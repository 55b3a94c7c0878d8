"""Sharded quantized EmbeddingCollection for inference (table-wise / row-wise / column-wise / table-row-wise placements over local
devices; reference torchrec/distributed/quant_embedding.py:597-1531)."""
from __future__ import annotations

from dataclasses import dataclass
from typing import Any, Dict, List, Optional, Sequence, Tuple, Type

import torch
from torch import nn

from ..quant.embedding_modules import EmbeddingCollection as QuantEmbeddingCollection
from ..sparse.jagged_tensor import JaggedTensor, KeyedJaggedTensor
from .embedding_types import BaseQuantEmbeddingSharder, quant_table_placement
from .engine import shards_of
from .types import LazyNoWait, NoWait, NullShardedModuleContext, ParameterSharding, ShardedModule, ShardingEnv, ShardingType


class ShardedQuantEmbeddingCollection(ShardedModule[List[KeyedJaggedTensor], List[torch.Tensor], Dict[str, JaggedTensor], NullShardedModuleContext]):
    """Sequence (unpooled) quantized lookups over local devices for every placement the planner can emit: a table's shards are
    rectangles (rank, row range, column range) and a feature's output is assembled from them -

        out_f[:, col_off : col_off + cols] += lookup(shard, ids_f - row_off)        (ids outside the shard's rows look up zeros)

    so table-wise is one full rectangle, column-wise fills disjoint column slices, row-wise adds row-disjoint partial results, and
    table-row-wise / grid are combinations. Per device the units are grouped by shard width into one quantized TBE launch each."""

    def __init__(self, module: QuantEmbeddingCollection, params: Dict[str, ParameterSharding], env: ShardingEnv, fused_params=None, device=None) -> None:
        super().__init__()
        from ..ops.quant_tbe import QuantTableBatchedEmbeddingBags, dequantize_rows

        self._device_type = "cuda" if torch.cuda.is_available() and (device is None or device.type == "cuda") else "cpu"
        tables = module.embedding_configs()
        self._tables = tables
        self._need_indices = module.need_indices()
        self._out_dtype = module.output_dtype()
        W = env.world_size
        self._feature_dim: Dict[str, int] = {f: t.embedding_dim for t in tables for f in t.feature_names}
        # (rank, shard width) -> units; a unit = (feature name, table idx, shard)
        groups: Dict[tuple, List[tuple]] = {}
        for ti, t in enumerate(tables):
            for sh in shards_of(ti, t, params[t.name]):
                for f in t.feature_names:
                    groups.setdefault((sh.rank, sh.cols), []).append((f, ti, sh))
        self._groups: List[tuple] = []
        self._group_units: List[Tuple[int, List[tuple]]] = []  # per group: (rank, its units)
        self._tbes = nn.ModuleList()
        for (r, cols), units in sorted(groups.items(), key=lambda kv: kv[0]):
            dev = torch.device("cuda", r) if self._device_type == "cuda" else torch.device("cpu")
            shard_keys: List[tuple] = []
            specs, locs, clfs = [], [], []
            for f, ti, sh in units:
                key = (ti, sh.row_off, sh.col_off)
                if key not in shard_keys:
                    shard_keys.append(key)
                    specs.append((f"{tables[ti].name}_{sh.row_off}_{sh.col_off}", sh.rows, sh.cols, tables[ti].data_type))
                    ps = params[tables[ti].name]
                    loc, clf = quant_table_placement(ps.compute_kernel, getattr(ps, "cache_params", None), fused_params)
                    locs.append(loc)
                    clfs.append(clf)
            fmap = [shard_keys.index((ti, sh.row_off, sh.col_off)) for _, ti, sh in units]
            tbe = QuantTableBatchedEmbeddingBags(specs, fmap, pooling_mode=2, output_dtype=self._out_dtype, device=dev, locations=locs,
                                                 cache_load_factor=clfs)
            for k, (ti, r0, c0) in enumerate(shard_keys):
                t = tables[ti]
                src = module.embeddings[t.name].weight
                rows_k, cols_k = specs[k][1], specs[k][2]
                if r0 == 0 and c0 == 0 and rows_k == t.num_embeddings and cols_k == t.embedding_dim:
                    dst = tbe.split_embedding_weights()[k]  # whole table: the quantized bytes as they are
                    dst.copy_(src.to(dst.device))
                    tbe.invalidate_cache(k)
                else:  # a rectangle of the table: re-quantized (row scales of column slices differ from the full row's)
                    full = dequantize_rows(src.to("cpu"), t.embedding_dim, t.data_type)
                    tbe.assign_from_float(k, full[r0 : r0 + rows_k, c0 : c0 + cols_k])
            self._tbes.append(tbe)
            row_offs = torch.tensor([sh.row_off for _, _, sh in units], dtype=torch.int64)
            self._groups.append((dev, [f for f, _, _ in units], [sh.col_off for _, _, sh in units], cols, row_offs))
            self._group_units.append((r, units))

    class _Ctx:
        """The batch's features travel from input_dist to output_dist (lengths / ids of the result are the caller's)."""

        features: Optional[KeyedJaggedTensor] = None

        def record_stream(self, stream) -> None:
            pass

    def create_context(self):
        return ShardedQuantEmbeddingCollection._Ctx()

    def input_dist(self, ctx, features: KeyedJaggedTensor):
        keys = features.keys()
        out = []
        for dev, feats, _, _, row_offs in self._groups:
            sub = features.permute([keys.index(f) for f in feats])  # (features repeat once per shard they have on this device)
            ro = row_offs.to(sub.values().device)
            if bool((row_offs != 0).any()):
                lpk = torch.tensor(sub.length_per_key(), dtype=torch.int64, device=ro.device)
                local = sub.values() - torch.repeat_interleave(ro, lpk, output_size=sub.values().numel()).to(sub.values().dtype)
                sub = KeyedJaggedTensor(keys=sub.keys(), values=local, lengths=sub.lengths(), stride=sub.stride())
            out.append(sub.to(dev, non_blocking=True))
        ctx.features = features
        return NoWait(NoWait(out))

    def compute(self, ctx, dist_input):
        return [(tbe(k.values(), k.offsets(), None, batch_size=k.stride()), k) for tbe, k in zip(self._tbes, dist_input)]

    def output_dist(self, ctx, output):
        dev0 = torch.device("cuda", 0) if self._device_type == "cuda" else torch.device("cpu")
        features: KeyedJaggedTensor = ctx.features
        keys = features.keys()
        lpk = features.length_per_key()
        vals = torch.split(features.values().to(dev0), lpk)
        lengths = features.lengths().to(dev0).view(len(keys), -1)
        acc: Dict[str, torch.Tensor] = {}
        for (emb, kjt), (_, feats, col_offs, cols, _) in zip(output, self._groups):
            parts = torch.split(emb.to(dev0), kjt.length_per_key(), dim=0)
            for f, c0, part in zip(feats, col_offs, parts):
                D = self._feature_dim[f]
                if cols == D and f not in acc:
                    acc[f] = part.clone() if part.device == emb.device else part  # full-width shard: no zero-filled buffer needed
                    continue
                if f not in acc:
                    acc[f] = torch.zeros(part.shape[0], D, dtype=part.dtype, device=dev0)
                acc[f][:, c0 : c0 + cols] += part
        res: Dict[str, JaggedTensor] = {}
        for i, k in enumerate(keys):
            if k in acc:
                res[k] = JaggedTensor(values=acc[k], lengths=lengths[i], weights=vals[i] if self._need_indices else None)
        return LazyNoWait(res)

    # ---- fused single-process multi-GPU path (CUDA) ---------------------------------------------------------------------------------
    def _plane(self) -> "_SequenceInferencePlane":
        pl = self.__dict__.get("_infer_plane")
        if pl is None:
            pl = self.__dict__["_infer_plane"] = _SequenceInferencePlane(self)
        return pl

    def forward_fused(self, features: KeyedJaggedTensor) -> Dict[str, JaggedTensor]:
        """``kjt_route`` on the input device routes every id exactly once per column slice of its feature, with its position inside the
        feature's values, straight into the memory of the device holding the shard; every group's quantized sequence lookup then stores
        its rows into one flat output on the first device at their final place (feature block, row, columns). Returns the same
        ``JaggedTensor`` per feature as the decomposed ``input_dist`` / ``compute`` / ``output_dist``."""
        return self._plane().run(features)

    def forward(self, features: KeyedJaggedTensor):
        if self._device_type == "cuda" and features.values().is_cuda and not features.variable_stride_per_key():
            return self.forward_fused(features)
        ctx = self.create_context()
        return self.output_dist(ctx, self.compute(ctx, self.input_dist(ctx, features).wait().wait())).wait()


INT64_MAX = (1 << 63) - 1


@dataclass
class SequenceUnits:
    """Static route / lookup table of the fused sequence path. A unit is (feature, shard); units are in device-major order and the units
    of one (rank, shard width) group of the module are contiguous, in the group's order (the group's TBE features)."""

    feature: List[str]
    rank: List[int]
    slot: List[int]        # index of the unit among its device's units
    row_lo: List[int]      # ids in [row_lo, row_hi) are the unit's (rebased by row_lo); whole-table units: 0, INT64_MAX
    row_hi: List[int]
    edge: List[int]        # bit 0: also takes the ids below 0 (shard starts at row 0), bit 1: the ids past the table (shard ends there)
    col: List[int]         # column offset of the shard inside its feature
    dim: List[int]         # the feature's full width
    group_slice: List[Tuple[int, int]]  # per module group: its units [u0, u1)
    dest_ustart: List[int]  # per device: its first unit; one more entry = number of units
    # one unit per distinct (feature, column offset) of a group / of a device: units sharing both cover the same column with disjoint
    # rows, so each id reaches at most one of them and these units' id counts bound the ids the group / device receives
    group_reps: List[List[int]]
    dev_reps: List[List[int]]


def sequence_units(group_units: Sequence[Tuple[int, Sequence[tuple]]], table_rows: Dict[int, int], feature_dim: Dict[str, int]) -> SequenceUnits:
    """The unit table of a sharded sequence collection: ``group_units`` = per group (rank, [(feature, table idx, shard)]), groups sorted
    by (rank, width). The shards of a table must tile it (every row and column in exactly one shard). An id goes to every shard whose
    rows hold it; shards starting at row 0 also take the ids below 0 and shards ending at the last row the ids past the table. So every
    (id, column) of a feature is routed to exactly one shard (the lookup stores zeros for an id outside the table), for any rectangle
    layout, including row shards cut into different column slices."""
    rects: Dict[int, set] = {}
    for _, units in group_units:
        for f, ti, sh in units:
            rects.setdefault(ti, set()).add((sh.row_off, sh.rows, sh.col_off, sh.cols, feature_dim[f]))
    for ti, rs in rects.items():
        R, D = table_rows[ti], next(iter(rs))[4]
        ok = all(r0 >= 0 and n > 0 and r0 + n <= R and c0 >= 0 and c > 0 and c0 + c <= D for r0, n, c0, c, _ in rs)
        ok = ok and sum(n * c for _, n, _, c, _ in rs) == R * D
        rl = sorted(rs)
        ok = ok and not any(a[0] < b[0] + b[1] and b[0] < a[0] + a[1] and a[2] < b[2] + b[3] and b[2] < a[2] + a[3]
                            for i, a in enumerate(rl) for b in rl[i + 1 :])
        if not ok:
            raise ValueError(f"table {ti}: its shards {rl} do not tile the {R} x {D} table")
    t = SequenceUnits([], [], [], [], [], [], [], [], [], [], [], [])
    n_dev = max((r for r, _ in group_units), default=-1) + 1
    per_dev = [0] * n_dev
    dev_keys: List[set] = [set() for _ in range(n_dev)]
    t.dev_reps = [[] for _ in range(n_dev)]
    for r, units in group_units:
        u0 = len(t.feature)
        keys: set = set()
        reps: List[int] = []
        for f, ti, sh in units:
            u = len(t.feature)
            R = table_rows[ti]
            t.feature.append(f)
            t.rank.append(r)
            t.slot.append(per_dev[r])
            per_dev[r] += 1
            if sh.row_off == 0 and sh.rows == R:
                t.row_lo.append(0)
                t.row_hi.append(INT64_MAX)
                t.edge.append(0)
            else:
                t.row_lo.append(sh.row_off)
                t.row_hi.append(sh.row_off + sh.rows)
                t.edge.append((1 if sh.row_off == 0 else 0) | (2 if sh.row_off + sh.rows == R else 0))
            t.col.append(sh.col_off)
            t.dim.append(feature_dim[f])
            if (f, sh.col_off) not in keys:
                keys.add((f, sh.col_off))
                reps.append(u)
            if (f, sh.col_off) not in dev_keys[r]:
                dev_keys[r].add((f, sh.col_off))
                t.dev_reps[r].append(u)
        t.group_slice.append((u0, len(t.feature)))
        t.group_reps.append(reps)
    t.dest_ustart = [0]
    for n in per_dev:
        t.dest_ustart.append(t.dest_ustart[-1] + n)
    assert t.rank == sorted(t.rank), "groups must be in device order"
    return t


def feature_bases(keys: Sequence[str], length_per_key: Sequence[int], feature_dim: Dict[str, int]) -> Tuple[Dict[str, int], int]:
    """Element offset of every served feature's [n_f, D_f] block in the flat sequence output (features in input key order), and the
    output's size."""
    bases, o = {}, 0
    for k, n in zip(keys, length_per_key):
        if k in feature_dim:
            bases[k] = o
            o += n * feature_dim[k]
    return bases, o


class _SequenceInferencePlane:
    """Static unit table + growable route buffers of the fused inference path of one sharded quantized sequence collection (one
    process, W devices)."""

    def __init__(self, m: ShardedQuantEmbeddingCollection) -> None:
        from ..ops import _lib

        self.m = m
        t = self.t = sequence_units(m._group_units, {ti: tc.num_embeddings for ti, tc in enumerate(m._tables)}, m._feature_dim)
        for u in range(len(t.feature)):
            if t.dim[u] % 4 or t.col[u] % 4:
                raise ValueError(f"feature {t.feature[u]}: the sequence lookup stores 4-element vectors, its width ({t.dim[u]}) and shard "
                                 f"column offsets ({t.col[u]}) must be multiples of 4")
        self.U = len(t.feature)
        self.W = W = len(t.dest_ustart) - 1
        self.devs = [torch.device("cuda", r) for r in range(W)]
        self.dev0 = self.devs[0]
        L = _lib.lib()
        used = sorted(set(t.rank))
        for a in used:
            for b in used:
                if a != b:
                    _lib.check(L.trb_enable_peer_access(a, b), f"trb_enable_peer_access({a},{b})")
        mk32 = lambda x, d: torch.tensor(x, dtype=torch.int32, device=d)
        self.u_lo = torch.tensor(t.row_lo, dtype=torch.int64, device=self.dev0)
        self.u_hi = torch.tensor(t.row_hi, dtype=torch.int64, device=self.dev0)
        self.u_dest = mk32(t.rank, self.dev0)
        self.u_slot = mk32(t.slot, self.dev0)
        self.u_edge = mk32(t.edge, self.dev0)
        self.dest_ustart = mk32(t.dest_ustart, self.dev0)
        self.overflow = torch.zeros(1, dtype=torch.int32, device=self.dev0)
        us = t.dest_ustart
        self.dev_col = [mk32(t.col[us[r] : us[r + 1]], self.devs[r]) for r in range(W)]
        self.dev_ostride = [mk32(t.dim[us[r] : us[r + 1]], self.devs[r]) for r in range(W)]
        self.streams = [torch.cuda.Stream(d) for d in self.devs]
        # per-unit feature bases of the current batch, rewritten (pinned non-blocking copy) on the stream of the device's lookups
        self.dev_obase = [torch.empty(us[r + 1] - us[r], dtype=torch.int64, device=d) for r, d in enumerate(self.devs)]
        for r in range(1, W):  # the lookups on streams[r] come after everything device r was asked to do so far (weights, these buffers)
            self.streams[r].wait_stream(torch.cuda.current_stream(self.devs[r]))
        self._key_cache: Dict[Tuple[str, ...], Tuple[torch.Tensor, List[int]]] = {}
        self._bases_key: Optional[tuple] = None
        self._last: Optional[Tuple[int, torch.cuda.Event]] = None  # (stream, end of the last eager call on it)
        self.B = -1
        self.cap = -1
        self.idx_dtype: Optional[torch.dtype] = None

    def _stream(self, r: int, main: torch.cuda.Stream) -> torch.cuda.Stream:
        """The stream that runs device r's lookups: the caller's stream on the first device, the plane's own stream elsewhere."""
        return main if r == 0 else self.streams[r]

    def _ensure(self, B: int, cap: int, idx_dtype: torch.dtype, main: torch.cuda.Stream) -> None:
        import ctypes

        from ..ops import _lib

        if B <= self.B and cap <= self.cap and idx_dtype == self.idx_dtype:
            return  # buffers are sized for the largest batch seen so far (serving batches vary): smaller ones use their front part
        self.idx_dtype = idx_dtype
        B = self.B = max(B, self.B)
        self.cap = max(cap, int(self.cap * 1.5) if self.cap > 0 else cap)
        us = self.t.dest_ustart
        self.off_bufs, self.val_bufs, self.pos_bufs = [], [], []
        for r, d in enumerate(self.devs):
            # allocated on the stream of device r's lookups: the memory is not handed to them before that stream's earlier work on it
            # is done, and the route (first device) runs after the previous call's lookups, which the caller's stream waited for.
            # The route stores every offset the lookups read, so nothing is initialised here.
            with torch.cuda.device(d), torch.cuda.stream(self._stream(r, main)):
                self.off_bufs.append(torch.empty((us[r + 1] - us[r]) * B + 1, dtype=torch.int32, device=d))
                self.val_bufs.append(torch.empty(self.cap, dtype=idx_dtype, device=d))
                self.pos_bufs.append(torch.empty(self.cap, dtype=torch.int32, device=d))
        L = _lib.lib()
        L.trb_kjt_route_workspace_bytes.restype = ctypes.c_int64
        self.route_ws = torch.empty(int(L.trb_kjt_route_workspace_bytes(self.U, B)), dtype=torch.uint8, device=self.dev0)

    def _bases(self, keys: Tuple[str, ...], lpk: List[int], main: torch.cuda.Stream) -> Tuple[Dict[str, int], int]:
        """Feature bases of the batch. The per-unit bases reach every device in one pinned non-blocking copy each, issued on the stream
        of that device's lookups (so they land before the lookups read them and after the previous lookups did), and are kept while the
        batch's lengths per key stay the same (so a CUDA graph captured after an eager call of the same batch copies nothing)."""
        m, t = self.m, self.t
        bases, total = feature_bases(keys, lpk, m._feature_dim)
        key = (keys, tuple(lpk))
        if key != self._bases_key:
            host = torch.tensor([bases[f] for f in t.feature], dtype=torch.int64).pin_memory()
            us = t.dest_ustart
            for r, d in enumerate(self.devs):
                if us[r + 1] > us[r]:
                    with torch.cuda.device(d), torch.cuda.stream(self._stream(r, main)):
                        self.dev_obase[r].copy_(host[us[r] : us[r + 1]], non_blocking=True)
            self._bases_key = key
        return bases, total

    def run(self, features: KeyedJaggedTensor) -> Dict[str, JaggedTensor]:
        import ctypes

        from ..ops import _lib

        m, t = self.m, self.t
        L = _lib.lib()
        if features.values().device != self.dev0:
            features = features.to(self.dev0, non_blocking=True)
        B = features.stride()
        keys = tuple(features.keys())
        values = features.values()
        lpk = features.length_per_key()
        hit = self._key_cache.get(keys)
        if hit is None:
            pos = {k: i for i, k in enumerate(keys)}
            kidx = [pos[f] for f in t.feature]
            hit = self._key_cache[keys] = (torch.tensor(kidx, dtype=torch.int32, device=self.dev0), kidx)
        u_key, kidx = hit
        n_of_unit = [lpk[k] for k in kidx]  # routed ids of a unit <= its feature's ids
        main = torch.cuda.current_stream(self.dev0)
        capturing = torch.cuda.is_current_stream_capturing()
        if self._last is not None and self._last[0] != main.cuda_stream and not capturing:
            # the buffers were last used from another stream: start after that call (a graph capture starts after a synchronize)
            main.wait_event(self._last[1])
        cap = max(32, max(sum(n_of_unit[u] for u in reps) for reps in t.dev_reps))
        self._ensure(B, cap, values.dtype, main)
        bases, total = self._bases(keys, lpk, main)
        out = torch.empty(total, dtype=m._out_dtype, device=self.dev0)
        offsets = features.offsets()
        code = L.trb_kjt_route_pos(
            _lib.ptr(offsets), int(offsets.dtype == torch.int64), _lib.ptr(values), int(values.dtype == torch.int64), ctypes.c_int64(values.numel()), B,
            _lib.ptr(u_key), _lib.ptr(self.u_lo), _lib.ptr(self.u_hi), _lib.ptr(self.u_dest), _lib.ptr(self.u_slot), _lib.ptr(self.dest_ustart),
            _lib.ptr(self.u_edge), self.U, self.W, _lib.ptr_array([b.data_ptr() for b in self.off_bufs]), 0,
            _lib.ptr_array([b.data_ptr() for b in self.val_bufs]), int(values.dtype == torch.int64), _lib.ptr_array([b.data_ptr() for b in self.pos_bufs]),
            ctypes.c_int64(self.cap), _lib.ptr(self.overflow), _lib.ptr(self.route_ws), ctypes.c_int64(self.route_ws.numel()),
            int(max(1, values.numel() // max(1, len(keys) * B))), _lib.stream_ptr(self.dev0))
        _lib.check(code, "trb_kjt_route_pos")
        ready = torch.cuda.Event()
        ready.record(main)
        done = []
        for r in range(self.W):
            groups = [gi for gi, (u0, u1) in enumerate(t.group_slice) if u1 > u0 and t.rank[u0] == r]
            if not groups:
                continue
            st = self.streams[r] if r != 0 else main
            with torch.cuda.device(self.devs[r]):
                if r != 0:
                    st.wait_event(ready)
                with torch.cuda.stream(st):
                    for gi in groups:  # one launch per (rank, width) group over its slice of the device's units
                        u0, u1 = t.group_slice[gi]
                        s0, s1 = t.slot[u0], t.slot[u0] + (u1 - u0)
                        m._tbes[gi].forward_scatter(self.val_bufs[r], self.off_bufs[r][s0 * B : s1 * B + 1], self.pos_bufs[r], B, out,
                                                    self.dev_obase[r][s0:s1], self.dev_ostride[r][s0:s1], self.dev_col[r][s0:s1],
                                                    sum(n_of_unit[u] for u in t.group_reps[gi]))
                    if r != 0:
                        ev = torch.cuda.Event()
                        ev.record(st)
                        done.append(ev)
        for ev in done:
            main.wait_event(ev)
        if not capturing:
            ev = torch.cuda.Event()
            ev.record(main)
            self._last = (main.cuda_stream, ev)
        lengths = features.lengths().view(len(keys), -1)
        vals = torch.split(values, lpk) if m._need_indices else None
        res: Dict[str, JaggedTensor] = {}
        for i, k in enumerate(keys):
            if k in bases:
                D = m._feature_dim[k]
                res[k] = JaggedTensor(values=out[bases[k] : bases[k] + lpk[i] * D].view(lpk[i], D), lengths=lengths[i],
                                      weights=vals[i] if vals is not None else None)
        return res


class QuantEmbeddingCollectionSharder(BaseQuantEmbeddingSharder[QuantEmbeddingCollection]):
    def shard(self, module, params, env, device=None, module_fqn=None):
        return ShardedQuantEmbeddingCollection(module, params, env, self.fused_params, device)

    def shardable_parameters(self, module: QuantEmbeddingCollection) -> Dict[str, nn.Parameter]:
        return {t.name: nn.Parameter(torch.empty(t.num_embeddings, t.embedding_dim, device="meta"), requires_grad=False) for t in module.embedding_configs()}

    def sharding_types(self, compute_device_type: str) -> List[str]:
        return [ShardingType.TABLE_WISE.value, ShardingType.ROW_WISE.value, ShardingType.COLUMN_WISE.value, ShardingType.TABLE_ROW_WISE.value,
                ShardingType.TABLE_COLUMN_WISE.value]

    @property
    def module_type(self) -> Type[QuantEmbeddingCollection]:
        return QuantEmbeddingCollection


class ShardedQuantManagedCollisionEmbeddingCollection(nn.Module):
    """Quantized sequence tables sharded like a plain quantized collection; the managed-collision collection is replicated (read-only
    when serving) and remaps the raw ids of the full batch before the lookup. Returns ``(embeddings, remapped features)``."""

    def __init__(self, module, params, env, fused_params=None, device=None) -> None:
        super().__init__()
        self._sharded = ShardedQuantEmbeddingCollection(module, params, env, fused_params, device)
        self._managed_collision_collection = module._managed_collision_collection
        self._configs = list(module.embedding_configs())

    def embedding_configs(self):
        return self._configs

    def forward(self, features: KeyedJaggedTensor):
        features = self._managed_collision_collection(features)
        return self._sharded(features), features


class QuantManagedCollisionEmbeddingCollectionSharder(QuantEmbeddingCollectionSharder):
    def shard(self, module, params, env, device=None, module_fqn=None):
        return ShardedQuantManagedCollisionEmbeddingCollection(module, params, env, self.fused_params, device)

    @property
    def module_type(self):
        from ..quant.embedding_modules import QuantManagedCollisionEmbeddingCollection

        return QuantManagedCollisionEmbeddingCollection
