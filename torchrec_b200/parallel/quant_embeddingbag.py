"""Sharded quantized (inference) embedding collections — single process driving several GPUs
(reference torchrec/distributed/quant_embeddingbag.py:171, quant_embedding.py:597, sharding/tw_sharding.py:466-584).

Inference has no process group (``ShardingEnv.from_local``): the module owns one quantized kernel per device.
Input dist = split the KJT per device + P2P copies (``KJTOneToAll``); output dist = NVLink copies back to the
first device, concatenated (TW/CW) or summed (RW)."""
from __future__ import annotations

from typing import Any, Dict, List, Optional, Tuple, Type

import torch
from torch import nn

from ..modules.embedding_configs import EmbeddingBagConfig, EmbeddingConfig, PoolingType
from ..modules.embedding_modules import get_embedding_names_by_table
from ..ops.quant_tbe import QuantTableBatchedEmbeddingBags
from ..quant.embedding_modules import EmbeddingBagCollection as QuantEmbeddingBagCollection
from ..quant.embedding_modules import EmbeddingCollection as QuantEmbeddingCollection
from ..types import DataType
from ..sparse.jagged_tensor import JaggedTensor, KeyedJaggedTensor, KeyedTensor
from .embedding_types import BaseQuantEmbeddingSharder, quant_table_placement
from .engine import shards_of
from .types import NullShardedModuleContext, ParameterSharding, ShardedModule, ShardingEnv, ShardingType, LazyNoWait, NoWait


def _dev(device_type: str, rank: int) -> torch.device:
    return torch.device("cpu") if device_type != "cuda" else torch.device("cuda", rank)


class ShardedQuantEmbeddingBagCollection(ShardedModule[List[KeyedJaggedTensor], List[torch.Tensor], KeyedTensor, NullShardedModuleContext]):
    """TW / CW / RW sharded quantized EBC for inference."""

    def __init__(self, module: QuantEmbeddingBagCollection, table_name_to_parameter_sharding: Dict[str, ParameterSharding], env: ShardingEnv,
                 fused_params: Optional[Dict[str, Any]] = None, device: Optional[torch.device] = None) -> None:
        super().__init__()
        self._env = env
        W = env.world_size
        self._device_type = "cuda" if (device is not None and device.type == "cuda") or (device is None and torch.cuda.is_available()) else "cpu"
        tables = module.embedding_bag_configs()
        self._tables = tables
        self._is_weighted = module.is_weighted()
        self._output_dtype = module.output_dtype()
        self._embedding_names = [n for ns in get_embedding_names_by_table(tables) for n in ns]
        self._dims = [t.embedding_dim for t in tables for _ in t.feature_names]
        self._feature_names = [f for t in tables for f in t.feature_names]
        feat_table = [ti for ti, t in enumerate(tables) for _ in t.feature_names]
        out_base = [0]
        for d in self._dims:
            out_base.append(out_base[-1] + d)
        self._total_cols = out_base[-1]
        src_weights = {t.name: module.embedding_bags[t.name].weight for t in tables}
        # per rank: list of (table idx, shard, feature idx)
        per_rank: List[List[Tuple[int, Any, int]]] = [[] for _ in range(W)]
        self._row_sharded_feature: Dict[int, List[Tuple[int, int, int]]] = {}
        for ti, t in enumerate(tables):
            ps = table_name_to_parameter_sharding[t.name]
            for s in shards_of(ti, t, ps):
                if t.data_type == DataType.FP8 and s.cols % 32 != 0:
                    raise ValueError(f"table {t.name}: block-scaled fp8 rows carry one scale per 32 elements, column shards must be multiples of 32 wide "
                                     f"(got {s.cols} of {t.embedding_dim}); use fewer column shards or another placement")
                for fi in [i for i, x in enumerate(feat_table) if x == ti]:
                    per_rank[s.rank].append((ti, s, fi))
        # inside a device, whole-table / column-shard units first, row-sharded units (summed at the destination) after them
        n_row_shards = {ti: len({(s.row_off, s.rows) for s in shards_of(ti, t, table_name_to_parameter_sharding[t.name])}) for ti, t in enumerate(tables)}
        for units in per_rank:
            units.sort(key=lambda u: n_row_shards[u[0]] > 1)
        self._per_rank = per_rank
        self._tbes = nn.ModuleList()
        self._rank_meta: List[List[Tuple[int, Any, int]]] = []
        for r in range(W):
            units = per_rank[r]
            dev = _dev(self._device_type, r)
            if not units:
                self._tbes.append(nn.Identity())
                self._rank_meta.append([])
                continue
            shard_keys: List[Tuple[int, int, int]] = []
            specs, locs, clfs = [], [], []
            for ti, s, fi in units:
                key = (ti, s.row_off, s.col_off)
                if key not in shard_keys:
                    shard_keys.append(key)
                    specs.append((f"{tables[ti].name}_{s.row_off}_{s.col_off}", s.rows, s.cols, tables[ti].data_type))
                    ps = table_name_to_parameter_sharding[tables[ti].name]
                    loc, clf = quant_table_placement(ps.compute_kernel, getattr(ps, "cache_params", None), fused_params)
                    locs.append(loc)
                    clfs.append(clf)
            fmap = [shard_keys.index((ti, s.row_off, s.col_off)) for ti, s, fi in units]
            pool = {tables[ti].pooling for ti, _, _ in units}
            tbe = QuantTableBatchedEmbeddingBags(specs, fmap, pooling_mode=0, output_dtype=self._output_dtype, device=dev, locations=locs,
                                                 cache_load_factor=clfs)
            # fill: dequantise the source slice and re-quantise the shard (column slices change the row scale)
            from ..ops.quant_tbe import dequantize_rows

            done = set()
            for (ti, s, fi), k in zip(units, fmap):
                if k in done:
                    continue
                done.add(k)
                full = dequantize_rows(src_weights[tables[ti].name].to("cpu"), tables[ti].embedding_dim, tables[ti].data_type)
                tbe.assign_from_float(k, full[s.row_off : s.row_off + s.rows, s.col_off : s.col_off + s.cols])
            self._tbes.append(tbe)
            self._rank_meta.append(units)
        self._mean_features = [fi for fi, ti in enumerate(feat_table) if tables[ti].pooling == PoolingType.MEAN]
        self._out_base = out_base

    def create_context(self) -> NullShardedModuleContext:
        return NullShardedModuleContext()

    # ---- fused single-process multi-GPU path (CUDA) ---------------------------------------------------------------------------------
    def _plane(self) -> "_InferencePlane":
        pl = self.__dict__.get("_infer_plane")
        if pl is None:
            pl = self.__dict__["_infer_plane"] = _InferencePlane(self)
        return pl

    def forward_fused(self, features: KeyedJaggedTensor) -> KeyedTensor:
        """One device-side pass per phase, no host round trip: ``kjt_route`` on the input device buckets / rebases / permutes the ids and
        stores every device's share straight into ITS memory (KJTOneToAll + bucketize of the reference in one kernel, peer stores);
        every device's quantized lookup kernel then stores its pooled rows straight into the output tensor on the first device at their
        final columns (EmbeddingsAllToOne / MergePooledEmbeddings as peer stores); row-sharded tables go through per-device staging
        slabs summed by one small kernel."""
        return self._plane().run(features)

    def input_dist(self, ctx, features: KeyedJaggedTensor):
        """Per device: the features of its units with ids filtered / rebased to the shard's row range."""
        pos = {k: i for i, k in enumerate(features.keys())}
        B = features.stride()
        out: List[Optional[KeyedJaggedTensor]] = []
        jt = features.to_dict()
        for r, units in enumerate(self._rank_meta):
            if not units:
                out.append(None)
                continue
            dev = _dev(self._device_type, r)
            vals, lens, ws = [], [], []
            for ti, s, fi in units:
                f = jt[self._feature_names[fi]]
                v, l = f.values(), f.lengths()
                w = f.weights_or_none()
                if s.rows != self._tables[ti].num_embeddings:
                    keep = (v >= s.row_off) & (v < s.row_off + s.rows)
                    seg = torch.repeat_interleave(torch.arange(B, device=v.device), l.long())
                    l = torch.zeros(B, dtype=l.dtype, device=v.device).index_add_(0, seg[keep], torch.ones(int(keep.sum()), dtype=l.dtype, device=v.device))
                    v = v[keep] - s.row_off
                    w = w[keep] if w is not None else None
                vals.append(v)
                lens.append(l)
                if w is not None:
                    ws.append(w)
            kjt = KeyedJaggedTensor(keys=[self._feature_names[fi] for _, _, fi in units], values=torch.cat(vals), lengths=torch.cat(lens),
                                    weights=torch.cat(ws) if ws else None, stride=B)
            out.append(kjt.to(dev, non_blocking=True))
        self._divisor = None
        if self._mean_features:
            lengths = features.lengths().view(len(features.keys()), B)
            self._divisor = {fi: lengths[pos[self._feature_names[fi]]].clamp(min=1).float() for fi in self._mean_features}
        return NoWait(NoWait(out))

    def compute(self, ctx, dist_input) -> List[Optional[torch.Tensor]]:
        outs = []
        for r, kjt in enumerate(dist_input):
            if kjt is None:
                outs.append(None)
                continue
            psw = kjt.weights_or_none() if self._is_weighted else None
            outs.append(self._tbes[r](kjt.values(), kjt.offsets(), psw, batch_size=kjt.stride()))
        return outs

    def output_dist(self, ctx, output):
        dev0 = _dev(self._device_type, 0)
        B = next(o.shape[0] for o in output if o is not None)
        res = torch.zeros(B, self._total_cols, dtype=self._output_dtype, device=dev0)
        for r, o in enumerate(output):
            if o is None:
                continue
            o = o.to(dev0, non_blocking=True)
            c = 0
            for ti, s, fi in self._rank_meta[r]:
                base = self._out_base[fi] + s.col_off
                res[:, base : base + s.cols] += o[:, c : c + s.cols]
                c += s.cols
        if self._divisor:
            for fi, d in self._divisor.items():
                res[:, self._out_base[fi] : self._out_base[fi + 1]] /= d.to(dev0).unsqueeze(1)
        return LazyNoWait(KeyedTensor(keys=self._embedding_names, length_per_key=self._dims, values=res))

    def forward(self, features: KeyedJaggedTensor):
        import os

        if self._device_type == "cuda" and features.values().is_cuda and not features.variable_stride_per_key() and os.environ.get("TRB_QUANT_FUSED", "1") != "0":
            return self.forward_fused(features)
        ctx = self.create_context()
        return self.output_dist(ctx, self.compute(ctx, self.input_dist(ctx, features).wait().wait())).wait()

    @property
    def unsharded_module_type(self):
        return QuantEmbeddingBagCollection


class _InferencePlane:
    """Static description + growable buffers of the fused inference path of one sharded quantized collection (one process, W devices)."""

    def __init__(self, m: ShardedQuantEmbeddingBagCollection) -> None:
        import ctypes

        from ..ops import _lib

        self.m = m
        self.W = W = len(m._rank_meta)
        self.devs = [_dev("cuda", r) for r in range(W)]
        self.dev0 = self.devs[0]
        L = _lib.lib()
        for a in range(W):
            for b in range(W):
                if a != b and m._rank_meta[a] is not None:
                    _lib.check(L.trb_enable_peer_access(a, b), f"trb_enable_peer_access({a},{b})")
        # lookup units in device-major order
        units = [(r, ti, s, fi) for r in range(W) for (ti, s, fi) in m._rank_meta[r]]
        self.U = len(units)
        self.units_per_dev = [len(m._rank_meta[r]) for r in range(W)]
        ustart = [0]
        for n in self.units_per_dev:
            ustart.append(ustart[-1] + n)
        self.ustart = ustart
        INT64_MAX = (1 << 63) - 1
        row_sharded = {ti: len({(s.row_off, s.rows) for _, tj, s, _ in units if tj == ti}) > 1 for _, ti, _, _ in units}
        mk32 = lambda x: torch.tensor(x, dtype=torch.int32, device=self.dev0)
        mk64 = lambda x: torch.tensor(x, dtype=torch.int64, device=self.dev0)
        self.feature_of_unit = [fi for _, _, _, fi in units]
        self.u_lo = mk64([s.row_off if row_sharded[ti] else 0 for _, ti, s, _ in units])
        self.u_hi = mk64([s.row_off + s.rows if row_sharded[ti] else INT64_MAX for _, ti, s, _ in units])
        self.u_dest = mk32([r for r, _, _, _ in units])
        self.u_slot = mk32([i - ustart[r] for i, (r, _, _, _) in enumerate(units)])
        self.u_cslice = mk32([0] * len(units))
        self.dest_ustart = mk32(ustart)
        self.overflow = torch.zeros(1, dtype=torch.int32, device=self.dev0)
        # output columns: direct units write their final columns of the result; row-sharded units write compact staging columns
        self.staged_cols: Dict[Tuple[int, int], int] = {}
        sc = 0
        for _, ti, s, fi in units:
            if row_sharded[ti] and (fi, s.col_off) not in self.staged_cols:
                self.staged_cols[(fi, s.col_off)] = sc
                sc += s.cols
        self.staged_width = (sc + 3) // 4 * 4
        self.dev_direct: List[Optional[torch.Tensor]] = []   # per device: feat_col override (int32) for the lookup kernel
        self.dev_is_staged: List[List[bool]] = []
        for r in range(W):
            cols, staged = [], []
            for ti, s, fi in m._rank_meta[r]:
                if row_sharded[ti]:
                    cols.append(self.staged_cols[(fi, s.col_off)])
                    staged.append(True)
                else:
                    cols.append(m._out_base[fi] + s.col_off)
                    staged.append(False)
            self.dev_direct.append(torch.tensor(cols, dtype=torch.int32, device=self.devs[r]) if cols else None)
            self.dev_is_staged.append(staged)
        if self.staged_cols:
            mask, dst = [0] * self.staged_width, [0] * self.staged_width
            for r, ti, s, fi in units:
                if row_sharded[ti]:
                    for c in range(s.cols):
                        mask[self.staged_cols[(fi, s.col_off)] + c] |= 1 << r
                        dst[self.staged_cols[(fi, s.col_off)] + c] = m._out_base[fi] + s.col_off + c
            self.stage_mask = torch.tensor(mask, dtype=torch.int64, device=self.dev0).to(torch.int32)
            self.stage_dst = mk32(dst)
        self.B = -1
        self.cap = -1
        self.streams = [torch.cuda.Stream(d) for d in self.devs]
        self._key_pos_cache: Dict[Tuple[str, ...], torch.Tensor] = {}

    def _ensure(self, B: int, n_ids: int, idx_dtype: torch.dtype, weighted: bool) -> None:
        from ..ops import _lib
        import ctypes

        need_cap = max(32, n_ids * max(1, max((len([1 for f in self.feature_of_unit if f == g]) for g in set(self.feature_of_unit)), default=1)))
        if B <= self.B and need_cap <= self.cap and idx_dtype == getattr(self, "idx_dtype", None) and weighted == getattr(self, "weighted", None):
            return  # buffers are sized for the largest batch seen so far (serving batches vary): smaller ones use their front part
        self.idx_dtype, self.weighted = idx_dtype, weighted
        B = self.B = max(B, self.B)
        self.cap = max(need_cap, int(self.cap * 1.5) if self.cap > 0 else need_cap)
        U_max = max(self.units_per_dev)
        self.off_bufs = [torch.zeros(U_max * B + 1, dtype=torch.int32, device=d) for d in self.devs]
        self.val_bufs = [torch.empty(self.cap, dtype=idx_dtype, device=d) for d in self.devs]
        self.wgt_bufs = [torch.empty(self.cap, dtype=torch.float32, device=d) for d in self.devs] if weighted else None
        L = _lib.lib()
        L.trb_kjt_route_workspace_bytes.restype = ctypes.c_int64
        self.route_ws = torch.empty(int(L.trb_kjt_route_workspace_bytes(self.U, B)), dtype=torch.uint8, device=self.dev0)
        self.staging = torch.zeros(self.W, B, self.staged_width, dtype=self.m._output_dtype, device=self.dev0) if self.staged_cols else None

    def run(self, features: KeyedJaggedTensor) -> KeyedTensor:
        import ctypes

        from ..ops import _lib

        m = self.m
        L = _lib.lib()
        if features.values().device != self.dev0:
            features = features.to(self.dev0, non_blocking=True)
        B = features.stride()
        values = features.values()
        weights = features.weights_or_none() if m._is_weighted else None
        self._ensure(B, values.numel(), values.dtype, weights is not None)
        keys = tuple(features.keys())
        u_key = self._key_pos_cache.get(keys)
        if u_key is None:
            pos = {k: i for i, k in enumerate(keys)}
            u_key = self._key_pos_cache[keys] = torch.tensor([pos[m._feature_names[fi]] for fi in self.feature_of_unit], dtype=torch.int32, device=self.dev0)
        offsets = features.offsets()
        main = torch.cuda.current_stream(self.dev0)
        n_bags = max(1, len(keys) * B)
        code = L.trb_kjt_route(
            _lib.ptr(offsets), int(offsets.dtype == torch.int64), _lib.ptr(values), int(values.dtype == torch.int64), _lib.ptr(weights), B, _lib.ptr(u_key),
            _lib.ptr(self.u_lo), _lib.ptr(self.u_hi), _lib.ptr(self.u_dest), _lib.ptr(self.u_slot), _lib.ptr(self.u_cslice), _lib.ptr(self.dest_ustart), self.U, self.W,
            _lib.ptr_array([t.data_ptr() for t in self.off_bufs]), 0, _lib.ptr_array([t.data_ptr() for t in self.val_bufs]), int(values.dtype == torch.int64),
            _lib.ptr_array([t.data_ptr() for t in self.wgt_bufs]) if weights is not None else ctypes.c_void_p(0), ctypes.c_int64(self.cap), ctypes.c_void_p(0), 1,
            _lib.ptr(self.overflow), _lib.ptr(self.route_ws), ctypes.c_int64(self.route_ws.numel()), int(max(1, values.numel() // n_bags)), _lib.stream_ptr(self.dev0))
        _lib.check(code, "trb_kjt_route")
        res = torch.zeros(B, m._total_cols, dtype=m._output_dtype, device=self.dev0) if (self.staged_cols or any(t is None for t in self.dev_direct)) else \
            torch.empty(B, m._total_cols, dtype=m._output_dtype, device=self.dev0)
        ready = torch.cuda.Event()
        ready.record(main)
        done = []
        esz = res.element_size()
        for r in range(self.W):
            tbe = m._tbes[r]
            if not m._rank_meta[r]:
                continue
            st = self.streams[r] if r != 0 else main
            with torch.cuda.device(self.devs[r]):
                if r != 0:
                    st.wait_event(ready)
                with torch.cuda.stream(st):
                    staged = self.dev_is_staged[r]
                    n_direct = staged.index(True) if True in staged else len(staged)
                    assert all(staged[n_direct:]), "row-sharded units follow whole-table units on a device"
                    F = len(staged)
                    psw = self.wgt_bufs[r] if weights is not None else None

                    def launch(f0: int, f1: int, out_ptr: int, out_stride: int) -> None:
                        if f1 <= f0:
                            return
                        if tbe._placed:  # host-resident tables (and their HBM row caches) next to HBM tables in the same launch
                            c = L.trb_qtbe_fwd_placed(
                                ctypes.c_void_p(tbe.feat_base.data_ptr() + 8 * f0), ctypes.c_void_p(tbe.feat_ctab.data_ptr() + 4 * f0),
                                _lib.ptr(tbe.cache_tabs), _lib.ptr(tbe.no_slot), ctypes.c_void_p(tbe.feat_rows.data_ptr() + 8 * f0),
                                ctypes.c_void_p(tbe.feat_dim.data_ptr() + 4 * f0), ctypes.c_void_p(self.dev_direct[r].data_ptr() + 4 * f0),
                                ctypes.c_void_p(tbe.feat_fmt.data_ptr() + 4 * f0), ctypes.c_void_p(tbe.feat_rb.data_ptr() + 4 * f0), _lib.ptr(self.val_bufs[r]),
                                int(self.idx_dtype == torch.int64), ctypes.c_void_p(self.off_bufs[r].data_ptr() + 4 * f0 * B), 0, _lib.ptr(psw),
                                ctypes.c_void_p(out_ptr), _lib.dtype_code(m._output_dtype), ctypes.c_int64(out_stride), B, f1 - f0, tbe.max_dim, 0, 1,
                                ctypes.c_int64(0), int(tbe._uniform_fmt), _lib.stream_ptr(self.devs[r]))
                            _lib.check(c, "trb_qtbe_fwd_placed")
                            return
                        c = L.trb_qtbe_fwd_ex(
                            _lib.ptr(tbe.weights), ctypes.c_void_p(tbe.feat_woff.data_ptr() + 8 * f0), ctypes.c_void_p(tbe.feat_rows.data_ptr() + 8 * f0),
                            ctypes.c_void_p(tbe.feat_dim.data_ptr() + 4 * f0), ctypes.c_void_p(self.dev_direct[r].data_ptr() + 4 * f0),
                            ctypes.c_void_p(tbe.feat_fmt.data_ptr() + 4 * f0), ctypes.c_void_p(tbe.feat_rb.data_ptr() + 4 * f0), _lib.ptr(self.val_bufs[r]),
                            int(self.idx_dtype == torch.int64), ctypes.c_void_p(self.off_bufs[r].data_ptr() + 4 * f0 * B), 0, _lib.ptr(psw), ctypes.c_void_p(out_ptr),
                            _lib.dtype_code(m._output_dtype), ctypes.c_int64(out_stride), B, f1 - f0, tbe.max_dim, 0, 1, ctypes.c_int64(0), int(tbe._uniform_fmt),
                            _lib.stream_ptr(self.devs[r]))
                        _lib.check(c, "trb_qtbe_fwd_ex")

                    if tbe._placed:
                        tbe._wait_admission()
                    launch(0, n_direct, res.data_ptr(), m._total_cols)  # pooled rows -> final columns of the result on device 0 (peer stores)
                    if n_direct < F:
                        launch(n_direct, F, self.staging.data_ptr() + r * B * self.staged_width * esz, self.staged_width)
                    if tbe._placed and tbe._cached:
                        tbe._admit()  # this device's admission, on its side stream
                    if r != 0:
                        ev = torch.cuda.Event()
                        ev.record(st)
                        done.append(ev)
        for ev in done:
            main.wait_event(ev)
        if self.staged_cols:
            code = L.trb_staging_reduce_cols(_lib.ptr(self.staging), _lib.dtype_code(m._output_dtype), _lib.ptr(res), _lib.dtype_code(m._output_dtype),
                                             _lib.ptr(self.stage_mask), _lib.ptr(self.stage_dst), B, self.staged_width, ctypes.c_int64(self.staged_width),
                                             ctypes.c_int64(m._total_cols), ctypes.c_int64(B * self.staged_width), self.W, _lib.stream_ptr(self.dev0))
            _lib.check(code, "trb_staging_reduce_cols")
        if m._mean_features:
            lengths = features.lengths().view(len(keys), B)
            pos = {k: i for i, k in enumerate(keys)}
            for fi in m._mean_features:
                res[:, m._out_base[fi] : m._out_base[fi + 1]] /= lengths[pos[m._feature_names[fi]]].clamp(min=1).to(res.dtype).unsqueeze(1)
        return KeyedTensor(keys=m._embedding_names, length_per_key=m._dims, values=res)


class QuantEmbeddingBagCollectionSharder(BaseQuantEmbeddingSharder[QuantEmbeddingBagCollection]):
    def shard(self, module, params, env, device=None, module_fqn=None) -> ShardedQuantEmbeddingBagCollection:
        return ShardedQuantEmbeddingBagCollection(module, params, env, self.fused_params, device=device)

    def shardable_parameters(self, module: QuantEmbeddingBagCollection) -> Dict[str, nn.Parameter]:
        return {name: nn.Parameter(torch.empty(t.num_embeddings, t.embedding_dim, device="meta"), requires_grad=False)
                for name, t in ((t.name, t) for t in module.embedding_bag_configs())}

    @property
    def module_type(self) -> Type[QuantEmbeddingBagCollection]:
        return QuantEmbeddingBagCollection


# ---- feature-processed / managed-collision quantized bags: the processors and the collision modules are replicated (they are small and
# read-only when serving), the tables are sharded like plain quantized bags ------------------------------------------------------------------------
class _PreprocessedShardedQuantModule(nn.Module):
    """``pre(features)`` on the full batch, then the sharded quantized lookup; with ``return_features`` the pre-processed (remapped)
    features are returned next to the embeddings like the unsharded module does."""

    def __init__(self, sharded: nn.Module, pre: nn.Module, return_features: bool, configs: List[Any]) -> None:
        super().__init__()
        self._sharded = sharded
        self._pre = pre
        self._return_features = return_features
        self._configs = list(configs)

    def embedding_bag_configs(self) -> List[Any]:
        return self._configs

    def forward(self, features: KeyedJaggedTensor):
        features = self._pre(features)
        out = self._sharded(features)
        return (out, features) if self._return_features else out

    def sharded_module_weights_spec(self):  # plan / weight-spec tooling looks through the wrapper
        return getattr(self._sharded, "sharded_module_weights_spec", lambda: {})()


class ShardedQuantFeatureProcessedEmbeddingBagCollection(_PreprocessedShardedQuantModule):
    def __init__(self, module, params, env, fused_params=None, device=None) -> None:
        super().__init__(ShardedQuantEmbeddingBagCollection(module, params, env, fused_params, device=device), module.feature_processor, False, module.embedding_bag_configs())

    @property
    def feature_processor(self) -> nn.Module:
        return self._pre


class ShardedQuantManagedCollisionEmbeddingBagCollection(_PreprocessedShardedQuantModule):
    def __init__(self, module, params, env, fused_params=None, device=None) -> None:
        super().__init__(ShardedQuantEmbeddingBagCollection(module, params, env, fused_params, device=device), module._managed_collision_collection, True, module.embedding_bag_configs())


def _quant_cls(name: str):
    from ..quant import embedding_modules as q

    return getattr(q, name)


class QuantFeatureProcessedEmbeddingBagCollectionSharder(QuantEmbeddingBagCollectionSharder):
    def shard(self, module, params, env, device=None, module_fqn=None):
        return ShardedQuantFeatureProcessedEmbeddingBagCollection(module, params, env, self.fused_params, device=device)

    @property
    def module_type(self):
        return _quant_cls("FeatureProcessedEmbeddingBagCollection")


class QuantManagedCollisionEmbeddingBagCollectionSharder(QuantEmbeddingBagCollectionSharder):
    def shard(self, module, params, env, device=None, module_fqn=None):
        return ShardedQuantManagedCollisionEmbeddingBagCollection(module, params, env, self.fused_params, device=device)

    @property
    def module_type(self):
        return _quant_cls("QuantManagedCollisionEmbeddingBagCollection")
