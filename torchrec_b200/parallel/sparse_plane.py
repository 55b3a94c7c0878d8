"""The NVLink sparse data plane: input dist, fused lookup + output dist, fused gradient dist + optimizer for the
model-parallel tables of one sharded module, over symmetric peer memory of ONE NVLink domain.

Everything a training step touches lives at a fixed address in symmetric buffers that are sized once (per local batch size
and id capacity), so that

* no size ever visits the host (reference: splits all-to-all + ``.tolist()``, dist_data.py:506-572),
* every phase is a handful of native launches over static shapes and can be replayed as a CUDA graph
  (``SparsePlane.use_graphs``): the host cost of the sparse half of a step is a few graph launches,
* the phases are plain methods (``push_input`` / ``forward`` / ``backward``) that a test can drive for W *virtual* ranks
  on ONE device (``LoopbackGroup``) — the same kernels, pointer tables and layouts as on W GPUs, checked against fp32
  PyTorch references by ``tests/test_sparse_plane_gpu.py``.

Per step and rank (W ranks, local batch B):

    push_input   kjt_route (3 launches)   offsets + ids [+ weights] of every lookup unit -> the OWNER's receive region
    barrier(1)                            (device side, epoch flags over NVLink)
    forward      tbe_pooled_fwd x groups  pooled rows -> the SAMPLE OWNER's [B, sum D] output (row-sharded tables: staging)
    barrier(0)   + staging reduce
    backward     grad_push                gradient column blocks -> the table owners' inboxes
    barrier(0)
                 tbe_bwd x groups         sort + exact fused optimizer over local memory

Slot discipline (what makes the fixed buffers race free; B = barrier of the phase):
  ids      3 slots  push(j) reuses the slot of batch j-3 and first waits for the LOCAL completion of batch j-2's last phase: that
                    rank passed B(j-2), so every peer has finished reading batch j-3 (they arrived at B(j-2) after it).
  out      slot 0 in training (a peer's forward(i+1) is behind its backward barrier of step i, which we only reach after our
                    dense backward(i) consumed out(i)); slots 1/2 alternate for forward-only steps.
  inbox    1 slot   peers push gradients of step i only after the forward barrier of step i, i.e. after our tbe_bwd(i-1).

FP8 wire (``wire_format``): when the engine's quantized-comms codecs ask for FP8 row-wise, the lookup stores directly written pooled
rows as e4m3 groups of R columns plus one fp32 scale per group into an FP8 region of the out slot, and the gradient push does the
same into an FP8 inbox; after the barrier one decode launch per direction fills the out slot / inbox in the wire dtype, so
``out_local`` and ``inbox_local`` keep their meaning. Row-sharded (staged) columns stay at the wire dtype: they are summed at the
destination, and a row-scaled format cannot be summed on the wire.
"""
from __future__ import annotations

import ctypes
import itertools
import logging
import os
from dataclasses import dataclass
from typing import Any, Dict, List, Optional, Sequence, Tuple

import torch

from ..ops import _lib
from ..ops import tbe as T
from .p2p import SymmetricBuffer, tensor_from_ptr

INT64_MAX = (1 << 63) - 1
FP8_ROW_DIMS = (32, 64, 128)  # a group of R columns is R / 4 float4 lanes of the lookup kernels, R / 8 lanes of the push: inside one warp

logger = logging.getLogger(__name__)
_logged_reasons: set = set()


def _align(x: int, a: int = 256) -> int:
    return (int(x) + a - 1) // a * a


# ---------------------------------------------------------------------------------------------------------------
# W virtual ranks on one device
# ---------------------------------------------------------------------------------------------------------------
class LoopbackGroup:
    """``W`` virtual ranks in ONE process on ONE device: every "symmetric" allocation is W ordinary device buffers and every
    virtual rank sees all of them as its peers. The driver (a test, ``__graft_entry__.smoke``) runs the phases of all
    virtual ranks in lock step on one stream, which is what the device barrier guarantees between real ranks."""

    def __init__(self, world: int, device: torch.device, peer_devices: Optional[Sequence[torch.device]] = None) -> None:
        """``peer_devices``: optional device of every virtual rank's buffers. ``[cuda:0, cuda:1]`` puts rank 1's memory on a second GPU
        of THIS process (peer access enabled), so rank 0's kernels really store over NVLink - the single-process harness that ``ncu``
        can profile (tools/peer_bench.py)."""
        self.world = world
        self.device = torch.device(device)
        self.peer_devices = [torch.device(d) for d in peer_devices] if peer_devices is not None else [self.device] * world
        assert len(self.peer_devices) == world
        if len({str(d) for d in self.peer_devices}) > 1:
            L = _lib.lib()
            idx = sorted({d.index for d in self.peer_devices})
            for a in idx:
                for b in idx:
                    if a != b:
                        _lib.check(L.trb_enable_peer_access(a, b), f"trb_enable_peer_access({a},{b})")
        self._allocs: Dict[int, List[torch.Tensor]] = {}
        self._views = [_LoopbackView(self, r) for r in range(world)]

    def view(self, rank: int) -> "_LoopbackView":
        return self._views[rank]


class _LoopbackView:
    is_loopback = True

    def __init__(self, group: LoopbackGroup, rank: int) -> None:
        self.group = group
        self.world = group.world
        self.rank = rank
        self.device = group.peer_devices[rank]
        self._seq = 0

    def alloc(self, nbytes: int) -> SymmetricBuffer:
        nbytes = _align(nbytes)
        bufs = self.group._allocs.get(self._seq)
        if bufs is None:
            bufs = self.group._allocs[self._seq] = [torch.zeros(nbytes, dtype=torch.uint8, device=self.group.peer_devices[r]) for r in range(self.world)]
        assert bufs[0].numel() == nbytes, "virtual ranks must allocate the same sizes in the same order"
        self._seq += 1
        return SymmetricBuffer(nbytes, bufs[self.rank].data_ptr(), [b.data_ptr() for b in bufs], self.device)

    def barrier(self, channel: int = 0) -> None:  # lock-step driver: nothing to wait for
        return None


class SingleRankGroup:
    """World of one: the "symmetric" buffers are plain device memory, there is nobody to wait for. Lets a single GPU run the same
    static-shape, graph-replayed sparse phases as a multi-GPU job."""

    is_loopback = False
    world = 1
    rank = 0

    def __init__(self, device: torch.device) -> None:
        self.device = torch.device(device)
        self._keep: List[torch.Tensor] = []

    def alloc(self, nbytes: int) -> SymmetricBuffer:
        t = torch.zeros(_align(nbytes), dtype=torch.uint8, device=self.device)
        self._keep.append(t)
        return SymmetricBuffer(t.numel(), t.data_ptr(), [t.data_ptr()], self.device)

    def barrier(self, channel: int = 0) -> None:
        return None


# ---------------------------------------------------------------------------------------------------------------
def select_wire_format(world: int, direct_cols: Sequence[Tuple[int, int]], push_cols: Sequence[Tuple[int, int, int]],
                       codecs) -> Tuple[Dict[str, Optional[Tuple[str, int]]], List[str]]:
    """What each direction of a plane carries: ``{"fwd": ("fp8", R) | None, "bwd": ("fp8", R) | None}`` (``None``: the wire dtype).

    ``direct_cols``: (output column, width) of every directly written unit, the columns the forward may quantize (row-sharded
    units are summed at the destination and keep the wire dtype); ``push_cols``: (output column, inbox column, width) of every unit
    the gradient push serves. A direction is FP8 when its codec reports ``fp8_row_dim`` R (FP8 row-wise), R is 32, 64 or 128 and
    every column offset and width of that direction is a multiple of R; one rank sends nothing over a wire. Also returns the
    reasons an FP8 direction was refused."""
    fmt: Dict[str, Optional[Tuple[str, int]]] = {"fwd": None, "bwd": None}
    why: List[str] = []
    if world <= 1 or codecs is None:
        return fmt, why
    spans = {"fwd": list(direct_cols), "bwd": [(c, w) for c, _i, w in push_cols] + [(i, w) for _c, i, w in push_cols]}
    for d, codec in (("fwd", getattr(codecs, "forward", None)), ("bwd", getattr(codecs, "backward", None))):
        R = getattr(codec, "fp8_row_dim", None)
        if R is None or not spans[d]:
            continue
        if R not in FP8_ROW_DIMS:
            why.append(f"{d}: FP8 row dim {R} is not one of {FP8_ROW_DIMS}")
            continue
        bad = [(c, w) for c, w in spans[d] if c % R or w % R]
        if bad:
            why.append(f"{d}: the column block at {bad[0][0]} of width {bad[0][1]} is not aligned to the FP8 row dim {R}")
            continue
        fmt[d] = ("fp8", R)
    return fmt, why


@dataclass
class RoutedIds:
    """Handle of a batch whose ids sit in receive slot ``slot`` of ``plane`` (what the input dist of the NVLink plane returns
    instead of a KeyedJaggedTensor; ``to_kjt()`` compacts it into one when a consumer needs the jagged view)."""

    plane: "SparsePlane"
    slot: int
    B_local: int
    _stride_per_rank: Optional[List[int]] = None

    def stride(self) -> int:
        return self.B_local * self.plane.W

    def record_stream(self, stream) -> None:  # symmetric buffers are not owned by the caching allocator
        return None

    def variable_stride_per_key(self) -> bool:
        return False

    def to_kjt(self):
        return self.plane.ids_to_kjt(self.slot)


class SparsePlane:
    N_ID_SLOTS = 3
    N_OUT_SLOTS = 3  # 0: training, 1/2: forward-only steps

    def __init__(self, eng, group, B_local: int, total_cols: int, capacity: int, idx_dtype: torch.dtype, weighted: bool,
                 key_of_feature: Optional[Sequence[int]] = None) -> None:
        self.eng = eng
        self.group = group
        self.W = W = eng._W
        self.rank = eng._rank
        self.device = eng._device
        self.B_local = B_local
        self.total_cols = total_cols
        self.capacity = int(capacity)
        self.idx_dtype = idx_dtype
        self.weighted = weighted
        self.wire_dtype = eng._output_dtype
        self.loopback = bool(getattr(group, "is_loopback", False))
        esz = torch.empty(0, dtype=self.wire_dtype).element_size()
        isz = 8 if idx_dtype == torch.int64 else 4
        units = eng._units
        U = len(units)
        self.U_d = eng._units_per_rank[self.rank]
        U_max = max(eng._units_per_rank) if eng._units_per_rank else 0

        # ---- route table (global unit order = destination-rank major) -----------------------------------------------
        kof = list(key_of_feature) if key_of_feature is not None else list(range(len(eng._feature_names)))
        mp_pos = {f: i for i, f in enumerate(eng._mp_features)}
        if key_of_feature is None:  # input KJT carries exactly the model-parallel features, in flat feature order
            kof = [mp_pos.get(f, -1) for f in range(len(eng._feature_names))]
        lo, hi, key, dest, slot_, csl = [], [], [], [], [], []
        cols_of_feature: Dict[int, List[int]] = {}
        for u in units:
            cols_of_feature.setdefault(u.feature, [])
            if u.shard.col_off not in cols_of_feature[u.feature]:
                cols_of_feature[u.feature].append(u.shard.col_off)
        for f in cols_of_feature:
            cols_of_feature[f].sort()
        for u in units:
            row_sharded = eng._table_row_sharded[u.shard.table_idx]
            lo.append(u.shard.row_off if row_sharded else 0)
            hi.append(u.shard.row_off + u.shard.rows if row_sharded else INT64_MAX)
            key.append(kof[u.feature])
            dest.append(u.shard.rank)
            slot_.append(u.gidx - eng._unit_start[u.shard.rank])
            csl.append(cols_of_feature[u.feature].index(u.shard.col_off))
        dev = self.device
        mk32 = lambda x: torch.tensor(x, dtype=torch.int32, device=dev)
        mk64 = lambda x: torch.tensor(x, dtype=torch.int64, device=dev)
        self.u_key, self.u_dest, self.u_slot, self.u_cslice = mk32(key), mk32(dest), mk32(slot_), mk32(csl)
        self.u_lo, self.u_hi = mk64(lo), mk64(hi)
        self.dest_ustart = mk32(eng._unit_start)
        self.U = U
        self.route_ws = torch.empty(self._route_ws_bytes(U, B_local), dtype=torch.uint8, device=dev)
        self.overflow = torch.zeros(1, dtype=torch.int32, device=dev)
        self._overflow_host = torch.zeros(1, dtype=torch.int32).pin_memory() if dev.type == "cuda" else torch.zeros(1, dtype=torch.int32)
        self._overflow_event: Optional[torch.cuda.Event] = None

        # ---- symmetric layout ------------------------------------------------------------------------------------------
        self.off_stride = _align(U_max * B_local + 1, 64)            # int32 elements between source regions
        self.off_bytes = _align(self.off_stride * 4 * W)
        self.val_bytes = _align(self.capacity * isz * W)
        self.wgt_bytes = _align(self.capacity * 4 * W) if weighted else 0
        self.id_slot_bytes = self.off_bytes + self.val_bytes + self.wgt_bytes
        self.slab_bytes = _align(B_local * total_cols * esz)
        dims_f = [eng._tables[ti].embedding_dim for ti in eng._feature_table]
        base_f = list(itertools.accumulate([0] + dims_f))
        self.base_f = base_f
        # gradient inbox [W * B_local, pitch]: the columns of MY units side by side, one row block per source rank
        chunks: List[List[int]] = []
        local_cols_per_rank: List[List[int]] = []
        vec = 8 if all(u.shard.cols % 8 == 0 and (base_f[u.feature] + u.shard.col_off) % 8 == 0 for u in units) and total_cols % 8 == 0 else 4
        self.push_vec = vec
        for r in range(W):
            c = 0
            cols_r = []
            for u in units[eng._unit_start[r] : eng._unit_start[r + 1]]:
                src0 = base_f[u.feature] + u.shard.col_off
                cols_r.append(c)
                for k in range(0, u.shard.cols, vec):
                    chunks.append([r, src0 + k, c + k])
                c += u.shard.cols
            local_cols_per_rank.append(cols_r)
        assert all(u.shard.cols % 4 == 0 for u in units)
        self.inbox_pitch = max(8, (max((sum(u.shard.cols for u in units[eng._unit_start[r] : eng._unit_start[r + 1]]) for r in range(W)), default=8) + 7) // 8 * 8)
        self.inbox_bytes = _align(W * B_local * self.inbox_pitch * esz) if W > 1 else 256  # one rank: the backward reads the gradient in place
        self.chunks = torch.tensor(chunks, dtype=torch.int32, device=dev).reshape(-1, 3).contiguous()
        self.local_cols = local_cols_per_rank[self.rank]
        # staging for row-sharded tables: slab j of rank d = partial sums computed by rank j, compact staged columns only
        staged_cols: Dict[Tuple[int, int], int] = {}
        sc = 0
        for u in units:
            if eng._table_row_sharded[u.shard.table_idx] and (u.feature, u.shard.col_off) not in staged_cols:
                staged_cols[(u.feature, u.shard.col_off)] = sc
                sc += u.shard.cols
        self.staged_width = max(4, (sc + 3) // 4 * 4) if staged_cols else 0
        self.has_staged = bool(staged_cols)
        self.stage_slab_bytes = _align(B_local * self.staged_width * esz) if self.has_staged else 0
        # ---- wire format (the user's quantized-comms codecs) -----------------------------------------------------------
        direct = [u for u in units if not eng._table_row_sharded[u.shard.table_idx]]
        push_cols = [(base_f[u.feature] + u.shard.col_off, local_cols_per_rank[u.shard.rank][i - eng._unit_start[u.shard.rank]], u.shard.cols)
                     for i, u in enumerate(units)]
        self.wire_format, why = select_wire_format(W, [(base_f[u.feature] + u.shard.col_off, u.shard.cols) for u in direct], push_cols,
                                                   getattr(eng, "_codecs", None))
        for msg in why:
            if msg not in _logged_reasons:
                _logged_reasons.add(msg)
                logger.warning(f"NVLink sparse plane keeps its {self.wire_dtype} wire: {msg}")
        self.fwd_q = self.wire_format["fwd"][1] if self.wire_format["fwd"] else 0  # FP8 row dim of the forward, 0 = wire dtype
        self.bwd_q = self.wire_format["bwd"][1] if self.wire_format["bwd"] else 0
        self.id_off = [i * self.id_slot_bytes for i in range(self.N_ID_SLOTS)]
        o = self.N_ID_SLOTS * self.id_slot_bytes
        self.out_off = [o + i * self.slab_bytes for i in range(self.N_OUT_SLOTS)]
        o += self.N_OUT_SLOTS * self.slab_bytes
        self.inbox_off = o
        o += self.inbox_bytes
        self.staging_off = o
        o += self.stage_slab_bytes * W
        # FP8 regions follow everything else: without an FP8 direction the layout above is all there is
        if self.fwd_q:  # per out slot: payload [B_local, fq_pitch] uint8 + scales [B_local, fq_spitch] fp32
            self.fq_pitch, self.fq_spitch = _align(total_cols, 16), (total_cols + self.fwd_q - 1) // self.fwd_q
            self.fq_off: List[Tuple[int, int]] = []
            for _ in range(self.N_OUT_SLOTS):
                pay = _align(B_local * self.fq_pitch)
                self.fq_off.append((o, o + pay))
                o += pay + _align(B_local * self.fq_spitch * 4)
            self.fq_cols = mk32(sorted({base_f[u.feature] + u.shard.col_off + c for u in direct for c in range(0, u.shard.cols, 16)}))
        if self.bwd_q:  # inbox: payload [W * B_local, bq_pitch] uint8 + scales [W * B_local, bq_spitch] fp32
            R = self.bwd_q
            self.bq_pitch, self.bq_spitch = _align(self.inbox_pitch, 16), (self.inbox_pitch + R - 1) // R
            pay = _align(W * B_local * self.bq_pitch)
            self.bq_off = (o, o + pay)
            o += pay + _align(W * B_local * self.bq_spitch * 4)
            # (destination rank, gradient column, inbox column) of every R-column group
            self.bq_chunks = torch.tensor([[u.shard.rank, c + k, i + k] for u, (c, i, w) in zip(units, push_cols) for k in range(0, w, R)],
                                          dtype=torch.int32, device=dev).reshape(-1, 3).contiguous()
            local_width = sum(u.shard.cols for u in eng._local_units)
            self.bq_cols = mk32(list(range(0, local_width, 16)))
        self.buf = group.alloc(o)

        # staged column bookkeeping for the reduce: contributors + destination column per staged 4-column vector
        if self.has_staged:
            mask = [0] * self.staged_width
            dst = [0] * self.staged_width
            for u in units:
                k = (u.feature, u.shard.col_off)
                if k in staged_cols:
                    for c in range(u.shard.cols):
                        mask[staged_cols[k] + c] |= 1 << u.shard.rank
                        dst[staged_cols[k] + c] = base_f[u.feature] + u.shard.col_off + c
            self.stage_mask = torch.tensor(mask, dtype=torch.int64, device=dev).to(torch.int32)
            self.stage_dst = mk32(dst)
        # per kernel group: metas (columns in the final output / in the staging slab / in the local inbox)
        self.group_meta: List[Optional[Dict[str, Any]]] = []
        for g in eng._groups:
            if g.tbe is None:
                self.group_meta.append(None)
                continue
            u0, u1 = g.unit_range
            gunits = eng._local_units[u0:u1]
            staged = [eng._table_row_sharded[u.shard.table_idx] for u in gunits]
            n_direct = staged.index(True) if True in staged else len(gunits)
            assert all(staged[n_direct:]), "row-sharded units must follow direct units inside a group"
            out_cols = [base_f[u.feature] + u.shard.col_off for u in gunits]
            full = g.tbe.meta.with_cols(out_cols, total_cols)
            stage_cols = [staged_cols.get((u.feature, u.shard.col_off), 0) for u in gunits]
            stg = g.tbe.meta.with_cols(stage_cols, self.staged_width) if self.has_staged else None
            local = g.tbe.meta.with_cols(self.local_cols[u0:u1], self.inbox_pitch)
            self.group_meta.append({"n_direct": n_direct, "n": len(gunits), "direct": _slice_meta(full, 0, n_direct),
                                    "staged": _slice_meta(stg, n_direct, len(gunits)) if stg is not None else None, "local": local})
        # backward workspace (one per group, static so that the backward can be captured)
        # one per (id slot, group): the id-dependent half of the backward (keys + sort) runs right after the input dist of a batch,
        # on an auxiliary stream, while earlier batches are still training
        self.bwd_ws: List[List[Optional[torch.Tensor]]] = []
        for _slot in range(self.N_ID_SLOTS):
            per_group: List[Optional[torch.Tensor]] = []
            for g in eng._groups:
                if g.tbe is None or self.capacity == 0:
                    per_group.append(None)
                    continue
                nb = T.backward_workspace_bytes(self.W * self.capacity, g.tbe.meta.max_dim, g.tbe.meta.total_rows) if dev.type == "cuda" else 0
                per_group.append(torch.empty(nb + 1024, dtype=torch.uint8, device=dev))
            self.bwd_ws.append(per_group)
        self.presort = os.environ.get("TRB_BWD_PRESORT", "1") != "0" and self.capacity > 0
        self._aux_stream: Optional[torch.cuda.Stream] = None
        self._prepared: List[Optional[torch.cuda.Event]] = [None] * self.N_ID_SLOTS
        self.psw_grad_buf = torch.zeros(self.W * self.capacity, dtype=torch.float32, device=dev) if weighted else None
        self.dummy = torch.zeros(1, device=dev, requires_grad=True)
        self.step = 0
        self.eval_step = 0
        self.external_push = False
        self._last_use: List[Optional[torch.cuda.Event]] = [None] * self.N_ID_SLOTS
        # CUDA graphs of the static phases, keyed by (phase, id slot, out slot)
        self.use_graphs = os.environ.get("TRB_SPARSE_GRAPHS", "1") != "0" and not self.loopback
        self._graphs: Dict[Tuple, Any] = {}
        self._graph_warm: Dict[Tuple, int] = {}
        self._graph_launches: Dict[Tuple, int] = {}

    # ---- helpers ----------------------------------------------------------------------------------------------------
    @staticmethod
    def _route_ws_bytes(U: int, B: int) -> int:
        if not _lib.available():
            return 16
        L = _lib.lib()
        L.trb_kjt_route_workspace_bytes.restype = ctypes.c_int64
        return int(L.trb_kjt_route_workspace_bytes(U, B))

    def out_local(self, slot: int) -> torch.Tensor:
        return self.buf.local(self.wire_dtype, (self.B_local, self.total_cols), self.out_off[slot])

    def inbox_local(self) -> torch.Tensor:
        return self.buf.local(self.wire_dtype, (self.W * self.B_local, self.inbox_pitch), self.inbox_off)

    def regions(self, slot: int) -> T.IdRegions:
        """This rank's receive slot as the kernels see it."""
        base = self.buf.local_ptr + self.id_off[slot]
        return T.IdRegions(idx_ptr=base + self.off_bytes, idx64=int(self.idx_dtype == torch.int64), off_ptr=base, off64=0,
                           psw_ptr=(base + self.off_bytes + self.val_bytes) if self.weighted else 0, n_src=self.W, idx_stride=self.capacity,
                           off_stride=self.off_stride, src_B=self.B_local)

    def _region_tensors(self, slot: int) -> Tuple[torch.Tensor, torch.Tensor, Optional[torch.Tensor]]:
        base = self.id_off[slot]
        off = self.buf.local(torch.int32, (self.W, self.off_stride), base)
        val = self.buf.local(self.idx_dtype, (self.W, self.capacity), base + self.off_bytes)
        wgt = self.buf.local(torch.float32, (self.W, self.capacity), base + self.off_bytes + self.val_bytes) if self.weighted else None
        return off, val, wgt

    def ids_to_kjt(self, slot: int):
        """Compact the receive slot into a regular KeyedJaggedTensor ([unit][source rank][sample] order). Host-syncing slow
        path for consumers that need the jagged view (lookup hooks, debugging, tests)."""
        from ..sparse.jagged_tensor import KeyedJaggedTensor

        off, val, wgt = self._region_tensors(slot)
        U_d, B = self.U_d, self.B_local
        lens = (off[:, 1 : U_d * B + 1] - off[:, : U_d * B]).view(self.W, U_d, B).permute(1, 0, 2).reshape(-1)
        vals, wts = [], []
        for ul in range(U_d):
            for s in range(self.W):
                a, b = int(off[s, ul * B]), int(off[s, (ul + 1) * B])
                vals.append(val[s, a:b])
                if wgt is not None:
                    wts.append(wgt[s, a:b])
        keys = [self.eng._feature_names[u.feature] for u in self.eng._local_units]
        return KeyedJaggedTensor(keys=keys, values=torch.cat(vals) if vals else val.new_zeros(0), weights=torch.cat(wts) if wts else None,
                                 lengths=lens.to(torch.int64), stride=self.W * B, stride_per_rank=[B] * self.W)

    # ---- phase 1: input dist ------------------------------------------------------------------------------------------
    def push_input(self, in_offsets: torch.Tensor, in_values: torch.Tensor, in_weights: Optional[torch.Tensor], avg_len_hint: int = 1,
                   training: Optional[bool] = None) -> RoutedIds:
        """Route the local batch to the owners of the lookup units (peer stores). Returns the handle of the batch."""
        assert in_values.dtype == self.idx_dtype, f"ids are {in_values.dtype}, plane was sized for {self.idx_dtype}"
        slot = self.step % self.N_ID_SLOTS
        self.step += 1
        stream = torch.cuda.current_stream(self.device) if self.device.type == "cuda" else None
        ev = self._last_use[(slot + 1) % self.N_ID_SLOTS]  # batch j-2: see the slot discipline in the module docstring
        if ev is not None and stream is not None:
            stream.wait_event(ev)
        self._check_overflow()
        base = self.id_off[slot]
        me = self.rank
        off_ptrs = [p + base + me * self.off_stride * 4 for p in self.buf.ptrs]
        isz = 8 if self.idx_dtype == torch.int64 else 4
        val_ptrs = [p + base + self.off_bytes + me * self.capacity * isz for p in self.buf.ptrs]
        wgt_ptrs = [p + base + self.off_bytes + self.val_bytes + me * self.capacity * 4 for p in self.buf.ptrs] if (self.weighted and in_weights is not None) else None
        L = _lib.lib()
        code = L.trb_kjt_route(
            _lib.ptr(in_offsets), int(in_offsets.dtype == torch.int64), _lib.ptr(in_values), int(in_values.dtype == torch.int64),
            _lib.ptr(in_weights.float() if (in_weights is not None and in_weights.dtype != torch.float32) else in_weights) if wgt_ptrs is not None else ctypes.c_void_p(0),
            self.B_local, _lib.ptr(self.u_key), _lib.ptr(self.u_lo), _lib.ptr(self.u_hi), _lib.ptr(self.u_dest), _lib.ptr(self.u_slot), _lib.ptr(self.u_cslice),
            _lib.ptr(self.dest_ustart), self.U, self.W, _lib.ptr_array(off_ptrs), 0, _lib.ptr_array(val_ptrs), int(self.idx_dtype == torch.int64),
            _lib.ptr_array(wgt_ptrs) if wgt_ptrs is not None else ctypes.c_void_p(0), ctypes.c_int64(self.capacity), ctypes.c_void_p(0), 1,
            _lib.ptr(self.overflow), _lib.ptr(self.route_ws), ctypes.c_int64(self.route_ws.numel()), int(avg_len_hint), _lib.stream_ptr(self.device))
        _lib.check(code, "trb_kjt_route")
        if stream is not None and not self.loopback:
            self._overflow_host.copy_(self.overflow, non_blocking=True)
            self._overflow_event = torch.cuda.Event()
            self._overflow_event.record(stream)
        self.group.barrier(1)
        if training is None:
            training = torch.is_grad_enabled()
        if self.presort and training and not self.loopback:
            self.prepare_backward(slot)
        return RoutedIds(self, slot, self.B_local, [self.B_local] * self.W)

    def prepare_backward(self, slot: int, fork: bool = True) -> None:
        """Id-dependent half of the fused backward (row keys + radix sort) of the batch in ``slot``, on an auxiliary stream forked
        from the current one: it overlaps the forward / the previous step instead of sitting between the dense backward and the
        optimizer update."""
        cur = torch.cuda.current_stream(self.device)
        if fork:
            if self._aux_stream is None:
                self._aux_stream = torch.cuda.Stream(self.device)
            aux = self._aux_stream
            aux.wait_stream(cur)
        else:
            aux = cur
        reg = self.regions(slot)
        with torch.cuda.stream(aux):
            self._backward_kernels(reg, slot, 1.0, phase=1)
            ev = torch.cuda.Event()
            ev.record(aux)
        self._prepared[slot] = ev

    def _check_overflow(self, wait: bool = False) -> None:
        ev = self._overflow_event
        if ev is None:
            return
        if wait:
            ev.synchronize()
        if ev.query():
            self._overflow_event = None
            if int(self._overflow_host[0]) != 0:
                raise RuntimeError(f"NVLink input dist overflow: a destination received more than {self.capacity} ids from one rank; raise "
                                   "TRB_MAX_IDS_PER_RANK / TRB_ID_CAPACITY_SLACK (the affected step looked up a truncated batch)")

    # ---- phase 2: lookup + output dist ---------------------------------------------------------------------------------
    def _ids_of(self, ids) -> Tuple[T.IdRegions, Optional[int]]:
        if isinstance(ids, RoutedIds):
            return self.regions(ids.slot), ids.slot
        # a regular distributed KJT (NCCL / feature-processor path): one source region
        values, offsets = ids.values(), ids.offsets()
        w = ids.weights_or_none() if self.weighted else None
        self._keep = (values, offsets, w)
        return T.IdRegions(values.data_ptr(), int(values.dtype == torch.int64), offsets.data_ptr(), int(offsets.dtype == torch.int64),
                           w.data_ptr() if w is not None else 0, 1, values.numel(), 0, ids.stride()), None

    def _forward_kernels(self, reg: T.IdRegions, out_slot: int, local_only: bool = False) -> None:
        eng = self.eng
        out_ptrs = self.buf.peer_ptrs(self.out_off[out_slot])
        stage_ptrs = [p + self.staging_off + self.rank * self.stage_slab_bytes for p in self.buf.ptrs]
        fp8 = None
        if self.fwd_q:  # direct columns go to the FP8 region of the out slot
            pay, sc = self.fq_off[out_slot]
            out_ptrs = self.buf.peer_ptrs(pay)
            fp8 = (self.buf.peer_ptrs(sc), self.fq_spitch, self.fwd_q)
        if local_only:  # measurement aid (bench.py): the same lookup with every destination aliased to local memory = no NVLink traffic
            out_ptrs = [self.buf.local_ptr + (self.fq_off[out_slot][0] if self.fwd_q else self.out_off[out_slot])] * self.W
            stage_ptrs = [self.buf.local_ptr + self.staging_off + self.rank * self.stage_slab_bytes] * self.W
            if fp8 is not None:
                fp8 = ([self.buf.local_ptr + self.fq_off[out_slot][1]] * self.W, self.fq_spitch, self.fwd_q)
        out_pitch = self.fq_pitch if self.fwd_q else self.total_cols
        for g, gm in zip(eng._groups, self.group_meta):
            if gm is None:
                continue
            u0, _ = g.unit_range
            mean = g.pooling == T.PoolingMode.MEAN
            if gm["direct"] is not None:
                T.pooled_forward_regions(gm["direct"], g.tbe.weights, reg.window(u0), mean, self.wire_dtype, out_ptrs, out_pitch, self.B_local, self.device, fp8=fp8)
            if gm["staged"] is not None:
                T.pooled_forward_regions(gm["staged"], g.tbe.weights, reg.window(u0 + gm["n_direct"]), False, self.wire_dtype, stage_ptrs, self.staged_width,
                                         self.B_local, self.device)

    def _staging_reduce(self, out_slot: int) -> None:
        if not self.has_staged:
            return
        L = _lib.lib()
        esz_code = _lib.dtype_code(self.wire_dtype)
        code = L.trb_staging_reduce_cols(ctypes.c_void_p(self.buf.local_ptr + self.staging_off), esz_code, _lib.ptr(self.out_local(out_slot)), esz_code,
                                         _lib.ptr(self.stage_mask), _lib.ptr(self.stage_dst), self.B_local, self.staged_width, ctypes.c_int64(self.staged_width),
                                         ctypes.c_int64(self.total_cols), ctypes.c_int64(self.stage_slab_bytes // torch.empty(0, dtype=self.wire_dtype).element_size()),
                                         self.W, _lib.stream_ptr(self.device))
        _lib.check(code, "trb_staging_reduce_cols")

    def _decode_out(self, out_slot: int) -> None:
        """FP8 payload + scales of the direct columns -> the out slot in the wire dtype (after the barrier; disjoint from the staged
        columns the staging reduce writes)."""
        if not self.fwd_q:
            return
        from . import p2p

        pay, sc = self.fq_off[out_slot]
        p2p.fp8_wire_decode(self.buf.local_ptr + pay, self.fq_pitch, self.buf.local_ptr + sc, self.fq_spitch, self.fwd_q, self.fq_cols, self.B_local,
                            self.out_local(out_slot))

    def _decode_inbox(self) -> None:
        """FP8 gradient inbox -> ``inbox_local()`` in the wire dtype (after the barrier, before the fused backward reads it)."""
        if not self.bwd_q:
            return
        from . import p2p

        pay, sc = self.bq_off
        p2p.fp8_wire_decode(self.buf.local_ptr + pay, self.bq_pitch, self.buf.local_ptr + sc, self.bq_spitch, self.bwd_q, self.bq_cols, self.W * self.B_local,
                            self.inbox_local())

    def forward(self, ids, training: bool) -> Tuple[torch.Tensor, int]:
        """Lookup + pooled output dist of the batch in ``ids``; returns (local ``[B_local, total_cols]`` output, out slot)."""
        reg, id_slot = self._ids_of(ids)
        if training:
            out_slot = 0
        else:
            out_slot = 1 + self.eval_step % 2
            self.eval_step += 1
        key = ("fwd", id_slot, out_slot)
        if self.use_graphs and id_slot is not None and self._graphable():
            self._run_graphed(key, lambda: self._forward_all(reg, out_slot))
        else:
            self._forward_all(reg, out_slot)
        self._mark_use(id_slot)
        return self.out_local(out_slot), out_slot

    def _forward_all(self, reg: T.IdRegions, out_slot: int) -> None:
        self._forward_kernels(reg, out_slot)
        self.group.barrier(0)
        self._staging_reduce(out_slot)
        self._decode_out(out_slot)

    # lock-step halves for the loopback driver
    def forward_kernels(self, ids, out_slot: int = 0) -> None:
        reg, _ = self._ids_of(ids)
        self._forward_kernels(reg, out_slot)

    def forward_finish(self, out_slot: int = 0) -> torch.Tensor:
        self._staging_reduce(out_slot)
        self._decode_out(out_slot)
        return self.out_local(out_slot)

    # ---- phase 3: gradient dist + fused optimizer ----------------------------------------------------------------------
    def _push_kernels(self, grad: torch.Tensor) -> None:
        from . import p2p

        if self.bwd_q:
            p2p.grad_push_fp8(grad, self.bq_chunks, self.bwd_q, self.buf.peer_ptrs(self.bq_off[0]), self.buf.peer_ptrs(self.bq_off[1]), self.bq_pitch,
                              self.bq_spitch, self.rank * self.B_local)
            return
        p2p.grad_push(grad, self.chunks, self.buf.peer_ptrs(self.inbox_off), self.wire_dtype, self.inbox_pitch, self.rank * self.B_local, 1.0, self.push_vec)

    def _backward_kernels(self, reg: T.IdRegions, id_slot: Optional[int], grad_scale: float, phase: int, want_psw: bool = False,
                          grad: Optional[torch.Tensor] = None) -> None:
        eng = self.eng
        Bg = self.W * self.B_local
        if self.W == 1 and grad is not None:  # one rank: gradient rows are read where autograd left them (no inbox, no copy)
            grad_ptrs, g_stride, g_dtype, mkey = [grad.data_ptr()], grad.stride(0), grad.dtype, "direct"
        else:
            grad_ptrs, g_stride, g_dtype, mkey = [self.buf.local_ptr + self.inbox_off], self.inbox_pitch, self.wire_dtype, "local"
        for gi, (g, gm) in enumerate(zip(eng._groups, self.group_meta)):
            if gm is None:
                continue
            u0, _ = g.unit_range
            mean = g.pooling == T.PoolingMode.MEAN
            w = reg.window(u0)
            if want_psw and phase != 1:
                T.psw_grad_regions(gm[mkey], g.tbe.weights, w, mean, grad_ptrs, g_stride, g_dtype, Bg, self.psw_grad_buf)
            if phase != 1:
                g.tbe._pre_update()
            if id_slot is not None:
                ws = self.bwd_ws[id_slot][gi]
            else:  # single-source KJT: positions vary per batch
                ws = T._workspace(T.backward_workspace_bytes(reg.positions, g.tbe.meta.max_dim, g.tbe.meta.total_rows), self.device)
            sr = g.tbe.stochastic_rounding and phase != 1
            T.fused_backward_regions(gm[mkey], g.tbe.weights, g.tbe.state1, g.tbe.state2, g.tbe.hyper_dev, g.tbe.opt_code, int(g.tbe.weight_decay_mode), w, mean,
                                     grad_ptrs, g_stride, g_dtype, grad_scale, Bg, ws, self.device,
                                     stochastic_rounding=sr, sr_seed=g.tbe.next_sr_seed() if sr else 0, phase=phase)

    def _apply_kernels(self, reg: T.IdRegions, id_slot: Optional[int], grad_scale: float, want_psw: bool, grad: Optional[torch.Tensor] = None) -> None:
        prepared = id_slot is not None and self._prepared[id_slot] is not None
        self._decode_inbox()
        self._backward_kernels(reg, id_slot, grad_scale, phase=2 if prepared else 0, want_psw=want_psw, grad=grad)

    def backward(self, ids, grad: torch.Tensor, grad_scale: float, want_psw: bool = False) -> None:
        reg, id_slot = self._ids_of(ids)
        if reg.n_src == 1:
            # single-source ids: positions = the KJT's id count; the static workspace was sized for W * capacity positions
            assert reg.idx_stride <= self.W * self.capacity, "distributed KJT larger than the plane's id capacity"
        prepared = id_slot is not None and self._prepared[id_slot] is not None
        if prepared:
            torch.cuda.current_stream(self.device).wait_event(self._prepared[id_slot])
        # the producer of `grad` may already have pushed it (DLRM: the push is captured inside the dense backward graph, where it
        # overlaps the deferred weight gradients); the flag is raised per step by that producer's forward
        ext = bool(self.external_push) and self.W > 1
        self.external_push = False
        key = ("bwd", id_slot, grad.data_ptr(), tuple(grad.shape), grad.stride(0), float(grad_scale), bool(want_psw), prepared, ext)
        if self.use_graphs and id_slot is not None and self._graphable():
            self._run_graphed(key, lambda: self._backward_all(reg, id_slot, grad, grad_scale, want_psw, ext))
        else:
            self._backward_all(reg, id_slot, grad, grad_scale, want_psw, ext)
        if prepared:
            self._prepared[id_slot] = None
        self._mark_use(id_slot)

    def _backward_all(self, reg: T.IdRegions, id_slot: Optional[int], grad: torch.Tensor, grad_scale: float, want_psw: bool, external_push: bool = False) -> None:
        if self.W == 1:
            self._apply_kernels(reg, id_slot, grad_scale, want_psw, grad=grad)
            return
        if not external_push:
            self._push_kernels(grad)
        self.group.barrier(0)
        self._apply_kernels(reg, id_slot, grad_scale, want_psw)

    def backward_push(self, grad: torch.Tensor) -> None:
        self._push_kernels(grad)

    def backward_apply(self, ids, grad_scale: float, want_psw: bool = False) -> None:
        reg, id_slot = self._ids_of(ids)
        self._apply_kernels(reg, id_slot, grad_scale, want_psw)
        if id_slot is not None:
            self._prepared[id_slot] = None

    # ---- CUDA graphs ---------------------------------------------------------------------------------------------------
    def _graphable(self) -> bool:
        for g in self.eng._groups:
            if g.tbe is None:
                continue
            if g.tbe.stochastic_rounding or g.tbe.__dict__.get("_fs") is not None or g.tbe._needs_step():
                return False  # per-step host state (rounding seed, step counter, 2D weight gathering) is baked into launches
        return True

    def _run_graphed(self, key: Tuple, fn) -> None:
        g = self._graphs.get(key)
        if g is not None:
            g.replay()
            _lib.add_launches(self._graph_launches[key])
            return
        warm = self._graph_warm.get(key, 0)
        if warm < 1 or len(self._graphs) >= 24:  # first occurrence eager (allocations, lazy init); cap the number of variants
            self._graph_warm[key] = warm + 1
            fn()
            return
        n0 = _lib.launch_count()
        graph = torch.cuda.CUDAGraph()
        # thread-local capture mode: the NCCL watchdog / other threads keep issuing (harmless) CUDA calls while we capture
        with torch.cuda.graph(graph, capture_error_mode="thread_local"):
            fn()
        self._graph_launches[key] = _lib.launch_count() - n0  # counted once by the capture, executed once by this first replay
        self._graphs[key] = graph
        graph.replay()

    def _mark_use(self, id_slot: Optional[int]) -> None:
        if id_slot is None or self.device.type != "cuda":
            return
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream(self.device))
        self._last_use[id_slot] = ev


def _slice_meta(m, a: int, b: int):
    if m is None or b <= a:
        return None
    return T.TbeMeta(m.feat_woff[a:b].contiguous(), m.feat_rows[a:b].contiguous(), m.feat_rowbase[a:b].contiguous(), m.feat_dim[a:b].contiguous(),
                     m.feat_col[a:b].contiguous(), m.h_woff[a:b], m.h_rows[a:b], m.h_rowbase[a:b], m.h_dim[a:b], m.h_col[a:b],
                     max(m.h_dim[a:b]), m.total_rows, m.total_cols, b - a)
