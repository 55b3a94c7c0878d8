"""Table-batched embedding (TBE) engine: one flat weight buffer for many tables, a single-launch
pooled / sequence forward and a fused exact backward+optimizer.

H100-native replacement for FBGEMM's ``SplitTableBatchedEmbeddingBagsCodegen`` /
``DenseTableBatchedEmbeddingBagsCodegen`` as used by the reference wrappers
(torchrec/distributed/batched_embedding_kernel.py:2915-3124, 3703-3826, 4636-4691).

CUDA tensors always run the sm_90a kernels in ``csrc/tbe_fwd.cu`` / ``csrc/tbe_bwd.cu``; CPU
tensors run the PyTorch reference implementation in this file (also the numerics oracle of the
GPU tests).
"""
from __future__ import annotations

import ctypes
import enum
import math
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

import torch
import torch.nn as nn

from . import _lib


class OptimType(enum.Enum):
    """Sparse optimizers fused into the TBE backward (reference: embedding_types.py:57-72)."""

    SGD = "sgd"
    EXACT_SGD = "exact_sgd"
    EXACT_ROWWISE_ADAGRAD = "exact_row_wise_adagrad"
    EXACT_ADAGRAD = "exact_adagrad"
    ADAM = "adam"
    ADAMW = "adamw"
    PARTIAL_ROWWISE_ADAM = "partial_row_wise_adam"
    LAMB = "lamb"
    PARTIAL_ROWWISE_LAMB = "partial_row_wise_lamb"
    LARS_SGD = "lars_sgd"
    LION = "lion"
    NONE = "none"  # dense gradient for an external optimizer / DDP

    def __str__(self) -> str:
        return self.value


_OPT_CODE = {
    OptimType.SGD: 0,
    OptimType.EXACT_SGD: 0,
    OptimType.EXACT_ROWWISE_ADAGRAD: 1,
    OptimType.EXACT_ADAGRAD: 2,
    OptimType.ADAM: 3,
    OptimType.ADAMW: 3,
    OptimType.PARTIAL_ROWWISE_ADAM: 4,
    OptimType.LAMB: 5,
    OptimType.PARTIAL_ROWWISE_LAMB: 6,
    OptimType.LARS_SGD: 7,
    OptimType.NONE: 8,
    OptimType.LION: 9,
}

# (state1 kind, state2 kind): "row" = one fp32 per row, "elem" = same shape as the weights
_OPT_STATE = {
    0: (None, None),
    1: ("row", None),
    2: ("elem", None),
    3: ("elem", "elem"),
    4: ("elem", "row"),
    5: ("elem", "elem"),
    6: ("elem", "row"),
    7: (None, None),
    8: (None, None),
    9: ("elem", None),
}

# names follow the reference's optimizer state keys (first state is always "momentum1",
# batched_embedding_kernel.py:1598-1608)
_OPT_STATE_NAMES = {
    1: ("momentum1", None),
    2: ("momentum1", None),
    3: ("momentum1", "momentum2"),
    4: ("momentum1", "momentum2"),
    5: ("momentum1", "momentum2"),
    6: ("momentum1", "momentum2"),
    9: ("momentum1", None),
}

HP_LR, HP_EPS, HP_BETA1, HP_BETA2, HP_WD, HP_STEP, HP_MAXGRAD, HP_MOMENTUM = range(8)


class WeightDecayMode(enum.IntEnum):
    NONE = 0
    L2 = 1
    DECOUPLE = 2


class EmbeddingLocation(enum.IntEnum):
    """Where a table-batched module keeps its rows (reference: fbgemm EmbeddingLocation / compute kernels
    FUSED, FUSED_UVM, FUSED_UVM_CACHING)."""

    DEVICE = 0            # HBM
    MANAGED = 1           # pinned host memory read / written zero-copy by the kernels (tables larger than HBM)
    MANAGED_CACHING = 2   # MANAGED backing store + software-managed HBM cache (ops/uvm.py)
    HOST = 3              # plain CPU


class PoolingMode(enum.IntEnum):
    SUM = 0
    MEAN = 1
    NONE = 2


@dataclass
class TbeMeta:
    """Per-feature descriptor tables of one TBE (device resident, built once per plan)."""

    feat_woff: torch.Tensor  # int64 [F]
    feat_rows: torch.Tensor  # int64 [F]
    feat_rowbase: torch.Tensor  # int64 [F]
    feat_dim: torch.Tensor  # int32 [F]
    feat_col: torch.Tensor  # int32 [F]
    h_woff: List[int] = field(default_factory=list)
    h_rows: List[int] = field(default_factory=list)
    h_rowbase: List[int] = field(default_factory=list)
    h_dim: List[int] = field(default_factory=list)
    h_col: List[int] = field(default_factory=list)
    max_dim: int = 0
    total_rows: int = 0
    total_cols: int = 0  # width of the output this TBE writes into
    num_features: int = 0

    @staticmethod
    def build(
        table_rows: Sequence[int],
        table_dims: Sequence[int],
        feature_table_map: Sequence[int],
        device: torch.device,
        feat_cols: Optional[Sequence[int]] = None,
        total_cols: Optional[int] = None,
    ) -> "TbeMeta":
        woff_t, rowbase_t = [], []
        w = r = 0
        for rows, dim in zip(table_rows, table_dims):
            if dim % 4 != 0:
                raise ValueError(f"embedding_dim must be a multiple of 4, got {dim}")
            woff_t.append(w)
            rowbase_t.append(r)
            w += rows * dim
            r += rows
        h_woff = [woff_t[t] for t in feature_table_map]
        h_rows = [table_rows[t] for t in feature_table_map]
        h_rowbase = [rowbase_t[t] for t in feature_table_map]
        h_dim = [table_dims[t] for t in feature_table_map]
        if feat_cols is None:
            h_col, c = [], 0
            for d in h_dim:
                h_col.append(c)
                c += d
            tot = c
        else:
            h_col = list(feat_cols)
            tot = total_cols if total_cols is not None else max((c + d for c, d in zip(h_col, h_dim)), default=0)
        if total_cols is not None:
            tot = total_cols
        mk64 = lambda x: torch.tensor(x, dtype=torch.int64, device=device)
        mk32 = lambda x: torch.tensor(x, dtype=torch.int32, device=device)
        return TbeMeta(
            mk64(h_woff), mk64(h_rows), mk64(h_rowbase), mk32(h_dim), mk32(h_col),
            h_woff, h_rows, h_rowbase, h_dim, h_col,
            max(h_dim) if h_dim else 0, r, tot, len(feature_table_map),
        )

    def with_cols(self, feat_cols: Sequence[int], total_cols: int) -> "TbeMeta":
        m = TbeMeta(
            self.feat_woff, self.feat_rows, self.feat_rowbase, self.feat_dim,
            torch.tensor(list(feat_cols), dtype=torch.int32, device=self.feat_dim.device),
            self.h_woff, self.h_rows, self.h_rowbase, self.h_dim, list(feat_cols),
            self.max_dim, self.total_rows, total_cols, self.num_features,
        )
        return m


# ----------------------------------------------------------------------------------------------
# reference (CPU / oracle) implementations
# ----------------------------------------------------------------------------------------------
def _ref_pooled_forward(meta: TbeMeta, weights, indices, offsets, psw, B: int, mean: bool, out_dtype, out=None) -> torch.Tensor:
    if out is None:
        out = torch.zeros(B, meta.total_cols, dtype=out_dtype, device=weights.device)
    offsets = offsets.to(torch.int64)
    indices = indices.to(torch.int64)
    for f in range(meta.num_features):
        D, rows = meta.h_dim[f], meta.h_rows[f]
        table = weights[meta.h_woff[f] : meta.h_woff[f] + rows * D].view(rows, D).float()
        off = offsets[f * B : (f + 1) * B + 1]
        lo, hi = int(off[0]), int(off[-1])
        idx = indices[lo:hi]
        lengths = off[1:] - off[:-1]
        valid = (idx >= 0) & (idx < rows)
        safe = torch.where(valid, idx, torch.zeros_like(idx))
        vals = table[safe]
        w = valid.to(torch.float32)
        if psw is not None:
            w = w * psw[lo:hi].float()
        vals = vals * w.unsqueeze(1)
        seg = torch.repeat_interleave(torch.arange(B, device=weights.device), lengths)
        pooled = torch.zeros(B, D, dtype=torch.float32, device=weights.device)
        pooled.index_add_(0, seg, vals)
        if mean:
            pooled = pooled / lengths.clamp(min=1).unsqueeze(1).float()
        out[:, meta.h_col[f] : meta.h_col[f] + D] = pooled.to(out.dtype)
    return out


def _ref_seq_forward(meta: TbeMeta, weights, indices, offsets, B: int, out_dtype) -> torch.Tensor:
    D = meta.h_dim[0] if meta.num_features else 0
    offsets = offsets.to(torch.int64)
    indices = indices.to(torch.int64)
    first = int(offsets[0]) if meta.num_features else 0
    total = (int(offsets[meta.num_features * B]) - first) if meta.num_features else 0
    out = torch.zeros(total, D, dtype=torch.float32, device=weights.device)
    for f in range(meta.num_features):
        rows = meta.h_rows[f]
        table = weights[meta.h_woff[f] : meta.h_woff[f] + rows * D].view(rows, D).float()
        lo, hi = int(offsets[f * B]), int(offsets[(f + 1) * B])
        idx = indices[lo:hi]
        valid = (idx >= 0) & (idx < rows)
        safe = torch.where(valid, idx, torch.zeros_like(idx))
        out[lo - first : hi - first] = table[safe] * valid.unsqueeze(1).float()
    return out.to(out_dtype)


def _ref_row_grads(meta: TbeMeta, indices, offsets, psw, grad: torch.Tensor, B: int, mean: bool, pooled: bool):
    """Yield (feature-group key, table view info, unique rows, summed grads) per table."""
    offsets = offsets.to(torch.int64)
    indices = indices.to(torch.int64)
    per_table: Dict[int, List[Tuple[torch.Tensor, torch.Tensor]]] = {}
    tinfo: Dict[int, Tuple[int, int, int]] = {}
    for f in range(meta.num_features):
        D, rows = meta.h_dim[f], meta.h_rows[f]
        if rows == 0:  # an empty shard shares its weight offset with the next table: nothing to update, and it must not alias that table's key
            continue
        lo, hi = int(offsets[f * B]), int(offsets[(f + 1) * B])
        idx = indices[lo:hi]
        if pooled:
            off = offsets[f * B : (f + 1) * B + 1]
            lengths = off[1:] - off[:-1]
            seg = torch.repeat_interleave(torch.arange(B, device=grad.device), lengths)
            g = grad[:, meta.h_col[f] : meta.h_col[f] + D].float()[seg]
            scale = torch.ones(hi - lo, dtype=torch.float32, device=grad.device)
            if psw is not None:
                scale = scale * psw[lo:hi].float()
            if mean:
                scale = scale / lengths.clamp(min=1).float()[seg]
            g = g * scale.unsqueeze(1)
        else:
            first = int(offsets[0])
            g = grad[lo - first : hi - first].float()
        valid = (idx >= 0) & (idx < rows)
        idx, g = idx[valid], g[valid]
        key = meta.h_woff[f]
        per_table.setdefault(key, []).append((idx, g))
        tinfo[key] = (rows, D, meta.h_rowbase[f])
    for key, parts in per_table.items():
        rows, D, rowbase = tinfo[key]
        idx = torch.cat([p[0] for p in parts])
        g = torch.cat([p[1] for p in parts])
        if idx.numel() == 0:
            continue
        uniq, inv = torch.unique(idx, return_inverse=True)
        gs = torch.zeros(uniq.numel(), D, dtype=torch.float32, device=g.device)
        gs.index_add_(0, inv, g)
        yield key, rows, D, rowbase, uniq, gs


def _ref_apply(opt: int, wd_mode: int, hyper: List[float], weights, state1, state2, key, rows, D, rowbase, uniq, g):
    lr, eps, b1, b2, wd, step, maxg = hyper[HP_LR], hyper[HP_EPS], hyper[HP_BETA1], hyper[HP_BETA2], hyper[HP_WD], hyper[HP_STEP], hyper[HP_MAXGRAD]
    table = weights[key : key + rows * D].view(rows, D)
    w = table[uniq].float()
    if maxg > 0:
        g = g.clamp(-maxg, maxg)
    if opt == 8:
        s = state1[key : key + rows * D].view(rows, D)
        s[uniq] += g
        return
    if wd_mode == 1:
        g = g + wd * w
    if wd_mode == 2 and opt in (0, 1, 2, 7):
        w = w * (1.0 - lr * wd)
    grow = rowbase + uniq
    if opt == 0:
        w = w - lr * g
    elif opt == 1:
        ns = state1[grow] + (g * g).sum(1) / D
        state1[grow] = ns
        w = w - (lr / (ns.sqrt() + eps)).unsqueeze(1) * g
    elif opt == 2:
        s = state1[key : key + rows * D].view(rows, D)
        ns = s[uniq] + g * g
        s[uniq] = ns
        w = w - lr * g / (ns.sqrt() + eps)
    elif opt in (3, 4, 5, 6):
        m = state1[key : key + rows * D].view(rows, D)
        mv = b1 * m[uniq] + (1 - b1) * g
        m[uniq] = mv
        if opt in (4, 6):
            vr = b2 * state2[grow] + (1 - b2) * (g * g).sum(1) / D
            state2[grow] = vr
            vv = vr.unsqueeze(1).expand_as(g)
        else:
            v = state2[key : key + rows * D].view(rows, D)
            vv = b2 * v[uniq] + (1 - b2) * g * g
            v[uniq] = vv
        bc1, bc2 = 1 - b1**step, 1 - b2**step
        upd = (mv / bc1) / ((vv / bc2).sqrt() + eps)
        lamb = opt in (5, 6)
        if lamb or wd_mode == 2:
            upd = upd + wd * w
        ratio = 1.0
        if lamb:
            un, wn = upd.norm(dim=1), w.norm(dim=1)
            ratio = torch.where((un > 0) & (wn > 0), wn / un, torch.ones_like(un)).unsqueeze(1)
        w = w - lr * ratio * upd
    elif opt == 9:
        m = state1[key : key + rows * D].view(rows, D)
        c = b1 * m[uniq] + (1 - b1) * g
        upd = torch.sign(c)
        if wd_mode == 2:
            upd = upd + wd * w
        w = w - lr * upd
        m[uniq] = b2 * m[uniq] + (1 - b2) * g
    elif opt == 7:
        eta = hyper[HP_MOMENTUM] if hyper[HP_MOMENTUM] > 0 else 0.001
        gn, wn = g.norm(dim=1), w.norm(dim=1)
        ratio = torch.where((gn > 0) & (wn > 0), eta * wn / (gn + wd * wn + eps), torch.ones_like(gn)).unsqueeze(1)
        w = w - lr * ratio * g
    if _SR_REF["on"] and table.dtype in (torch.bfloat16, torch.float16):
        table[uniq] = stochastic_round(w, table.dtype, _SR_REF["gen"])
    else:
        table[uniq] = w.to(table.dtype)


_SR_REF = {"on": False, "gen": None}  # set around the reference backward by fused_backward(stochastic_rounding=...)


def stochastic_round(x: torch.Tensor, dtype: torch.dtype, generator: Optional[torch.Generator] = None) -> torch.Tensor:
    """Unbiased rounding of fp32 ``x`` to bf16 / fp16: up with probability (x - lo) / (hi - lo) (torch mirror of the kernel's
    ``trb_sr_bf16`` / ``trb_sr_half``; FBGEMM ``stochastic_rounding=True``)."""
    x = x.float()
    if dtype == torch.bfloat16:
        bits = x.contiguous().view(torch.int32)
        noise = torch.randint(0, 1 << 16, x.shape, generator=generator, device=x.device, dtype=torch.int32)
        finite = torch.isfinite(x)
        out = torch.where(finite, (bits + noise) & ~0xFFFF, bits & ~0xFFFF)
        return out.view(torch.float32).to(torch.bfloat16)
    near = x.to(dtype)
    nf = near.float()
    other = torch.nextafter(near, torch.where(x > nf, torch.full_like(near, float("inf")), torch.full_like(near, float("-inf"))))
    span = (other.float() - nf).abs()
    pr = torch.where(span > 0, (x - nf).abs() / span, torch.zeros_like(x))
    u = torch.rand(x.shape, generator=generator, device=x.device)
    return torch.where((u < pr) & torch.isfinite(other.float()), other, near)


def _ref_fused_backward(meta, weights, state1, state2, hyper, opt, wd_mode, indices, offsets, psw, grad, B, mean, pooled=True):
    with torch.no_grad():
        for key, rows, D, rowbase, uniq, gs in _ref_row_grads(meta, indices, offsets, psw, grad, B, mean, pooled):
            _ref_apply(opt, wd_mode, hyper, weights, state1, state2, key, rows, D, rowbase, uniq, gs)


# ----------------------------------------------------------------------------------------------
# native launchers
# ----------------------------------------------------------------------------------------------
def _is64(t: torch.Tensor) -> int:
    if t.dtype == torch.int64:
        return 1
    if t.dtype == torch.int32:
        return 0
    raise TypeError(f"indices/offsets must be int32 or int64, got {t.dtype}")


def pooled_forward(
    meta: TbeMeta,
    weights: torch.Tensor,
    indices: torch.Tensor,
    offsets: torch.Tensor,
    per_sample_weights: Optional[torch.Tensor],
    B: int,
    mean: bool,
    out_dtype: torch.dtype,
    out: Optional[torch.Tensor] = None,
    out_ptrs: Optional[Sequence[int]] = None,
    out_stride: Optional[int] = None,
    B_local: Optional[int] = None,
) -> Optional[torch.Tensor]:
    """Pooled lookup. ``out_ptrs`` (peer-mapped raw pointers, one per destination rank) turns the
    call into the fused lookup + all-to-all; otherwise a local ``[B, total_cols]`` tensor is
    written/returned."""
    if not _lib.use_cuda_kernels(weights, indices):
        if out_ptrs is not None:
            raise RuntimeError("peer-pointer outputs need CUDA")
        return _ref_pooled_forward(meta, weights, indices, offsets, per_sample_weights, B, mean, out_dtype, out)
    if out_ptrs is None:
        if out is None:
            out = torch.empty(B, meta.total_cols, dtype=out_dtype, device=indices.device)
        assert out.stride(1) == 1
        out_ptrs = [out.data_ptr()]
        out_stride = out.stride(0)
        B_local = B
    assert indices.is_contiguous() and offsets.is_contiguous()
    L = _lib.lib()
    code = L.trb_tbe_pooled_fwd(
        _lib.ptr(weights), _lib.dtype_code(weights.dtype),
        _lib.ptr(meta.feat_woff), _lib.ptr(meta.feat_rows), _lib.ptr(meta.feat_dim), _lib.ptr(meta.feat_col),
        _lib.ptr(indices), _is64(indices), _lib.ptr(offsets), _is64(offsets),
        _lib.ptr(per_sample_weights), _lib.ptr_array(out_ptrs), len(out_ptrs),
        _lib.dtype_code(out_dtype), ctypes.c_int64(out_stride), B, B_local, meta.num_features,
        meta.max_dim, int(mean), _lib.stream_ptr(indices.device),
    )
    _lib.check(code, "trb_tbe_pooled_fwd")
    return out


def sequence_forward(meta: TbeMeta, weights, indices, offsets, B: int, out_dtype: torch.dtype) -> torch.Tensor:
    if not _lib.use_cuda_kernels(weights, indices):
        return _ref_seq_forward(meta, weights, indices, offsets, B, out_dtype)
    D = meta.h_dim[0] if meta.num_features else 0
    n = indices.numel()
    out = torch.empty(n, D, dtype=out_dtype, device=indices.device)
    if n == 0:
        return out
    L = _lib.lib()
    code = L.trb_tbe_seq_fwd(
        _lib.ptr(weights), _lib.dtype_code(weights.dtype), _lib.ptr(meta.feat_woff), _lib.ptr(meta.feat_rows),
        _lib.ptr(indices), _is64(indices), _lib.ptr(offsets), _is64(offsets), meta.num_features, B, D,
        _lib.ptr(out), _lib.dtype_code(out_dtype), ctypes.c_int64(n), _lib.stream_ptr(indices.device),
    )
    _lib.check(code, "trb_tbe_seq_fwd")
    return out


_WS_CACHE: Dict[Tuple[int, int], torch.Tensor] = {}


def _workspace(nbytes: int, device: torch.device) -> torch.Tensor:
    key = (device.index if device.index is not None else torch.cuda.current_device(), torch.cuda.current_stream(device).cuda_stream)
    ws = _WS_CACHE.get(key)
    if ws is None or ws.numel() < nbytes:
        with torch.inference_mode(False):  # cached across calls: must not become an inference tensor (a training step writes into it later)
            ws = torch.empty(int(nbytes * 1.25) + 1024, dtype=torch.uint8, device=device)
        _WS_CACHE[key] = ws
    return ws


def fused_backward(
    meta: TbeMeta,
    weights: torch.Tensor,
    state1: Optional[torch.Tensor],
    state2: Optional[torch.Tensor],
    hyper_dev: torch.Tensor,
    hyper_host: List[float],
    opt: int,
    wd_mode: int,
    indices: torch.Tensor,
    offsets: torch.Tensor,
    per_sample_weights: Optional[torch.Tensor],
    B: int,
    mean: bool,
    grad: Optional[torch.Tensor] = None,
    grad_ptrs: Optional[Sequence[int]] = None,
    grad_stride: Optional[int] = None,
    grad_dtype: Optional[torch.dtype] = None,
    B_local: Optional[int] = None,
    stochastic_rounding: bool = False,
    sr_seed: int = 0,
) -> None:
    """Exact fused backward + optimizer for a pooled lookup (gradient rows may live on peers). ``stochastic_rounding`` applies to
    bf16 / fp16 tables only: the updated row is rounded up or down with probability proportional to the distance."""
    if not _lib.use_cuda_kernels(weights, indices):
        assert grad is not None
        _SR_REF["on"] = bool(stochastic_rounding)
        _SR_REF["gen"] = torch.Generator().manual_seed(int(sr_seed) & 0x7FFFFFFF) if stochastic_rounding else None
        try:
            _ref_fused_backward(meta, weights, state1, state2, hyper_host, opt, wd_mode, indices, offsets, per_sample_weights, grad, B, mean)
        finally:
            _SR_REF["on"] = False
        return
    n = indices.numel()
    if n == 0:
        return
    if grad_ptrs is None:
        assert grad is not None
        if grad.stride(1) != 1:
            grad = grad.contiguous()
        grad_ptrs = [grad.data_ptr()]
        grad_stride = grad.stride(0)
        grad_dtype = grad.dtype
        B_local = B
    L = _lib.lib()
    L.trb_tbe_bwd_workspace_bytes.restype = ctypes.c_int64
    nbytes = L.trb_tbe_bwd_workspace_bytes(ctypes.c_int64(n), meta.max_dim, ctypes.c_int64(meta.total_rows))
    ws = _workspace(nbytes, indices.device)
    code = L.trb_tbe_bwd_fused_ex(
        _lib.ptr(weights), _lib.dtype_code(weights.dtype), _lib.ptr(state1), _lib.ptr(state2), _lib.ptr(hyper_dev),
        opt, wd_mode, _lib.ptr(meta.feat_woff), _lib.ptr(meta.feat_rows), _lib.ptr(meta.feat_rowbase),
        _lib.ptr(meta.feat_dim), _lib.ptr(meta.feat_col), _lib.ptr(indices), _is64(indices), _lib.ptr(offsets),
        _is64(offsets), _lib.ptr(per_sample_weights), _lib.ptr_array(grad_ptrs), len(grad_ptrs),
        _lib.dtype_code(grad_dtype), ctypes.c_int64(grad_stride), ctypes.c_int64(n), ctypes.c_int64(meta.total_rows),
        B, B_local, meta.num_features, meta.max_dim, int(mean), _lib.ptr(ws), int(bool(stochastic_rounding)), ctypes.c_uint64(int(sr_seed) & 0xFFFFFFFFFFFFFFFF),
        _lib.stream_ptr(indices.device),
    )
    _lib.check(code, "trb_tbe_bwd_fused_ex")


@dataclass
class IdRegions:
    """Ids of a lookup delivered as per-source regions of one receive slot (NVLink input dist, csrc/kjt_route.cu): source
    rank s wrote offsets ``[F_total * src_B + 1]`` (relative) at ``off_ptr + s * off_stride`` elements and its ids at
    ``idx_ptr + s * idx_stride`` elements. ``window(u0)`` moves the offsets pointer to the first feature of a kernel group."""

    idx_ptr: int
    idx64: int
    off_ptr: int
    off64: int
    psw_ptr: int
    n_src: int
    idx_stride: int
    off_stride: int
    src_B: int

    def window(self, first_feature: int) -> "IdRegions":
        esz = 8 if self.off64 else 4
        return IdRegions(self.idx_ptr, self.idx64, self.off_ptr + first_feature * self.src_B * esz, self.off64, self.psw_ptr, self.n_src, self.idx_stride,
                         self.off_stride, self.src_B)

    @property
    def positions(self) -> int:
        return self.n_src * self.idx_stride


def pooled_forward_regions(meta: TbeMeta, weights: torch.Tensor, ids: IdRegions, mean: bool, out_dtype: torch.dtype, out_ptrs: Sequence[int],
                           out_stride: int, B_local: int, device: torch.device) -> None:
    """Pooled lookup over per-source id regions, pooled rows stored into ``out_ptrs`` (one buffer per destination rank)."""
    L = _lib.lib()
    B = ids.n_src * ids.src_B
    code = L.trb_tbe_pooled_fwd_ms(
        _lib.ptr(weights), _lib.dtype_code(weights.dtype), _lib.ptr(meta.feat_woff), _lib.ptr(meta.feat_rows), _lib.ptr(meta.feat_dim), _lib.ptr(meta.feat_col),
        ctypes.c_void_p(ids.idx_ptr), ids.idx64, ctypes.c_void_p(ids.off_ptr), ids.off64, ctypes.c_void_p(ids.psw_ptr), ids.n_src,
        ctypes.c_int64(ids.idx_stride), ctypes.c_int64(ids.off_stride), _lib.ptr_array(out_ptrs), len(out_ptrs), _lib.dtype_code(out_dtype),
        ctypes.c_int64(out_stride), B, B_local, meta.num_features, meta.max_dim, int(mean), _lib.stream_ptr(device))
    _lib.check(code, "trb_tbe_pooled_fwd_ms")


def backward_workspace_bytes(n_positions: int, max_dim: int, total_rows: int) -> int:
    L = _lib.lib()
    L.trb_tbe_bwd_workspace_bytes.restype = ctypes.c_int64
    return int(L.trb_tbe_bwd_workspace_bytes(ctypes.c_int64(n_positions), max_dim, ctypes.c_int64(total_rows)))


def fused_backward_regions(meta: TbeMeta, weights: torch.Tensor, state1, state2, hyper_dev: torch.Tensor, opt: int, wd_mode: int, ids: IdRegions, mean: bool,
                           grad_ptrs: Sequence[int], grad_stride: int, grad_dtype: torch.dtype, grad_scale: float, B_local: int, workspace: torch.Tensor,
                           device: torch.device, stochastic_rounding: bool = False, sr_seed: int = 0, phase: int = 0) -> None:
    """Fused backward + optimizer over per-source id regions (gradient rows in ``grad_ptrs`` buffers, scaled by ``grad_scale``).
    ``phase`` 1 runs only the id-dependent half (key build + radix sort into ``workspace``) - callable as soon as the ids exist, on
    any stream; ``phase`` 2 runs the gradient-dependent half (run walk + optimizer) over a prepared workspace; 0 = both."""
    L = _lib.lib()
    B = ids.n_src * ids.src_B
    code = L.trb_tbe_bwd_fused_phase(
        _lib.ptr(weights), _lib.dtype_code(weights.dtype), _lib.ptr(state1), _lib.ptr(state2), _lib.ptr(hyper_dev), opt, wd_mode,
        _lib.ptr(meta.feat_woff), _lib.ptr(meta.feat_rows), _lib.ptr(meta.feat_rowbase), _lib.ptr(meta.feat_dim), _lib.ptr(meta.feat_col),
        ctypes.c_void_p(ids.idx_ptr), ids.idx64, ctypes.c_void_p(ids.off_ptr), ids.off64, ctypes.c_void_p(ids.psw_ptr), ids.n_src,
        ctypes.c_int64(ids.idx_stride), ctypes.c_int64(ids.off_stride), _lib.ptr_array(grad_ptrs), len(grad_ptrs), _lib.dtype_code(grad_dtype),
        ctypes.c_int64(grad_stride), ctypes.c_float(grad_scale), ctypes.c_int64(ids.positions), ctypes.c_int64(meta.total_rows), B, B_local,
        meta.num_features, meta.max_dim, int(mean), _lib.ptr(workspace), int(bool(stochastic_rounding)), ctypes.c_uint64(int(sr_seed) & 0xFFFFFFFFFFFFFFFF),
        int(phase), _lib.stream_ptr(device))
    _lib.check(code, "trb_tbe_bwd_fused_phase")


def psw_grad_regions(meta: TbeMeta, weights: torch.Tensor, ids: IdRegions, mean: bool, grad_ptrs: Sequence[int], grad_stride: int, grad_dtype: torch.dtype,
                     B_local: int, out: torch.Tensor) -> torch.Tensor:
    """Per-sample-weight gradient over per-source id regions; ``out`` is fp32 ``[positions]`` (position = s * idx_stride + i)."""
    L = _lib.lib()
    B = ids.n_src * ids.src_B
    code = L.trb_tbe_psw_grad_ms(
        _lib.ptr(weights), _lib.dtype_code(weights.dtype), _lib.ptr(meta.feat_woff), _lib.ptr(meta.feat_rows), _lib.ptr(meta.feat_dim), _lib.ptr(meta.feat_col),
        ctypes.c_void_p(ids.idx_ptr), ids.idx64, ctypes.c_void_p(ids.off_ptr), ids.off64, ids.n_src, ctypes.c_int64(ids.idx_stride),
        ctypes.c_int64(ids.off_stride), _lib.ptr_array(grad_ptrs), len(grad_ptrs), _lib.dtype_code(grad_dtype), ctypes.c_int64(grad_stride), _lib.ptr(out),
        B, B_local, meta.num_features, meta.max_dim, int(mean), _lib.stream_ptr(out.device))
    _lib.check(code, "trb_tbe_psw_grad_ms")
    return out


def psw_grad(meta: TbeMeta, weights: torch.Tensor, indices: torch.Tensor, offsets: torch.Tensor, B: int, mean: bool, grad: Optional[torch.Tensor] = None,
             grad_ptrs: Optional[Sequence[int]] = None, grad_stride: Optional[int] = None, grad_dtype: Optional[torch.dtype] = None,
             B_local: Optional[int] = None) -> torch.Tensor:
    """Gradient of the pooled lookup w.r.t. per-sample weights: ``d psw[i] = <grad[bag(i)], W[idx[i]]>`` (fp32 ``[n]``).
    Call BEFORE ``fused_backward`` (which updates the rows in place). csrc/tbe_psw_grad.cu."""
    n = indices.numel()
    if not _lib.use_cuda_kernels(weights, indices):
        assert grad is not None
        out = torch.zeros(n, dtype=torch.float32, device=weights.device)
        off = offsets.to(torch.int64)
        for f in range(meta.num_features):
            o = off[f * B : (f + 1) * B + 1]
            lo, hi = int(o[0]), int(o[-1])
            if hi <= lo:
                continue
            D, col, rows = meta.h_dim[f], meta.h_col[f], meta.h_rows[f]
            lengths = o[1:] - o[:-1]
            b = torch.repeat_interleave(torch.arange(B, device=off.device), lengths, output_size=hi - lo)
            idx = indices[lo:hi].long()
            ok = (idx >= 0) & (idx < rows)
            w = weights[meta.h_woff[f] : meta.h_woff[f] + rows * D].view(rows, D)[idx.clamp(0, rows - 1)].float()
            v = (w * grad[b, col : col + D].float()).sum(1) * ok
            if mean:
                v = v / lengths[b].clamp(min=1).float()
            out[lo:hi] = v
        return out
    out = torch.zeros(n, dtype=torch.float32, device=indices.device)
    if n == 0:
        return out
    if grad_ptrs is None:
        assert grad is not None
        if grad.stride(1) != 1:
            grad = grad.contiguous()
        grad_ptrs, grad_stride, grad_dtype, B_local = [grad.data_ptr()], grad.stride(0), grad.dtype, B
    L = _lib.lib()
    code = L.trb_tbe_psw_grad(_lib.ptr(weights), _lib.dtype_code(weights.dtype), _lib.ptr(meta.feat_woff), _lib.ptr(meta.feat_rows), _lib.ptr(meta.feat_dim),
                              _lib.ptr(meta.feat_col), _lib.ptr(indices), _is64(indices), _lib.ptr(offsets), _is64(offsets), _lib.ptr_array(grad_ptrs),
                              len(grad_ptrs), _lib.dtype_code(grad_dtype), ctypes.c_int64(grad_stride), _lib.ptr(out), B, B_local, meta.num_features,
                              meta.max_dim, int(mean), _lib.stream_ptr(indices.device))
    _lib.check(code, "trb_tbe_psw_grad")
    return out


def sequence_backward(meta, weights, state1, state2, hyper_dev, hyper_host, opt, wd_mode, indices, offsets, B, grad, stochastic_rounding: bool = False, sr_seed: int = 0):
    """Backward of the unpooled lookup: position i contributes grad[i] to row indices[i].
    Expressed as a pooled backward with one bag per position (column offset 0, stride D)."""
    if not _lib.use_cuda_kernels(weights, indices):
        _SR_REF["on"] = bool(stochastic_rounding)
        _SR_REF["gen"] = torch.Generator().manual_seed(int(sr_seed) & 0x7FFFFFFF) if stochastic_rounding else None
        try:
            _ref_fused_backward(meta, weights, state1, state2, hyper_host, opt, wd_mode, indices, offsets, None, grad, B, False, pooled=False)
        finally:
            _SR_REF["on"] = False
        return
    n = indices.numel()
    if n == 0:
        return
    # Per-position bags: feature f owns positions [offsets[f*B], offsets[(f+1)*B]); build a
    # [F * n + 1] offsets array where bag (f, i) is non-empty only if position i belongs to f.
    F = meta.num_features
    off = offsets.to(torch.int64)
    fstart = off[torch.arange(0, F + 1, device=off.device) * B]  # [F+1]
    pos = torch.arange(n + 1, device=off.device, dtype=torch.int64)
    bag_off = torch.minimum(torch.maximum(pos.unsqueeze(0), fstart[:-1].unsqueeze(1)), fstart[1:].unsqueeze(1))
    # rows: f, cols: position boundary -> flatten as F bags-of-n with shared final sentinel
    flat = torch.cat([bag_off[:, :-1].reshape(-1), fstart[-1:].reshape(1)]).contiguous()
    seq_meta = meta.with_cols([0] * F, meta.h_dim[0])
    fused_backward(seq_meta, weights, state1, state2, hyper_dev, hyper_host, opt, wd_mode, indices, flat, None, n, False, grad=grad.contiguous(),
                   stochastic_rounding=stochastic_rounding, sr_seed=sr_seed)


# ----------------------------------------------------------------------------------------------
# nn.Module front-end
# ----------------------------------------------------------------------------------------------
class _PooledLookupFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, dummy, tbe: "TableBatchedEmbeddingBags", indices, offsets, psw, B):
        ctx.tbe = tbe
        ctx.B = B
        ctx.save_for_backward(indices, offsets, psw)
        return pooled_forward(tbe.meta, tbe.weights, indices, offsets, psw, B, tbe.pooling_mode == PoolingMode.MEAN, tbe.output_dtype)

    @staticmethod
    def backward(ctx, grad):
        indices, offsets, psw = ctx.saved_tensors
        tbe = ctx.tbe
        if tbe.__dict__.get("_fs") is not None:
            tbe._fs.before_backward()
        gpsw = None
        if psw is not None and ctx.needs_input_grad[4]:
            # windowed offsets (engine groups) index into the full values tensor: the gradient is positional
            gpsw = psw_grad(tbe.meta, tbe.weights.detach(), indices, offsets, ctx.B, tbe.pooling_mode == PoolingMode.MEAN, grad=grad).to(psw.dtype)
        dense = tbe._backward(indices, offsets, psw, grad, ctx.B)
        return dense, None, None, None, gpsw, None


class _SeqLookupFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, dummy, tbe: "TableBatchedEmbeddingBags", indices, offsets, B):
        ctx.tbe = tbe
        ctx.B = B
        ctx.save_for_backward(indices, offsets)
        return sequence_forward(tbe.meta, tbe.weights, indices, offsets, B, tbe.output_dtype)

    @staticmethod
    def backward(ctx, grad):
        indices, offsets = ctx.saved_tensors
        if ctx.tbe.__dict__.get("_fs") is not None:
            ctx.tbe._fs.before_backward()
        dense = ctx.tbe._backward_seq(indices, offsets, grad, ctx.B)
        return dense, None, None, None, None


class TableBatchedEmbeddingBags(nn.Module):
    """Many embedding tables in one flat buffer with a single-launch lookup and a fused optimizer.

    Args mirror what the reference hands to FBGEMM (batched_embedding_kernel.py:3744-3765):
    ``embedding_specs`` = [(rows, dim)], ``feature_table_map`` maps each feature to its table.
    With ``optimizer=OptimType.NONE`` the module behaves like the dense TBE: ``weights.grad`` is
    produced for an external optimizer / DDP.
    """

    def __init__(
        self,
        embedding_specs: Sequence[Tuple[int, int]],
        feature_table_map: Optional[Sequence[int]] = None,
        pooling_mode: PoolingMode = PoolingMode.SUM,
        weights_precision: torch.dtype = torch.float32,
        output_dtype: torch.dtype = torch.float32,
        optimizer: OptimType = OptimType.EXACT_SGD,
        learning_rate: float = 0.01,
        eps: float = 1.0e-8,
        beta1: float = 0.9,
        beta2: float = 0.999,
        weight_decay: float = 0.0,
        weight_decay_mode: WeightDecayMode = WeightDecayMode.NONE,
        max_gradient: float = 0.0,
        momentum: float = 0.0,
        device: Optional[torch.device] = None,
        table_names: Optional[Sequence[str]] = None,
        location: "EmbeddingLocation" = None,  # type: ignore[assignment]
        stochastic_rounding: bool = True,
        sr_seed: int = 0,
    ) -> None:
        super().__init__()
        # FBGEMM default: low-precision (fp16 / bf16) tables are updated with stochastic rounding; no effect on fp32 tables
        self.stochastic_rounding = bool(stochastic_rounding) and weights_precision in (torch.float16, torch.bfloat16)
        self._sr_seed, self._sr_calls = int(sr_seed), 0
        device = torch.device(device) if device is not None else torch.device("cpu")
        self.embedding_specs = [(int(r), int(d)) for r, d in embedding_specs]
        self.feature_table_map = list(feature_table_map) if feature_table_map is not None else list(range(len(self.embedding_specs)))
        self.pooling_mode = PoolingMode(pooling_mode)
        self.output_dtype = output_dtype
        self.optimizer = optimizer
        if optimizer == OptimType.ADAMW:
            weight_decay_mode = WeightDecayMode.DECOUPLE
        self.opt_code = _OPT_CODE[optimizer]
        self.weight_decay_mode = WeightDecayMode(weight_decay_mode)
        self.location = EmbeddingLocation(location) if location is not None else (EmbeddingLocation.HOST if torch.device(device or "cpu").type == "cpu" else EmbeddingLocation.DEVICE)
        self.table_names = list(table_names) if table_names is not None else [f"t{i}" for i in range(len(self.embedding_specs))]
        rows = [r for r, _ in self.embedding_specs]
        dims = [d for _, d in self.embedding_specs]
        self._is_meta = device.type == "meta"
        total = sum(r * d for r, d in self.embedding_specs)
        self.total_rows = sum(rows)
        dense = optimizer == OptimType.NONE
        if dense:
            self.weights = nn.Parameter(torch.empty(total, dtype=weights_precision, device=device), requires_grad=True)
        else:
            # fused tables are updated in-kernel: a plain buffer, never seen by autograd / DDP / dense optimizers
            self.register_buffer("weights", self._alloc(total, weights_precision, device, big=True), persistent=False)
        self._dummy = nn.Parameter(torch.zeros(1, device=device if not self._is_meta else "cpu"), requires_grad=True) if not dense else None
        if not self._is_meta:
            self.meta = TbeMeta.build(rows, dims, self.feature_table_map, device)
        k1, k2 = _OPT_STATE[self.opt_code]
        # element-wise optimizer state follows the weights' location; row-wise state (4 B / row) stays in HBM
        mk = lambda kind: None if kind is None else (torch.zeros(self.total_rows, dtype=torch.float32, device=device) if kind == "row"
                                                     else self._alloc(total, torch.float32, device, big=True).zero_())
        self.register_buffer("state1", mk(k1), persistent=False)
        self.register_buffer("state2", mk(k2), persistent=False)
        self._state_kinds = (k1, k2)
        self.hyper_host = [learning_rate, eps, beta1, beta2, weight_decay, 0.0, max_gradient, momentum]
        hdev = torch.tensor(self.hyper_host, dtype=torch.float32, device=device if not self._is_meta else "cpu")
        self.register_buffer("hyper_dev", hdev, persistent=False)
        self._hyper_pinned: Optional[torch.Tensor] = None
        self._auto_step = True
        if not self._is_meta:
            self.init_parameters()

    def _alloc(self, n: int, dtype: torch.dtype, device: torch.device, big: bool) -> torch.Tensor:
        if big and self.location == EmbeddingLocation.MANAGED and device.type == "cuda":
            return torch.empty(n, dtype=dtype, pin_memory=True)  # UVA: the same pointer is valid inside kernels
        return torch.empty(n, dtype=dtype, device=device)

    def _apply(self, fn, recurse: bool = True):
        """``.to(device)`` / ``.cuda()`` must not drag zero-copy host tables into HBM."""
        if self.location != EmbeddingLocation.MANAGED:
            return super()._apply(fn, recurse)
        keep = {k: self._buffers[k] for k in ("weights", "state1", "state2") if self._buffers.get(k) is not None and not self._buffers[k].is_cuda}
        for k in keep:
            self._buffers[k] = None
        super()._apply(fn, recurse)
        for k, v in keep.items():
            self._buffers[k] = v
        return self

    # ---- parameters -------------------------------------------------------------------------
    @torch.no_grad()
    def init_parameters(self, init_ranges: Optional[Sequence[Tuple[float, float]]] = None) -> None:
        for t, w in enumerate(self.split_embedding_weights()):
            rows = self.embedding_specs[t][0]
            lo, hi = init_ranges[t] if init_ranges is not None else (-math.sqrt(1.0 / max(rows, 1)), math.sqrt(1.0 / max(rows, 1)))
            if w.dtype == torch.float32:
                w.uniform_(lo, hi)
            else:
                w.copy_(torch.empty(w.shape, dtype=torch.float32, device=w.device).uniform_(lo, hi))

    def split_embedding_weights(self) -> List[torch.Tensor]:
        out, o = [], 0
        for r, d in self.embedding_specs:
            out.append(self.weights.detach()[o : o + r * d].view(r, d))
            o += r * d
        return out

    def split_optimizer_states(self) -> List[Dict[str, torch.Tensor]]:
        """Per table {state name: tensor view} (row-wise states are 1-D [rows])."""
        names = _OPT_STATE_NAMES.get(self.opt_code, (None, None))
        res: List[Dict[str, torch.Tensor]] = []
        eo = ro = 0
        for r, d in self.embedding_specs:
            st: Dict[str, torch.Tensor] = {}
            for buf, kind, name in ((self.state1, self._state_kinds[0], names[0]), (self.state2, self._state_kinds[1], names[1])):
                if buf is None or name is None:
                    continue
                st[name] = buf[ro : ro + r] if kind == "row" else buf[eo : eo + r * d].view(r, d)
            res.append(st)
            eo += r * d
            ro += r
        return res

    # ---- hyper-parameters -------------------------------------------------------------------
    def _push_hyper(self) -> None:
        if self.hyper_dev.is_cuda:
            if self._hyper_pinned is None:
                self._hyper_pinned = torch.empty(8, dtype=torch.float32).pin_memory()
            self._hyper_pinned.copy_(torch.tensor(self.hyper_host, dtype=torch.float32))
            self.hyper_dev.copy_(self._hyper_pinned, non_blocking=True)
        else:
            self.hyper_dev.copy_(torch.tensor(self.hyper_host, dtype=torch.float32))

    def set_learning_rate(self, lr: float) -> None:
        if self.hyper_host[HP_LR] != lr:
            self.hyper_host[HP_LR] = float(lr)
            self._push_hyper()

    def get_learning_rate(self) -> float:
        return self.hyper_host[HP_LR]

    def set_optimizer_step(self, step: int) -> None:
        self.hyper_host[HP_STEP] = float(step)
        self._push_hyper()

    def _needs_step(self) -> bool:
        return self.opt_code in (3, 4, 5, 6)

    # ---- forward / backward -----------------------------------------------------------------
    def forward(self, indices: torch.Tensor, offsets: torch.Tensor, per_sample_weights: Optional[torch.Tensor] = None, batch_size: Optional[int] = None) -> torch.Tensor:
        F = len(self.feature_table_map)
        B = batch_size if batch_size is not None else (offsets.numel() - 1) // max(F, 1)
        anchor = self.weights if self._dummy is None else self._dummy
        fs = self.__dict__.get("_fs")  # FULLY_SHARDED 2D strategy (parallel/fully_sharded.py): full weights only around the kernels
        if fs is not None:
            fs.before_forward()
        if self.pooling_mode == PoolingMode.NONE:
            out = _SeqLookupFn.apply(anchor, self, indices, offsets, B)
        else:
            out = _PooledLookupFn.apply(anchor, self, indices, offsets, per_sample_weights, B)
        if fs is not None and torch.is_grad_enabled():
            fs.after_forward()
        return out

    def next_sr_seed(self) -> int:
        """Seed of the next backward's rounding noise (changes every call, reproducible for a given ``sr_seed``)."""
        self._sr_calls += 1
        return (self._sr_seed * 0x9E3779B1 + self._sr_calls * 0x85EBCA77) & 0xFFFFFFFFFFFF

    def _pre_update(self) -> None:
        if self._needs_step() and self._auto_step:
            self.hyper_host[HP_STEP] += 1.0
            self._push_hyper()

    def _backward(self, indices, offsets, psw, grad, B) -> Optional[torch.Tensor]:
        mean = self.pooling_mode == PoolingMode.MEAN
        if self.opt_code == 8:
            gw = torch.zeros(self.weights.numel(), dtype=torch.float32, device=self.weights.device)
            fused_backward(self.meta, self.weights.detach(), gw, None, self.hyper_dev, self.hyper_host, 8, 0, indices, offsets, psw, B, mean, grad=grad)
            return gw.to(self.weights.dtype)
        self._pre_update()
        fused_backward(self.meta, self.weights.detach(), self.state1, self.state2, self.hyper_dev, self.hyper_host, self.opt_code, int(self.weight_decay_mode), indices, offsets, psw, B, mean, grad=grad,
                       stochastic_rounding=self.stochastic_rounding, sr_seed=self.next_sr_seed())
        return torch.zeros_like(self._dummy)

    def _backward_seq(self, indices, offsets, grad, B) -> Optional[torch.Tensor]:
        if self.opt_code == 8:
            gw = torch.zeros(self.weights.numel(), dtype=torch.float32, device=self.weights.device)
            sequence_backward(self.meta, self.weights.detach(), gw, None, self.hyper_dev, self.hyper_host, 8, 0, indices, offsets, B, grad)
            return gw.to(self.weights.dtype)
        self._pre_update()
        sequence_backward(self.meta, self.weights.detach(), self.state1, self.state2, self.hyper_dev, self.hyper_host, self.opt_code, int(self.weight_decay_mode), indices, offsets, B, grad,
                          stochastic_rounding=self.stochastic_rounding, sr_seed=self.next_sr_seed())
        return torch.zeros_like(self._dummy)
