"""Variable batch per feature (VBE): padding to a uniform batch, the inverse-index expansion of the pooled rows and its gradient.

A VBE ``KeyedJaggedTensor`` carries ``B_f`` de-duplicated bags for feature ``f`` and ``inverse_indices = (keys, [R, B])``: sample
``b`` uses bag ``inv[r(f), b]``. ``pad_offsets`` appends empty bags so the lookup kernels see an ordinary uniform batch,
``vbe_expand`` computes ``out[b, cols(f)] = pooled[inv[r(f), b], cols(f)]`` and, backward, the segmented sum over the samples that
referenced each bag. On CUDA these are the kernels of ``csrc/vbe.cu`` (one launch forward; a sorted transpose of the inverse indices
and a deterministic reduce backward); on the CPU, and for layouts the kernels do not serve (column blocks that are not multiples of
16 bytes, dtypes other than bf16 / fp32), the per-name ``index_select`` formulation ``expand_eager`` runs. The choice is made from
the tensors alone.
"""
from __future__ import annotations

import ctypes
from typing import TYPE_CHECKING, Dict, List, Optional, Sequence, Tuple

import torch

from . import _lib

if TYPE_CHECKING:
    from ..sparse.jagged_tensor import KeyedJaggedTensor

_KERNEL_DTYPES = (torch.bfloat16, torch.float32)


def pad_offsets(kjt: "KeyedJaggedTensor", B: int) -> "KeyedJaggedTensor":
    """Variable batch per feature -> uniform stride ``B`` (>= every ``B_f``) by appending empty bags; values and weights untouched."""
    from ..sparse.jagged_tensor import KeyedJaggedTensor

    spk = kjt.stride_per_key()
    F = len(spk)
    assert all(b <= B for b in spk), f"cannot pad per-feature batch sizes {spk} to {B}"
    off = kjt.offsets()
    sizes = torch.tensor(spk, dtype=torch.int32)
    if F * B == 0:
        out = off.new_zeros(1)
    elif _lib.use_cuda_kernels(off):
        # the batch sizes are host data: one pinned, non-blocking copy
        sizes = sizes.pin_memory().to(off.device, non_blocking=True)
        out = torch.empty(F * B + 1, dtype=off.dtype, device=off.device)
        code = _lib.lib().trb_vbe_pad_offsets(_lib.ptr(off), int(off.dtype == torch.int64), _lib.ptr(sizes), F, ctypes.c_int64(B), _lib.ptr(out),
                                              _lib.stream_ptr(off.device))
        _lib.check(code, "trb_vbe_pad_offsets")
    else:
        sizes = sizes.long()
        base = torch.cumsum(sizes, 0) - sizes
        pos = base.unsqueeze(1) + torch.minimum(torch.arange(B).unsqueeze(0), sizes.unsqueeze(1))
        out = torch.cat([off[pos.reshape(-1).to(off.device)], off[-1:]])
    return KeyedJaggedTensor(keys=kjt.keys(), values=kjt.values(), weights=kjt.weights_or_none(), offsets=out, stride=B)


def expand_eager(pooled: torch.Tensor, inverse_indices: Tuple[List[str], torch.Tensor], names: Sequence[str], dims: Sequence[int]) -> torch.Tensor:
    """``out[b, cols(name)] = pooled[inv[row(feature of name), b], cols(name)]``, one ``index_select`` per embedding name (reference
    embeddingbag.py:405 / VariableBatchPooledEmbeddingsAllToAll semantics). Names whose feature has no inverse row pass through."""
    keys, idx = inverse_indices
    row = {k: i for i, k in enumerate(keys)}
    outs = []
    c = 0
    for name, d in zip(names, dims):
        feat = name.split("@")[0]
        outs.append(pooled[:, c : c + d].index_select(0, idx[row[feat]].long()) if feat in row else pooled[:, c : c + d])
        c += d
    return torch.cat(outs, dim=1)


class _ColTable:
    """Static maps between 16-byte column vectors and inverse rows: ``col_row[v]`` (-1 = identity) and its transpose."""

    def __init__(self, keys: Sequence[str], names: Sequence[str], dims: Sequence[int], esz: int, device: torch.device) -> None:
        per = 16 // esz
        row = {k: i for i, k in enumerate(keys)}
        col_row: List[int] = []
        vecs: List[List[int]] = [[] for _ in keys]
        for name, d in zip(names, dims):
            r = row.get(name.split("@")[0], -1)
            if r >= 0:
                vecs[r].extend(range(len(col_row), len(col_row) + d // per))
            col_row.extend([r] * (d // per))
        self.cols_vec = len(col_row)
        self.has_identity = -1 in col_row
        self.max_nv = max((len(v) for v in vecs), default=0)
        off = [0]
        for v in vecs:
            off.append(off[-1] + len(v))
        self.col_row = torch.tensor(col_row, dtype=torch.int32, device=device)
        self.row_vec_off = torch.tensor(off, dtype=torch.int32, device=device)
        self.row_vecs = torch.tensor([x for v in vecs for x in v], dtype=torch.int32, device=device)


class VbeIndex:
    """What the expansion of one batch needs: the inverse indices, the static column -> inverse-row table of the collection and (built
    once per batch, ids only) the CSR transpose of the inverse indices that the gradient reduce walks. ``tables`` is the cache of
    column tables of the collection that owns ``names`` and ``dims`` (they are static per inverse-key order, element size and
    device); without one the table lives as long as this index."""

    def __init__(self, inverse_indices: Tuple[List[str], torch.Tensor], names: Sequence[str], dims: Sequence[int], src_rows: int,
                 tables: Optional[Dict[Tuple, _ColTable]] = None) -> None:
        keys, inv = inverse_indices
        self.inverse_indices = inverse_indices
        self.keys = tuple(keys)
        self.inv = inv if inv.is_contiguous() else inv.contiguous()
        self.names, self.dims = tuple(names), tuple(dims)
        self.R, self.B = int(inv.shape[0]), int(inv.shape[1])
        self.S = int(src_rows)
        self._csr: Optional[Tuple[torch.Tensor, torch.Tensor, torch.Tensor]] = None
        self._tables: Dict[Tuple, _ColTable] = tables if tables is not None else {}

    def record_stream(self, stream: torch.Stream) -> None:
        """The index is built on the stream of the input dist and read, forward and backward, on the compute stream ``stream``: keep
        the inverse indices and the CSR out of the allocator's hands until that stream is done with them."""
        if self.inv.is_cuda:
            self.inv.record_stream(stream)
            for t in self._csr or ():
                t.record_stream(stream)

    def col_table(self, esz: int) -> Optional[_ColTable]:
        """The table for elements of ``esz`` bytes; None when an embedding column block is not a whole number of 16-byte vectors."""
        if any((d * esz) % 16 for d in self.dims):
            return None
        key = (self.keys, esz, str(self.inv.device))
        t = self._tables.get(key)
        if t is None:
            t = self._tables[key] = _ColTable(self.keys, self.names, self.dims, esz, self.inv.device)
        return t

    def kernels_serve(self, pooled: torch.Tensor) -> Optional[_ColTable]:
        """The column table when the native kernels run this expansion, else None (the eager formulation runs)."""
        if not (pooled.is_cuda and self.inv.device == pooled.device and _lib.use_cuda_kernels(pooled)):
            return None
        if pooled.dtype not in _KERNEL_DTYPES or pooled.dim() != 2 or self.inv.dtype not in (torch.int32, torch.int64) or self.R == 0:
            return None
        if pooled.shape[1] != sum(self.dims) or pooled.shape[0] != self.S or self.S == 0:
            return None
        t = self.col_table(pooled.element_size())
        if t is None or (t.has_identity and self.S != self.B):
            return None
        return t

    @torch.no_grad()
    def csr(self) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """(seg_off ``[R * S + 1]``, seg_b ``[R * B]``, long-segment lists): segment ``r * S + u`` holds, ascending, the samples ``b`` with
        ``inv[r, b] == u``."""
        if self._csr is None:
            L = _lib.lib()
            L.trb_vbe_csr_workspace_bytes.restype = ctypes.c_int64
            L.trb_vbe_long_list_elems.restype = ctypes.c_int64
            R, B = ctypes.c_int64(self.R), ctypes.c_int64(self.B)
            ws_bytes, n_list = int(L.trb_vbe_csr_workspace_bytes(R, B)), int(L.trb_vbe_long_list_elems(R, B))
            _lib.check(min(ws_bytes, n_list, 0), "trb_vbe_csr_workspace_bytes")
            dev = self.inv.device
            seg_off = torch.empty(self.R * self.S + 1, dtype=torch.int32, device=dev)
            seg_b = torch.empty(self.R * self.B, dtype=torch.int32, device=dev)
            lists = torch.empty(n_list, dtype=torch.int32, device=dev)
            ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
            code = L.trb_vbe_csr(_lib.ptr(self.inv), int(self.inv.dtype == torch.int64), R, B, ctypes.c_int64(self.S), _lib.ptr(seg_off), _lib.ptr(seg_b),
                                 _lib.ptr(lists), _lib.ptr(ws), ctypes.c_int64(ws_bytes), _lib.stream_ptr(dev))
            _lib.check(code, "trb_vbe_csr")
            self._csr = (seg_off, seg_b, lists)
        return self._csr


class _VbeExpandFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, pooled: torch.Tensor, index: VbeIndex, table: _ColTable) -> torch.Tensor:
        pooled = pooled.contiguous()
        out = torch.empty(index.B, pooled.shape[1], dtype=pooled.dtype, device=pooled.device)
        code = _lib.lib().trb_vbe_expand(_lib.ptr(pooled), _lib.ptr(out), _lib.ptr(table.col_row), _lib.ptr(index.inv), int(index.inv.dtype == torch.int64),
                                         ctypes.c_int64(index.B), ctypes.c_int64(index.S), table.cols_vec, _lib.stream_ptr(pooled.device))
        _lib.check(code, "trb_vbe_expand")
        ctx.index, ctx.table = index, table
        return out

    @staticmethod
    def backward(ctx, grad: torch.Tensor):
        index, table = ctx.index, ctx.table
        grad = grad.contiguous()
        seg_off, seg_b, lists = index.csr()
        L = _lib.lib()
        L.trb_vbe_reduce_workspace_bytes.restype = ctypes.c_int64
        R, B = ctypes.c_int64(index.R), ctypes.c_int64(index.B)
        ws_bytes = int(L.trb_vbe_reduce_workspace_bytes(R, B, table.max_nv))
        _lib.check(min(ws_bytes, 0), "trb_vbe_reduce_workspace_bytes")
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=grad.device)
        out = torch.empty(index.S, grad.shape[1], dtype=grad.dtype, device=grad.device)
        code = L.trb_vbe_reduce(_lib.ptr(grad), _lib.ptr(out), _lib.dtype_code(grad.dtype), _lib.ptr(table.col_row), _lib.ptr(table.row_vec_off),
                                _lib.ptr(table.row_vecs), table.max_nv, _lib.ptr(seg_off), _lib.ptr(seg_b), _lib.ptr(lists), R, B, ctypes.c_int64(index.S),
                                table.cols_vec, _lib.ptr(ws), ctypes.c_int64(ws_bytes), _lib.stream_ptr(grad.device))
        _lib.check(code, "trb_vbe_reduce")
        return out, None, None


def vbe_expand(pooled: torch.Tensor, index: VbeIndex) -> torch.Tensor:
    """Undo the de-duplication of a VBE batch: ``[S, sum D]`` pooled rows -> ``[B, sum D]`` per-sample rows (differentiable)."""
    table = index.kernels_serve(pooled)
    if table is None:
        return expand_eager(pooled, index.inverse_indices, index.names, index.dims)
    return _VbeExpandFn.apply(pooled, index, table)
