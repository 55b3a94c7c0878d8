"""Jagged / sparse utility ops (the ``torch.ops.fbgemm.*`` sparse-op surface the reference uses,
SURVEY §2.4(b)), implemented for both CPU (PyTorch reference) and CUDA (sm_90a kernels in
``csrc/jagged_ops.cu`` where a hot path needs one; composition of stream-ordered torch ops
otherwise). No op here performs a hidden host sync unless its output size is data dependent and
the caller did not pass it.
"""
from __future__ import annotations

import ctypes
from typing import Dict, List, Optional, Sequence, Tuple

import torch

from . import _lib


def asynchronous_complete_cumsum(x: torch.Tensor) -> torch.Tensor:
    """[n] -> [n+1] exclusive prefix sum with the total appended (works on 1-D or 2-D rows)."""
    if x.dim() == 1:
        out = x.new_zeros(x.numel() + 1)
        torch.cumsum(x, 0, out=out[1:])
        return out
    out = x.new_zeros(x.shape[0], x.shape[1] + 1)
    torch.cumsum(x, 1, out=out[:, 1:])
    return out


def asynchronous_inclusive_cumsum(x: torch.Tensor) -> torch.Tensor:
    return torch.cumsum(x, 0)


def asynchronous_exclusive_cumsum(x: torch.Tensor) -> torch.Tensor:
    return torch.cumsum(x, 0) - x


def offsets_range(offsets: torch.Tensor, range_size: int) -> torch.Tensor:
    """arange restarting at every segment start: positions of each element inside its segment."""
    if range_size == 0:
        return offsets.new_zeros(0)
    starts = offsets
    ends = torch.cat([offsets[1:], offsets.new_tensor([range_size])])
    seg_start = torch.repeat_interleave(starts, ends - starts, output_size=range_size)
    return torch.arange(range_size, device=offsets.device, dtype=offsets.dtype) - seg_start


def invert_permute(permute: torch.Tensor) -> torch.Tensor:
    inv = torch.empty_like(permute)
    inv[permute.long()] = torch.arange(permute.numel(), device=permute.device, dtype=permute.dtype)
    return inv


def segment_sum_csr(batch_size: int, csr_seg: torch.Tensor, values: torch.Tensor) -> torch.Tensor:
    """Sum ``values`` over segments given by offsets ``csr_seg`` counted in units of ``batch_size`` rows."""
    if values.is_cuda and _lib.available() and values.dtype in (torch.float32, torch.int64, torch.int32) and csr_seg.dtype in (torch.int32, torch.int64) \
            and values.is_contiguous() and csr_seg.is_contiguous():
        n_seg = csr_seg.numel() - 1
        out = torch.empty(n_seg, dtype=values.dtype, device=values.device)
        code = _lib.lib().trb_segment_sum_csr(_lib.ptr(values), _lib.dtype_code(values.dtype), _lib.ptr(csr_seg), int(csr_seg.dtype == torch.int64), _lib.ptr(out),
                                              ctypes.c_int64(n_seg), int(batch_size), _lib.stream_ptr(values.device))
        _lib.check(code, "trb_segment_sum_csr")
        return out
    seg_off = csr_seg.long() * batch_size
    lengths = seg_off[1:] - seg_off[:-1]
    seg = torch.repeat_interleave(torch.arange(lengths.numel(), device=values.device), lengths, output_size=values.numel())
    out = torch.zeros(lengths.numel(), dtype=values.dtype, device=values.device)
    out.index_add_(0, seg, values)
    return out


def _segment_gather_index(in_starts: torch.Tensor, seg_lengths: torch.Tensor, total: int) -> torch.Tensor:
    """Index tensor that concatenates ranges [in_starts[k], in_starts[k]+seg_lengths[k])."""
    out_off = torch.cumsum(seg_lengths, 0) - seg_lengths
    seg = torch.repeat_interleave(torch.arange(seg_lengths.numel(), device=seg_lengths.device), seg_lengths, output_size=total)
    return in_starts[seg] + (torch.arange(total, device=seg_lengths.device) - out_off[seg])


def permute_2D_sparse_data(
    permute: torch.Tensor,
    lengths: torch.Tensor,
    values: torch.Tensor,
    weights: Optional[torch.Tensor] = None,
    permuted_lengths_sum: Optional[int] = None,
) -> Tuple[torch.Tensor, torch.Tensor, Optional[torch.Tensor]]:
    """Permute the rows (features) of a [F, B] jagged layout. ``permute`` may repeat / drop rows."""
    F, B = lengths.shape
    if _lib.use_cuda_kernels(values) and values.numel() > 0 and permuted_lengths_sum is not None:
        return _permute_2d_cuda(permute, lengths, values, weights, permuted_lengths_sum)
    perm = permute.long()
    out_lengths = lengths[perm]
    len_per_key = lengths.sum(1)
    in_key_off = torch.cumsum(len_per_key, 0) - len_per_key
    out_len_per_key = len_per_key[perm]
    total = int(out_len_per_key.sum()) if permuted_lengths_sum is None else permuted_lengths_sum
    if total == 0:
        return out_lengths, values.new_zeros((0,) + tuple(values.shape[1:])), (None if weights is None else weights.new_zeros((0,) + tuple(weights.shape[1:])))
    idx = _segment_gather_index(in_key_off[perm], out_len_per_key, total)
    return out_lengths, values[idx], (None if weights is None else weights[idx])


def _permute_2d_cuda(permute, lengths, values, weights, total):
    F, B = lengths.shape
    P = permute.numel()
    L = _lib.lib()
    lengths = lengths.contiguous()
    permute = permute.to(torch.int32).contiguous()
    out_lengths = torch.empty(P, B, dtype=lengths.dtype, device=lengths.device)
    in_off = asynchronous_complete_cumsum(lengths.view(-1).to(torch.int64))
    out_values = torch.empty(total, dtype=values.dtype, device=values.device)
    out_weights = None if weights is None else torch.empty(total, dtype=weights.dtype, device=weights.device)
    # out lengths + out offsets
    out_lengths.copy_(lengths[permute.long()])
    out_off = asynchronous_complete_cumsum(out_lengths.view(-1).to(torch.int64))
    code = L.trb_permute_2d_data(
        _lib.ptr(permute), P, B, _lib.ptr(in_off), _lib.ptr(out_off),
        _lib.ptr(values), _lib.ptr(out_values), values.element_size(),
        _lib.ptr(weights), _lib.ptr(out_weights), 0 if weights is None else weights.element_size(),
        _lib.stream_ptr(values.device),
    )
    _lib.check(code, "trb_permute_2d_data")
    return out_lengths, out_values, out_weights


def permute_1D_sparse_data(
    permute: torch.Tensor,
    lengths: torch.Tensor,
    values: torch.Tensor,
    weights: Optional[torch.Tensor] = None,
    permuted_lengths_sum: Optional[int] = None,
) -> Tuple[torch.Tensor, torch.Tensor, Optional[torch.Tensor]]:
    """Permute variable-length segments of a 1-D jagged array."""
    perm = permute.long()
    out_lengths = lengths[perm]
    in_off = torch.cumsum(lengths, 0) - lengths
    total = int(out_lengths.sum()) if permuted_lengths_sum is None else permuted_lengths_sum
    if total == 0:
        return out_lengths, values.new_zeros((0,) + tuple(values.shape[1:])), (None if weights is None else weights.new_zeros((0,) + tuple(weights.shape[1:])))
    idx = _segment_gather_index(in_off[perm], out_lengths, total)
    return out_lengths, values[idx], (None if weights is None else weights[idx])


def expand_into_jagged_permute(permute: torch.Tensor, input_offsets: torch.Tensor, output_offsets: torch.Tensor, output_size: int) -> torch.Tensor:
    in_len = input_offsets[1:] - input_offsets[:-1]
    perm = permute.long()
    seg_len = in_len[perm]
    return _segment_gather_index(input_offsets[:-1][perm], seg_len, output_size)


def block_bucketize_sparse_features(
    lengths: torch.Tensor,
    indices: torch.Tensor,
    bucketize_pos: bool,
    sequence: bool,
    block_sizes: torch.Tensor,
    my_size: int,
    weights: Optional[torch.Tensor] = None,
    batch_size_per_feature: Optional[torch.Tensor] = None,
    max_B: int = -1,
    block_bucketize_pos: Optional[List[torch.Tensor]] = None,
    keep_orig_idx: bool = False,
    total_num_blocks: Optional[torch.Tensor] = None,
    keep_orig_idx_per_feature: Optional[torch.Tensor] = None,
) -> Tuple[torch.Tensor, torch.Tensor, Optional[torch.Tensor], Optional[torch.Tensor], Optional[torch.Tensor]]:
    """Row-wise bucketization: id -> (bucket = id // block_size[f], local id = id % block_size[f]).

    Input layout lengths [F*B] (feature major). Output lengths [my_size * F * B] ordered
    (bucket, feature, sample); values re-sorted accordingly (stable within a bag). Returns
    (new_lengths, new_indices, new_weights, new_pos, unbucketize_permute).
    Parity: fbgemm.block_bucketize_sparse_features as called at embedding_sharding.py:312.
    """
    n = indices.numel()
    FB = lengths.numel()
    F = block_sizes.numel()
    B = FB // max(F, 1)
    dev = indices.device
    if (indices.is_cuda and _lib.available() and not keep_orig_idx and batch_size_per_feature is None and keep_orig_idx_per_feature is None
            and FB > 0 and my_size <= 4096 and indices.dtype in (torch.int32, torch.int64)):
        return _block_bucketize_cuda(lengths, indices, bucketize_pos, sequence, block_sizes, my_size, weights, block_bucketize_pos, F, B)
    lengths64 = lengths.to(torch.int64)
    bag = torch.repeat_interleave(torch.arange(FB, device=dev), lengths64, output_size=n)
    feat = bag // max(B, 1)
    if block_bucketize_pos is not None:
        bucket = torch.empty(n, dtype=torch.int64, device=dev)
        local = torch.empty(n, dtype=indices.dtype, device=dev)
        for f in range(F):
            m = feat == f
            pos = block_bucketize_pos[f].to(indices.dtype)
            b_ = torch.bucketize(indices[m], pos[1:], right=True).clamp(max=my_size - 1)
            bucket[m] = b_
            local[m] = indices[m] - pos[b_]
    else:
        bs = block_sizes.to(indices.dtype)[feat]
        blk = torch.div(indices, bs, rounding_mode="floor")
        in_range = blk < my_size
        # ids past the last block wrap round-robin (fbgemm semantics for un-hashed overflow ids)
        bucket = torch.where(in_range, blk, indices % my_size).to(torch.int64)
        local = torch.where(in_range, indices - blk * bs, torch.div(indices, my_size, rounding_mode="floor"))
    if keep_orig_idx:
        local = indices
    new_bag = bucket * FB + bag
    order = torch.argsort(new_bag, stable=True)
    new_lengths = torch.zeros(my_size * FB, dtype=lengths.dtype, device=dev)
    new_lengths.index_add_(0, new_bag, torch.ones(n, dtype=lengths.dtype, device=dev))
    new_indices = local[order]
    new_weights = None if weights is None else weights[order]
    new_pos = None
    if bucketize_pos:
        off = torch.cumsum(lengths64, 0) - lengths64
        pos_in_bag = torch.arange(n, device=dev) - off[bag]
        new_pos = pos_in_bag[order].to(indices.dtype)
    unbucketize = None
    if sequence:
        unbucketize = torch.empty(n, dtype=indices.dtype, device=dev)
        unbucketize[order] = torch.arange(n, device=dev, dtype=indices.dtype)
    return new_lengths, new_indices, new_weights, new_pos, unbucketize


_BB_TABLES: dict = {}


def _block_bucketize_cuda(lengths, indices, bucketize_pos, sequence, block_sizes, my_size, weights, block_bucketize_pos, F: int, B: int):
    """Device-side bucketization through the routing kernels of ``csrc/kjt_route.cu`` (3 launches, no host sync): the "units" are the
    (bucket, feature) pairs in output order; a unit keeps the ids of its row block (or, past the table's last block, the ids whose
    remainder modulo ``my_size`` is the bucket) and rebases them."""
    dev = indices.device
    INT64_MAX = (1 << 63) - 1
    key = (F, my_size, block_sizes.data_ptr(), None if block_bucketize_pos is None else tuple(t.data_ptr() for t in block_bucketize_pos), str(dev))
    tab = _BB_TABLES.get(key)
    if tab is None:
        bs = block_sizes.to(device=dev, dtype=torch.int64)
        j = torch.arange(my_size, device=dev, dtype=torch.int64).unsqueeze(1)  # [my_size, 1]
        if block_bucketize_pos is None:
            lo = (j * bs.unsqueeze(0)).reshape(-1)
            hi = ((j + 1) * bs.unsqueeze(0)).reshape(-1)
            wrap = (bs * my_size).unsqueeze(0).expand(my_size, F).reshape(-1).contiguous()
        else:
            pos = torch.stack([p.to(device=dev, dtype=torch.int64) for p in block_bucketize_pos], dim=1)  # [my_size + 1, F]
            lo, hi = pos[:-1].reshape(-1).contiguous(), pos[1:].reshape(-1).clone()
            hi.view(my_size, F)[-1] = INT64_MAX  # ids past the last boundary stay in the last bucket
            wrap = None
        u_key = torch.arange(F, device=dev, dtype=torch.int32).repeat(my_size)
        zero = torch.zeros(my_size * F, dtype=torch.int32, device=dev)
        tab = (lo.contiguous(), hi.contiguous(), wrap, u_key, zero, torch.arange(my_size * F, device=dev, dtype=torch.int32),
               torch.arange(my_size, device=dev, dtype=torch.int32).repeat_interleave(F),
               torch.tensor([0, my_size * F], dtype=torch.int32, device=dev), torch.zeros(1, dtype=torch.int32, device=dev))
        _BB_TABLES[key] = tab
    lo, hi, wrap, u_key, zero, slot, rem, ustart, overflow = tab
    U = my_size * F
    n = indices.numel()
    in_off = asynchronous_complete_cumsum(lengths.to(torch.int64))
    L = _lib.lib()
    L.trb_kjt_route_workspace_bytes.restype = ctypes.c_int64
    ws = torch.empty(int(L.trb_kjt_route_workspace_bytes(U, B)), dtype=torch.uint8, device=dev)
    new_len32 = torch.empty(U * B + 1, dtype=torch.int32, device=dev)
    out_off = torch.empty(U * B + 1, dtype=torch.int32, device=dev)
    new_indices = torch.empty(n, dtype=indices.dtype, device=dev)
    new_weights = torch.empty(n, dtype=torch.float32, device=dev) if weights is not None else None
    new_pos = torch.empty(n, dtype=torch.int64, device=dev) if bucketize_pos else None
    unbucketize = torch.empty(n, dtype=torch.int64, device=dev) if sequence else None
    w32 = weights.float().contiguous() if weights is not None else None
    code = L.trb_kjt_route_ex(
        _lib.ptr(in_off), 1, _lib.ptr(indices), int(indices.dtype == torch.int64), _lib.ptr(w32), B, _lib.ptr(u_key), _lib.ptr(lo), _lib.ptr(hi), _lib.ptr(zero),
        _lib.ptr(slot), _lib.ptr(zero), _lib.ptr(ustart), U, 1, _lib.ptr_array([out_off.data_ptr()]), 0, _lib.ptr_array([new_indices.data_ptr()]),
        int(indices.dtype == torch.int64), _lib.ptr_array([new_weights.data_ptr()]) if new_weights is not None else ctypes.c_void_p(0), ctypes.c_int64(max(n, 1)),
        _lib.ptr(unbucketize), 1, _lib.ptr(new_pos), _lib.ptr(wrap), _lib.ptr(rem) if wrap is not None else ctypes.c_void_p(0), my_size, ctypes.c_void_p(0), _lib.ptr(new_len32),
        _lib.ptr(overflow), _lib.ptr(ws), ctypes.c_int64(ws.numel()), int(max(1, n // max(F * B, 1))), _lib.stream_ptr(dev))
    _lib.check(code, "trb_kjt_route_ex")
    new_lengths = new_len32[: U * B].to(lengths.dtype)
    if new_weights is not None and weights.dtype != torch.float32:
        new_weights = new_weights.to(weights.dtype)
    return (new_lengths, new_indices, new_weights, None if new_pos is None else new_pos.to(indices.dtype),
            None if unbucketize is None else unbucketize.to(indices.dtype))


def jagged_to_padded_dense(values: torch.Tensor, offsets: Sequence[torch.Tensor], max_lengths: Sequence[int], padding_value: float = 0.0) -> torch.Tensor:
    if values.is_cuda and _lib.available() and values.dim() <= 2 and values.is_contiguous() and (values[0:1].numel() * values.element_size()) % 4 == 0 and values.numel() > 0 \
            and values.element_size() in (4, 8) :
        off64 = offsets[0].to(torch.int64).contiguous()
        N, max_len = off64.numel() - 1, int(max_lengths[0])
        trail = tuple(values.shape[1:])
        out = torch.empty((N, max_len) + trail, dtype=values.dtype, device=values.device)
        row_bytes = values[0:1].numel() * values.element_size()
        if values.element_size() == 4:
            pad = torch.tensor([padding_value], dtype=values.dtype).view(torch.int32).item() & 0xFFFFFFFF
            code = _lib.lib().trb_jagged_to_padded_dense(_lib.ptr(values), _lib.ptr(off64), _lib.ptr(out), ctypes.c_int64(N), max_len, int(row_bytes),
                                                         ctypes.c_uint32(pad), _lib.stream_ptr(values.device))
            _lib.check(code, "trb_jagged_to_padded_dense")
            return out
    off = offsets[0].long()
    N = off.numel() - 1
    max_len = max_lengths[0]
    lengths = off[1:] - off[:-1]
    trail = values.shape[1:]
    out = values.new_full((N, max_len) + tuple(trail), padding_value)
    if values.numel() == 0 or N == 0:
        return out
    n = values.shape[0]
    seg = torch.repeat_interleave(torch.arange(N, device=values.device), lengths, output_size=n)
    pos = torch.arange(n, device=values.device) - off[:-1][seg]
    keep = pos < max_len
    out[seg[keep], pos[keep]] = values[keep]
    return out


def jagged_2d_to_dense(values: torch.Tensor, offsets: torch.Tensor, max_sequence_length: int) -> torch.Tensor:
    return jagged_to_padded_dense(values, [offsets], [max_sequence_length], 0.0)


def jagged_1d_to_dense(values: torch.Tensor, offsets: torch.Tensor, max_sequence_length: int, padding_value: float) -> torch.Tensor:
    return jagged_to_padded_dense(values, [offsets], [max_sequence_length], padding_value)


def dense_to_jagged(dense: torch.Tensor, offsets: Sequence[torch.Tensor], total_L: Optional[int] = None) -> Tuple[torch.Tensor, List[torch.Tensor]]:
    if dense.is_cuda and _lib.available() and total_L is not None and dense.is_contiguous() and dense.element_size() == 4 and dense.dim() in (2, 3):
        off64 = offsets[0].to(torch.int64).contiguous()
        trail = tuple(dense.shape[2:])
        out = torch.empty((int(total_L),) + trail, dtype=dense.dtype, device=dense.device)
        row_bytes = (dense[0, 0:1].numel()) * 4
        code = _lib.lib().trb_dense_to_jagged(_lib.ptr(dense), _lib.ptr(off64), _lib.ptr(out), ctypes.c_int64(dense.shape[0]), int(dense.shape[1]), int(row_bytes),
                                              _lib.stream_ptr(dense.device))
        _lib.check(code, "trb_dense_to_jagged")
        return out, list(offsets)
    off = offsets[0].long()
    lengths = off[1:] - off[:-1]
    N, max_len = dense.shape[0], dense.shape[1]
    mask = torch.arange(max_len, device=dense.device).unsqueeze(0) < lengths.unsqueeze(1)
    return dense[mask], list(offsets)


def jagged_index_select_2d(values: torch.Tensor, lengths: torch.Tensor, indices: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    off = torch.cumsum(lengths, 0) - lengths
    out_len = lengths[indices.long()]
    total = int(out_len.sum())
    if total == 0:
        return values[:0], out_len
    idx = _segment_gather_index(off[indices.long()], out_len, total)
    return values[idx], out_len


def keyed_jagged_index_select_dim1(
    values: torch.Tensor, lengths: torch.Tensor, offsets: torch.Tensor, indices: torch.Tensor, batch_size: int,
    weights: Optional[torch.Tensor] = None, selected_lengths_sum: Optional[int] = None,
) -> List[torch.Tensor]:
    """Select the same batch positions from every key of a [F, B] jagged layout."""
    F = lengths.numel() // batch_size
    idx = indices.long()
    sel = (torch.arange(F, device=lengths.device).unsqueeze(1) * batch_size + idx.unsqueeze(0)).reshape(-1)
    out_len = lengths[sel]
    total = int(out_len.sum()) if selected_lengths_sum is None else selected_lengths_sum
    if total == 0:
        res = [values[:0], out_len]
    else:
        g = _segment_gather_index(offsets[:-1][sel], out_len, total)
        res = [values[g], out_len]
        if weights is not None:
            res.append(weights[g])
            return res
    if weights is not None:
        res.append(weights[:0])
    return res


def batch_index_select_dim0(inputs: torch.Tensor, indices: torch.Tensor, input_num_indices: List[int], input_rows: List[int], input_columns: List[int], permute_output_dim_0_1: bool = False) -> torch.Tensor:
    outs = []
    io = ii = 0
    for n_idx, rows, cols in zip(input_num_indices, input_rows, input_columns):
        block = inputs[io : io + rows * cols].view(rows, cols)
        outs.append(block[indices[ii : ii + n_idx].long()])
        io += rows * cols
        ii += n_idx
    if permute_output_dim_0_1:
        return torch.cat(outs, dim=1).reshape(-1)
    return torch.cat([o.reshape(-1) for o in outs])


def jagged_unique_indices(hash_size_cumsum: torch.Tensor, hash_size_offsets: torch.Tensor, offsets: torch.Tensor, indices: torch.Tensor):
    """Per-table unique of a multi-feature id list. Returns (output_lengths, output_offsets, unique_indices, reverse_index) like the
    fbgemm op (reference embedding.py:1404).

    ``hash_size_cumsum`` [F + 1]: linearisation base of every feature (features of one table share the base of the table).
    ``hash_size_offsets``: feature ranges of the tables - entry i covers features [hso[i], hso[i + 1]); the reference passes one entry
    per feature (empty ranges for the non-first features of a table), one entry per table works too. All unique ids of a table are put
    into the first bag of its first feature (any split over the bags of the table is a valid KJT; this one needs no division)."""
    n = indices.numel()
    FB = offsets.numel() - 1
    F = hash_size_cumsum.numel() - 1
    B = FB // max(F, 1)
    dev = indices.device
    cum = hash_size_cumsum.long()
    lengths = offsets[1:] - offsets[:-1]
    bag = torch.repeat_interleave(torch.arange(FB, device=dev), lengths, output_size=n)
    feat = bag // max(B, 1)
    lin = indices.long() + cum[feat]
    uniq, inv = torch.unique(lin, return_inverse=True)  # sorted
    hso = hash_size_offsets.long()
    first, end = hso[:-1], hso[1:]
    real = end > first
    first, end = first[real], end[real]
    lo, hi = cum[first], cum[end]  # linearised id range of every table
    counts = torch.searchsorted(uniq, hi) - torch.searchsorted(uniq, lo)
    out_lengths = torch.zeros(FB, dtype=offsets.dtype, device=dev)
    out_lengths[first * B] = counts.to(offsets.dtype)
    out_offsets = asynchronous_complete_cumsum(out_lengths)
    table = torch.searchsorted(hi, uniq, right=True).clamp(max=max(hi.numel() - 1, 0))
    base = lo[table] if lo.numel() else torch.zeros_like(uniq)
    return out_lengths, out_offsets, (uniq - base).to(indices.dtype), inv


def group_index_select_dim0(inputs: Sequence[torch.Tensor], indices: Sequence[torch.Tensor]) -> List[torch.Tensor]:
    """``[x.index_select(0, i) for x, i in zip(inputs, indices)]`` as one op (fbgemm ``group_index_select_dim0``: a single
    launch over a group of tensors with different row counts / widths; used by the reference's pooled-embedding arch and VBE
    re-expansion, SURVEY 2.4b). Same-width members are gathered by one kernel over their concatenation; autograd flows through."""
    assert len(inputs) == len(indices)
    out: List[Optional[torch.Tensor]] = [None] * len(inputs)
    by_shape: Dict[Tuple, List[int]] = {}
    for k, x in enumerate(inputs):
        by_shape.setdefault((tuple(x.shape[1:]), x.dtype, x.device), []).append(k)
    for ks in by_shape.values():
        if len(ks) == 1:
            k = ks[0]
            out[k] = inputs[k].index_select(0, indices[k].long())
            continue
        base, cat_idx = 0, []
        for k in ks:
            cat_idx.append(indices[k].long() + base)
            base += inputs[k].shape[0]
        gathered = torch.cat([inputs[k] for k in ks], dim=0).index_select(0, torch.cat(cat_idx))
        pos = 0
        for k in ks:
            n = indices[k].numel()
            out[k] = gathered[pos : pos + n]
            pos += n
    return out  # type: ignore[return-value]


def permute_2D_sparse_data_input1D(permute: torch.Tensor, lengths: torch.Tensor, values: torch.Tensor, stride: int,
                                   weights: Optional[torch.Tensor] = None, permuted_lengths_sum: Optional[int] = None):
    """``permute_2D_sparse_data`` for lengths given flat (``[F * stride]``); returns flat permuted lengths (fbgemm op of the same
    name, used by the KJT all-to-all recat)."""
    F = lengths.numel() // max(stride, 1)
    pl, pv, pw = permute_2D_sparse_data(permute, lengths.view(F, stride), values, weights, permuted_lengths_sum)
    return pl.reshape(-1), pv, pw


_PERMUTE_TABLES: dict = {}


def permute_pooled_embs(pooled: torch.Tensor, offset_dim_list: Sequence[int], permute_list: Sequence[int]) -> torch.Tensor:
    """Column-block permutation of a [B, sum(D)] tensor (PermutePooledEmbeddings)."""
    if pooled.is_cuda and _lib.available() and pooled.dim() == 2 and pooled.is_contiguous() and not pooled.requires_grad and len(permute_list) > 0:
        esz = pooled.element_size()
        widths = [offset_dim_list[p + 1] - offset_dim_list[p] for p in permute_list]
        if all((w * esz) % 4 == 0 and (offset_dim_list[p] * esz) % 4 == 0 for w, p in zip(widths, permute_list)) and sum(widths) == pooled.shape[1]:
            key = (tuple(offset_dim_list), tuple(permute_list), esz, str(pooled.device))
            src = _PERMUTE_TABLES.get(key)
            if src is None:
                words = []
                for p in permute_list:
                    words.extend(range(offset_dim_list[p] * esz // 4, offset_dim_list[p + 1] * esz // 4))
                src = _PERMUTE_TABLES[key] = torch.tensor(words, dtype=torch.int32, device=pooled.device)
            out = torch.empty_like(pooled)
            code = _lib.lib().trb_permute_pooled_embs(_lib.ptr(pooled), _lib.ptr(out), _lib.ptr(src), ctypes.c_int64(pooled.shape[0]), int(src.numel()),
                                                      _lib.stream_ptr(pooled.device))
            _lib.check(code, "trb_permute_pooled_embs")
            return out
    cols = []
    for p in permute_list:
        cols.append(torch.arange(offset_dim_list[p], offset_dim_list[p + 1], device=pooled.device))
    if not cols:
        return pooled[:, :0]
    return pooled.index_select(1, torch.cat(cols))


def fused_nbit_rowwise_quantize(weight: torch.Tensor, bit_rate: int) -> torch.Tensor:
    """Row-wise N-bit quantization with fused fp16 (scale, bias) tail — the layout of fbgemm
    ``FloatOrHalfToFusedNBitRowwiseQuantizedSBHalf`` (quant/embedding_modules.py:264).
    Returns uint8 [rows, ceil(D*bits/8) + 4]."""
    assert bit_rate in (2, 4, 8)
    w = weight.float()
    rows, D = w.shape
    if rows == 0:  # an empty row shard (row-wise sharding of a table with fewer rows than ranks)
        return torch.zeros(0, (D * bit_rate + 7) // 8 + 4, dtype=torch.uint8, device=w.device)
    mn = w.min(dim=1, keepdim=True).values
    mx = w.max(dim=1, keepdim=True).values
    qmax = float((1 << bit_rate) - 1)
    mn16 = mn.half().float()
    scale = ((mx - mn16) / qmax).half().float()
    scale = torch.where(scale == 0, torch.ones_like(scale), scale)
    q = torch.clamp(torch.round((w - mn16) / scale), 0, qmax).to(torch.uint8)
    per_byte = 8 // bit_rate
    pad = (-D) % per_byte
    if pad:
        q = torch.cat([q, q.new_zeros(rows, pad)], 1)
    q = q.view(rows, -1, per_byte)
    packed = torch.zeros(rows, q.shape[1], dtype=torch.uint8, device=w.device)
    for i in range(per_byte):
        packed |= q[:, :, i] << (i * bit_rate)
    tail = torch.cat([scale.half().view(torch.uint8).view(rows, 2), mn16.half().view(torch.uint8).view(rows, 2)], 1)
    return torch.cat([packed, tail], 1)


def fused_nbit_rowwise_dequantize(q: torch.Tensor, bit_rate: int, D: int) -> torch.Tensor:
    rows = q.shape[0]
    if rows == 0:
        return torch.zeros(0, D, dtype=torch.float32, device=q.device)
    per_byte = 8 // bit_rate
    nbytes = (D + per_byte - 1) // per_byte
    packed = q[:, :nbytes]
    tail = q[:, nbytes : nbytes + 4].contiguous()
    scale = tail[:, 0:2].contiguous().view(torch.float16).float()
    bias = tail[:, 2:4].contiguous().view(torch.float16).float()
    mask = (1 << bit_rate) - 1
    parts = [((packed >> (i * bit_rate)) & mask) for i in range(per_byte)]
    vals = torch.stack(parts, dim=2).reshape(rows, -1)[:, :D].float()
    return vals * scale + bias
