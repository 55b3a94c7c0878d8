"""Inference table-batched embedding over quantized rows (``csrc/tbe_quant.cu``).

Replaces fbgemm ``IntNBitTableBatchedEmbeddingBagsCodegen`` (reference quant/embedding_modules.py:425-442).
Row formats: FP32, FP16, BF16, INT8 / INT4 / INT2 (row-wise, fused fp16 scale+bias tail) and
block-scaled FP8 (e4m3 + one fp16 scale per 32 elements)."""
from __future__ import annotations

import ctypes
from typing import Dict, List, Optional, Sequence, Tuple

import torch
import torch.nn as nn

from ..types import DataType
from . import _lib
from . import jagged as J

FMT = {DataType.FP32: 0, DataType.FP16: 1, DataType.BF16: 2, DataType.INT8: 3, DataType.INT4: 4, DataType.INT2: 5, DataType.FP8: 6}
_BITS = {DataType.INT8: 8, DataType.INT4: 4, DataType.INT2: 2}
FP8_BLOCK = 32


def row_bytes(dim: int, data_type: DataType, row_alignment: int = 16) -> int:
    if data_type == DataType.FP32:
        n = dim * 4
    elif data_type in (DataType.FP16, DataType.BF16):
        n = dim * 2
    elif data_type in _BITS:
        n = (dim * _BITS[data_type] + 7) // 8 + 4
    elif data_type == DataType.FP8:
        n = dim + (dim // FP8_BLOCK) * 2
    else:
        raise ValueError(data_type)
    return (n + row_alignment - 1) // row_alignment * row_alignment


def quantize_rows(weight: torch.Tensor, data_type: DataType, row_alignment: int = 16) -> torch.Tensor:
    """fp32 [rows, dim] -> uint8 [rows, row_bytes] in the kernel's row format."""
    rows, dim = weight.shape
    rb = row_bytes(dim, data_type, row_alignment)
    out = torch.zeros(rows, rb, dtype=torch.uint8, device=weight.device)
    w = weight.float()
    if data_type == DataType.FP32:
        out[:, : dim * 4] = w.contiguous().view(torch.uint8).view(rows, dim * 4)
    elif data_type == DataType.FP16:
        out[:, : dim * 2] = w.half().contiguous().view(torch.uint8).view(rows, dim * 2)
    elif data_type == DataType.BF16:
        out[:, : dim * 2] = w.bfloat16().contiguous().view(torch.uint8).view(rows, dim * 2)
    elif data_type in _BITS:
        q = J.fused_nbit_rowwise_quantize(w, _BITS[data_type])
        out[:, : q.shape[1]] = q
    elif data_type == DataType.FP8:
        assert dim % FP8_BLOCK == 0, f"block-scaled fp8 needs dim % {FP8_BLOCK} == 0"
        blocks = w.view(rows, dim // FP8_BLOCK, FP8_BLOCK)
        amax = blocks.abs().amax(dim=2, keepdim=True).clamp(min=1e-12)
        scale = (amax / 448.0).half().float().clamp(min=6e-8)
        q = (blocks / scale).to(torch.float8_e4m3fn).view(torch.uint8).view(rows, dim)
        out[:, :dim] = q
        out[:, dim : dim + (dim // FP8_BLOCK) * 2] = scale.half().contiguous().view(torch.uint8).view(rows, (dim // FP8_BLOCK) * 2)
    else:
        raise ValueError(data_type)
    return out


def dequantize_rows(q: torch.Tensor, dim: int, data_type: DataType) -> torch.Tensor:
    rows = q.shape[0]
    if data_type == DataType.FP32:
        return q[:, : dim * 4].contiguous().view(torch.float32).view(rows, dim)
    if data_type == DataType.FP16:
        return q[:, : dim * 2].contiguous().view(torch.float16).view(rows, dim).float()
    if data_type == DataType.BF16:
        return q[:, : dim * 2].contiguous().view(torch.bfloat16).view(rows, dim).float()
    if data_type in _BITS:
        return J.fused_nbit_rowwise_dequantize(q, _BITS[data_type], dim)
    if data_type == DataType.FP8:
        vals = q[:, :dim].contiguous().view(torch.float8_e4m3fn).float().view(rows, dim // FP8_BLOCK, FP8_BLOCK)
        scale = q[:, dim : dim + (dim // FP8_BLOCK) * 2].contiguous().view(torch.float16).float().view(rows, dim // FP8_BLOCK, 1)
        return (vals * scale).view(rows, dim)
    raise ValueError(data_type)


class QuantTableBatchedEmbeddingBags(nn.Module):
    """Inference TBE: ``embedding_specs`` = [(name, rows, dim, DataType)]; weights live in one uint8 buffer."""

    def __init__(self, embedding_specs: Sequence[Tuple[str, int, int, DataType]], feature_table_map: Optional[Sequence[int]] = None,
                 pooling_mode: int = 0, output_dtype: torch.dtype = torch.float32, device: Optional[torch.device] = None, row_alignment: int = 16) -> None:
        super().__init__()
        device = torch.device(device) if device is not None else torch.device("cpu")
        self.embedding_specs = list(embedding_specs)
        self.feature_table_map = list(feature_table_map) if feature_table_map is not None else list(range(len(self.embedding_specs)))
        self.pooling_mode = pooling_mode  # 0 sum, 1 mean, 2 none
        self.output_dtype = output_dtype
        self.row_alignment = row_alignment
        self._row_bytes = [row_bytes(d, dt, row_alignment) for _, _, d, dt in self.embedding_specs]
        offs, o = [], 0
        for (_, r, _, _), rb in zip(self.embedding_specs, self._row_bytes):
            offs.append(o)
            o += r * rb
        self._table_off = offs
        self.register_buffer("weights", torch.zeros(o, dtype=torch.uint8, device=device), persistent=False)
        fm = self.feature_table_map
        mk64 = lambda x: torch.tensor(x, dtype=torch.int64, device=device)
        mk32 = lambda x: torch.tensor(x, dtype=torch.int32, device=device)
        self._h_dim = [self.embedding_specs[t][2] for t in fm]
        cols, c = [], 0
        for d in self._h_dim:
            cols.append(c)
            c += d
        self._h_col, self.total_cols = cols, c
        if device.type != "meta":
            self.register_buffer("feat_woff", mk64([offs[t] for t in fm]), persistent=False)
            self.register_buffer("feat_rows", mk64([self.embedding_specs[t][1] for t in fm]), persistent=False)
            self.register_buffer("feat_dim", mk32(self._h_dim), persistent=False)
            self.register_buffer("feat_col", mk32(cols), persistent=False)
            self.register_buffer("feat_fmt", mk32([FMT[self.embedding_specs[t][3]] for t in fm]), persistent=False)
            self.register_buffer("feat_rb", mk32([self._row_bytes[t] for t in fm]), persistent=False)
        self.max_dim = max(self._h_dim) if self._h_dim else 0
        fmts = {FMT[dt] for _, _, _, dt in self.embedding_specs}
        # one row format for the whole launch + rows made of whole 16-byte vectors -> the vector kernel (tbe_quant.cu: qtbe_fwd_vec_kernel);
        # elements per vector: 16 for the 8-bit formats, 8 for fp16 / bf16, 32 for int4
        epv = {FMT[DataType.INT8]: 16, FMT[DataType.FP8]: 16, FMT[DataType.FP16]: 8, FMT[DataType.BF16]: 8, FMT[DataType.INT4]: 32}
        one = next(iter(fmts)) if len(fmts) == 1 else -1
        aligned = one in epv and all(d % epv[one] == 0 for d in self._h_dim) and all(rb % 16 == 0 for rb in self._row_bytes)
        self._uniform_fmt = one if aligned else -1

    def split_embedding_weights(self) -> List[torch.Tensor]:
        """Per table uint8 [rows, row_bytes] views."""
        return [self.weights[o : o + r * rb].view(r, rb) for (_, r, _, _), rb, o in zip(self.embedding_specs, self._row_bytes, self._table_off)]

    @torch.no_grad()
    def assign_from_float(self, table_idx: int, weight: torch.Tensor) -> None:
        name, rows, dim, dt = self.embedding_specs[table_idx]
        self.split_embedding_weights()[table_idx].copy_(quantize_rows(weight.to(self.weights.device), dt, self.row_alignment))

    def dequantized_table(self, table_idx: int) -> torch.Tensor:
        _, _, dim, dt = self.embedding_specs[table_idx]
        return dequantize_rows(self.split_embedding_weights()[table_idx], dim, dt)

    def forward(self, indices: torch.Tensor, offsets: torch.Tensor, per_sample_weights: Optional[torch.Tensor] = None, batch_size: Optional[int] = None) -> torch.Tensor:
        F = len(self.feature_table_map)
        B = batch_size if batch_size is not None else (offsets.numel() - 1) // max(F, 1)
        pooled = self.pooling_mode != 2
        if not _lib.use_cuda_kernels(self.weights):
            return self._ref_forward(indices, offsets, per_sample_weights, B, pooled)
        n = indices.numel()
        if pooled:
            out = torch.empty(B, self.total_cols, dtype=self.output_dtype, device=self.weights.device)
            stride = self.total_cols
        else:
            D = self._h_dim[0]
            out = torch.empty(n, D, dtype=self.output_dtype, device=self.weights.device)
            stride = D
        L = _lib.lib()
        code = L.trb_qtbe_fwd_ex(_lib.ptr(self.weights), _lib.ptr(self.feat_woff), _lib.ptr(self.feat_rows), _lib.ptr(self.feat_dim), _lib.ptr(self.feat_col),
                              _lib.ptr(self.feat_fmt), _lib.ptr(self.feat_rb), _lib.ptr(indices), 1 if indices.dtype == torch.int64 else 0,
                              _lib.ptr(offsets), 1 if offsets.dtype == torch.int64 else 0, _lib.ptr(per_sample_weights), _lib.ptr(out),
                              _lib.dtype_code(self.output_dtype), ctypes.c_int64(stride), B, F, self.max_dim, int(self.pooling_mode == 1), int(pooled),
                              ctypes.c_int64(n), int(self._uniform_fmt), _lib.stream_ptr(self.weights.device))
        _lib.check(code, "trb_qtbe_fwd_ex")
        return out

    def _ref_forward(self, indices, offsets, psw, B: int, pooled: bool) -> torch.Tensor:
        offsets = offsets.long()
        indices = indices.long()
        F = len(self.feature_table_map)
        if not pooled:
            D = self._h_dim[0]
            out = torch.zeros(indices.numel(), D, dtype=torch.float32, device=indices.device)
        else:
            out = torch.zeros(B, self.total_cols, dtype=torch.float32, device=indices.device)
        tables = {t: self.dequantized_table(t) for t in set(self.feature_table_map)}
        for f, t in enumerate(self.feature_table_map):
            tab = tables[t]
            off = offsets[f * B : (f + 1) * B + 1]
            lo, hi = int(off[0]), int(off[-1])
            idx = indices[lo:hi]
            valid = (idx >= 0) & (idx < tab.shape[0])
            vals = tab[torch.where(valid, idx, torch.zeros_like(idx))] * valid.unsqueeze(1)
            if not pooled:
                out[lo:hi] = vals
                continue
            if psw is not None:
                vals = vals * psw[lo:hi].float().unsqueeze(1)
            lengths = off[1:] - off[:-1]
            seg = torch.repeat_interleave(torch.arange(B, device=indices.device), lengths)
            pooled_v = torch.zeros(B, tab.shape[1], device=indices.device).index_add_(0, seg, vals)
            if self.pooling_mode == 1:
                pooled_v = pooled_v / lengths.clamp(min=1).unsqueeze(1)
            out[:, self._h_col[f] : self._h_col[f] + tab.shape[1]] = pooled_v
        return out.to(self.output_dtype)
