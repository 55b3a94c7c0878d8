"""Quantized communication codecs (reference torchrec/distributed/fbgemm_qcomm_codec.py:31-254).

``CommType`` FP32 / FP16 / BF16 / FP8 / INT8 wire formats for the pooled all-to-all, reduce-scatter and
sequence all-to-all of the portable transport. FP8 / INT8 are row-wise scaled (one fp32 scale per ``row_dim``
elements) and therefore not usable for reductions on the wire: reduce-scatter falls back to BF16 (FP16 on CPU).

The fused NVLink plane (``sparse_plane.py``) reads ``fp8_row_dim`` of the codecs: an FP8 row-wise codec makes its kernels carry the
pooled rows and the gradients of directly written columns as e4m3 groups of that many columns plus one fp32 scale (the arithmetic
of ``trb_qcomm_encode`` / ``trb_qcomm_decode``, csrc/qcomm_fp8.cuh). Every other codec leaves the plane at its wire dtype."""
from __future__ import annotations

import logging
from dataclasses import dataclass
from enum import Enum, unique
from typing import Dict, List, Optional

import torch

from .types import CommOp, QuantizedCommCodec, QuantizedCommCodecs

logger = logging.getLogger(__name__)


@unique
class CommType(Enum):
    FP32 = "fp32"
    FP16 = "fp16"
    BF16 = "bf16"
    FP8 = "fp8"
    INT8 = "int8"
    MX4 = "mx4"

    def __str__(self) -> str:
        return self.value


@dataclass
class QCommsConfig:
    """Wire precision of forward (activations) and backward (gradients) embedding collectives."""

    forward_precision: CommType = CommType.FP32
    backward_precision: CommType = CommType.FP32
    forward_loss_scale: Optional[float] = None
    backward_loss_scale: Optional[float] = None
    fp8_quantize_dim: Optional[int] = None
    fp8_quantize_dim_bwd: Optional[int] = None
    fp8_bwd_uses_143: Optional[bool] = False
    mx4_quantize_dim: Optional[int] = None
    mx4_quantize_dim_bwd: Optional[int] = None
    mx4_rounding_mode: Optional[str] = None

    def __post_init__(self) -> None:
        if self.forward_precision != CommType.FP8 and self.backward_precision != CommType.FP8 and (
                self.fp8_quantize_dim is not None or self.fp8_quantize_dim_bwd is not None):
            raise ValueError(f"fp8_quantize_dim is set to {self.fp8_quantize_dim} and fp8_quantize_dim_bwd is set to {self.fp8_quantize_dim_bwd} but no FP8 precision is found in forward or backward precisions")
        if self.backward_precision == CommType.FP8 and self.fp8_quantize_dim_bwd is None:
            self.fp8_quantize_dim_bwd = self.fp8_quantize_dim
            logger.warning(f"No override of FP8 bwd row dim, using general FP8 row dim for backward: {self.fp8_quantize_dim_bwd} ")


class _CastCodec:
    def __init__(self, dtype: torch.dtype, loss_scale: Optional[float] = None) -> None:
        self._dtype = dtype
        self._loss_scale = loss_scale

    def encode(self, input_tensor: torch.Tensor, ctx=None) -> torch.Tensor:
        if self._loss_scale is not None:
            input_tensor = input_tensor * self._loss_scale
        return input_tensor.to(self._dtype)

    def decode(self, input_tensor: torch.Tensor, ctx=None) -> torch.Tensor:
        out = input_tensor.float()
        if self._loss_scale is not None:
            out = out / self._loss_scale
        return out

    @property
    def quantized_dtype(self) -> torch.dtype:
        return self._dtype

    @property
    def fp8_row_dim(self) -> Optional[int]:
        return None

    def calc_quantized_size(self, input_len: int, ctx=None) -> int:
        return input_len

    def create_context(self):
        return None

    def padded_size(self, input_tensor, dim_per_rank, my_rank, qcomm_ctx):
        return input_tensor.shape[0], 0


_CODEC_ID = {"fp8": 0, "int8": 1, "mx4": 2}


def _native(kind: str, encode: bool, x: torch.Tensor, rows: int, row_dim: int) -> torch.Tensor:
    """CUDA tensors go through the codec kernels of ``ops/csrc/qcomm.cu`` (one warp per row / per 32-element group)."""
    import ctypes

    from ..ops import _lib

    L = _lib.lib()
    cid = _CODEC_ID[kind]
    if encode:
        L.trb_qcomm_encoded_bytes.restype = ctypes.c_int64
        nbytes = int(L.trb_qcomm_encoded_bytes(cid, ctypes.c_int64(rows), row_dim))
        out = torch.empty(nbytes, dtype=torch.uint8, device=x.device)
        _lib.check(L.trb_qcomm_encode(cid, _lib.ptr(x), _lib.ptr(out), ctypes.c_int64(rows), row_dim, _lib.stream_ptr(x.device)), "trb_qcomm_encode")
    else:
        out = torch.empty(rows * row_dim, dtype=torch.float32, device=x.device)
        _lib.check(L.trb_qcomm_decode(cid, _lib.ptr(x), _lib.ptr(out), ctypes.c_int64(rows), row_dim, _lib.stream_ptr(x.device)), "trb_qcomm_decode")
    return out


class _RowwiseCodec:
    """Row-wise scaled 8-bit codec, uint8 wire. Per row of ``row_dim`` elements:
    FP8  ``[row_dim x e4m3][fp32 scale = amax / 448]``;  INT8  ``[row_dim x uint8][fp32 scale][fp32 bias = row min]``.
    CUDA tensors use the codec kernels, CPU tensors the PyTorch mirror of the same layout (gloo tests, numerics oracle)."""

    def __init__(self, row_dim: int, fp8: bool) -> None:
        self._row_dim = row_dim
        self._fp8 = fp8
        self._tail = 4 if fp8 else 8

    def _rows(self, n: int) -> int:
        assert n % self._row_dim == 0, f"tensor size {n} is not a multiple of the quantization row dim {self._row_dim}"
        return n // self._row_dim

    def encode(self, x: torch.Tensor, ctx=None) -> torch.Tensor:
        flat = x.reshape(-1).float().contiguous()
        rows = self._rows(flat.numel())
        if flat.is_cuda:
            return _native("fp8" if self._fp8 else "int8", True, flat, rows, self._row_dim)
        m = flat.view(rows, self._row_dim)
        if self._fp8:
            amax = m.abs().amax(dim=1, keepdim=True)
            scale = torch.where(amax > 0, amax / 448.0, torch.ones_like(amax))
            q = (m / scale).to(torch.float8_e4m3fn).view(torch.uint8)
            tail = scale.view(torch.uint8).view(rows, 4)
        else:
            lo, hi = m.amin(dim=1, keepdim=True), m.amax(dim=1, keepdim=True)
            scale = torch.where(hi > lo, (hi - lo) / 255.0, torch.ones_like(hi))
            q = torch.clamp(torch.round((m - lo) / scale), 0, 255).to(torch.uint8)
            tail = torch.cat([scale.view(torch.uint8).view(rows, 4), lo.contiguous().view(torch.uint8).view(rows, 4)], dim=1)
        return torch.cat([q, tail], dim=1).reshape(-1)

    def decode(self, x: torch.Tensor, ctx=None) -> torch.Tensor:
        rows = x.numel() // (self._row_dim + self._tail)
        if x.is_cuda:
            return _native("fp8" if self._fp8 else "int8", False, x.contiguous(), rows, self._row_dim)
        m = x.view(rows, self._row_dim + self._tail)
        q = m[:, : self._row_dim].contiguous()
        scale = m[:, self._row_dim : self._row_dim + 4].contiguous().view(torch.float32)
        if self._fp8:
            return (q.view(torch.float8_e4m3fn).float() * scale).reshape(-1)
        bias = m[:, self._row_dim + 4 :].contiguous().view(torch.float32)
        return (q.float() * scale + bias).reshape(-1)

    @property
    def quantized_dtype(self) -> torch.dtype:
        return torch.uint8

    @property
    def fp8_row_dim(self) -> Optional[int]:
        """Elements per fp32 scale when this is the FP8 row-wise codec, ``None`` for INT8."""
        return self._row_dim if self._fp8 else None

    def calc_quantized_size(self, input_len: int, ctx=None) -> int:
        return self._rows(input_len) * (self._row_dim + self._tail)

    def create_context(self):
        return None

    def padded_size(self, input_tensor, dim_per_rank, my_rank, qcomm_ctx):
        return input_tensor.shape[0], 0


_E2M1 = [0.0, 0.5, 1.0, 1.5, 2.0, 3.0, 4.0, 6.0]
_E2M1_EDGES = [0.25, 0.75, 1.25, 1.75, 2.5, 3.5, 5.0]


class _Mx4Codec:
    """MX4 (OCP microscaling): groups of 32 elements share one power-of-two scale (e8m0 byte), every element is a 4-bit e2m1 value:
    17 bytes per 32 elements = 4.25 bits per element on the wire."""

    GROUP = 32

    def __init__(self, row_dim: Optional[int] = None) -> None:
        self._row_dim = row_dim or 32

    def encode(self, x: torch.Tensor, ctx=None) -> torch.Tensor:
        flat = x.reshape(-1).float().contiguous()
        n = flat.numel()
        if flat.is_cuda:
            return _native("mx4", True, flat, 1, n)
        groups = (n + 31) // 32
        m = torch.zeros(groups * 32, dtype=torch.float32)
        m[:n] = flat
        m = m.view(groups, 32)
        amax = m.abs().amax(dim=1)
        e = torch.where(amax > 0, torch.floor(torch.log2(amax.clamp(min=1e-38))) - 2, torch.full_like(amax, -127.0)).clamp(-127, 127)
        scaled = m * torch.exp2(-e).unsqueeze(1)
        mag = torch.bucketize(scaled.abs(), torch.tensor(_E2M1_EDGES), right=True).to(torch.uint8)
        q = mag | ((scaled < 0).to(torch.uint8) << 3)
        packed = q[:, 0::2] | (q[:, 1::2] << 4)
        return torch.cat([(e + 127).to(torch.uint8).unsqueeze(1), packed], dim=1).reshape(-1)

    def decode(self, x: torch.Tensor, ctx=None, n: Optional[int] = None) -> torch.Tensor:
        groups = x.numel() // 17
        n = groups * 32 if n is None else n
        if x.is_cuda:
            return _native("mx4", False, x.contiguous(), 1, groups * 32)[:n]
        m = x.view(groups, 17)
        scale = torch.exp2(m[:, 0].float() - 127.0).unsqueeze(1)
        b = m[:, 1:]
        q = torch.stack([b & 15, b >> 4], dim=2).reshape(groups, 32)
        vals = torch.tensor(_E2M1)[(q & 7).long()] * torch.where((q & 8) > 0, -1.0, 1.0)
        return (vals * scale).reshape(-1)[:n]

    @property
    def quantized_dtype(self) -> torch.dtype:
        return torch.uint8

    @property
    def fp8_row_dim(self) -> Optional[int]:
        return None

    def calc_quantized_size(self, input_len: int, ctx=None) -> int:
        return (input_len + 31) // 32 * 17

    def create_context(self):
        return None

    def padded_size(self, input_tensor, dim_per_rank, my_rank, qcomm_ctx):
        return input_tensor.shape[0], 0


def get_qcomm_codec(comm_type: CommType, loss_scale: Optional[float], row_dim: Optional[int], is_fwd: bool = True):
    if comm_type == CommType.FP32:
        return _CastCodec(torch.float32, None)
    if comm_type == CommType.FP16:
        return _CastCodec(torch.float16, loss_scale)
    if comm_type == CommType.BF16:
        return _CastCodec(torch.bfloat16, loss_scale)
    if comm_type == CommType.FP8:
        return _RowwiseCodec(row_dim or 32, fp8=True)
    if comm_type == CommType.MX4:
        return _Mx4Codec(row_dim)
    if comm_type == CommType.INT8:
        return _RowwiseCodec(row_dim or 32, fp8=False)
    raise ValueError(comm_type)


def get_qcomm_codecs(qcomms_config: Optional[QCommsConfig]) -> QuantizedCommCodecs:
    codecs = QuantizedCommCodecs()
    if qcomms_config is not None:
        codecs.forward = get_qcomm_codec(qcomms_config.forward_precision, qcomms_config.forward_loss_scale, qcomms_config.fp8_quantize_dim, True)
        codecs.backward = get_qcomm_codec(qcomms_config.backward_precision, qcomms_config.backward_loss_scale,
                                          qcomms_config.fp8_quantize_dim_bwd if qcomms_config.backward_precision == CommType.FP8 else qcomms_config.fp8_quantize_dim, False)
    return codecs


def get_qcomm_codecs_registry(qcomms_config: QCommsConfig, comm_ops: Optional[List[CommOp]] = None, device: Optional[torch.device] = None) -> Optional[Dict[str, QuantizedCommCodecs]]:
    """Per comm op codecs. FP8/INT8/MX4 cannot be summed on the wire: reduce-scatter uses BF16 (FP16 on CPU)."""
    if qcomms_config.forward_precision == CommType.FP32 and qcomms_config.backward_precision == CommType.FP32:
        return None
    if comm_ops is None:
        comm_ops = [CommOp.POOLED_EMBEDDINGS_ALL_TO_ALL, CommOp.POOLED_EMBEDDINGS_REDUCE_SCATTER, CommOp.SEQUENCE_EMBEDDINGS_ALL_TO_ALL]
    registry: Dict[str, QuantizedCommCodecs] = {}
    on_cpu = device is not None and device.type == "cpu"
    for comm_op in comm_ops:
        cfg = qcomms_config
        if comm_op == CommOp.POOLED_EMBEDDINGS_REDUCE_SCATTER:
            fix = lambda t: (CommType.FP16 if on_cpu else CommType.BF16) if t in (CommType.FP8, CommType.INT8, CommType.MX4) else t
            cfg = QCommsConfig(forward_precision=fix(cfg.forward_precision), backward_precision=fix(cfg.backward_precision),
                               forward_loss_scale=cfg.forward_loss_scale, backward_loss_scale=cfg.backward_loss_scale)
        if on_cpu:
            swap = lambda t: CommType.FP16 if t == CommType.BF16 else t
            cfg = QCommsConfig(forward_precision=swap(cfg.forward_precision), backward_precision=swap(cfg.backward_precision),
                               forward_loss_scale=cfg.forward_loss_scale, backward_loss_scale=cfg.backward_loss_scale,
                               fp8_quantize_dim=cfg.fp8_quantize_dim, fp8_quantize_dim_bwd=cfg.fp8_quantize_dim_bwd)
        registry[comm_op.name] = get_qcomm_codecs(cfg)
    return registry
