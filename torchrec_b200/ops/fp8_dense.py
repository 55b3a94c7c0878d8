"""FP8 (e4m3) dense inference: the number format, its CPU mirror, and the front end of ``csrc/gemm_fp8.cu``.

Format (the CUDA kernels reproduce it bit for bit):

* values: ``torch.float8_e4m3fn``, round to nearest even, saturating to +-448;
* activations ``[M, K]``: one scale per row per block of 128 consecutive columns (the last block may be partial);
* weights ``[N, K]`` (nn.Linear layout): one scale per output channel;
* every scale is a power of two: the smallest ``s`` with ``amax <= 448 * s`` (``s = 1`` for an all-zero block, ``s >= 2**-126``),
  taken from the exponent bits of ``amax`` plus one exact comparison. Dividing by ``s`` is exact, so the e4m3 cast is the only rounding.

Quantized activations are a pair ``(q, scales)``: ``q`` e4m3 ``[M, Kp]`` with ``Kp`` = K rounded up to 16 (zero columns after K) and
``scales`` fp32 ``[ceil(Kp / 128), Mp]``, ``Mp`` = M rounded up to 128, transposed so that the GEMM loads the 128 scales of one row tile
and K-block with one bulk copy. Code outside this module reads the layout only through :func:`row_block_scales`.

``gemm_fp8`` computes ``act(sw[n] * sum_kb sa[m, kb] * (A_q[m, kb] . W_q[n, kb]^T) + bias[n])`` with a bf16 output or an fp8 output
(quantized in the epilogue, the input format of the next fp8 layer). CUDA tensors run the kernels; CPU tensors run the emulation
(dequantize, fp32 matmul), which the CPU tests and CPU modules use. :func:`gemm_fp8_reference` is the float64 oracle of the tests.
"""
from __future__ import annotations

import ctypes
from typing import Optional, Tuple

import torch

from . import _lib

E4M3 = torch.float8_e4m3fn
E4M3_MAX = 448.0
BLOCK = 128  # columns per activation scale block
ROW_TILE = 128  # rows per GEMM tile: the scale rows are padded to a multiple of it
ACT_NONE, ACT_RELU = 0, 1


def padded_k(K: int) -> int:
    """Width of a quantized row: K rounded up to 16 (16-byte TMA rows)."""
    return (K + 15) // 16 * 16


def _scale_rows(M: int) -> int:
    return (M + ROW_TILE - 1) // ROW_TILE * ROW_TILE


def pow2_scale(amax: torch.Tensor) -> torch.Tensor:
    """The block scale of blocks with largest magnitudes ``amax`` (fp32): the smallest power of two ``s`` with ``amax <= 448 s``,
    1 for zero blocks, at least 2**-126. With ``amax = f 2^E`` (1 <= f < 2) and 448 = 1.75 2^8 the candidate is 2^(E - 8), and one
    exact comparison decides between it and 2^(E - 7)."""
    amax = amax.to(torch.float32)
    e = ((amax.view(torch.int32) >> 23) & 0xFF) - 127 - 8
    e = torch.clamp(e, min=-126)
    cand = ((e + 127) << 23).to(torch.int32).view(torch.float32)
    e = torch.where(amax <= E4M3_MAX * cand, e, e + 1)
    s = ((e + 127) << 23).to(torch.int32).view(torch.float32)
    return torch.where(amax > 0, s, torch.ones_like(s))


def _to_e4m3(x: torch.Tensor) -> torch.Tensor:
    # |x| <= 448 by construction of the scale; the clamp only mirrors the kernels' saturating cast
    return torch.clamp(x, -E4M3_MAX, E4M3_MAX).to(E4M3)


def quantize_rows_reference(x: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """CPU mirror of ``trb_fp8_quantize_rows``: ``x [M, K]`` -> ``(q e4m3 [M, Kp], scales fp32 [ceil(Kp / 128), Mp])``."""
    assert x.dim() == 2
    M, K = x.shape
    Kp = padded_k(K)
    KB = (Kp + BLOCK - 1) // BLOCK
    xf = torch.zeros(M, KB * BLOCK, dtype=torch.float32, device=x.device)
    xf[:, :K] = x.to(torch.float32)
    blocks = xf.view(M, KB, BLOCK)
    s = pow2_scale(blocks.abs().amax(dim=2))  # [M, KB]
    q = _to_e4m3(blocks * (1.0 / s).unsqueeze(2)).view(M, KB * BLOCK)[:, :Kp].contiguous()
    scales = torch.ones(KB, _scale_rows(M), dtype=torch.float32, device=x.device)
    scales[:, :M] = s.t()
    return q, scales


def quantize_rows(x: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """``x`` bf16 / fp32 ``[M, K]`` (any row pitch) -> ``(q, scales)``: the CUDA kernel on CUDA tensors, the reference on CPU."""
    if not _lib.use_cuda_kernels(x):
        return quantize_rows_reference(x)
    assert x.dim() == 2 and x.stride(1) == 1 and x.dtype in (torch.bfloat16, torch.float32), (x.shape, x.stride(), x.dtype)
    M, K = x.shape
    Kp = padded_k(K)
    q = torch.empty(M, Kp, dtype=E4M3, device=x.device)
    scales = torch.empty((Kp + BLOCK - 1) // BLOCK, _scale_rows(M), dtype=torch.float32, device=x.device)
    code = _lib.lib().trb_fp8_quantize_rows(_lib.ptr(x), ctypes.c_int64(x.stride(0)), int(x.dtype == torch.bfloat16), M, K, _lib.ptr(q),
                                            ctypes.c_int64(q.stride(0)), _lib.ptr(scales), ctypes.c_int64(scales.stride(0)), _lib.stream_ptr(x.device))
    _lib.check(code, "trb_fp8_quantize_rows")
    return q, scales


def quantize_weight(w: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """nn.Linear weight ``[N, K]`` -> ``(q e4m3 [N, Kp], channel scales fp32 [N])`` (zero columns after K). One-time model
    transformation: plain tensor ops on ``w``'s device, same rule as the kernels."""
    assert w.dim() == 2
    N, K = w.shape
    wf = w.detach().to(torch.float32)
    s = pow2_scale(wf.abs().amax(dim=1))
    q = torch.zeros(N, padded_k(K), dtype=E4M3, device=w.device)
    q[:, :K] = _to_e4m3(wf * (1.0 / s).unsqueeze(1))
    return q, s.contiguous()


def row_block_scales(scales: torch.Tensor, M: int) -> torch.Tensor:
    """``[M, ceil(Kp / 128)]`` view of the block scales of an M-row quantized activation."""
    return scales[:, :M].t()


def dequantize(q: torch.Tensor, scales: torch.Tensor, K: Optional[int] = None) -> torch.Tensor:
    """fp32 value of a quantized activation ``(q, scales)`` (``K``: drop the padding columns) or, with 1-D ``scales``, of a quantized
    weight."""
    qf = q.to(torch.float32)
    if scales.dim() == 1:
        out = qf * scales.to(qf.device).unsqueeze(1)
    else:
        M, Kp = q.shape
        s = row_block_scales(scales, M).to(qf.device)
        out = qf * s.repeat_interleave(BLOCK, dim=1)[:, :Kp]
    return out if K is None else out[:, :K]


def gemm_fp8_reference(a_q: torch.Tensor, sa: torch.Tensor, w_q: torch.Tensor, sw: torch.Tensor, bias: Optional[torch.Tensor] = None,
                       act: int = ACT_NONE) -> torch.Tensor:
    """float64 oracle of ``trb_gemm_fp8`` on the same quantized operands (the pre-rounding output, ``[M, N]`` float64, computed on
    the operands' device)."""
    M, Kp = a_q.shape
    a = a_q.to(torch.float64)
    w = w_q.to(torch.float64)
    sab = row_block_scales(sa, M).to(torch.float64)  # [M, KB]
    out = torch.zeros(M, w.shape[0], dtype=torch.float64, device=a.device)
    for kb in range(sab.shape[1]):
        k0, k1 = kb * BLOCK, min(Kp, (kb + 1) * BLOCK)
        out += sab[:, kb : kb + 1] * (a[:, k0:k1] @ w[:, k0:k1].t())
    out = out * sw.to(torch.float64).unsqueeze(0)
    if bias is not None:
        out = out + bias.to(torch.float64).unsqueeze(0)
    if act == ACT_RELU:
        out = torch.clamp(out, min=0.0)
    return out


def gemm_fp8(a_q: torch.Tensor, sa: torch.Tensor, w_q: torch.Tensor, sw: torch.Tensor, bias: Optional[torch.Tensor] = None, act: int = ACT_NONE,
             out_fp8: bool = False):
    """``act(sw[n] * sum_kb sa[m, kb] (A_q . W_q^T)_kb + bias[n])``. ``out_fp8=False``: bf16 ``[M, N]``; ``out_fp8=True``: the quantized
    output ``(q, scales)``, block scales computed in the epilogue. N must be a multiple of 16 and ``a_q``, ``w_q`` share the padded width."""
    M, Kp = a_q.shape
    N = w_q.shape[0]
    assert w_q.shape[1] == Kp and N % 16 == 0 and act in (ACT_NONE, ACT_RELU), (a_q.shape, w_q.shape, act)
    if not _lib.use_cuda_kernels(a_q):
        y = dequantize(a_q, sa) @ dequantize(w_q, sw).t()
        if bias is not None:
            y = y + bias.to(torch.float32)
        if act == ACT_RELU:
            y = torch.relu(y)
        return quantize_rows_reference(y) if out_fp8 else y.to(torch.bfloat16)
    assert a_q.dtype == E4M3 and w_q.dtype == E4M3 and a_q.stride(1) == 1 and w_q.stride(1) == 1
    assert sa.dtype == torch.float32 and sa.is_contiguous() and sa.shape[1] >= _scale_rows(M) and sa.shape[0] == (Kp + BLOCK - 1) // BLOCK
    assert sw.dtype == torch.float32 and sw.is_contiguous() and sw.numel() == N
    if bias is not None:
        assert bias.dtype == torch.float32 and bias.is_contiguous() and bias.numel() == N
    if out_fp8:
        out = torch.empty(M, N, dtype=E4M3, device=a_q.device)
        out_scales = torch.empty((N + BLOCK - 1) // BLOCK, _scale_rows(M), dtype=torch.float32, device=a_q.device)
    else:
        out = torch.empty(M, N, dtype=torch.bfloat16, device=a_q.device)
        out_scales = None
    code = _lib.lib().trb_gemm_fp8(
        _lib.ptr(a_q), ctypes.c_int64(a_q.stride(0)), _lib.ptr(sa), ctypes.c_int64(sa.stride(0)), _lib.ptr(w_q), ctypes.c_int64(w_q.stride(0)),
        _lib.ptr(sw), _lib.ptr(bias), int(act), _lib.ptr(out), ctypes.c_int64(out.stride(0)), int(out_fp8), _lib.ptr(out_scales),
        ctypes.c_int64(out_scales.stride(0) if out_scales is not None else 0), M, N, Kp, _lib.stream_ptr(a_q.device))
    _lib.check(code, "trb_gemm_fp8")
    return (out, out_scales) if out_fp8 else out
