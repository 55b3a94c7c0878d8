"""Python front-end of the hand-written wgmma GEMM (``csrc/gemm_wgmma.cu``).

``gemm_bf16_tn(a, b)`` computes ``act(alpha * a @ b.T + bias)`` with a ``[M, K]`` and b ``[N, K]``
(both bf16, K-major). ``LinearActFn`` is the autograd op behind ``Perceptron``:

    forward : y  = act(x W^T + b)                      one fused kernel (bias + ReLU in the epilogue)
    dgrad   : dx = (dy ⊙ act') W   = gemm(dy', W^T)     ReLU mask fused in the *previous* layer's dgrad epilogue
    wgrad   : dW = dy'^T x         = gemm(dy'^T, x^T)   operands transposed by a small tiled kernel, fp32 out
    bgrad   : db = colsum(dy')

Weights stay fp32 master copies (nn.Linear parameters); bf16 operand copies are made per call.
"""
from __future__ import annotations

import ctypes
import os
from typing import Optional, Tuple

import torch

from . import _lib

ACT_NONE, ACT_RELU, ACT_SIGMOID, ACT_RELU_GRAD = 0, 1, 2, 3


def _check_bf16_2d(t: torch.Tensor, name: str) -> None:
    assert t.is_cuda and t.dtype == torch.bfloat16 and t.dim() == 2 and t.stride(1) == 1, f"{name}: need a row-major bf16 CUDA matrix"
    assert t.stride(0) % 8 == 0 and t.shape[1] % 8 == 0, f"{name}: K and the row pitch must be multiples of 8 (16 B TMA alignment)"
    assert t.data_ptr() % 16 == 0, f"{name}: base pointer must be 16 B aligned"


def gemm_bf16(a: torch.Tensor, b: torch.Tensor, a_mn: bool = False, b_mn: bool = False, bias: Optional[torch.Tensor] = None,
              act: int = ACT_NONE, out_dtype: torch.dtype = torch.bfloat16, mask: Optional[torch.Tensor] = None, alpha: float = 1.0,
              out: Optional[torch.Tensor] = None, split_k: int = 1, tile_n: int = 0, mask_bits: Optional[torch.Tensor] = None,
              relu_bits_out: Optional[torch.Tensor] = None, colsum_ws: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``act(alpha * op(a) @ op(b)^T + bias)`` on the wgmma kernel (128 x 64 tiles for N <= 64, 128 x 128 otherwise). ``tile_n``: the
    tile width the caller sized ``split_k`` for (a hint; the kernel's tile depends on N only). ``relu_bits_out`` (int32
    ``[M, ceil(N / 32)]``, with ``ACT_RELU``): receives one bit per output (> 0); ``mask_bits`` (same layout, with ``ACT_RELU_GRAD``): used instead of re-reading ``mask``.

    ``a_mn=False``: a is ``[M, K]`` (K-major);  ``a_mn=True``: a is ``[K, M]`` (consumed MN-major, no transpose copy).
    ``b_mn=False``: b is ``[N, K]``;            ``b_mn=True``: b is ``[K, N]``.
    ``mask`` (bf16 [M, N]) with ``ACT_RELU_GRAD`` zeroes outputs where mask <= 0."""
    _check_bf16_2d(a, "a")
    _check_bf16_2d(b, "b")
    if a_mn:
        K, M = a.shape
    else:
        M, K = a.shape
    if b_mn:
        Kb, N = b.shape
    else:
        N, Kb = b.shape
    assert Kb == K and N % 8 == 0, (a.shape, b.shape, a_mn, b_mn)
    if out is None:
        out = torch.empty(M, N, dtype=out_dtype, device=a.device)
    assert out.stride(1) == 1 and out.dtype in (torch.bfloat16, torch.float32)
    if bias is not None:
        assert bias.dtype == torch.float32 and bias.is_contiguous() and bias.numel() == N
    if act == ACT_RELU_GRAD:
        assert mask is not None and mask.dtype == torch.bfloat16 and mask.shape == (M, N) and mask.stride(1) == 1 and mask.stride(0) % 8 == 0
    bits = mask_bits if act == ACT_RELU_GRAD else (relu_bits_out if act == ACT_RELU else None)
    ld_bits = 0
    if bits is not None:
        assert bits.dtype == torch.int32 and bits.dim() == 2 and bits.shape[0] == M and bits.stride(1) == 1 and bits.stride(0) * 32 >= N and bits.device == a.device
        ld_bits = bits.stride(0)
    if colsum_ws is not None:  # fp32 [ceil(M / 32), N]: per-32-row column sums of the bf16 output, written by the epilogue
        assert colsum_ws.dtype == torch.float32 and colsum_ws.is_contiguous() and tuple(colsum_ws.shape) == ((M + 31) // 32, N) and out.dtype == torch.bfloat16 and split_k <= 1
    L = _lib.lib()
    code = L.trb_gemm_bf16_ex3(
        _lib.ptr(a), ctypes.c_int64(a.stride(0)), int(a_mn), _lib.ptr(b), ctypes.c_int64(b.stride(0)), int(b_mn), _lib.ptr(out),
        ctypes.c_int64(out.stride(0)), 1 if out.dtype == torch.float32 else 0, M, N, K, _lib.ptr(bias), act, _lib.ptr(mask),
        ctypes.c_int64(mask.stride(0) if mask is not None else 0), ctypes.c_float(alpha), int(split_k), int(tile_n),
        _lib.ptr(mask_bits if act == ACT_RELU_GRAD else None), _lib.ptr(relu_bits_out if act == ACT_RELU else None), ctypes.c_int64(ld_bits),
        _lib.ptr(colsum_ws), _lib.stream_ptr(a.device),
    )
    _lib.check(code, "trb_gemm_bf16_ex3")
    return out


def colsum_from_partials(ws: torch.Tensor) -> torch.Tensor:
    """``ws [P, N]`` (the epilogue column sums of a GEMM, ``colsum_ws``) -> fp32 ``[N]``, fixed summation order."""
    P, N = ws.shape
    out = torch.empty(N, dtype=torch.float32, device=ws.device)
    code = _lib.lib().trb_colsum_partials(_lib.ptr(ws), int(P), int(N), _lib.ptr(out), _lib.stream_ptr(ws.device))
    _lib.check(code, "trb_colsum_partials")
    return out


def gemm_bf16_tn(a: torch.Tensor, b: torch.Tensor, bias: Optional[torch.Tensor] = None, act: int = ACT_NONE,
                 out_dtype: torch.dtype = torch.bfloat16, mask: Optional[torch.Tensor] = None, alpha: float = 1.0,
                 out: Optional[torch.Tensor] = None, split_k: int = 1, relu_bits_out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``act(alpha * a @ b.T + bias)`` with a ``[M, K]`` and b ``[N, K]`` (both K-major)."""
    return gemm_bf16(a, b, False, False, bias, act, out_dtype, mask, alpha, out, split_k, relu_bits_out=relu_bits_out)


def transpose_bf16(x: torch.Tensor, pad_cols_to: int = 8) -> torch.Tensor:
    """``x [R, C]`` -> ``[C, R_pad]`` bf16 with the row pitch padded to a multiple of 8 (zero filled)."""
    assert x.is_cuda and x.dtype == torch.bfloat16 and x.dim() == 2 and x.stride(1) == 1
    R, C = x.shape
    Rp = (R + pad_cols_to - 1) // pad_cols_to * pad_cols_to
    out = torch.zeros(C, Rp, dtype=torch.bfloat16, device=x.device) if Rp != R else torch.empty(C, R, dtype=torch.bfloat16, device=x.device)
    L = _lib.lib()
    code = L.trb_transpose_bf16(_lib.ptr(x), _lib.ptr(out), R, C, ctypes.c_int64(x.stride(0)), ctypes.c_int64(out.stride(0)), _lib.stream_ptr(x.device))
    _lib.check(code, "trb_transpose_bf16")
    return out


def colsum_bf16(x: torch.Tensor) -> torch.Tensor:
    assert x.is_cuda and x.dtype == torch.bfloat16 and x.dim() == 2 and x.stride(1) == 1
    out = torch.empty(x.shape[1], dtype=torch.float32, device=x.device)
    L = _lib.lib()
    code = L.trb_colsum_bf16(_lib.ptr(x), _lib.ptr(out), x.shape[0], x.shape[1], ctypes.c_int64(x.stride(0)), _lib.stream_ptr(x.device))
    _lib.check(code, "trb_colsum_bf16")
    return out


_SMS = {}


def _num_sms(device: torch.device) -> int:
    idx = device.index if device.index is not None else torch.cuda.current_device()
    if idx not in _SMS:
        _SMS[idx] = torch.cuda.get_device_properties(idx).multi_processor_count
    return _SMS[idx]


# ReLU layers emit a bit mask of their output for the following layer's masked dgrad (TRB_GEMM_RELU_BITS=0: re-read the activation)
RELU_BITS = os.environ.get("TRB_GEMM_RELU_BITS", "1") != "0"


def _best_split(tiles: int, K: int, sms: int) -> int:
    """Split-K factor that fills whole waves of the grid: maximise tiles*s / (ceil(tiles*s / sms) * sms) over splits that keep
    >= 512 reduction elements each (fewer, fuller waves beat many splits: every split adds a pass of fp32 atomics)."""
    best, best_score = 1, -1.0
    for s in range(1, max(1, min(64, K // 512)) + 1):
        items = tiles * s
        score = items / (((items + sms - 1) // sms) * sms) - 0.004 * s
        if score > best_score:
            best, best_score = s, score
    return best


# CTAs of the GEMM kernel resident per SM (csrc/gemm_wgmma.cu: __launch_bounds__(288, 2), a 96 KB operand ring each): one wave of the
# grid is GEMM_CTAS_PER_SM x SMs tiles
GEMM_CTAS_PER_SM = 2


def _wgrad_plan(n_out: int, n_in: int, batch: int, sms: int) -> "tuple[int, int]":
    """(split_k, tile_n) of the weight-gradient GEMM ``[n_out, n_in] = gy^T[n_out, batch] . x[batch, n_in]`` on 128 x 128 tiles."""
    tiles = ((n_out + 127) // 128) * ((n_in + 127) // 128)
    return _best_split(tiles, batch, GEMM_CTAS_PER_SM * sms), 128


COLSUM_OVERLAP = os.environ.get("TRB_COLSUM_OVERLAP", "1") != "0"
DEFER_WGRAD = os.environ.get("TRB_DEFER_WGRAD", "1") != "0"
_COLSUM_STREAMS: dict = {}


def _colsum_stream(device: torch.device) -> "torch.cuda.Stream":
    key = device.index if device.index is not None else torch.cuda.current_device()
    st = _COLSUM_STREAMS.get(key)
    if st is None:
        st = _COLSUM_STREAMS[key] = torch.cuda.Stream(device=device)
    return st


_DEFER_SCOPE = {"on": False}


class defer_wgrad_scope:
    """``with defer_wgrad_scope():`` around a CUDA-graph capture whose module inputs pass through ``DeferredGradJoin``: weight / bias
    gradients of every ``LinearActFn`` inside are left on the side stream until that node joins them."""

    def __enter__(self):
        self._prev = _DEFER_SCOPE["on"]
        _DEFER_SCOPE["on"] = True
        return self

    def __exit__(self, *exc):
        _DEFER_SCOPE["on"] = self._prev
        return False


class DeferredGradJoin(torch.autograd.Function):
    """Identity on the inputs of a module whose backward is captured into a CUDA graph. Its backward is the LAST node of that
    backward: it runs ``on_backward`` (e.g. the NVLink gradient push of the embedding gradients, so that the transfer is part of the
    graph and overlaps the deferred weight gradients) and then joins the side stream that carries the deferred wgrad / bias-grad
    kernels of every ``LinearActFn`` above it."""

    @staticmethod
    def forward(ctx, on_backward, *tensors):
        ctx.on_backward = on_backward
        ctx.device = tensors[0].device
        return tuple(t.view_as(t) for t in tensors)

    @staticmethod
    def backward(ctx, *grads):
        if ctx.on_backward is not None:
            ctx.on_backward(grads)
        if ctx.device.type == "cuda":
            torch.cuda.current_stream(ctx.device).wait_stream(_colsum_stream(ctx.device))
        return (None,) + tuple(grads)


def cast_pad_weights(weights) -> list:
    """bf16 GEMM operands ``[N, Kp]`` (K zero-padded to a multiple of 8) of several fp32 ``[N, K]`` weights with ONE kernel launch
    (one flat allocation, per-layer views). ``LinearActFn`` takes them through its ``wb`` argument."""
    import numpy as np

    ws = [w.detach() for w in weights]
    assert 0 < len(ws) <= 16 and all(w.is_cuda and w.dtype == torch.float32 and w.dim() == 2 and w.is_contiguous() for w in ws)
    Kps = [(w.shape[1] + 7) // 8 * 8 for w in ws]
    sizes = [w.shape[0] * kp for w, kp in zip(ws, Kps)]
    flat = torch.empty(sum(sizes), dtype=torch.bfloat16, device=ws[0].device)
    outs, o = [], 0
    for w, kp, n in zip(ws, Kps, sizes):
        outs.append(flat[o : o + n].view(w.shape[0], kp))
        o += n
    L = _lib.lib()
    n = len(ws)
    src = (ctypes.c_void_p * n)(*[w.data_ptr() for w in ws])
    dst = (ctypes.c_void_p * n)(*[t.data_ptr() for t in outs])
    i32 = lambda xs: np.ascontiguousarray(np.array(xs, dtype=np.int32)).ctypes.data_as(ctypes.c_void_p)
    rows, Ks, Kpa = np.array([w.shape[0] for w in ws], dtype=np.int32), np.array([w.shape[1] for w in ws], dtype=np.int32), np.array(Kps, dtype=np.int32)
    code = L.trb_multi_cast_pad_bf16(src, dst, rows.ctypes.data_as(ctypes.c_void_p), Ks.ctypes.data_as(ctypes.c_void_p), Kpa.ctypes.data_as(ctypes.c_void_p), n,
                                     _lib.stream_ptr(ws[0].device))
    _lib.check(code, "trb_multi_cast_pad_bf16")
    return outs


# Bias gradients from the dgrad epilogue of the layer above (``colsum_ws``) instead of a separate column-sum kernel. OFF by default:
# the column sums add shuffles and a named barrier to the epilogue of the dgrad GEMMs on the critical path, while the separate ``trb_colsum``
# kernels run beside them on their side stream. Opt in with TRB_EPI_COLSUM=1.
EPI_COLSUM = os.environ.get("TRB_EPI_COLSUM", "0") == "1"


def _pad_k(t: torch.Tensor, Kp: int) -> torch.Tensor:
    if t.shape[1] == Kp:
        return t
    return torch.nn.functional.pad(t, (0, Kp - t.shape[1]))


class LinearActFn(torch.autograd.Function):
    """``act(x @ W^T + b)`` on the wgmma kernel; bf16 activations, fp32 master weights."""

    @staticmethod
    def forward(ctx, x: torch.Tensor, weight: torch.Tensor, bias: Optional[torch.Tensor], act: int, wb: Optional[torch.Tensor] = None) -> torch.Tensor:
        N, K = weight.shape
        Kp = (K + 7) // 8 * 8
        xb = x if x.dtype == torch.bfloat16 else x.to(torch.bfloat16)
        pre_padded = xb.shape[1] == Kp and Kp != K  # producer already emitted the zero K-padding
        xb = _pad_k(xb, Kp)
        if xb.stride(1) != 1 or xb.stride(0) % 8 != 0:
            xb = xb.contiguous()
        if wb is None or tuple(wb.shape) != (N, Kp):  # (``cast_pad_weights`` of the enclosing MLP made the operand already)
            wb = _pad_k(weight.detach().to(torch.bfloat16), Kp)
        relu_bits = None
        if act == ACT_RELU and RELU_BITS:
            # one bit per output for the next layer's masked dgrad (it would otherwise re-read this whole activation)
            relu_bits = torch.empty(xb.shape[0], (N + 31) // 32, dtype=torch.int32, device=xb.device)
        y = gemm_bf16_tn(xb, wb, bias.detach() if bias is not None else None, act, relu_bits_out=relu_bits)
        # If this layer's input is the ReLU output of the previous fused layer, the ReLU gradient mask
        # of that layer is applied in *this* layer's dgrad epilogue (mask = saved input > 0).
        ctx.mask_input = bool(getattr(x, "_trb_relu_out", False)) and xb is x
        ctx.mask_bits = getattr(x, "_trb_relu_bits", None) if ctx.mask_input else None
        if act == ACT_RELU:
            y._trb_relu_out = True  # python attribute travels with the tensor object to the next layer
            y._trb_relu_bits = relu_bits
        ctx.act = act
        ctx.K = K
        ctx.has_bias = bias is not None
        ctx.x_dtype = x.dtype
        ctx.pre_padded = pre_padded
        ctx.save_for_backward(xb, wb, y)
        return y

    @staticmethod
    def backward(ctx, gy: torch.Tensor):
        xb, wb, y = ctx.saved_tensors
        act = ctx.act
        already_masked = bool(getattr(gy, "_trb_masked", False))
        gy = gy if gy.dtype == torch.bfloat16 else gy.to(torch.bfloat16)
        if gy.stride(1) != 1 or gy.stride(0) % 8 != 0:
            gy = gy.contiguous()
        if act == ACT_RELU:
            if not already_masked:
                gy = torch.where(y > 0, gy, torch.zeros_like(gy))
        elif act == ACT_SIGMOID:
            yf = y.float()
            gy = (gy.float() * yf * (1.0 - yf)).to(torch.bfloat16)
        M = gy.shape[0]
        gx = gw = gb = None
        # The weight / bias gradients are OFF the critical chain of the backward (the next layer only needs gx). On CUDA they go to a
        # side stream: the bias gradient (column sums of gy, a pure HBM stream) runs beside the tensor-core-bound GEMMs, and inside
        # a CUDA-graph capture the wgrad GEMM is DEFERRED too - the side stream is not joined per layer but once, by the node that
        # ends the captured backward (``DeferredGradJoin``), so the dgrad chain reaches the embedding gradients early and the NVLink
        # gradient dist overlaps the remaining wgrad work.
        want_w = ctx.needs_input_grad[1]
        want_b = ctx.has_bias and ctx.needs_input_grad[2]
        capturing = gy.is_cuda and DEFER_WGRAD and _DEFER_SCOPE["on"] and torch.cuda.is_current_stream_capturing()
        side = None
        if gy.is_cuda and (want_w or want_b) and (capturing or (COLSUM_OVERLAP and want_b and (ctx.needs_input_grad[0] or want_w))):
            cur = torch.cuda.current_stream(gy.device)
            side = _colsum_stream(gy.device)
            side.wait_stream(cur)
        # gy was written by the dgrad GEMM of the layer above: its epilogue may have left the column sums behind (EPI_COLSUM)
        parts = getattr(gy, "_trb_colsum_ws", None)
        if parts is not None and (parts.shape[1] != gy.shape[1] or parts.shape[0] != (M + 31) // 32):
            parts = None
        bias_grad = (lambda: colsum_from_partials(parts)) if parts is not None else (lambda: colsum_bf16(gy))
        if want_b:
            if side is not None:
                with torch.cuda.stream(side):
                    gb = bias_grad()
                gb.record_stream(cur)
                if parts is not None:
                    parts.record_stream(side)
            else:
                gb = bias_grad()

        def wgrad():
            # gw[N, Kp] = gy^T . x with BOTH operands consumed MN-major straight from their row-major storage
            split, tile_n = _wgrad_plan(gy.shape[1], xb.shape[1], M, _num_sms(gy.device))
            g = gemm_bf16(gy, xb, a_mn=True, b_mn=True, out_dtype=torch.float32, split_k=split, tile_n=tile_n)[:, : ctx.K]
            if g.stride(1) != 1 or g.shape[1] != g.stride(0):
                g = g.contiguous()
            return g

        if want_w and capturing:
            gy.record_stream(side)  # read by the deferred kernels after this node returned and dropped its reference
            with torch.cuda.stream(side):
                gw = wgrad()
            gw.record_stream(cur)
        if ctx.needs_input_grad[0]:
            # dgrad: gx[M, Kp] = gy[M, N] . W[N, Kp]; W is consumed as an MN-major B operand (no transpose)
            if ctx.mask_input and xb.shape[1] == ctx.K:
                # the masked output IS the pre-activation gradient of the layer below: its bias gradient (column sums) comes out of
                # this GEMM's epilogue instead of a second pass over the [M, K] tensor (trb_colsum was ~9 % of the DLRM step)
                ws = torch.empty((M + 31) // 32, xb.shape[1], dtype=torch.float32, device=gy.device) if (EPI_COLSUM and gy.is_cuda) else None
                gx = gemm_bf16(gy, wb, b_mn=True, act=ACT_RELU_GRAD, mask=xb, mask_bits=ctx.mask_bits, colsum_ws=ws)
                gx._trb_masked = True
                if ws is not None:
                    gx._trb_colsum_ws = ws
            else:
                gx = gemm_bf16(gy, wb, b_mn=True)
                if not ctx.pre_padded:
                    gx = gx[:, : ctx.K]
            if ctx.x_dtype != torch.bfloat16:
                gx = gx.to(ctx.x_dtype)
        if want_w and not capturing:
            gw = wgrad()
        if side is not None and (not capturing or not ctx.needs_input_grad[0]):
            # eager: the results are consumed right after this node (AccumulateGrad) -> join now. Captured: only the LAST node of the
            # chain (no input gradient wanted) joins; chains that continue are joined by DeferredGradJoin at the module inputs.
            torch.cuda.current_stream(gy.device).wait_stream(side)
        return gx, gw, gb, None, None
