"""Dense-arch kernels front-end: fused Linear+bias+activation (wgmma GEMM), dot interaction.

``set_dense_backend("wgmma")`` routes ``Perceptron`` layers and ``InteractionArch`` through the
hand-written sm_90a kernels in ``csrc/gemm_wgmma.cu`` / ``csrc/interaction.cu`` (bf16 operands,
fp32 accumulation in registers, bias+ReLU fused in the epilogue). ``"torch"`` keeps stock PyTorch ops
(used on CPU and as the numerics oracle).
"""
from __future__ import annotations

import ctypes
from typing import Callable, Optional

import torch
import torch.nn as nn

from . import _lib

_BACKEND = "torch"

ACT_NONE, ACT_RELU, ACT_SIGMOID = 0, 1, 2


def set_dense_backend(name: str) -> None:
    global _BACKEND
    if name not in ("torch", "wgmma"):
        raise ValueError(name)
    if name == "wgmma":
        _lib.lib()
    _BACKEND = name


def get_dense_backend() -> str:
    return _BACKEND


def fused_act_code(act) -> Optional[int]:
    if act is torch.relu or act is torch.nn.functional.relu or isinstance(act, nn.ReLU):
        return ACT_RELU
    if act is torch.sigmoid or isinstance(act, nn.Sigmoid):
        return ACT_SIGMOID
    if act is None or isinstance(act, nn.Identity):
        return ACT_NONE
    return None


def can_fuse(x: torch.Tensor, linear: nn.Linear) -> bool:
    if _BACKEND != "wgmma" or not x.is_cuda or x.dim() != 2:
        return False
    # TMA needs 16-byte aligned row pitches: K and N multiples of 8 bf16 elements
    # N must be a multiple of 8 (16-byte TMA rows of the transposed operands); K is zero-padded to 8
    return linear.out_features % 8 == 0


def linear_act(x: torch.Tensor, weight: torch.Tensor, bias: Optional[torch.Tensor], act: int, wb: Optional[torch.Tensor] = None) -> torch.Tensor:
    from .gemm import LinearActFn

    return LinearActFn.apply(x, weight, bias, act, wb)


def cast_weights_once(linears) -> Optional[list]:
    """bf16 operands of a stack of fused Linear layers made by ONE kernel (``gemm.cast_pad_weights``); None when the stack is not on
    the wgmma path (the layers then cast their own weights)."""
    if _BACKEND != "wgmma" or not linears or len(linears) > 16:
        return None
    ws = [l.weight for l in linears]
    if not all(w.is_cuda and w.dtype == torch.float32 and w.is_contiguous() and l.out_features % 8 == 0 for w, l in zip(ws, linears)):
        return None
    from .gemm import cast_pad_weights

    return cast_pad_weights(ws)


def dot_interaction(dense: torch.Tensor, sparse: torch.Tensor) -> torch.Tensor:
    """DLRM pairwise dot interaction. dense [B, D], sparse [B, F, D] ->
    [B, D + (F+1)F/2] = cat(dense, strictly-lower-triangular(X X^T)) with X = [dense; sparse].
    Parity: models/dlrm.py:210-222."""
    if _BACKEND == "wgmma" and dense.is_cuda:
        from . import interaction as _inter

        if _inter.supported(dense, sparse):
            return _inter.DotInteractionFn.apply(dense, sparse)
    B, D = dense.shape
    F = sparse.shape[1]
    combined = torch.cat((dense.unsqueeze(1), sparse.to(dense.dtype)), dim=1)
    inter = torch.bmm(combined, combined.transpose(1, 2))
    idx = _triu_flat_index(F + 1, dense.device)
    flat = inter.reshape(B, (F + 1) * (F + 1)).index_select(1, idx)
    return torch.cat((dense, flat), dim=1)


_TRIU_CACHE: dict = {}


def _triu_flat_index(n: int, device: torch.device) -> torch.Tensor:
    key = (n, str(device))
    if key not in _TRIU_CACHE:
        # a cached tensor must not be an inference tensor: the first caller may be a predict module under torch.inference_mode(), a later
        # one a training step that saves the index for backward
        with torch.inference_mode(False):
            ti = torch.triu_indices(n, n, offset=1, device=device)
            _TRIU_CACHE[key] = ti[0] * n + ti[1]
    return _TRIU_CACHE[key]
