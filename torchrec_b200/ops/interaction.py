"""DLRM dot interaction on wgmma tensor cores (``csrc/interaction.cu``)."""
from __future__ import annotations

import ctypes

import torch

from . import _lib


def _ceil8(x: int) -> int:
    return (x + 7) // 8 * 8


def supported(dense: torch.Tensor, sparse: torch.Tensor) -> bool:
    """Shapes the kernels cover: D % 16 == 0 with 16 <= D <= 256 and 1 <= F <= 127 (one 128-row MMA tile per sample at most)."""
    if not (dense.is_cuda and dense.dim() == 2 and sparse.dim() == 3):
        return False
    D = dense.shape[1]
    return (sparse.shape[2] == D and D % 16 == 0 and 16 <= D <= 256 and 1 <= sparse.shape[1] <= 127
            and sparse.dtype in (torch.float32, torch.bfloat16) and sparse.stride(2) == 1 and sparse.stride(1) == D
            and sparse.stride(0) % 8 == 0)


class DotInteractionFn(torch.autograd.Function):
    """``cat(dense, triu(X X^T, 1))`` with X = [dense; sparse]. Returns a bf16 ``[B, ceil8(D + R(R-1)/2)]``
    tensor whose tail columns are zero (consumed as K-padding by the next fused Linear)."""

    @staticmethod
    def forward(ctx, dense: torch.Tensor, sparse: torch.Tensor) -> torch.Tensor:
        B, D = dense.shape
        F = sparse.shape[1]
        db = dense if dense.dtype == torch.bfloat16 else dense.to(torch.bfloat16)
        if db.stride(1) != 1 or db.stride(0) % 8 != 0:
            db = db.contiguous()
        out_cols = D + (F + 1) * F // 2
        ld = _ceil8(out_cols)
        out = torch.empty(B, ld, dtype=torch.bfloat16, device=dense.device)
        L = _lib.lib()
        code = L.trb_interaction_fwd(_lib.ptr(db), ctypes.c_int64(db.stride(0)), _lib.ptr(sparse), ctypes.c_int64(sparse.stride(0)),
                                     1 if sparse.dtype == torch.float32 else 0, _lib.ptr(out), ctypes.c_int64(ld), B, F, D,
                                     _lib.stream_ptr(dense.device))
        _lib.check(code, "trb_interaction_fwd")
        ctx.save_for_backward(db, sparse)
        ctx.dense_dtype = dense.dtype
        ctx.out_cols = out_cols
        out._trb_logical_cols = out_cols  # consumers treat columns >= out_cols as zero K-padding
        return out

    @staticmethod
    def backward(ctx, gout: torch.Tensor):
        db, sparse = ctx.saved_tensors
        B, D = db.shape
        F = sparse.shape[1]
        ld = _ceil8(ctx.out_cols)
        g = gout if gout.dtype == torch.bfloat16 else gout.to(torch.bfloat16)
        if g.shape[1] != ld or g.stride(1) != 1 or g.stride(0) % 8 != 0:
            g2 = torch.zeros(B, ld, dtype=torch.bfloat16, device=g.device)
            g2[:, : g.shape[1]] = g
            g = g2
        g_dense = torch.empty(B, D, dtype=torch.bfloat16, device=g.device)
        g_sparse = torch.empty(B, F, D, dtype=sparse.dtype, device=g.device)
        L = _lib.lib()
        code = L.trb_interaction_bwd(_lib.ptr(db), ctypes.c_int64(db.stride(0)), _lib.ptr(sparse), ctypes.c_int64(sparse.stride(0)),
                                     1 if sparse.dtype == torch.float32 else 0, _lib.ptr(g), ctypes.c_int64(g.stride(0)), _lib.ptr(g_dense),
                                     ctypes.c_int64(D), _lib.ptr(g_sparse), ctypes.c_int64(F * D), 1 if sparse.dtype == torch.float32 else 0,
                                     B, F, D, _lib.stream_ptr(g.device))
        _lib.check(code, "trb_interaction_bwd")
        if ctx.dense_dtype != torch.bfloat16:
            g_dense = g_dense.to(ctx.dense_dtype)
        return g_dense, g_sparse
