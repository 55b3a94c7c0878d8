"""Cross networks (DCN family). Reference torchrec/modules/crossnet.py:21-380."""
import os
from typing import Callable, Optional, Union

import torch
from torch import nn


class CrossNet(nn.Module):
    """Full-rank cross network: ``x_{l+1} = x_0 * (W_l x_l + b_l) + x_l``."""

    def __init__(self, in_features: int, num_layers: int) -> None:
        super().__init__()
        self._num_layers = num_layers
        self.kernels: nn.ParameterList = nn.ParameterList(
            [nn.Parameter(nn.init.xavier_normal_(torch.empty(in_features, in_features))) for _ in range(num_layers)])
        self.bias: nn.ParameterList = nn.ParameterList(
            [nn.Parameter(nn.init.zeros_(torch.empty(in_features, 1))) for _ in range(num_layers)])

    def forward(self, input: torch.Tensor) -> torch.Tensor:
        x_0 = input.unsqueeze(2)  # (B, N, 1)
        x_l = x_0
        for layer in range(self._num_layers):
            xl_w = torch.matmul(self.kernels[layer], x_l)
            x_l = x_0 * (xl_w + self.bias[layer]) + x_l
        return torch.squeeze(x_l, dim=2)


_FUSED_COMBINE = os.environ.get("TRB_CROSS_FUSED", "1") != "0"


class _CrossCombine(torch.autograd.Function):
    """``y = x0 * u + xl`` on bf16 CUDA tensors: one element-wise kernel forward; backward ``gu = g * x0`` and ``gx0 = g * u`` in one
    kernel (x_0 feeds every cross layer: autograd sums the per-layer ``gx0`` terms), ``gxl = g`` without a kernel."""

    @staticmethod
    def forward(ctx, x0: torch.Tensor, u: torch.Tensor, xl: torch.Tensor) -> torch.Tensor:
        import ctypes

        from ..ops import _lib

        u = u.contiguous()
        xl = xl.contiguous()
        y = torch.empty_like(x0)
        code = _lib.lib().trb_cross_fwd(_lib.ptr(x0), _lib.ptr(u), _lib.ptr(xl), _lib.ptr(y), ctypes.c_int64(x0.numel()), _lib.stream_ptr(x0.device))
        _lib.check(code, "trb_cross_fwd")
        ctx.save_for_backward(x0, u)
        return y

    @staticmethod
    def backward(ctx, g: torch.Tensor):
        import ctypes

        from ..ops import _lib

        x0, u = ctx.saved_tensors
        g = g.contiguous() if g.dtype == torch.bfloat16 else g.to(torch.bfloat16).contiguous()
        gu = torch.empty_like(u)
        gx0 = torch.empty_like(x0)
        code = _lib.lib().trb_cross_bwd(_lib.ptr(g), _lib.ptr(x0), _lib.ptr(u), _lib.ptr(gu), _lib.ptr(gx0), ctypes.c_int64(x0.numel()), _lib.stream_ptr(x0.device))
        _lib.check(code, "trb_cross_bwd")
        return gx0, gu, g


class LowRankCrossNet(nn.Module):
    """Low-rank cross network: ``x_{l+1} = x_0 * (W_l (V_l x_l) + b_l) + x_l`` (DCN-v2)."""

    def __init__(self, in_features: int, num_layers: int, low_rank: int = 1) -> None:
        super().__init__()
        assert low_rank >= 1, "Low rank must be larger or equal to 1"
        self._num_layers = num_layers
        self._low_rank = low_rank
        W_kernels = nn.ParameterList()
        for _ in range(num_layers):
            Wp = nn.Parameter(torch.empty(in_features, low_rank))
            nn.init.xavier_normal_(Wp)
            W_kernels.append(Wp)
        V_kernels = nn.ParameterList()
        for _ in range(num_layers):
            Vp = nn.Parameter(torch.empty(low_rank, in_features))
            nn.init.xavier_normal_(Vp)
            V_kernels.append(Vp)
        self.W_kernels = W_kernels
        self.V_kernels = V_kernels
        self.bias: nn.ParameterList = nn.ParameterList(
            [nn.Parameter(nn.init.zeros_(torch.empty(in_features))) for _ in range(num_layers)])

    def _wgmma_ok(self, x: torch.Tensor) -> bool:
        from ..ops import dense as _dense

        return (_dense.get_dense_backend() == "wgmma" and x.is_cuda and x.dim() == 2 and x.shape[1] % 8 == 0 and self._low_rank % 8 == 0)

    def forward(self, input: torch.Tensor) -> torch.Tensor:
        x_0 = input
        x_l = x_0
        if self._wgmma_ok(input):
            # both projections on the hand-written sm_90a GEMM (bf16 operands, fp32 accumulation in registers, bias fused in the
            # epilogue of the second one); the Hadamard + residual stay element-wise in the activation dtype
            from ..ops import dense as _dense

            x_0 = x_0.to(torch.bfloat16).contiguous()
            x_l = x_0
            combine = _CrossCombine.apply if (x_0.numel() % 8 == 0 and _FUSED_COMBINE) else (lambda a, u, b: a * u + b)
            for layer in range(self._num_layers):
                x_l_v = _dense.linear_act(x_l, self.V_kernels[layer], None, _dense.ACT_NONE)
                x_l_w = _dense.linear_act(x_l_v, self.W_kernels[layer], self.bias[layer], _dense.ACT_NONE)
                x_l = combine(x_0, x_l_w, x_l)  # one kernel forward, one backward (ops/csrc/crossnet.cu)
            return x_l.to(input.dtype) if input.dtype != torch.bfloat16 else x_l
        for layer in range(self._num_layers):
            x_l_v = torch.nn.functional.linear(x_l, self.V_kernels[layer])
            x_l_w = torch.nn.functional.linear(x_l_v, self.W_kernels[layer])
            x_l = x_0 * (x_l_w + self.bias[layer]) + x_l
        return x_l


class VectorCrossNet(nn.Module):
    """Vector (DCN-v1) cross network: ``x_{l+1} = x_0 * (w_l^T x_l) + b_l + x_l``."""

    def __init__(self, in_features: int, num_layers: int) -> None:
        super().__init__()
        self._num_layers = num_layers
        self.kernels: nn.ParameterList = nn.ParameterList(
            [nn.Parameter(nn.init.xavier_normal_(torch.empty(in_features, 1))) for _ in range(num_layers)])
        self.bias: nn.ParameterList = nn.ParameterList(
            [nn.Parameter(nn.init.zeros_(torch.empty(in_features, 1))) for _ in range(num_layers)])

    def forward(self, input: torch.Tensor) -> torch.Tensor:
        x_0 = input.unsqueeze(2)
        x_l = x_0
        for layer in range(self._num_layers):
            xl_w = torch.tensordot(x_l, self.kernels[layer], dims=([1], [0]))
            x_l = torch.matmul(x_0, xl_w) + self.bias[layer] + x_l
        return torch.squeeze(x_l, dim=2)


class LowRankMixtureCrossNet(nn.Module):
    """Mixture of low-rank experts cross network (DCN-Mix)."""

    def __init__(self, in_features: int, num_layers: int, num_experts: int = 1, low_rank: int = 1,
                 activation: Union[nn.Module, Callable[[torch.Tensor], torch.Tensor]] = torch.relu) -> None:
        super().__init__()
        assert num_experts >= 1 and low_rank >= 1
        self._num_layers = num_layers
        self._num_experts = num_experts
        self._low_rank = low_rank
        self._in_features = in_features
        self.U_kernels = nn.ParameterList([
            nn.Parameter(nn.init.xavier_normal_(torch.empty(num_experts, in_features, low_rank))) for _ in range(num_layers)])
        self.V_kernels = nn.ParameterList([
            nn.Parameter(nn.init.xavier_normal_(torch.empty(num_experts, low_rank, in_features))) for _ in range(num_layers)])
        self.bias = nn.ParameterList([nn.Parameter(nn.init.zeros_(torch.empty(in_features, 1))) for _ in range(num_layers)])
        self.gates: Optional[nn.Module] = nn.ModuleList([nn.Linear(in_features, 1, bias=False) for _ in range(num_experts)]) if num_experts > 1 else None
        self._activation = activation
        self.C_kernels = nn.ParameterList([
            nn.Parameter(nn.init.xavier_normal_(torch.empty(num_experts, low_rank, low_rank))) for _ in range(num_layers)])

    def forward(self, input: torch.Tensor) -> torch.Tensor:
        x_0 = input.unsqueeze(2)
        x_l = x_0
        for layer in range(self._num_layers):
            if self._num_experts > 1:
                gating = [self.gates[i](x_l.squeeze(2)) for i in range(self._num_experts)]
                gating = torch.stack(gating, 1)  # (B, E, 1)
            experts = []
            for i in range(self._num_experts):
                expert = torch.matmul(self.V_kernels[layer][i], x_l)
                expert = torch.matmul(self.C_kernels[layer][i], self._activation(expert))
                expert = torch.matmul(self.U_kernels[layer][i], self._activation(expert))
                expert = x_0 * (expert + self.bias[layer])
                experts.append(expert.squeeze(2))
            experts = torch.stack(experts, 2)  # (B, N, E)
            if self._num_experts > 1:
                moe = torch.matmul(experts, torch.nn.functional.softmax(gating, 1))
                x_l = moe + x_l
            else:
                x_l = experts + x_l
        return torch.squeeze(x_l, dim=2)
