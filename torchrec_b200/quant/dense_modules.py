"""FP8 inference forms of the dense-arch modules: ``Fp8MLP`` (for ``modules.mlp.MLP``) and ``Fp8LowRankCrossNet`` (for
``modules.crossnet.LowRankCrossNet``), built with ``from_float`` and normally installed by
``inference.modules.quantize_dense(module, torch.float8_e4m3fn)``.

They hold e4m3 weights, fp32 power-of-two channel scales and fp32 biases as buffers (format: ``ops/fp8_dense.py``). On CUDA every
projection runs on the FP8 wgmma GEMM (``ops/csrc/gemm_fp8.cu``); on CPU the same chain runs the emulation (dequantize, fp32
matmul), so swapping and state dicts can be checked without a GPU. Inference only: there is no backward.
"""
from __future__ import annotations

from typing import List, Optional

import torch
from torch import nn

from ..modules.crossnet import LowRankCrossNet, _CrossCombine
from ..modules.mlp import MLP, Perceptron
from ..ops import dense as _dense
from ..ops import fp8_dense as F8

_FP8_ACTS = {_dense.ACT_NONE: F8.ACT_NONE, _dense.ACT_RELU: F8.ACT_RELU}


class Fp8Linear(nn.Module):
    """One ``act(x W^T + b)`` layer in FP8: ``weight`` e4m3 ``[N, Kp]``, ``weight_scale`` fp32 ``[N]``, ``bias`` fp32 ``[N]`` or None."""

    def __init__(self, in_features: int, out_features: int, act: int, bias: bool, device: Optional[torch.device] = None) -> None:
        super().__init__()
        self.in_features = in_features
        self.out_features = out_features
        self.act = act
        self.register_buffer("weight", torch.zeros(out_features, F8.padded_k(in_features), dtype=F8.E4M3, device=device))
        self.register_buffer("weight_scale", torch.ones(out_features, dtype=torch.float32, device=device))
        self.register_buffer("bias", torch.zeros(out_features, dtype=torch.float32, device=device) if bias else None)

    @staticmethod
    def eligible(p: nn.Module) -> bool:
        """A Perceptron whose activation the FP8 epilogue fuses (none / ReLU) and whose output width is a multiple of 16."""
        return isinstance(p, Perceptron) and p._linear.out_features % 16 == 0 and _dense.fused_act_code(p._activation_fn) in _FP8_ACTS

    @classmethod
    def from_float(cls, p: Perceptron) -> "Fp8Linear":
        lin = p._linear
        m = cls(lin.in_features, lin.out_features, _FP8_ACTS[_dense.fused_act_code(p._activation_fn)], lin.bias is not None, device=lin.weight.device)
        q, s = F8.quantize_weight(lin.weight)
        m.weight.copy_(q)
        m.weight_scale.copy_(s)
        if lin.bias is not None:
            m.bias.copy_(lin.bias.detach().float())
        return m

    def extra_repr(self) -> str:
        return f"in_features={self.in_features}, out_features={self.out_features}, act={self.act}, bias={self.bias is not None}"


class Fp8MLP(nn.Module):
    """``MLP`` with its eligible layers (``Fp8Linear.eligible``) in FP8. The input is quantized once; consecutive FP8 layers hand the
    activation over in FP8 (the producer's epilogue quantizes it); the last FP8 layer of a run writes bf16. Ineligible layers keep
    their ``Perceptron`` and get that bf16 (or the caller's) tensor. Zero-padded input columns of a producer are accepted."""

    def __init__(self, layers: List[nn.Module]) -> None:
        super().__init__()
        self._mlp = nn.Sequential(*layers)

    @staticmethod
    def eligible(mlp: nn.Module) -> bool:
        return isinstance(mlp, MLP) and any(Fp8Linear.eligible(p) for p in mlp._mlp)

    @classmethod
    def from_float(cls, mlp: MLP) -> "Fp8MLP":
        return cls([Fp8Linear.from_float(p) if Fp8Linear.eligible(p) else p for p in mlp._mlp])

    def forward(self, input: torch.Tensor) -> torch.Tensor:
        layers = list(self._mlp)
        x, xq = input, None
        for i, layer in enumerate(layers):
            if not isinstance(layer, Fp8Linear):
                x = layer(x)
                continue
            if xq is None:
                if x.shape[-1] != layer.in_features:  # producer emitted zero-padded columns
                    x = x[:, : layer.in_features]
                if x.stride(-1) != 1:
                    x = x.contiguous()
                xq = F8.quantize_rows(x)
            to_fp8 = i + 1 < len(layers) and isinstance(layers[i + 1], Fp8Linear)
            y = F8.gemm_fp8(xq[0], xq[1], layer.weight, layer.weight_scale, layer.bias, layer.act, out_fp8=to_fp8)
            if to_fp8:
                xq = y
            else:
                x, xq = y, None
        return x


class Fp8LowRankCrossNet(nn.Module):
    """``LowRankCrossNet`` in FP8. Per layer: quantize ``x_l``, ``V_l x_l`` with an FP8-out epilogue, ``W_l (.) + b_l`` with a bf16
    output ``u``, then ``x_{l+1} = x_0 * u + x_l`` (``trb_cross_fwd`` on CUDA). Needs ``in_features`` and ``low_rank`` multiples of 16."""

    def __init__(self, in_features: int, num_layers: int, low_rank: int, device: Optional[torch.device] = None) -> None:
        super().__init__()
        self._in_features = in_features
        self._num_layers = num_layers
        self._low_rank = low_rank
        for l in range(num_layers):
            self.register_buffer(f"v_weight_{l}", torch.zeros(low_rank, F8.padded_k(in_features), dtype=F8.E4M3, device=device))
            self.register_buffer(f"v_scale_{l}", torch.ones(low_rank, dtype=torch.float32, device=device))
            self.register_buffer(f"w_weight_{l}", torch.zeros(in_features, F8.padded_k(low_rank), dtype=F8.E4M3, device=device))
            self.register_buffer(f"w_scale_{l}", torch.ones(in_features, dtype=torch.float32, device=device))
            self.register_buffer(f"bias_{l}", torch.zeros(in_features, dtype=torch.float32, device=device))

    @staticmethod
    def eligible(m: nn.Module) -> bool:
        return isinstance(m, LowRankCrossNet) and m._num_layers > 0 and m._low_rank % 16 == 0 and m.bias[0].numel() % 16 == 0

    @classmethod
    def from_float(cls, m: LowRankCrossNet) -> "Fp8LowRankCrossNet":
        D = m.bias[0].numel()
        out = cls(D, m._num_layers, m._low_rank, device=m.bias[0].device)
        for l in range(m._num_layers):
            vq, vs = F8.quantize_weight(m.V_kernels[l])
            wq, ws = F8.quantize_weight(m.W_kernels[l])
            getattr(out, f"v_weight_{l}").copy_(vq)
            getattr(out, f"v_scale_{l}").copy_(vs)
            getattr(out, f"w_weight_{l}").copy_(wq)
            getattr(out, f"w_scale_{l}").copy_(ws)
            getattr(out, f"bias_{l}").copy_(m.bias[l].detach().float())
        return out

    def forward(self, input: torch.Tensor) -> torch.Tensor:
        x0 = input.to(torch.bfloat16).contiguous()
        xl = x0
        for l in range(self._num_layers):
            q, s = F8.quantize_rows(xl)
            vq, vs = F8.gemm_fp8(q, s, getattr(self, f"v_weight_{l}"), getattr(self, f"v_scale_{l}"), None, F8.ACT_NONE, out_fp8=True)
            u = F8.gemm_fp8(vq, vs, getattr(self, f"w_weight_{l}"), getattr(self, f"w_scale_{l}"), getattr(self, f"bias_{l}"), F8.ACT_NONE)
            if x0.is_cuda and x0.numel() % 8 == 0:
                xl = _CrossCombine.apply(x0, u, xl)
            else:
                xl = torch.addcmul(xl.float(), x0.float(), u.float()).to(torch.bfloat16)
        return xl if input.dtype == torch.bfloat16 else xl.to(input.dtype)
