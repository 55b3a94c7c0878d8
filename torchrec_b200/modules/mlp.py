"""Perceptron / MLP (reference torchrec/modules/mlp.py:18-190).

On CUDA with bf16/fp16 compute enabled (``torchrec_b200.ops.dense.set_dense_backend``) a
``Linear + bias + ReLU`` layer runs as ONE hand-written wgmma GEMM kernel with the bias
and activation fused into the epilogue (``csrc/gemm_wgmma.cu``); otherwise plain PyTorch.
"""
from typing import Callable, List, Optional, Union

import torch
from torch import nn

from ..ops import dense as _dense
from .activation import SwishLayerNorm
from .utils import extract_module_or_tensor_callable


class Perceptron(nn.Module):
    """Linear layer followed by an activation."""

    def __init__(
        self,
        in_size: int,
        out_size: int,
        bias: bool = True,
        activation: Union[nn.Module, Callable[[torch.Tensor], torch.Tensor]] = torch.relu,
        device: Optional[torch.device] = None,
        dtype: torch.dtype = torch.float32,
    ) -> None:
        super().__init__()
        self._out_size = out_size
        self._in_size = in_size
        self._linear: nn.Linear = nn.Linear(self._in_size, self._out_size, bias=bias, device=device, dtype=dtype)
        self._activation_fn = activation

    def forward(self, input: torch.Tensor, wb: Optional[torch.Tensor] = None) -> torch.Tensor:
        act = self._activation_fn
        fused = _dense.fused_act_code(act)
        if fused is not None and _dense.can_fuse(input, self._linear):
            return _dense.linear_act(input, self._linear.weight, self._linear.bias, fused, wb)
        if input.shape[-1] != self._in_size:  # producer emitted zero-padded columns (see ops.interaction)
            input = input[..., : self._in_size]
        if input.dtype != self._linear.weight.dtype and input.is_floating_point():
            input = input.to(self._linear.weight.dtype)
        return act(self._linear(input))


class MLP(nn.Module):
    """Stack of Perceptrons. ``activation`` may be ``"relu"``, ``"sigmoid"``, ``"swish_layernorm"``,
    a callable, or a module (factory)."""

    def __init__(
        self,
        in_size: int,
        layer_sizes: List[int],
        bias: bool = True,
        activation: Union[str, Callable[[], nn.Module], nn.Module, Callable[[torch.Tensor], torch.Tensor]] = torch.relu,
        device: Optional[torch.device] = None,
        dtype: torch.dtype = torch.float32,
        activation_on_last: bool = True,
    ) -> None:
        super().__init__()
        last = len(layer_sizes) - 1
        if activation == "relu":
            activation = torch.relu
        elif activation == "sigmoid":
            activation = torch.sigmoid
        if not isinstance(activation, str):
            self._mlp: nn.Module = nn.Sequential(*[
                Perceptron(
                    layer_sizes[i - 1] if i > 0 else in_size, layer_sizes[i], bias=bias,
                    activation=nn.Identity() if (not activation_on_last and i == last) else extract_module_or_tensor_callable(activation), device=device, dtype=dtype,
                )
                for i in range(len(layer_sizes))
            ])
        elif activation == "swish_layernorm":
            self._mlp = nn.Sequential(*[
                Perceptron(
                    layer_sizes[i - 1] if i > 0 else in_size, layer_sizes[i], bias=bias,
                    activation=nn.Identity() if (not activation_on_last and i == last) else SwishLayerNorm(layer_sizes[i], device=device), device=device,
                )
                for i in range(len(layer_sizes))
            ])
        else:
            raise ValueError(f"This MLP only supports str version activation function of relu, sigmoid, and swish_layernorm, got {activation}")

    def forward(self, input: torch.Tensor) -> torch.Tensor:
        layers = list(self._mlp)
        if input.is_cuda and input.dim() == 2 and len(layers) > 1 and all(isinstance(l, Perceptron) and _dense.fused_act_code(l._activation_fn) is not None for l in layers):
            # wgmma path: the bf16 operands of every layer come from ONE cast kernel in front of the stack
            wbs = _dense.cast_weights_once([l._linear for l in layers])
            if wbs is not None:
                x = input
                for l, wb in zip(layers, wbs):
                    x = l(x, wb)
                return x
        return self._mlp(input)
