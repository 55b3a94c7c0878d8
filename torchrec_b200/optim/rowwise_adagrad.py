"""Row-wise Adagrad (pure PyTorch reference optimizer; reference torchrec/optim/rowwise_adagrad.py).

One accumulator per embedding row: ``sum[r] += mean(grad[r]^2)``, ``w[r] -= lr * grad[r] /
(sqrt(sum[r]) + eps)``. Used (a) as the tag class for ``apply_optimizer_in_backward`` — the sharded
tables then run the fused sm_90a kernel — and (b) as the CPU golden implementation in tests.
"""
from typing import Any, Dict, Iterable, List, Optional

import torch
from torch import Tensor
from torch.optim.optimizer import Optimizer


class RowWiseAdagrad(Optimizer):
    def __init__(self, params: Iterable[torch.nn.Parameter], lr: float = 1e-2, lr_decay: float = 0.0, weight_decay: float = 0.0,
                 initial_accumulator_value: float = 0.0, eps: float = 1e-10, *, maximize: bool = False, **unused: Any) -> None:
        if lr < 0.0:
            raise ValueError(f"Invalid learning rate: {lr}")
        if eps < 0.0:
            raise ValueError(f"Invalid epsilon value: {eps}")
        defaults = dict(lr=lr, lr_decay=lr_decay, eps=eps, weight_decay=weight_decay, initial_accumulator_value=initial_accumulator_value, maximize=maximize)
        super().__init__(params, defaults)
        for group in self.param_groups:
            for p in group["params"]:
                state = self.state[p]
                state["step"] = torch.tensor(0.0)
                init_value = complex(initial_accumulator_value, initial_accumulator_value) if torch.is_complex(p) else initial_accumulator_value
                state["sum"] = torch.full_like(p, init_value, memory_format=torch.preserve_format).mean(axis=1).view(-1, 1) if p.dim() == 2 else torch.full_like(p, init_value)

    def __setstate__(self, state: Dict[str, Any]) -> None:
        super().__setstate__(state)
        for group in self.param_groups:
            group.setdefault("maximize", False)

    @torch.no_grad()
    def step(self, closure: Any = None) -> Optional[torch.Tensor]:
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        for group in self.param_groups:
            for p in group["params"]:
                if p.grad is None:
                    continue
                state = self.state[p]
                state["step"] += 1
                step = float(state["step"])
                grad = p.grad
                if grad.is_sparse:
                    grad = grad.to_dense()
                if group["maximize"]:
                    grad = -grad
                if group["weight_decay"] != 0:
                    grad = grad.add(p, alpha=group["weight_decay"])
                clr = group["lr"] / (1 + (step - 1) * group["lr_decay"])
                touched = (grad != 0).any(dim=1, keepdim=True) if grad.dim() == 2 else torch.ones_like(grad, dtype=torch.bool)
                state["sum"].add_((grad * grad).mean(dim=1, keepdim=True) if grad.dim() == 2 else grad * grad)
                std = state["sum"].sqrt().add_(group["eps"])
                p.add_(torch.where(touched, -clr * grad / std, torch.zeros_like(grad)))
        return loss
