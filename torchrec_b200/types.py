"""Core enums / mixins (reference torchrec/types.py:17-72)."""
from __future__ import annotations

from abc import abstractmethod
from enum import Enum, unique

import torch
from torch import nn


class CacheMixin:
    """Modules that cache computed values during forward; ``clear_cache`` drops them."""

    @abstractmethod
    def clear_cache(self) -> None:
        ...


class CopyMixIn:
    @abstractmethod
    def copy(self, device: torch.device) -> nn.Module:
        ...


class ModuleCopyMixin(CopyMixIn):
    def copy(self, device: torch.device) -> nn.Module:
        return self.to(device)  # type: ignore[attr-defined]


class ModuleNoCopyMixin(CopyMixIn):
    def copy(self, device: torch.device) -> nn.Module:
        return self  # type: ignore[return-value]


@unique
class DataType(Enum):
    """Embedding storage data types."""

    FP32 = "FP32"
    FP16 = "FP16"
    BF16 = "BF16"
    INT64 = "INT64"
    INT32 = "INT32"
    INT8 = "INT8"
    UINT8 = "UINT8"
    INT4 = "INT4"
    INT2 = "INT2"
    FP8 = "FP8"  # block-scaled fp8 (e4m3 + fp16 scale per 32 elements)

    def __str__(self) -> str:
        return self.value
