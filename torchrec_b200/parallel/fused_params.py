"""Accessors for the ``fused_params`` dict that sharders pass down to the table-batched kernels (reference
torchrec/distributed/fused_params.py:43-160). Keys the engine understands: optimizer hyper-parameters (``optimizer``,
``learning_rate``, ``eps``, ``beta1/2``, ``weight_decay``, ``weight_decay_mode``, ``max_gradient``, ``momentum``), ``stochastic_rounding``,
``cache_load_factor`` / ``cache_algorithm`` (UVM caching), ``output_dtype``, plus the inference-side switches below."""
from __future__ import annotations

from typing import Any, Dict, Iterable, Optional

import torch

FUSED_PARAM_REGISTER_TBE_BOOL: str = "__register_tbes_in_named_modules"
FUSED_PARAM_QUANT_STATE_DICT_SPLIT_SCALE_BIAS: str = "__register_quant_state_dict_split_scale_bias"
FUSED_PARAM_TBE_ROW_ALIGNMENT: str = "__register_tbe_row_alignment"
FUSED_PARAM_BOUNDS_CHECK_MODE: str = "__register_tbe_bounds_check_mode"
FUSED_PARAM_LENGTHS_TO_OFFSETS_LOOKUP: str = "__register_lengths_to_offsets_lookup"
_INTERNAL = (FUSED_PARAM_REGISTER_TBE_BOOL, FUSED_PARAM_QUANT_STATE_DICT_SPLIT_SCALE_BIAS, FUSED_PARAM_TBE_ROW_ALIGNMENT, FUSED_PARAM_BOUNDS_CHECK_MODE,
             FUSED_PARAM_LENGTHS_TO_OFFSETS_LOOKUP)


class TBEToRegisterMixIn:
    """Modules that own table-batched kernels expose them here so export / inspection tooling can find them."""

    def get_tbes_to_register(self) -> Dict[Any, Any]:
        raise NotImplementedError


def get_tbes_to_register_from_iterable(iterable: Iterable[torch.nn.Module]) -> Dict[Any, Any]:
    tbes: Dict[Any, Any] = {}
    for m in iterable:
        if isinstance(m, TBEToRegisterMixIn):
            tbes.update(m.get_tbes_to_register())
    return tbes


def is_fused_param_register_tbe(fused_params: Optional[Dict[str, Any]]) -> bool:
    return bool(fused_params and fused_params.get(FUSED_PARAM_REGISTER_TBE_BOOL, False))


def get_fused_param_tbe_row_alignment(fused_params: Optional[Dict[str, Any]]) -> Optional[int]:
    return None if not fused_params else fused_params.get(FUSED_PARAM_TBE_ROW_ALIGNMENT)


def fused_param_bounds_check_mode(fused_params: Optional[Dict[str, Any]]) -> Optional[Any]:
    return None if not fused_params else fused_params.get(FUSED_PARAM_BOUNDS_CHECK_MODE)


def fused_param_lengths_to_offsets_lookup(fused_params: Optional[Dict[str, Any]]) -> bool:
    return bool(fused_params and fused_params.get(FUSED_PARAM_LENGTHS_TO_OFFSETS_LOOKUP, False))


def is_fused_param_quant_state_dict_split_scale_bias(fused_params: Optional[Dict[str, Any]]) -> bool:
    return bool(fused_params and fused_params.get(FUSED_PARAM_QUANT_STATE_DICT_SPLIT_SCALE_BIAS, False))


def tbe_fused_params(fused_params: Optional[Dict[str, Any]]) -> Optional[Dict[str, Any]]:
    """The subset that is handed to the kernel constructor (internal ``__register_*`` switches stripped)."""
    if not fused_params:
        return None
    return {k: v for k, v in fused_params.items() if k not in _INTERNAL}


def get_embedding_table_index_type(fused_params: Optional[Dict[str, Any]]) -> torch.dtype:
    return (fused_params or {}).get("embedding_table_index_type", torch.int64)


def get_embedding_table_offset_type(fused_params: Optional[Dict[str, Any]]) -> torch.dtype:
    return (fused_params or {}).get("embedding_table_offset_type", torch.int64)
