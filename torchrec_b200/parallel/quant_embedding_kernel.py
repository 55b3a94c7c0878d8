"""Per-group inference kernels over row-wise quantized tables.

Reference: ``torchrec/distributed/quant_embedding_kernel.py`` (``QuantBatchedEmbeddingBag`` :247-511, ``QuantBatchedEmbedding`` :514-711,
``_quantize_weight`` :100-120, ``_copy_config`` :57-97). The reference instantiates FBGEMM ``IntNBitTableBatchedEmbeddingBagsCodegen``; here the kernel is
``ops/quant_tbe.py: QuantTableBatchedEmbeddingBags`` (``ops/csrc/tbe_quant.cu``: INT8 / INT4 / INT2 / FP16 / FP8 rows with a fused fp16 scale+bias,
16-byte row alignment).
"""
from __future__ import annotations

import copy
from typing import Any, Dict, Iterator, List, Optional, Tuple

import torch
import torch.distributed as dist
from torch import nn

from ..modules.embedding_configs import DataType, PoolingType, data_type_to_dtype
from ..ops.quant_tbe import QuantTableBatchedEmbeddingBags, dequantize_rows, quantize_rows, row_bytes
from ..sparse.jagged_tensor import KeyedJaggedTensor
from .embedding_kernel import BaseEmbedding, get_state_dict
from .embedding_types import GroupedEmbeddingConfig, ShardedEmbeddingTable, quant_table_placement


def _copy_config(original: GroupedEmbeddingConfig, data_type: DataType, sparse_type: Any = None, device: Optional[torch.device] = None) -> GroupedEmbeddingConfig:
    """The same group with every table re-typed to ``data_type`` (rows are re-sized by the kernel's row layout)."""
    cfg = copy.deepcopy(original)
    cfg.data_type = data_type
    for t in cfg.embedding_tables:
        t.data_type = data_type
    return cfg


def _quantize_weight(state_dict: Dict[str, torch.Tensor], data_type: DataType) -> List[Tuple[torch.Tensor, Optional[torch.Tensor]]]:
    """float table -> (quantized uint8 rows, fp16 scale/bias columns) per table, in ``state_dict`` order."""
    out: List[Tuple[torch.Tensor, Optional[torch.Tensor]]] = []
    for w in state_dict.values():
        w = w.float() if isinstance(w, torch.Tensor) else w.local_shards()[0].tensor.float()
        q = quantize_rows(w, data_type)
        out.append((q, _scale_bias_tail(q, w.shape[1], data_type)))
    return out


_NBITS = {DataType.INT8: 8, DataType.INT4: 4, DataType.INT2: 2}


def _scale_bias_tail(q: torch.Tensor, dim: int, data_type: DataType) -> Optional[torch.Tensor]:
    """View of the fused fp16 (scale, bias) pair that follows the packed payload of an INT-N row; None for float rows."""
    if data_type not in _NBITS:
        return None
    payload = (dim * _NBITS[data_type] + 7) // 8
    return q[:, payload : payload + 4]


def _get_runtime_device(device: Optional[torch.device], config: GroupedEmbeddingConfig, shard_index: Optional[int] = None) -> torch.device:
    if device is not None and device.type != "meta":
        return device
    if device is not None and device.type == "meta":
        return torch.device("cpu")
    return torch.device("cuda", torch.cuda.current_device()) if torch.cuda.is_available() else torch.device("cpu")


def _unwrap_kjt(features: KeyedJaggedTensor) -> Tuple[torch.Tensor, torch.Tensor, Optional[torch.Tensor]]:
    """(int32 indices, int32 offsets, weights) - the inference kernels index with 32-bit ids (reference :181-191)."""
    return features.values().int(), features.offsets().int(), features.weights_or_none()


class _QuantBase(BaseEmbedding):
    _POOLED = True

    def __init__(self, config: GroupedEmbeddingConfig, pg: Optional[dist.ProcessGroup] = None, device: Optional[torch.device] = None,
                 fused_params: Optional[Dict[str, Any]] = None, shard_index: Optional[int] = None) -> None:
        super().__init__()
        self._config = config
        self._pg = pg
        self._pooling = config.pooling
        self._is_weighted = config.is_weighted
        self._quant_state_dict_split_scale_bias = bool((fused_params or {}).get("quant_state_dict_split_scale_bias", False))
        dev = _get_runtime_device(device, config, shard_index)
        out_dtype = (fused_params or {}).get("output_dtype", torch.float32)
        if isinstance(out_dtype, DataType):
            out_dtype = data_type_to_dtype(out_dtype)
        mode = 2 if not self._POOLED else (1 if config.pooling == PoolingType.MEAN else 0)
        # per table: HBM / pinned host / pinned host + HBM row cache, from the table's compute kernel (quant / quant_uvm / quant_uvm_caching)
        placement = [quant_table_placement(t.compute_kernel, None, {**(fused_params or {}), **(config.fused_params or {}), **(t.fused_params or {})})
                     for t in config.embedding_tables]
        self._emb_module = QuantTableBatchedEmbeddingBags(
            embedding_specs=[(t.name, t.local_rows, t.local_cols, t.data_type) for t in config.embedding_tables],
            feature_table_map=[i for i, t in enumerate(config.embedding_tables) for _ in t.feature_names],
            pooling_mode=mode, output_dtype=out_dtype, device=dev, row_alignment=int((fused_params or {}).get("row_alignment", 16)),
            locations=[loc for loc, _ in placement], cache_load_factor=[clf for _, clf in placement],
        )
        self._runtime_device = dev

    @property
    def config(self) -> GroupedEmbeddingConfig:
        return self._config

    @property
    def emb_module(self) -> QuantTableBatchedEmbeddingBags:
        return self._emb_module

    def get_tbes_to_register(self) -> Dict[QuantTableBatchedEmbeddingBags, GroupedEmbeddingConfig]:
        return {self._emb_module: self._config}

    def forward(self, features: KeyedJaggedTensor) -> torch.Tensor:
        idx, off, w = _unwrap_kjt(features)
        F = max(len(self._emb_module.feature_table_map), 1)
        return self._emb_module(idx, off, w if (self._POOLED and self._is_weighted) else None, batch_size=(off.numel() - 1) // F)

    def split_embedding_weights(self) -> List[Tuple[torch.Tensor, Optional[torch.Tensor]]]:
        """(uint8 rows, scale/bias bytes or None) per table - the pair layout FBGEMM's ``split_embedding_weights(split_scale_shifts=True)`` returns."""
        out = []
        for t, w in zip(self._config.embedding_tables, self._emb_module.split_embedding_weights()):
            out.append((w, _scale_bias_tail(w, t.local_cols, t.data_type)))
        return out

    def named_split_embedding_weights(self, prefix: str = "", recurse: bool = True, remove_duplicate: bool = True) -> Iterator[Tuple[str, torch.Tensor]]:
        for t, (w, _) in zip(self._config.embedding_tables, self.split_embedding_weights()):
            yield (f"{prefix}.{t.name}.weight" if prefix else f"{t.name}.weight"), w

    def state_dict(self, destination: Optional[Dict[str, Any]] = None, prefix: str = "", keep_vars: bool = False) -> Dict[str, Any]:  # type: ignore[override]
        return get_state_dict(self._config.embedding_tables, [w for w, _ in self.split_embedding_weights()], self._pg, destination, prefix)

    def named_buffers(self, prefix: str = "", recurse: bool = True, remove_duplicate: bool = True) -> Iterator[Tuple[str, torch.Tensor]]:
        for t, (w, _) in zip(self._config.embedding_tables, self.split_embedding_weights()):
            yield (f"{prefix}.{t.name}.weight" if prefix else f"{t.name}.weight"), w

    def named_parameters(self, prefix: str = "", recurse: bool = True, remove_duplicate: bool = True) -> Iterator[Tuple[str, nn.Parameter]]:
        yield from ()

    @classmethod
    def from_float(cls, module: BaseEmbedding, use_precomputed_fake_quant: bool = False) -> "_QuantBase":
        """Quantize a trained float kernel's tables row by row into a new inference kernel (reference :478-511)."""
        cfg = module.config
        data_type = getattr(getattr(module, "qconfig", None), "data_type", None) or DataType.INT8
        ret = cls(_copy_config(cfg, data_type), pg=getattr(module, "_pg", None), device=next(iter(module.split_embedding_weights())).device)
        for i, w in enumerate(module.split_embedding_weights()):
            ret._emb_module.assign_from_float(i, w.float())
        return ret


class QuantBatchedEmbeddingBag(_QuantBase):
    """Pooled quantized lookup (reference :247)."""

    _POOLED = True


class QuantBatchedEmbedding(_QuantBase):
    """Sequence quantized lookup: output ``[sum(lengths), D]`` (reference :514)."""

    _POOLED = False


class IntNBitTableBatchedEmbeddingBagsCodegenWithLength(QuantTableBatchedEmbeddingBags):
    """Variant taking ``lengths`` instead of ``offsets`` (reference :227-244: keeps the cumsum out of the traced graph)."""

    def forward(self, indices: torch.Tensor, lengths: torch.Tensor, per_sample_weights: Optional[torch.Tensor] = None) -> torch.Tensor:  # type: ignore[override]
        offsets = torch.zeros(lengths.numel() + 1, dtype=torch.int32, device=lengths.device)
        torch.cumsum(lengths.reshape(-1), 0, out=offsets[1:])
        return super().forward(indices, offsets, per_sample_weights)
