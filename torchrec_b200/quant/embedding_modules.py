"""Quantized (inference) embedding collections (reference torchrec/quant/embedding_modules.py:206-1359).

``EmbeddingBagCollection.from_float(ebc)`` / ``EmbeddingCollection.from_float(ec)`` build modules whose tables are
row-wise INT8 / INT4 / INT2, FP16 or block-scaled FP8 and run the sm_90a quantized lookup kernel. State-dict layout
follows the reference: ``embedding_bags.<table>.weight`` (uint8 rows incl. the fused scale/bias tail)."""
from __future__ import annotations

import copy
from typing import Any, Callable, Dict, List, Optional, Tuple

import torch
import torch.nn as nn

from ..modules.embedding_configs import DATA_TYPE_NUM_BITS, DataType, EmbeddingBagConfig, EmbeddingConfig, PoolingType, dtype_to_data_type
from ..modules.embedding_modules import (
    EmbeddingBagCollection as OriginalEmbeddingBagCollection,
    EmbeddingBagCollectionInterface,
    EmbeddingCollection as OriginalEmbeddingCollection,
    EmbeddingCollectionInterface,
    get_embedding_names_by_table,
)
from ..ops.quant_tbe import QuantTableBatchedEmbeddingBags, quantize_rows
from ..sparse.jagged_tensor import JaggedTensor, KeyedJaggedTensor, KeyedTensor

MODULE_ATTR_REGISTER_TBES_BOOL: str = "__register_tbes_in_named_modules"
MODULE_ATTR_QUANT_STATE_DICT_SPLIT_SCALE_BIAS: str = "__quant_state_dict_split_scale_bias"
MODULE_ATTR_ROW_ALIGNMENT_INT: str = "__register_row_alignment_in_named_modules"
MODULE_ATTR_EMB_CONFIG_NAME_TO_NUM_ROWS_POST_PRUNING_DICT: str = "__emb_name_to_num_rows_post_pruning"
DEFAULT_ROW_ALIGNMENT = 16


def quant_prep_enable_quant_state_dict_split_scale_bias(module: nn.Module) -> None:
    setattr(module, MODULE_ATTR_QUANT_STATE_DICT_SPLIT_SCALE_BIAS, True)


def quant_prep_enable_register_tbes(module: nn.Module, module_types: List[type]) -> None:
    for m in module.modules():
        if type(m) in module_types:
            setattr(m, MODULE_ATTR_REGISTER_TBES_BOOL, True)


def quant_prep_customize_row_alignment(module: nn.Module, module_types: List[type], row_alignment: int) -> None:
    for m in module.modules():
        if type(m) in module_types:
            setattr(m, MODULE_ATTR_ROW_ALIGNMENT_INT, row_alignment)


def quantize_state_dict(module: nn.Module, table_name_to_quantized_weights: Dict[str, Tuple[torch.Tensor, Optional[torch.Tensor]]],
                        table_name_to_data_type: Dict[str, DataType], table_name_to_num_embeddings_post_pruning: Optional[Dict[str, int]] = None) -> torch.device:
    """Quantize every ``*.weight`` of ``module.state_dict()`` row-wise into ``table_name_to_quantized_weights``."""
    device = torch.device("cpu")
    for key, tensor in module.state_dict().items():
        splits = key.split(".")
        assert splits[-1] == "weight"
        table_name = splits[-2]
        data_type = table_name_to_data_type[table_name]
        t = tensor
        if hasattr(t, "local_shards"):
            t = t.local_shards()[0].tensor
        if t.is_meta:
            continue
        device = t.device
        if table_name_to_num_embeddings_post_pruning and table_name in table_name_to_num_embeddings_post_pruning:
            t = t[: table_name_to_num_embeddings_post_pruning[table_name]]
        q = quantize_rows(t.float(), data_type, DEFAULT_ROW_ALIGNMENT)
        table_name_to_quantized_weights[table_name] = (q, None)
    return device


def _data_type_of(qconfig_dtype: Any, per_table: Optional[Dict[str, Any]], name: str) -> DataType:
    dt = per_table.get(name) if per_table and name in per_table else qconfig_dtype
    if isinstance(dt, DataType):
        return dt
    return dtype_to_data_type(dt)


class EmbeddingBagCollection(EmbeddingBagCollectionInterface):
    """Quantized EmbeddingBagCollection: KJT -> KeyedTensor via the quantized table-batched kernel."""

    def __init__(self, tables: List[EmbeddingBagConfig], is_weighted: bool, device: torch.device, output_dtype: torch.dtype = torch.float,
                 table_name_to_quantized_weights: Optional[Dict[str, Tuple[torch.Tensor, Optional[torch.Tensor]]]] = None, register_tbes: bool = False,
                 quant_state_dict_split_scale_bias: bool = False, row_alignment: int = DEFAULT_ROW_ALIGNMENT, cache_features_order: bool = False) -> None:
        super().__init__()
        self._is_weighted = is_weighted
        self._embedding_bag_configs: List[EmbeddingBagConfig] = tables
        self._device = torch.device(device)
        self._output_dtype = output_dtype
        self.row_alignment = row_alignment
        names = set()
        for t in tables:
            if t.name in names:
                raise ValueError(f"Duplicate table name {t.name}")
            names.add(t.name)
        # one kernel per pooling type
        self._groups: List[Tuple[PoolingType, List[int]]] = []
        for pt in (PoolingType.SUM, PoolingType.MEAN):
            idxs = [i for i, t in enumerate(tables) if t.pooling == pt]
            if idxs:
                self._groups.append((pt, idxs))
        self._tbes = nn.ModuleList()
        self._group_features: List[List[str]] = []
        for pt, idxs in self._groups:
            specs = [(tables[i].name, tables[i].num_embeddings_post_pruning or tables[i].num_embeddings, tables[i].embedding_dim, tables[i].data_type) for i in idxs]
            fmap = [k for k, i in enumerate(idxs) for _ in tables[i].feature_names]
            tbe = QuantTableBatchedEmbeddingBags(specs, fmap, pooling_mode=1 if pt == PoolingType.MEAN else 0, output_dtype=output_dtype,
                                                 device=self._device, row_alignment=row_alignment)
            if table_name_to_quantized_weights and self._device.type != "meta":
                for k, i in enumerate(idxs):
                    if tables[i].name in table_name_to_quantized_weights:
                        q = table_name_to_quantized_weights[tables[i].name][0]
                        tbe.split_embedding_weights()[k].copy_(q.to(self._device))
            self._tbes.append(tbe)
            self._group_features.append([f for i in idxs for f in tables[i].feature_names])
        self._embedding_names: List[str] = [n for ns in get_embedding_names_by_table(tables) for n in ns]
        self._length_per_key: List[int] = [t.embedding_dim for t in tables for _ in t.feature_names]
        self._feature_names: List[str] = [f for t in tables for f in t.feature_names]
        # output column order = table order; group outputs are re-ordered once
        order = []
        for (pt, idxs), feats in zip(self._groups, self._group_features):
            for i in idxs:
                for f in tables[i].feature_names:
                    order.append((i, f))
        flat = [(i, f) for i, t in enumerate(tables) for f in t.feature_names]
        self._needs_regroup = order != flat
        self._group_key_order = order
        self._flat_key_order = flat
        self.embedding_bags = nn.ModuleDict({t.name: nn.Module() for t in tables})
        for (pt, idxs), tbe in zip(self._groups, self._tbes):
            for k, i in enumerate(idxs):
                self.embedding_bags[tables[i].name].register_buffer("weight", tbe.split_embedding_weights()[k], persistent=True)

    def forward(self, features: KeyedJaggedTensor) -> KeyedTensor:
        outs = []
        for feats, tbe in zip(self._group_features, self._tbes):
            sub = features if feats == features.keys() else features.permute([features.keys().index(f) for f in feats])
            psw = sub.weights_or_none() if self._is_weighted else None
            outs.append(tbe(sub.values(), sub.offsets(), psw, batch_size=sub.stride()).to(self._output_dtype))
        vals = outs[0] if len(outs) == 1 else torch.cat(outs, dim=1)
        if self._needs_regroup:
            dims = {k: self._embedding_bag_configs[k[0]].embedding_dim for k in self._group_key_order}
            start, c = {}, 0
            for k in self._group_key_order:
                start[k] = c
                c += dims[k]
            idx = torch.cat([torch.arange(start[k], start[k] + dims[k], device=vals.device) for k in self._flat_key_order])
            vals = vals.index_select(1, idx)
        return KeyedTensor(keys=self._embedding_names, length_per_key=self._length_per_key, values=vals)

    @classmethod
    def from_float(cls, module: OriginalEmbeddingBagCollection, use_precomputed_fake_quant: bool = False) -> "EmbeddingBagCollection":
        qconfig = getattr(module, "qconfig", None)
        assert qconfig is not None, "EmbeddingBagCollection input float module must have qconfig defined"
        per_table = getattr(qconfig, "per_table_weight_dtype", None)
        w = qconfig.weight
        wdtype = w().dtype if callable(w) else w
        tables = []
        name_to_dt = {}
        for cfg in module.embedding_bag_configs():
            dt = _data_type_of(wdtype, per_table, cfg.name)
            c = copy.deepcopy(cfg)
            c.data_type = dt
            tables.append(c)
            name_to_dt[cfg.name] = dt
        qw: Dict[str, Tuple[torch.Tensor, Optional[torch.Tensor]]] = {}
        device = quantize_state_dict(module, qw, name_to_dt, getattr(module, MODULE_ATTR_EMB_CONFIG_NAME_TO_NUM_ROWS_POST_PRUNING_DICT, None))
        act = qconfig.activation
        out_dtype = act().dtype if callable(act) else (act if isinstance(act, torch.dtype) else torch.float)
        return cls(tables, module.is_weighted(), device=device, output_dtype=out_dtype, table_name_to_quantized_weights=qw,
                   register_tbes=getattr(module, MODULE_ATTR_REGISTER_TBES_BOOL, False),
                   quant_state_dict_split_scale_bias=getattr(module, MODULE_ATTR_QUANT_STATE_DICT_SPLIT_SCALE_BIAS, False),
                   row_alignment=getattr(module, MODULE_ATTR_ROW_ALIGNMENT_INT, DEFAULT_ROW_ALIGNMENT))

    def embedding_bag_configs(self) -> List[EmbeddingBagConfig]:
        return self._embedding_bag_configs

    def is_weighted(self) -> bool:
        return self._is_weighted

    def output_dtype(self) -> torch.dtype:
        return self._output_dtype

    @property
    def device(self) -> torch.device:
        return self._device


class EmbeddingCollection(EmbeddingCollectionInterface):
    """Quantized EmbeddingCollection (sequence embeddings)."""

    def __init__(self, tables: List[EmbeddingConfig], device: torch.device, need_indices: bool = False, output_dtype: torch.dtype = torch.float,
                 table_name_to_quantized_weights: Optional[Dict[str, Tuple[torch.Tensor, Optional[torch.Tensor]]]] = None, register_tbes: bool = False,
                 quant_state_dict_split_scale_bias: bool = False, row_alignment: int = DEFAULT_ROW_ALIGNMENT, cache_features_order: bool = False) -> None:
        super().__init__()
        self._embedding_configs = tables
        self._need_indices = need_indices
        self._output_dtype = output_dtype
        self._device = torch.device(device)
        self._embedding_dim = tables[0].embedding_dim if tables else -1
        for t in tables:
            if t.embedding_dim != self._embedding_dim:
                raise ValueError("All tables in a EmbeddingCollection are required to have same embedding dimension.")
        specs = [(t.name, t.num_embeddings_post_pruning or t.num_embeddings, t.embedding_dim, t.data_type) for t in tables]
        fmap = [k for k, t in enumerate(tables) for _ in t.feature_names]
        self._tbe = QuantTableBatchedEmbeddingBags(specs, fmap, pooling_mode=2, output_dtype=output_dtype, device=self._device, row_alignment=row_alignment)
        if table_name_to_quantized_weights and self._device.type != "meta":
            for k, t in enumerate(tables):
                if t.name in table_name_to_quantized_weights:
                    self._tbe.split_embedding_weights()[k].copy_(table_name_to_quantized_weights[t.name][0].to(self._device))
        self._feature_names = [f for t in tables for f in t.feature_names]
        self._embedding_names_by_table = get_embedding_names_by_table(tables)
        self._embedding_names = [n for ns in self._embedding_names_by_table for n in ns]
        self.embeddings = nn.ModuleDict({t.name: nn.Module() for t in tables})
        for k, t in enumerate(tables):
            self.embeddings[t.name].register_buffer("weight", self._tbe.split_embedding_weights()[k], persistent=True)

    def forward(self, features: KeyedJaggedTensor) -> Dict[str, JaggedTensor]:
        sub = features if self._feature_names == features.keys() else features.permute([features.keys().index(f) for f in self._feature_names])
        emb = self._tbe(sub.values(), sub.offsets(), None, batch_size=sub.stride()).to(self._output_dtype)
        lpk = sub.length_per_key()
        parts = torch.split(emb, lpk, dim=0)
        vals = torch.split(sub.values(), lpk) if self._need_indices else None
        B = sub.stride()
        lengths = sub.lengths().view(len(self._feature_names), B)
        return {name: JaggedTensor(values=parts[i], lengths=lengths[i], weights=vals[i] if vals is not None else None)
                for i, name in enumerate(self._embedding_names)}

    @classmethod
    def from_float(cls, module: OriginalEmbeddingCollection, use_precomputed_fake_quant: bool = False) -> "EmbeddingCollection":
        qconfig = getattr(module, "qconfig", None)
        assert qconfig is not None, "EmbeddingCollection input float module must have qconfig defined"
        per_table = getattr(qconfig, "per_table_weight_dtype", None)
        w = qconfig.weight
        wdtype = w().dtype if callable(w) else w
        tables, name_to_dt = [], {}
        for cfg in module.embedding_configs():
            dt = _data_type_of(wdtype, per_table, cfg.name)
            c = copy.deepcopy(cfg)
            c.data_type = dt
            tables.append(c)
            name_to_dt[cfg.name] = dt
        qw: Dict[str, Tuple[torch.Tensor, Optional[torch.Tensor]]] = {}
        device = quantize_state_dict(module, qw, name_to_dt)
        act = qconfig.activation
        out_dtype = act().dtype if callable(act) else (act if isinstance(act, torch.dtype) else torch.float)
        return cls(tables, device=device, need_indices=module.need_indices(), output_dtype=out_dtype, table_name_to_quantized_weights=qw)

    def embedding_configs(self) -> List[EmbeddingConfig]:
        return self._embedding_configs

    def need_indices(self) -> bool:
        return self._need_indices

    def embedding_dim(self) -> int:
        return self._embedding_dim

    def embedding_names_by_table(self) -> List[List[str]]:
        return self._embedding_names_by_table

    def output_dtype(self) -> torch.dtype:
        return self._output_dtype

    @property
    def device(self) -> torch.device:
        return self._device


# ---- feature-processed and managed-collision variants ----------------------------------------------------------------------------------------------------
MODULE_ATTR_CACHE_FEATURES_ORDER = "__cache_features_order"


def for_each_module_of_type_do(module: nn.Module, module_types: List[type], op: Callable[[nn.Module], None]) -> None:
    """``op(m)`` for every sub-module (the root included) whose type is one of ``module_types``."""
    for m in module.modules():
        if any(type(m) is t for t in module_types):
            op(m)


def quant_prep_enable_quant_state_dict_split_scale_bias_for_types(module: nn.Module, module_types: List[type]) -> None:
    """Mark the float modules of these types: their quantized versions keep scale / bias as separate state-dict tensors."""
    for_each_module_of_type_do(module, module_types, lambda m: setattr(m, MODULE_ATTR_QUANT_STATE_DICT_SPLIT_SCALE_BIAS, True))


def quant_prep_enable_cache_features_order(module: nn.Module, module_types: List[type]) -> None:
    """Mark the float modules of these types: their quantized versions remember the feature permutation of the first batch (inputs
    always arrive in the same key order when serving)."""
    for_each_module_of_type_do(module, module_types, lambda m: setattr(m, MODULE_ATTR_CACHE_FEATURES_ORDER, True))


def _quantized_tables(configs, qconfig, pruning: Optional[Dict[str, int]] = None):
    per_table = getattr(qconfig, "per_table_weight_dtype", None)
    w = qconfig.weight
    wdtype = w().dtype if callable(w) else w
    tables, name_to_dt = [], {}
    for cfg in configs:
        c = copy.deepcopy(cfg)
        c.data_type = _data_type_of(wdtype, per_table, cfg.name)
        if pruning and cfg.name in pruning:
            c.num_embeddings_post_pruning = pruning[cfg.name]
        tables.append(c)
        name_to_dt[cfg.name] = c.data_type
    act = qconfig.activation
    out_dtype = act().dtype if callable(act) else (act if isinstance(act, torch.dtype) else torch.float)
    return tables, name_to_dt, out_dtype


class FeatureProcessedEmbeddingBagCollection(EmbeddingBagCollection):
    """Quantized bags behind (float) feature processors: ``forward`` applies the processors to the KJT, then looks up
    (reference quant/embedding_modules.py:636)."""

    def __init__(self, tables: List[EmbeddingBagConfig], is_weighted: bool, device: torch.device, output_dtype: torch.dtype = torch.float,
                 table_name_to_quantized_weights: Optional[Dict[str, Tuple[torch.Tensor, Optional[torch.Tensor]]]] = None, register_tbes: bool = False,
                 quant_state_dict_split_scale_bias: bool = False, row_alignment: int = DEFAULT_ROW_ALIGNMENT, feature_processor: Optional[nn.Module] = None,
                 cache_features_order: bool = False) -> None:
        super().__init__(tables, is_weighted, device, output_dtype, table_name_to_quantized_weights, register_tbes, quant_state_dict_split_scale_bias, row_alignment,
                         cache_features_order)
        assert feature_processor is not None, "Use EmbeddingBagCollection for no feature_processor"
        self.feature_processor = feature_processor

    def forward(self, features: KeyedJaggedTensor) -> KeyedTensor:
        return super().forward(self.feature_processor(features))

    def _get_name(self) -> str:
        return "QuantFeatureProcessedEmbeddingBagCollection"

    @classmethod
    def from_float(cls, module: nn.Module, use_precomputed_fake_quant: bool = False) -> "FeatureProcessedEmbeddingBagCollection":
        assert hasattr(module, "qconfig"), "FeatureProcessedEmbeddingBagCollection input float module must have qconfig defined"
        ebc = module._embedding_bag_collection
        pruning = getattr(module, MODULE_ATTR_EMB_CONFIG_NAME_TO_NUM_ROWS_POST_PRUNING_DICT, None)
        tables, name_to_dt, out_dtype = _quantized_tables(ebc.embedding_bag_configs(), module.qconfig, pruning)
        qw: Dict[str, Tuple[torch.Tensor, Optional[torch.Tensor]]] = {}
        device = quantize_state_dict(ebc, qw, name_to_dt, pruning)
        fp = module._feature_processors
        return cls(tables, ebc.is_weighted(), device=device, output_dtype=out_dtype, table_name_to_quantized_weights=qw,
                   register_tbes=getattr(module, MODULE_ATTR_REGISTER_TBES_BOOL, False),
                   quant_state_dict_split_scale_bias=getattr(ebc, MODULE_ATTR_QUANT_STATE_DICT_SPLIT_SCALE_BIAS, False),
                   row_alignment=getattr(ebc, MODULE_ATTR_ROW_ALIGNMENT_INT, DEFAULT_ROW_ALIGNMENT), feature_processor=fp.to(device) if device.type != "meta" else fp,
                   cache_features_order=getattr(module, MODULE_ATTR_CACHE_FEATURES_ORDER, False))


def _freeze_mcc(mcc: nn.Module) -> None:
    """Serving: the managed-collision modules only look ids up (no insertion, no eviction)."""
    for m in getattr(mcc, "_managed_collision_modules", {}).values():
        if hasattr(m, "reset_inference_mode"):
            m.reset_inference_mode()
        elif hasattr(m, "_is_inference"):
            m._is_inference = True
        m.train(False)


class QuantManagedCollisionEmbeddingCollection(EmbeddingCollection):
    """Quantized sequence embeddings behind a managed-collision collection: raw ids are remapped to table slots (read-only), then
    looked up; ``forward`` returns ``(embeddings, remapped features)`` (reference quant/embedding_modules.py:1050)."""

    def __init__(self, tables: List[EmbeddingConfig], device: torch.device, need_indices: bool = False, output_dtype: torch.dtype = torch.float,
                 table_name_to_quantized_weights: Optional[Dict[str, Tuple[torch.Tensor, Optional[torch.Tensor]]]] = None, register_tbes: bool = False,
                 quant_state_dict_split_scale_bias: bool = False, row_alignment: int = DEFAULT_ROW_ALIGNMENT, managed_collision_collection: Optional[nn.Module] = None,
                 return_remapped_features: bool = False, cache_features_order: bool = False) -> None:
        super().__init__(tables, device, need_indices, output_dtype, table_name_to_quantized_weights, register_tbes, quant_state_dict_split_scale_bias, row_alignment,
                         cache_features_order)
        assert managed_collision_collection, "Managed collision collection cannot be None"
        self._managed_collision_collection = managed_collision_collection
        self._return_remapped_features = return_remapped_features
        assert [c.name for c in self.embedding_configs()] == [c.name for c in managed_collision_collection.embedding_configs()], \
            "Embedding Collection and Managed Collision Collection must contain the same Embedding Configs"
        _freeze_mcc(managed_collision_collection)

    def forward(self, features: KeyedJaggedTensor):
        features = self._managed_collision_collection(features)
        return super().forward(features), features

    def train(self, mode: bool = True):
        super().train(mode)
        _freeze_mcc(self._managed_collision_collection)  # serving never inserts or evicts, whatever mode the parent model is put in
        return self

    def _get_name(self) -> str:
        return "QuantManagedCollisionEmbeddingCollection"

    @classmethod
    def from_float(cls, module: nn.Module, return_remapped_features: bool = False) -> "QuantManagedCollisionEmbeddingCollection":
        assert hasattr(module, "qconfig"), "QuantManagedCollisionEmbeddingCollection input float module must have qconfig defined"
        ec = module._embedding_module
        tables, name_to_dt, out_dtype = _quantized_tables(ec.embedding_configs(), module.qconfig)
        qw: Dict[str, Tuple[torch.Tensor, Optional[torch.Tensor]]] = {}
        device = quantize_state_dict(ec, qw, name_to_dt)
        return cls(tables, device=device, need_indices=ec.need_indices(), output_dtype=out_dtype, table_name_to_quantized_weights=qw,
                   register_tbes=getattr(module, MODULE_ATTR_REGISTER_TBES_BOOL, False),
                   quant_state_dict_split_scale_bias=getattr(ec, MODULE_ATTR_QUANT_STATE_DICT_SPLIT_SCALE_BIAS, False),
                   row_alignment=getattr(ec, MODULE_ATTR_ROW_ALIGNMENT_INT, DEFAULT_ROW_ALIGNMENT), managed_collision_collection=module._managed_collision_collection,
                   return_remapped_features=return_remapped_features or module._return_remapped_features,
                   cache_features_order=getattr(ec, MODULE_ATTR_CACHE_FEATURES_ORDER, False))


class QuantManagedCollisionEmbeddingBagCollection(EmbeddingBagCollection):
    """Quantized bags behind a managed-collision collection; ``forward`` returns ``(KeyedTensor, remapped features)``."""

    def __init__(self, tables: List[EmbeddingBagConfig], is_weighted: bool, device: torch.device, output_dtype: torch.dtype = torch.float,
                 table_name_to_quantized_weights: Optional[Dict[str, Tuple[torch.Tensor, Optional[torch.Tensor]]]] = None, register_tbes: bool = False,
                 quant_state_dict_split_scale_bias: bool = False, row_alignment: int = DEFAULT_ROW_ALIGNMENT, managed_collision_collection: Optional[nn.Module] = None,
                 return_remapped_features: bool = False, cache_features_order: bool = False) -> None:
        super().__init__(tables, is_weighted, device, output_dtype, table_name_to_quantized_weights, register_tbes, quant_state_dict_split_scale_bias, row_alignment,
                         cache_features_order)
        assert managed_collision_collection, "Managed collision collection cannot be None"
        self._managed_collision_collection = managed_collision_collection
        self._return_remapped_features = return_remapped_features
        assert [c.name for c in self.embedding_bag_configs()] == [c.name for c in managed_collision_collection.embedding_configs()], \
            "Embedding Bag Collection and Managed Collision Collection must contain the same Embedding Configs"
        _freeze_mcc(managed_collision_collection)

    def forward(self, features: KeyedJaggedTensor):
        features = self._managed_collision_collection(features)
        return super().forward(features), features

    def train(self, mode: bool = True):
        super().train(mode)
        _freeze_mcc(self._managed_collision_collection)  # serving never inserts or evicts, whatever mode the parent model is put in
        return self

    def _get_name(self) -> str:
        return "QuantManagedCollisionEmbeddingBagCollection"

    @classmethod
    def from_float(cls, module: nn.Module, return_remapped_features: bool = False) -> "QuantManagedCollisionEmbeddingBagCollection":
        assert hasattr(module, "qconfig"), "QuantManagedCollisionEmbeddingBagCollection input float module must have qconfig defined"
        ebc = module._embedding_module
        tables, name_to_dt, out_dtype = _quantized_tables(ebc.embedding_bag_configs(), module.qconfig)
        qw: Dict[str, Tuple[torch.Tensor, Optional[torch.Tensor]]] = {}
        device = quantize_state_dict(ebc, qw, name_to_dt)
        return cls(tables, ebc.is_weighted(), device=device, output_dtype=out_dtype, table_name_to_quantized_weights=qw,
                   register_tbes=getattr(module, MODULE_ATTR_REGISTER_TBES_BOOL, False),
                   quant_state_dict_split_scale_bias=getattr(ebc, MODULE_ATTR_QUANT_STATE_DICT_SPLIT_SCALE_BIAS, False),
                   row_alignment=getattr(ebc, MODULE_ATTR_ROW_ALIGNMENT_INT, DEFAULT_ROW_ALIGNMENT), managed_collision_collection=module._managed_collision_collection,
                   return_remapped_features=return_remapped_features or module._return_remapped_features,
                   cache_features_order=getattr(ebc, MODULE_ATTR_CACHE_FEATURES_ORDER, False))
