"""Embedding runtime types (reference torchrec/distributed/embedding_types.py)."""
from __future__ import annotations

import abc
import copy
from dataclasses import dataclass, field
from enum import Enum, unique
import logging
from typing import Any, Callable, Dict, Generic, Iterator, List, Optional, Tuple, Type, TypeVar, Union

import torch
from torch import nn

logger = logging.getLogger(__name__)

from ..modules.embedding_configs import DataType, EmbeddingTableConfig, PoolingType
from ..ops.tbe import OptimType  # noqa: F401  (re-export: reference exposes OptimType here)
from ..sparse.jagged_tensor import KeyedJaggedTensor
from ..streamable import Multistreamable
from .types import (
    EmbeddingModuleShardingPlan,
    ModuleSharder,
    ParameterSharding,
    QuantizedCommCodecs,
    ShardedModule,
    ShardingType,
    ShardMetadata,
)


@unique
class EmbeddingComputeKernel(Enum):
    DENSE = "dense"  # dense gradients, external optimizer (DP tables)
    FUSED = "fused"  # HBM tables, optimizer fused into the backward kernel
    FUSED_UVM = "fused_uvm"  # host-resident table accessed over PCIe/C2C
    FUSED_UVM_CACHING = "fused_uvm_caching"  # host table + HBM cache
    QUANT = "quant"  # row-wise quantized inference tables
    QUANT_UVM = "quant_uvm"
    QUANT_UVM_CACHING = "quant_uvm_caching"
    KEY_VALUE = "key_value"
    SSD_VIRTUAL_TABLE = "ssd_virtual_table"
    DRAM_VIRTUAL_TABLE = "dram_virtual_table"
    CUSTOMIZED_KERNEL = "customized_kernel"


def compute_kernel_to_embedding_location(compute_kernel: EmbeddingComputeKernel) -> str:
    if compute_kernel in (EmbeddingComputeKernel.DENSE, EmbeddingComputeKernel.FUSED, EmbeddingComputeKernel.QUANT):
        return "device"
    if compute_kernel in (EmbeddingComputeKernel.FUSED_UVM, EmbeddingComputeKernel.QUANT_UVM, EmbeddingComputeKernel.KEY_VALUE,
                          EmbeddingComputeKernel.SSD_VIRTUAL_TABLE, EmbeddingComputeKernel.DRAM_VIRTUAL_TABLE):
        return "managed"
    return "managed_caching"


_QUANT_KERNELS = (EmbeddingComputeKernel.QUANT, EmbeddingComputeKernel.QUANT_UVM, EmbeddingComputeKernel.QUANT_UVM_CACHING)


def quant_table_placement(compute_kernel: Any, cache_params: Any = None, fused_params: Optional[Dict[str, Any]] = None) -> Tuple[Any, float]:
    """(``EmbeddingLocation``, cache load factor) of a quantized inference table planned with ``compute_kernel``: ``quant`` -> HBM,
    ``quant_uvm`` -> pinned host memory, ``quant_uvm_caching`` -> pinned host memory + HBM row cache. The load factor comes from
    ``cache_params.load_factor``, then ``fused_params["cache_load_factor"]``, then the planner's default (the order of the training
    lookup engine)."""
    from ..ops.tbe import EmbeddingLocation
    from .planner.constants import UVM_CACHING_RATIO

    ck = EmbeddingComputeKernel(compute_kernel) if isinstance(compute_kernel, str) else compute_kernel
    loc = EmbeddingLocation.DEVICE
    if ck in _QUANT_KERNELS:
        loc = {"device": EmbeddingLocation.DEVICE, "managed": EmbeddingLocation.MANAGED,
               "managed_caching": EmbeddingLocation.MANAGED_CACHING}[compute_kernel_to_embedding_location(ck)]
    clf = getattr(cache_params, "load_factor", None) if cache_params is not None else None
    if not clf:
        clf = (fused_params or {}).get("cache_load_factor")
    return loc, float(clf) if clf else UVM_CACHING_RATIO


class KJTList(Multistreamable):
    """List of KJTs (one per sharding group) that crosses streams together."""

    def __init__(self, features: List[KeyedJaggedTensor]) -> None:
        self.features = features

    def __len__(self) -> int:
        return len(self.features)

    def __setitem__(self, key: int, item: KeyedJaggedTensor) -> None:
        self.features[key] = item

    def __getitem__(self, key: int) -> KeyedJaggedTensor:
        return self.features[key]

    def __iter__(self) -> Iterator[KeyedJaggedTensor]:
        return iter(self.features)

    def record_stream(self, stream: torch.Stream) -> None:
        for f in self.features:
            f.record_stream(stream)


class InputDistOutputs(Multistreamable):
    def __init__(self, features: KJTList, unbucketize_permute_tensor: Optional[torch.Tensor] = None,
                 bucket_mapping_tensor: Optional[torch.Tensor] = None, bucketized_length: Optional[torch.Tensor] = None) -> None:
        self.features = features
        self.unbucketize_permute_tensor = unbucketize_permute_tensor
        self.bucket_mapping_tensor = bucket_mapping_tensor
        self.bucketized_length = bucketized_length

    def record_stream(self, stream: torch.Stream) -> None:
        self.features.record_stream(stream)
        for t in (self.unbucketize_permute_tensor, self.bucket_mapping_tensor, self.bucketized_length):
            if t is not None and t.is_cuda:
                t.record_stream(stream)


@dataclass
class ShardedConfig:
    local_rows: int = 0
    local_cols: int = 0


@dataclass
class ShardedMetaConfig(ShardedConfig):
    local_metadata: Optional[ShardMetadata] = None
    global_metadata: Optional[Any] = None
    dtensor_metadata: Optional[Any] = None


@dataclass
class EmbeddingAttributes:
    compute_kernel: EmbeddingComputeKernel = EmbeddingComputeKernel.DENSE


@dataclass
class ShardedEmbeddingTable(ShardedMetaConfig, EmbeddingAttributes, EmbeddingTableConfig):
    """One local shard of a table + its optimizer parameters."""

    fused_params: Optional[Dict[str, Any]] = None


@dataclass
class GroupedEmbeddingConfig:
    data_type: DataType
    pooling: PoolingType
    is_weighted: bool
    has_feature_processor: bool
    compute_kernel: EmbeddingComputeKernel
    embedding_tables: List[ShardedEmbeddingTable]
    fused_params: Optional[Dict[str, Any]] = None

    def feature_hash_sizes(self) -> List[int]:
        return [t.num_embeddings for t in self.embedding_tables for _ in t.feature_names]

    def num_features(self) -> int:
        return sum(t.num_features() for t in self.embedding_tables)

    def dim_sum(self) -> int:
        return sum(t.num_features() * t.local_cols for t in self.embedding_tables)

    def table_names(self) -> List[str]:
        return [t.name for t in self.embedding_tables]

    def feature_names(self) -> List[str]:
        return [f for t in self.embedding_tables for f in t.feature_names]

    def embedding_dims(self) -> List[int]:
        return [t.local_cols for t in self.embedding_tables for _ in t.feature_names]

    def embedding_names(self) -> List[str]:
        return [n for t in self.embedding_tables for n in t.embedding_names]


F = TypeVar("F", bound=Multistreamable)
T = TypeVar("T")
M = TypeVar("M", bound=nn.Module)


class BaseEmbeddingLookup(abc.ABC, nn.Module, Generic[F, T]):
    @abc.abstractmethod
    def forward(self, sparse_features: F) -> T:
        ...


class FeatureShardingMixIn:
    def feature_names(self) -> List[str]:
        raise NotImplementedError

    def feature_names_per_rank(self) -> List[List[str]]:
        raise NotImplementedError

    def features_per_rank(self) -> List[int]:
        raise NotImplementedError


class ListOfKJTList(Multistreamable):
    """Per device one ``KJTList`` (inference: one process drives several devices)."""

    def __init__(self, features: List[KJTList]) -> None:
        self.features_list = features

    def __len__(self) -> int:
        return len(self.features_list)

    def __setitem__(self, key: int, item: KJTList) -> None:
        self.features_list[key] = item

    def __getitem__(self, key: int) -> KJTList:
        return self.features_list[key]

    def __iter__(self) -> Iterator[KJTList]:
        return iter(self.features_list)

    def record_stream(self, stream: torch.Stream) -> None:
        for f in self.features_list:
            f.record_stream(stream)


@dataclass
class DTensorMetadata:
    """How a table shard appears as a DTensor: mesh, placements, global size and stride."""

    mesh: Optional[Any] = None
    placements: Optional[Tuple[Any, ...]] = None
    size: Optional[Tuple[int, ...]] = None
    stride: Optional[Tuple[int, ...]] = None


class BaseEmbeddingUpdate(abc.ABC, nn.Module, Generic[F]):
    """Interface of embedding implementations that take row updates (``forward(embeddings)`` writes them into the tables)."""

    @abc.abstractmethod
    def forward(self, embeddings: F) -> None:
        ...


class BaseGroupedFeatureProcessor(nn.Module):
    """Interface of feature processors applied to the features of one table group: KJT in, KJT out."""

    @abc.abstractmethod
    def forward(self, features: KeyedJaggedTensor) -> KeyedJaggedTensor:
        ...


class _TableFeatureSharding(FeatureShardingMixIn):
    """The features of the tables placed with one sharding type, and which rank looks them up."""

    def __init__(self, names: List[str], per_rank: List[List[str]]) -> None:
        self._names, self._per_rank = names, per_rank

    def feature_names(self) -> List[str]:
        return list(self._names)

    def feature_names_per_rank(self) -> List[List[str]]:
        return [list(x) for x in self._per_rank]

    def features_per_rank(self) -> List[int]:
        return [len(x) for x in self._per_rank]


class ModuleShardingMixIn:
    """Access to a sharded module's sharding scheme: sharding type -> the features sharded that way (per rank)."""

    @property
    def shardings(self) -> Dict[str, FeatureShardingMixIn]:
        plan = getattr(self, "_plan", None)
        cfgs = self.embedding_bag_configs() if hasattr(self, "embedding_bag_configs") else self.embedding_configs() if hasattr(self, "embedding_configs") else None
        if plan is None or cfgs is None:
            raise NotImplementedError
        world = getattr(getattr(self, "_env", None), "world_size", 1)
        out: Dict[str, FeatureShardingMixIn] = {}
        by_type: Dict[str, Tuple[List[str], List[List[str]]]] = {}
        for c in cfgs:
            ps = plan[c.name]
            names, per_rank = by_type.setdefault(ps.sharding_type, ([], [[] for _ in range(world)]))
            names.extend(c.feature_names)
            for r in (ps.ranks if ps.ranks else range(world)):
                if r < world:
                    per_rank[r].extend(c.feature_names)
        for st, (names, per_rank) in by_type.items():
            out[st] = _TableFeatureSharding(names, per_rank)
        return out


Out = TypeVar("Out")
CompIn = TypeVar("CompIn", KJTList, ListOfKJTList, KeyedJaggedTensor)
DistOut = TypeVar("DistOut")
ShrdCtx = TypeVar("ShrdCtx", bound=Multistreamable)


class ShardedEmbeddingModule(ShardedModule[CompIn, DistOut, Out, ShrdCtx], ModuleShardingMixIn):
    """What every model-parallel embedding module offers besides the ``ShardedModule`` stages: its sharding scheme (``shardings``),
    cache prefetch over its lookups, and tracker callbacks - ``register_post_lookup_tracker_fn(fn)``: ``fn(features, embeddings,
    module, extra)`` for every lookup of this rank (the distributed features, i.e. the ids this rank looks up; this framework's fused
    kernels do not materialise per-id embeddings at that point, ``embeddings`` is None - the delta tracker reads rows by id instead),
    ``register_post_odist_tracker_fn(fn)``: ``fn()`` after every output dist has been issued."""

    post_lookup_tracker_fn: Optional[Callable[..., None]] = None
    post_odist_tracker_fn: Optional[Callable[..., None]] = None
    _remove_lookup_tracker: Optional[Callable[[], None]] = None

    def register_post_lookup_tracker_fn(self, record_fn: Callable[..., None]) -> None:
        if self.post_lookup_tracker_fn is not None:
            logger.warning("[ModelDeltaTracker] Custom record function already defined, overriding with new callable")
            if self._remove_lookup_tracker is not None:
                self._remove_lookup_tracker()
        self.post_lookup_tracker_fn = record_fn
        engine = getattr(self, "engine", None)
        if engine is not None:
            self._remove_lookup_tracker = engine.register_lookup_hook(lambda eng, feats: record_fn(feats, None, self, None))

    def register_post_odist_tracker_fn(self, record_fn: Callable[..., None]) -> None:
        if self.post_odist_tracker_fn is not None:
            logger.warning("[ModelDeltaTracker] Compaction function already defined, overriding with new callable")
        self.post_odist_tracker_fn = record_fn

    @property
    def unsharded_module_type(self) -> Type[nn.Module]:
        return nn.Module


class BaseEmbeddingSharder(ModuleSharder[M]):
    """Common sharder behaviour: supported sharding types / compute kernels and fused params
    (reference embedding_types.py:513-606)."""

    def __init__(self, fused_params: Optional[Dict[str, Any]] = None, qcomm_codecs_registry: Optional[Dict[str, QuantizedCommCodecs]] = None) -> None:
        super().__init__(qcomm_codecs_registry=qcomm_codecs_registry)
        self._fused_params = copy.deepcopy(fused_params) if fused_params is not None else fused_params

    def sharding_types(self, compute_device_type: str) -> List[str]:
        types = [
            ShardingType.DATA_PARALLEL.value,
            ShardingType.TABLE_WISE.value,
            ShardingType.COLUMN_WISE.value,
            ShardingType.TABLE_COLUMN_WISE.value,
            ShardingType.ROW_WISE.value,
            ShardingType.TABLE_ROW_WISE.value,
            ShardingType.GRID_SHARD.value,
        ]
        return types

    def compute_kernels(self, sharding_type: str, compute_device_type: str) -> List[str]:
        ret: List[str] = []
        if sharding_type != ShardingType.DATA_PARALLEL.value:
            ret += [EmbeddingComputeKernel.FUSED.value]
            if compute_device_type in {"cuda"}:
                ret += [EmbeddingComputeKernel.FUSED_UVM.value, EmbeddingComputeKernel.FUSED_UVM_CACHING.value, EmbeddingComputeKernel.KEY_VALUE.value]
        else:
            ret.append(EmbeddingComputeKernel.DENSE.value)
        return ret

    @property
    def fused_params(self) -> Optional[Dict[str, Any]]:
        return self._fused_params

    def storage_usage(self, tensor: torch.Tensor, compute_device_type: str, compute_kernel: str) -> Dict[str, int]:
        tensor_bytes = tensor.element_size() * tensor.nelement()
        if compute_kernel in {EmbeddingComputeKernel.FUSED_UVM.value, EmbeddingComputeKernel.FUSED_UVM_CACHING.value,
                              EmbeddingComputeKernel.KEY_VALUE.value}:
            assert compute_device_type in {"cuda"}
            return {"DDR": tensor_bytes}
        storage_map = {"cuda": "HBM", "cpu": "DDR", "mtia": "DDR"}
        return {storage_map[compute_device_type]: tensor_bytes}


class BaseQuantEmbeddingSharder(ModuleSharder[M]):
    def __init__(self, fused_params: Optional[Dict[str, Any]] = None, shardable_params: Optional[List[str]] = None) -> None:
        super().__init__()
        self._fused_params = copy.deepcopy(fused_params) if fused_params is not None else fused_params
        self._shardable_params: List[str] = shardable_params if shardable_params else []

    def sharding_types(self, compute_device_type: str) -> List[str]:
        return [ShardingType.TABLE_WISE.value, ShardingType.ROW_WISE.value, ShardingType.COLUMN_WISE.value]

    def compute_kernels(self, sharding_type: str, compute_device_type: str) -> List[str]:
        ret = [EmbeddingComputeKernel.QUANT.value]
        if compute_device_type in {"cuda"}:
            ret += [EmbeddingComputeKernel.QUANT_UVM.value, EmbeddingComputeKernel.QUANT_UVM_CACHING.value]
        return ret

    @property
    def fused_params(self) -> Optional[Dict[str, Any]]:
        return self._fused_params

    def storage_usage(self, tensor: torch.Tensor, compute_device_type: str, compute_kernel: str) -> Dict[str, int]:
        tensor_bytes = tensor.element_size() * tensor.nelement() + tensor.shape[0] * 4
        if compute_kernel in {EmbeddingComputeKernel.QUANT_UVM.value, EmbeddingComputeKernel.QUANT_UVM_CACHING.value}:
            return {"DDR": tensor_bytes}
        storage_map = {"cuda": "HBM", "cpu": "DDR", "mtia": "DDR"}
        return {storage_map[compute_device_type]: tensor_bytes}
