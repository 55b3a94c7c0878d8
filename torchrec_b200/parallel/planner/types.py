"""Planner data model (reference torchrec/distributed/planner/types.py:55-1480): ``Topology`` (devices,
capacities, bandwidths), ``Storage`` / ``Perf`` algebra, ``Shard`` / ``ShardingOption`` (one candidate
way of sharding one table), ``ParameterConstraints`` and the proposer / partitioner / estimator ABCs."""
from __future__ import annotations

import abc
import hashlib
from copy import deepcopy
from dataclasses import dataclass, field
from enum import Enum
from typing import Any, Dict, List, Optional, Tuple, Union, cast

import torch
from torch import nn

from ...modules.embedding_configs import DataType
from ..embedding_types import EmbeddingComputeKernel
from ..types import CacheParams, KeyValueParams, ModuleSharder, ShardingPlan
from .constants import (
    BATCH_SIZE,
    BWD_COMPUTE_MULTIPLIER,
    CROSS_NODE_BANDWIDTH,
    DDR_CAP,
    DDR_MEM_BW,
    HBM_CAP,
    HBM_MEM_BW,
    HBM_TO_DDR_MEM_BW,
    INTRA_NODE_BANDWIDTH,
    POOLING_FACTOR,
    SSD_CAP,
    SSD_MEM_BW,
    UVM_CACHING_RATIO,
    WEIGHTED_KERNEL_MULTIPLIER,
)


class PlannerErrorType(Enum):
    INSUFFICIENT_STORAGE = "insufficient_storage"
    STRICT_CONSTRAINTS = "strict_constraints"
    PARTITION = "partition"
    PLANNER_INPUT_CONTEXT_MISMATCH = "planner_input_context_mismatch"
    PLAN_LOADING_FAILED = "plan_loading_failed"
    INVALID_RANK_ASSIGNMENT = "invalid_rank_assignment"
    INVALID_COMPUTE_KERNEL = "invalid_compute_kernel"
    MISSING_MODULE_IN_PLAN = "missing_module_in_plan"
    OTHER = "other"


class PlannerError(Exception):
    def __init__(self, message: str, error_type: PlannerErrorType = PlannerErrorType.OTHER) -> None:
        self.error_type = error_type
        super().__init__(message)


@dataclass
class Perf:
    """Per-shard cost breakdown in ms."""

    fwd_compute: float = 0.0
    fwd_comms: float = 0.0
    bwd_compute: float = 0.0
    bwd_comms: float = 0.0
    prefetch_compute: float = 0.0
    input_dist_comms: float = 0.0

    @property
    def total(self) -> float:
        # the row prefetch of UVM-cached tables is pipelined with the previous step's compute
        return max(self.fwd_compute + self.bwd_compute + self.fwd_comms + self.bwd_comms + self.input_dist_comms, self.prefetch_compute)

    def __add__(self, other: "Perf") -> "Perf":
        return Perf(self.fwd_compute + other.fwd_compute, self.fwd_comms + other.fwd_comms, self.bwd_compute + other.bwd_compute,
                    self.bwd_comms + other.bwd_comms, self.prefetch_compute + other.prefetch_compute, self.input_dist_comms + other.input_dist_comms)

    def __hash__(self) -> int:
        return hash((self.fwd_compute, self.fwd_comms, self.bwd_compute, self.bwd_comms, self.prefetch_compute, self.input_dist_comms))


@dataclass
class Storage:
    """HBM / DDR bytes."""

    hbm: int
    ddr: int
    ssd: int = 0

    def __add__(self, other: "Storage") -> "Storage":
        return Storage(self.hbm + other.hbm, self.ddr + other.ddr, self.ssd + other.ssd)

    def __sub__(self, other: "Storage") -> "Storage":
        return Storage(self.hbm - other.hbm, self.ddr - other.ddr, self.ssd - other.ssd)

    def __hash__(self) -> int:
        return hash((self.hbm, self.ddr, self.ssd))

    def fits_in(self, other: "Storage") -> bool:
        return self.hbm <= other.hbm and self.ddr <= other.ddr and self.ssd <= other.ssd


@dataclass
class DeviceHardware:
    rank: int
    storage: Storage
    perf: Perf


class CustomTopologyData:
    """Per-rank overrides of Topology fields (heterogeneous clusters)."""

    supported_fields = ["ddr_cap", "hbm_cap"]

    def __init__(self, data: Dict[str, List[int]], world_size: int) -> None:
        assert all(key in self.supported_fields for key in data.keys()), f"{data.keys()} not supported in CustomTopologyData"
        assert all(len(v) == world_size for v in data.values()), f"{data.values()} must be positive"
        self._data = data
        self._world_size = world_size

    def get_data(self, key: str) -> List[int]:
        assert key in self.supported_fields
        return self._data[key]

    def has_data(self, key: str) -> bool:
        return key in self._data


class CollectiveType(Enum):
    ALL_TO_ALL = "all_to_all"
    REDUCE_SCATTER = "reduce_scatter"
    ALL_GATHER = "all_gather"
    ALL_REDUCE = "all_reduce"


class GeneralizedCommsBandwidth(abc.ABC):
    @abc.abstractmethod
    def get_bw(self, local_world_size: int, world_size: int, collective_type: CollectiveType) -> float:
        ...

    @property
    @abc.abstractmethod
    def intra_host_bw(self) -> float:
        ...

    @property
    @abc.abstractmethod
    def inter_host_bw(self) -> float:
        ...


class BasicCommsBandwidths(GeneralizedCommsBandwidth):
    """Two-level bandwidth model: NVLink inside a domain, NIC across."""

    def __init__(self, inter_host_bw: float = CROSS_NODE_BANDWIDTH, intra_host_bw: float = INTRA_NODE_BANDWIDTH) -> None:
        self.name = "BasicCommsBandwidths"
        self._inter_host_bw = inter_host_bw
        self._intra_host_bw = intra_host_bw

    def get_bw(self, local_world_size: int, world_size: int, collective_type: CollectiveType) -> float:
        return self.intra_host_bw if world_size <= local_world_size else self.inter_host_bw

    @property
    def inter_host_bw(self) -> float:
        return self._inter_host_bw

    @property
    def intra_host_bw(self) -> float:
        return self._intra_host_bw


class Topology:
    """Cluster description used by the planner. Defaults model 8xH100 per NVLink domain."""

    def __init__(
        self,
        world_size: int,
        compute_device: str,
        hbm_cap: Optional[int] = None,
        ddr_cap: Optional[int] = None,
        local_world_size: Optional[int] = None,
        hbm_mem_bw: float = HBM_MEM_BW,
        ddr_mem_bw: float = DDR_MEM_BW,
        hbm_to_ddr_mem_bw: float = HBM_TO_DDR_MEM_BW,
        intra_host_bw: float = INTRA_NODE_BANDWIDTH,
        inter_host_bw: float = CROSS_NODE_BANDWIDTH,
        bwd_compute_multiplier: float = BWD_COMPUTE_MULTIPLIER,
        custom_topology_data: Optional[CustomTopologyData] = None,
        weighted_feature_bwd_compute_multiplier: float = WEIGHTED_KERNEL_MULTIPLIER,
        uneven_sharding_perf_multiplier: float = 1.0,
        generalized_comms_bandwidths: Optional[GeneralizedCommsBandwidth] = None,
        pod_size: Optional[int] = None,
        ssd_cap: Optional[int] = None,
        ssd_mem_bw: float = SSD_MEM_BW,
    ) -> None:
        assert compute_device in ["cpu", "cuda", "mtia"], f"unsupported compute device {compute_device}"
        self._compute_device = compute_device
        self._world_size = world_size
        hbm_per_device = [0] * world_size
        if self._compute_device == "cuda":
            hbm_per_device = [hbm_cap if hbm_cap else HBM_CAP] * world_size
        ddr_cap_per_rank = [ddr_cap if ddr_cap else DDR_CAP] * world_size
        if custom_topology_data:
            if custom_topology_data.has_data("hbm_cap"):
                hbm_per_device = custom_topology_data.get_data("hbm_cap")
            if custom_topology_data.has_data("ddr_cap"):
                ddr_cap_per_rank = custom_topology_data.get_data("ddr_cap")
        ssd = ssd_cap if ssd_cap else SSD_CAP
        self._devices: List[DeviceHardware] = [
            DeviceHardware(rank=rank, storage=Storage(hbm=hbm_per_device[rank], ddr=ddr_cap_per_rank[rank], ssd=ssd), perf=Perf())
            for rank in range(world_size)
        ]
        self._local_world_size: int = local_world_size if local_world_size else min(world_size, 8)
        # an NVLink "pod" (e.g. NVL72) widens the intra group beyond one host
        self._pod_size = pod_size
        if pod_size:
            self._local_world_size = min(world_size, self._local_world_size * pod_size)
        self._hbm_mem_bw = hbm_mem_bw
        self._ddr_mem_bw = ddr_mem_bw
        self._ssd_mem_bw = ssd_mem_bw
        self._hbm_to_ddr_mem_bw = hbm_to_ddr_mem_bw
        self._comms_bandwidths: GeneralizedCommsBandwidth = generalized_comms_bandwidths or BasicCommsBandwidths(
            intra_host_bw=intra_host_bw, inter_host_bw=inter_host_bw)
        self._bwd_compute_multiplier = bwd_compute_multiplier
        self._custom_topology_data = custom_topology_data
        self._weighted_feature_bwd_compute_multiplier = weighted_feature_bwd_compute_multiplier
        self._uneven_sharding_perf_multiplier = uneven_sharding_perf_multiplier

    @property
    def compute_device(self) -> str:
        return self._compute_device

    @property
    def devices(self) -> List[DeviceHardware]:
        return self._devices

    @property
    def world_size(self) -> int:
        return self._world_size

    @property
    def local_world_size(self) -> int:
        return self._local_world_size

    @property
    def pod_size(self) -> Optional[int]:
        return self._pod_size

    @property
    def hbm_mem_bw(self) -> float:
        return self._hbm_mem_bw

    @property
    def ddr_mem_bw(self) -> float:
        return self._ddr_mem_bw

    @property
    def ssd_mem_bw(self) -> float:
        return self._ssd_mem_bw

    @property
    def hbm_to_ddr_mem_bw(self) -> float:
        return self._hbm_to_ddr_mem_bw

    @property
    def intra_host_bw(self) -> float:
        return self._comms_bandwidths.intra_host_bw

    @property
    def inter_host_bw(self) -> float:
        return self._comms_bandwidths.inter_host_bw

    @property
    def comms_bandwidths(self) -> GeneralizedCommsBandwidth:
        return self._comms_bandwidths

    @property
    def bwd_compute_multiplier(self) -> float:
        return self._bwd_compute_multiplier

    @property
    def weighted_feature_bwd_compute_multiplier(self) -> float:
        return self._weighted_feature_bwd_compute_multiplier

    @property
    def uneven_sharding_perf_multiplier(self) -> float:
        return self._uneven_sharding_perf_multiplier

    def _hash(self) -> int:
        parts = [self._world_size, self._compute_device, self._local_world_size, self._hbm_mem_bw, self._ddr_mem_bw, self.intra_host_bw,
                 self.inter_host_bw, tuple((d.storage.hbm, d.storage.ddr) for d in self._devices)]
        return int(hashlib.sha256(repr(parts).encode()).hexdigest()[:15], 16)

    def __repr__(self) -> str:
        topology_repr: str = f"world_size={self._world_size} \n"
        topology_repr += f"compute_device={self._compute_device}\n"
        topology_repr += "devices=\n"
        for idx, device in enumerate(self._devices):
            topology_repr += f"\tdevice {idx} {device}\n"
        topology_repr += f"local_world_size={self._local_world_size} \n"
        topology_repr += f"intra_host_bw={self.intra_host_bw} \n"
        topology_repr += f"inter_host_bw={self.inter_host_bw} \n"
        return topology_repr


# ---- sharding options --------------------------------------------------------------------------------------
@dataclass
class Shard:
    """One shard of a candidate sharding: size [rows, cols], offset, estimated storage/perf, rank."""

    size: List[int]
    offset: List[int]
    storage: Optional[Storage] = None
    perf: Optional[Perf] = None
    rank: Optional[int] = None

    def __hash__(self) -> int:
        return hash((tuple(self.size), tuple(self.offset), self.storage, self.perf, self.rank))

    def __str__(self) -> str:
        return f"Shard size: {tuple(self.size)}, offset: {tuple(self.offset)}, storage: {self.storage}, perf: {self.perf}, rank: {self.rank}"


class ShardingOption:
    """One (table, sharding type, compute kernel, shard geometry) candidate."""

    def __init__(
        self,
        name: str,
        tensor: torch.Tensor,
        module: Tuple[str, nn.Module],
        input_lengths: List[float],
        batch_size: int,
        sharding_type: str,
        partition_by: str,
        compute_kernel: str,
        shards: List[Shard],
        cache_params: Optional[CacheParams] = None,
        enforce_hbm: Optional[bool] = None,
        stochastic_rounding: Optional[bool] = None,
        bounds_check_mode: Optional[Any] = None,
        dependency: Optional[str] = None,
        is_pooled: Optional[bool] = None,
        feature_names: Optional[List[str]] = None,
        output_dtype: Optional[DataType] = None,
        key_value_params: Optional[KeyValueParams] = None,
    ) -> None:
        self.name = name
        self._tensor = tensor
        self._module = module
        self.input_lengths = input_lengths
        self.batch_size = batch_size
        self.sharding_type = sharding_type
        self.partition_by = partition_by
        self.compute_kernel = compute_kernel
        self.shards = shards
        self.cache_params = cache_params
        self.enforce_hbm = enforce_hbm
        self.stochastic_rounding = stochastic_rounding
        self.bounds_check_mode = bounds_check_mode
        self.dependency = dependency
        self._is_pooled = is_pooled
        self.is_weighted: Optional[bool] = None
        self.feature_names: Optional[List[str]] = feature_names
        self.output_dtype: Optional[DataType] = output_dtype
        self.key_value_params: Optional[KeyValueParams] = key_value_params

    @property
    def tensor(self) -> torch.Tensor:
        return self._tensor

    @property
    def module(self) -> Tuple[str, nn.Module]:
        return self._module

    @property
    def fqn(self) -> str:
        return self.module[0] + "." + self.name

    @property
    def cache_load_factor(self) -> Optional[float]:
        return self.cache_params.load_factor if self.cache_params is not None else None

    @property
    def path(self) -> str:
        return self.module[0]

    @property
    def num_shards(self) -> int:
        return len(self.shards)

    @property
    def num_inputs(self) -> int:
        return len(self.input_lengths)

    @property
    def total_storage(self) -> Storage:
        storage = Storage(hbm=0, ddr=0)
        for shard in self.shards:
            storage += cast(Storage, shard.storage)
        return storage

    @property
    def total_perf(self) -> float:
        return sum(cast(Perf, shard.perf).total for shard in self.shards)

    @property
    def is_pooled(self) -> bool:
        if self._is_pooled is None:
            self._is_pooled = ShardingOption.module_pooled(self.module[1], self.name)
        return self._is_pooled

    @staticmethod
    def module_pooled(module: nn.Module, sharding_option_name: str) -> bool:
        from ...modules.embedding_modules import EmbeddingCollectionInterface

        if isinstance(module, EmbeddingCollectionInterface) or type(module).__name__ in ("ManagedCollisionEmbeddingCollection", "EmbeddingCollection"):
            return False
        for submodule in module.modules():
            if isinstance(submodule, EmbeddingCollectionInterface):
                for name, _ in submodule.named_parameters():
                    if sharding_option_name in name:
                        return False
        return True

    def storage_hash(self) -> int:
        """Identity of this option BEFORE planning (fqn, sharding type, kernel, cache load factor, shard count): the key under which
        a stored plan keeps the shards it chose for it (BLAKE2b, 56 bits - stable across processes and machines)."""
        key = f"{self.fqn}|{self.sharding_type}|{self.compute_kernel}|{self.cache_load_factor}|{self.num_shards}"
        return int.from_bytes(hashlib.blake2b(key.encode("utf-8"), digest_size=7).digest(), byteorder="big")

    def __hash__(self) -> int:
        return hash((self.fqn, self.sharding_type, self.compute_kernel, tuple(self.shards), self.cache_params))

    def __deepcopy__(self, memo: Optional[Dict[int, "ShardingOption"]]) -> "ShardingOption":
        cls = self.__class__
        result = cls.__new__(cls)
        for k, v in self.__dict__.items():
            if k in ["_tensor", "_module"]:
                setattr(result, k, v)
            else:
                setattr(result, k, deepcopy(v, memo))
        return result

    def __str__(self) -> str:
        return (f"ShardingOption(fqn={self.fqn}, sharding_type={self.sharding_type}, compute_kernel={self.compute_kernel}, "
                f"shards={[str(s) for s in self.shards]})")


class PartitionByType(Enum):
    DEVICE = "device"  # each shard may go to any device
    HOST = "host"  # all shards of the option go to the devices of one host
    UNIFORM = "uniform"  # one shard per device
    MULTI_HOST = "multi_host"  # column shards across hosts, each row-split inside its host (GRID)


@dataclass
class ParameterConstraints:
    """User constraints / hints for one table (reference planner/types.py:1344)."""

    sharding_types: Optional[List[str]] = None
    compute_kernels: Optional[List[str]] = None
    min_partition: Optional[int] = None  # column-wise shard width
    pooling_factors: List[float] = field(default_factory=lambda: [POOLING_FACTOR])
    num_poolings: Optional[List[float]] = None
    batch_sizes: Optional[List[int]] = None
    is_weighted: bool = False
    cache_params: Optional[CacheParams] = None
    enforce_hbm: Optional[bool] = None
    stochastic_rounding: Optional[bool] = None
    bounds_check_mode: Optional[Any] = None
    feature_names: Optional[List[str]] = None
    output_dtype: Optional[DataType] = None
    device_group: Optional[str] = None
    key_value_params: Optional[KeyValueParams] = None
    use_gpu_rank_broadcast: Optional[bool] = None


class PlannerInputContext:
    pass


class PartitionError(PlannerError):
    def __init__(self, message: str) -> None:
        super().__init__(message, PlannerErrorType.PARTITION)


class StorageReservation(abc.ABC):
    @abc.abstractmethod
    def reserve(self, topology: Topology, batch_size: int, module: nn.Module, sharders: List[ModuleSharder[nn.Module]],
                constraints: Optional[Dict[str, ParameterConstraints]] = None) -> Topology:
        ...

    @property
    @abc.abstractmethod
    def last_reserved_topology(self) -> Optional[Topology]:
        ...


class PerfModel(abc.ABC):
    @abc.abstractmethod
    def rate(self, plan: List[ShardingOption]) -> float:
        ...


class ShardEstimator(abc.ABC):
    @abc.abstractmethod
    def __init__(self, topology: Topology, constraints: Optional[Dict[str, ParameterConstraints]] = None) -> None:
        ...

    @abc.abstractmethod
    def estimate(self, sharding_options: List[ShardingOption], sharder_map: Optional[Dict[str, ModuleSharder[nn.Module]]] = None) -> None:
        ...


class Enumerator(abc.ABC):
    @abc.abstractmethod
    def __init__(self, topology: Topology, batch_size: int = BATCH_SIZE, constraints: Optional[Dict[str, ParameterConstraints]] = None,
                 estimator: Optional[Union[ShardEstimator, List[ShardEstimator]]] = None) -> None:
        ...

    @abc.abstractmethod
    def enumerate(self, module: nn.Module, sharders: List[ModuleSharder[nn.Module]]) -> List[ShardingOption]:
        ...

    @abc.abstractmethod
    def populate_estimates(self, sharding_options: List[ShardingOption]) -> None:
        ...


class Proposer(abc.ABC):
    @abc.abstractmethod
    def load(self, search_space: List[ShardingOption], enumerator: Optional[Enumerator] = None) -> None:
        ...

    @abc.abstractmethod
    def feedback(self, partitionable: bool, plan: Optional[List[ShardingOption]] = None, perf_rating: Optional[float] = None,
                 storage_constraint: Optional[Topology] = None) -> None:
        ...

    @abc.abstractmethod
    def propose(self) -> Optional[List[ShardingOption]]:
        ...


class Partitioner(abc.ABC):
    @abc.abstractmethod
    def partition(self, proposal: List[ShardingOption], storage_constraint: Topology) -> List[ShardingOption]:
        ...


class Stats(abc.ABC):
    @abc.abstractmethod
    def log(self, sharding_plan: ShardingPlan, topology: Topology, batch_size: int, storage_reservation: StorageReservation, num_proposals: int,
            num_plans: int, run_time: float, best_plan: List[ShardingOption], constraints: Optional[Dict[str, ParameterConstraints]] = None,
            sharders: Optional[List[ModuleSharder[nn.Module]]] = None, debug: bool = False) -> None:
        ...


# ---- stored plans ------------------------------------------------------------------------------------------------------------------------------------
@dataclass
class PlanDebugStats:
    """What is logged about how a plan came about."""

    planner_type: str
    timeout_seconds: Optional[int]


class PlanLoader(abc.ABC):
    """Source of a previously computed plan: re-use it instead of searching again (restarts), or start the next search from it.
    ``load`` returns {``ShardingOption.storage_hash()``: the option with the shards the stored plan chose}; ``plan_context_hash`` the
    hash of the planner inputs the plan was computed for (checked against the current planner before the plan is used)."""

    @abc.abstractmethod
    def load(self) -> Optional[Dict[int, "ShardingOption"]]:
        ...

    @abc.abstractmethod
    def plan_context_hash(self) -> Optional[str]:
        ...

    def get_plan_id(self) -> Optional[str]:
        return None


@dataclass
class CriticalPathEstimate:
    comms_estimate: float
    comp_estimate: float

    def total(self) -> float:
        return self.comms_estimate + self.comp_estimate


# ---- topology from configuration layers -----------------------------------------------------------------------------------------------------------------
class TopologyConfigBase(abc.ABC):
    """A layer of topology configuration with an open key-value side channel (``additional_params``) for data the schema does not
    know (per-device capacities of a heterogeneous job, hardware generation, experiments)."""

    additional_params: Dict[str, Any]

    def get_param(self, key: str, default: Any = None) -> Any:
        return self.additional_params.get(key, default)

    def has_param(self, key: str) -> bool:
        return key in self.additional_params

    @abc.abstractmethod
    def validate(self) -> None:
        ...


@dataclass(frozen=True)
class HardwareConfig(TopologyConfigBase):
    """What the hardware offers (detected or looked up per machine type): capacities in bytes, bandwidths in bytes / ms. Subclass with
    defaults for a machine type (e.g. an H100 HGX host: 80 GB HBM, NVLink 4 intra-host bandwidth)."""

    hbm_cap_bytes: Optional[int] = None
    ddr_cap_bytes: Optional[int] = None
    ssd_cap_bytes: Optional[int] = None
    intra_host_bw: Optional[float] = None
    inter_host_bw: Optional[float] = None
    hbm_mem_bw: Optional[float] = None
    ddr_mem_bw: Optional[float] = None
    hbm_to_ddr_mem_bw: Optional[float] = None
    ssd_mem_bw: Optional[float] = None
    additional_params: Dict[str, Any] = field(default_factory=dict)

    def validate(self) -> None:
        for name in ("hbm_cap_bytes", "ddr_cap_bytes", "ssd_cap_bytes", "intra_host_bw", "inter_host_bw", "hbm_mem_bw", "ddr_mem_bw", "hbm_to_ddr_mem_bw", "ssd_mem_bw"):
            v = getattr(self, name)
            if v is not None and v < 0:
                raise ValueError(f"{name} must not be negative, got {v}")


@dataclass(frozen=True)
class TrainerConfig(TopologyConfigBase):
    """What the job asks for - wins over the hardware layer: world size (required), ranks per host, capacity overrides, dry-run
    capacities (plan for hardware that is not there), hosts per NVLink domain (``pod_size``)."""

    world_size: Optional[int] = None
    local_world_size: Optional[int] = None
    hbm_cap_bytes: Optional[int] = None
    ddr_cap_bytes: Optional[int] = None
    ssd_cap_bytes: Optional[int] = None
    is_dry_run: bool = False
    dry_run_hbm_bytes: Optional[int] = None
    dry_run_ddr_bytes: Optional[int] = None
    pod_size: Optional[int] = None
    additional_params: Dict[str, Any] = field(default_factory=dict)

    def validate(self) -> None:
        if self.world_size is None:
            raise ValueError("world_size must be provided in TrainerConfig")
        if self.pod_size is not None and self.pod_size > self.world_size:
            raise ValueError(f"pod_size ({self.pod_size}) cannot be greater than world_size ({self.world_size})")


@dataclass(frozen=True)
class KernelConfig(TopologyConfigBase):
    """What the compute kernels need the cost model to know: device type, backward / weighted-feature / uneven-shard multipliers,
    whether bandwidths come from the hardware layer, an explicit collective bandwidth model."""

    compute_device: str = "cuda"
    bwd_compute_multiplier: float = BWD_COMPUTE_MULTIPLIER
    weighted_feature_bwd_compute_multiplier: float = WEIGHTED_KERNEL_MULTIPLIER
    uneven_sharding_perf_multiplier: float = 1.0
    use_hardware_based_bandwidth: bool = False
    generalized_comms_bandwidths: Optional[GeneralizedCommsBandwidth] = None
    additional_params: Dict[str, Any] = field(default_factory=dict)

    def validate(self) -> None:
        if self.compute_device not in ("cpu", "cuda", "mtia"):
            raise ValueError(f"compute_device must be one of ('cpu', 'cuda', 'mtia'), got {self.compute_device}")


class TopologyFactory:
    """``Topology`` from the three layers: trainer (explicit) > hardware (detected) > built-in defaults."""

    @staticmethod
    def create_topology(trainer_config: TrainerConfig, hardware_config: Optional[HardwareConfig] = None, kernel_config: Optional[KernelConfig] = None) -> "Topology":
        hardware, kernel = hardware_config or HardwareConfig(), kernel_config or KernelConfig()
        trainer_config.validate()
        hardware.validate()
        kernel.validate()
        first = lambda *xs: next((x for x in xs if x is not None), None)  # noqa: E731
        kw: Dict[str, Any] = {"world_size": trainer_config.world_size, "compute_device": kernel.compute_device, "bwd_compute_multiplier": kernel.bwd_compute_multiplier,
                              "weighted_feature_bwd_compute_multiplier": kernel.weighted_feature_bwd_compute_multiplier,
                              "uneven_sharding_perf_multiplier": kernel.uneven_sharding_perf_multiplier}
        if trainer_config.local_world_size is not None:
            kw["local_world_size"] = trainer_config.local_world_size
        if trainer_config.pod_size is not None:
            kw["pod_size"] = trainer_config.pod_size
        hbm, ddr, ssd = first(trainer_config.hbm_cap_bytes, hardware.hbm_cap_bytes), first(trainer_config.ddr_cap_bytes, hardware.ddr_cap_bytes), \
            first(trainer_config.ssd_cap_bytes, hardware.ssd_cap_bytes)
        if trainer_config.is_dry_run:
            hbm, ddr = first(trainer_config.dry_run_hbm_bytes, hbm), first(trainer_config.dry_run_ddr_bytes, ddr)
        for key, v in (("hbm_cap", hbm), ("ddr_cap", ddr), ("ssd_cap", ssd)):
            if v is not None:
                kw[key] = v
        custom = trainer_config.get_param("custom_topology_data")
        if custom is not None:
            kw["custom_topology_data"] = custom
        hw = kernel.use_hardware_based_bandwidth
        kw["hbm_mem_bw"] = first(hardware.hbm_mem_bw if hw else None, HBM_MEM_BW)
        kw["ddr_mem_bw"] = first(hardware.ddr_mem_bw if hw else None, DDR_MEM_BW)
        kw["ssd_mem_bw"] = first(hardware.ssd_mem_bw if hw else None, SSD_MEM_BW)
        kw["hbm_to_ddr_mem_bw"] = first(hardware.hbm_to_ddr_mem_bw if hw else None, HBM_TO_DDR_MEM_BW)
        if kernel.generalized_comms_bandwidths is not None:
            kw["generalized_comms_bandwidths"] = kernel.generalized_comms_bandwidths
        else:
            kw["intra_host_bw"] = first(hardware.intra_host_bw if hw else None, INTRA_NODE_BANDWIDTH)
            kw["inter_host_bw"] = first(hardware.inter_host_bw if hw else None, CROSS_NODE_BANDWIDTH)
        topology = Topology(**kw)
        topology.created_by_factory = True
        return topology


# ---- planner context hashing ---------------------------------------------------------------------------------------------------------------------------------
HUNDRED_GB = 100 * 1024 * 1024 * 1024


def hash_sha256_to_int(hashable_list: List[Any]) -> int:
    return int(hashlib.sha256(str(hashable_list).encode("utf-8")).hexdigest(), 16)


def hash_sha256_str(hashable_list: List[Any]) -> str:
    return hashlib.sha256(str(hashable_list).encode("utf-8")).hexdigest()


def round_to_nearest(x: int, unit: int) -> int:
    """Round to the nearest unit (e.g. 100 GB)."""
    return round(x / unit) * unit


def _topology_hash_components(topology: "Topology", round_unit: int = HUNDRED_GB) -> List[Any]:
    """The fields of a topology that decide a plan; device memory rounded to ``round_unit`` so that small driver / OS differences
    between otherwise identical machines do not invalidate a stored plan."""
    devices = [(d.rank, round_to_nearest(d.storage.hbm, round_unit), round_to_nearest(d.storage.ddr, round_unit), round_to_nearest(getattr(d.storage, "ssd", 0), round_unit))
               for d in topology.devices]
    return [topology.world_size, topology.compute_device, devices, topology.local_world_size, getattr(topology, "intra_group_size", topology.local_world_size),
            topology.hbm_mem_bw, topology.ddr_mem_bw, topology.ssd_mem_bw, topology.hbm_to_ddr_mem_bw, topology.comms_bandwidths.intra_host_bw,
            topology.comms_bandwidths.inter_host_bw, topology.bwd_compute_multiplier, topology.weighted_feature_bwd_compute_multiplier,
            topology.uneven_sharding_perf_multiplier]


def _shard_hash_components(shard: "Shard") -> tuple:
    st = shard.storage
    return (tuple(shard.size), tuple(shard.offset), shard.rank, (st.hbm, st.ddr, getattr(st, "ssd", 0)) if st else None)


def _build_hashable_list(topology: "Topology", batch_size: int, enumerator: "Enumerator", storage_reservation: "StorageReservation",
                         constraints: Optional[Dict[str, "ParameterConstraints"]]) -> List[Any]:
    assert hasattr(enumerator, "last_stored_search_space"), "This enumerator is not compatible with hashing"
    search_space = enumerator.last_stored_search_space
    assert search_space is not None, "Unable to hash planner context without an enumerator that has a precomputed search space"
    reserved = storage_reservation.last_reserved_topology
    assert reserved is not None, "Unable to hash planner context without a storage reservation that has a precomputed topology"
    return [hash_sha256_to_int(_topology_hash_components(topology)), batch_size,
            [[so.fqn, so.sharding_type, so.compute_kernel, tuple(_shard_hash_components(sh) for sh in so.shards), so.cache_params] for so in search_space],
            type(storage_reservation).__name__, hash_sha256_to_int(_topology_hash_components(reserved)),
            tuple((k, hash_sha256_str([repr(v)])) for k, v in sorted(constraints.items())) if constraints else None]


def hash_planner_context_inputs(topology: "Topology", batch_size: int, enumerator: "Enumerator", storage_reservation: "StorageReservation",
                                constraints: Optional[Dict[str, "ParameterConstraints"]], hash_function: Callable[[List[Any]], int] = hash_sha256_to_int) -> int:
    """Hash of everything a plan depends on (topology, batch size, enumerated search space, reservation policy and reserved
    topology, constraints): equal hashes <=> a stored plan is valid for this planner."""
    return hash_function(_build_hashable_list(topology, batch_size, enumerator, storage_reservation, constraints))


def hash_planner_context_inputs_str(topology: "Topology", batch_size: int, enumerator: "Enumerator", storage_reservation: "StorageReservation",
                                    constraints: Optional[Dict[str, "ParameterConstraints"]], hash_function: Callable[[List[Any]], str] = hash_sha256_str) -> str:
    return hash_function(_build_hashable_list(topology, batch_size, enumerator, storage_reservation, constraints))


# ---- picklable sharder snapshot (the estimators work from this, not from live sharder objects) ---------------------------------------------------------------
class StorageUsageType(Enum):
    """Which storage formula a sharder uses: its own ``storage_usage`` (DEFAULT), the training embedding sharders' (BASE), the
    quantized inference sharders' (BASE_QUANT)."""

    DEFAULT = "default"
    BASE = "base"
    BASE_QUANT = "base_quant"


@dataclass
class SharderData:
    fused_params: Dict[str, Any]
    qcomm_dtype_sizes: Dict[str, Tuple[float, float]]
    storage_usage_type: StorageUsageType


SharderDataMap = Dict[str, SharderData]
