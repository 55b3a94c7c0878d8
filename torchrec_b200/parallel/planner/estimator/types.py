"""Data types of the annotation-driven perf estimator.

Reference: ``torchrec/distributed/planner/estimator/types.py`` (``PerfCoefficient`` :67, ``EstimatorPerfCoefficients`` :82, ``PrefetchCoefficients`` :90,
``PerfCoefficientConfig`` :104, ``HardwarePerfConfig`` :190, ``ShardPerfContext`` :493).
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Any, Dict, List, Optional

from ...embedding_types import EmbeddingComputeKernel
from ...types import ShardingType
from .. import constants as K


@dataclass
class PerfCoefficient:
    """Linear model of one pass: ``bytes = a * input_read + b * lookup + c * output_write + d * hash_size`` (then divided by the device bandwidth)."""

    input_read_size_multiplier: float = 1.0
    lookup_size_multiplier: float = 1.0
    embedding_output_multiplier: float = 1.0
    hash_size_multiplier: float = 0.0


@dataclass
class EstimatorPerfCoefficients:
    fwd: PerfCoefficient = field(default_factory=PerfCoefficient)
    bwd: PerfCoefficient = field(default_factory=lambda: PerfCoefficient(lookup_size_multiplier=K.BWD_COMPUTE_MULTIPLIER, embedding_output_multiplier=1.0))


@dataclass
class PrefetchCoefficients:
    expected_num_lookups_coefficient: float = 1.0
    expected_num_unique_lookups_coefficient: float = 1.0
    expected_size_cache_fetches_coefficient: float = 1.0


@dataclass
class PerfCoefficientConfig:
    """Coefficients per sharding type (``default`` when a type has no entry)."""

    default: EstimatorPerfCoefficients = field(default_factory=EstimatorPerfCoefficients)
    per_sharding_type: Dict[str, EstimatorPerfCoefficients] = field(default_factory=dict)
    prefetch: PrefetchCoefficients = field(default_factory=PrefetchCoefficients)

    def get(self, sharding_type: str) -> EstimatorPerfCoefficients:
        return self.per_sharding_type.get(sharding_type, self.default)


class HardwarePerfConfig:
    """Bandwidths of one hardware generation (bytes / ms). Subclass and decorate with ``annotations.hbm_mem_bw(...)`` etc., or pass values here.
    The defaults are the H100 / NVLink-4 numbers of ``planner/constants.py``."""

    name: str = "default"
    hbm_mem_bw: float = K.HBM_MEM_BW
    ddr_mem_bw: float = K.DDR_MEM_BW
    ssd_mem_bw: float = K.SSD_MEM_BW
    hbm_to_ddr_mem_bw: float = K.HBM_TO_DDR_MEM_BW
    intra_host_bw: float = K.INTRA_NODE_BANDWIDTH
    inter_host_bw: float = K.CROSS_NODE_BANDWIDTH
    bwd_compute_multiplier: float = K.BWD_COMPUTE_MULTIPLIER
    weighted_feature_bwd_compute_multiplier: float = K.WEIGHTED_KERNEL_MULTIPLIER
    uneven_sharding_perf_multiplier: float = 1.0
    use_min_dim_for_lookup: bool = False
    use_block_usage_penalty: bool = True
    use_bytes_for_input_read_size: bool = True
    input_data_type_size: float = float(K.BIGINT_DTYPE)
    supported_sharding_types: Optional[List[str]] = None
    coefficients: PerfCoefficientConfig = PerfCoefficientConfig()
    _device_bw_overrides: Dict[Any, float] = {}

    def __init__(self, **overrides: Any) -> None:
        for k, v in overrides.items():
            if not hasattr(type(self), k):
                raise TypeError(f"unknown hardware field {k!r}")
            setattr(self, k, v)

    def get_device_bw(self, compute_device: str, compute_kernel: str, caching_ratio: Optional[float] = None, prefetch_pipeline: bool = False) -> Optional[float]:
        """Effective bandwidth a lookup kernel sees; ``annotations.device_bw`` entries win over the ``kernel_bw_lookup`` table."""
        key = (compute_device, compute_kernel)
        if key in self._device_bw_overrides:
            v = self._device_bw_overrides[key]
            return v(self, caching_ratio, prefetch_pipeline) if callable(v) else v
        return K.kernel_bw_lookup(compute_device, compute_kernel, self.hbm_mem_bw, self.ddr_mem_bw, self.hbm_to_ddr_mem_bw, caching_ratio, prefetch_pipeline)

    def get_comms_bw(self, world_size: int, local_world_size: int) -> float:
        """Per-direction bytes / ms of one rank inside the job's all-to-all: inside one NVLink domain the all-to-all efficiency of
        that world size applies to the single-peer rate (``planner/calibration.py``); across hosts the NIC is the limit."""
        if world_size > local_world_size:
            return self.inter_host_bw
        from ..calibration import ALL_TO_ALL_EFFICIENCY, PEER_STORE_GBPS, all_to_all_gbps

        return self.intra_host_bw * all_to_all_gbps(world_size) / PEER_STORE_GBPS


@dataclass
class ShardPerfContext:
    """Everything an evaluator needs to cost ONE shard of ONE sharding option."""

    sharding_type: str
    compute_kernel: str
    compute_device: str
    world_size: int
    local_world_size: int
    batch_sizes: List[int]
    input_lengths: List[float]
    num_poolings: List[float]
    hash_size: int
    emb_dim: int
    shard_rows: int
    shard_cols: int
    num_row_shards: int
    table_data_type_size: float
    output_data_type_size: float
    fwd_a2a_comm_data_type_size: float
    bwd_a2a_comm_data_type_size: float
    fwd_sr_comm_data_type_size: float
    bwd_sr_comm_data_type_size: float
    is_pooled: bool
    is_weighted: bool = False
    is_inference: bool = False
    caching_ratio: Optional[float] = None
    prefetch_pipeline: bool = False
    expected_cache_fetches: float = 0.0
    uneven_sharding_perf_multiplier: float = 1.0
    device_bw: float = 0.0
    comms_bw: float = 0.0

    # -- derived sizes (bytes) --
    @property
    def batch_multiplier(self) -> float:
        return 1.0 if self.sharding_type == ShardingType.DATA_PARALLEL.value else float(self.world_size)

    @property
    def num_ids(self) -> float:
        n = sum(l * p * b for l, p, b in zip(self.input_lengths, self.num_poolings, self.batch_sizes)) * self.batch_multiplier
        if self.sharding_type in (ShardingType.ROW_WISE.value, ShardingType.TABLE_ROW_WISE.value, ShardingType.GRID_SHARD.value):
            n /= max(1, self.num_row_shards)
        return n

    @property
    def num_bags(self) -> float:
        return sum(p * b for p, b in zip(self.num_poolings, self.batch_sizes)) * self.batch_multiplier

    def input_read_size(self, input_data_type_size: float) -> float:
        return self.num_ids * input_data_type_size * (2.0 if self.is_weighted else 1.0)

    @property
    def lookup_size(self) -> float:
        return self.num_ids * self.shard_cols * self.table_data_type_size

    @property
    def output_write_size(self) -> float:
        return (self.num_bags if self.is_pooled else self.num_ids) * self.shard_cols * self.output_data_type_size
