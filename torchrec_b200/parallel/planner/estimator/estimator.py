"""Per-sharding-type perf evaluators + the estimator that drives them.

Reference: ``torchrec/distributed/planner/estimator/estimator.py`` - ``EmbeddingShardingPerfEvaluator`` :65-1110, ``TableWiseEvaluator`` :1113,
``RowWiseEvaluator`` :1157, ``TableRowWiseEvaluator`` :1319, ``DataParallelEvaluator`` :1512, CW / TWCW / GRID :1604-1620, ``EmbeddingPerfEstimator`` :1623,
``EmbeddingPerfEstimatorFactory`` :1779, inference evaluators :1939-1992, ``compute_block_usage_penalty`` :1995, ``get_embedding_perf_sharding_evaluator`` :2033.

Every cost is bytes / bandwidth (ms). An evaluator owns the formulas of one sharding type; a hardware config may override any single formula with an
annotated method (``annotations.py``). The formulas model THIS framework's kernels: lookup + output all-to-all fused over NVLink inside a host (the
transfer hides behind the gathers), row-wise partial pools reduced at the destination, hierarchical two-hop dists for host-local row shards.
"""
from __future__ import annotations

from abc import ABC
from typing import Any, Callable, Dict, List, Optional, Type

import torch
from torch import nn

from ...embedding_types import EmbeddingComputeKernel
from ...types import ModuleSharder, ShardingType
from .. import calibration as CAL
from .. import constants as K
from ..types import ParameterConstraints, Perf, PlannerError, ShardEstimator, ShardingOption, Topology
import importlib

A = importlib.import_module(__package__ + ".annotations")  # (``from . import annotations`` would pick up the __future__ feature of that name)
from .config import EmbeddingPerfEstimatorConfig
from .types import EstimatorPerfCoefficients, HardwarePerfConfig, PerfCoefficient, ShardPerfContext


def compute_block_usage_penalty(embedding_dim: int) -> float:
    """A warp moves 512 B per request: rows narrower than 128 fp32 waste part of it (``calibration.py``)."""
    if embedding_dim >= K.FULL_BLOCK_EMB_DIM:
        return 1.0
    return K.HALF_BLOCK_PENALTY if embedding_dim >= K.FULL_BLOCK_EMB_DIM // 2 else K.QUARTER_BLOCK_PENALTY


class EmbeddingShardingPerfEvaluator(ABC):
    """Template: ``evaluate(ctx)`` -> ``Perf``; each term first looks for an annotated override on the config."""

    sharding_type: str = ""
    is_inference: bool = False

    def __init__(self, config: Optional[HardwarePerfConfig] = None) -> None:
        self.config = config or EmbeddingPerfEstimatorConfig()

    # -- coefficients --
    def _coeff(self, ctx: ShardPerfContext, fwd: bool) -> PerfCoefficient:
        custom = (A.get_fwd_coefficient if fwd else A.get_bwd_coefficient)(self.config, ctx.sharding_type)
        if custom is not None:
            return custom(ctx)
        c = self.config.coefficients.get(ctx.sharding_type)
        return c.fwd if fwd else c.bwd

    def _penalty(self, ctx: ShardPerfContext) -> float:
        return compute_block_usage_penalty(ctx.shard_cols) if self.config.use_block_usage_penalty else 1.0

    def _pass_bytes(self, ctx: ShardPerfContext, c: PerfCoefficient) -> float:
        in_size = ctx.input_read_size(self.config.input_data_type_size) if self.config.use_bytes_for_input_read_size else ctx.num_ids
        out = self.output_write_size(ctx)
        return (c.input_read_size_multiplier * in_size + c.lookup_size_multiplier * ctx.lookup_size * self._penalty(ctx)
                + c.embedding_output_multiplier * out + c.hash_size_multiplier * ctx.shard_rows * ctx.shard_cols * ctx.table_data_type_size)

    # -- terms (defaults) --
    def output_write_size(self, ctx: ShardPerfContext) -> float:
        custom = A.get_output_write_size(self.config, ctx.sharding_type)
        return custom(ctx) if custom is not None else ctx.output_write_size

    def forward_compute(self, ctx: ShardPerfContext) -> float:
        t = self._pass_bytes(ctx, self._coeff(ctx, True)) / ctx.device_bw
        return t * (self.config.weighted_feature_bwd_compute_multiplier if ctx.is_weighted else 1.0) * ctx.uneven_sharding_perf_multiplier

    def backward_compute(self, ctx: ShardPerfContext) -> float:
        t = self._pass_bytes(ctx, self._coeff(ctx, False)) / ctx.device_bw
        return t * (self.config.weighted_feature_bwd_compute_multiplier if ctx.is_weighted else 1.0) * ctx.uneven_sharding_perf_multiplier

    def _remote_fraction(self, ctx: ShardPerfContext) -> float:
        return (ctx.world_size - 1) / ctx.world_size if ctx.world_size > 1 else 0.0

    def input_dist_comms(self, ctx: ShardPerfContext) -> float:
        return ctx.input_read_size(self.config.input_data_type_size) * self._remote_fraction(ctx) / ctx.comms_bw

    def fwd_comms(self, ctx: ShardPerfContext) -> float:
        return 0.0

    def bwd_comms(self, ctx: ShardPerfContext) -> float:
        return 0.0

    def prefetch_compute(self, ctx: ShardPerfContext) -> float:
        if not ctx.prefetch_pipeline or ctx.caching_ratio is None:
            return 0.0
        pc = self.config.coefficients.prefetch
        misses = ctx.expected_cache_fetches if ctx.expected_cache_fetches > 0 else ctx.num_ids * max(0.0, 1.0 - ctx.caching_ratio) * pc.expected_num_unique_lookups_coefficient
        return misses * pc.expected_size_cache_fetches_coefficient * ctx.shard_cols * ctx.table_data_type_size / self.config.hbm_to_ddr_mem_bw

    # -- driver --
    def _term(self, name: str, getter: Callable[[Any, str], Optional[Callable[..., float]]], ctx: ShardPerfContext) -> float:
        custom = getter(self.config, ctx.sharding_type)
        return float(custom(ctx)) if custom is not None else float(getattr(self, name)(ctx))

    def evaluate(self, ctx: ShardPerfContext) -> Perf:
        fwd_compute = self._term("forward_compute", A.get_forward_compute, ctx)
        fwd_comms = self._term("fwd_comms", A.get_fwd_comms, ctx)
        fwd_compute, fwd_comms = self._overlap(ctx, fwd_compute, fwd_comms)
        if self.is_inference or ctx.is_inference:
            bwd_compute = bwd_comms = 0.0
        else:
            bwd_compute = self._term("backward_compute", A.get_backward_compute, ctx)
            bwd_comms = self._term("bwd_comms", A.get_bwd_comms, ctx)
            bwd_compute, bwd_comms = self._overlap(ctx, bwd_compute, bwd_comms)
        return Perf(fwd_compute=fwd_compute, fwd_comms=fwd_comms, bwd_compute=bwd_compute, bwd_comms=bwd_comms,
                    prefetch_compute=self._term("prefetch_compute", A.get_prefetch_compute, ctx), input_dist_comms=self._term("input_dist_comms", A.get_input_dist_comms, ctx))

    def _overlap(self, ctx: ShardPerfContext, compute: float, comms: float):
        return compute, comms


class TableWiseEvaluator(EmbeddingShardingPerfEvaluator):
    sharding_type = ShardingType.TABLE_WISE.value

    def fwd_comms(self, ctx: ShardPerfContext) -> float:
        return ctx.num_bags * ctx.shard_cols * ctx.fwd_a2a_comm_data_type_size * self._remote_fraction(ctx) / ctx.comms_bw if ctx.is_pooled else \
            ctx.num_ids * ctx.shard_cols * ctx.fwd_a2a_comm_data_type_size * self._remote_fraction(ctx) / ctx.comms_bw

    def bwd_comms(self, ctx: ShardPerfContext) -> float:
        rows = ctx.num_bags if ctx.is_pooled else ctx.num_ids
        return rows * ctx.shard_cols * ctx.bwd_a2a_comm_data_type_size * self._remote_fraction(ctx) / ctx.comms_bw

    def bwd_comms(self, ctx: ShardPerfContext) -> float:  # noqa: F811 - fused variant below wraps the plain formula
        rows = ctx.num_bags if ctx.is_pooled else ctx.num_ids
        full = rows * ctx.shard_cols * ctx.bwd_a2a_comm_data_type_size * self._remote_fraction(ctx) / ctx.comms_bw
        if ctx.world_size <= ctx.local_world_size and ctx.compute_device == "cuda" and ctx.is_pooled:
            # the gradient push is captured inside the dense backward graph and runs beside the deferred weight-gradient GEMMs
            full *= CAL.GRAD_PUSH_EXPOSED
        return full

    def _overlap(self, ctx: ShardPerfContext, compute: float, comms: float):
        # fused lookup + output dist: T = lookup + transfer - overlap(W) * min(lookup, transfer)   (calibration.py)
        if ctx.world_size <= ctx.local_world_size and ctx.compute_device == "cuda":
            comms -= min(compute, comms) * CAL.fused_overlap(ctx.world_size)
        return compute, comms


class ColumnWiseEvaluator(TableWiseEvaluator):
    sharding_type = ShardingType.COLUMN_WISE.value


class TableColumnWiseEvaluator(TableWiseEvaluator):
    sharding_type = ShardingType.TABLE_COLUMN_WISE.value


class RowWiseEvaluator(EmbeddingShardingPerfEvaluator):
    sharding_type = ShardingType.ROW_WISE.value

    def forward_compute(self, ctx: ShardPerfContext) -> float:
        base = super().forward_compute(ctx)
        # destination-side reduce of the partial pools: read one slab per row shard, write one
        reduce_bytes = (ctx.num_bags / max(ctx.world_size, 1)) * ctx.shard_cols * ctx.output_data_type_size * (ctx.num_row_shards + 1) if ctx.is_pooled else 0.0
        return base + reduce_bytes / self.config.hbm_mem_bw

    def fwd_comms(self, ctx: ShardPerfContext) -> float:
        rows = ctx.num_bags if ctx.is_pooled else ctx.num_ids
        size = ctx.fwd_sr_comm_data_type_size if ctx.is_pooled else ctx.fwd_a2a_comm_data_type_size
        return rows * ctx.shard_cols * size * self._remote_fraction(ctx) / ctx.comms_bw

    def bwd_comms(self, ctx: ShardPerfContext) -> float:
        rows = ctx.num_bags if ctx.is_pooled else ctx.num_ids
        size = ctx.bwd_sr_comm_data_type_size if ctx.is_pooled else ctx.bwd_a2a_comm_data_type_size
        return rows * ctx.shard_cols * size * self._remote_fraction(ctx) / ctx.comms_bw


class TableRowWiseEvaluator(RowWiseEvaluator):
    sharding_type = ShardingType.TABLE_ROW_WISE.value

    def _two_hop(self, ctx: ShardPerfContext, elem: float) -> float:
        rows = ctx.num_bags if ctx.is_pooled else ctx.num_ids
        nbytes = rows * ctx.shard_cols * elem
        L, W_ = ctx.local_world_size, ctx.world_size
        if W_ <= L:
            return nbytes * ((W_ - 1) / W_ if W_ > 1 else 0.0) / self.config.intra_host_bw
        nodes = W_ / L
        return nbytes * ((L - 1) / L) / self.config.intra_host_bw + nbytes / L * ((nodes - 1) / nodes) / self.config.inter_host_bw

    def fwd_comms(self, ctx: ShardPerfContext) -> float:
        return self._two_hop(ctx, ctx.fwd_sr_comm_data_type_size)

    def bwd_comms(self, ctx: ShardPerfContext) -> float:
        return self._two_hop(ctx, ctx.bwd_sr_comm_data_type_size)


class GridShardEvaluator(TableRowWiseEvaluator):
    sharding_type = ShardingType.GRID_SHARD.value


class DataParallelEvaluator(EmbeddingShardingPerfEvaluator):
    sharding_type = ShardingType.DATA_PARALLEL.value

    def input_dist_comms(self, ctx: ShardPerfContext) -> float:
        return 0.0

    def backward_compute(self, ctx: ShardPerfContext) -> float:
        # dense gradient + an element-wise optimizer pass over the WHOLE table (read w, read g, write w)
        return super().backward_compute(ctx) + ctx.shard_rows * ctx.shard_cols * ctx.table_data_type_size * 3 / ctx.device_bw

    def bwd_comms(self, ctx: ShardPerfContext) -> float:
        if ctx.world_size <= 1:
            return 0.0
        table = ctx.shard_rows * ctx.shard_cols * ctx.table_data_type_size
        return 2 * table * self._remote_fraction(ctx) / ctx.comms_bw  # all-reduce = reduce-scatter + all-gather


class InferenceShardingPerfEvaluator(EmbeddingShardingPerfEvaluator):
    is_inference = True


class TableWiseInferenceEvaluator(InferenceShardingPerfEvaluator, TableWiseEvaluator):
    pass


class RowWiseInferenceEvaluator(InferenceShardingPerfEvaluator, RowWiseEvaluator):
    pass


class TableRowWiseInferenceEvaluator(InferenceShardingPerfEvaluator, TableRowWiseEvaluator):
    pass


class ColumnWiseInferenceEvaluator(InferenceShardingPerfEvaluator, ColumnWiseEvaluator):
    pass


class DataParallelInferenceEvaluator(InferenceShardingPerfEvaluator, DataParallelEvaluator):
    pass


class TableColumnWiseInferenceEvaluator(InferenceShardingPerfEvaluator, TableColumnWiseEvaluator):
    pass


class GridShardInferenceEvaluator(InferenceShardingPerfEvaluator, GridShardEvaluator):
    pass


_TRAIN: Dict[str, Type[EmbeddingShardingPerfEvaluator]] = {c.sharding_type: c for c in (
    TableWiseEvaluator, RowWiseEvaluator, TableRowWiseEvaluator, DataParallelEvaluator, ColumnWiseEvaluator, TableColumnWiseEvaluator, GridShardEvaluator)}
_INFER: Dict[str, Type[EmbeddingShardingPerfEvaluator]] = {c.sharding_type: c for c in (
    TableWiseInferenceEvaluator, RowWiseInferenceEvaluator, TableRowWiseInferenceEvaluator, DataParallelInferenceEvaluator, ColumnWiseInferenceEvaluator,
    TableColumnWiseInferenceEvaluator, GridShardInferenceEvaluator)}


def get_embedding_perf_sharding_evaluator(sharding_type: str, config: Optional[HardwarePerfConfig] = None, is_inference: bool = False) -> EmbeddingShardingPerfEvaluator:
    table = _INFER if is_inference else _TRAIN
    if sharding_type not in table:
        raise PlannerError(f"no perf evaluator for sharding type {sharding_type}")
    if config is not None and config.supported_sharding_types is not None and sharding_type not in config.supported_sharding_types:
        raise PlannerError(f"hardware config {config.name} does not support sharding type {sharding_type}")
    return table[sharding_type](config)


class EmbeddingPerfEstimator(ShardEstimator):
    """Fills ``shard.perf`` of every sharding option through the evaluator of its sharding type."""

    def __init__(self, topology: Topology, constraints: Optional[Dict[str, ParameterConstraints]] = None, is_inference: bool = False,
                 config: Optional[HardwarePerfConfig] = None) -> None:
        self._topology = topology
        self._constraints = constraints
        self._is_inference = is_inference
        if config is None:  # the topology's numbers are authoritative unless a config says otherwise
            config = EmbeddingPerfEstimatorConfig(hbm_mem_bw=topology.hbm_mem_bw, ddr_mem_bw=topology.ddr_mem_bw, hbm_to_ddr_mem_bw=topology.hbm_to_ddr_mem_bw,
                                                  intra_host_bw=topology.intra_host_bw, inter_host_bw=topology.inter_host_bw,
                                                  bwd_compute_multiplier=topology.bwd_compute_multiplier,
                                                  weighted_feature_bwd_compute_multiplier=topology.weighted_feature_bwd_compute_multiplier)
        self._config = config
        self._evaluators: Dict[str, EmbeddingShardingPerfEvaluator] = {}

    @property
    def config(self) -> HardwarePerfConfig:
        return self._config

    def _evaluator(self, sharding_type: str) -> EmbeddingShardingPerfEvaluator:
        if sharding_type not in self._evaluators:
            self._evaluators[sharding_type] = get_embedding_perf_sharding_evaluator(sharding_type, self._config, self._is_inference)
        return self._evaluators[sharding_type]

    def estimate(self, sharding_options: List[ShardingOption], sharder_map: Optional[Dict[str, ModuleSharder[nn.Module]]] = None) -> None:
        if not sharder_map:
            assert not sharding_options, "sharder_map not provided for sharding_options"
            return
        for so in sharding_options:
            ev = self._evaluator(so.sharding_type)
            for shard in so.shards:
                shard.perf = ev.evaluate(self.build_context(so, shard))

    def build_context(self, so: ShardingOption, shard: Any) -> ShardPerfContext:
        from ....modules.embedding_configs import DATA_TYPE_NUM_BITS

        topo = self._topology
        c = self._constraints.get(so.name) if self._constraints else None
        num_poolings = c.num_poolings if c and c.num_poolings else [1.0] * so.num_inputs
        batch_sizes = c.batch_sizes if c and c.batch_sizes else [so.batch_size] * so.num_inputs
        out_elem = DATA_TYPE_NUM_BITS[so.output_dtype] / 8 if so.output_dtype else 4.0
        prefetch = bool(so.cache_params and so.cache_params.prefetch_pipeline)
        bw = self._config.get_device_bw(topo.compute_device, so.compute_kernel, so.cache_load_factor, prefetch)
        if bw is None:
            raise PlannerError(f"No kernel bandwidth for compute device {topo.compute_device}, compute kernel {so.compute_kernel}")
        rows, cols = shard.size
        expected = 0.0
        stats = getattr(so.cache_params, "stats", None) if so.cache_params else None
        if stats is not None and so.cache_load_factor is not None:
            expected = float(stats.expected_miss_rate(so.cache_load_factor)) * sum(l * p * b for l, p, b in zip(so.input_lengths, num_poolings, batch_sizes)) * topo.world_size
        return ShardPerfContext(
            sharding_type=so.sharding_type, compute_kernel=so.compute_kernel, compute_device=topo.compute_device, world_size=topo.world_size,
            local_world_size=topo.local_world_size, batch_sizes=list(batch_sizes), input_lengths=list(so.input_lengths), num_poolings=list(num_poolings),
            hash_size=so.tensor.shape[0], emb_dim=so.tensor.shape[1], shard_rows=rows, shard_cols=cols,
            num_row_shards=len({(s.offset[0], s.size[0]) for s in so.shards}), table_data_type_size=float(so.tensor.element_size()), output_data_type_size=out_elem,
            fwd_a2a_comm_data_type_size=out_elem, bwd_a2a_comm_data_type_size=out_elem, fwd_sr_comm_data_type_size=out_elem, bwd_sr_comm_data_type_size=out_elem,
            is_pooled=so.is_pooled, is_weighted=bool(c.is_weighted) if c and c.is_weighted is not None else bool(so.is_weighted), is_inference=self._is_inference,
            caching_ratio=so.cache_load_factor, prefetch_pipeline=prefetch, expected_cache_fetches=expected,
            uneven_sharding_perf_multiplier=self._config.uneven_sharding_perf_multiplier, device_bw=bw,
            comms_bw=self._config.get_comms_bw(topo.world_size, topo.local_world_size))


EmbeddingPerfEstimatorV2 = EmbeddingPerfEstimator  # the annotation-driven estimator under its versioned name


class EmbeddingPerfEstimatorFactory:
    """Registry of hardware configs by name: ``EmbeddingPerfEstimatorFactory.create("h100", topology)`` (reference :1779-1936)."""

    _registry: Dict[str, Type[HardwarePerfConfig]] = {}

    @classmethod
    def register(cls, name: str, config_cls: Optional[Type[HardwarePerfConfig]] = None):
        def deco(c: Type[HardwarePerfConfig]) -> Type[HardwarePerfConfig]:
            cls._registry[name] = c
            return c

        return deco(config_cls) if config_cls is not None else deco

    @classmethod
    def available(cls) -> List[str]:
        return sorted(cls._registry)

    @classmethod
    def get_config(cls, name: str) -> HardwarePerfConfig:
        if name not in cls._registry:
            raise PlannerError(f"unknown hardware config {name!r}; registered: {cls.available()}")
        return cls._registry[name]()

    @classmethod
    def create(cls, name: Optional[str], topology: Topology, constraints: Optional[Dict[str, ParameterConstraints]] = None, is_inference: bool = False) -> EmbeddingPerfEstimator:
        return EmbeddingPerfEstimator(topology, constraints, is_inference, config=None if name is None else cls.get_config(name))


from .config import GB200PerfConfig  # noqa: E402

EmbeddingPerfEstimatorFactory.register("h100", EmbeddingPerfEstimatorConfig)
EmbeddingPerfEstimatorFactory.register("gb200", GB200PerfConfig)
