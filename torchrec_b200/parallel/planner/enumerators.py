"""Search-space enumeration + shard cost estimators.

``EmbeddingEnumerator`` (reference planner/enumerators.py:75-553) lists every legal
(table x sharding type x compute kernel x column split) as a ``ShardingOption``.
``EmbeddingStorageEstimator`` / ``EmbeddingPerfEstimator`` (reference shard_estimators.py, estimator/)
annotate each shard with HBM/DDR bytes and a forward/backward compute+comms time. The perf model is
re-derived for this framework's kernels: lookups stream ``rows touched x row bytes`` at HBM bandwidth,
output dists move ``B x D`` per peer over NVLink (fused into the lookup / backward kernels, so comms of
TW/CW and compute overlap: the slower of the two is charged), row-wise adds the staging reduce.
"""
from __future__ import annotations

import logging
import math
from typing import Dict, List, Optional, Tuple, Union, cast

import torch
from torch import nn

from ...modules.embedding_configs import DATA_TYPE_NUM_BITS, DataType
from ...modules.embedding_configs import dtype_to_data_type as _dtype_to_data_type
from ..embedding_types import EmbeddingComputeKernel
from ..sharding_plan import calculate_shard_sizes_and_offsets
from ..types import CacheParams, KeyValueParams, ModuleSharder, ShardingType
from .calibration import GRAD_PUSH_EXPOSED, PEER_STORE_GBPS, all_to_all_gbps, fused_overlap
from .constants import (
    BIGINT_DTYPE,
    FULL_BLOCK_EMB_DIM,
    HALF_BLOCK_PENALTY,
    POOLING_FACTOR,
    QUARTER_BLOCK_PENALTY,
    UVM_CACHING_RATIO,
    kernel_bw_lookup,
)
from .types import (
    Enumerator,
    ParameterConstraints,
    PartitionByType,
    Perf,
    PlannerError,
    PlannerErrorType,
    Shard,
    ShardEstimator,
    ShardingOption,
    Storage,
    Topology,
)
from .utils import sharder_name

logger = logging.getLogger(__name__)

GUARDED_COMPUTE_KERNELS = {EmbeddingComputeKernel.KEY_VALUE, EmbeddingComputeKernel.SSD_VIRTUAL_TABLE, EmbeddingComputeKernel.DRAM_VIRTUAL_TABLE}


def get_partition_by_type(sharding_type: str) -> str:
    device = {ShardingType.TABLE_WISE.value, ShardingType.COLUMN_WISE.value}
    host = {ShardingType.TABLE_ROW_WISE.value, ShardingType.TABLE_COLUMN_WISE.value}
    uniform = {ShardingType.ROW_WISE.value, ShardingType.DATA_PARALLEL.value}
    multi_host = {ShardingType.GRID_SHARD.value}
    if sharding_type in device:
        return PartitionByType.DEVICE.value
    if sharding_type in host:
        return PartitionByType.HOST.value
    if sharding_type in uniform:
        return PartitionByType.UNIFORM.value
    if sharding_type in multi_host:
        return PartitionByType.MULTI_HOST.value
    raise ValueError(f"Unrecognized or unsupported sharding type provided: {sharding_type}")


def _tensor_dtype_bytes(t: torch.Tensor) -> float:
    return t.element_size()


# ---- storage ---------------------------------------------------------------------------------------------
class EmbeddingStorageEstimator(ShardEstimator):
    """HBM / DDR per shard: weights + optimizer state + input/output buffers of the sharding type."""

    def __init__(self, topology: Topology, constraints: Optional[Dict[str, ParameterConstraints]] = None, pipeline_type=None,
                 run_embedding_at_peak_memory: bool = False, is_inference: bool = False) -> None:
        self._topology = topology
        self._constraints = constraints
        self._pipeline_type = pipeline_type
        self._run_embedding_at_peak_memory = run_embedding_at_peak_memory
        self._is_inference = is_inference

    def estimate(self, sharding_options: List[ShardingOption], sharder_map: Optional[Dict[str, ModuleSharder[nn.Module]]] = None) -> None:
        if not sharder_map:
            assert not sharding_options, "sharder_map not provided for sharding_options"
            return
        for so in sharding_options:
            sharder = sharder_map[sharder_name(type(so.module[1]))]
            c = self._constraints.get(so.name) if self._constraints else None
            caching_ratio = so.cache_load_factor
            num_poolings = c.num_poolings if c and c.num_poolings else [1.0] * so.num_inputs
            batch_sizes = c.batch_sizes if c and c.batch_sizes else [so.batch_size] * so.num_inputs
            opt_mult = self._optimizer_multiplier(so)
            elem = _tensor_dtype_bytes(so.tensor)
            out_elem = DATA_TYPE_NUM_BITS[so.output_dtype] / 8 if so.output_dtype else 4.0
            world, local = self._topology.world_size, self._topology.local_world_size
            for shard in so.shards:
                rows, cols = shard.size
                weight = rows * cols * elem
                # row-wise optimizer state: 1 fp32 per row; element-wise: same size as the weights
                opt_bytes = rows * 4 if opt_mult == "row" else (rows * cols * 4 * (opt_mult if isinstance(opt_mult, (int, float)) else 0))
                hbm = ddr = 0.0
                if so.compute_kernel in (EmbeddingComputeKernel.FUSED_UVM.value, EmbeddingComputeKernel.QUANT_UVM.value, EmbeddingComputeKernel.KEY_VALUE.value):
                    ddr += weight + opt_bytes
                elif so.compute_kernel in (EmbeddingComputeKernel.FUSED_UVM_CACHING.value, EmbeddingComputeKernel.QUANT_UVM_CACHING.value):
                    ratio = caching_ratio if caching_ratio is not None else UVM_CACHING_RATIO
                    ddr += weight + opt_bytes
                    hbm += ratio * (weight + opt_bytes)
                elif self._topology.compute_device == "cuda":
                    hbm += weight + (0 if self._is_inference else opt_bytes)
                else:
                    ddr += weight + (0 if self._is_inference else opt_bytes)
                # activations: ids in + pooled rows out for the *global* batch this shard serves
                io = self._io_bytes(so, shard, batch_sizes, num_poolings, world, local, out_elem)
                if self._topology.compute_device == "cuda":
                    hbm += io
                else:
                    ddr += io
                shard.storage = Storage(hbm=int(math.ceil(hbm)), ddr=int(math.ceil(ddr)))

    def _optimizer_multiplier(self, so: ShardingOption):
        if self._is_inference or so.compute_kernel in (EmbeddingComputeKernel.QUANT.value, EmbeddingComputeKernel.QUANT_UVM.value,
                                                       EmbeddingComputeKernel.QUANT_UVM_CACHING.value):
            return 0
        if so.compute_kernel == EmbeddingComputeKernel.DENSE.value:
            return 1  # dense gradient buffer
        t = so.tensor
        classes = getattr(t, "_optimizer_classes", None) or ([getattr(t, "_optimizer_class")] if getattr(t, "_optimizer_class", None) else [])
        names = {c.__name__ for c in classes}
        if names & {"RowWiseAdagrad"}:
            return "row"
        if names & {"Adam", "AdamW", "LAMB"}:
            return 2
        if names & {"PartialRowWiseAdam", "PartialRowWiseLAMB", "Adagrad"}:
            return 1
        if names & {"SGD", "LarsSGD"}:
            return 0
        return "row"

    def _io_bytes(self, so: ShardingOption, shard: Shard, batch_sizes, num_poolings, world, local, out_elem) -> float:
        st = so.sharding_type
        if st == ShardingType.DATA_PARALLEL.value:
            mult = 1
        elif st in (ShardingType.TABLE_ROW_WISE.value, ShardingType.GRID_SHARD.value):
            mult = world  # ids of every rank's batch (bucketised) arrive here
        else:
            mult = world
        ids = sum(l * n * b for l, n, b in zip(so.input_lengths, num_poolings, batch_sizes)) * mult
        if st in (ShardingType.ROW_WISE.value, ShardingType.TABLE_ROW_WISE.value, ShardingType.GRID_SHARD.value):
            ids = ids / max(1, len({tuple([s.offset[0], s.size[0]]) for s in so.shards}))
        in_bytes = ids * BIGINT_DTYPE
        out_rows = sum(n * b for n, b in zip(num_poolings, batch_sizes)) * mult if so.is_pooled else ids
        out_bytes = out_rows * shard.size[1] * out_elem
        pipeline_mult = 2.0 if self._pipeline_type is not None else 1.0  # double-buffered in-flight batches
        return in_bytes * pipeline_mult + out_bytes


# ---- perf ----------------------------------------------------------------------------------------------------
class EmbeddingPerfEstimator(ShardEstimator):
    """Forward / backward compute and comms per shard for every sharding type."""

    def __init__(self, topology: Topology, constraints: Optional[Dict[str, ParameterConstraints]] = None, is_inference: bool = False) -> None:
        self._topology = topology
        self._constraints = constraints
        self._is_inference = is_inference

    def estimate(self, sharding_options: List[ShardingOption], sharder_map: Optional[Dict[str, ModuleSharder[nn.Module]]] = None) -> None:
        if not sharder_map:
            assert not sharding_options, "sharder_map not provided for sharding_options"
            return
        topo = self._topology
        for so in sharding_options:
            c = self._constraints.get(so.name) if self._constraints else None
            num_poolings = c.num_poolings if c and c.num_poolings else [1.0] * so.num_inputs
            batch_sizes = c.batch_sizes if c and c.batch_sizes else [so.batch_size] * so.num_inputs
            is_weighted = bool(c.is_weighted) if c else bool(so.is_weighted)
            elem = _tensor_dtype_bytes(so.tensor)
            out_elem = DATA_TYPE_NUM_BITS[so.output_dtype] / 8 if so.output_dtype else 4.0
            caching_ratio = so.cache_load_factor
            prefetch = bool(so.cache_params and so.cache_params.prefetch_pipeline)
            bw = kernel_bw_lookup(topo.compute_device, so.compute_kernel, topo.hbm_mem_bw, topo.ddr_mem_bw, topo.hbm_to_ddr_mem_bw, caching_ratio, prefetch)
            if bw is None:
                raise PlannerError(f"No kernel bandwidth for compute device {topo.compute_device}, compute kernel {so.compute_kernel}")
            W, L = topo.world_size, topo.local_world_size
            intra, inter = topo.intra_host_bw, topo.inter_host_bw
            comm_bw = intra * all_to_all_gbps(W) / PEER_STORE_GBPS if W <= L else inter  # all-to-all efficiency of this world size (calibration.py)
            n_row_shards = len({(s.offset[0], s.size[0]) for s in so.shards})
            for shard in so.shards:
                rows, cols = shard.size
                dim_penalty = 1.0
                if cols < FULL_BLOCK_EMB_DIM:
                    dim_penalty = HALF_BLOCK_PENALTY if cols >= FULL_BLOCK_EMB_DIM // 2 else QUARTER_BLOCK_PENALTY
                st = so.sharding_type
                # ids this shard looks up per step and pooled rows it emits
                if st == ShardingType.DATA_PARALLEL.value:
                    batch_mult = 1.0
                else:
                    batch_mult = float(W)
                ids = sum(l * n * b for l, n, b in zip(so.input_lengths, num_poolings, batch_sizes)) * batch_mult
                if st in (ShardingType.ROW_WISE.value, ShardingType.TABLE_ROW_WISE.value, ShardingType.GRID_SHARD.value):
                    ids /= max(1, n_row_shards)
                bags = sum(n * b for n, b in zip(num_poolings, batch_sizes)) * batch_mult
                out_rows = bags if so.is_pooled else ids
                gather_bytes = ids * cols * elem
                out_bytes = out_rows * cols * out_elem
                fwd_compute = (gather_bytes + out_bytes) * dim_penalty / bw
                if is_weighted:
                    fwd_compute *= topo.weighted_feature_bwd_compute_multiplier
                bwd_compute = fwd_compute * topo.bwd_compute_multiplier
                # comms: bytes that leave / enter this rank
                remote_frac = (W - 1) / W if W > 1 else 0.0
                if st == ShardingType.DATA_PARALLEL.value:
                    fwd_comms = 0.0
                    # dense all-reduce of the table gradient (ring / NVLS): ~2x table bytes
                    bwd_comms = (2 * rows * cols * elem * remote_frac) / comm_bw if W > 1 else 0.0
                    bwd_compute = fwd_compute * topo.bwd_compute_multiplier + rows * cols * elem * 3 / bw  # dense optimizer pass
                else:
                    fwd_comms = out_bytes * remote_frac / comm_bw
                    bwd_comms = fwd_comms
                    if st in (ShardingType.ROW_WISE.value, ShardingType.TABLE_ROW_WISE.value, ShardingType.GRID_SHARD.value):
                        # destination-side staging reduce: read n_row_shards slabs + write one
                        fwd_compute += (bags / max(W, 1)) * cols * out_elem * (n_row_shards + 1) / topo.hbm_mem_bw
                        if W > L and st != ShardingType.ROW_WISE.value:
                            # hierarchical: intra-node reduce first, then 1/L of the bytes cross nodes
                            fwd_comms = out_bytes * ((L - 1) / L) / intra + out_bytes / L * ((W / L - 1) / (W / L)) / inter
                            bwd_comms = fwd_comms
                    if W <= L and st in (ShardingType.TABLE_WISE.value, ShardingType.COLUMN_WISE.value, ShardingType.TABLE_COLUMN_WISE.value):
                        # fused lookup + NVLink store: transfer overlaps the gathers tile by tile
                        fwd_comms -= min(fwd_compute, fwd_comms) * fused_overlap(W)
                        bwd_comms *= GRAD_PUSH_EXPOSED  # pushed from inside the dense backward graph, beside the deferred wgrad GEMMs
                input_dist = ids * BIGINT_DTYPE * remote_frac / comm_bw if st != ShardingType.DATA_PARALLEL.value else 0.0
                prefetch_compute = 0.0
                if prefetch and caching_ratio is not None:
                    miss = max(0.0, 1.0 - caching_ratio)
                    prefetch_compute = ids * miss * cols * elem / topo.hbm_to_ddr_mem_bw
                if self._is_inference:
                    bwd_compute = bwd_comms = 0.0
                shard.perf = Perf(fwd_compute=fwd_compute, fwd_comms=fwd_comms, bwd_compute=bwd_compute, bwd_comms=bwd_comms,
                                  prefetch_compute=prefetch_compute, input_dist_comms=input_dist)


# ---- enumerator ------------------------------------------------------------------------------------------------
class EmbeddingEnumerator(Enumerator):
    """Generates the sharding options of every shardable parameter of a model."""

    def __init__(self, topology: Topology, batch_size: int, constraints: Optional[Dict[str, ParameterConstraints]] = None,
                 estimator: Optional[Union[ShardEstimator, List[ShardEstimator]]] = None, use_exact_enumerate_order: Optional[bool] = False) -> None:
        self._compute_device: str = topology.compute_device
        self._world_size: int = topology.world_size
        self._local_world_size: int = topology.local_world_size
        self._batch_size: int = batch_size
        self._constraints = constraints
        self._sharder_map: Dict[str, ModuleSharder[nn.Module]] = {}
        self._use_exact_enumerate_order = bool(use_exact_enumerate_order)
        self._last_stored_search_space: Optional[List[ShardingOption]] = None
        if estimator:
            self._estimators: List[ShardEstimator] = [estimator] if not isinstance(estimator, list) else estimator
        else:
            self._estimators = [EmbeddingPerfEstimator(topology=topology, constraints=constraints),
                                EmbeddingStorageEstimator(topology=topology, constraints=constraints)]

    def enumerate(self, module: nn.Module, sharders: List[ModuleSharder[nn.Module]]) -> List[ShardingOption]:
        self._sharder_map = {sharder_name(sharder.module_type): sharder for sharder in sharders}
        sharding_options: List[ShardingOption] = []
        named_modules_queue = [("", module)]
        while named_modules_queue:
            child_path, child_module = named_modules_queue.pop(0 if self._use_exact_enumerate_order else -1)
            sharder_key = sharder_name(type(child_module))
            sharder = self._sharder_map.get(sharder_key, None)
            if not sharder:
                for n, m in child_module.named_children():
                    named_modules_queue.append((child_path + "." + n if child_path != "" else n, m))
                continue
            is_weighted = bool(child_module.is_weighted()) if hasattr(child_module, "is_weighted") else False
            feature_by_table = self._feature_names(child_module)
            for name, param in sharder.shardable_parameters(child_module).items():
                c = self._constraints.get(name) if self._constraints else None
                input_lengths = list(c.pooling_factors) if c and c.pooling_factors else [POOLING_FACTOR]
                n_feat = len(feature_by_table.get(name, [name]))
                if len(input_lengths) == 1 and n_feat > 1:
                    input_lengths = input_lengths * n_feat
                sharding_options_per_table: List[ShardingOption] = []
                allowed_sharding_types = self._filter_sharding_types(name, sharder.sharding_types(self._compute_device))
                for sharding_type in allowed_sharding_types:
                    for compute_kernel in self._filter_compute_kernels(name, sharder.compute_kernels(sharding_type, self._compute_device), sharding_type):
                        col_wise_shard_dim = c.min_partition if c else None
                        try:
                            shard_sizes, shard_offsets = calculate_shard_sizes_and_offsets(
                                tensor=param, world_size=self._world_size, local_world_size=self._local_world_size,
                                sharding_type=sharding_type, col_wise_shard_dim=col_wise_shard_dim)
                        except ValueError:
                            continue
                        if sharding_type in (ShardingType.COLUMN_WISE.value, ShardingType.TABLE_COLUMN_WISE.value) and len(shard_sizes) == 1 and \
                                any(t not in (ShardingType.COLUMN_WISE.value, ShardingType.TABLE_COLUMN_WISE.value) for t in allowed_sharding_types):
                            continue  # identical to table-wise (kept when column-wise is all the user allows: a narrow table yields one slice)
                        if sharding_type == ShardingType.GRID_SHARD.value and (self._world_size <= self._local_world_size or len(shard_sizes) == self._local_world_size):
                            continue  # needs several hosts and several column shards
                        if sharding_type in (ShardingType.TABLE_ROW_WISE.value,) and self._world_size <= self._local_world_size and \
                                ShardingType.ROW_WISE.value in allowed_sharding_types:
                            continue  # equals row-wise on one NVLink domain (kept when it is the only type the user allows)
                        if sharding_type == ShardingType.TABLE_COLUMN_WISE.value and (self._world_size <= self._local_world_size or len(shard_sizes) > self._local_world_size):
                            continue
                        # wire / output dtype of the pooled embeddings: the constraint wins, else the sharder's fused_params["output_dtype"]
                        sharder_out_dtype = None
                        fp = getattr(sharder, "fused_params", None) or {}
                        if fp.get("output_dtype") is not None:
                            od = fp["output_dtype"]
                            sharder_out_dtype = od if isinstance(od, DataType) else _dtype_to_data_type(od)
                        sharding_options_per_table.append(ShardingOption(
                            name=name, tensor=param, module=(child_path, child_module), input_lengths=input_lengths, batch_size=self._batch_size,
                            compute_kernel=compute_kernel, sharding_type=sharding_type, partition_by=get_partition_by_type(sharding_type),
                            shards=[Shard(size=list(size), offset=list(offset)) for size, offset in zip(shard_sizes, shard_offsets)],
                            cache_params=c.cache_params if c else None, enforce_hbm=c.enforce_hbm if c else None,
                            stochastic_rounding=c.stochastic_rounding if c else None, bounds_check_mode=c.bounds_check_mode if c else None,
                            feature_names=feature_by_table.get(name), output_dtype=(c.output_dtype if c and c.output_dtype is not None else sharder_out_dtype),
                            key_value_params=c.key_value_params if c else None,
                        ))
                        sharding_options_per_table[-1].is_weighted = is_weighted
                if not sharding_options_per_table:
                    raise RuntimeError(f"No available sharding type and compute kernel combination after applying user provided constraints for {name}. "
                                       f"Module: {sharder_key}, sharder: {sharder.__class__.__name__}, compute device: {self._compute_device}.")
                sharding_options.extend(sharding_options_per_table)
        self.populate_estimates(sharding_options)
        self._last_stored_search_space = sharding_options
        return sharding_options

    @property
    def last_stored_search_space(self) -> Optional[List[ShardingOption]]:
        return self._last_stored_search_space

    def populate_estimates(self, sharding_options: List[ShardingOption]) -> None:
        for estimator in self._estimators:
            estimator.estimate(sharding_options, self._sharder_map)

    @staticmethod
    def _feature_names(module: nn.Module) -> Dict[str, List[str]]:
        out: Dict[str, List[str]] = {}
        for attr in ("embedding_bag_configs", "embedding_configs"):
            if hasattr(module, attr):
                try:
                    for cfg in getattr(module, attr)():
                        out[cfg.name] = list(cfg.feature_names)
                except TypeError:
                    pass
        return out

    def _filter_sharding_types(self, name: str, allowed_sharding_types: List[str]) -> List[str]:
        if not self._constraints or not self._constraints.get(name):
            return allowed_sharding_types
        constraints = self._constraints.get(name)
        if not constraints.sharding_types:
            return allowed_sharding_types
        filtered = list(set(constraints.sharding_types) & set(allowed_sharding_types))
        if not filtered:
            logger.warn(f"No available sharding types after applying user provided constraints for {name}. Constrained sharding types: "
                        f"{constraints.sharding_types}, allowed sharding types: {allowed_sharding_types}")
        return [t for t in allowed_sharding_types if t in filtered]

    def _filter_compute_kernels(self, name: str, allowed_compute_kernels: List[str], sharding_type: str) -> List[str]:
        if not self._constraints or not self._constraints.get(name) or not self._constraints[name].compute_kernels:
            filtered = [k for k in allowed_compute_kernels if k not in {g.value for g in GUARDED_COMPUTE_KERNELS}]
        else:
            constraints = self._constraints[name]
            filtered = [k for k in allowed_compute_kernels if k in set(constraints.compute_kernels)]
        if EmbeddingComputeKernel.DENSE.value in filtered and EmbeddingComputeKernel.FUSED.value in filtered:
            filtered.remove(EmbeddingComputeKernel.DENSE.value)  # fused is a strict improvement
        if not filtered:
            logger.warning(f"No available compute kernels after applying user provided constraints for {name}; allowed: {allowed_compute_kernels}")
        return filtered


def get_partition_by_type_for_option(so: ShardingOption) -> str:
    return get_partition_by_type(so.sharding_type)
