"""Per-group training kernels: one ``TableBatchedEmbeddingBags`` per ``GroupedEmbeddingConfig``.

Reference: ``torchrec/distributed/batched_embedding_kernel.py`` - ``BaseBatchedEmbeddingBag`` :2915-3124, ``BatchedFusedEmbeddingBag`` :3703-3826,
``BatchedDenseEmbeddingBag`` :4636, the sequence twins :1729-2913, ``EmbeddingFusedOptimizer`` :1195-1624 and the key-value (virtual table) variants
:1917-2508 / :3127-3700. The reference builds FBGEMM ``SplitTableBatchedEmbeddingBagsCodegen`` / ``DenseTableBatchedEmbeddingBagsCodegen`` / SSD TBEs; here
every variant is the same hand-written sm_90a kernel family (``ops/csrc/tbe_fwd.cu`` / ``tbe_bwd.cu`` through ``ops/tbe.py``) configured by

* the optimizer (``OptimType.NONE`` -> dense gradient for DDP / an external optimizer, anything else -> fused into the backward),
* the pooling mode (SUM / MEAN for bags, NONE for sequence lookups),
* where the rows live: HBM (``fused``), host-mapped (``fused_uvm``) or host rows behind an HBM row cache (``fused_uvm_caching`` and the key-value kernels,
  ``ops/uvm.py``) - on an 80 GB part the cache variant is what the reference's SSD/DRAM virtual tables become.
"""
from __future__ import annotations

import copy
import itertools
from collections import OrderedDict
from dataclasses import dataclass
from typing import Any, Dict, Generic, Iterator, List, Optional, Tuple, TypeVar

import torch
import torch.distributed as dist
from torch import nn

from ..modules.embedding_configs import DataType, PoolingType, data_type_to_dtype
from ..ops.tbe import EmbeddingLocation, OptimType, PoolingMode, TableBatchedEmbeddingBags
from ..optim.fused import FusedOptimizer, FusedOptimizerModule
from ..sparse.jagged_tensor import KeyedJaggedTensor
from .embedding_kernel import BaseEmbedding, get_state_dict
from .embedding_types import EmbeddingComputeKernel, GroupedEmbeddingConfig, ShardedEmbeddingTable
from .types import LazyAwaitable

SplitWeightType = TypeVar("SplitWeightType")


class ReduceScatterResizeAwaitable(LazyAwaitable[torch.Tensor]):
    """Waits an async reduce-scatter of a padded gradient and trims the padding rows (fully-sharded 2D tables, reference :125-171)."""

    def __init__(self, async_work: Optional[Any], output_tensor: torch.Tensor, unpadded_rows: int) -> None:
        super().__init__()
        self._work, self._out, self._rows = async_work, output_tensor, unpadded_rows

    def _wait_impl(self) -> torch.Tensor:
        if self._work is not None:
            self._work.wait()
        return self._out[: self._rows]


@dataclass
class ShardParams:
    """Layout of a fully-sharded (2D) kernel's weight buffer inside a replica group (reference :606-612)."""

    embedding_dim: int
    local_rows: List[int]
    shard_rows: List[int]
    padded_rows: List[int]


def _assert_local_cols_divisible_by_4(config: GroupedEmbeddingConfig) -> None:
    """The lookup kernels move rows as 16-byte vectors (reference :1906-1914 has the same rule for FBGEMM)."""
    for t in config.embedding_tables:
        if t.local_cols % 4 != 0:
            raise ValueError(f"table {t.name}: local_cols {t.local_cols} is not divisible by 4")


def _location_of(kernel: EmbeddingComputeKernel) -> Tuple[EmbeddingLocation, bool]:
    """compute kernel -> (row location, needs the HBM row cache)."""
    k = kernel.value if isinstance(kernel, EmbeddingComputeKernel) else str(kernel)
    if k == "fused_uvm":
        return EmbeddingLocation.MANAGED, False
    if k in ("fused_uvm_caching", "key_value", "ssd_virtual_table", "dram_virtual_table"):
        return EmbeddingLocation.MANAGED_CACHING, True
    return EmbeddingLocation.DEVICE, False


def _optimizer_kwargs(fused_params: Optional[Dict[str, Any]]) -> Dict[str, Any]:
    """``fused_params`` of a sharder (FBGEMM spelling) -> TableBatchedEmbeddingBags keyword arguments."""
    from .embeddingbag import optimizer_spec_from

    spec, _ = optimizer_spec_from(None, fused_params)
    return dict(optimizer=spec.optim, learning_rate=spec.lr, eps=spec.eps, beta1=spec.beta1, beta2=spec.beta2, weight_decay=spec.weight_decay,
                weight_decay_mode=spec.weight_decay_mode, max_gradient=spec.max_gradient, momentum=spec.momentum, stochastic_rounding=spec.stochastic_rounding)


def _build_tbe(config: GroupedEmbeddingConfig, device: Optional[torch.device], pooling: PoolingMode, dense: bool) -> nn.Module:
    _assert_local_cols_divisible_by_4(config)
    specs = [(t.local_rows, t.local_cols) for t in config.embedding_tables]
    ftm = [i for i, t in enumerate(config.embedding_tables) for _ in t.feature_names]
    dtype = torch.float32 if config.data_type == DataType.FP32 else data_type_to_dtype(config.data_type)
    fp = dict(config.fused_params or {})
    out_dtype = fp.get("output_dtype", torch.float32)
    if isinstance(out_dtype, DataType):
        out_dtype = data_type_to_dtype(out_dtype)
    dev = torch.device(device) if device is not None else torch.device("cpu")
    kwargs: Dict[str, Any] = dict(embedding_specs=specs, feature_table_map=ftm, pooling_mode=pooling, weights_precision=dtype, output_dtype=out_dtype,
                                  device=dev, table_names=[t.name for t in config.embedding_tables])
    if dense:
        kwargs["optimizer"] = OptimType.NONE
        return TableBatchedEmbeddingBags(**kwargs)
    kwargs.update(_optimizer_kwargs(fp))
    loc, cached = _location_of(config.compute_kernel)
    if dev.type != "cuda":
        loc, cached = EmbeddingLocation.HOST, False
    if cached:
        from ..ops.uvm import UvmCachedEmbeddingBags

        kwargs.pop("stochastic_rounding", None)
        return UvmCachedEmbeddingBags(cache_load_factor=float(fp.get("cache_load_factor", 0.2)), **kwargs)
    return TableBatchedEmbeddingBags(location=loc, **kwargs)


def _init_ranges(config: GroupedEmbeddingConfig) -> List[Tuple[float, float]]:
    out = []
    for t in config.embedding_tables:
        lo = t.get_weight_init_min() if hasattr(t, "get_weight_init_min") else -(1.0 / t.num_embeddings) ** 0.5
        hi = t.get_weight_init_max() if hasattr(t, "get_weight_init_max") else (1.0 / t.num_embeddings) ** 0.5
        out.append((float(lo), float(hi)))
    return out


# ---- fused optimizer view of ONE kernel ------------------------------------------------------------------------------
class EmbeddingFusedOptimizer(FusedOptimizer):
    """KeyedOptimizer over the optimizer state that lives inside a fused kernel (reference :1195-1624).

    ``params`` maps ``{table}.weight`` to the table's weight view (or the ShardedTensor when ``create_for_table`` is given shard metadata);
    ``state[param]`` holds ``{table}.{state name}`` views (row-wise states are 1-D ``[local_rows]``, like FBGEMM's ``momentum1`` of row-wise Adagrad).
    ``step`` only pushes hyper-parameters: the update already happened inside the backward kernel."""

    def __init__(self, config: GroupedEmbeddingConfig, emb_module: nn.Module, pg: Optional[dist.ProcessGroup] = None,
                 create_for_table: Optional[str] = None, param_weight_for_table: Optional[nn.Parameter] = None,
                 embedding_weights_by_table: Optional[List[torch.Tensor]] = None, all_optimizer_states: Optional[List[Dict[str, torch.Tensor]]] = None) -> None:
        self._emb_module = emb_module
        self._pg = pg
        weights = embedding_weights_by_table if embedding_weights_by_table is not None else emb_module.split_embedding_weights()
        states = all_optimizer_states if all_optimizer_states is not None else emb_module.split_optimizer_states()
        tables = config.embedding_tables
        sd = get_state_dict(tables, list(weights), pg)
        params: Dict[str, Any] = OrderedDict()
        state: Dict[Any, Any] = OrderedDict()
        seen: Dict[str, Any] = {}
        for t, w, st in zip(tables, weights, states):
            if create_for_table is not None and t.name != create_for_table:
                continue
            key = f"{t.name}.weight"
            p = param_weight_for_table if (param_weight_for_table is not None and create_for_table == t.name) else sd[key]
            if key in seen:  # a second local shard of the same table (column-wise): states are concatenated along dim 1 / shared per row
                prev = state[seen[key]]
                for name, v in st.items():
                    k = f"{t.name}.{name}"
                    if k in prev and v.dim() == 2:
                        prev[k] = torch.cat([prev[k], v], dim=1)
                continue
            seen[key] = p
            params[key] = p
            state[p] = {f"{t.name}.{name}": v for name, v in st.items()}
        lr = emb_module.get_learning_rate() if hasattr(emb_module, "get_learning_rate") else 0.01
        groups = [{"params": list(params.values()), "lr": lr}]
        super().__init__(params, state, groups)

    def zero_grad(self, set_to_none: bool = False) -> None:
        pass  # sparse gradients never materialise

    def step(self, closure: Any = None) -> None:
        self._emb_module.set_learning_rate(self.param_groups[0]["lr"])

    def set_optimizer_step(self, step: int) -> None:
        self._emb_module.set_optimizer_step(step)

    def update_hyper_parameters(self, params_dict: Dict[str, Any]) -> None:
        if "lr" in params_dict:
            self.param_groups[0]["lr"] = float(params_dict["lr"])
            self._emb_module.set_learning_rate(float(params_dict["lr"]))
        host = getattr(self._emb_module, "hyper_host", None)
        if host is not None:
            for name, slot in (("eps", 1), ("beta1", 2), ("beta2", 3), ("weight_decay", 4)):
                if name in params_dict:
                    host[slot] = float(params_dict[name])
            if hasattr(self._emb_module, "_push_hyper"):
                self._emb_module._push_hyper()


class KeyValueEmbeddingFusedOptimizer(EmbeddingFusedOptimizer):
    """Optimizer view of a key-value kernel: states are read through the row cache (flushes first) - reference :615-1049."""

    def __init__(self, config: GroupedEmbeddingConfig, emb_module: nn.Module, pg: Optional[dist.ProcessGroup] = None) -> None:
        if hasattr(emb_module, "flush"):
            emb_module.flush()
        super().__init__(config, emb_module, pg)


class ZeroCollisionKeyValueEmbeddingFusedOptimizer(KeyValueEmbeddingFusedOptimizer):
    """reference :1052-1192 (bucketised virtual tables); same state layout here."""


# ---- named parameters -----------------------------------------------------------------------------------------------
def _gen_named_parameters_by_table_fused(emb_module: nn.Module, table_name_to_count: Dict[str, int], config: GroupedEmbeddingConfig,
                                         pg: Optional[dist.ProcessGroup] = None) -> Iterator[Tuple[str, nn.Parameter]]:
    """One ``TableBatchedEmbeddingSlice`` per table over the flat fused buffer, each carrying its own fused-optimizer view (reference :1649-1701)."""
    from .composable.table_batched_embedding_slice import TableBatchedEmbeddingSlice

    weights = emb_module.split_embedding_weights()
    flat = emb_module.weights
    done: Dict[str, Any] = {}
    off = 0
    spans: Dict[str, List[Tuple[int, int, int]]] = OrderedDict()
    for t, w in zip(config.embedding_tables, weights):
        n = w.numel()
        spans.setdefault(t.name, []).append((off, off + n, t.local_cols))
        off += n
    for name, lst in spans.items():
        start, end = lst[0][0], lst[-1][1]
        cols = lst[0][2]
        try:
            p = TableBatchedEmbeddingSlice(flat, start, end, (end - start) // cols, cols)
        except Exception:
            p = nn.Parameter(flat.detach()[start:end].view(-1, cols), requires_grad=False)
        p._in_backward_optimizers = [EmbeddingFusedOptimizer(config, emb_module, pg, create_for_table=name, param_weight_for_table=p)]  # type: ignore[attr-defined]
        done[name] = p
        yield name, p


def _gen_named_parameters_by_table_dense(emb_module: nn.Module, table_name_to_count: Dict[str, int], config: GroupedEmbeddingConfig) -> Iterator[Tuple[str, nn.Parameter]]:
    """Per-table slices of the dense kernel's single autograd Parameter (reference :1704-1726)."""
    from .composable.table_batched_embedding_slice import TableBatchedEmbeddingSlice

    off = 0
    spans: Dict[str, List[Tuple[int, int, int]]] = OrderedDict()
    for t in config.embedding_tables:
        n = t.local_rows * t.local_cols
        spans.setdefault(t.name, []).append((off, off + n, t.local_cols))
        off += n
    for name, lst in spans.items():
        start, end, cols = lst[0][0], lst[-1][1], lst[0][2]
        try:
            yield name, TableBatchedEmbeddingSlice(emb_module.weights, start, end, (end - start) // cols, cols)
        except Exception:
            yield name, nn.Parameter(emb_module.weights.detach()[start:end].view(-1, cols))


# ---- kernels --------------------------------------------------------------------------------------------------------
class _BatchedBase(BaseEmbedding, Generic[SplitWeightType]):
    _POOLED = True
    _DENSE = False

    def __init__(self, config: GroupedEmbeddingConfig, pg: Optional[dist.ProcessGroup] = None, device: Optional[torch.device] = None,
                 sharding_type: Optional[Any] = None, env: Optional[Any] = None) -> None:
        super().__init__()
        self._config = config
        self._pg = pg
        self._device = torch.device(device) if device is not None else torch.device("cpu")
        self._sharding_type = sharding_type
        self._env = env
        self._pooling = PoolingMode.NONE if not self._POOLED else (PoolingMode.MEAN if config.pooling == PoolingType.MEAN else PoolingMode.SUM)
        self._local_rows = [t.local_rows for t in config.embedding_tables]
        self._local_cols = [t.local_cols for t in config.embedding_tables]
        self._weight_init_mins = [r[0] for r in _init_ranges(config)]
        self._weight_init_maxs = [r[1] for r in _init_ranges(config)]
        self._num_embeddings = [t.num_embeddings for t in config.embedding_tables]
        self._feature_table_map: List[int] = [i for i, t in enumerate(config.embedding_tables) for _ in t.feature_names]
        self.table_name_to_count: Dict[str, int] = {}
        for t in config.embedding_tables:
            self.table_name_to_count[t.name] = self.table_name_to_count.get(t.name, 0) + 1
        self._emb_module = _build_tbe(config, self._device, self._pooling, self._DENSE)
        self._param_per_table: Dict[str, nn.Parameter] = {}
        if self._device.type != "meta":
            self.init_parameters()

    # ---- reference surface ----
    @property
    def config(self) -> GroupedEmbeddingConfig:
        return self._config

    @property
    def emb_module(self) -> nn.Module:
        return self._emb_module

    def init_parameters(self) -> None:
        """Uniform init in each table's ``[weight_init_min, weight_init_max]``; a config's ``init_fn`` wins (reference :3017-3035)."""
        self._emb_module.init_parameters(list(zip(self._weight_init_mins, self._weight_init_maxs)))
        for t, w in zip(self._config.embedding_tables, self.split_embedding_weights()):
            fn = getattr(t, "init_fn", None)
            if fn is not None:
                tmp = torch.empty(w.shape, dtype=torch.float32, device=w.device)
                fn(tmp)
                w.copy_(tmp)

    def forward(self, features: KeyedJaggedTensor) -> torch.Tensor:
        self._track_raw_ids(features)
        weights = features.weights_or_none() if (self._POOLED and self._config.is_weighted) else None
        F = max(len(self._feature_table_map), 1)
        offsets = features.offsets()
        B = (offsets.numel() - 1) // F
        return self._emb_module(features.values(), offsets, weights, batch_size=B)

    def split_embedding_weights(self) -> List[torch.Tensor]:
        return self._emb_module.split_embedding_weights()

    def named_split_embedding_weights(self, prefix: str = "", recurse: bool = True, remove_duplicate: bool = True) -> Iterator[Tuple[str, torch.Tensor]]:
        for t, w in zip(self._config.embedding_tables, self.split_embedding_weights()):
            yield (f"{prefix}.{t.name}.weight" if prefix else f"{t.name}.weight"), w

    def state_dict(self, destination: Optional[Dict[str, Any]] = None, prefix: str = "", keep_vars: bool = False) -> Dict[str, Any]:  # type: ignore[override]
        self.flush()
        return get_state_dict(self._config.embedding_tables, self.split_embedding_weights(), self._pg, destination, prefix)

    def load_state_dict(self, state_dict: Dict[str, Any], strict: bool = True) -> Any:  # type: ignore[override]
        missing: List[str] = []
        for t, w in zip(self._config.embedding_tables, self.split_embedding_weights()):
            key = f"{t.name}.weight"
            if key not in state_dict:
                missing.append(key)
                continue
            src = state_dict[key]
            if hasattr(src, "local_shards"):
                shards = src.local_shards()
                md = t.local_metadata
                src = next((s.tensor for s in shards if md is None or list(s.metadata.shard_offsets) == list(md.shard_offsets)), shards[0].tensor)
            w.copy_(src.to(w.dtype))
        if hasattr(self._emb_module, "load_rows_changed"):
            self._emb_module.load_rows_changed()
        if strict and missing:
            raise RuntimeError(f"missing keys: {missing}")
        return torch.nn.modules.module._IncompatibleKeys(missing, [])

    def named_buffers(self, prefix: str = "", recurse: bool = True, remove_duplicate: bool = True) -> Iterator[Tuple[str, torch.Tensor]]:
        yield from ()

    def flush(self) -> None:
        if hasattr(self._emb_module, "flush"):
            self._emb_module.flush()

    def purge(self) -> None:
        if hasattr(self._emb_module, "flush"):
            self._emb_module.flush(invalidate=True)

    def prefetch(self, features: KeyedJaggedTensor, forward_stream: Optional[torch.cuda.Stream] = None) -> None:
        if hasattr(self._emb_module, "prefetch"):
            F = max(len(self._feature_table_map), 1)
            self._emb_module.prefetch(features.values(), features.offsets(), (features.offsets().numel() - 1) // F)


class _FusedMixin(FusedOptimizerModule):
    _emb_module: nn.Module
    _config: GroupedEmbeddingConfig
    _pg: Optional[dist.ProcessGroup]
    _OPTIM_CLS = EmbeddingFusedOptimizer

    def _init_fused(self) -> None:
        self._optim = self._OPTIM_CLS(self._config, self._emb_module, self._pg)
        self._param_per_table = dict(_gen_named_parameters_by_table_fused(self._emb_module, self.table_name_to_count, self._config, self._pg))  # type: ignore[attr-defined]

    @property
    def fused_optimizer(self) -> FusedOptimizer:
        return self._optim

    def named_parameters(self, prefix: str = "", recurse: bool = True, remove_duplicate: bool = True) -> Iterator[Tuple[str, nn.Parameter]]:
        """Per-table parameters tagged with ``_in_backward_optimizers`` - they never receive ``.grad`` (reference :3793-3806)."""
        for name, p in self._param_per_table.items():  # type: ignore[attr-defined]
            yield (f"{prefix}.{name}.weight" if prefix else f"{name}.weight"), p


class BaseBatchedEmbeddingBag(_BatchedBase[SplitWeightType]):
    """Pooled lookup over one group of tables (reference :2915)."""

    _POOLED = True


class BaseBatchedEmbedding(_BatchedBase[SplitWeightType]):
    """Sequence (un-pooled) lookup over one group of tables: output ``[sum(lengths), D]`` (reference :1729)."""

    _POOLED = False


class BatchedFusedEmbeddingBag(BaseBatchedEmbeddingBag[torch.Tensor], _FusedMixin):
    """Pooled lookup with the optimizer fused into the backward kernel; HBM / host-mapped / cached rows by compute kernel (reference :3703)."""

    def __init__(self, config: GroupedEmbeddingConfig, pg: Optional[dist.ProcessGroup] = None, device: Optional[torch.device] = None,
                 sharding_type: Optional[Any] = None, env: Optional[Any] = None) -> None:
        super().__init__(config, pg, device, sharding_type, env)
        self._init_fused()


class BatchedFusedEmbedding(BaseBatchedEmbedding[torch.Tensor], _FusedMixin):
    """Sequence twin of ``BatchedFusedEmbeddingBag`` (reference :2510)."""

    def __init__(self, config: GroupedEmbeddingConfig, pg: Optional[dist.ProcessGroup] = None, device: Optional[torch.device] = None,
                 sharding_type: Optional[Any] = None, env: Optional[Any] = None) -> None:
        super().__init__(config, pg, device, sharding_type, env)
        self._init_fused()


class _DenseMixin:
    def named_parameters(self, prefix: str = "", recurse: bool = True, remove_duplicate: bool = True) -> Iterator[Tuple[str, nn.Parameter]]:
        """The combined flat Parameter under the reference's combined key (``t1_t2.weight``): DDP / dense optimizers see ONE tensor (reference :4676-4688)."""
        key = "_".join(dict.fromkeys(t.name for t in self._config.embedding_tables))  # type: ignore[attr-defined]
        yield (f"{prefix}.{key}.weight" if prefix else f"{key}.weight"), self._emb_module.weights  # type: ignore[attr-defined]

    def named_parameters_by_table(self) -> Iterator[Tuple[str, nn.Parameter]]:
        yield from _gen_named_parameters_by_table_dense(self._emb_module, self.table_name_to_count, self._config)  # type: ignore[attr-defined]


class BatchedDenseEmbeddingBag(_DenseMixin, BaseBatchedEmbeddingBag[torch.Tensor]):
    """Pooled lookup whose backward writes a dense ``weights.grad`` (data-parallel tables under DDP) - reference :4636."""

    _DENSE = True


class BatchedDenseEmbedding(_DenseMixin, BaseBatchedEmbedding[torch.Tensor]):
    """reference :2858."""

    _DENSE = True


# ---- fully-sharded (2D) kernels: weights of a replica group are themselves row-sharded over the group --------------------
class _FullyShardedMixin:
    """``ShardingStrategy.FULLY_SHARDED`` of ``DMPCollection``: between the forward lookup and the backward each replica keeps 1/R of the
    (replica-averaged) flat weight buffer; it is all-gathered back before the fused backward (reference :2647-2855, :4423-4633). The state machine
    is ``parallel/fully_sharded.py: FullyShardedTBEWeights`` attached to the kernel (``tbe._fs``); the lookup autograd functions drive it."""

    def _init_fully_sharded(self, env: Any) -> None:
        from .fully_sharded import attach

        self._replica_pg = getattr(env, "replica_pg", None)
        R = dist.get_world_size(self._replica_pg) if self._replica_pg is not None else 1
        rows = [t.local_rows for t in self._config.embedding_tables]  # type: ignore[attr-defined]
        padded = [-(-r // R) * R for r in rows]
        self._shard_params = ShardParams(embedding_dim=max(self._local_cols), local_rows=rows, shard_rows=[p // R for p in padded], padded_rows=padded)  # type: ignore[attr-defined]
        self._fs = attach(self._emb_module, self._replica_pg) if self._replica_pg is not None else None  # type: ignore[attr-defined]

    @property
    def shard_params(self) -> ShardParams:
        return self._shard_params

    def _all_gather_table_weights(self) -> None:
        """Bring the full (averaged) buffer back, e.g. before a forward or a state_dict."""
        if self._fs is not None:
            self._fs.gather()


class ShardedBatchedFusedEmbeddingBag(BatchedFusedEmbeddingBag, _FullyShardedMixin):
    def __init__(self, config: GroupedEmbeddingConfig, pg: Optional[dist.ProcessGroup] = None, device: Optional[torch.device] = None,
                 sharding_type: Optional[Any] = None, env: Optional[Any] = None) -> None:
        super().__init__(config, pg, device, sharding_type, env)
        self._init_fully_sharded(env)

    def forward(self, features: KeyedJaggedTensor) -> torch.Tensor:
        self._all_gather_table_weights()
        return super().forward(features)


class ShardedBatchedFusedEmbedding(BatchedFusedEmbedding, _FullyShardedMixin):
    def __init__(self, config: GroupedEmbeddingConfig, pg: Optional[dist.ProcessGroup] = None, device: Optional[torch.device] = None,
                 sharding_type: Optional[Any] = None, env: Optional[Any] = None) -> None:
        super().__init__(config, pg, device, sharding_type, env)
        self._init_fully_sharded(env)

    def forward(self, features: KeyedJaggedTensor) -> torch.Tensor:
        self._all_gather_table_weights()
        return super().forward(features)


# ---- key-value (virtual table) kernels: host-resident rows behind an HBM cache ------------------------------------------
class _KeyValueMixin(_FusedMixin):
    _OPTIM_CLS = KeyValueEmbeddingFusedOptimizer

    def _force_cached(self, config: GroupedEmbeddingConfig) -> GroupedEmbeddingConfig:
        cfg = copy.copy(config)
        if cfg.compute_kernel not in (EmbeddingComputeKernel.KEY_VALUE, EmbeddingComputeKernel.FUSED_UVM_CACHING):
            cfg.compute_kernel = EmbeddingComputeKernel.KEY_VALUE
        return cfg

    def get_named_split_embedding_weights_snapshot(self, prefix: str = "") -> Iterator[Tuple[str, torch.Tensor, Optional[torch.Tensor], Optional[torch.Tensor], Optional[torch.Tensor]]]:
        """(name, weights, weight ids, bucket counts, metadata) after a cache flush - the checkpoint view of a virtual table (reference :2040-2070)."""
        self.flush()  # type: ignore[attr-defined]
        for t, w in zip(self._config.embedding_tables, self.split_embedding_weights()):  # type: ignore[attr-defined]
            name = f"{prefix}.{t.name}.weight" if prefix else f"{t.name}.weight"
            yield name, w, None, None, None


class KeyValueEmbeddingBag(_KeyValueMixin, BaseBatchedEmbeddingBag[torch.Tensor]):
    """reference :3127 - SSD / DRAM backed TBE; here host rows + HBM row cache (``UvmCachedEmbeddingBags``)."""

    def __init__(self, config: GroupedEmbeddingConfig, pg: Optional[dist.ProcessGroup] = None, device: Optional[torch.device] = None,
                 sharding_type: Optional[Any] = None, env: Optional[Any] = None, backend_type: Any = None) -> None:
        super().__init__(self._force_cached(config), pg, device, sharding_type, env)
        self._backend_type = backend_type
        self._init_fused()


class KeyValueEmbedding(_KeyValueMixin, BaseBatchedEmbedding[torch.Tensor]):
    """reference :1917."""

    def __init__(self, config: GroupedEmbeddingConfig, pg: Optional[dist.ProcessGroup] = None, device: Optional[torch.device] = None,
                 sharding_type: Optional[Any] = None, env: Optional[Any] = None, backend_type: Any = None) -> None:
        super().__init__(self._force_cached(config), pg, device, sharding_type, env)
        self._backend_type = backend_type
        self._init_fused()


class _ZeroCollisionMixin(_KeyValueMixin):
    """Virtual tables addressed by bucketised ids: ``total_num_buckets`` buckets are range-split over the shards; a local id is
    ``global id - bucket_offset * bucket_size`` (reference ``_get_sharded_local_buckets_for_zero_collision`` :562-603)."""

    _OPTIM_CLS = ZeroCollisionKeyValueEmbeddingFusedOptimizer

    def _init_buckets(self) -> None:
        self._bucket_offsets: List[Tuple[int, int]] = []
        self._bucket_sizes: List[int] = []
        for t in self._config.embedding_tables:  # type: ignore[attr-defined]
            total = getattr(t, "total_num_buckets", None) or 1
            size = -(-t.num_embeddings // total)
            row0 = t.local_metadata.shard_offsets[0] if t.local_metadata is not None else 0
            start = row0 // size
            end = -(-(row0 + t.local_rows) // size)
            self._bucket_offsets.append((start, end))
            self._bucket_sizes.append(size)

    def get_sharded_local_buckets(self) -> List[Tuple[int, int, int]]:
        return [(a, b, s) for (a, b), s in zip(self._bucket_offsets, self._bucket_sizes)]


def _get_sharded_local_buckets_for_zero_collision(embedding_tables: List[ShardedEmbeddingTable], pg: Optional[dist.ProcessGroup] = None) -> List[Tuple[int, int, int]]:
    out = []
    for t in embedding_tables:
        total = getattr(t, "total_num_buckets", None) or 1
        size = -(-t.num_embeddings // total)
        row0 = t.local_metadata.shard_offsets[0] if t.local_metadata is not None else 0
        out.append((row0 // size, -(-(row0 + t.local_rows) // size), size))
    return out


class ZeroCollisionKeyValueEmbeddingBag(_ZeroCollisionMixin, BaseBatchedEmbeddingBag[torch.Tensor]):
    """reference :3314."""

    def __init__(self, config: GroupedEmbeddingConfig, pg: Optional[dist.ProcessGroup] = None, device: Optional[torch.device] = None,
                 sharding_type: Optional[Any] = None, env: Optional[Any] = None, backend_type: Any = None) -> None:
        super().__init__(self._force_cached(config), pg, device, sharding_type, env)
        self._init_buckets()
        self._init_fused()


class ZeroCollisionKeyValueEmbedding(_ZeroCollisionMixin, BaseBatchedEmbedding[torch.Tensor]):
    """reference :2106."""

    def __init__(self, config: GroupedEmbeddingConfig, pg: Optional[dist.ProcessGroup] = None, device: Optional[torch.device] = None,
                 sharding_type: Optional[Any] = None, env: Optional[Any] = None, backend_type: Any = None) -> None:
        super().__init__(self._force_cached(config), pg, device, sharding_type, env)
        self._init_buckets()
        self._init_fused()


class ZeroCollisionEmbeddingCache(ZeroCollisionKeyValueEmbedding):
    """HBM-only cache front of a remote virtual table (reference :2450): rows not in the cache read as zeros until written back."""


class ZeroCollisionEmbeddingEnrichmentCache(ZeroCollisionKeyValueEmbedding):
    """reference :2480."""
