"""ShardedEmbeddingBagCollection + sharder (reference torchrec/distributed/embeddingbag.py).

One ``ShardedLookupEngine`` (see ``engine.py``) serves every model-parallel table of the module
regardless of sharding type; data-parallel tables run a dense local kernel wrapped in DDP. The
module keeps the reference contract: ``input_dist -> compute -> output_dist`` returning a
``LazyAwaitable[KeyedTensor]``, ``state_dict`` keys ``embedding_bags.<table>.weight`` backed by
``ShardedTensor``, a ``fused_optimizer`` with per-table state keys ``<table>.momentum1``.
"""
from __future__ import annotations

import copy
from collections import OrderedDict
from dataclasses import dataclass, field
from typing import Any, Dict, Iterator, List, Mapping, Optional, Set, Tuple, Type, Union

import torch
import torch.distributed as dist
from torch import nn
from torch.distributed._shard.sharded_tensor import Shard, ShardedTensor, ShardedTensorMetadata, TensorProperties
from torch.nn.parallel import DistributedDataParallel

from ..modules.embedding_configs import BaseEmbeddingConfig, DataType, EmbeddingBagConfig, PoolingType, data_type_to_dtype
from ..modules.embedding_modules import EmbeddingBagCollection, EmbeddingBagCollectionInterface, get_embedding_names_by_table
from ..ops import vbe as V
from ..ops.tbe import OptimType, PoolingMode, TableBatchedEmbeddingBags, WeightDecayMode
from ..optim.fused import EmptyFusedOptimizer, FusedOptimizer, FusedOptimizerModule
from ..optim.keyed import CombinedOptimizer, KeyedOptimizer
from ..sparse.jagged_tensor import KeyedJaggedTensor, KeyedTensor
from ..streamable import Multistreamable
from .embedding_types import BaseEmbeddingSharder, EmbeddingComputeKernel, KJTList, ShardedEmbeddingModule
from .engine import OptimizerSpec, ShardedLookupEngine, TableShard
from .sharding_plan import placement
from .types import (
    Awaitable,
    EmbeddingModuleShardingPlan,
    LazyAwaitable,
    NoWait,
    ParameterSharding,
    QuantizedCommCodecs,
    ShardedModule,
    ShardingEnv,
    ShardingType,
    ShardMetadata,
    CommOp,
)


# ---- optimizer tags -> fused optimizer spec -----------------------------------------------------------
def optimizer_spec_from(param: Optional[torch.Tensor], fused_params: Optional[Dict[str, Any]]) -> Tuple[OptimizerSpec, bool]:
    """Read ``apply_optimizer_in_backward`` tags (and sharder ``fused_params``) into an OptimizerSpec.
    Returns (spec, has_in_backward_optimizer). Mapping parity: reference distributed/utils.py:325-341."""
    from ..optim import optimizers as shells
    from ..optim.rowwise_adagrad import RowWiseAdagrad

    spec = OptimizerSpec()
    fp = dict(fused_params or {})
    tagged = False
    cls = kwargs = None
    if param is not None:
        classes = getattr(param, "_optimizer_classes", None)
        if classes:
            cls = classes[0]
            kw_list = getattr(param, "_optimizer_kwargs_list", None)
            kwargs = kw_list[0] if kw_list else getattr(param, "_optimizer_kwargs", {})
        elif getattr(param, "_optimizer_class", None) is not None:
            cls = param._optimizer_class
            kwargs = getattr(param, "_optimizer_kwargs", {})
    if cls is not None:
        tagged = True
        kwargs = dict(kwargs or {})
        mapping = {
            torch.optim.SGD: OptimType.EXACT_SGD, shells.SGD: OptimType.EXACT_SGD,
            torch.optim.Adagrad: OptimType.EXACT_ADAGRAD, shells.Adagrad: OptimType.EXACT_ADAGRAD,
            torch.optim.Adam: OptimType.ADAM, shells.Adam: OptimType.ADAM, torch.optim.AdamW: OptimType.ADAMW,
            RowWiseAdagrad: OptimType.EXACT_ROWWISE_ADAGRAD,
            shells.PartialRowWiseAdam: OptimType.PARTIAL_ROWWISE_ADAM, shells.LAMB: OptimType.LAMB,
            shells.PartialRowWiseLAMB: OptimType.PARTIAL_ROWWISE_LAMB, shells.LarsSGD: OptimType.LARS_SGD,
        }
        if cls not in mapping:
            raise ValueError(f"Cannot fuse optimizer {cls} into the embedding backward kernel")
        spec.optim = mapping[cls]
        if "lr" in kwargs:
            spec.lr = float(kwargs["lr"])
        if "eps" in kwargs:
            spec.eps = float(kwargs["eps"])
        if "betas" in kwargs:
            spec.beta1, spec.beta2 = float(kwargs["betas"][0]), float(kwargs["betas"][1])
        if "weight_decay" in kwargs and kwargs["weight_decay"]:
            spec.weight_decay = float(kwargs["weight_decay"])
            spec.weight_decay_mode = WeightDecayMode.DECOUPLE if cls is torch.optim.AdamW else WeightDecayMode.L2
        if cls is torch.optim.Adagrad:
            spec.eps = float(kwargs.get("eps", 1e-10))
        if "momentum" in kwargs:
            spec.momentum = float(kwargs["momentum"])
        if "eta" in kwargs:
            spec.momentum = float(kwargs["eta"])
    if "optimizer" in fp:
        o = fp["optimizer"]
        if isinstance(o, OptimType):
            spec.optim = o
        else:
            key = str(getattr(o, "value", o))
            try:
                spec.optim = OptimType(key)
            except ValueError:  # enum NAME spelling ("EXACT_ROWWISE_ADAGRAD"), as FBGEMM's ``EmbOptimType.X`` prints
                spec.optim = OptimType[key.split(".")[-1].upper()]
        tagged = True
    for src, dst in (("learning_rate", "lr"), ("eps", "eps"), ("beta1", "beta1"), ("beta2", "beta2"), ("weight_decay", "weight_decay"),
                     ("max_gradient", "max_gradient"), ("momentum", "momentum")):
        if src in fp:
            setattr(spec, dst, float(fp[src]))
    if "weight_decay_mode" in fp:
        spec.weight_decay_mode = WeightDecayMode(int(getattr(fp["weight_decay_mode"], "value", fp["weight_decay_mode"])))
    if fp.get("stochastic_rounding") is not None:
        spec.stochastic_rounding = bool(fp["stochastic_rounding"])
    return spec, tagged


# ---- fused optimizer view -----------------------------------------------------------------------------------
def _sharded_tensor_from_local(local: List[Tuple[torch.Tensor, List[int], List[int]]], global_shards: List[Tuple[List[int], List[int], int]],
                               size: List[int], dtype: torch.dtype, pg: Optional[dist.ProcessGroup], device_type: str, local_size: int, rank: int):
    """Build a ShardedTensor from local shard tensors + the global shard layout (no communication)."""
    if pg is None or not dist.is_initialized():
        return local[0][0] if len(local) == 1 else torch.cat([t for t, _, _ in local], dim=len(size) - 1)
    # shard layouts are written in ranks of the SHARDING group (2D parallel: a sub-group of the job); ShardedTensor wants global ranks
    try:
        to_global = (lambda r: r) if pg is dist.group.WORLD else (lambda r: dist.get_global_rank(pg, r))
        to_global(0)
    except Exception:
        to_global = lambda r: r

    def dev_of(r: int) -> str:
        if r == rank and local:
            d = local[0][0].device
            return f"rank:{to_global(r)}/{d.type}" + (f":{d.index}" if d.index is not None else "")
        return placement(device_type, to_global(r), local_size)

    metas = [ShardMetadata(shard_offsets=list(o), shard_sizes=list(s), placement=dev_of(r)) for o, s, r in global_shards]
    local_shards = [Shard(tensor=t, metadata=ShardMetadata(shard_offsets=list(o), shard_sizes=list(s), placement=dev_of(rank))) for t, o, s in local]
    md = ShardedTensorMetadata(
        shards_metadata=metas, size=torch.Size(size),
        tensor_properties=TensorProperties(dtype=dtype, layout=torch.strided, requires_grad=False, memory_format=torch.contiguous_format, pin_memory=False),
    )
    return ShardedTensor._init_from_local_shards_and_global_metadata(local_shards, md, process_group=pg)


_MESH_CACHE: Dict[Any, Any] = {}


def _mesh_of(env: ShardingEnv, device_type: str):
    """1-D device mesh over the sharding group (created once per group; collective on first use)."""
    mesh = getattr(env, "device_mesh", None)
    if isinstance(mesh, (list, tuple)):  # 2D parallel: a [replicas][shards] rank matrix (DMPCollection._create_process_groups)
        key = (tuple(tuple(r) for r in mesh), device_type)
        if key not in _MESH_CACHE:
            from torch.distributed.device_mesh import DeviceMesh

            _MESH_CACHE[key] = DeviceMesh(device_type, torch.tensor(mesh, dtype=torch.int64), mesh_dim_names=("replicate", "shard"))
        return _MESH_CACHE[key]
    if mesh is not None:
        return mesh
    key = (id(env.process_group), device_type)
    if key not in _MESH_CACHE:
        from torch.distributed.device_mesh import init_device_mesh

        _MESH_CACHE[key] = init_device_mesh(device_type, (env.world_size,))
    return _MESH_CACHE[key]


def _dtensor_from_local(local: List[Tuple[torch.Tensor, List[int], List[int]]], size: List[int], sharding_type: str, env: ShardingEnv, device_type: str):
    """``env.output_dtensor`` layout of a sharded table / optimizer state: a ``DTensor`` whose local tensor is a ``LocalShardsWrapper``
    holding this rank's shards with their offsets (several for column-wise tables), placements by sharding type - whole tables
    ``Replicate()`` (one owner, every other rank holds no shard), row-sharded ``Shard(0)``, column-sharded and table-row-wise
    ``Shard(1)``; 2D parallelism prepends ``Replicate()`` over the replica dimension. No communication, no copies.
    Parity: reference embedding_kernel.py:350-520, sharding/{tw,rw,cw,twrw,grid}_sharding.py DTensorMetadata."""
    from torch.distributed.tensor import DTensor, Replicate
    from torch.distributed.tensor import Shard as DShard

    from .shards_wrapper import LocalShardsWrapper

    mesh = _mesh_of(env, device_type)
    if sharding_type in (ShardingType.TABLE_WISE.value, ShardingType.DATA_PARALLEL.value):
        inner = Replicate()
    elif sharding_type == ShardingType.ROW_WISE.value:
        inner = DShard(0)
    else:  # COLUMN_WISE, TABLE_COLUMN_WISE, TABLE_ROW_WISE, GRID_SHARD
        inner = DShard(1) if len(size) > 1 else DShard(0)
    placements = (Replicate(),) * (mesh.ndim - 1) + (inner,)
    wrapper = LocalShardsWrapper([t for t, _, _ in local], [tuple(o) for _, o, _ in local])
    stride = (size[1], 1) if len(size) == 2 else (1,)
    return DTensor.from_local(wrapper, mesh, placements, run_check=False, shape=torch.Size(size), stride=stride)


def _sharded_view(local, global_shards, size, dtype, sharding_type: str, env: ShardingEnv, pg, device_type: str, local_size: int):
    """State-dict value of a sharded tensor in the layout the environment asks for (DTensor or ShardedTensor)."""
    if getattr(env, "output_dtensor", False) and pg is not None and dist.is_initialized():
        return _dtensor_from_local(local, size, sharding_type, env, device_type)
    return _sharded_tensor_from_local(local, global_shards, size, dtype, pg, device_type, local_size, env.rank)


def _local_pieces_with_offsets(src) -> Optional[List[Tuple[torch.Tensor, List[int]]]]:
    """(tensor, offsets) of the rank-local shards of a ShardedTensor / DTensor(LocalShardsWrapper); None for plain tensors."""
    if isinstance(src, ShardedTensor):
        return [(sh.tensor, list(sh.metadata.shard_offsets)) for sh in src.local_shards()]
    try:
        from torch.distributed.tensor import DTensor
    except Exception:  # pragma: no cover
        return None
    if isinstance(src, DTensor):
        loc = src.to_local()
        if hasattr(loc, "shards_with_offsets"):
            return [(t, list(o)) for t, o in loc.shards_with_offsets()]
        return None
    return None


class EmbeddingFusedOptimizer(FusedOptimizer):
    """KeyedOptimizer view over the optimizer state living inside the table kernels. ``step`` is a
    no-op apart from pushing the learning rate (reference batched_embedding_kernel.py:1195-1624)."""

    def __init__(self, sharded_module: "ShardedEmbeddingBagCollection", prefix: str = "embedding_bags") -> None:
        self._module = sharded_module
        params: Dict[str, Any] = {}
        state: Dict[Any, Any] = {}
        groups: List[Dict[str, Any]] = []
        by_table = sharded_module._table_state_tensors()
        for table, (param, st) in by_table.items():
            key = f"{prefix}.{table}.weight"
            params[key] = param
            state[param] = {f"{table}.{name}": t for name, t in st.items()}
        lrs = {}
        for g in sharded_module._engine.groups if sharded_module._engine is not None else []:
            if g.tbe is None:
                continue
            ps = [params[f"{prefix}.{s.name}.weight"] for s in g.local_shards if f"{prefix}.{s.name}.weight" in params]
            uniq = list(OrderedDict((id(p), p) for p in ps).values())
            groups.append({"params": uniq, "lr": g.opt.lr, "_tbe": g.tbe})
        super().__init__(params, state, groups)

    def zero_grad(self, set_to_none: bool = False) -> None:
        pass

    def step(self, closure: Any = None) -> None:
        for group in self.param_groups:
            tbe = group.get("_tbe")
            if tbe is not None:
                tbe.set_learning_rate(group["lr"])

    def set_optimizer_step(self, step: int) -> None:
        for group in self.param_groups:
            tbe = group.get("_tbe")
            if tbe is not None:
                tbe.set_optimizer_step(step)

    def state_dict(self) -> Dict[str, Any]:
        sd = super().state_dict()
        return sd


# ---- contexts / awaitables -------------------------------------------------------------------------------------
class EmbeddingBagCollectionContext(Multistreamable):
    def __init__(self) -> None:
        self.batch_size_per_rank: Optional[List[int]] = None
        self.mean_divisor: Optional[torch.Tensor] = None
        self.dp_features: Optional[KeyedJaggedTensor] = None
        self.inverse_indices: Optional[Tuple[List[str], torch.Tensor]] = None
        self.sharding_contexts: List[Any] = []
        self.B_local: int = 0
        self.variable_batch_per_feature: bool = False
        self.vbe_full: bool = False  # VBE batch padded to the width of its inverse indices: it takes the NVLink plane
        self.vbe_index: Optional[V.VbeIndex] = None  # inverse indices + their CSR, read by the expansion and by its backward

    def record_stream(self, stream: torch.Stream) -> None:
        if self.mean_divisor is not None and self.mean_divisor.is_cuda:
            self.mean_divisor.record_stream(stream)
        if self.dp_features is not None:
            self.dp_features.record_stream(stream)
        if self.vbe_index is not None:
            self.vbe_index.record_stream(stream)


class _InputDistAwaitable(Awaitable[Awaitable[KJTList]]):
    def __init__(self, inner: Awaitable[Awaitable[KeyedJaggedTensor]]) -> None:
        super().__init__()
        self._inner = inner

    def _wait_impl(self) -> Awaitable[KJTList]:
        return _InputDistTensorsAwaitable(self._inner.wait())


class _InputDistTensorsAwaitable(Awaitable[KJTList]):
    def __init__(self, inner: Awaitable[KeyedJaggedTensor]) -> None:
        super().__init__()
        self._inner = inner

    def _wait_impl(self) -> KJTList:
        return KJTList([self._inner.wait()])


class EmbeddingBagCollectionAwaitable(LazyAwaitable[KeyedTensor]):
    def __init__(self, finish) -> None:
        super().__init__()
        self._finish = finish

    def _wait_impl(self) -> KeyedTensor:
        return self._finish()


class _TableParam(nn.Module):
    """Holder so that ``embedding_bags.<table>.weight`` exists in the module tree."""

    def __init__(self, weight: Optional[nn.Parameter]) -> None:
        super().__init__()
        if weight is not None:
            self.weight = weight


class _DenseLookup(nn.Module):
    """Data-parallel tables: replicated dense kernel; gradients flow to ``weights`` for DDP."""

    def __init__(self, tbe: TableBatchedEmbeddingBags) -> None:
        super().__init__()
        self.tbe = tbe

    def forward(self, indices: torch.Tensor, offsets: torch.Tensor, psw: Optional[torch.Tensor], batch_size: int) -> torch.Tensor:
        return self.tbe(indices, offsets, psw, batch_size=batch_size)


class ShardedEmbeddingBagCollection(
    ShardedEmbeddingModule[KJTList, List[torch.Tensor], KeyedTensor, EmbeddingBagCollectionContext],
    FusedOptimizerModule,
):
    """Sharded ``EmbeddingBagCollection``."""

    def __init__(
        self,
        module: EmbeddingBagCollectionInterface,
        table_name_to_parameter_sharding: Dict[str, ParameterSharding],
        env: ShardingEnv,
        fused_params: Optional[Dict[str, Any]] = None,
        device: Optional[torch.device] = None,
        qcomm_codecs_registry: Optional[Dict[str, QuantizedCommCodecs]] = None,
        module_fqn: Optional[str] = None,
    ) -> None:
        super().__init__(qcomm_codecs_registry=qcomm_codecs_registry)
        self._module_fqn = module_fqn
        self._env = env
        self._pg = env.process_group
        self._device = torch.device(device) if device is not None else torch.device("cpu")
        self._is_weighted = module.is_weighted()
        self._embedding_bag_configs: List[EmbeddingBagConfig] = module.embedding_bag_configs()
        self._plan = table_name_to_parameter_sharding
        self._fused_params = fused_params
        tables = self._embedding_bag_configs
        self._table_names = [t.name for t in tables]
        self._embedding_names: List[str] = [n for names in get_embedding_names_by_table(tables) for n in names]
        self._embedding_dims: List[int] = [t.embedding_dim for t in tables for _ in t.feature_names]
        self._feature_names: List[str] = [f for t in tables for f in t.feature_names]
        self._feature_table: List[int] = [ti for ti, t in enumerate(tables) for _ in t.feature_names]
        self._total_cols = sum(self._embedding_dims)
        self._out_base = [0]
        for d in self._embedding_dims:
            self._out_base.append(self._out_base[-1] + d)

        # optimizer specs from apply_optimizer_in_backward tags on the unsharded module's params
        opt_specs: Dict[str, OptimizerSpec] = {}
        self._fused_tables: Set[str] = set()
        src_params = dict(module.named_parameters()) if isinstance(module, nn.Module) else {}
        for t in tables:
            p = src_params.get(f"embedding_bags.{t.name}.weight")
            spec, tagged = optimizer_spec_from(p, fused_params)
            opt_specs[t.name] = spec
        if getattr(module, "_trb_opt_specs", None):  # re-sharding keeps the optimizers of the module being replaced
            opt_specs.update(module._trb_opt_specs)
        self._opt_specs = opt_specs
        codecs = None
        if qcomm_codecs_registry is not None:
            codecs = qcomm_codecs_registry.get(CommOp.POOLED_EMBEDDINGS_ALL_TO_ALL.name, None)
        output_dtype = torch.float32
        if fused_params and fused_params.get("output_dtype") is not None:
            od = fused_params["output_dtype"]
            output_dtype = od if isinstance(od, torch.dtype) else data_type_to_dtype(od)

        self._dp_tables = [ti for ti, t in enumerate(tables) if self._plan[t.name].sharding_type == ShardingType.DATA_PARALLEL.value]
        self._has_mp = len(self._dp_tables) < len(tables)
        self._engine: Optional[ShardedLookupEngine] = None
        if self._has_mp:
            self._engine = ShardedLookupEngine(
                tables=tables, feature_names=self._feature_names, feature_table=self._feature_table, plan=self._plan, env=env,
                device=self._device, pooled=True, is_weighted=self._is_weighted, opt_specs=opt_specs, output_dtype=output_dtype,
                qcomm_codecs=codecs,
            )
        # ---- data-parallel tables --------------------------------------------------------------------
        self._dp_lookup: Optional[nn.Module] = None
        self._dp_features: List[int] = [fi for fi, ti in enumerate(self._feature_table) if ti in self._dp_tables]
        self._dp_cols: List[int] = []
        if self._dp_tables:
            pool = {getattr(tables[ti], "pooling", PoolingType.SUM) for ti in self._dp_tables}
            # SUM and MEAN tables replicated in one collection: the kernel sums, the MEAN features are divided by their bag lengths
            # afterwards through the same per-(sample, feature) divisor the row-sharded MEAN tables use (``ctx.mean_divisor``)
            self._dp_post_mean_features = [fi for fi in self._dp_features if getattr(tables[self._feature_table[fi]], "pooling", PoolingType.SUM) == PoolingType.MEAN] \
                if len(pool) > 1 else []
            if len(pool) > 1:
                pool = {PoolingType.SUM}
            local_idx = {ti: i for i, ti in enumerate(self._dp_tables)}
            dp_tbe = TableBatchedEmbeddingBags(
                embedding_specs=[(tables[ti].num_embeddings, tables[ti].embedding_dim) for ti in self._dp_tables],
                feature_table_map=[local_idx[self._feature_table[fi]] for fi in self._dp_features],
                pooling_mode=PoolingMode.MEAN if pool.pop() == PoolingType.MEAN else PoolingMode.SUM,
                optimizer=OptimType.NONE, device=self._device, table_names=[tables[ti].name for ti in self._dp_tables],
            )
            self._dp_tbe = dp_tbe
            lookup = _DenseLookup(dp_tbe)
            if self._pg is not None and env.world_size > 1 and self._device.type != "meta":
                with torch.no_grad():
                    dist.broadcast(dp_tbe.weights.data, src=dist.get_global_rank(self._pg, 0) if hasattr(dist, "get_global_rank") else 0, group=self._pg)
                lookup = DistributedDataParallel(lookup, device_ids=[self._device] if self._device.type == "cuda" else None,
                                                 process_group=self._pg, gradient_as_bucket_view=True, broadcast_buffers=False)
            self._dp_lookup = lookup
            for fi in self._dp_features:
                self._dp_cols.extend(range(self._out_base[fi], self._out_base[fi + 1]))

        # ---- copy initial weights from a materialised unsharded module --------------------------------------
        self._init_from(module)
        # ---- parameter views embedding_bags.<table>.weight ------------------------------------------------------
        self.embedding_bags = nn.ModuleDict()
        self._build_param_views()
        # ---- mean pooling handled after the reduce (row-sharded MEAN tables) -----------------------------------
        self._post_mean_feature: List[bool] = list(self._engine._post_mean_feature) if self._engine is not None else [False] * len(self._feature_names)
        for fi in getattr(self, "_dp_post_mean_features", []):
            self._post_mean_feature[fi] = True
        self._post_mean = any(self._post_mean_feature)
        self._features_order: Optional[List[int]] = None
        self._has_features_permute = False
        self._optim: Optional[KeyedOptimizer] = None
        self._vbe_col_tables: Dict[Tuple, Any] = {}  # static column -> inverse-row tables of VBE batches (ops/vbe.py), per inverse-key order

    # ---- construction helpers -----------------------------------------------------------------------------
    @torch.no_grad()
    def _init_from(self, module: nn.Module) -> None:
        if self._device.type == "meta":
            return
        tables = {t.name: t for t in self._embedding_bag_configs}
        src = {}
        if hasattr(module, "embedding_bags"):
            for name, bag in module.embedding_bags.items():
                w = getattr(bag, "weight", None)
                if w is not None and w.device.type != "meta":
                    src[name] = w
        for shard, wview, _st, _tbe in (self._engine.local_shard_views() if self._engine is not None else []):
            cfg = tables[shard.name]
            if shard.name in src:
                wview.copy_(src[shard.name][shard.row_off : shard.row_off + shard.rows, shard.col_off : shard.col_off + shard.cols])
            else:
                if wview.numel() > 0:
                    if wview.dtype == torch.float32:
                        wview.uniform_(cfg.get_weight_init_min(), cfg.get_weight_init_max())
                    else:
                        init = torch.empty(wview.shape, dtype=torch.float32, device=wview.device).uniform_(cfg.get_weight_init_min(), cfg.get_weight_init_max())
                        wview.copy_(init)
        if self._dp_tables:
            for ti, w in zip(self._dp_tables, self._dp_tbe.split_embedding_weights()):
                cfg = self._embedding_bag_configs[ti]
                if cfg.name in src:
                    w.copy_(src[cfg.name])
                else:
                    w.uniform_(cfg.get_weight_init_min(), cfg.get_weight_init_max())
            if self._pg is not None and self._env.world_size > 1:
                dist.broadcast(self._dp_tbe.weights.data, src=dist.get_global_rank(self._pg, 0), group=self._pg)

    def prefetch(self, ctx, dist_input) -> None:
        """Stage the rows of an already-distributed batch into the HBM caches of UVM_CACHING tables (prefetch pipeline)."""
        if self._engine is not None and len(dist_input) > 0 and isinstance(dist_input[0], KeyedJaggedTensor):
            self._engine.prefetch(dist_input[0])  # (batches routed through the NVLink plane never hit cached tables: nothing to stage)

    def reset_rows(self, table: str, global_rows: torch.Tensor) -> int:
        """Re-initialise rows of a sharded table (managed-collision eviction / ITEP); see engine.reset_rows."""
        return self._engine.reset_rows(table, global_rows) if self._engine is not None else 0

    def _local_shards_by_table(self) -> Dict[str, List[Tuple[TableShard, torch.Tensor, Dict[str, torch.Tensor], TableBatchedEmbeddingBags]]]:
        res: Dict[str, List] = {}
        if self._engine is not None:
            for item in self._engine.local_shard_views():
                res.setdefault(item[0].name, []).append(item)
        return res

    def _build_param_views(self) -> None:
        by_table = self._local_shards_by_table()
        self._table_params: Dict[str, nn.Parameter] = {}
        for ti, cfg in enumerate(self._embedding_bag_configs):
            if ti in self._dp_tables:
                w = self._dp_tbe.split_embedding_weights()[self._dp_tables.index(ti)]
                p = nn.Parameter(w, requires_grad=False)
                self.embedding_bags[cfg.name] = _TableParam(p)
                self._table_params[cfg.name] = p
                continue
            shards = by_table.get(cfg.name, [])
            if not shards:
                self.embedding_bags[cfg.name] = _TableParam(None)
                continue
            # column shards on one rank are exposed side by side (reference concatenates CW shards)
            views = [w for _, w, _, _ in shards]
            w = views[0] if len(views) == 1 else views[0]
            p = nn.Parameter(w, requires_grad=False)
            p._in_backward_optimizers = [None]  # type: ignore[attr-defined]
            self.embedding_bags[cfg.name] = _TableParam(p)
            self._table_params[cfg.name] = p

    def _global_shards(self, name: str) -> List[Tuple[List[int], List[int], int]]:
        spec = self._plan[name].sharding_spec
        from .sharding_plan import placement_rank

        return [(list(s.shard_offsets), list(s.shard_sizes), placement_rank(s.placement)) for s in spec.shards]  # type: ignore[union-attr]

    def _table_state_tensors(self) -> Dict[str, Tuple[nn.Parameter, Dict[str, Any]]]:
        """table -> (param, {state name: ShardedTensor / tensor}) for the fused optimizer view."""
        from .comm import get_local_size

        res: Dict[str, Tuple[nn.Parameter, Dict[str, Any]]] = {}
        by_table = self._local_shards_by_table()
        local_size = get_local_size(self._env.world_size)
        for cfg in self._embedding_bag_configs:
            shards = by_table.get(cfg.name)
            if not shards or cfg.name not in self._table_params:
                continue
            gshards = self._global_shards(cfg.name)
            names = list(shards[0][2].keys())
            st: Dict[str, Any] = {}
            for n in names:
                first = shards[0][2][n]
                if first.dim() == 1:  # row-wise state: 1-D, sharded like the rows (one entry per row shard / column shard)
                    local = [(s_st[n], [s.row_off + self._cw_row_shift(cfg, s)], [s.rows]) for s, _, s_st, _ in shards]
                    g = [([o[0] + self._cw_row_shift_g(cfg, o, gshards)], [sz[0]], r) for o, sz, r in gshards]
                    size = [self._rowwise_state_size(cfg, gshards)]
                else:
                    local = [(s_st[n], [s.row_off, s.col_off], [s.rows, s.cols]) for s, _, s_st, _ in shards]
                    g = gshards
                    size = [cfg.num_embeddings, cfg.embedding_dim]
                st[n] = _sharded_view(local, g, size, torch.float32, self._plan[cfg.name].sharding_type, self._env, self._pg, self._device.type, local_size)
            res[cfg.name] = (self._table_params[cfg.name], st)
        return res

    # Row-wise optimizer state of column-sharded tables: every column shard keeps its own per-row
    # state; they are laid out one after another along dim 0 (reference
    # batched_embedding_kernel.py:1259-1329 does the same trick).
    def _cw_row_shift(self, cfg: BaseEmbeddingConfig, s: TableShard) -> int:
        gshards = self._global_shards(cfg.name)
        cols = sorted({o[1] for o, _, _ in gshards})
        return cols.index(s.col_off) * cfg.num_embeddings

    def _cw_row_shift_g(self, cfg, off, gshards) -> int:
        cols = sorted({o[1] for o, _, _ in gshards})
        return cols.index(off[1]) * cfg.num_embeddings

    def _rowwise_state_size(self, cfg, gshards) -> int:
        return len({o[1] for o, _, _ in gshards}) * cfg.num_embeddings

    # ---- ShardedModule contract -----------------------------------------------------------------------------
    def create_context(self) -> EmbeddingBagCollectionContext:
        return EmbeddingBagCollectionContext()

    def _setup_feature_order(self, features: KeyedJaggedTensor) -> None:
        keys = features.keys()
        pos = {k: i for i, k in enumerate(keys)}
        order = [pos[f] for f in self._feature_names]
        self._features_order = order
        self._has_features_permute = order != list(range(len(keys)))

    def _plane_serves(self, B: int) -> bool:
        """A uniform batch of ``B`` samples per feature takes the NVLink plane (fused input dist, lookup + output dist)."""
        eng = self._engine
        return eng is not None and not self._needs_dist_kjt and eng.fused_available(None) and eng._uniform_batch(B)

    def _pad_vbe(self, ctx: EmbeddingBagCollectionContext, features: KeyedJaggedTensor) -> KeyedJaggedTensor:
        """Variable batch per feature -> one stride by appending empty bags (values untouched). A device batch with inverse indices
        ``[R, B]`` whose features all have ``B_f <= B`` is padded to ``B`` when the NVLink plane serves that stride: ``B`` is the same
        every step, so the plane's buffers, its CUDA graphs and the uniform-batch check see one size (``ctx.vbe_full``). Any other
        batch - and any batch the plane does not serve, whose bags travel through the routed input dist and the collective output
        dist - is padded to ``max_f B_f`` only. The expansion index (CSR of the inverse indices, ids only) is built here, next to the
        routing work, and kept in the context for the backward."""
        inv = features.inverse_indices_or_none()
        spk = features.stride_per_key()
        stride = max(spk) if spk else 0
        ctx.vbe_full = (inv is not None and features.values().is_cuda and inv[1].is_cuda and stride <= inv[1].shape[1]
                        and self._plane_serves(inv[1].shape[1]))
        if ctx.vbe_full:
            stride = inv[1].shape[1]
        padded = V.pad_offsets(features, stride)
        if inv is not None:
            ctx.vbe_index = V.VbeIndex(inv, self._embedding_names, self._embedding_dims, src_rows=stride, tables=self._vbe_col_tables)
            if ctx.vbe_full and torch.is_grad_enabled():
                ctx.vbe_index.csr()
        return padded

    def _vbe_expand(self, ctx: EmbeddingBagCollectionContext, kt: KeyedTensor) -> KeyedTensor:
        """Undo the de-duplication of a VBE batch: out[b, cols(f)] = pooled[inverse_indices[f, b], cols(f)]."""
        index = ctx.vbe_index
        if index is None:
            return kt
        return KeyedTensor(keys=kt.keys(), length_per_key=kt.length_per_key(), values=V.vbe_expand(kt.values(), index), key_dim=1)

    def input_dist(self, ctx: EmbeddingBagCollectionContext, features: KeyedJaggedTensor) -> Awaitable[Awaitable[KJTList]]:
        if self._features_order is None:
            self._setup_feature_order(features)
        if features.variable_stride_per_key():
            # VBE: ship the de-duplicated bags (padded to one stride), expand with inverse_indices after the output dist
            ctx.inverse_indices = features.inverse_indices_or_none()
            ctx.variable_batch_per_feature = True
            features = self._pad_vbe(ctx, features)
        with torch.no_grad():
            eng = self._engine
            if ctx.vbe_full or (not ctx.variable_batch_per_feature and self._plane_serves(features.stride())):
                # NVLink plane: bucketize + feature permute + peer write in one device-side pass, straight from the batch's KJT
                # (any mix of sharding types); the only host work is picking the slot
                order = self._features_order
                B = features.stride()
                ctx.B_local = B
                if self._post_mean:
                    ctx.mean_divisor = self._mean_divisor(features.permute(order) if self._has_features_permute else features)
                if self._dp_tables:
                    ctx.dp_features = features.permute([order[fi] for fi in self._dp_features])
                return _InputDistAwaitable(NoWait(NoWait(eng.plane_input_dist(features, order, self._total_cols, training=self.training))))
            if not self._post_mean and eng is not None and not eng._row_sharded:
                # fast path: input order -> unit order in ONE key permutation (feature order, model-parallel subset and unit
                # replication composed on the host once) instead of three KJT permutes per step
                comp = self.__dict__.get("_composed_perm")
                if comp is None:
                    order = self._features_order
                    mp_unit = [order[eng.mp_features[p]] for p in eng._perm_features]
                    dp = [order[fi] for fi in self._dp_features]
                    comp = self.__dict__["_composed_perm"] = (mp_unit, dp, mp_unit == list(range(len(features.keys()))))
                mp_unit, dp, identity = comp
                ctx.B_local = features.stride()
                if self._dp_tables:
                    ctx.dp_features = features.permute(dp)
                return _InputDistAwaitable(eng.input_dist_routed(features if identity else features.permute(mp_unit)))
            if self._has_features_permute:
                features = features.permute(self._features_order)
            B = features.stride()
            ctx.B_local = B
            if self._post_mean:
                ctx.mean_divisor = self._mean_divisor(features)
            if self._dp_tables:
                ctx.dp_features = features.permute(self._dp_features) if len(self._dp_features) != len(self._feature_names) else features
            if self._engine is None:
                return NoWait(NoWait(KJTList([])))
            mp = features
            if len(self._engine.mp_features) != len(self._feature_names):
                mp = features.permute(self._engine.mp_features)
            aw, _ = self._engine.input_dist(mp)
            return _InputDistAwaitable(aw)

    # feature processors compute per-id weights ON the distributed KJT (and need their gradient): those modules ask for a real KJT
    _needs_dist_kjt: bool = False

    def _mean_divisor(self, features: KeyedJaggedTensor) -> torch.Tensor:
        """``[B, total_cols]`` factors 1 / bag length for the MEAN-pooled row-sharded features (divided after the reduce), 1 elsewhere;
        ``features`` in flat feature order."""
        B = features.stride()
        lengths = features.lengths().view(len(self._feature_names), B).t().float()  # [B, F]
        mask = self.__dict__.get("_post_mean_mask")
        if mask is None or mask.device != lengths.device:
            mask = self.__dict__["_post_mean_mask"] = torch.tensor(self._post_mean_feature, device=lengths.device)
            self.__dict__["_embedding_dims_t"] = torch.tensor(self._embedding_dims, device=lengths.device)
        div = torch.where(mask.unsqueeze(0), 1.0 / lengths.clamp(min=1.0), torch.ones_like(lengths))
        return torch.repeat_interleave(div, self.__dict__["_embedding_dims_t"], dim=1, output_size=self._total_cols)

    def compute(self, ctx: EmbeddingBagCollectionContext, dist_input: KJTList) -> List[torch.Tensor]:
        outs: List[torch.Tensor] = []
        if self._engine is not None:
            kjt = dist_input[0]
            if not isinstance(kjt, KeyedJaggedTensor):  # handle of the NVLink plane consumed through the 3-phase API: jagged view
                kjt = kjt.to_kjt()
            spr = kjt._stride_per_rank
            ctx.batch_size_per_rank = spr if spr is not None else None
            outs.append(self._engine.lookup(kjt))
        return outs

    def output_dist(self, ctx: EmbeddingBagCollectionContext, output: List[torch.Tensor]) -> LazyAwaitable[KeyedTensor]:
        mp_aw: Optional[Awaitable[torch.Tensor]] = None
        if self._engine is not None:
            mp_aw = self._engine.output_dist(output[0], ctx.batch_size_per_rank)
        dp_out: Optional[torch.Tensor] = None
        if self._dp_lookup is not None:
            f = ctx.dp_features
            psw = f.weights_or_none() if self._is_weighted else None
            dp_out = self._dp_lookup(f.values(), f.offsets(), psw, f.stride())

        def finish() -> KeyedTensor:
            mp = mp_aw.wait() if mp_aw is not None else None
            eng = self._engine if self._engine is not None else _COMBINE_ONLY
            vals = eng.combine(mp, dp_out, self._dp_cols, self._total_cols, ctx.mean_divisor)
            kt = KeyedTensor(keys=self._embedding_names, length_per_key=self._embedding_dims, values=vals, key_dim=1)
            return self._vbe_expand(ctx, kt) if ctx.variable_batch_per_feature else kt

        return EmbeddingBagCollectionAwaitable(finish)

    def compute_and_output_dist(self, ctx: EmbeddingBagCollectionContext, input: KJTList) -> LazyAwaitable[KeyedTensor]:
        eng = self._engine
        if eng is not None and len(input) > 0:
            kjt = input[0]
            spr = kjt._stride_per_rank
            if eng.fused_available(spr):
                return self._fused_compute_and_output_dist(ctx, kjt)
        return self.output_dist(ctx, self.compute(ctx, input))

    def _fused_compute_and_output_dist(self, ctx: EmbeddingBagCollectionContext, kjt: KeyedJaggedTensor) -> LazyAwaitable[KeyedTensor]:
        """Single-NVLink-domain fast path: lookup fused with the pooled output dist (see engine.py)."""
        from .comm_ops import get_gradient_division

        eng = self._engine
        W = self._env.world_size
        B_local = kjt.stride() // W
        scale = 1.0 / W if get_gradient_division() else 1.0
        dp = None
        if self._dp_lookup is not None:
            # replicated tables: looked up locally, pooled rows written straight into their columns of the output buffer inside
            # the fused op; their dense gradient is all-reduced inside its backward (no copies of the [B, sum(D)] tensor)
            if not hasattr(self, "_dp_meta_cols"):
                self._dp_meta_cols = self._dp_tbe.meta.with_cols([self._out_base[fi] for fi in self._dp_features], self._total_cols)
            dp = (self._dp_tbe, self._dp_meta_cols, ctx.dp_features, self._pg)
        vals = eng.fused_lookup_dist(kjt, B_local, self._total_cols, scale, dp)
        if ctx.mean_divisor is not None:
            vals = vals * ctx.mean_divisor.to(vals.dtype)
        kt = KeyedTensor(keys=self._embedding_names, length_per_key=self._embedding_dims, values=vals, key_dim=1)
        if ctx.variable_batch_per_feature:
            kt = self._vbe_expand(ctx, kt)
        return EmbeddingBagCollectionAwaitable(lambda: kt)

    # ---- parameters / state ------------------------------------------------------------------------------------
    def named_parameters(self, prefix: str = "", recurse: bool = True, remove_duplicate: bool = True) -> Iterator[Tuple[str, nn.Parameter]]:
        for name, p in self._table_params.items():
            if self._dp_tables and name in [self._embedding_bag_configs[ti].name for ti in self._dp_tables]:
                continue
            yield (prefix + "." if prefix else "") + f"embedding_bags.{name}.weight", p
        if self._dp_lookup is not None:
            yield (prefix + "." if prefix else "") + self._dp_param_name(), self._dp_tbe.weights

    def _dp_param_name(self) -> str:
        """Structural name of the flat data-parallel weight (what DDP sees)."""
        for n, p in nn.Module.named_parameters(self):
            if p is self._dp_tbe.weights:
                return n
        return "_dp_lookup.tbe.weights"

    def named_buffers(self, prefix: str = "", recurse: bool = True, remove_duplicate: bool = True) -> Iterator[Tuple[str, torch.Tensor]]:
        yield from ()

    def sharded_parameter_names(self, prefix: str = "") -> Iterator[str]:
        dp_names = {self._embedding_bag_configs[ti].name for ti in self._dp_tables}
        for name in self._table_params:
            if name not in dp_names:
                yield (prefix + "." if prefix else "") + f"embedding_bags.{name}.weight"
        if self._dp_lookup is not None:
            # replicated tables are all-reduced by their own DDP wrapper: hide them from the outer DDP
            yield (prefix + "." if prefix else "") + self._dp_param_name()
        # the engine's storage (autograd anchor parameters) is rank-private: keep it out of DDP
        for n, _ in nn.Module.named_parameters(self):
            if n.startswith("_engine."):
                yield (prefix + "." if prefix else "") + n

    def state_dict(self, destination: Optional[Dict[str, Any]] = None, prefix: str = "", keep_vars: bool = False) -> Dict[str, Any]:
        from .comm import get_local_size

        if destination is None:
            destination = OrderedDict()
        local_size = get_local_size(self._env.world_size)
        by_table = self._local_shards_by_table()
        for ti, cfg in enumerate(self._embedding_bag_configs):
            key = f"{prefix}embedding_bags.{cfg.name}.weight"
            if ti in self._dp_tables:
                w = self._dp_tbe.split_embedding_weights()[self._dp_tables.index(ti)]
                destination[key] = w if keep_vars else w.detach()
                continue
            shards = by_table.get(cfg.name, [])
            dtype = torch.float32 if cfg.data_type == DataType.FP32 else data_type_to_dtype(cfg.data_type)
            local = [(w, [s.row_off, s.col_off], [s.rows, s.cols]) for s, w, _, _ in shards]
            if self._pg is None or not dist.is_initialized():
                destination[key] = self._assemble_local(cfg, local)
            else:
                destination[key] = _sharded_view(local, self._global_shards(cfg.name), [cfg.num_embeddings, cfg.embedding_dim], dtype,
                                                 self._plan[cfg.name].sharding_type, self._env, self._pg, self._device.type, local_size)
        return destination

    def _assemble_local(self, cfg, local) -> torch.Tensor:
        if len(local) == 1 and list(local[0][0].shape) == [cfg.num_embeddings, cfg.embedding_dim]:
            return local[0][0]
        full = torch.zeros(cfg.num_embeddings, cfg.embedding_dim, dtype=local[0][0].dtype, device=local[0][0].device)
        for t, o, s in local:
            full[o[0] : o[0] + s[0], o[1] : o[1] + s[1]] = t
        return full

    @torch.no_grad()
    def load_state_dict(self, state_dict: Mapping[str, Any], strict: bool = True, assign: bool = False):
        """Accepts ShardedTensors (same layout), or full unsharded tensors (sliced by shard offsets)."""
        missing, unexpected = [], []
        by_table = self._local_shards_by_table()
        expected = set()
        for ti, cfg in enumerate(self._embedding_bag_configs):
            key = f"embedding_bags.{cfg.name}.weight"
            expected.add(key)
            if key not in state_dict:
                missing.append(key)
                continue
            src = state_dict[key]
            if ti in self._dp_tables:
                dst = self._dp_tbe.split_embedding_weights()[self._dp_tables.index(ti)]
                dst.copy_(src.local_tensor() if isinstance(src, ShardedTensor) else src)
                continue
            pieces = _local_pieces_with_offsets(src)
            for s, w, _, _ in by_table.get(cfg.name, []):
                if pieces is not None:  # ShardedTensor / DTensor over local shards: match shards by their offsets
                    hit = [t for t, off in pieces if off == [s.row_off, s.col_off]]
                    if not hit:
                        raise RuntimeError(f"{key}: no local shard at offsets {[s.row_off, s.col_off]} in the loaded {type(src).__name__}")
                    w.copy_(hit[0])
                else:  # full unsharded tensor (or a plain DTensor's local tensor): slice this shard's window
                    full = src.full_tensor() if hasattr(src, "full_tensor") and not isinstance(src, ShardedTensor) else src
                    w.copy_(full[s.row_off : s.row_off + s.rows, s.col_off : s.col_off + s.cols])
        for k in state_dict.keys():
            if k not in expected:
                unexpected.append(k)
        if strict and (missing or unexpected):
            raise RuntimeError(f"Error(s) in loading state_dict: missing {missing}, unexpected {unexpected}")
        return torch.nn.modules.module._IncompatibleKeys(missing, unexpected)

    def _load_from_state_dict(self, state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys, error_msgs):
        sub = {k[len(prefix):]: v for k, v in state_dict.items() if k.startswith(prefix)}
        res = self.load_state_dict(sub, strict=False)
        missing_keys.extend(prefix + k for k in res.missing_keys)

    @property
    def fused_optimizer(self) -> KeyedOptimizer:
        if self._optim is None:
            self._optim = EmbeddingFusedOptimizer(self) if self._engine is not None else CombinedOptimizer([])
        return self._optim

    def embedding_bag_configs(self) -> List[EmbeddingBagConfig]:
        return self._embedding_bag_configs

    def is_weighted(self) -> bool:
        return self._is_weighted

    @property
    def unsharded_module_type(self) -> Type[EmbeddingBagCollection]:
        return EmbeddingBagCollection

    @property
    def engine(self) -> Optional[ShardedLookupEngine]:
        return self._engine


class _CombineOnly:
    """Stand-in used when a collection has only data-parallel tables."""

    def combine(self, mp, dp, dp_cols, total_cols, div):
        if dp_cols == list(range(total_cols)):
            return dp if div is None else dp * div
        inv = [0] * total_cols
        for src, dst in enumerate(dp_cols):
            inv[dst] = src
        out = dp.index_select(1, torch.tensor(inv, device=dp.device))
        return out if div is None else out * div


_COMBINE_ONLY = _CombineOnly()


class EmbeddingBagCollectionSharder(BaseEmbeddingSharder[EmbeddingBagCollection]):
    """Shards an ``EmbeddingBagCollection`` (reference embeddingbag.py:2207)."""

    def shard(self, module: EmbeddingBagCollection, params: Dict[str, ParameterSharding], env: ShardingEnv,
              device: Optional[torch.device] = None, module_fqn: Optional[str] = None) -> ShardedEmbeddingBagCollection:
        return ShardedEmbeddingBagCollection(module=module, table_name_to_parameter_sharding=params, env=env, fused_params=self.fused_params,
                                             device=device, qcomm_codecs_registry=self.qcomm_codecs_registry, module_fqn=module_fqn)

    def shardable_parameters(self, module: EmbeddingBagCollection) -> Dict[str, nn.Parameter]:
        return {name.split(".")[0]: param for name, param in module.embedding_bags.named_parameters()}

    @property
    def module_type(self) -> Type[EmbeddingBagCollection]:
        return EmbeddingBagCollection


# ---- nn.EmbeddingBag ------------------------------------------------------------------------------------------------
class _BagAsCollection(nn.Module):
    """Present one ``nn.EmbeddingBag`` as a single-table collection (table ``weight``-> feature ``dummy_feature``)."""

    def __init__(self, bag: nn.EmbeddingBag, table_name: str) -> None:
        super().__init__()
        pooling = {"sum": PoolingType.SUM, "mean": PoolingType.MEAN}.get(bag.mode)
        if pooling is None:
            raise ValueError(f"nn.EmbeddingBag mode '{bag.mode}' cannot be sharded (sum / mean only)")
        self._cfg = EmbeddingBagConfig(name=table_name, embedding_dim=bag.embedding_dim, num_embeddings=bag.num_embeddings, feature_names=["dummy_feature"], pooling=pooling)
        self.embedding_bags = nn.ModuleDict({table_name: bag})

    def embedding_bag_configs(self) -> List[EmbeddingBagConfig]:
        return [self._cfg]

    def is_weighted(self) -> bool:
        return True


class _BagAwaitable(LazyAwaitable[torch.Tensor]):
    def __init__(self, inner: LazyAwaitable[KeyedTensor]) -> None:
        super().__init__()
        self._inner = inner

    def _wait_impl(self) -> torch.Tensor:
        return self._inner.wait().values()


class ShardedEmbeddingBag(ShardedModule, FusedOptimizerModule):
    """Sharded ``nn.EmbeddingBag``: ``forward(input, offsets=None, per_sample_weights=None) -> Tensor [B, D]``
    (reference embeddingbag.py:2286-2507)."""

    def __init__(self, module: nn.EmbeddingBag, table_name_to_parameter_sharding: Dict[str, ParameterSharding], env: ShardingEnv,
                 fused_params: Optional[Dict[str, Any]] = None, device: Optional[torch.device] = None) -> None:
        super().__init__()
        assert len(table_name_to_parameter_sharding) == 1, "expect one and only one table (weight) in an nn.EmbeddingBag plan"
        self._table_name = next(iter(table_name_to_parameter_sharding))  # "weight"
        adapter = _BagAsCollection(module, self._table_name)
        w = module.weight
        # optimizer tags live on the bag's parameter; expose them under the collection's parameter name
        self._ebc = ShardedEmbeddingBagCollection(adapter, table_name_to_parameter_sharding, env, fused_params, device)
        self._device = self._ebc._device

    def create_context(self) -> EmbeddingBagCollectionContext:
        return self._ebc.create_context()

    def _to_kjt(self, input: torch.Tensor, offsets: Optional[torch.Tensor], per_sample_weights: Optional[torch.Tensor]) -> KeyedJaggedTensor:
        if input.dim() == 2:
            B, L = input.shape
            offsets = torch.arange(0, B * L + 1, L, device=input.device)
            input = input.reshape(-1)
            if per_sample_weights is not None:
                per_sample_weights = per_sample_weights.reshape(-1)
        else:
            assert offsets is not None, "1-D input needs offsets"
            if offsets.numel() == 0 or int(offsets[-1]) != input.numel():  # nn.EmbeddingBag default: no trailing offset
                offsets = torch.cat([offsets, offsets.new_tensor([input.numel()])])
        w = per_sample_weights if per_sample_weights is not None else torch.ones(input.numel(), device=input.device)
        return KeyedJaggedTensor(keys=["dummy_feature"], values=input, offsets=offsets, weights=w)

    def input_dist(self, ctx, input: torch.Tensor, offsets: Optional[torch.Tensor] = None, per_sample_weights: Optional[torch.Tensor] = None):
        return self._ebc.input_dist(ctx, self._to_kjt(input, offsets, per_sample_weights))

    def compute(self, ctx, dist_input):
        return self._ebc.compute(ctx, dist_input)

    def output_dist(self, ctx, output) -> LazyAwaitable[torch.Tensor]:
        return _BagAwaitable(self._ebc.output_dist(ctx, output))

    def compute_and_output_dist(self, ctx, input) -> LazyAwaitable[torch.Tensor]:
        return _BagAwaitable(self._ebc.compute_and_output_dist(ctx, input))

    def named_parameters(self, prefix: str = "", recurse: bool = True, remove_duplicate: bool = True):
        for n, p in self._ebc.named_parameters("", recurse):
            yield (prefix + "." if prefix else "") + "weight", p

    def sharded_parameter_names(self, prefix: str = "") -> Iterator[str]:
        yield from self._ebc.sharded_parameter_names((prefix + "." if prefix else "") + "_ebc")

    def state_dict(self, destination=None, prefix: str = "", keep_vars: bool = False):
        inner = self._ebc.state_dict(None, "", keep_vars)
        destination = OrderedDict() if destination is None else destination
        destination[prefix + "weight"] = inner[f"embedding_bags.{self._table_name}.weight"]
        return destination

    def load_state_dict(self, state_dict, strict: bool = True, assign: bool = False):
        return self._ebc.load_state_dict({f"embedding_bags.{self._table_name}.weight": state_dict["weight"]}, strict)

    @property
    def fused_optimizer(self) -> KeyedOptimizer:
        return self._ebc.fused_optimizer

    @property
    def engine(self):
        return self._ebc.engine


class EmbeddingBagSharder(BaseEmbeddingSharder[nn.EmbeddingBag]):
    """Shards a bare ``nn.EmbeddingBag`` (reference embeddingbag.py:2510)."""

    def shard(self, module: nn.EmbeddingBag, params: Dict[str, ParameterSharding], env: ShardingEnv, device: Optional[torch.device] = None,
              module_fqn: Optional[str] = None) -> ShardedEmbeddingBag:
        return ShardedEmbeddingBag(module, params, env, self.fused_params, device)

    def shardable_parameters(self, module: nn.EmbeddingBag) -> Dict[str, nn.Parameter]:
        return {name: param for name, param in module.named_parameters()}

    @property
    def module_type(self) -> Type[nn.EmbeddingBag]:
        return nn.EmbeddingBag
