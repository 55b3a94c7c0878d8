"""The composable sharding framework: ``EmbeddingSharding`` = input dist + lookup + output dist for the tables of ONE sharding type.

Reference: ``torchrec/distributed/embedding_sharding.py`` - ``bucketize_kjt_before_all2all`` :268-353, ``bucketize_kjt_inference`` :356-437,
``group_tables`` :552-683, ``KJTListAwaitable`` :690-725, ``KJTListSplitsAwaitable`` :844-891, ``FusedKJTListSplitsAwaitable`` :907-1052,
``ListOfKJTList*`` :1055-1112, ``EmbeddingShardingContext`` :1115, ``BaseSparseFeaturesDist`` / ``BaseEmbeddingDist`` :1125-1167,
``EmbeddingSharding`` :1170-1248, ``EmbeddingShardingInfo`` :1251.

How this relates to ``parallel/engine.py``: the sharded modules of this framework do not instantiate one ``EmbeddingSharding`` per type - the engine cuts
every table into rectangles and runs one route / lookup / combine for all types (DESIGN.md section 2). The classes below and ``parallel/sharding/*`` are
the same stages in the reference's decomposed form, built from the portable collectives of ``dist_data.py``; they are what a custom sharded module,
the inference path and the tests of individual stages use. Both forms share the kernels (``ops/tbe.py``) and the collectives.
"""
from __future__ import annotations

import abc
import copy
from dataclasses import dataclass, field
from typing import Any, Dict, Generic, List, Optional, Tuple, TypeVar, Union

import torch
import torch.distributed as dist
from torch import nn
from torch.autograd.profiler import record_function

from ..modules.embedding_configs import DataType, PoolingType
from ..ops import jagged as J
from ..sparse.jagged_tensor import KeyedJaggedTensor
from ..streamable import Multistreamable
from .dist_data import KJTAllToAllTensorsAwaitable, SplitsAllToAllAwaitable
from .embedding_dim_bucketer import EmbDimBucketer, EmbDimBucketerPolicy, should_do_dim_bucketing
from .embedding_types import (
    BaseEmbeddingLookup,
    EmbeddingComputeKernel,
    FeatureShardingMixIn,
    GroupedEmbeddingConfig,
    KJTList,
    ShardedEmbeddingTable,
)
from .types import Awaitable, EmbeddingEvent, NoWait, ParameterSharding, QuantizedCommCodecs, ShardingEnv, ShardMetadata

C = TypeVar("C", bound=Multistreamable)
F = TypeVar("F", bound=Multistreamable)
T = TypeVar("T")
W = TypeVar("W")

CACHE_LOAD_FACTOR_STR = "cache_load_factor"
USE_ONE_TBE_PER_TABLE = "use_one_tbe_per_table"


# ---- bucketization ---------------------------------------------------------------------------------------------------
def bucketize_kjt_before_all2all(
    kjt: KeyedJaggedTensor,
    num_buckets: int,
    block_sizes: torch.Tensor,
    total_num_blocks: Optional[torch.Tensor] = None,
    output_permute: bool = False,
    bucketize_pos: bool = False,
    block_bucketize_row_pos: Optional[List[torch.Tensor]] = None,
    keep_original_indices: bool = False,
) -> Tuple[KeyedJaggedTensor, Optional[torch.Tensor]]:
    """Row-wise routing: id -> (bucket = owner rank, local id). The result has ``num_buckets * F`` keys (bucket major) so a plain KJT all-to-all
    with ``splits=[F] * num_buckets`` delivers bucket ``r`` to rank ``r``. With ``output_permute`` the permutation that restores the original value
    order is returned (sequence embeddings need it after the output all-to-all). ``bucketize_pos`` replaces the weights with each id's position in
    its bag (position-weighted feature processors). ``block_bucketize_row_pos`` gives per-feature uneven shard boundaries."""
    num_features = len(kjt.keys())
    assert block_sizes.numel() == num_features, f"block_sizes has {block_sizes.numel()} entries for {num_features} features"
    block_sizes = block_sizes.to(kjt.values().device)
    bspf = None
    max_B = -1
    if kjt.variable_stride_per_key():
        bspf = torch.tensor([sum(s) for s in kjt.stride_per_key_per_rank()], dtype=torch.int64, device=kjt.values().device)
        max_B = int(max(sum(s) for s in kjt.stride_per_key_per_rank()))
    with record_function("## bucketize_kjt_before_all2all ##"):
        lengths, ids, weights, pos, unbucketize = J.block_bucketize_sparse_features(
            kjt.lengths().view(-1), kjt.values(), bucketize_pos=bucketize_pos, sequence=output_permute, block_sizes=block_sizes, my_size=num_buckets,
            weights=kjt.weights_or_none(), batch_size_per_feature=bspf, max_B=max_B, block_bucketize_pos=block_bucketize_row_pos,
            keep_orig_idx=keep_original_indices, total_num_blocks=total_num_blocks,
        )
    out_weights = pos if bucketize_pos else weights
    if kjt.variable_stride_per_key():
        spkpr = [list(s) for _ in range(num_buckets) for s in kjt.stride_per_key_per_rank()]
        out = KeyedJaggedTensor(keys=list(kjt.keys()) * num_buckets, values=ids, weights=out_weights, lengths=lengths.view(-1), stride_per_key_per_rank=spkpr)
    else:
        out = KeyedJaggedTensor(keys=list(kjt.keys()) * num_buckets, values=ids, weights=out_weights, lengths=lengths.view(-1), stride=kjt.stride())
    return out, unbucketize


def bucketize_kjt_inference(
    kjt: KeyedJaggedTensor,
    num_buckets: int,
    block_sizes: torch.Tensor,
    total_num_buckets: Optional[torch.Tensor] = None,
    bucketize_pos: bool = False,
    block_bucketize_row_pos: Optional[List[torch.Tensor]] = None,
    is_sequence: bool = False,
    keep_original_indices: bool = False,
) -> Tuple[KeyedJaggedTensor, Optional[torch.Tensor], Optional[torch.Tensor]]:
    """Inference flavour: also returns the bucket of every id (``bucket_mapping``) for sequence outputs that are gathered back per device
    (reference :356-437)."""
    out, unbucketize = bucketize_kjt_before_all2all(kjt, num_buckets, block_sizes, total_num_buckets, output_permute=is_sequence, bucketize_pos=bucketize_pos,
                                                    block_bucketize_row_pos=block_bucketize_row_pos, keep_original_indices=keep_original_indices)
    bucket_mapping = None
    if is_sequence:
        per_bucket = out.lengths().view(num_buckets, -1).sum(1)
        sorted_bucket = torch.repeat_interleave(torch.arange(num_buckets, device=per_bucket.device), per_bucket)
        bucket_mapping = sorted_bucket[unbucketize.long()] if unbucketize is not None and unbucketize.numel() else sorted_bucket
    return out, unbucketize, bucket_mapping


def bucketize_embeddings_before_all2all_write(kjt: KeyedJaggedTensor, embeddings: torch.Tensor, num_buckets: int, block_sizes: torch.Tensor,
                                             block_bucketize_row_pos: Optional[List[torch.Tensor]] = None) -> Tuple[KeyedJaggedTensor, torch.Tensor]:
    """Route (id, new row) pairs of an embedding UPDATE to the row owners: ids are bucketized like a lookup, the rows follow the same permutation
    (reference :773-841)."""
    out, unbucketize = bucketize_kjt_before_all2all(kjt, num_buckets, block_sizes, output_permute=True, block_bucketize_row_pos=block_bucketize_row_pos)
    assert unbucketize is not None
    order = torch.empty_like(unbucketize)
    order[unbucketize.long()] = torch.arange(unbucketize.numel(), device=unbucketize.device, dtype=unbucketize.dtype)
    return out, embeddings.view(kjt.values().numel(), -1)[order.long()]


# ---- table grouping --------------------------------------------------------------------------------------------------
def _get_weighted_avg_cache_load_factor(embedding_tables: List[ShardedEmbeddingTable]) -> Optional[float]:
    """Row-weighted mean of the tables' cache load factors: ONE cache serves the whole group (reference :440-465)."""
    num = den = 0.0
    for t in embedding_tables:
        clf = (t.fused_params or {}).get(CACHE_LOAD_FACTOR_STR)
        if clf is not None:
            num += float(clf) * t.num_embeddings
            den += t.num_embeddings
    return None if den == 0 else num / den


def _get_grouping_fused_params(fused_params: Optional[Dict[str, Any]], name: str) -> Optional[Dict[str, Any]]:
    """fused_params without the keys that must not split groups (cache load factor is averaged; one-TBE-per-table becomes the table's name)."""
    if fused_params is None:
        return None
    fp = dict(fused_params)
    fp.pop(CACHE_LOAD_FACTOR_STR, None)
    if fp.get(USE_ONE_TBE_PER_TABLE):
        fp[USE_ONE_TBE_PER_TABLE] = name
    return fp


def _get_compute_kernel_type(compute_kernel: EmbeddingComputeKernel) -> EmbeddingComputeKernel:
    """All HBM/host fused flavours and all quant flavours can share a TBE (reference :496-513)."""
    if compute_kernel in (EmbeddingComputeKernel.FUSED, EmbeddingComputeKernel.FUSED_UVM, EmbeddingComputeKernel.FUSED_UVM_CACHING):
        return EmbeddingComputeKernel.FUSED
    if compute_kernel in (EmbeddingComputeKernel.QUANT, EmbeddingComputeKernel.QUANT_UVM, EmbeddingComputeKernel.QUANT_UVM_CACHING):
        return EmbeddingComputeKernel.QUANT
    return compute_kernel


def _prefetch_and_cached(table: ShardedEmbeddingTable) -> bool:
    """Cached tables that take part in the prefetch pipeline get their own groups per dim bucket (reference :516-539)."""
    if table.compute_kernel not in (EmbeddingComputeKernel.FUSED_UVM_CACHING, EmbeddingComputeKernel.QUANT_UVM_CACHING, EmbeddingComputeKernel.KEY_VALUE):
        return False
    return bool((table.fused_params or {}).get("prefetch_pipeline", False))


def _all_tables_are_quant_kernel(tables: List[ShardedEmbeddingTable]) -> bool:
    return all(t.compute_kernel == EmbeddingComputeKernel.QUANT for t in tables)


def group_tables(tables_per_rank: List[List[ShardedEmbeddingTable]]) -> List[List[GroupedEmbeddingConfig]]:
    """Per rank: partition the local shards into groups that can share ONE kernel launch.

    Tables share a group when they agree on (fused_params minus per-table keys, compute-kernel family, data type, pooling, weighted-ness,
    feature-processor, [dim bucket for cached prefetch tables], virtual-table-ness). Parity: reference :552-683. The single-launch TBE here handles
    mixed dims, so - like FBGEMM - dims only split groups for cached tables (cache rows are sized per group)."""

    def group_one_rank(tables: List[ShardedEmbeddingTable]) -> List[GroupedEmbeddingConfig]:
        groups: Dict[Tuple, List[ShardedEmbeddingTable]] = {}
        order: List[Tuple] = []
        cached_tables = [t for t in tables if _prefetch_and_cached(t)]
        bucketer = EmbDimBucketer(cached_tables, EmbDimBucketerPolicy.CACHELINE_BUCKETS if should_do_dim_bucketing(cached_tables) else EmbDimBucketerPolicy.SINGLE_BUCKET) if cached_tables else None
        is_inference = _all_tables_are_quant_kernel(tables)
        for t in tables:
            fp = _get_grouping_fused_params(t.fused_params, t.name)
            fp_key = tuple(sorted((k, str(v)) for k, v in (fp or {}).items()))
            dim_bucket = bucketer.get_bucket(t.local_cols, t.data_type) if (bucketer is not None and _prefetch_and_cached(t)) else -1
            key = (
                fp_key,
                _get_compute_kernel_type(t.compute_kernel).value,
                # inference TBEs hold mixed row formats in one buffer; training groups are per dtype
                None if is_inference else t.data_type,
                t.pooling, t.is_weighted, t.has_feature_processor, dim_bucket,
                bool(getattr(t, "use_virtual_table", False)), bool(getattr(t, "enable_embedding_update", False)),
            )
            if key not in groups:
                groups[key] = []
                order.append(key)
            groups[key].append(t)
        out: List[GroupedEmbeddingConfig] = []
        for key in order:
            ts = groups[key]
            fp = _get_grouping_fused_params(ts[0].fused_params, ts[0].name)
            clf = _get_weighted_avg_cache_load_factor(ts)
            if clf is not None:
                fp = dict(fp or {})
                fp[CACHE_LOAD_FACTOR_STR] = clf
            kernels = {t.compute_kernel for t in ts}
            # a group that mixes HBM and cached tables is promoted to the cached kernel (rows that fit stay resident anyway)
            kernel = ts[0].compute_kernel
            for cand in (EmbeddingComputeKernel.FUSED_UVM_CACHING, EmbeddingComputeKernel.FUSED_UVM, EmbeddingComputeKernel.QUANT_UVM_CACHING, EmbeddingComputeKernel.QUANT_UVM):
                if cand in kernels:
                    kernel = cand
                    break
            out.append(GroupedEmbeddingConfig(data_type=ts[0].data_type, pooling=ts[0].pooling, is_weighted=ts[0].is_weighted,
                                              has_feature_processor=ts[0].has_feature_processor, compute_kernel=kernel, embedding_tables=ts, fused_params=fp))
        return out

    return [group_one_rank(tables) for tables in tables_per_rank]


# ---- awaitables of the two-stage input dist ----------------------------------------------------------------------------
class KJTListAwaitable(Awaitable[KJTList]):
    """Second stage of several KJT all-to-alls: ``wait()`` returns the received KJTs as a ``KJTList`` and fills the sharding contexts."""

    def __init__(self, awaitables: List[Awaitable[KeyedJaggedTensor]], ctx: C) -> None:
        super().__init__()
        self.awaitables = awaitables
        self.ctx = ctx

    def _wait_impl(self) -> KJTList:
        kjts = [w.wait() for w in self.awaitables]
        _set_sharding_context_post_a2a(kjts, self.ctx)
        return KJTList(kjts)


def _set_sharding_context_post_a2a(kjts: List[KeyedJaggedTensor], ctx: C) -> None:
    """Per-rank batch sizes seen AFTER the all-to-all: the output dists split by them (variable batch per rank / per feature)."""
    for kjt, sctx in zip(kjts, getattr(ctx, "sharding_contexts", [])):
        if hasattr(sctx, "batch_size_per_rank_per_feature") and kjt.variable_stride_per_key() and kjt.stride_per_key_per_rank():
            spkpr = kjt.stride_per_key_per_rank()
            sctx.batch_size_per_rank_per_feature = [[spkpr[f][r] for f in range(len(spkpr))] for r in range(len(spkpr[0]))]
        if hasattr(sctx, "lengths_after_input_dist"):
            sctx.lengths_after_input_dist = kjt.lengths()


def _set_sharding_context_intra_a2a(tensors_awaitables: List[Awaitable[KeyedJaggedTensor]], ctx: C) -> None:
    """Between the stages: per-rank strides and split sizes learnt from the size exchange."""
    for aw, sctx in zip(tensors_awaitables, getattr(ctx, "sharding_contexts", [])):
        if isinstance(aw, KJTAllToAllTensorsAwaitable):
            vi = aw._input.dist_labels().index("values")
            # the sequence output all-to-all runs the input dist backwards: it SENDS what was received and RECEIVES what was sent
            if hasattr(sctx, "input_splits"):
                sctx.input_splits = list(aw._output_splits[vi])
            if hasattr(sctx, "output_splits"):
                sctx.output_splits = list(aw._input_splits[vi])
            if hasattr(sctx, "sparse_features_recat"):
                sctx.sparse_features_recat = aw._recat
            if hasattr(sctx, "batch_size_per_rank") and aw._stride_per_rank is not None:
                sctx.batch_size_per_rank = list(aw._stride_per_rank)


def _split(flat_list: List[T], splits: List[int]) -> List[List[T]]:
    out, o = [], 0
    for s in splits:
        out.append(flat_list[o : o + s])
        o += s
    return out


class KJTListSplitsAwaitable(Awaitable[Awaitable[KJTList]], Generic[C]):
    """First stage of the input dists of one module (one per sharding type): ``wait()`` finishes every size exchange and launches the tensor
    all-to-alls (reference :844-891)."""

    def __init__(self, awaitables: List[Awaitable[Awaitable[KeyedJaggedTensor]]], ctx: C, module_fqn: Optional[str] = None,
                 sharding_types: Optional[List[str]] = None) -> None:
        super().__init__()
        self.awaitables = awaitables
        self.ctx = ctx
        self._module_fqn = module_fqn
        self._sharding_types = sharding_types

    def _wait_impl(self) -> KJTListAwaitable:
        tensors_awaitables = [w.wait() for w in self.awaitables]
        _set_sharding_context_intra_a2a(tensors_awaitables, self.ctx)
        return KJTListAwaitable(tensors_awaitables, self.ctx)


@dataclass
class KJTSplitsAllToAllMeta:
    """What one KJT all-to-all would have exchanged on its own - input of the fused size exchange."""

    pg: dist.ProcessGroup
    _input: KeyedJaggedTensor
    splits: List[int]
    splits_tensors: List[torch.Tensor]
    input_splits: List[List[int]]
    input_tensors: List[torch.Tensor]
    labels: List[str]
    keys: List[str]
    device: torch.device
    stagger: int
    splits_cumsum: List[int] = field(default_factory=list)


class FusedKJTListSplitsAwaitable(Awaitable[List[KJTListAwaitable]]):
    """ONE size all-to-all for the input dists of ALL pipelined modules (reference :907-1052): the small int exchange is latency bound
    (a launch + a host sync each), so N modules x S shardings exchanges collapse into one."""

    def __init__(self, requests: List[KJTListSplitsAwaitable[C]], contexts: List[C], pg: Optional[dist.ProcessGroup]) -> None:
        super().__init__()
        self._contexts = contexts
        self._awaitables: List[Union[KJTSplitsAllToAllMeta, Awaitable[Awaitable[KeyedJaggedTensor]]]] = [a for r in requests for a in r.awaitables]
        self._lengths = [len(r.awaitables) for r in requests]
        self._output_lengths = [len(a.splits_tensors) for a in self._awaitables if isinstance(a, KJTSplitsAllToAllMeta)]
        self._splits_awaitable: Optional[SplitsAllToAllAwaitable] = None
        rows = [t for a in self._awaitables if isinstance(a, KJTSplitsAllToAllMeta) for t in a.splits_tensors]
        if rows and pg is not None:
            self._splits_awaitable = SplitsAllToAllAwaitable(rows, pg)

    def _wait_impl(self) -> List[KJTListAwaitable]:
        splits_per_awaitable: List[List[List[int]]] = []
        if self._splits_awaitable is not None:
            splits_per_awaitable = _split(self._splits_awaitable.wait(), self._output_lengths)
        tensors_awaitables: List[Awaitable[KeyedJaggedTensor]] = []
        it = iter(splits_per_awaitable)
        for a in self._awaitables:
            if not isinstance(a, KJTSplitsAllToAllMeta):
                tensors_awaitables.append(a.wait())
                continue
            output_splits = next(it)
            stride_per_rank = None
            if not a._input.variable_stride_per_key():
                stride_per_rank = output_splits.pop()
            tensors_awaitables.append(KJTAllToAllTensorsAwaitable(
                pg=a.pg, input=a._input, splits=a.splits, input_splits=a.input_splits, output_splits=output_splits, input_tensors=a.input_tensors,
                labels=a.labels, keys=a.keys, device=a.device, stagger=a.stagger, stride_per_rank=stride_per_rank))
        out: List[KJTListAwaitable] = []
        for group, ctx in zip(_split(tensors_awaitables, self._lengths), self._contexts):
            _set_sharding_context_intra_a2a(group, ctx)
            out.append(KJTListAwaitable(group, ctx))
        return out


def kjt_splits_meta(pg: dist.ProcessGroup, kjt: KeyedJaggedTensor, splits: List[int], stagger: int = 1) -> KJTSplitsAllToAllMeta:
    """Describe a KJT all-to-all without launching its size exchange (the pipelines swap ``KJTAllToAll.forward`` for this when fusing)."""
    import itertools

    cumsum = [0] + list(itertools.accumulate(splits))
    rank = dist.get_rank(pg)
    tensor_splits = kjt.dist_splits(splits)
    dev = kjt.device()
    rows = [torch.tensor(s, device=dev, dtype=torch.int64) for s in tensor_splits]
    if not kjt.variable_stride_per_key():
        rows.append(torch.tensor([kjt.stride()] * pg.size(), device=dev, dtype=torch.int64))
    return KJTSplitsAllToAllMeta(pg=pg, _input=kjt, splits=splits, splits_tensors=rows, input_splits=tensor_splits, input_tensors=kjt.dist_tensors(),
                                 labels=kjt.dist_labels(), keys=kjt.keys()[cumsum[rank] : cumsum[rank + 1]], device=dev, stagger=stagger, splits_cumsum=cumsum)


class ListOfKJTList(Multistreamable):
    def __init__(self, features: List[KJTList]) -> None:
        self.features_list = features

    def __len__(self) -> int:
        return len(self.features_list)

    def __getitem__(self, key: int) -> KJTList:
        return self.features_list[key]

    def __iter__(self):
        return iter(self.features_list)

    def record_stream(self, stream: torch.Stream) -> None:
        for f in self.features_list:
            f.record_stream(stream)


class ListOfKJTListAwaitable(Awaitable[ListOfKJTList]):
    def __init__(self, awaitables: List[Awaitable[KJTList]]) -> None:
        super().__init__()
        self.awaitables = awaitables

    def _wait_impl(self) -> ListOfKJTList:
        return ListOfKJTList([w.wait() for w in self.awaitables])


class ListOfKJTListSplitsAwaitable(Awaitable[Awaitable[ListOfKJTList]]):
    def __init__(self, awaitables: List[Awaitable[Awaitable[KJTList]]]) -> None:
        super().__init__()
        self.awaitables = awaitables

    def _wait_impl(self) -> Awaitable[ListOfKJTList]:
        return ListOfKJTListAwaitable([w.wait() for w in self.awaitables])


# ---- the framework ---------------------------------------------------------------------------------------------------
class EmbeddingShardingContext(Multistreamable):
    """What the output dist must know about the batch the input dist saw (variable batch sizes)."""

    def __init__(self, batch_size_per_rank: Optional[List[int]] = None, batch_size_per_rank_per_feature: Optional[List[List[int]]] = None,
                 batch_size_per_feature_pre_a2a: Optional[List[int]] = None, variable_batch_per_feature: bool = False) -> None:
        super().__init__()
        self.batch_size_per_rank: List[int] = batch_size_per_rank if batch_size_per_rank is not None else []
        self.batch_size_per_rank_per_feature: List[List[int]] = batch_size_per_rank_per_feature if batch_size_per_rank_per_feature is not None else []
        self.batch_size_per_feature_pre_a2a: List[int] = batch_size_per_feature_pre_a2a if batch_size_per_feature_pre_a2a is not None else []
        self.variable_batch_per_feature: bool = variable_batch_per_feature

    def record_stream(self, stream: torch.Stream) -> None:
        pass


class BaseSparseFeaturesDist(abc.ABC, nn.Module, Generic[F]):
    """Input dist of one sharding: local KJT -> ``Awaitable[Awaitable[F]]`` (sizes, then tensors)."""

    @abc.abstractmethod
    def forward(self, sparse_features: KeyedJaggedTensor) -> Union[Awaitable[Awaitable[F]], F]:
        ...


class BaseSparseFeaturesWriteDist(abc.ABC, nn.Module, Generic[F]):
    """Input dist of an embedding UPDATE: ids + new rows -> the row owners."""

    @abc.abstractmethod
    def forward(self, sparse_features: KeyedJaggedTensor, embeddings: torch.Tensor) -> Union[Awaitable[Awaitable[F]], F]:
        ...


class BaseEmbeddingDist(abc.ABC, nn.Module, Generic[C, T, W]):
    """Output dist of one sharding: local lookup result -> ``Awaitable`` of this rank's samples' embeddings."""

    @abc.abstractmethod
    def forward(self, local_embs: T, sharding_ctx: Optional[C] = None) -> Union[Awaitable[W], W]:
        ...


class EmbeddingSharding(abc.ABC, Generic[C, F, T, W], FeatureShardingMixIn):
    """One sharding type's three stages + its naming (reference :1170-1248)."""

    def __init__(self, qcomm_codecs_registry: Optional[Dict[str, QuantizedCommCodecs]] = None) -> None:
        self._qcomm_codecs_registry = qcomm_codecs_registry

    @property
    def qcomm_codecs_registry(self) -> Optional[Dict[str, QuantizedCommCodecs]]:
        return self._qcomm_codecs_registry

    @abc.abstractmethod
    def create_input_dist(self, device: Optional[torch.device] = None) -> BaseSparseFeaturesDist[F]:
        ...

    @abc.abstractmethod
    def create_output_dist(self, device: Optional[torch.device] = None) -> BaseEmbeddingDist[C, T, W]:
        ...

    @abc.abstractmethod
    def create_lookup(self, device: Optional[torch.device] = None, fused_params: Optional[Dict[str, Any]] = None,
                      feature_processor: Optional[nn.Module] = None) -> BaseEmbeddingLookup[F, T]:
        ...

    def create_write_dist(self, device: Optional[torch.device] = None) -> BaseSparseFeaturesWriteDist[F]:
        raise NotImplementedError(f"{type(self).__name__} does not support embedding updates")

    def create_update(self, device: Optional[torch.device] = None, fused_params: Optional[Dict[str, Any]] = None,
                      feature_processor: Optional[nn.Module] = None) -> nn.Module:
        raise NotImplementedError(f"{type(self).__name__} does not support embedding updates")

    @abc.abstractmethod
    def embedding_dims(self) -> List[int]:
        ...

    @abc.abstractmethod
    def embedding_shard_metadata(self) -> List[Optional[ShardMetadata]]:
        ...

    @abc.abstractmethod
    def embedding_names(self) -> List[str]:
        ...

    @abc.abstractmethod
    def embedding_names_per_rank(self) -> List[List[str]]:
        ...

    def embedding_tables(self) -> List[ShardedEmbeddingTable]:
        raise NotImplementedError

    def uncombined_embedding_dims(self) -> List[int]:
        return self.embedding_dims()

    def uncombined_embedding_names(self) -> List[str]:
        return self.embedding_names()


@dataclass
class EmbeddingShardingInfo:
    """One table as the sharded module hands it to an ``EmbeddingSharding``: config + placement + the parameter to copy rows from."""

    embedding_config: Any  # EmbeddingTableConfig
    param_sharding: ParameterSharding
    param: torch.Tensor
    fused_params: Optional[Dict[str, Any]] = None
