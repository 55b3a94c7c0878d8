"""Sharded quantized EmbeddingCollection for inference (table-wise / row-wise / column-wise / table-row-wise placements over local
devices; reference torchrec/distributed/quant_embedding.py:597-1531)."""
from __future__ import annotations

from typing import Any, Dict, List, Optional, Type

import torch
from torch import nn

from ..quant.embedding_modules import EmbeddingCollection as QuantEmbeddingCollection
from ..sparse.jagged_tensor import JaggedTensor, KeyedJaggedTensor
from .embedding_types import BaseQuantEmbeddingSharder, quant_table_placement
from .engine import shards_of
from .types import LazyNoWait, NoWait, NullShardedModuleContext, ParameterSharding, ShardedModule, ShardingEnv, ShardingType


class ShardedQuantEmbeddingCollection(ShardedModule[List[KeyedJaggedTensor], List[torch.Tensor], Dict[str, JaggedTensor], NullShardedModuleContext]):
    """Sequence (unpooled) quantized lookups over local devices for every placement the planner can emit: a table's shards are
    rectangles (rank, row range, column range) and a feature's output is assembled from them -

        out_f[:, col_off : col_off + cols] += lookup(shard, ids_f - row_off)        (ids outside the shard's rows look up zeros)

    so table-wise is one full rectangle, column-wise fills disjoint column slices, row-wise adds row-disjoint partial results, and
    table-row-wise / grid are combinations. Per device the units are grouped by shard width into one quantized TBE launch each."""

    def __init__(self, module: QuantEmbeddingCollection, params: Dict[str, ParameterSharding], env: ShardingEnv, fused_params=None, device=None) -> None:
        super().__init__()
        from ..ops.quant_tbe import QuantTableBatchedEmbeddingBags, dequantize_rows

        self._device_type = "cuda" if torch.cuda.is_available() and (device is None or device.type == "cuda") else "cpu"
        tables = module.embedding_configs()
        self._tables = tables
        self._need_indices = module.need_indices()
        self._out_dtype = module.output_dtype()
        W = env.world_size
        self._feature_dim: Dict[str, int] = {f: t.embedding_dim for t in tables for f in t.feature_names}
        # (rank, shard width) -> units; a unit = (feature name, table idx, shard)
        groups: Dict[tuple, List[tuple]] = {}
        for ti, t in enumerate(tables):
            for sh in shards_of(ti, t, params[t.name]):
                for f in t.feature_names:
                    groups.setdefault((sh.rank, sh.cols), []).append((f, ti, sh))
        self._groups: List[tuple] = []
        self._tbes = nn.ModuleList()
        for (r, cols), units in sorted(groups.items(), key=lambda kv: kv[0]):
            dev = torch.device("cuda", r) if self._device_type == "cuda" else torch.device("cpu")
            shard_keys: List[tuple] = []
            specs, locs, clfs = [], [], []
            for f, ti, sh in units:
                key = (ti, sh.row_off, sh.col_off)
                if key not in shard_keys:
                    shard_keys.append(key)
                    specs.append((f"{tables[ti].name}_{sh.row_off}_{sh.col_off}", sh.rows, sh.cols, tables[ti].data_type))
                    ps = params[tables[ti].name]
                    loc, clf = quant_table_placement(ps.compute_kernel, getattr(ps, "cache_params", None), fused_params)
                    locs.append(loc)
                    clfs.append(clf)
            fmap = [shard_keys.index((ti, sh.row_off, sh.col_off)) for _, ti, sh in units]
            tbe = QuantTableBatchedEmbeddingBags(specs, fmap, pooling_mode=2, output_dtype=self._out_dtype, device=dev, locations=locs,
                                                 cache_load_factor=clfs)
            for k, (ti, r0, c0) in enumerate(shard_keys):
                t = tables[ti]
                src = module.embeddings[t.name].weight
                rows_k, cols_k = specs[k][1], specs[k][2]
                if r0 == 0 and c0 == 0 and rows_k == t.num_embeddings and cols_k == t.embedding_dim:
                    dst = tbe.split_embedding_weights()[k]  # whole table: the quantized bytes as they are
                    dst.copy_(src.to(dst.device))
                    tbe.invalidate_cache(k)
                else:  # a rectangle of the table: re-quantized (row scales of column slices differ from the full row's)
                    full = dequantize_rows(src.to("cpu"), t.embedding_dim, t.data_type)
                    tbe.assign_from_float(k, full[r0 : r0 + rows_k, c0 : c0 + cols_k])
            self._tbes.append(tbe)
            row_offs = torch.tensor([sh.row_off for _, _, sh in units], dtype=torch.int64)
            self._groups.append((dev, [f for f, _, _ in units], [sh.col_off for _, _, sh in units], cols, row_offs))

    class _Ctx:
        """The batch's features travel from input_dist to output_dist (lengths / ids of the result are the caller's)."""

        features: Optional[KeyedJaggedTensor] = None

        def record_stream(self, stream) -> None:
            pass

    def create_context(self):
        return ShardedQuantEmbeddingCollection._Ctx()

    def input_dist(self, ctx, features: KeyedJaggedTensor):
        keys = features.keys()
        out = []
        for dev, feats, _, _, row_offs in self._groups:
            sub = features.permute([keys.index(f) for f in feats])  # (features repeat once per shard they have on this device)
            ro = row_offs.to(sub.values().device)
            if bool((row_offs != 0).any()):
                lpk = torch.tensor(sub.length_per_key(), dtype=torch.int64, device=ro.device)
                local = sub.values() - torch.repeat_interleave(ro, lpk, output_size=sub.values().numel()).to(sub.values().dtype)
                sub = KeyedJaggedTensor(keys=sub.keys(), values=local, lengths=sub.lengths(), stride=sub.stride())
            out.append(sub.to(dev, non_blocking=True))
        ctx.features = features
        return NoWait(NoWait(out))

    def compute(self, ctx, dist_input):
        return [(tbe(k.values(), k.offsets(), None, batch_size=k.stride()), k) for tbe, k in zip(self._tbes, dist_input)]

    def output_dist(self, ctx, output):
        dev0 = torch.device("cuda", 0) if self._device_type == "cuda" else torch.device("cpu")
        features: KeyedJaggedTensor = ctx.features
        keys = features.keys()
        lpk = features.length_per_key()
        vals = torch.split(features.values().to(dev0), lpk)
        lengths = features.lengths().to(dev0).view(len(keys), -1)
        acc: Dict[str, torch.Tensor] = {}
        for (emb, kjt), (_, feats, col_offs, cols, _) in zip(output, self._groups):
            parts = torch.split(emb.to(dev0), kjt.length_per_key(), dim=0)
            for f, c0, part in zip(feats, col_offs, parts):
                D = self._feature_dim[f]
                if cols == D and f not in acc:
                    acc[f] = part.clone() if part.device == emb.device else part  # full-width shard: no zero-filled buffer needed
                    continue
                if f not in acc:
                    acc[f] = torch.zeros(part.shape[0], D, dtype=part.dtype, device=dev0)
                acc[f][:, c0 : c0 + cols] += part
        res: Dict[str, JaggedTensor] = {}
        for i, k in enumerate(keys):
            if k in acc:
                res[k] = JaggedTensor(values=acc[k], lengths=lengths[i], weights=vals[i] if self._need_indices else None)
        return LazyNoWait(res)

    def forward(self, features: KeyedJaggedTensor):
        ctx = self.create_context()
        return self.output_dist(ctx, self.compute(ctx, self.input_dist(ctx, features).wait().wait())).wait()


class QuantEmbeddingCollectionSharder(BaseQuantEmbeddingSharder[QuantEmbeddingCollection]):
    def shard(self, module, params, env, device=None, module_fqn=None):
        return ShardedQuantEmbeddingCollection(module, params, env, self.fused_params, device)

    def shardable_parameters(self, module: QuantEmbeddingCollection) -> Dict[str, nn.Parameter]:
        return {t.name: nn.Parameter(torch.empty(t.num_embeddings, t.embedding_dim, device="meta"), requires_grad=False) for t in module.embedding_configs()}

    def sharding_types(self, compute_device_type: str) -> List[str]:
        return [ShardingType.TABLE_WISE.value, ShardingType.ROW_WISE.value, ShardingType.COLUMN_WISE.value, ShardingType.TABLE_ROW_WISE.value,
                ShardingType.TABLE_COLUMN_WISE.value]

    @property
    def module_type(self) -> Type[QuantEmbeddingCollection]:
        return QuantEmbeddingCollection


class ShardedQuantManagedCollisionEmbeddingCollection(nn.Module):
    """Quantized sequence tables sharded like a plain quantized collection; the managed-collision collection is replicated (read-only
    when serving) and remaps the raw ids of the full batch before the lookup. Returns ``(embeddings, remapped features)``."""

    def __init__(self, module, params, env, fused_params=None, device=None) -> None:
        super().__init__()
        self._sharded = ShardedQuantEmbeddingCollection(module, params, env, fused_params, device)
        self._managed_collision_collection = module._managed_collision_collection
        self._configs = list(module.embedding_configs())

    def embedding_configs(self):
        return self._configs

    def forward(self, features: KeyedJaggedTensor):
        features = self._managed_collision_collection(features)
        return self._sharded(features), features


class QuantManagedCollisionEmbeddingCollectionSharder(QuantEmbeddingCollectionSharder):
    def shard(self, module, params, env, device=None, module_fqn=None):
        return ShardedQuantManagedCollisionEmbeddingCollection(module, params, env, self.fused_params, device)

    @property
    def module_type(self):
        from ..quant.embedding_modules import QuantManagedCollisionEmbeddingCollection

        return QuantManagedCollisionEmbeddingCollection
