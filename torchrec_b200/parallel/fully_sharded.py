"""FULLY_SHARDED 2D strategy: between the forward lookup and the backward of a step, every replica of an embedding shard keeps
only 1/R of the (replica-averaged) flat weight buffer.

Parity: reference ``ShardedBatchedFusedEmbeddingBag`` (batched_embedding_kernel.py:4425-4640): after the forward lookup the
flat TBE weights are ``reduce_scatter_tensor(AVG)``-ed over the replica group and the full buffer is released; a backward
pre-hook ``all_gather_into_tensor``s it back before the fused backward + optimizer runs. Net effect per step: replicas are
averaged every step (no periodic ``DMPCollection.sync`` of the weights) and the full copy is not resident while the dense
part of the model runs — with 80 GB of HBM per GPU that is what lets one replica group hold tables sized for the whole group.

Here it is a small state machine attached to a ``TableBatchedEmbeddingBags`` (``tbe._fs``) and driven from the lookup
autograd functions (eager lookup and the fused NVLink lookup + dist)."""
from __future__ import annotations

from typing import Optional

import torch
import torch.distributed as dist


class FullyShardedTBEWeights:
    def __init__(self, tbe: torch.nn.Module, replica_pg: Optional[dist.ProcessGroup]) -> None:
        self.tbe = tbe
        self.pg = replica_pg
        self.R = dist.get_world_size(replica_pg) if replica_pg is not None else 1
        self.rank = dist.get_rank(replica_pg) if replica_pg is not None else 0
        w = tbe.weights.data
        self.numel = w.numel()
        self.shape = tuple(w.shape)
        self.shard_numel = (self.numel + self.R - 1) // self.R
        self.padded = self.shard_numel * self.R
        self.nbytes = w.untyped_storage().nbytes()
        self.shard: Optional[torch.Tensor] = None
        self.sharded = False
        self._native = replica_pg is not None and dist.get_backend(replica_pg) == "nccl"

    # -- forward lookup is done: average over the replicas, keep my slice, drop the full buffer ---------------------------
    @torch.no_grad()
    def after_forward(self) -> None:
        if self.R == 1 or self.sharded or not self.tbe.training:
            return
        w = self.tbe.weights.data
        flat = w.reshape(-1)
        if self.padded != self.numel:
            flat = torch.nn.functional.pad(flat, (0, self.padded - self.numel))
        out = torch.empty(self.shard_numel, dtype=w.dtype, device=w.device)
        if self._native:
            dist.reduce_scatter_tensor(out, flat, op=dist.ReduceOp.AVG, group=self.pg)
        else:  # gloo (CPU tests): no reduce-scatter, no AVG
            tmp = flat.clone() if flat.data_ptr() == w.data_ptr() else flat
            dist.all_reduce(tmp, op=dist.ReduceOp.SUM, group=self.pg)
            out.copy_(tmp[self.rank * self.shard_numel : (self.rank + 1) * self.shard_numel] / self.R)
        self.shard = out
        w.untyped_storage().resize_(0)
        self.sharded = True

    # -- before the fused backward (or the next forward / a state_dict): restore the full, averaged buffer ----------------
    @torch.no_grad()
    def gather(self) -> None:
        if not self.sharded:
            return
        w = self.tbe.weights.data
        w.untyped_storage().resize_(self.nbytes)
        flat = w.reshape(-1)
        assert self.shard is not None
        if self.padded == self.numel and self._native:
            dist.all_gather_into_tensor(flat, self.shard, group=self.pg)
        else:
            parts = [torch.empty_like(self.shard) for _ in range(self.R)]
            dist.all_gather(parts, self.shard, group=self.pg)
            flat.copy_(torch.cat(parts)[: self.numel])
        self.shard = None
        self.sharded = False

    before_backward = gather
    before_forward = gather


def attach(tbe: torch.nn.Module, replica_pg: Optional[dist.ProcessGroup]) -> Optional[FullyShardedTBEWeights]:
    """Enable the strategy for one TBE (device-resident tables only: host-mapped storage cannot be released and re-grown)."""
    loc = getattr(getattr(tbe, "location", None), "name", "DEVICE")
    if tbe.weights.device.type == "meta" or loc in ("MANAGED", "MANAGED_CACHING"):
        return None
    fs = FullyShardedTBEWeights(tbe, replica_pg)
    tbe._fs = fs
    return fs
