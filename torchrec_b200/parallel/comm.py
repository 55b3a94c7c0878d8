"""Process-group topology helpers (reference torchrec/distributed/comm.py:38-335).

On an 8-GPU HGX box every GPU reaches every peer at full NVLink bandwidth through NVSwitch, so
the "node" (intra) group normally equals the world; the intra/cross split is kept for multi-node
jobs and for simulating hierarchies on one host (tests override LOCAL_WORLD_SIZE).
"""
from __future__ import annotations

import logging
import os
from typing import List, Optional, Tuple

import torch
import torch.distributed as dist

logger = logging.getLogger(__name__)

_INTRA_PG: Optional[dist.ProcessGroup] = None
_CROSS_PG: Optional[dist.ProcessGroup] = None
_PG_KEY: Optional[Tuple[int, int]] = None


def _env2int(env_list: List[str], default: int = -1) -> int:
    for e in env_list:
        val = int(os.environ.get(e, -1))
        if val >= 0:
            return val
    return default


def get_local_size(world_size: Optional[int] = None) -> int:
    """Ranks per NVLink domain ("node"). ``TOPOLOGY_DOMAIN_MULTIPLE`` widens it to a pod."""
    if world_size is None:
        world_size = dist.get_world_size() if dist.is_initialized() else 1
    local_size = _env2int(["LOCAL_WORLD_SIZE", "MPI_LOCALNRANKS", "OMPI_COMM_WORLD_LOCAL_SIZE", "MV2_COMM_WORLD_LOCAL_SIZE"], 8)
    local_size *= max(_env2int(["TOPOLOGY_DOMAIN_MULTIPLE"], 1), 1)
    if local_size == -1 or world_size % local_size != 0:
        logging.warning("Could not determine LOCAL_WORLD_SIZE from environment, falling back to WORLD_SIZE.")
        local_size = world_size
    return min(local_size, world_size)


def get_local_rank(world_size: Optional[int] = None, rank: Optional[int] = None) -> int:
    my_local_rank = _env2int(["LOCAL_RANK", "MPI_LOCALRANKID", "OMPI_COMM_WORLD_LOCAL_RANK", "MV2_COMM_WORLD_LOCAL_RANK"], -1)
    local_size = get_local_size(world_size)
    if my_local_rank == -1 or my_local_rank >= local_size:
        if rank is None:
            rank = dist.get_rank() if dist.is_initialized() else 0
        my_local_rank = rank % local_size
    return my_local_rank


def get_group_rank(world_size: Optional[int] = None, rank: Optional[int] = None) -> int:
    if rank is None:
        rank = dist.get_rank() if dist.is_initialized() else 0
    return rank // get_local_size(world_size)


def get_num_groups(world_size: Optional[int] = None) -> int:
    if world_size is None:
        world_size = dist.get_world_size() if dist.is_initialized() else 1
    return world_size // get_local_size(world_size)


_NODE_GROUP_SIZE_2D: Optional[int] = None  # set while the process groups of a 2D-parallel job are built


def get_node_group_size(world_size: Optional[int] = None) -> int:
    """Ranks per node as the current sharding group sees it: the 2D node group size when one is active, else the local world size."""
    return get_local_size(world_size) if _NODE_GROUP_SIZE_2D is None else _NODE_GROUP_SIZE_2D


def get_topology_domain_multiple() -> Optional[int]:
    """Hosts per high-bandwidth domain (an NVLink / NVSwitch pod spanning several hosts, e.g. NVL72): ``TOPOLOGY_DOMAIN_MULTIPLE``."""
    v = _env2int(["TOPOLOGY_DOMAIN_MULTIPLE"], -1)
    return None if v == -1 else v


def get_topology_group_world_size(world_size: Optional[int] = None) -> int:
    """Processes linked by the high-bandwidth fabric: hosts per domain x ranks per host (the local world size when no domain multiple is
    set); the world size must be a multiple of it."""
    multiple = get_topology_domain_multiple()
    if multiple is None:
        return get_local_size(world_size)
    per_host = _env2int(["LOCAL_WORLD_SIZE", "MPI_LOCALNRANKS", "OMPI_COMM_WORLD_LOCAL_SIZE", "MV2_COMM_WORLD_LOCAL_SIZE"], 8)  # ``get_local_size`` already spans the domain
    per_domain = multiple * per_host
    world_size = dist.get_world_size() if world_size is None else world_size
    if world_size % per_domain != 0:
        raise ValueError(f"World size {world_size} is not a multiple of the topology group: {per_domain}")
    return per_domain


def intra_and_cross_node_pg(device: Optional[torch.device] = None, backend: Optional[str] = None) -> Tuple[Optional[dist.ProcessGroup], Optional[dist.ProcessGroup]]:
    """(intra-node group, cross-node group of same-local-rank peers); cached."""
    global _INTRA_PG, _CROSS_PG, _PG_KEY
    my_size = dist.get_world_size()
    my_rank = dist.get_rank()
    my_local_rank = get_local_rank(my_size, my_rank)
    local_size = get_local_size(my_size)
    my_group_rank = get_group_rank(my_size, my_rank)
    group_count = get_num_groups(my_size)
    if backend is None:
        backend = dist.get_backend()
    key = (my_size, local_size)
    if _PG_KEY != key:
        _INTRA_PG = _CROSS_PG = None
        _PG_KEY = key
    if _INTRA_PG is None:
        for group_rank in range(group_count):
            peers = [group_rank * local_size + r for r in range(local_size)]
            pg = dist.new_group(backend=backend, ranks=peers)
            if my_group_rank == group_rank:
                _INTRA_PG = pg
        dist.barrier()
    if _CROSS_PG is None:
        for l_rank in range(local_size):
            peers = [l_rank + g * local_size for g in range(group_count)]
            pg = dist.new_group(backend=backend, ranks=peers)
            if l_rank == my_local_rank:
                _CROSS_PG = pg
        dist.barrier()
    return _INTRA_PG, _CROSS_PG


def intra_and_cross_node_pg_2D(env, device: Optional[torch.device] = None) -> Tuple[Optional[dist.ProcessGroup], Optional[dist.ProcessGroup]]:
    """Intra / cross node groups inside one sharding group of a 2D-parallel job."""
    backend = dist.get_backend(env.sharding_pg)
    my_rank = dist.get_rank()
    ranks = dist.get_process_group_ranks(env.sharding_pg)
    local_size = env.node_group_size if env.node_group_size else get_local_size(len(ranks))
    local_size = min(local_size, len(ranks))
    global _NODE_GROUP_SIZE_2D
    _NODE_GROUP_SIZE_2D = local_size
    intra = cross = None
    world = dist.get_world_size()
    step = env.num_sharding_groups
    for g in range(step):
        group_ranks = list(range(g, world, step)) if not env.use_inter_host_allreduce else list(range(g * len(ranks), (g + 1) * len(ranks)))
        for n in range(len(group_ranks) // local_size):
            peers = group_ranks[n * local_size : (n + 1) * local_size]
            pg = dist.new_group(backend=backend, ranks=peers)
            if my_rank in peers:
                intra = pg
        for l in range(local_size):
            peers = group_ranks[l::local_size]
            pg = dist.new_group(backend=backend, ranks=peers)
            if my_rank in peers:
                cross = pg
    dist.barrier()
    return intra, cross
