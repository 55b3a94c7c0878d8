"""Measured costs of THIS framework's kernels on H100, the numbers the planner's perf model is built from.

Measured on one H100 80GB HBM3 (SXM, 700 W power limit) with ``tools/kernel_bench.py`` (CUDA events, L2 flushed, median):

* device-to-device copy: 3015 and 3029 GB/s (read + write bytes) in two runs
* the lookup kernels at the shape of the busiest rank of an 8-GPU DLRM job (below)

Not measured on H100, because that needs several GPUs of one NVLink domain: the per-peer NVLink rate (the data sheet's 450 GB/s per
direction stands in for it), how much an all-to-all of W ranks derates it, how much of the transfer the fused lookup + output dist hides
and how much of the gradient push stays exposed. The model applies no derating and gives no overlap credit for these until they are
measured. Nothing here is inherited from the reference's A100-era constants (``planner/constants.py:16-45`` there: 2.455 batched-copy
factor, 9.22 data-parallel factor, /10 UVM rule ...).
"""
from __future__ import annotations

from typing import Dict

GB = 1024 * 1024 * 1024

COPY_GBPS: float = 3020.0

# ---- NVLink 4 through NVSwitch ------------------------------------------------------------------------------------------------
# one direction, one peer: H100 SXM data sheet (18 links, 900 GB/s bidirectional)
PEER_STORE_GBPS: float = 450.0
# all-to-all among W ranks with both directions busy, as a fraction of PEER_STORE_GBPS (not measured on H100: no derating)
ALL_TO_ALL_EFFICIENCY: Dict[int, float] = {1: 1.0}


def all_to_all_gbps(world_size: int) -> float:
    """Per-direction GB/s one rank sustains inside an all-to-all of ``world_size`` ranks of one NVLink domain."""
    if world_size in ALL_TO_ALL_EFFICIENCY:
        eff = ALL_TO_ALL_EFFICIENCY[world_size]
    else:
        known = sorted(ALL_TO_ALL_EFFICIENCY)
        lo = max((k for k in known if k <= world_size), default=known[0])
        hi = min((k for k in known if k >= world_size), default=known[-1])
        eff = ALL_TO_ALL_EFFICIENCY[lo] if lo == hi else ALL_TO_ALL_EFFICIENCY[lo] + (ALL_TO_ALL_EFFICIENCY[hi] - ALL_TO_ALL_EFFICIENCY[lo]) * (world_size - lo) / (hi - lo)
    return PEER_STORE_GBPS * eff


# ---- table-batched lookup kernels -------------------------------------------------------------------------------------------------
# forward (tbe_pooled_fwd_chunk, one-hot fp32 rows -> bf16): 4 tables of 20 M rows x 262144 samples, 814 MB of row reads + pooled writes
# in 297 us = 2.74 TB/s of algorithmic bytes, 90 % of the copy bandwidth
LOOKUP_FWD_EFFICIENCY: float = 0.90
# backward (tbe_bwd walk + span kernels, row-wise Adagrad; keys + radix sort run on an auxiliary stream, off the critical path): the same
# 1.05 M ids, 1.04 M distinct rows: 1.34 GB of gradient rows + row read-modify-writes + row state in 776 us = 1.73 TB/s, 57 %
LOOKUP_BWD_EFFICIENCY: float = 0.57
# rows narrower than one 512 B warp request (dim 64 / dim 32) against dim 128: model assumptions, not measured on H100
HALF_ROW_PENALTY: float = 1.15
QUARTER_ROW_PENALTY: float = 1.75


def fused_overlap(world_size: int) -> float:
    """Share of min(lookup, transfer) that the fused lookup + output-dist kernel hides: T = lookup + transfer - overlap * min(...).
    Not measured on H100: no overlap credit."""
    return 0.0


# gradient dist: captured inside the dense backward graph beside the deferred weight-gradient GEMMs; the share of the push that stays
# exposed is not measured on H100: all of it
GRAD_PUSH_EXPOSED: float = 1.0
