"""Hardware model constants of the planner — H100 SXM / NVLink-4 defaults.

The reference models an A100-era box (HBM 32 GB @ 897 GB/s, 600 GB/s intra-node, 12.5 GB/s cross-node,
planner/constants.py:16-36); here the defaults describe one 8xH100 SXM HGX node: 80 GB HBM3 per GPU, the copy bandwidth
measured on one H100 (``calibration.py``), NVLink 4 through NVSwitch at the data sheet's 450 GB/s per direction with every peer at
full bandwidth, 400 Gb/s NICs across nodes. Kernel-cost factors live in ``calibration.py`` with their measurements.
"""
from typing import Dict, Optional

from ..embedding_types import EmbeddingComputeKernel

MAX_SIZE: int = (1 << 63) - 1

from .calibration import COPY_GBPS, HALF_ROW_PENALTY, LOOKUP_BWD_EFFICIENCY, LOOKUP_FWD_EFFICIENCY, PEER_STORE_GBPS, QUARTER_ROW_PENALTY

INTRA_NODE_BANDWIDTH: float = PEER_STORE_GBPS * 1024 * 1024 * 1024 / 1000  # bytes / ms  (NVLink 4, per direction, one peer)
CROSS_NODE_BANDWIDTH: float = 50 * 1024 * 1024 * 1024 / 1000  # bytes / ms  (400 Gb/s NIC)

MIN_CW_DIM: int = 128
POOLING_FACTOR: float = 1.0

BIGINT_DTYPE: int = 8

HBM_CAP: int = 80 * 1024 * 1024 * 1024  # 80 GB HBM3
DDR_CAP: int = 2048 * 1024 * 1024 * 1024
SSD_CAP: int = 16 * 1024 * 1024 * 1024 * 1024
DDR_MEM_BW: float = 400 * 1024 * 1024 * 1024 / 1000  # bytes / ms
HBM_MEM_BW: float = COPY_GBPS * 1024 * 1024 * 1024 / 1000  # bytes / ms (measured device-to-device copy)
SSD_MEM_BW: float = 7 * 1024 * 1024 * 1024 / 1000
HBM_TO_DDR_MEM_BW: float = 55 * 1024 * 1024 * 1024 / 1000  # PCIe Gen5 x16
UVM_CACHING_RATIO: float = 0.2
BATCH_SIZE: int = 512

FULL_BLOCK_EMB_DIM: int = 128  # one warp moves a 512 B (128 x fp32) row per request
HALF_BLOCK_PENALTY: float = HALF_ROW_PENALTY
QUARTER_BLOCK_PENALTY: float = QUARTER_ROW_PENALTY
# backward = gradient row + row read + row write per id at the measured backward efficiency, relative to the forward's (row + pooled row):
# (256 + 512 + 512) / LOOKUP_BWD_EFFICIENCY vs (512 + 256) / LOOKUP_FWD_EFFICIENCY for fp32 rows / bf16 outputs
BWD_COMPUTE_MULTIPLIER: float = round(((256 + 512 + 512) / LOOKUP_BWD_EFFICIENCY) / ((512 + 256) / LOOKUP_FWD_EFFICIENCY), 2)
WEIGHTED_KERNEL_MULTIPLIER: float = 1.1  # one more 4 B load + multiply per id (weighted TBE forward / backward)


def kernel_bw_lookup(compute_device: str, compute_kernel: str, hbm_mem_bw: float, ddr_mem_bw: float, hbm_to_ddr_mem_bw: float,
                     caching_ratio: Optional[float] = None, prefetch_pipeline: bool = False) -> Optional[float]:
    """Effective bandwidth (bytes/ms) a lookup kernel sees for a compute kernel / placement."""
    caching_ratio = caching_ratio if caching_ratio else UVM_CACHING_RATIO
    lookup: Dict = {
        ("cpu", EmbeddingComputeKernel.DENSE.value): 0.5 * ddr_mem_bw,
        ("cpu", EmbeddingComputeKernel.FUSED.value): 1 * ddr_mem_bw,
        ("cpu", EmbeddingComputeKernel.QUANT.value): 1 * ddr_mem_bw,
        ("cuda", EmbeddingComputeKernel.DENSE.value): 0.5 * hbm_mem_bw,
        ("cuda", EmbeddingComputeKernel.FUSED.value): LOOKUP_FWD_EFFICIENCY * hbm_mem_bw,
        # zero-copy host rows: every gathered row is one PCIe read of a 512 B line; random reads reach about half of the link's streaming rate
        ("cuda", EmbeddingComputeKernel.FUSED_UVM.value): 0.5 * hbm_to_ddr_mem_bw,
        # hits at the HBM lookup rate, misses through the row mover over PCIe (time adds up: harmonic mix, not a weighted mean of rates)
        ("cuda", EmbeddingComputeKernel.FUSED_UVM_CACHING.value): 1.0 / (caching_ratio / (LOOKUP_FWD_EFFICIENCY * hbm_mem_bw) + (1 - caching_ratio) / (0.5 * hbm_to_ddr_mem_bw)),
        ("cuda", EmbeddingComputeKernel.QUANT.value): LOOKUP_FWD_EFFICIENCY * hbm_mem_bw,
        ("cuda", EmbeddingComputeKernel.QUANT_UVM.value): 0.5 * hbm_to_ddr_mem_bw,
        ("cuda", EmbeddingComputeKernel.QUANT_UVM_CACHING.value): 1.0 / (caching_ratio / (LOOKUP_FWD_EFFICIENCY * hbm_mem_bw) + (1 - caching_ratio) / (0.5 * hbm_to_ddr_mem_bw)),
        ("cuda", EmbeddingComputeKernel.KEY_VALUE.value): hbm_to_ddr_mem_bw,
        ("cuda", EmbeddingComputeKernel.SSD_VIRTUAL_TABLE.value): SSD_MEM_BW,
        ("cuda", EmbeddingComputeKernel.DRAM_VIRTUAL_TABLE.value): hbm_to_ddr_mem_bw,
    }
    if prefetch_pipeline and compute_device == "cuda" and compute_kernel == EmbeddingComputeKernel.FUSED_UVM_CACHING.value:
        return lookup.get(("cuda", EmbeddingComputeKernel.FUSED.value))
    return lookup.get((compute_device, compute_kernel))

NUM_POOLINGS: float = 1.0  # poolings per feature and example unless a constraint says otherwise
