"""Stock hardware configs (reference ``planner/estimator/config.py:69`` ``EmbeddingPerfEstimatorConfig``)."""
from __future__ import annotations

from .. import constants as K
from .annotations import hbm_mem_bw, hbm_to_ddr_mem_bw, inter_host_bw, intra_host_bw
from .types import HardwarePerfConfig


class EmbeddingPerfEstimatorConfig(HardwarePerfConfig):
    """The planner's default: one 8 x H100 HGX node (``planner/constants.py``)."""

    name = "h100"


@hbm_mem_bw(K.HBM_MEM_BW)
@intra_host_bw(K.INTRA_NODE_BANDWIDTH)
@inter_host_bw(K.CROSS_NODE_BANDWIDTH)
@hbm_to_ddr_mem_bw(450 * 1024 * 1024 * 1024 / 1000)
class GB200PerfConfig(HardwarePerfConfig):
    """Grace-Blackwell: the host link is NVLink-C2C (~450 GB/s per direction) instead of PCIe - host-resident tables are an order cheaper."""

    name = "gb200"
