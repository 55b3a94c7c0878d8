"""Pin the calling process to the CPUs that are NUMA-local to its GPU.

On a two-socket GPU host the GPU hangs off one socket (``nvidia-smi topo -m``: "CPU Affinity 32-63,96-127"). A rank that the
scheduler happens to place on the other socket allocates its pinned staging buffers there and every H2D copy crosses the
socket interconnect; the end-to-end step time then varies run to run on the same build.
The reference leaves placement to the launcher (``torchx`` / ``numactl``); here it is one call."""
from __future__ import annotations

import os
from typing import Optional, Set


def gpu_local_cpus(device_index: int) -> Optional[Set[int]]:
    """CPU ids NVML reports as local to ``device_index`` (None if NVML is unavailable)."""
    try:
        import pynvml

        pynvml.nvmlInit()
        try:
            visible = os.environ.get("CUDA_VISIBLE_DEVICES")
            if visible:
                tok = visible.split(",")[device_index].strip()
                handle = pynvml.nvmlDeviceGetHandleByUUID(tok) if tok.startswith("GPU-") else pynvml.nvmlDeviceGetHandleByIndex(int(tok))
            else:
                handle = pynvml.nvmlDeviceGetHandleByIndex(device_index)
            n_words = (os.cpu_count() + 63) // 64
            words = pynvml.nvmlDeviceGetCpuAffinity(handle, n_words)
        finally:
            pynvml.nvmlShutdown()
        cpus = {w * 64 + b for w, word in enumerate(words) for b in range(64) if (int(word) >> b) & 1}
        if cpus:
            return cpus
    except Exception:
        pass
    return _sysfs_local_cpus(device_index)


def _sysfs_local_cpus(device_index: int) -> Optional[Set[int]]:
    """Fallback without NVML: the PCI device's ``local_cpulist`` in sysfs."""
    try:
        import torch

        pr = torch.cuda.get_device_properties(device_index)
        path = f"/sys/bus/pci/devices/{pr.pci_domain_id:04x}:{pr.pci_bus_id:02x}:{pr.pci_device_id:02x}.0/local_cpulist"
        with open(path) as f:
            text = f.read().strip()
        cpus: Set[int] = set()
        for part in text.split(","):
            if "-" in part:
                a, b = part.split("-")
                cpus.update(range(int(a), int(b) + 1))
            elif part:
                cpus.add(int(part))
        return cpus or None
    except Exception:
        return None


def bind_to_gpu_numa(device_index: int) -> Optional[Set[int]]:
    """Restrict the process to the intersection of its current CPU set and the GPU-local CPUs. Returns the new set, or None
    when nothing was changed (no NVML, empty intersection, platform without ``sched_setaffinity``)."""
    if not hasattr(os, "sched_setaffinity"):
        return None
    local = gpu_local_cpus(device_index)
    if not local:
        return None
    try:
        allowed = os.sched_getaffinity(0)
        target = allowed & local
        if not target or target == allowed:
            return None
        os.sched_setaffinity(0, target)
        return target
    except OSError:
        return None
