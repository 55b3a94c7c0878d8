"""Quantized lookups from HBM, from pinned host memory (zero-copy) and from host memory behind the HBM row cache.

    python tools/quant_offload_bench.py --rows 2000000 --tables 8 --dim 128 --batches 512,4096,32768

For every row format (FP8, INT8), batch size and id distribution (uniform, Zipf(1.05)) it times DEVICE, MANAGED and MANAGED_CACHING
(each load factor) with CUDA events after warm-up, and prints one JSON line per case: ms per batch, cache hit rate, host bytes read per
batch (misses x row bytes; every id of a MANAGED table) and the host-link rate that implies. The card name and its power limit are read
in the same run. Sizes are flags so the tables fit the host memory of the machine at hand (8 x rows x row bytes of pinned memory)."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from torchrec_b200.ops.quant_tbe import QuantTableBatchedEmbeddingBags  # noqa: E402
from torchrec_b200.ops.tbe import EmbeddingLocation as EL  # noqa: E402
from torchrec_b200.types import DataType  # noqa: E402


def card() -> dict:
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout
        name, power = q.strip().splitlines()[0].split(", ")
        return {"gpu": name, "power_limit": power}
    except Exception:
        return {"gpu": torch.cuda.get_device_name(), "power_limit": "unknown"}


def ids(rng, dist: str, n: int, rows: int) -> np.ndarray:
    if dist == "uniform":
        return rng.integers(0, rows, size=n)
    return (rng.zipf(1.05, size=n) - 1) % rows


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--tables", type=int, default=8)
    ap.add_argument("--dim", type=int, default=128)
    ap.add_argument("--batches", default="512,4096,32768")
    ap.add_argument("--formats", default="FP8,INT8")
    ap.add_argument("--dists", default="uniform,zipf")
    ap.add_argument("--load-factors", default="0.05,0.2")
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--iters", type=int, default=50)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    info = card()
    T = a.tables
    placements = [("DEVICE", EL.DEVICE, 0.0), ("MANAGED", EL.MANAGED, 0.0)] + \
        [(f"MANAGED_CACHING@{lf}", EL.MANAGED_CACHING, float(lf)) for lf in a.load_factors.split(",")]
    for fmt in a.formats.split(","):
        dt = getattr(DataType, fmt)
        specs = [(f"t{i}", a.rows, a.dim, dt) for i in range(T)]
        src = QuantTableBatchedEmbeddingBags(specs, device=dev)
        for t in range(T):
            src.split_embedding_weights()[t].random_(0, 120)  # arbitrary bytes: the lookup cost does not depend on them
        rb = src._row_bytes[0]
        for name, loc, lf in placements:
            if loc == EL.DEVICE:
                mod = src
            else:
                mod = QuantTableBatchedEmbeddingBags(specs, device=dev, locations=[loc] * T, cache_load_factor=lf or 0.2)
                for t in range(T):
                    mod.split_embedding_weights()[t].copy_(src.split_embedding_weights()[t])
                mod.invalidate_cache()
            for B in (int(x) for x in a.batches.split(",")):
                for dist in a.dists.split(","):
                    rng = np.random.default_rng(0)
                    batches = []
                    for _ in range(8):
                        v = np.concatenate([ids(rng, dist, B, a.rows) for _ in range(T)])
                        batches.append(torch.from_numpy(v).to(torch.int32).to(dev))
                    off = torch.arange(T * B + 1, dtype=torch.int32, device=dev)
                    for i in range(a.warmup):
                        mod(batches[i % 8], off)
                    s0 = mod.cache_stats() if loc == EL.MANAGED_CACHING else {}
                    torch.cuda.synchronize()
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for i in range(a.iters):
                        mod(batches[i % 8], off)
                    e1.record()
                    torch.cuda.synchronize()
                    ms = e0.elapsed_time(e1) / a.iters
                    if loc == EL.MANAGED_CACHING:
                        s1 = mod.cache_stats()
                        look = sum(s1[k]["lookups"] - s0[k]["lookups"] for k in s1)
                        hits = sum(s1[k]["hits"] - s0[k]["hits"] for k in s1)
                        hit_rate = hits / max(look, 1)
                        host_bytes = (look - hits) / a.iters * rb
                    else:
                        hit_rate = None
                        host_bytes = 0.0 if loc == EL.DEVICE else T * B * rb
                    print(json.dumps({"format": fmt, "placement": name, "B": B, "ids": dist, "tables": T, "rows": a.rows, "dim": a.dim,
                                      "ms_per_batch": round(ms, 4), "hit_rate": None if hit_rate is None else round(hit_rate, 4),
                                      "host_bytes_per_batch": int(host_bytes), "host_GBps": round(host_bytes / (ms * 1e-3) / 1e9, 2), **info}),
                          flush=True)
            if mod is not src:
                del mod
                torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
