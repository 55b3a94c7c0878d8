"""Sharded quantized sequence lookups (ShardedQuantEmbeddingCollection): the fused path against the decomposed
input_dist / compute / output_dist of the same module.

    python tools/quant_ec_bench.py --rows 200000 --tables 4 --ids-per-bag 50 --batches 256,4096

For INT8 and FP8 rows, D in {64, 128}, every batch size and the placements table-wise, column-wise (two halves) and row-wise (4 row
shards), all shards on cuda:0, it times both paths with CUDA events after warm-up: the two alternate, each runs twice, and every run
reports the median of --iters calls. One JSON line per case: ms per call, host enqueue ms (median time until the call returns, without
a synchronize), device operations per call (kernels and copies, from one profiled call of each path), and bytes of rows gathered and
of rows written by the lookups (from shapes). The card name, its power limit and its SM clock limit are read in the same run."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from torchrec_b200.ops.quant_tbe import row_bytes  # noqa: E402
from torchrec_b200.types import DataType  # noqa: E402


def card() -> dict:
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout
        name, power, sm = q.strip().splitlines()[0].split(", ")
        return {"gpu": name, "power_limit": power, "sm_clock_max": sm}
    except Exception:
        return {"gpu": torch.cuda.get_device_name(), "power_limit": "unknown", "sm_clock_max": "unknown"}


def build(fmt: str, T: int, rows: int, dim: int, placement: str):
    from torchrec_b200.inference.modules import quantize_inference_model
    from torchrec_b200.modules.embedding_configs import EmbeddingConfig
    from torchrec_b200.modules.embedding_modules import EmbeddingCollection
    from torchrec_b200.parallel.quant_embedding import ShardedQuantEmbeddingCollection
    from torchrec_b200.parallel.types import EnumerableShardingSpec, ParameterSharding, ShardingEnv, ShardMetadata

    tables = [EmbeddingConfig(name=f"t{i}", embedding_dim=dim, num_embeddings=rows, feature_names=[f"f{i}"]) for i in range(T)]

    class M(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.ec = EmbeddingCollection(tables=tables)

    torch.manual_seed(0)
    qec = quantize_inference_model(M(), quantization_dtype=getattr(DataType, fmt), output_dtype=torch.float32).ec
    if placement == "tw":
        shards, kind = [(0, 0, rows, dim)], "table_wise"
    elif placement == "cw":
        shards, kind = [(0, 0, rows, dim // 2), (0, dim // 2, rows, dim // 2)], "column_wise"
    else:
        q = rows // 4
        shards, kind = [(i * q, 0, q if i < 3 else rows - 3 * q, dim) for i in range(4)], "row_wise"
    plan = {t.name: ParameterSharding(sharding_type=kind, compute_kernel="quant", ranks=[0] * len(shards), sharding_spec=EnumerableShardingSpec(
        [ShardMetadata(shard_sizes=[r, c], shard_offsets=[ro, co], placement="rank:0/cuda:0") for ro, co, r, c in shards])) for t in tables}
    return ShardedQuantEmbeddingCollection(qec, plan, ShardingEnv.from_local(1, 0), device=torch.device("cuda:0")), shards


def batch(T: int, B: int, L: int, rows: int, dev):
    from torchrec_b200.sparse import KeyedJaggedTensor

    g = torch.Generator().manual_seed(1)
    lens = torch.randint(L // 2, L + L // 2 + 1, (T * B,), generator=g)
    vals = torch.randint(0, rows, (int(lens.sum()),), generator=g)
    kjt = KeyedJaggedTensor(keys=[f"f{i}" for i in range(T)], values=vals.to(dev), lengths=lens.to(dev), stride=B)
    kjt.length_per_key()
    return kjt


def time_path(fn, iters: int):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    dev_ms, host_ms = [], []
    for _ in range(iters):
        s.record()
        t0 = time.perf_counter()
        fn()
        host_ms.append((time.perf_counter() - t0) * 1e3)
        e.record()
        e.synchronize()
        dev_ms.append(s.elapsed_time(e))
    return statistics.median(dev_ms), statistics.median(host_ms)


def device_ops(fn) -> int:
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(1 for ev in prof.events() if ev.device_type.name == "CUDA")


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=200_000)
    ap.add_argument("--tables", type=int, default=4)
    ap.add_argument("--ids-per-bag", type=int, default=50)
    ap.add_argument("--batches", default="256,4096")
    ap.add_argument("--dims", default="64,128")
    ap.add_argument("--formats", default="INT8,FP8")
    ap.add_argument("--placements", default="tw,cw,rw")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "the benchmark times the GPU"
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    print(json.dumps(card()), flush=True)
    for fmt in a.formats.split(","):
        for dim in (int(x) for x in a.dims.split(",")):
            for placement in a.placements.split(","):
                m, shards = build(fmt, a.tables, a.rows, dim, placement)
                for B in (int(x) for x in a.batches.split(",")):
                    kjt = batch(a.tables, B, a.ids_per_bag, a.rows, dev)
                    n = kjt.values().numel()

                    def decomposed():
                        ctx = m.create_context()
                        return m.output_dist(ctx, m.compute(ctx, m.input_dist(ctx, kjt).wait().wait())).wait()

                    paths = {"fused": lambda: m.forward_fused(kjt), "decomposed": decomposed}
                    for fn in paths.values():
                        for _ in range(a.warmup):
                            fn()
                    torch.cuda.synchronize()
                    res = {k: [] for k in paths}
                    for _ in range(2):  # alternate the two paths, each twice
                        for k, fn in paths.items():
                            res[k].append(time_path(fn, a.iters))
                    ops = {k: device_ops(fn) for k, fn in paths.items()}
                    dt = getattr(DataType, fmt)
                    gathered = n * (sum(row_bytes(c, dt) for _, _, _, c in shards) if placement == "cw" else row_bytes(dim, dt))
                    written = n * dim * 4
                    # the decomposed row-wise path looks every id up on every row shard (zero rows for the ids outside it)
                    dec_written = written * (len(shards) if placement == "rw" else 1)
                    for k in paths:
                        print(json.dumps({"format": fmt, "dim": dim, "placement": placement, "B": B, "ids": n, "path": k,
                                          "ms": [round(x[0], 4) for x in res[k]], "host_enqueue_ms": [round(x[1], 4) for x in res[k]],
                                          "device_ops_per_call": ops[k], "rows_gathered_bytes": gathered,
                                          "rows_written_bytes": written if k == "fused" else dec_written}), flush=True)
                del m
                torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
