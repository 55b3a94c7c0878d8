"""Serving latency of the DLRM predictor: eager executor path against CUDA-graph replay (``inference.graphed.GraphedPredictor``).

    python tools/serve_latency_bench.py --rows 100000 --batches 1,16,64,256,1024,2048 --iters 200

The model is the bench's DLRM shape served from one GPU: 26 quantized tables at D = 128 (INT8 rows under the bf16 dense arch, FP8 rows
under the FP8 dense arch; --rows caps every table so that the float tables can be built and quantized on the host), dense arch
512-256-128, over arch 1024-1024-512-256-1, 13 float features, one id per feature. For every batch size both paths start from the
same pinned slab in the serving core's layout and end with the predictions in host memory, as the server's executor runs them:

* eager: one H2D copy of the slab, KJT views, the predict call, ``.cpu()`` of the result;
* graphed: one H2D copy into the predictor's static slab, ingest + predict replayed from the bucket's graph, a copy into a pinned buffer
  and a stream synchronize. The buckets are the measured batch sizes, with the default id capacity of a 16 MiB slab.

The two alternate call by call after warm-up. Per path it reports the median and p99 of the host wall time per prediction (slab to
host result, ending in a synchronize) and of the device time between CUDA events recorded before the H2D copy and after the D2H copy,
plus the largest difference between the two paths' predictions. The card name, power limit and SM clock limit are read in the same
run. Without a GPU the script fails."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout
    name, power, sm = q.strip().splitlines()[0].split(", ")
    return {"gpu": name, "power_limit": power, "sm_clock_max": sm}


def build(dense_kind: str, rows: int, dev: torch.device):
    from torchrec_b200.inference.modules import quantize_dense, quantize_inference_model, shard_quant_model
    from torchrec_b200.models.dlrm import DLRM
    from torchrec_b200.modules.embedding_configs import EmbeddingBagConfig
    from torchrec_b200.modules.embedding_modules import EmbeddingBagCollection
    from torchrec_b200.types import DataType

    torch.manual_seed(0)
    keys = [f"cat_{i}" for i in range(26)]
    tables = [EmbeddingBagConfig(name=f"t_{k}", embedding_dim=128, num_embeddings=rows, feature_names=[k]) for k in keys]
    model = DLRM(EmbeddingBagCollection(tables), 13, [512, 256, 128], [1024, 1024, 512, 256, 1], dense_device=dev).eval()
    q = quantize_inference_model(model, quantization_dtype=DataType.FP8 if dense_kind == "fp8" else DataType.INT8, output_dtype=torch.float32)
    q, _ = shard_quant_model(q, world_size=1)
    if dense_kind == "fp8":
        q = quantize_dense(q, torch.float8_e4m3fn)

    def predict(dense, kjt, _wkjt):
        return q(dense, kjt).sigmoid().reshape(-1)

    return keys, predict


def pct(xs, p):
    return float(np.percentile(np.asarray(xs), p))


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000)
    ap.add_argument("--batches", default="1,16,64,256,1024,2048")
    ap.add_argument("--dense", default="bf16,fp8")
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("serve_latency_bench needs a CUDA device")
    from torchrec_b200.inference.graphed import GraphedPredictor, pack_slab
    from torchrec_b200.inference.server import ServerConfig, batch_views
    from torchrec_b200.ops import dense as _dense

    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    _dense.set_dense_backend("wgmma")
    info = card()
    batches = [int(b) for b in args.batches.split(",")]
    cfg = ServerConfig()
    results = []
    for dense_kind in args.dense.split(","):
        keys, predict = build(dense_kind, args.rows, dev)
        gp = GraphedPredictor(predict, batches, num_float=13, id_list_keys=keys, device=dev, buffer_bytes=cfg.buffer_bytes, max_batch_size=cfg.max_batch_size)
        gp.capture()
        stream = torch.cuda.Stream(dev)
        out_host = torch.empty(cfg.max_batch_size, dtype=torch.float32, pin_memory=True)
        rng = np.random.default_rng(0)
        for B in batches:
            slabs = []
            for _ in range(8):
                lengths = np.ones(26 * B, dtype=np.int32)
                slab, d = pack_slab(B, rng.random((B, 13), dtype=np.float32), (lengths, rng.integers(0, args.rows, size=26 * B)), None, 26)
                slabs.append((slab.pin_memory(), d))

            def eager(slab, d):
                buf = slab[: d.total_bytes].to(dev, non_blocking=True)
                return predict(*batch_views(buf, d, keys, ())).float().reshape(d.batch_size, -1).cpu()

            def graphed(slab, d):
                gp.slab[: d.total_bytes].copy_(slab[: d.total_bytes], non_blocking=True)
                out = gp.run(gp.slab, d).reshape(-1)
                res = out_host[: out.numel()]
                res.copy_(out, non_blocking=True)
                stream.synchronize()
                return res.clone()

            wall = {"eager": [], "graphed": []}
            devt = {"eager": [], "graphed": []}
            diff = 0.0
            with torch.inference_mode(), torch.cuda.stream(stream):
                for it in range(args.warmup + args.iters):
                    slab, d = slabs[it % len(slabs)]
                    outs = {}
                    for name, fn in (("eager", eager), ("graphed", graphed)) if it % 2 == 0 else (("graphed", graphed), ("eager", eager)):
                        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        t0 = time.perf_counter()
                        e0.record(stream)
                        o = fn(slab, d)
                        e1.record(stream)
                        t1 = time.perf_counter()
                        e1.synchronize()
                        outs[name] = o.reshape(-1)
                        if it >= args.warmup:
                            wall[name].append((t1 - t0) * 1e3)
                            devt[name].append(e0.elapsed_time(e1))
                    diff = max(diff, float((outs["eager"] - outs["graphed"]).abs().max()))
            r = {"dense": dense_kind, "rows_format": "FP8" if dense_kind == "fp8" else "INT8", "B": B, "iters": args.iters,
                 "max_abs_diff": diff, **info}
            for name in ("eager", "graphed"):
                r[f"{name}_wall_ms_p50"], r[f"{name}_wall_ms_p99"] = pct(wall[name], 50), pct(wall[name], 99)
                r[f"{name}_dev_ms_p50"], r[f"{name}_dev_ms_p99"] = pct(devt[name], 50), pct(devt[name], 99)
            r["wall_speedup_p50"] = r["eager_wall_ms_p50"] / r["graphed_wall_ms_p50"]
            print(json.dumps(r), flush=True)
            results.append(r)
        del gp
        torch.cuda.empty_cache()
    print(f"\n{info['gpu']}, power limit {info['power_limit']}, max SM clock {info['sm_clock_max']}; host wall / device ms, median (p99)")
    print("| dense | B | eager wall | graphed wall | eager device | graphed device | wall speed-up |")
    print("|---|---|---|---|---|---|---|")
    for r in results:
        f = lambda k: f"{r[k + '_p50']:.3f} ({r[k + '_p99']:.3f})"
        print(f"| {r['dense']} | {r['B']} | {f('eager_wall_ms')} | {f('graphed_wall_ms')} | {f('eager_dev_ms')} | {f('graphed_dev_ms')} | "
              f"{r['wall_speedup_p50']:.2f}x |")
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(results, fh, indent=1)


if __name__ == "__main__":
    main()
