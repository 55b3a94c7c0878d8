"""Training HBM cache of fused_uvm_caching tables: prefetch cost and step time, this build against another ``ops/uvm.py``.

    python tools/uvm_cache_bench.py [--baseline path/to/older/uvm.py] [--tables 26 --rows 2000000 --dim 128 --batch 32768]

Workload: ``--tables`` tables of ``--rows`` x ``--dim`` fp32 rows in pinned host memory behind a cache of ``cache_load_factor`` 0.2,
one id per table and sample drawn from a Zipf law (a = 1.05), row-wise Adagrad. The cache starts cold; ``--warmup`` steps fill it.

Two measurements per implementation, the implementations alternating ``--rounds`` times:
  * module: ``prefetch`` + forward + backward of one ``UvmCachedEmbeddingBags`` on the current stream. Reported: device time of the
    prefetch (CUDA events), host time of the ``prefetch`` call, host enqueue time of the whole step and step time (synchronised), hit rate.
  * pipeline: a one-GPU sharded EBC of the same tables (compute kernel fused_uvm_caching) under a small dense model, stepped through
    PrefetchTrainPipelineSparseDist and TrainPipelineSparseDist. Reported: step time (synchronised at the end of the window).
``--baseline`` loads another ``ops/uvm.py`` (for instance the parent commit's) in place of this one. Results: one JSON line per run,
and the list of them in ``--out`` (default: uvm_cache_bench.json in the temporary directory)."""
from __future__ import annotations

import argparse
import importlib.util
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402


def _load_uvm(path):
    import torchrec_b200.ops.uvm as cur

    if path is None:
        return cur
    spec = importlib.util.spec_from_file_location("torchrec_b200.ops._uvm_baseline", path)
    mod = importlib.util.module_from_spec(spec)
    sys.modules[spec.name] = mod
    spec.loader.exec_module(mod)
    return mod


def _zipf_batches(n, T, rows, B, dev, seed):
    g = torch.Generator().manual_seed(seed)
    out = []
    # inverse-CDF sampling of a Zipf(1.05) law truncated to `rows`, shuffled per table so hot ids differ between tables
    ranks = torch.arange(1, rows + 1, dtype=torch.float64)
    cdf = torch.cumsum(ranks.pow(-1.05), 0)
    cdf /= cdf[-1].clone()
    perms = [torch.randperm(rows, generator=g) for _ in range(T)]
    for _ in range(n):
        u = torch.rand(T, B, generator=g, dtype=torch.float64)
        r = torch.searchsorted(cdf, u).clamp_(max=rows - 1)
        ids = torch.stack([perms[t][r[t]] for t in range(T)]).reshape(-1)
        out.append((ids.to(dev), torch.arange(0, T * B + 1, device=dev)))
    return out


def _module_run(uvm, a, batches, warmup, steps):
    from torchrec_b200.ops.tbe import OptimType, PoolingMode

    dev = torch.device("cuda:0")
    specs = [(a.rows, a.dim)] * a.tables
    m = uvm.UvmCachedEmbeddingBags(specs, list(range(a.tables)), cache_load_factor=0.2, device=dev, pooling_mode=PoolingMode.SUM,
                                   optimizer=OptimType.EXACT_ROWWISE_ADAGRAD, learning_rate=0.01, eps=1e-8)
    gout = torch.randn(a.batch, a.tables * a.dim, device=dev)
    s0 = None
    pf_dev, pf_host, enq, step = [], [], [], []
    for i in range(warmup + steps):
        idx, off = batches[i % len(batches)]
        if i == warmup:
            torch.cuda.synchronize()
            s0 = dict(m.stats)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        e0.record()
        m.prefetch(idx, off, a.batch)
        e1.record()
        t1 = time.perf_counter()
        m(idx, off, None, batch_size=a.batch).backward(gout)
        t2 = time.perf_counter()
        torch.cuda.synchronize()
        t3 = time.perf_counter()
        if i >= warmup:
            pf_dev.append(e0.elapsed_time(e1) * 1e3)
            pf_host.append((t1 - t0) * 1e6)
            enq.append((t2 - t0) * 1e6)
            step.append((t3 - t0) * 1e6)
    s1 = m.stats
    hits, misses = s1["hits"] - s0["hits"], s1["misses"] - s0["misses"]
    med = lambda xs: sorted(xs)[len(xs) // 2]
    res = {"prefetch_device_us": med(pf_dev), "prefetch_host_us": med(pf_host), "step_enqueue_us": med(enq), "step_us": med(step),
           "hit_rate": hits / max(hits + misses, 1), "evictions": s1["evictions"] - s0["evictions"]}
    del m
    torch.cuda.empty_cache()
    return res


def _pipeline_run(uvm, a, batches, warmup, steps):
    import torchrec_b200.ops.uvm as cur_uvm
    from torchrec_b200.models.dlrm import DLRM, DLRMTrain
    from torchrec_b200.modules.embedding_configs import EmbeddingBagConfig
    from torchrec_b200.modules.embedding_modules import EmbeddingBagCollection
    from torchrec_b200.optim.apply_optimizer_in_backward import apply_optimizer_in_backward
    from torchrec_b200.optim.rowwise_adagrad import RowWiseAdagrad
    from torchrec_b200.parallel import sharding_plan as sp
    from torchrec_b200.parallel import train_pipeline as tp
    from torchrec_b200.parallel.embeddingbag import EmbeddingBagCollectionSharder
    from torchrec_b200.parallel.model_parallel import DistributedModelParallel
    from torchrec_b200.parallel.types import CacheParams, ShardingPlan
    from torchrec_b200.sparse import KeyedJaggedTensor
    from torchrec_b200.datasets.utils import Batch

    dev = torch.device("cuda:0")
    keys = [f"f{i}" for i in range(a.tables)]

    def build():
        saved = cur_uvm.UvmCachedEmbeddingBags
        cur_uvm.UvmCachedEmbeddingBags = uvm.UvmCachedEmbeddingBags  # the sharded kernel imports the class at construction
        try:
            ebc = EmbeddingBagCollection([EmbeddingBagConfig(name=f"t{i}", embedding_dim=a.dim, num_embeddings=a.rows, feature_names=[keys[i]])
                                          for i in range(a.tables)], device=torch.device("meta"))
            apply_optimizer_in_backward(RowWiseAdagrad, ebc.parameters(), {"lr": 0.01})
            model = DLRMTrain(DLRM(ebc, 13, [512, a.dim], [512, 256, 1], dense_device=dev))
            plan = sp.construct_module_sharding_plan(ebc, {f"t{i}": sp.table_wise(rank=0, compute_kernel="fused_uvm_caching") for i in range(a.tables)},
                                                     sharder=EmbeddingBagCollectionSharder(), world_size=1, local_size=1, device_type="cuda")
            for i in range(a.tables):
                plan[f"t{i}"].cache_params = CacheParams(load_factor=0.2)
            return DistributedModelParallel(model, device=dev, plan=ShardingPlan({"model.sparse_arch.embedding_bag_collection": plan}),
                                            sharders=[EmbeddingBagCollectionSharder()])
        finally:
            cur_uvm.UvmCachedEmbeddingBags = saved

    host = []
    g = torch.Generator().manual_seed(5)
    for idx, _off in batches:
        host.append(Batch(dense_features=torch.randn(a.batch, 13, generator=g).pin_memory(),
                          sparse_features=KeyedJaggedTensor(keys=keys, values=idx.cpu().pin_memory(), lengths=torch.ones(a.tables * a.batch, dtype=torch.int32)),
                          labels=torch.randint(0, 2, (a.batch,), generator=g).float().pin_memory()))
    res = {}
    # each pipeline on a fresh model, so both start from a cold cache and see the same batches
    for name, cls in (("prefetch_pipeline", tp.PrefetchTrainPipelineSparseDist), ("sparse_dist_pipeline", tp.TrainPipelineSparseDist)):
        dmp = build()
        opt = torch.optim.SGD([p for p in dmp.parameters() if p.requires_grad], lr=0.01)
        pipe = cls(dmp, opt, dev)
        n = warmup + steps
        it = iter([host[i % len(host)] for i in range(n)])
        for _ in range(warmup):
            pipe.progress(it)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        k = 0
        while True:
            try:
                pipe.progress(it)
                k += 1
            except StopIteration:
                break
        torch.cuda.synchronize()
        res[f"{name}_step_us"] = (time.perf_counter() - t0) * 1e6 / max(k, 1)
        del dmp, opt, pipe
        torch.cuda.empty_cache()
    return res


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--baseline", default=None, help="path of another ops/uvm.py to compare against")
    ap.add_argument("--tables", type=int, default=26)
    ap.add_argument("--rows", type=int, default=2_000_000)
    ap.add_argument("--dim", type=int, default=128)
    ap.add_argument("--batch", type=int, default=32768)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--no-pipeline", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("uvm_cache_bench needs a GPU")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(f"# GPU: {smi}", flush=True)
    impls = {"this": _load_uvm(None)}
    if a.baseline:
        impls["baseline"] = _load_uvm(a.baseline)
    batches = _zipf_batches(a.warmup + a.steps, a.tables, a.rows, a.batch, torch.device("cuda:0"), seed=1)
    out = a.out or os.path.join(tempfile.gettempdir(), "uvm_cache_bench.json")
    os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
    results = []
    for r in range(a.rounds):
        for name, uvm in impls.items():
            res = {"impl": name, "round": r, "gpu": smi, "tables": a.tables, "rows": a.rows, "dim": a.dim, "batch": a.batch}
            res.update(_module_run(uvm, a, batches, a.warmup, a.steps))
            if not a.no_pipeline:
                res.update(_pipeline_run(uvm, a, batches, a.warmup, a.steps))
            print(json.dumps(res), flush=True)
            results.append(res)
            with open(out, "w") as f:
                json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
