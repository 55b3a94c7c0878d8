"""YAML-driven train-pipeline benchmark (reference torchrec/distributed/benchmark/benchmark_train_pipeline.py + yaml/*.yml).

    python -m torchrec_b200.benchmarks.benchmark_train_pipeline --yaml torchrec_b200/benchmarks/yaml/sparse_dist.yml
    torchrun --nproc-per-node 8 -m torchrec_b200.benchmarks.benchmark_train_pipeline --yaml ... 

Config keys (all optional): model {name: dlrm|deepfm, dense_arch, over_arch, embedding_dim}, tables {num, rows, pooling},
run {batch_size, steps, warmup, pipelines: [base, sparse_dist, sparse_dist_lite, fused_sparse_dist, semi_sync, prefetch],
sharding: table_wise|row_wise|column_wise|planner, dense_backend: torch|wgmma}. Prints one JSON line per pipeline."""
from __future__ import annotations

import argparse
import json
import os
import time
from typing import Any, Dict, List

import torch
import torch.distributed as dist

DEFAULT: Dict[str, Any] = {
    "model": {"name": "dlrm", "dense_arch": [64, 32], "over_arch": [64, 1], "embedding_dim": 32},
    "tables": {"num": 8, "rows": 10000, "pooling": 4},
    # sharding: table_wise | row_wise | column_wise | table_row_wise | grid_shard | planner;  compute_kernel: fused | fused_uvm | fused_uvm_caching | key_value
    # (cache_load_factor for the cached kernels);  pipelines: see PIPELINES;  eval_every: N -> an eval forward every N steps (EvalPipelineSparseDist);
    # grad_accumulation: N -> optimizer step every N batches;  mpzch: rows of the zero-collision remapper in front of every table (0 = off)
    "run": {"batch_size": 256, "steps": 10, "warmup": 3, "pipelines": ["base", "sparse_dist"], "sharding": "table_wise", "dense_backend": "torch",
            "compute_kernel": "fused", "cache_load_factor": 0.2, "eval_every": 0, "grad_accumulation": 1, "local_world_size": 0},
}

PIPELINES = {"base": "TrainPipelineBase", "sparse_dist": "TrainPipelineSparseDist", "sparse_dist_lite": "TrainPipelineSparseDistLite",
             "fused_sparse_dist": "TrainPipelineFusedSparseDist", "semi_sync": "TrainPipelineSemiSync", "prefetch": "PrefetchTrainPipelineSparseDist",
             "emb_stash": "TrainPipelineSparseDistEmbStash", "opt_stash": "TrainPipelineSparseDistOptStash", "bwd_opt": "TrainPipelineSparseDistBwdOpt", "prefetch_ems": "TrainPipelinePrefetchEMS"}


def _merge(a: Dict[str, Any], b: Dict[str, Any]) -> Dict[str, Any]:
    out = dict(a)
    for k, v in (b or {}).items():
        out[k] = _merge(a.get(k, {}), v) if isinstance(v, dict) else v
    return out


def build(cfg: Dict[str, Any], device: torch.device, world: int):
    from ..models.deepfm import SimpleDeepFMNN
    from ..models.dlrm import DLRM, DLRMTrain
    from ..modules.embedding_configs import EmbeddingBagConfig
    from ..modules.embedding_modules import EmbeddingBagCollection
    from ..ops import dense as _dense
    from ..optim.apply_optimizer_in_backward import apply_optimizer_in_backward
    from ..optim.keyed import CombinedOptimizer, KeyedOptimizerWrapper
    from ..optim.optimizers import in_backward_optimizer_filter
    from ..optim.rowwise_adagrad import RowWiseAdagrad
    from ..parallel import sharding_plan as sp
    from ..parallel.embeddingbag import EmbeddingBagCollectionSharder
    from ..parallel.model_parallel import DistributedModelParallel
    from ..parallel.types import ShardingPlan

    m, t, r = cfg["model"], cfg["tables"], cfg["run"]
    keys = [f"f{i}" for i in range(t["num"])]
    tables = [EmbeddingBagConfig(name=f"t{i}", embedding_dim=m["embedding_dim"], num_embeddings=t["rows"], feature_names=[keys[i]]) for i in range(t["num"])]
    ebc = EmbeddingBagCollection(tables, device=torch.device("meta"))
    apply_optimizer_in_backward(RowWiseAdagrad, ebc.parameters(), {"lr": 0.01})
    if m["name"] == "dlrm":
        model = DLRMTrain(DLRM(ebc, 13, list(m["dense_arch"]) + [m["embedding_dim"]], list(m["over_arch"]), dense_device=device))
        path = "model.sparse_arch.embedding_bag_collection"
    else:
        class _Train(torch.nn.Module):
            def __init__(self) -> None:
                super().__init__()
                self.model = SimpleDeepFMNN(13, ebc, 64, 16)
                for name, child in self.model.named_children():  # dense parts to the device; the (meta) EBC is materialised by DMP
                    if child is not self.model.sparse_arch:
                        child.to(device)

            def forward(self, batch):
                logits = self.model(batch.dense_features, batch.sparse_features).squeeze(-1)
                loss = torch.nn.functional.binary_cross_entropy(logits, batch.labels.float())
                return loss, (loss.detach(), logits.detach(), batch.labels)

        model, path = _Train(), "model.sparse_arch.embedding_bag_collection"
    if device.type == "cuda":
        _dense.set_dense_backend(r["dense_backend"])
    kernel = r.get("compute_kernel", "fused")
    fused_params = {"cache_load_factor": r.get("cache_load_factor", 0.2)} if kernel in ("fused_uvm_caching", "key_value") else None
    sharder = EmbeddingBagCollectionSharder(fused_params=fused_params)
    local = r.get("local_world_size") or world
    if r["sharding"] == "planner":
        plan = None
        if kernel != "fused":  # constrain the planner to the requested kernel
            from ..parallel.planner import EmbeddingShardingPlanner, Topology
            from ..parallel.planner.types import ParameterConstraints

            cons = {tb.name: ParameterConstraints(compute_kernels=[kernel]) for tb in tables}
            planner = EmbeddingShardingPlanner(topology=Topology(world_size=world, local_world_size=local, compute_device=device.type), batch_size=r["batch_size"], constraints=cons)
            plan = planner.collective_plan(model, [sharder], dist.group.WORLD) if world > 1 else planner.plan(model, [sharder])
    else:
        hosts = max(world // local, 1)
        gen = {"table_wise": lambda i: sp.table_wise(rank=i % world, compute_kernel=kernel), "row_wise": lambda i: sp.row_wise(compute_kernel=kernel),
               "column_wise": lambda i: sp.column_wise(ranks=[(i + j) % world for j in range(min(world, 2))], compute_kernel=kernel) if world > 1 else sp.table_wise(rank=0, compute_kernel=kernel),
               "table_row_wise": lambda i: sp.table_row_wise(host_index=i % hosts, compute_kernel=kernel),
               "grid_shard": lambda i: sp.grid_shard(host_indexes=list(range(hosts)), compute_kernel=kernel) if hosts > 1 else sp.table_row_wise(host_index=0, compute_kernel=kernel)}[r["sharding"]]
        mp = sp.construct_module_sharding_plan(ebc, {tb.name: gen(i) for i, tb in enumerate(tables)}, sharder=sharder, world_size=world, local_size=local, device_type=device.type)
        plan = ShardingPlan({path: mp})
    dmp = DistributedModelParallel(model, device=device, plan=plan, sharders=[sharder])
    dense_opt = KeyedOptimizerWrapper(dict(in_backward_optimizer_filter(dmp.named_parameters())), lambda p: torch.optim.SGD(p, lr=0.01))
    return dmp, CombinedOptimizer([dmp.fused_optimizer, dense_opt]), keys


class _EveryN:
    """Optimizer facade for gradient accumulation: ``step`` / ``zero_grad`` act on every N-th call (gradients of the dense part add up in
    between; the fused embedding optimizer applies per batch, as in the reference's accumulation pipelines)."""

    def __init__(self, opt, n: int) -> None:
        self._opt, self._n, self._k = opt, n, 0

    def zero_grad(self, *a, **kw):
        if self._k % self._n == 0:
            self._opt.zero_grad(*a, **kw)

    def step(self, *a, **kw):
        self._k += 1
        if self._k % self._n == 0:
            return self._opt.step(*a, **kw)
        return None

    def __getattr__(self, name):
        return getattr(self._opt, name)


def run(cfg: Dict[str, Any]) -> List[Dict[str, Any]]:
    from ..datasets.random import RandomRecDataset
    from ..parallel import train_pipeline as tp

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    cuda = torch.cuda.is_available()
    device = torch.device(f"cuda:{int(os.environ.get('LOCAL_RANK', '0'))}") if cuda else torch.device("cpu")
    if cuda:
        torch.cuda.set_device(device)
    if world > 1 and not dist.is_initialized():
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        dist.init_process_group(backend="nccl" if cuda else "gloo")
    r, t = cfg["run"], cfg["tables"]
    from ..parallel.train_pipeline import experimental_pipelines as xp

    classes = {k: getattr(tp, v, None) or getattr(xp, v) for k, v in PIPELINES.items()}
    results = []
    for name in r["pipelines"]:
        dmp, opt, keys = build(cfg, device, world)
        ds = RandomRecDataset(keys, r["batch_size"], hash_sizes=[t["rows"]] * t["num"], ids_per_features=[t["pooling"]] * t["num"], num_dense=13, manual_seed=rank,
                              num_generated_batches=4, pin_memory=cuda)
        batches = ds.batch_generator._generated_batches
        step_opt = opt
        if int(r.get("grad_accumulation", 1)) > 1:  # optimizer step every N batches (the pipelines call .step() / .zero_grad() every batch)
            step_opt = _EveryN(opt, int(r["grad_accumulation"]))
        pipe = classes[name](dmp, step_opt, device)
        eval_pipe = tp.EvalPipelineSparseDist(dmp, opt, device) if int(r.get("eval_every", 0)) > 0 and hasattr(tp, "EvalPipelineSparseDist") else None
        total = r["warmup"] + r["steps"]
        it = iter(batches[i % len(batches)] for i in range(total + 4))
        for _ in range(r["warmup"]):
            pipe.progress(it)
        if cuda:
            torch.cuda.synchronize()
        if world > 1:
            dist.barrier()
        t0 = time.perf_counter()
        for i in range(r["steps"]):
            pipe.progress(it)
            if eval_pipe is not None and (i + 1) % int(r["eval_every"]) == 0:
                dmp.eval()
                with torch.no_grad():
                    eval_pipe.progress(iter([batches[0], batches[1]]))
                dmp.train()
        if cuda:
            torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        res = {"pipeline": name, "ms_per_step": dt / r["steps"] * 1e3, "samples_per_s": r["batch_size"] * world * r["steps"] / dt, "world": world, "device": device.type,
               "sharding": r["sharding"], "batch_size": r["batch_size"]}
        if cuda:
            res["peak_mem_gb"] = torch.cuda.max_memory_allocated(device) / 1e9
        results.append(res)
        if rank == 0:
            print(json.dumps(res))
        # the stashing pipelines park tensors in the process-wide manager: bring them back so the model of this run can be freed
        from ..parallel.memory_stashing import MemoryStashingManager

        MemoryStashingManager.reset()
    return results


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--yaml", type=str, default=None)
    a = ap.parse_args()
    cfg = DEFAULT
    if a.yaml:
        import yaml

        with open(a.yaml) as f:
            cfg = _merge(DEFAULT, yaml.safe_load(f))
    run(cfg)
    if dist.is_initialized():
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
