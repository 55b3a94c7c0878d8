#!/usr/bin/env python
"""Variable-batch-per-feature (VBE) kernels against the eager formulation, ONE GPU.

At ``B`` samples and ``F`` features of width ``D`` (default 32768, 26 x 128 bf16): the inverse-index expansion (``trb_vbe_expand``),
the per-batch CSR build (``trb_vbe_csr``) and the gradient reduce (``trb_vbe_reduce``), for de-duplication ratios ``B_f / B`` of
1.0, 0.25 and 0.02 with Zipf-distributed referrers and for the worst case of one bag referenced by every sample of every feature.
The eager formulation (one ``index_select`` per feature + ``cat`` forward, one ``index_add_`` per feature + ``cat`` backward) is
timed in the same loop, alternating with the kernels. Times are CUDA-event medians over ``--iters`` launches after warm-up; bytes
are the compulsory traffic computed from the shapes (the expansion reads each referenced bag once and writes ``B x sum D``; the
reduce reads ``B x sum D`` and writes every bag). Last, a one-GPU sharded-collection training step on VBE batches (F tables,
fused row-wise Adagrad) through the NVLink-plane path, in blocks of ``--steps`` steps (host clock around a synchronised block)
alternating with the unfused path of such a batch (padding to ``max_f B_f``, routed input dist, separate lookup, eager expansion). One JSON line per measurement; the card and its power limit are read in
the same run.

    python tools/vbe_bench.py [--batch 32768] [--features 26] [--dim 128] [--iters 200] [--out results.jsonl]
"""
import argparse
import json
import os
import subprocess
import sys
import time
import types
from unittest import mock

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from torchrec_b200.ops import vbe as V  # noqa: E402


def card() -> dict:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30).stdout
        name, limit = [x.strip() for x in out.strip().splitlines()[0].split(",")]
    except Exception:
        name, limit = torch.cuda.get_device_name(0), "unknown"
    return {"gpu": name, "power_limit": limit}


def zipf_inverse(F: int, B: int, bags: int, seed: int, dev) -> torch.Tensor:
    """[F, B] inverse indices over ``bags`` bags per feature, P(bag u) ~ 1 / (u + 1)^1.05, bag ids shuffled per feature."""
    g = torch.Generator(device=dev).manual_seed(seed)
    p = 1.0 / torch.arange(1, bags + 1, device=dev, dtype=torch.float64) ** 1.05
    rows = []
    for _ in range(F):
        draw = torch.multinomial(p.float(), B, replacement=True, generator=g)
        rows.append(torch.randperm(bags, device=dev, generator=g)[draw])
    return torch.stack(rows)


def eager_reduce(grad: torch.Tensor, inv: torch.Tensor, dims, S: int) -> torch.Tensor:
    outs, c = [], 0
    for r, d in enumerate(dims):
        outs.append(torch.zeros(S, d, dtype=grad.dtype, device=grad.device).index_add_(0, inv[r], grad[:, c : c + d]))
        c += d
    return torch.cat(outs, 1)


def time_alternating(fns: dict, iters: int, warm: int = 10) -> dict:
    """Median CUDA-event time (ms) of every callable, launched in turn ``iters`` times."""
    for _ in range(warm):
        for fn in fns.values():
            fn()
    torch.cuda.synchronize()
    events = {k: [] for k in fns}
    for _ in range(iters):
        for k, fn in fns.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            events[k].append((e0, e1))
    torch.cuda.synchronize()
    return {k: sorted(a.elapsed_time(b) for a, b in v)[len(v) // 2] for k, v in events.items()}


def kernel_cases(a, emit) -> None:
    dev = torch.device("cuda:0")
    B, F, D = a.batch, a.features, a.dim
    dtype = torch.bfloat16
    esz = 2
    names = [f"f{i}" for i in range(F)]
    dims = [D] * F
    C = F * D
    pooled = torch.randn(B, C, device=dev).to(dtype)
    grad = torch.randn(B, C, device=dev).to(dtype)
    cases = [(f"ratio_{r}", zipf_inverse(F, B, max(1, int(r * B)), 1, dev)) for r in (1.0, 0.25, 0.02)]
    cases.append(("hot_bag", torch.zeros(F, B, dtype=torch.int64, device=dev)))
    for case, inv in cases:
        index = V.VbeIndex((names, inv), names, dims, src_rows=B)
        table = index.kernels_serve(pooled)
        assert table is not None
        index.csr()
        ctx = types.SimpleNamespace(index=index, table=table)
        seg = index.csr()[0]
        lens = (seg[1:] - seg[:-1])
        with torch.no_grad():
            assert torch.equal(V.vbe_expand(pooled, index), V.expand_eager(pooled, (names, inv), names, dims))
            t = time_alternating({
                "expand": lambda: V.vbe_expand(pooled, index),
                "expand_eager": lambda: V.expand_eager(pooled, (names, inv), names, dims),
                "csr": lambda: V.VbeIndex((names, inv), names, dims, src_rows=B).csr(),
                "reduce": lambda: V._VbeExpandFn.backward(ctx, grad),
                "reduce_eager": lambda: eager_reduce(grad, inv, dims, B),
            }, a.iters)
        n = F * B
        distinct = int((lens > 0).sum())  # pooled row blocks the expansion has to read: the bags somebody references
        nbytes = {
            "expand": (B * C + distinct * D) * esz + n * 8, "expand_eager": (B * C + distinct * D) * esz + n * 8,
            "csr": n * 8 + n * 4 + (n + 1) * 4,
            "reduce": 2 * B * C * esz + n * 4 + (n + 1) * 4, "reduce_eager": 2 * B * C * esz + n * 8,
        }
        for k, ms in t.items():
            emit({"case": case, "op": k, "ms": round(ms, 4), "bytes": nbytes[k], "GBps": round(nbytes[k] / ms / 1e6, 1), "B": B, "F": F, "D": D, "dtype": "bf16",
                  "referenced_bags": distinct, "max_referrers": int(lens.max()), "long_segments": int((lens > 256).sum())})


def training_step(a, emit) -> None:
    from torchrec_b200.modules.embedding_configs import EmbeddingBagConfig
    from torchrec_b200.modules.embedding_modules import EmbeddingBagCollection
    from torchrec_b200.optim.apply_optimizer_in_backward import apply_optimizer_in_backward
    from torchrec_b200.optim.rowwise_adagrad import RowWiseAdagrad
    from torchrec_b200.parallel import sharding_plan as sp
    from torchrec_b200.parallel.embeddingbag import EmbeddingBagCollectionSharder
    from torchrec_b200.parallel.model_parallel import DistributedModelParallel
    from torchrec_b200.parallel.types import ShardingPlan
    from torchrec_b200.sparse.jagged_tensor import KeyedJaggedTensor

    dev = torch.device("cuda:0")
    B, F, D, rows, ratio = a.batch, a.features, a.dim, 100_000, 0.25
    bags = max(1, int(ratio * B))
    keys = [f"f{i}" for i in range(F)]
    ebc = EmbeddingBagCollection([EmbeddingBagConfig(name=f"t{i}", embedding_dim=D, num_embeddings=rows, feature_names=[keys[i]]) for i in range(F)],
                                 device=torch.device("meta"))
    apply_optimizer_in_backward(RowWiseAdagrad, ebc.parameters(), {"lr": 0.05})
    plan = sp.construct_module_sharding_plan(ebc, {f"t{i}": sp.table_wise(rank=0) for i in range(F)}, sharder=EmbeddingBagCollectionSharder(), world_size=1,
                                             local_size=1, device_type="cuda")

    class Wrap(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.ebc = ebc

        def forward(self, k):
            return self.ebc(k).values()

    dmp = DistributedModelParallel(Wrap(), device=dev, plan=ShardingPlan({"ebc": plan}), sharders=[EmbeddingBagCollectionSharder()])
    g = torch.Generator(device=dev).manual_seed(2)
    lengths = torch.randint(1, 4, (F * bags,), device=dev, generator=g)
    values = torch.randint(0, rows, (int(lengths.sum()),), device=dev, generator=g)
    kjt = KeyedJaggedTensor(keys=keys, values=values, lengths=lengths, stride_per_key_per_rank=[[bags]] * F,
                            inverse_indices=(keys, zipf_inverse(F, B, bags, 3, dev)))
    grad = torch.randn(B, F * D, device=dev)
    sharded = dmp.module.ebc

    def block() -> float:
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(a.steps):
            dmp(kjt).backward(grad)
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) / a.steps * 1e3

    # the unfused path of a VBE batch on the same module: padded to max_f B_f, routed input dist, separate lookup, collective-shaped
    # output dist, per-name index_select expansion
    former = (mock.patch.object(type(sharded), "_plane_serves", lambda self, B: False),
              mock.patch.object(type(sharded._engine), "fused_available", lambda self, spr: False),
              mock.patch.object(V.VbeIndex, "kernels_serve", lambda self, pooled: None))
    times = {"plane + vbe kernels": [], "unfused path (eager expansion)": []}
    for rnd in range(4):  # alternating blocks; the first round warms both paths up and is dropped
        t = block()
        with former[0], former[1], former[2]:
            t_old = block()
        if rnd:
            times["plane + vbe kernels"].append(t)
            times["unfused path (eager expansion)"].append(t_old)
    for k, v in times.items():
        emit({"case": f"sharded_ebc_step_ratio_{ratio}", "op": f"forward+backward, fused row-wise Adagrad: {k}", "ms": round(sorted(v)[len(v) // 2], 3),
              "ms_blocks": [round(x, 3) for x in v], "B": B, "F": F, "D": D, "rows_per_table": rows, "bags_per_feature": bags, "ids": int(values.numel()),
              "dtype": "fp32", "steps_per_block": a.steps})


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32768)
    ap.add_argument("--features", type=int, default=26)
    ap.add_argument("--dim", type=int, default=128)
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--steps", type=int, default=400)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("vbe_bench.py measures on a GPU and found none")
    hw = card()
    sink = open(a.out, "w") if a.out else None

    def emit(rec: dict) -> None:
        line = json.dumps({**rec, **hw})
        print(line, flush=True)
        if sink:
            sink.write(line + "\n")

    kernel_cases(a, emit)
    training_step(a, emit)
    if sink:
        sink.close()


if __name__ == "__main__":
    main()
