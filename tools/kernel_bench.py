#!/usr/bin/env python
"""Per-kernel roofline table of the sparse / quantized / codec / jagged kernels at the DLRM headline shapes, ONE GPU.

Every peer kernel runs in loopback (W virtual ranks, all symmetric buffers on this device), so the numbers are the HBM side of the
kernels; the NVLink side is `tools/peer_bench.py` (2 GPUs, one process) and `bench.py --measure-comm` (N processes).
For each case: device time (CUDA events, L2 flushed before every iteration, median), the bytes the kernel has to move by its own
definition (compulsory traffic), GB/s, and the fraction of the device-to-device copy bandwidth measured at start-up on this GPU.

    python tools/kernel_bench.py [--batch 32768] [--iters 15] [--only tbe_fwd] [--md kernel_roofline.md]
"""
import argparse
import gc
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from torchrec_b200.modules.embedding_configs import DataType, EmbeddingBagConfig  # noqa: E402
from torchrec_b200.modules.embedding_modules import EmbeddingBagCollection  # noqa: E402
from torchrec_b200.ops.tbe import OptimType  # noqa: E402
from torchrec_b200.parallel import sharding_plan as sp  # noqa: E402
from torchrec_b200.parallel.embeddingbag import EmbeddingBagCollectionSharder  # noqa: E402
from torchrec_b200.parallel.engine import OptimizerSpec, ShardedLookupEngine  # noqa: E402
from torchrec_b200.parallel.sparse_plane import LoopbackGroup  # noqa: E402
from torchrec_b200.parallel.types import ShardingEnv  # noqa: E402
from torchrec_b200.sparse.jagged_tensor import KeyedJaggedTensor  # noqa: E402

CRITEO = [39884406, 39043, 17289, 7420, 20263, 3, 7120, 1543, 63, 38532951, 2953546, 403346, 10, 2208, 11938, 155, 4, 976, 14,
          39979771, 25641295, 39664984, 585935, 12972, 108, 36]


def copy_gbs(dev: torch.device, nbytes: int = 2 << 30, iters: int = 10) -> float:
    """Device-to-device copy bandwidth (read + write bytes per second), median of ``iters`` CUDA-event timed copies."""
    src = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    dst = torch.empty_like(src)
    for _ in range(3):
        dst.copy_(src)
    ts = []
    for _ in range(iters):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        dst.copy_(src)
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) * 1e-3)
    del src, dst
    torch.cuda.empty_cache()
    return 2.0 * nbytes / sorted(ts)[len(ts) // 2] / 1e9


class Bench:
    def __init__(self, a) -> None:
        self.a = a
        self.dev = torch.device("cuda:0")
        self.flush = None if a.no_flush else torch.empty(256 << 20, dtype=torch.uint8, device=self.dev)
        self.rows = []
        self.hbm = copy_gbs(self.dev)
        print(f"{torch.cuda.get_device_name(self.dev)}: device-to-device copy {self.hbm:.0f} GB/s", flush=True)

    def run(self, name: str, fn, nbytes: float, note: str = "") -> None:
        if self.a.only and self.a.only not in name:
            return
        for _ in range(self.a.warm):
            fn()
        torch.cuda.synchronize()
        ts = []
        for _ in range(self.a.iters):
            if self.flush is not None:
                self.flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1) * 1e3)
        us = sorted(ts)[len(ts) // 2]
        gbs = nbytes / (us * 1e-6) / 1e9
        self.rows.append((name, us, nbytes / 1e6, gbs, 100.0 * gbs / self.hbm, note))
        print(f"{name:34s} {us:9.1f} us  {nbytes / 1e6:9.1f} MB  {gbs:8.1f} GB/s  {100.0 * gbs / self.hbm:5.1f} % of copy bw   {note}", flush=True)


def engine(tables, names, plan, env, dev, out_dtype=torch.bfloat16):
    return ShardedLookupEngine(tables, names, list(range(len(tables))), plan, env, dev, pooled=True, is_weighted=False,
                               opt_specs={t.name: OptimizerSpec(optim=getattr(OptimType, os.environ.get("KB_OPT", "EXACT_ROWWISE_ADAGRAD"))) for t in tables}, output_dtype=out_dtype)


def sparse_cases(bn: Bench) -> None:
    a, dev = bn.a, bn.dev
    B, D = a.batch, 128
    rows = [min(r, a.row_cap) for r in CRITEO]
    F = len(rows)
    tables = [EmbeddingBagConfig(name=f"t{i}", embedding_dim=D, num_embeddings=r, feature_names=[f"f{i}"]) for i, r in enumerate(rows)]
    names = [f"f{i}" for i in range(F)]
    ebc = EmbeddingBagCollection(tables=tables, device=torch.device("meta"))
    g = torch.Generator().manual_seed(0)
    vals = torch.cat([torch.randint(0, r, (B,), generator=g) for r in rows]).to(dev)
    kjt = KeyedJaggedTensor(keys=names, values=vals, lengths=torch.ones(F * B, dtype=torch.int64, device=dev), stride=B)
    N = F * B
    uniq = sum(int(torch.unique(vals[i * B : (i + 1) * B]).numel()) for i in range(F))

    # ---- one rank (the N=1 bench path: SingleRankGroup) ----
    plan = sp.construct_module_sharding_plan(ebc, {t.name: sp.table_wise(rank=0) for t in tables}, sharder=EmbeddingBagCollectionSharder(),
                                             world_size=1, local_size=1, device_type="cuda")
    eng = engine(tables, names, plan, ShardingEnv.from_local(1, 0), dev)
    ids = eng.plane_input_dist(kjt, None, F * D, capacity=N + 64, training=False)
    pl = ids.plane
    reg = pl.regions(ids.slot)
    isz = vals.element_size()
    bn.run("kjt_route (len + scan + write) W=1", lambda: pl.push_input(kjt.offsets(), kjt.values(), None, 1, training=False), 2.0 * N * (isz + 4),
           "ids + offsets read once, written once")
    ids = pl.push_input(kjt.offsets(), kjt.values(), None, 1, training=False)
    reg = pl.regions(ids.slot)
    bn.run("tbe_pooled_fwd fp32 rows -> bf16", lambda: pl._forward_kernels(reg, 0), N * D * (4 + 2) + N * isz,
           f"{N} rows x 512 B gathered, bf16 pooled rows stored")
    grad = torch.randn(B, F * D, device=dev).to(torch.bfloat16)
    bn.run("tbe_bwd phase 1 (keys + radix sort)", lambda: pl._backward_kernels(reg, ids.slot, 1.0, phase=1), N * (isz + 8 + 8 + 4 + 4),
           "id read, 64-bit key + payload through the sort passes (lower bound: one pass)")
    pl._backward_kernels(reg, ids.slot, 1.0, phase=1)
    bn.run("tbe_bwd phase 2 (rowwise adagrad)", lambda: pl._backward_kernels(reg, ids.slot, 1.0, phase=2, grad=grad),
           N * D * 2 + uniq * (2 * D * 4 + 8), f"{N} bf16 grad rows read, {uniq} unique rows read-modify-written (+ 4 B state each way)")

    # ---- 4 virtual ranks: routing with destinations, staged (row-wise) reduce, gradient push ----
    W = 4
    del eng, pl
    torch.cuda.empty_cache()
    small = [EmbeddingBagConfig(name=f"s{i}", embedding_dim=D, num_embeddings=min(r, 2_000_000), feature_names=[f"f{i}"]) for i, r in enumerate(rows)]
    ebc2 = EmbeddingBagCollection(tables=small, device=torch.device("meta"))
    per = {t.name: (sp.row_wise() if i == 0 else sp.table_wise(rank=i % W)) for i, t in enumerate(small)}
    plan2 = sp.construct_module_sharding_plan(ebc2, per, sharder=EmbeddingBagCollectionSharder(), world_size=W, local_size=W, device_type="cuda")
    group = LoopbackGroup(W, dev)
    engs = [engine(small, names, plan2, ShardingEnv.from_loopback(W, r, group), dev) for r in range(W)]
    vals2 = torch.cat([torch.randint(0, t.num_embeddings, (B,), generator=g) for t in small]).to(dev)
    kjt2 = KeyedJaggedTensor(keys=names, values=vals2, lengths=torch.ones(N, dtype=torch.int64, device=dev), stride=B)
    rids = [e.plane_input_dist(kjt2, None, F * D, capacity=N + 64, training=False) for e in engs]
    p0 = rids[0].plane
    bn.run(f"kjt_route W={W} (1 RW + 25 TW units)", lambda: p0.push_input(kjt2.offsets(), kjt2.values(), None, 1, training=False), 2.0 * N * (isz + 4),
           "destinations are the 4 virtual ranks' id regions")
    grad2 = torch.randn(B, F * D, device=dev).to(torch.bfloat16)
    bn.run(f"trb_grad_push W={W} (persistent, 2 CTA/SM)", lambda: p0._push_kernels(grad2), 2.0 * B * F * D * 2, "bf16 [B, 3328] read, column slices stored to the owners' inboxes")
    if p0.has_staged:
        bn.run(f"trb_staging_reduce_cols W={W}", lambda: p0._staging_reduce(0), (W + 1) * B * p0.staged_width * 2, "row-wise partial sums of W sources -> output columns")


def n8_rank_cases(bn: Bench) -> None:
    """What the busiest rank of the 8-GPU DLRM job runs locally: 4 of the large tables, the GLOBAL batch (8 x 32768 samples), every id
    a different row (no duplicates to merge) - the backward is a pure random 512 B read-modify-write stream."""
    a, dev = bn.a, bn.dev
    B, D, F = 8 * a.batch, 128, 4
    rows = [min(r, a.row_cap) for r in (39884406, 38532951, 39979771, 39664984)]
    tables = [EmbeddingBagConfig(name=f"t{i}", embedding_dim=D, num_embeddings=r, feature_names=[f"f{i}"]) for i, r in enumerate(rows)]
    names = [f"f{i}" for i in range(F)]
    ebc = EmbeddingBagCollection(tables=tables, device=torch.device("meta"))
    g = torch.Generator().manual_seed(0)
    vals = torch.cat([torch.randint(0, r, (B,), generator=g) for r in rows]).to(dev)
    kjt = KeyedJaggedTensor(keys=names, values=vals, lengths=torch.ones(F * B, dtype=torch.int64, device=dev), stride=B)
    N = F * B
    uniq = sum(int(torch.unique(vals[i * B : (i + 1) * B]).numel()) for i in range(F))
    plan = sp.construct_module_sharding_plan(ebc, {t.name: sp.table_wise(rank=0) for t in tables}, sharder=EmbeddingBagCollectionSharder(),
                                             world_size=1, local_size=1, device_type="cuda")
    eng = engine(tables, names, plan, ShardingEnv.from_local(1, 0), dev)
    ids = eng.plane_input_dist(kjt, None, F * D, capacity=N + 64, training=False)
    pl = ids.plane
    reg = pl.regions(ids.slot)
    isz = vals.element_size()
    bn.run(f"N=8 busiest rank: tbe_pooled_fwd (4 x {rows[0] // 1_000_000}M-row tables, {B} samples)", lambda: pl._forward_kernels(reg, 0), N * D * (4 + 2) + N * isz,
           f"{N} rows x 512 B gathered")
    grad = torch.randn(B, F * D, device=dev).to(torch.bfloat16)
    pl._backward_kernels(reg, ids.slot, 1.0, phase=1)
    bn.run("N=8 busiest rank: tbe_bwd phase 2 (all ids distinct)", lambda: pl._backward_kernels(reg, ids.slot, 1.0, phase=2, grad=grad),
           N * D * 2 + uniq * (2 * D * 4 + 8), f"{uniq} unique rows read-modify-written")
    del eng, pl
    torch.cuda.empty_cache()


def quant_cases(bn: Bench) -> None:
    from torchrec_b200.ops.quant_tbe import QuantTableBatchedEmbeddingBags

    dev, B, D = bn.dev, bn.a.batch, 128
    rows = [min(r, 4_000_000) for r in CRITEO]
    F = len(rows)
    g = torch.Generator().manual_seed(1)
    idx = torch.cat([torch.randint(0, r, (B,), generator=g) for r in rows]).to(dev).to(torch.int32)
    off = torch.arange(F * B + 1, dtype=torch.int32, device=dev)
    for dt, label in ((DataType.INT8, "int8 rows"), (DataType.FP8, "fp8 block-scaled rows"), (DataType.INT4, "int4 rows"), (DataType.FP16, "fp16 rows")):
        q = QuantTableBatchedEmbeddingBags([(f"t{i}", r, D, dt) for i, r in enumerate(rows)], output_dtype=torch.bfloat16, device=dev)
        q.weights.random_(0, 255)
        rb = q._row_bytes[0]
        bn.run(f"qtbe_fwd {label} -> bf16", lambda q=q: q(idx, off, None, B), F * B * (rb + D * 2 + 4), f"{rb} B rows")
        del q


def codec_cases(bn: Bench) -> None:
    from torchrec_b200.parallel.qcomm_codec import CommType, get_qcomm_codec

    dev, B = bn.dev, bn.a.batch
    x = torch.randn(B, 26 * 128, device=dev)
    for ct in (CommType.FP8, CommType.INT8, CommType.MX4):
        try:
            c = get_qcomm_codec(ct, None, 128, True)
            y = c.encode(x)
            bn.run(f"qcomm encode fp32 -> {ct.name}", lambda c=c: c.encode(x), x.numel() * 4 + y.numel() * y.element_size())
            bn.run(f"qcomm decode {ct.name} -> fp32", lambda c=c, y=y: c.decode(y), x.numel() * 4 + y.numel() * y.element_size())
        except Exception as e:  # pragma: no cover
            print(f"codec {ct}: {e}")


def jagged_cases(bn: Bench) -> None:
    from torchrec_b200.ops import jagged as J

    dev = bn.dev
    Bj, maxL, D = 65536, 32, 64
    lengths = torch.randint(0, maxL + 1, (Bj,), device=dev)
    offs = torch.zeros(Bj + 1, dtype=torch.int64, device=dev)
    offs[1:] = lengths.cumsum(0)
    L = int(offs[-1])
    v = torch.randn(L, D, device=dev)
    bn.run("jagged_to_padded_dense", lambda: J.jagged_to_padded_dense(v, [offs], [maxL], 0.0), L * D * 4 + Bj * maxL * D * 4)
    dense = J.jagged_to_padded_dense(v, [offs], [maxL], 0.0)
    bn.run("dense_to_jagged", lambda: J.dense_to_jagged(dense, [offs], L), 2.0 * L * D * 4)
    T, Bk = 26, 32768
    ln = torch.randint(0, 3, (T * Bk,), device=dev)
    vals = torch.randint(0, 1 << 20, (int(ln.sum()),), device=dev)
    perm = torch.randperm(T, device=dev).to(torch.int32)
    nv = int(vals.numel())
    bn.run("permute_2D_sparse_data", lambda: J.permute_2D_sparse_data(perm, ln.view(T, Bk), vals, None, nv), 2.0 * (vals.numel() * 8 + T * Bk * 8))
    bsz = torch.full((T,), (1 << 20) // 8 + 1, dtype=torch.int64, device=dev)
    bn.run("block_bucketize_sparse_features W=8", lambda: J.block_bucketize_sparse_features(ln, vals, False, True, bsz, 8), 2.0 * (vals.numel() * 8 + T * Bk * 8) + vals.numel() * 8)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32768)
    ap.add_argument("--row-cap", type=int, default=20_000_000)
    ap.add_argument("--iters", type=int, default=15)
    ap.add_argument("--only", type=str, default="")
    ap.add_argument("--no-flush", action="store_true")
    ap.add_argument("--warm", type=int, default=2)
    ap.add_argument("--skip", type=str, default="")
    ap.add_argument("--md", type=str, default="")
    a = ap.parse_args()
    torch.cuda.set_device(0)
    bn = Bench(a)
    for nm, fn in (("sparse", sparse_cases), ("n8rank", n8_rank_cases), ("quant", quant_cases), ("codec", codec_cases), ("jagged", jagged_cases)):
        if nm in a.skip.split(","):
            continue
        try:
            fn(bn)
        except Exception as e:  # keep going: one family failing must not lose the others' numbers
            import traceback

            traceback.print_exc()
            print(f"[{nm}] failed: {e}", flush=True)
        gc.collect()  # the engines of a family hold reference cycles: free their tables before the next family allocates
        torch.cuda.empty_cache()
    if a.md:
        with open(a.md, "w") as f:
            f.write(f"| kernel (DLRM shapes, batch {a.batch}, 26 x dim 128) | us | compulsory MB | GB/s | % of measured copy bw ({bn.hbm:.0f} GB/s, {torch.cuda.get_device_name(bn.dev)}) | bytes counted |\n|---|---|---|---|---|---|\n")
            for name, us, mb, gbs, pct, note in bn.rows:
                f.write(f"| `{name}` | {us:.1f} | {mb:.1f} | {gbs:.0f} | {pct:.1f} | {note} |\n")


if __name__ == "__main__":
    main()
