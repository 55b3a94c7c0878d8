#!/usr/bin/env python
"""Single-process NVLink microbenchmark of the sparse plane's peer kernels (what `ncu` can attach to: one process, two GPUs).

Virtual rank 0 lives on cuda:0, virtual rank 1's symmetric buffers on cuda:1 (peer access enabled): rank 0's fused lookup + output
dist and its gradient push store half of their rows over NVLink exactly like in a 2-process job. Reports time, bytes stored into the
peer and GB/s for
    fwd_fused   tbe_pooled_fwd with [local, peer] destinations      fwd_local   same lookup, both destinations local
    push        trb_grad_push into [local, peer] inboxes            copy        torch peer copy of the same number of bytes (reference)
    decode_out  FP8 out slot -> wire dtype (fp8 wire only)          decode_in   FP8 gradient inbox -> wire dtype (fp8 wire only)

``--wire bf16,fp8`` runs the plane with each wire in turn (fp8: the FP8 row-wise quantized-comms codec, row dim ``--row-dim``),
alternating them ``--repeats`` times; bytes are what is actually stored into the peer (payload + scales for fp8). With one GPU
(``--loopback``) both virtual ranks live on cuda:0: the numbers are then the cost of the quantizing stores and of the decode passes,
not an NVLink effect.

    python tools/peer_bench.py [--tables 13] [--batch 32768] [--dim 128] [--iters 20] [--only fwd_fused] [--wire bf16,fp8] [--loopback]
"""
import argparse
import gc
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from torchrec_b200.modules.embedding_configs import EmbeddingBagConfig  # noqa: E402
from torchrec_b200.modules.embedding_modules import EmbeddingBagCollection  # noqa: E402
from torchrec_b200.ops.tbe import OptimType  # noqa: E402
from torchrec_b200.parallel import sharding_plan as sp  # noqa: E402
from torchrec_b200.parallel.embeddingbag import EmbeddingBagCollectionSharder  # noqa: E402
from torchrec_b200.parallel.engine import OptimizerSpec, ShardedLookupEngine  # noqa: E402
from torchrec_b200.parallel.qcomm_codec import CommType, QCommsConfig, get_qcomm_codecs  # noqa: E402
from torchrec_b200.parallel.sparse_plane import LoopbackGroup  # noqa: E402
from torchrec_b200.parallel.types import ShardingEnv  # noqa: E402
from torchrec_b200.sparse.jagged_tensor import KeyedJaggedTensor  # noqa: E402


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--tables", type=int, default=13, help="tables owned by rank 0 (rank 1 owns as many)")
    ap.add_argument("--rows", type=int, default=4_000_000)
    ap.add_argument("--batch", type=int, default=32768)
    ap.add_argument("--dim", type=int, default=128)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--only", type=str, default="")
    ap.add_argument("--wire", type=str, default="bf16,fp8", help="comma-separated wires to alternate: bf16 | fp8")
    ap.add_argument("--row-dim", type=int, default=32)
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--loopback", action="store_true", help="both virtual ranks on cuda:0 (one GPU: no NVLink traffic)")
    a = ap.parse_args()
    if not a.loopback:
        assert torch.cuda.device_count() >= 2, "needs 2 GPUs in one process (or --loopback)"
    d0 = torch.device("cuda:0")
    d1 = d0 if a.loopback else torch.device("cuda:1")
    torch.cuda.set_device(d0)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().splitlines()
    print(f"cards: {q}  mode: {'loopback on cuda:0 (NVLink effect not measured)' if a.loopback else 'rank 1 on cuda:1 over NVLink'}")
    W, T, B, D = 2, a.tables, a.batch, a.dim
    tables = [EmbeddingBagConfig(name=f"t{i}", embedding_dim=D, num_embeddings=a.rows if i % 2 == 0 else 5000, feature_names=[f"f{i}"]) for i in range(2 * T)]
    ebc = EmbeddingBagCollection(tables=tables, device=torch.device("meta"))
    plan = sp.construct_module_sharding_plan(ebc, {t.name: sp.table_wise(rank=i // T) for i, t in enumerate(tables)}, sharder=EmbeddingBagCollectionSharder(),
                                             world_size=W, local_size=W, device_type="cuda")
    names = [f"f{i}" for i in range(2 * T)]
    g = torch.Generator().manual_seed(0)
    vals = torch.cat([torch.randint(0, t.num_embeddings, (B,), generator=g) for t in tables])
    total_cols = 2 * T * D
    grad = torch.randn(B, total_cols, device=d0).to(torch.bfloat16)

    def make(wire):
        codecs = get_qcomm_codecs(QCommsConfig(forward_precision=CommType.FP8, backward_precision=CommType.FP8, fp8_quantize_dim=a.row_dim)) if wire == "fp8" else None
        group = LoopbackGroup(W, d0, peer_devices=[d0, d1])
        opt = {t.name: OptimizerSpec(optim=OptimType.EXACT_ROWWISE_ADAGRAD) for t in tables}
        eng = ShardedLookupEngine(tables, names, list(range(2 * T)), plan, ShardingEnv.from_loopback(W, 0, group), d0, pooled=True, is_weighted=False,
                                  opt_specs=opt, output_dtype=torch.bfloat16, qcomm_codecs=codecs)
        # rank 1's engine only exists to make the "collective" allocations (its buffers live on cuda:1)
        with torch.cuda.device(d1):
            eng1 = ShardedLookupEngine(tables, names, list(range(2 * T)), plan, ShardingEnv.from_loopback(W, 1, group), d1, pooled=True, is_weighted=False,
                                       opt_specs=opt, output_dtype=torch.bfloat16, qcomm_codecs=codecs)
        kjt = KeyedJaggedTensor(keys=names, values=vals.to(d0), lengths=torch.ones(2 * T * B, dtype=torch.int64, device=d0), stride=B)
        ids0 = eng.plane_input_dist(kjt, None, total_cols, capacity=T * B + 64)
        with torch.cuda.device(d1):
            kjt1 = KeyedJaggedTensor(keys=names, values=vals.to(d1), lengths=torch.ones(2 * T * B, dtype=torch.int64, device=d1), stride=B)
            eng1.plane_input_dist(kjt1, None, total_cols, capacity=T * B + 64)  # fills rank 0's regions for source 1 (peer stores 1 -> 0)
        torch.cuda.synchronize(d0)
        torch.cuda.synchronize(d1)
        pl = ids0.plane
        assert (pl.wire_format["fwd"] is not None) == (wire == "fp8"), pl.wire_format
        # bytes stored into the peer: rank 0's T tables x the B samples of rank 1 (forward), the gradient columns of rank 1's T tables
        # for rank 0's B samples (push); fp8 = 1 byte per element + one fp32 scale per row_dim elements
        per_elem = 1 + 4 / a.row_dim if wire == "fp8" else 2
        remote = int(B * T * D * per_elem)
        return pl, pl.regions(ids0.slot), remote, (eng, eng1)

    wires = [w for w in a.wire.split(",") if w]
    for rep_i in range(a.repeats):
        for wire in wires:
            pl, reg, remote, _keep = make(wire)
            src = torch.empty(remote, dtype=torch.uint8, device=d0)
            dst = torch.empty(remote, dtype=torch.uint8, device=d1)
            cases = {
                "fwd_fused": (lambda: pl._forward_kernels(reg, 0), remote),
                "fwd_local": (lambda: pl._forward_kernels(reg, 0, local_only=True), 0),
                "push": (lambda: pl._push_kernels(grad), remote),
                "copy": (lambda: dst.copy_(src, non_blocking=True), remote),
            }
            if wire == "fp8":
                cases["decode_out"] = (lambda: pl._decode_out(0), 0)
                cases["decode_in"] = (lambda: pl._decode_inbox(), 0)
            for name, (fn, nbytes) in cases.items():
                if a.only and a.only != name:
                    continue
                for _ in range(3):
                    fn()
                torch.cuda.synchronize(d0)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(a.iters):
                    fn()
                e1.record()
                torch.cuda.synchronize(d0)
                ms = e0.elapsed_time(e1) / a.iters
                rate = f"{nbytes / (ms * 1e-3) / 1e9:7.1f} GB/s to the peer" if nbytes else ""
                print(f"run {rep_i} wire {wire:4s} {name:10s} {ms * 1e3:8.1f} us   peer bytes {nbytes / 1e6:7.1f} MB   {rate}")
            del pl, reg, _keep, cases, src, dst
            gc.collect()
            torch.cuda.empty_cache()

if __name__ == "__main__":
    main()
