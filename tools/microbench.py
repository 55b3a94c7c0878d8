"""Per-op micro-benchmarks on one H100 (CUDA events, L2 flushed between iterations, median of N).
Usage: python tools/microbench.py [gemm] [interaction] [tbe]   -> prints markdown tables."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from torchrec_b200.ops import gemm as G  # noqa: E402
from torchrec_b200.ops import interaction as I  # noqa: E402
from torchrec_b200.ops import tbe as T  # noqa: E402

dev = torch.device("cuda:0")
_flush = None


def timeit(fn, iters=15, warm=3):
    global _flush
    if _flush is None:
        _flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    for _ in range(warm):
        fn()
    ts = []
    for _ in range(iters):
        _flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) * 1e3)
    ts.sort()
    return ts[len(ts) // 2]


def bench_gemm():
    print("| GEMM (M,N,K) | layout | us | TFLOP/s |\n|---|---|---|---|")
    M = 32768
    for (N, K) in [(1024, 480), (1024, 1024), (512, 1024), (256, 512), (512, 16), (256, 512), (128, 256)]:
        a = torch.randn(M, max(K, 8), device=dev).bfloat16()
        w = torch.randn(N, max(K, 8), device=dev).bfloat16()
        bias = torch.zeros(N, device=dev)
        us = timeit(lambda: G.gemm_bf16(a, w, bias=bias, act=G.ACT_RELU))
        print(f"| {M},{N},{K} | fwd (K-major) | {us:.1f} | {2 * M * N * K / us / 1e6:.0f} |")
        gy = torch.randn(M, N, device=dev).bfloat16()
        wt = w  # dgrad: gy [M,N] @ w [N,K] -> [M,K]; b consumed MN-major
        if K % 8 == 0 and K >= 64:
            us = timeit(lambda: G.gemm_bf16(gy, wt, b_mn=True))
            print(f"| {M},{K},{N} | dgrad (B MN-major) | {us:.1f} | {2 * M * N * K / us / 1e6:.0f} |")
            sp, tn = G._wgrad_plan(N, a.shape[1], M, torch.cuda.get_device_properties(dev).multi_processor_count)
            us = timeit(lambda: G.gemm_bf16(gy, a, a_mn=True, b_mn=True, out_dtype=torch.float32, split_k=sp, tile_n=tn))
            print(f"| {N},{K},{M} | wgrad (A,B MN-major, split-K {sp}, tile_n {tn}) | {us:.1f} | {2 * M * N * K / us / 1e6:.0f} |")


def bench_gemmx():
    """Mainloop vs epilogue: sweep K at fixed M, N."""
    print("| M,N,K | variant | us | TFLOP/s |\n|---|---|---|---|")
    M, N = 32768, 1024
    for K in (512, 1024, 2048, 4096):
        a = torch.randn(M, K, device=dev).bfloat16()
        w = torch.randn(N, K, device=dev).bfloat16()
        wt = w.t().contiguous()
        bias = torch.zeros(N, device=dev)
        out = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
        mask = torch.randn(M, N, device=dev).bfloat16()
        for name, fn in [
            ("K-major B, bias+relu", lambda: G.gemm_bf16(a, w, bias=bias, act=G.ACT_RELU, out=out)),
            ("K-major B, plain", lambda: G.gemm_bf16(a, w, out=out)),
            ("MN-major B, plain", lambda: G.gemm_bf16(a, wt, b_mn=True, out=out)),
            ("MN-major B, relu-grad mask", lambda: G.gemm_bf16(a, wt, b_mn=True, out=out, act=G.ACT_RELU_GRAD, mask=mask)),
        ]:
            us = timeit(fn)
            print(f"| {M},{N},{K} | {name} | {us:.1f} | {2 * M * N * K / us / 1e6:.0f} |")


def bench_colsum():
    print("| colsum bf16 [32768, N] | us | GB/s |\n|---|---|---|")
    tot = 0.0
    tiny = torch.zeros(8, device=dev)
    print(f"| (timing floor: one tiny kernel) | {timeit(lambda: tiny.add_(1.0)):.1f} | |")
    for N in (1024, 1024, 512, 256, 512, 256, 128):
        x = torch.randn(32768, N, device=dev).bfloat16()
        us = timeit(lambda: G.colsum_bf16(x))
        tot += us
        ref = x.float().sum(0)
        err = (G.colsum_bf16(x) - ref).abs().max().item()
        print(f"| {N} | {us:.1f} | {x.numel() * 2 / us / 1e3:.0f} | err {err:.3f}")
    print(f"| total (the 7 bias gradients of one DLRM step) | {tot:.1f} | |")


INTERACTION_SHAPES = [(16, 26), (32, 26), (32, 40), (48, 26), (64, 8), (64, 26), (64, 40), (96, 26), (128, 15), (128, 26), (128, 31),
                      (128, 63), (128, 100), (192, 26), (256, 26), (256, 127)]


def bench_interaction():
    """Kernel vs the eager PyTorch formulation (ops/dense.py) at B = 32768, bf16. Bytes moved are the least the op must move:
    fwd reads X [B, F+1, D] and writes the padded output; bwd reads X and the output gradient and writes dX."""
    from torchrec_b200.ops import dense as DN

    print(f"GPU: {torch.cuda.get_device_name(dev)}")
    print("| interaction (D, F) | pass | kernel us | eager us | GB moved | kernel GB/s | eager GB/s | eager / kernel |\n|---|---|---|---|---|---|---|---|")
    B = 32768
    for D, F in INTERACTION_SHAPES:
        dense = torch.randn(B, D, device=dev).bfloat16().requires_grad_()
        sparse = torch.randn(B, F, D, device=dev).bfloat16().requires_grad_()
        assert I.supported(dense, sparse), (D, F)
        out = I.DotInteractionFn.apply(dense, sparse)
        g = torch.randn_like(out)
        DN.set_dense_backend("torch")
        out_e = DN.dot_interaction(dense, sparse)
        g_e = g[:, : out_e.shape[1]].contiguous()
        x_bytes = B * (F + 1) * D * 2
        for name, gb, fk, fe in (
            ("fwd", (x_bytes + out.numel() * 2) / 1e9, lambda: I.DotInteractionFn.apply(dense, sparse), lambda: DN.dot_interaction(dense, sparse)),
            ("bwd", (2 * x_bytes + out.numel() * 2) / 1e9, lambda: torch.autograd.grad(out, (dense, sparse), g, retain_graph=True),
             lambda: torch.autograd.grad(out_e, (dense, sparse), g_e, retain_graph=True)),
        ):
            uk, ue = timeit(fk), timeit(fe)
            print(f"| {D}, {F} | {name} | {uk:.1f} | {ue:.1f} | {gb:.3f} | {gb / uk * 1e6:.0f} | {gb / ue * 1e6:.0f} | {ue / uk:.2f} |")
        del dense, sparse, out, g, out_e, g_e
        torch.cuda.empty_cache()


def bench_tbe(rows_per_table=40_000_000, n_tables=8):
    print("| TBE (fp32 rows, D=128, pooling 1) | us | GB moved | GB/s |\n|---|---|---|---|")
    B, D = 32768, 128
    for rows in (rows_per_table, 1_000_000):
        tbe = T.TableBatchedEmbeddingBags([(rows, D)] * n_tables, list(range(n_tables)), pooling_mode=T.PoolingMode.SUM, optimizer=T.OptimType.EXACT_ROWWISE_ADAGRAD,
                                          learning_rate=0.01, device=dev, output_dtype=torch.bfloat16)
        idx = torch.randint(0, rows, (n_tables * B,), device=dev)
        off = torch.arange(0, n_tables * B + 1, device=dev)
        out = tbe(idx, off, None, batch_size=B)
        g = torch.randn_like(out)
        us = timeit(lambda: tbe(idx, off, None, batch_size=B))
        gb = (n_tables * B * D * 4 + out.numel() * 2) / 1e9
        print(f"| fwd {n_tables} x {rows} rows | {us:.1f} | {gb:.3f} | {gb / us * 1e6:.0f} |")
        us = timeit(lambda: out.backward(g, retain_graph=True))
        gb = (n_tables * B * D * 4 * 2 + out.numel() * 2) / 1e9
        print(f"| bwd+adagrad {n_tables} x {rows} rows | {us:.1f} | {gb:.3f} | {gb / us * 1e6:.0f} |")
        del tbe


if __name__ == "__main__":
    which = sys.argv[1:] or ["gemm", "interaction", "tbe"]
    for w in which:
        {"gemm": bench_gemm, "interaction": bench_interaction, "tbe": bench_tbe, "colsum": bench_colsum, "gemmx": bench_gemmx}[w]()
        print()
