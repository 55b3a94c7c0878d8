"""The 13 forward and dgrad GEMMs of the one-GPU DLRM training step (batch 32768), each with the epilogue the step runs it with:
CUDA-event time per GEMM (median of 20, L2 flushed before each) on seeded inputs, and optionally the outputs, to compare two builds.

    python tools/gemm_step_bench.py [--save DIR]            # time; --save: write every output (and ReLU bit mask) to DIR
    python tools/gemm_step_bench.py --compare DIR_A DIR_B   # bit-equality / max difference of two --save directories

Run the first form from each source tree to time or compare two builds of the kernel library."""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

M = 32768
# (name, N, K) forward: bias + ReLU + ReLU bits
FWD = [("fwd bot0", 512, 16), ("fwd bot1", 256, 512), ("fwd bot2", 128, 256), ("fwd top0", 1024, 480), ("fwd top1", 1024, 1024),
       ("fwd top2", 512, 1024), ("fwd top3", 256, 512)]
# (name, N, K, masked) dgrad dx [M, N] = dy [M, K] . W [K, N] (MN-major B); masked: ReLU-gradient mask from the bits of the layer below
DGRAD = [("dgrad bot1", 512, 256, True), ("dgrad bot2", 256, 128, True), ("dgrad top0", 480, 1024, False),
         ("dgrad top1", 1024, 1024, True), ("dgrad top2", 1024, 512, True), ("dgrad top3", 512, 256, True)]


def _cases(dev):
    from torchrec_b200.ops.gemm import ACT_RELU, ACT_RELU_GRAD, gemm_bf16

    g = torch.Generator(device=dev).manual_seed(2024)
    rnd = lambda *s: (torch.randn(*s, device=dev, generator=g) * 0.3).to(torch.bfloat16)
    for name, N, K in FWD:
        x, w, bias = rnd(M, K), rnd(N, K), torch.randn(N, device=dev, generator=g)
        y = torch.empty(M, N, dtype=torch.bfloat16, device=dev)
        bits = torch.empty(M, (N + 31) // 32, dtype=torch.int32, device=dev)
        yield name, N, K, (lambda x=x, w=w, bias=bias, y=y, bits=bits: gemm_bf16(x, w, bias=bias, act=ACT_RELU, relu_bits_out=bits, out=y)), (y, bits)
    for name, N, K, masked in DGRAD:
        dy, w = rnd(M, K), rnd(K, N)
        dx = torch.empty(M, N, dtype=torch.bfloat16, device=dev)
        if masked:
            act = torch.relu(torch.randn(M, N, device=dev, generator=g)).to(torch.bfloat16)
            words = ((act > 0).view(M, N // 32, 32).long() << torch.arange(32, device=dev)).sum(-1)  # bit n % 32 of word n / 32
            bits = torch.where(words >= 2 ** 31, words - 2 ** 32, words).to(torch.int32)
            fn = lambda dy=dy, w=w, act=act, bits=bits, dx=dx: gemm_bf16(dy, w, b_mn=True, act=ACT_RELU_GRAD, mask=act, mask_bits=bits, out=dx)
        else:
            fn = lambda dy=dy, w=w, dx=dx: gemm_bf16(dy, w, b_mn=True, out=dx)
        yield name, N, K, fn, (dx,)


def run(save_dir):
    dev = torch.device("cuda:0")
    props = torch.cuda.get_device_properties(dev)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    print(f"# {props.name}, {props.multi_processor_count} SMs\n\n| GEMM | M,N,K | us | TFLOP/s |\n|---|---|---|---|")
    total = 0.0
    for name, N, K, fn, outs in _cases(dev):
        for _ in range(3):
            fn()
        ts = []
        for _ in range(20):
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1) * 1e3)
        us = sorted(ts)[len(ts) // 2]
        total += us
        print(f"| {name} | {M},{N},{K} | {us:.1f} | {2 * M * N * K / us / 1e6:.0f} |")
        if save_dir:
            os.makedirs(save_dir, exist_ok=True)
            torch.save([t.cpu() for t in outs], os.path.join(save_dir, name.replace(" ", "_") + ".pt"))
    print(f"\nsum of medians: {total:.1f} us")


def compare(a_dir, b_dir):
    print("| GEMM | bit-identical | max abs diff | elements differing |\n|---|---|---|---|")
    for name in [f[0] for f in FWD] + [d[0] for d in DGRAD]:
        fn = name.replace(" ", "_") + ".pt"
        a, b = torch.load(os.path.join(a_dir, fn)), torch.load(os.path.join(b_dir, fn))
        same = all(torch.equal(x, y) for x, y in zip(a, b))
        diff = (a[0].float() - b[0].float()).abs()
        print(f"| {name} | {'yes' if same else 'no'} | {diff.max().item():.3g} | {int((diff != 0).sum())} |")


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--save", default="")
    ap.add_argument("--compare", nargs=2, default=None)
    args = ap.parse_args()
    if args.compare:
        compare(*args.compare)
    else:
        run(args.save)
