"""Run ONE GEMM shape a few times (target for `ncu -k regex:gemm_bf16_wgmma --launch-skip 2 -c 1`).
Usage: python tools/gemm_one.py M N K [tile_n] [mode: 0 plain, 1 bias+relu, 2 masked dgrad]"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from torchrec_b200.ops import gemm as G  # noqa: E402

M, N, K = (int(x) for x in sys.argv[1:4])
tile_n = int(sys.argv[4]) if len(sys.argv) > 4 else 0
bias_relu = int(sys.argv[5]) if len(sys.argv) > 5 else 1
dev = torch.device("cuda:0")
a = torch.randn(M, K, device=dev).bfloat16()
w = torch.randn(N, K, device=dev).bfloat16()
bias = torch.zeros(N, device=dev)
out = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
mask = torch.randn(M, N, device=dev).bfloat16()
wt = w.t().contiguous()
for _ in range(5):
    if bias_relu == 2:  # masked dgrad: B consumed MN-major, ReLU-gradient mask in the epilogue
        G.gemm_bf16(a, wt, b_mn=True, out=out, act=G.ACT_RELU_GRAD, mask=mask, tile_n=tile_n)
    elif bias_relu:
        G.gemm_bf16(a, w, bias=bias, act=G.ACT_RELU, out=out, tile_n=tile_n)
    else:
        G.gemm_bf16(a, w, out=out, tile_n=tile_n)
torch.cuda.synchronize()
print("ok", float(out.float().abs().mean()))
