"""Split-K fp32 weight gradients ``gw = gy^T . x`` (both operands MN-major) against an fp32 reference built from the same bf16
operands: the seven wgrads of the DLRM training step as ``LinearActFn.backward`` runs them (including the 479- and 13-wide inputs and
their slice), split factors 1, 2, the planned one and 64, M and N tails, a K that is not a multiple of the split, an output a tensor
map cannot describe (cooperative kernel, fp32 atomics) and capture / replay in a CUDA graph. Split-K outputs with a describable output
run on the ping-pong kernel, each K-slice's partial tile added through TMA reduce-adds."""
import pytest
import torch

pytestmark = pytest.mark.gpu

M_STEP = 32768  # bench.py's batch
# (name, n_out, n_in) of the step's weight gradients: bottom MLP 13 -> 512 -> 256 -> 128, top MLP 479 -> 1024 -> 1024 -> 512 -> 256
WGRADS = [("bot0", 512, 13), ("bot1", 256, 512), ("bot2", 128, 256), ("top0", 1024, 479), ("top1", 1024, 1024), ("top2", 512, 1024),
          ("top3", 256, 512)]


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _operands(batch, n_out, n_in, seed):
    """gy [batch, n_out] and x [batch, Kp] (bf16, columns >= n_in zero, as LinearActFn pads them) and the fp32 reference [n_out, n_in]."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    Kp = (n_in + 7) // 8 * 8
    gy = (torch.randn(batch, n_out, device="cuda", generator=g) * 0.3).to(torch.bfloat16)
    x = torch.zeros(batch, Kp, dtype=torch.bfloat16, device="cuda")
    x[:, :n_in] = (torch.randn(batch, n_in, device="cuda", generator=g) * 0.3).to(torch.bfloat16)
    ref = gy.float().t() @ x[:, :n_in].float()
    return gy, x, ref


def _close(out, ref):
    # fp32 sums of up to 32768 products of magnitude ~0.1 (results ~16): a few ulps of the accumulation order, far below one product
    torch.testing.assert_close(out, ref, rtol=1e-3, atol=1e-2)


def _wgrad(gy, x, split, out=None):
    from torchrec_b200.ops.gemm import gemm_bf16

    return gemm_bf16(gy, x, a_mn=True, b_mn=True, out_dtype=torch.float32, split_k=split, out=out)


def _kernels(fn):
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.key for e in prof.key_averages() if "gemm_bf16_wgmma" in e.key]


@pytest.mark.parametrize("idx,name,n_out,n_in", [(i,) + w for i, w in enumerate(WGRADS)], ids=[w[0] for w in WGRADS])
def test_step_wgrads_planned(idx, name, n_out, n_in):
    """As LinearActFn.backward runs them: the planned split, then the slice to the unpadded width (and the copy that makes it dense)."""
    from torchrec_b200.ops.gemm import _wgrad_plan

    gy, x, ref = _operands(M_STEP, n_out, n_in, seed=idx)
    split, _ = _wgrad_plan(n_out, x.shape[1], M_STEP, _sms())
    gw = _wgrad(gy, x, split)[:, :n_in].contiguous()
    assert gw.shape == (n_out, n_in)
    _close(gw, ref)


@pytest.mark.parametrize("name,n_out,n_in", [WGRADS[3], WGRADS[6], WGRADS[2]], ids=["top0", "top3", "bot2"])
@pytest.mark.parametrize("split", [1, 2, "plan", 64])
def test_split_factors(name, n_out, n_in, split):
    from torchrec_b200.ops.gemm import _wgrad_plan

    gy, x, ref = _operands(M_STEP, n_out, n_in, seed=7)
    if split == "plan":
        split = _wgrad_plan(n_out, x.shape[1], M_STEP, _sms())[0]
    _close(_wgrad(gy, x, split)[:, :n_in], ref)


@pytest.mark.parametrize("batch,n_out,n_in,split", [
    (4096, 200, 136, 4),     # M and N tails of the 128 x 128 tiles
    (3000, 256, 256, 5),     # K = 47 k-blocks (a 56-element tail): slices of 10 k-blocks, the last one of 7
    (1000, 328, 264, 64),    # 16 k-blocks: the split is cut to 16 one-k-block slices
    (33000, 136, 1032, 9),   # M, N and K tails together, more items than the grid
])
def test_tails(batch, n_out, n_in, split):
    gy, x, ref = _operands(batch, n_out, n_in, seed=batch)
    _close(_wgrad(gy, x, split), ref)


def test_routes_by_tensor_map():
    """A 16 B aligned output runs the ping-pong kernel; a row pitch of 130 floats (not a multiple of 16 B) cannot be described by a
    tensor map and falls back to the cooperative kernel's fp32 atomics. Both are checked against the reference."""
    gy, x, ref = _operands(8192, 256, 128, seed=3)
    names = _kernels(lambda: _wgrad(gy, x, 8))
    assert names and all("pingpong" in k for k in names), names
    buf = torch.full((256, 130), float("nan"), device="cuda")
    out = buf[:, :128]
    names = _kernels(lambda: _wgrad(gy, x, 8, out=out))
    assert names and all("persistent" in k for k in names), names
    _close(out, ref)


def test_cuda_graph_replay():
    """Memset and split-K GEMM captured into a CUDA graph (as in the captured dense backward), replayed on new operands."""
    gy, x, _ = _operands(M_STEP, 1024, 479, seed=11)
    from torchrec_b200.ops.gemm import _wgrad_plan

    split = _wgrad_plan(1024, x.shape[1], M_STEP, _sms())[0]
    out = torch.empty(1024, x.shape[1], device="cuda")
    _wgrad(gy, x, split, out=out)  # warm-up (kernel attributes, tensor-map encoder)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        _wgrad(gy, x, split, out=out)
    for seed in (12, 13):
        gy2, x2, ref = _operands(M_STEP, 1024, 479, seed=seed)
        gy.copy_(gy2)
        x.copy_(x2)
        out.fill_(float("nan"))
        graph.replay()
        torch.cuda.synchronize()
        _close(out[:, :479], ref)
