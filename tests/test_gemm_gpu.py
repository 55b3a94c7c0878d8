"""wgmma GEMM / fused Linear numerics vs fp32 PyTorch."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _ref(a, b, bias, act):
    y = a.float() @ b.float().t()
    if bias is not None:
        y = y + bias
    if act == 1:
        y = torch.relu(y)
    elif act == 2:
        y = torch.sigmoid(y)
    return y


@pytest.mark.parametrize("M,N,K", [(128, 128, 64), (256, 256, 512), (1000, 512, 256), (4096, 1024, 480), (300, 64, 16), (128, 8, 1024), (4096, 128, 2048), (38000, 512, 192), (20000, 1024, 320)])
@pytest.mark.parametrize("act", [0, 1])
def test_gemm_bf16_tn(M, N, K, act):
    from torchrec_b200.ops.gemm import gemm_bf16_tn

    torch.manual_seed(0)
    dev = torch.device("cuda:0")
    a = (torch.randn(M, K, device=dev) * 0.5).to(torch.bfloat16)
    b = (torch.randn(N, K, device=dev) * 0.5).to(torch.bfloat16)
    bias = torch.randn(N, device=dev)
    out = gemm_bf16_tn(a, b, bias, act)
    ref = _ref(a, b, bias, act)
    torch.testing.assert_close(out.float(), ref, rtol=2e-2, atol=2e-1 if K > 512 else 6e-2)
    out32 = gemm_bf16_tn(a, b, None, 0, out_dtype=torch.float32)
    torch.testing.assert_close(out32, _ref(a, b, None, 0), rtol=1e-3, atol=1e-2)


def test_gemm_split_k_and_mask():
    from torchrec_b200.ops.gemm import ACT_RELU_GRAD, gemm_bf16_tn

    dev = torch.device("cuda:0")
    torch.manual_seed(1)
    a = (torch.randn(256, 8192, device=dev) * 0.1).to(torch.bfloat16)
    b = (torch.randn(128, 8192, device=dev) * 0.1).to(torch.bfloat16)
    out = gemm_bf16_tn(a, b, out_dtype=torch.float32, split_k=16)
    torch.testing.assert_close(out, a.float() @ b.float().t(), rtol=1e-3, atol=2e-2)
    a2 = (torch.randn(512, 256, device=dev)).to(torch.bfloat16)
    b2 = (torch.randn(128, 256, device=dev)).to(torch.bfloat16)
    mask = torch.randn(512, 128, device=dev).to(torch.bfloat16)
    o = gemm_bf16_tn(a2, b2, act=ACT_RELU_GRAD, mask=mask)
    ref = (a2.float() @ b2.float().t()) * (mask.float() > 0)
    torch.testing.assert_close(o.float(), ref, rtol=2e-2, atol=1e-1)


def test_linear_act_autograd_matches_torch():
    from torchrec_b200.ops import dense
    from torchrec_b200.modules.mlp import MLP

    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    ref = MLP(13, [64, 32, 16], device=dev)
    mine = MLP(13, [64, 32, 16], device=dev)
    mine.load_state_dict(ref.state_dict())
    x = torch.randn(512, 13, device=dev)
    yr = ref(x)
    dense.set_dense_backend("wgmma")
    try:
        ym = mine(x)
    finally:
        dense.set_dense_backend("torch")
    torch.testing.assert_close(ym.float(), yr, rtol=5e-2, atol=5e-2)
    g = torch.randn_like(yr)
    yr.backward(g)
    ym.backward(g.to(ym.dtype))
    for (n, pr), (_, pm) in zip(ref.named_parameters(), mine.named_parameters()):
        cos = torch.nn.functional.cosine_similarity(pm.grad.flatten().float(), pr.grad.flatten().float(), dim=0)
        assert float(cos) > 0.99, (n, float(cos))


@pytest.mark.parametrize("a_mn,b_mn", [(True, True), (False, True), (True, False)])
@pytest.mark.parametrize("M,N,K", [(256, 128, 512), (1024, 512, 4096), (128, 16, 333), (480, 1024, 1000), (38016, 256, 136), (1024, 1024, 40000)])
def test_gemm_mn_major_operands(a_mn, b_mn, M, N, K):
    from torchrec_b200.ops.gemm import gemm_bf16

    dev = torch.device("cuda:0")
    torch.manual_seed(2)
    if not a_mn or not b_mn:
        K = (K + 7) // 8 * 8
    A = (torch.randn(M, K, device=dev) * 0.3).to(torch.bfloat16)
    Bm = (torch.randn(N, K, device=dev) * 0.3).to(torch.bfloat16)
    a = A.t().contiguous() if a_mn else A
    b = Bm.t().contiguous() if b_mn else Bm
    out = gemm_bf16(a, b, a_mn=a_mn, b_mn=b_mn, out_dtype=torch.float32)
    ref = A.float() @ Bm.float().t()
    torch.testing.assert_close(out, ref, rtol=1e-3, atol=2e-2)
    out2 = gemm_bf16(a, b, a_mn=a_mn, b_mn=b_mn, out_dtype=torch.float32, split_k=4)
    torch.testing.assert_close(out2, ref, rtol=1e-3, atol=2e-2)
    if N % 256 == 0:  # split-K on 128 x 256 tiles (the wgrad plan of wide layers)
        out3 = gemm_bf16(a, b, a_mn=a_mn, b_mn=b_mn, out_dtype=torch.float32, split_k=5, tile_n=256)
        torch.testing.assert_close(out3, ref, rtol=1e-3, atol=2e-2)


def test_wgrad_plan_fills_the_grid():
    from torchrec_b200.ops.gemm import _wgrad_plan

    for n_out, n_in in [(1024, 1024), (512, 1024), (256, 512), (1024, 480), (512, 16), (128, 256)]:
        s, tn = _wgrad_plan(n_out, n_in, 32768, 132)
        tiles = ((n_out + 127) // 128) * ((n_in + tn - 1) // tn) * s
        assert tn == 128
        assert tiles >= 0.85 * 132, (n_out, n_in, s, tn)


@pytest.mark.parametrize("N", [128, 256, 480, 1024])
def test_colsum_variants(N, monkeypatch):
    from torchrec_b200.ops.gemm import colsum_bf16

    x = (torch.randn(5003, N, device="cuda:0") * 0.5).to(torch.bfloat16)
    torch.testing.assert_close(colsum_bf16(x), x.float().sum(0), rtol=1e-3, atol=5e-2)
    xs = x[:, : N // 2] if (N // 2) % 8 == 0 else x  # strided view
    torch.testing.assert_close(colsum_bf16(xs), xs.float().sum(0), rtol=1e-3, atol=5e-2)


@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (False, True), (True, True), (True, False)])
@pytest.mark.parametrize("M,N,K,split", [(256, 256, 64, 1), (512, 256, 512, 1), (4096, 1024, 480, 1), (5000, 480, 1024, 1), (1024, 1024, 40000, 9),
                                         (40000, 512, 200, 1), (256, 512, 32768, 37), (300, 264, 136, 1)])
def test_gemm_cta_pair_kernel(a_mn, b_mn, M, N, K, split):
    """The shapes the CTA-pair kernel took on Blackwell (tile hint 512), now on the wgmma kernel: fp32 matmul reference over all operand
    majors, tails in M / N / K, deep split-K."""
    from torchrec_b200.ops.gemm import ACT_RELU, gemm_bf16

    dev = torch.device("cuda:0")
    torch.manual_seed(5)
    K = (K + 7) // 8 * 8
    if a_mn:
        M = (M + 7) // 8 * 8
    A = (torch.randn(M, K, device=dev) * 0.3).to(torch.bfloat16)
    Bm = (torch.randn(N, K, device=dev) * 0.3).to(torch.bfloat16)
    a = A.t().contiguous() if a_mn else A
    b = Bm.t().contiguous() if b_mn else Bm
    ref = A.float() @ Bm.float().t()
    out = gemm_bf16(a, b, a_mn=a_mn, b_mn=b_mn, out_dtype=torch.float32, split_k=split, tile_n=512)
    torch.testing.assert_close(out, ref, rtol=2e-3, atol=3e-2 if K < 10000 else 0.2)
    if split == 1:
        bias = torch.randn(N, device=dev)
        out_b = gemm_bf16(a, b, a_mn=a_mn, b_mn=b_mn, bias=bias, act=ACT_RELU, tile_n=512)
        torch.testing.assert_close(out_b.float(), torch.relu(ref + bias), rtol=2e-2, atol=6e-2)


def test_low_rank_crossnet_on_wgmma_matches_torch():
    from torchrec_b200.modules.crossnet import LowRankCrossNet
    from torchrec_b200.ops import dense as D

    dev = torch.device("cuda:0")
    torch.manual_seed(3)
    net = LowRankCrossNet(in_features=256, num_layers=2, low_rank=64).to(dev)
    with torch.no_grad():
        for b in net.bias:
            b.normal_(0, 0.1)
    x = (torch.randn(1000, 256, device=dev) * 0.5).requires_grad_()
    prev = D.get_dense_backend()
    try:
        D.set_dense_backend("torch")
        ref = net(x)
        ref.sum().backward()
        gref, gw_ref = x.grad.clone(), net.W_kernels[0].grad.clone()
        x.grad = None
        net.zero_grad()
        D.set_dense_backend("wgmma")
        out = net(x)
        out.sum().backward()
    finally:
        D.set_dense_backend(prev)
    torch.testing.assert_close(out, ref, rtol=3e-2, atol=6e-2)
    torch.testing.assert_close(x.grad, gref, rtol=5e-2, atol=1e-1)
    torch.testing.assert_close(net.W_kernels[0].grad, gw_ref, rtol=5e-2, atol=2.0)


@pytest.mark.parametrize("tile_n", [0, 128, 256, 512])
@pytest.mark.parametrize("M,N,K", [(512, 256, 128), (1000, 480, 256), (4100, 1024, 512), (300, 64, 64)])
def test_relu_bit_mask_roundtrip(M, N, K, tile_n):
    """Forward ReLU epilogue writes 1 bit per output; the masked dgrad consumes the bits instead of the bf16 activation."""
    from torchrec_b200.ops.gemm import ACT_RELU, ACT_RELU_GRAD, gemm_bf16

    # tile_n is only a hint to the kernel (its tile depends on N); every value a caller may pass is kept here and must give the same bits
    dev = torch.device("cuda:0")
    torch.manual_seed(11)
    a = (torch.randn(M, K, device=dev) * 0.3).to(torch.bfloat16)
    w = (torch.randn(N, K, device=dev) * 0.3).to(torch.bfloat16)
    bias = torch.randn(N, device=dev) * 0.1
    words = (N + 31) // 32
    bits = torch.full((M, words), -1, dtype=torch.int32, device=dev)
    y = gemm_bf16(a, w, bias=bias, act=ACT_RELU, relu_bits_out=bits, tile_n=tile_n)
    cols = torch.arange(N, device=dev)
    got = ((bits[:, cols // 32] >> (cols % 32)) & 1).bool()
    assert torch.equal(got, y > 0)
    gy = (torch.randn(M, N, device=dev) * 0.5).to(torch.bfloat16)
    wt = (torch.randn(N, N, device=dev) * 0.1).to(torch.bfloat16)          # dgrad of a following N -> N layer: [M, N] = gy [M, N] . W [N, N]
    ref = gemm_bf16(gy, wt, b_mn=True, act=ACT_RELU_GRAD, mask=y, tile_n=tile_n)
    out = gemm_bf16(gy, wt, b_mn=True, act=ACT_RELU_GRAD, mask=y, mask_bits=bits, tile_n=tile_n)
    assert torch.equal(out, ref)
    assert torch.equal(out == 0, (ref == 0)) and bool(((out != 0) <= (y > 0)).all())


@pytest.mark.parametrize("M,N,K,masked", [(32768, 1024, 1024, True), (4096, 512, 256, True), (1000, 480, 1024, False), (333, 64, 512, False), (8192, 256, 512, True)])
def test_epilogue_column_sums_equal_the_column_sums_of_the_output(M, N, K, masked):
    """The dgrad epilogue's per-32-row column sums (bias gradient of the layer below) reduce to exactly the column sums of the bf16
    tensor the GEMM wrote (same rounded values, fp32 accumulation)."""
    from torchrec_b200.ops.gemm import ACT_NONE, ACT_RELU_GRAD, colsum_from_partials, gemm_bf16

    torch.manual_seed(M + N)
    dev = "cuda"
    gy = torch.randn(M, K, device=dev).to(torch.bfloat16)
    w = (torch.randn(K, N, device=dev) / K ** 0.5).to(torch.bfloat16)  # [K, N]: consumed MN-major like a dgrad
    mask = torch.randn(M, N, device=dev).to(torch.bfloat16) if masked else None
    ws = torch.full(((M + 31) // 32, N), float("nan"), device=dev)
    out = gemm_bf16(gy, w, b_mn=True, act=ACT_RELU_GRAD if masked else ACT_NONE, mask=mask, colsum_ws=ws)
    ref_out = gemm_bf16(gy, w, b_mn=True, act=ACT_RELU_GRAD if masked else ACT_NONE, mask=mask)
    assert torch.equal(out, ref_out), "asking for the column sums must not change the output"
    assert not torch.isnan(ws).any()
    got = colsum_from_partials(ws)
    want = out.float().sum(0)
    torch.testing.assert_close(got, want, rtol=1e-4, atol=1e-2)
    # per-slab partials: rows 32p .. 32p+31
    p = (M // 32) // 2
    torch.testing.assert_close(ws[p], out[32 * p : 32 * p + 32].float().sum(0), rtol=1e-5, atol=1e-4)


def test_mlp_bias_gradients_from_the_epilogue_match_the_separate_colsum(monkeypatch):
    import torchrec_b200.ops.dense as Dn
    import torchrec_b200.ops.gemm as G
    from torchrec_b200.modules.mlp import MLP

    prev = Dn._BACKEND
    Dn.set_dense_backend("wgmma")
    try:
        torch.manual_seed(0)
        mlp = MLP(480, [1024, 512, 256], device=torch.device("cuda"))
        x = torch.randn(4096, 480, device="cuda").to(torch.bfloat16)
        grads = {}
        for flag in (True, False):
            monkeypatch.setattr(G, "EPI_COLSUM", flag)
            mlp.zero_grad()
            mlp(x).float().square().mean().backward()
            grads[flag] = [p.grad.clone() for p in mlp.parameters()]
        for a, b in zip(grads[True], grads[False]):
            torch.testing.assert_close(a, b, rtol=1e-4, atol=1e-5)
    finally:
        Dn._BACKEND = prev
