"""Every tile path of the wgmma GEMM (128 x 64, persistent 128 x 128 and 128 x 256; TMA-store and direct-store epilogues) against
an fp32 PyTorch reference: N around the tile widths, M and K tails, all operand majors, every fused epilogue option and split-K."""
import pytest
import torch

pytestmark = pytest.mark.gpu

NS = [64, 128, 136, 256, 264, 480, 512, 1024]
MAJORS = [(False, False), (False, True), (True, False), (True, True)]


def _operands(M, N, K, a_mn, b_mn, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    A = (torch.randn(M, K, device="cuda", generator=g) * 0.3).to(torch.bfloat16)
    Bm = (torch.randn(N, K, device="cuda", generator=g) * 0.3).to(torch.bfloat16)
    a = A.t().contiguous() if a_mn else A
    b = Bm.t().contiguous() if b_mn else Bm
    return A, Bm, a, b


def _close(out, ref, K):
    torch.testing.assert_close(out.float(), ref, rtol=2e-2, atol=0.05 + 0.004 * K ** 0.5)


@pytest.mark.parametrize("a_mn,b_mn", MAJORS)
@pytest.mark.parametrize("N", NS)
@pytest.mark.parametrize("M,K", [(72, 40), (1000, 200), (384, 64)])
def test_tile_paths_plain(M, N, K, a_mn, b_mn):
    """M < 128 / M % 128 != 0, K < 64 / K % 64 != 0, bf16 (TMA store) and fp32 (direct store) outputs."""
    from torchrec_b200.ops.gemm import gemm_bf16

    A, Bm, a, b = _operands(M, N, K, a_mn, b_mn, M + N + K)
    ref = A.float() @ Bm.float().t()
    _close(gemm_bf16(a, b, a_mn=a_mn, b_mn=b_mn), ref, K)
    torch.testing.assert_close(gemm_bf16(a, b, a_mn=a_mn, b_mn=b_mn, out_dtype=torch.float32), ref, rtol=1e-3, atol=1e-2)


@pytest.mark.parametrize("N", [128, 256, 1024])
@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (False, True)])
def test_more_tiles_than_sms(N, a_mn, b_mn):
    """M = 32768: the persistent loop walks several tiles per CTA."""
    from torchrec_b200.ops.gemm import ACT_RELU, gemm_bf16

    M, K = 32768, 136
    A, Bm, a, b = _operands(M, N, K, a_mn, b_mn, N)
    bias = torch.randn(N, device="cuda")
    ref = torch.relu(A.float() @ Bm.float().t() + bias)
    _close(gemm_bf16(a, b, a_mn=a_mn, b_mn=b_mn, bias=bias, act=ACT_RELU), ref, K)


@pytest.mark.parametrize("N", NS)
@pytest.mark.parametrize("b_mn", [False, True])
def test_epilogue_options(N, b_mn):
    from torchrec_b200.ops.gemm import ACT_RELU, ACT_RELU_GRAD, ACT_SIGMOID, colsum_from_partials, gemm_bf16

    M, K = 1000, 200
    A, Bm, a, b = _operands(M, N, K, False, b_mn, 7 * N)
    acc = A.float() @ Bm.float().t()
    bias = torch.randn(N, device="cuda")
    words = (N + 31) // 32

    # alpha + bias + ReLU, with and without the bit mask: the bits must not change the output
    y = gemm_bf16(a, b, b_mn=b_mn, bias=bias, act=ACT_RELU, alpha=0.5)
    _close(y, torch.relu(0.5 * acc + bias), K)
    bits = torch.full((M, words), -1, dtype=torch.int32, device="cuda")
    y_b = gemm_bf16(a, b, b_mn=b_mn, bias=bias, act=ACT_RELU, alpha=0.5, relu_bits_out=bits)
    assert torch.equal(y_b, y)
    cols = torch.arange(N, device="cuda")
    assert torch.equal(((bits[:, cols // 32] >> (cols % 32)) & 1).bool(), y > 0)

    # sigmoid
    _close(gemm_bf16(a, b, b_mn=b_mn, bias=bias, act=ACT_SIGMOID), torch.sigmoid(acc + bias), K)

    # ReLU gradient with a bf16 mask and with the bits: identical outputs
    g_mask = gemm_bf16(a, b, b_mn=b_mn, act=ACT_RELU_GRAD, mask=y)
    _close(g_mask, acc * (y.float() > 0), K)
    assert torch.equal(gemm_bf16(a, b, b_mn=b_mn, act=ACT_RELU_GRAD, mask=y, mask_bits=bits), g_mask)

    # column sums of the bf16 output: never change the output, reduce to its column sums
    ws = torch.full(((M + 31) // 32, N), float("nan"), device="cuda")
    g_cs = gemm_bf16(a, b, b_mn=b_mn, act=ACT_RELU_GRAD, mask=y, colsum_ws=ws)
    assert torch.equal(g_cs, g_mask)
    torch.testing.assert_close(colsum_from_partials(ws), g_mask.float().sum(0), rtol=1e-4, atol=1e-2)

    # ldo > N, bf16 and fp32: the columns past N keep their contents
    for dt in (torch.bfloat16, torch.float32):
        wide = torch.full((M, N + 24), 7.0, dtype=dt, device="cuda")
        out = wide[:, :N]
        gemm_bf16(a, b, b_mn=b_mn, bias=bias, out=out)
        _close(out, acc + bias, K)
        assert bool((wide[:, N:] == 7.0).all())


def test_unaligned_output_falls_back_to_direct_stores():
    """An output whose base is 8 B but not 16 B aligned cannot be described by a tensor map: the same values are stored directly."""
    from torchrec_b200.ops.gemm import ACT_RELU, gemm_bf16

    M, N, K = 500, 512, 128
    A, Bm, a, b = _operands(M, N, K, False, False, 3)
    bias = torch.randn(N, device="cuda")
    ref = gemm_bf16(a, b, bias=bias, act=ACT_RELU)
    buf = torch.zeros(M * N + 8, dtype=torch.bfloat16, device="cuda")
    out = buf[4 : 4 + M * N].view(M, N)
    assert out.data_ptr() % 16 != 0
    gemm_bf16(a, b, bias=bias, act=ACT_RELU, out=out)
    assert torch.equal(out, ref)


@pytest.mark.parametrize("a_mn,b_mn", MAJORS)
@pytest.mark.parametrize("N", [64, 136, 264, 1024])
def test_split_k(N, a_mn, b_mn):
    from torchrec_b200.ops.gemm import gemm_bf16

    M, K = 264, 5000
    A, Bm, a, b = _operands(M, N, K, a_mn, b_mn, 11 + N)
    ref = A.float() @ Bm.float().t()
    for split in (3, 16):
        out = gemm_bf16(a, b, a_mn=a_mn, b_mn=b_mn, out_dtype=torch.float32, split_k=split, tile_n=128)
        torch.testing.assert_close(out, ref, rtol=2e-3, atol=5e-2)
