"""The ping-pong wgmma GEMM (bf16 output without split-K, N > 128, except plain MN-major-B products: each consumer warpgroup owns
whole 128 x 128 tiles and the two alternate) against an fp32 reference: every forward and dgrad GEMM of the DLRM training step with
the epilogue it uses there (two of them run on the cooperative kernel), M and N tails, uneven tile counts per CTA and per
warpgroup, grids smaller than the GPU, and the direct-store epilogue."""
import pytest
import torch

pytestmark = pytest.mark.gpu

M_STEP = 32768  # bench.py's batch
# (name, N, K) of the step's forward GEMMs: bottom MLP 13 (padded to 16) -> 512 -> 256 -> 128, top MLP 480 -> 1024 -> 1024 -> 512 -> 256
FWD = [("bot0", 512, 16), ("bot1", 256, 512), ("bot2", 128, 256), ("top0", 1024, 480), ("top1", 1024, 1024), ("top2", 512, 1024),
       ("top3", 256, 512)]
# (name, N, K, masked) of the dgrad GEMMs dx [M, N] = dy [M, K] . W [K, N]; masked: the input is the ReLU output of the layer below,
# whose gradient mask (bits) is applied in the epilogue. top0's input is the interaction output (no mask); bot0's input needs none.
DGRAD = [("bot1", 512, 256, True), ("bot2", 256, 128, True), ("top0", 480, 1024, False), ("top1", 1024, 1024, True),
         ("top2", 1024, 512, True), ("top3", 512, 256, True)]


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _randn(shape, g, scale=0.3):
    return (torch.randn(*shape, device="cuda", generator=g) * scale).to(torch.bfloat16)


def _close(out, ref, K):
    torch.testing.assert_close(out.float(), ref, rtol=2e-2, atol=0.05 + 0.004 * K ** 0.5)


def _pack_bits(pos: torch.Tensor) -> torch.Tensor:
    """bool [M, N] -> int32 [M, ceil(N / 32)], bit n % 32 of word n / 32 (the layout of relu_bits_out / mask_bits)."""
    M, N = pos.shape
    words = (N + 31) // 32
    padded = torch.zeros(M, words * 32, dtype=torch.int64, device=pos.device)
    padded[:, :N] = pos.long()
    w = (padded.view(M, words, 32) << torch.arange(32, device=pos.device)).sum(-1)
    return torch.where(w >= 2 ** 31, w - 2 ** 32, w).to(torch.int32)


def _check_forward(M, N, K, seed, out=None, a_mn=False):
    from torchrec_b200.ops.gemm import ACT_RELU, gemm_bf16

    g = torch.Generator(device="cuda").manual_seed(seed)
    x, w = _randn((M, K), g), _randn((N, K), g)
    bias = torch.randn(N, device="cuda", generator=g)
    ref = torch.relu(x.float() @ w.float().t() + bias)
    bits = torch.full((M, (N + 31) // 32), -1, dtype=torch.int32, device="cuda")
    a = x.t().contiguous() if a_mn else x
    y = gemm_bf16(a, w, a_mn=a_mn, bias=bias, act=ACT_RELU, relu_bits_out=bits, out=out)
    _close(y, ref, K)
    assert torch.equal(bits, _pack_bits(y > 0))
    return y


def _check_dgrad(M, N, K, masked, seed, out=None):
    """dx = dy . W with W [K, N] consumed MN-major; masked: ReLU-gradient mask from bits and from the bf16 activation, and the
    epilogue column sums."""
    from torchrec_b200.ops.gemm import ACT_RELU_GRAD, colsum_from_partials, gemm_bf16

    g = torch.Generator(device="cuda").manual_seed(seed)
    dy, w = _randn((M, K), g), _randn((K, N), g)
    acc = dy.float() @ w.float()
    if not masked:
        dx = gemm_bf16(dy, w, b_mn=True, out=out)
        _close(dx, acc, K)
        return dx
    act = torch.relu(_randn((M, N), g, 1.0))  # the forward activation of the layer below: about half zeros
    bits = _pack_bits(act > 0)
    dx = gemm_bf16(dy, w, b_mn=True, act=ACT_RELU_GRAD, mask=act, mask_bits=bits, out=out)
    _close(dx, acc * (act.float() > 0), K)
    assert torch.equal(gemm_bf16(dy, w, b_mn=True, act=ACT_RELU_GRAD, mask=act), dx)
    ws = torch.full(((M + 31) // 32, N), float("nan"), device="cuda")
    assert torch.equal(gemm_bf16(dy, w, b_mn=True, act=ACT_RELU_GRAD, mask=act, mask_bits=bits, colsum_ws=ws), dx)
    torch.testing.assert_close(colsum_from_partials(ws), dx.float().sum(0), rtol=1e-4, atol=2e-2)
    return dx


@pytest.mark.parametrize("name,N,K", FWD, ids=[f[0] for f in FWD])
def test_step_forward(name, N, K):
    """bias + ReLU + ReLU bits, as the step's forward layers run."""
    _check_forward(M_STEP, N, K, seed=N + K)


@pytest.mark.parametrize("name,N,K,masked", DGRAD, ids=[d[0] for d in DGRAD])
def test_step_dgrad(name, N, K, masked):
    """ReLU-gradient mask from bits (bf16 mask: same output) and column sums, or a plain dgrad into the interaction output."""
    _check_dgrad(M_STEP, N, K, masked, seed=3 * N + K)


@pytest.mark.parametrize("M", [1, 72, 200, 1000, 32768 + 72])
@pytest.mark.parametrize("N", [136, 264, 480])
def test_tails(M, N):
    """M tails (a tile whose second 64-row half is empty or partial) and N tails (N = 136: a last tile of 8 columns)."""
    _check_forward(M, N, 200, seed=M + N)
    _check_dgrad(M, N, 136, True, seed=M + 2 * N)


@pytest.mark.parametrize("extra", [0, 5])
def test_odd_tiles_per_cta(extra):
    """3 tiles per CTA (warpgroup 0 runs two, warpgroup 1 one), and 3 or 4 when `extra` tiles are left over."""
    N = 256
    M = 128 * (3 * _sms() + extra) // 2  # (N / 128 = 2 tiles per 128-row block)
    _check_forward(M, N, 192, seed=11 + extra)
    _check_dgrad(M, N, 320, True, seed=13 + extra)


@pytest.mark.parametrize("tiles", ["fewer_than_sms", "fewer_than_2x_sms"])
def test_small_grids(tiles):
    """One tile per CTA (warpgroup 1 has none), and some CTAs with two."""
    N = 256  # 2 tiles per 128-row block
    m_blocks = 4 if tiles == "fewer_than_sms" else (_sms() + 14) // 2
    _check_forward(128 * m_blocks - 40, N, 256, seed=m_blocks)
    _check_dgrad(128 * m_blocks - 40, N, 512, True, seed=m_blocks + 1)


@pytest.mark.parametrize("a_mn", [False, True])
def test_long_k_operand_majors(a_mn):
    """Long K (many ring passes per tile), with A K-major and MN-major."""
    _check_forward(2048 + 64, 384, 2048 + 8, seed=17, a_mn=a_mn)


def test_unaligned_output_direct_store():
    """An output whose base is 8 B but not 16 B aligned cannot be described by a tensor map: the ping-pong kernel stores from the
    fragment layout, with the same epilogues and the same values."""
    M, N = 3000, 264
    buf = torch.zeros(M * N + 8, dtype=torch.bfloat16, device="cuda")
    out = buf[4 : 4 + M * N].view(M, N)
    assert out.data_ptr() % 16 != 0
    y = _check_forward(M, N, 256, seed=5, out=out)
    assert torch.equal(y, _check_forward(M, N, 256, seed=5))
    dx = _check_dgrad(M, N, 384, True, seed=6, out=out)
    assert torch.equal(dx, _check_dgrad(M, N, 384, True, seed=6))
