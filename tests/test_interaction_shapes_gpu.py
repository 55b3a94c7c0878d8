"""wgmma dot interaction at every covered shape: D % 16 == 0 with 16 <= D <= 256, 1 <= F <= 127.

Exact tests draw dense, sparse and the output gradient from the dyadic grid k / 8 (|k| <= 8). Every product is a multiple of
1/64 and every sum of up to 256 such terms is exact in fp32 (and bf16 holds every input exactly), so the kernel's output and
gradients must equal a float64 reference rounded once to the output dtype, bit for bit."""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
PACKING_F = [1, 15, 16, 31, 32, 63, 64, 127]  # R = F + 1 on both sides of 16, 32, 64 and at 128


def _ceil8(x):
    return (x + 7) // 8 * 8


def _dyadic(*shape, gen):
    return torch.randint(-8, 9, shape, generator=gen, dtype=torch.int64).double().div_(8.0)


def _ref64(dense, sparse):
    B, D = dense.shape
    F = sparse.shape[1]
    c = torch.cat((dense.unsqueeze(1), sparse), dim=1)
    z = torch.bmm(c, c.transpose(1, 2))
    ti = torch.triu_indices(F + 1, F + 1, offset=1, device=dense.device)
    return torch.cat((dense, z[:, ti[0], ti[1]]), dim=1)


def _samples_per_tile(F):
    R = F + 1
    return 8 if R <= 16 else 4 if R <= 32 else 2 if R <= 64 else 1


def _check_exact(B, F, D, sparse_dtype, seed=0, dense_pitch=None, sparse_pitch=None, sparse_off=0):
    """Kernel forward + backward against the float64 reference, bit for bit. dense_pitch / sparse_pitch (> D, > F * D) place the
    inputs as strided views into wider rows (sparse at column sparse_off of a KeyedTensor-like [B, total] values tensor)."""
    from torchrec_b200.ops import interaction as I

    gen = torch.Generator().manual_seed(seed)
    d64, s64 = _dyadic(B, D, gen=gen), _dyadic(B, F, D, gen=gen)
    n = D + (F + 1) * F // 2
    ld = _ceil8(n)
    g64 = _dyadic(B, n, gen=gen)

    dense_store = torch.zeros(B, dense_pitch or D, dtype=torch.bfloat16, device=DEV)
    dense_store[:, :D] = d64.to(torch.bfloat16).to(DEV)
    dense = dense_store[:, :D]
    sp_store = torch.zeros(B, sparse_pitch or F * D, dtype=sparse_dtype, device=DEV)
    sp_store[:, sparse_off : sparse_off + F * D] = s64.reshape(B, F * D).to(sparse_dtype).to(DEV)
    sparse = sp_store[:, sparse_off : sparse_off + F * D].view(B, F, D)
    dense.requires_grad_(True)
    sparse.requires_grad_(True)
    assert I.supported(dense, sparse)

    out = I.DotInteractionFn.apply(dense, sparse)
    assert out.shape == (B, ld) and out.dtype == torch.bfloat16 and out._trb_logical_cols == n
    d64r, s64r = d64.clone().requires_grad_(True), s64.clone().requires_grad_(True)
    ref = _ref64(d64r, s64r)
    assert torch.equal(out[:, :n].cpu(), ref.detach().to(torch.bfloat16)), "forward"
    assert torch.count_nonzero(out[:, n:]).item() == 0, "tail columns"

    g = torch.zeros(B, ld, dtype=torch.bfloat16, device=DEV)
    g[:, :n] = g64.to(torch.bfloat16).to(DEV)
    out.backward(g)
    ref.backward(g64)
    assert dense.grad.dtype == torch.bfloat16 and sparse.grad.dtype == sparse_dtype
    assert torch.equal(dense.grad.cpu(), d64r.grad.to(torch.bfloat16)), "dense gradient"
    assert torch.equal(sparse.grad.cpu(), s64r.grad.to(sparse_dtype)), "sparse gradient"


@pytest.mark.parametrize("sparse_dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("D", [16, 64, 256])
@pytest.mark.parametrize("F", PACKING_F)
def test_exact_packing_boundaries(F, D, sparse_dtype):
    _check_exact(37, F, D, sparse_dtype, seed=F * 1000 + D)


@pytest.mark.parametrize("sparse_dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("D", [16, 32, 48, 64, 96, 128, 192, 256])
def test_exact_every_width_f26(D, sparse_dtype):
    _check_exact(300, 26, D, sparse_dtype, seed=D)


@pytest.mark.parametrize("D", [48, 64, 256])
@pytest.mark.parametrize("F", [15, 31, 63, 127])
def test_exact_batch_tails(F, D):
    spt = _samples_per_tile(F)
    for B in sorted({1, spt - 1, spt + 1, 5003} - {0}):
        _check_exact(B, F, D, torch.bfloat16, seed=B)


@pytest.mark.parametrize("sparse_dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("D,F", [(64, 26), (48, 40), (256, 9), (16, 100)])
def test_exact_strided_inputs(D, F, sparse_dtype):
    # sparse: a [B, F, D] view at column 3 * D of a [B, (F + 5) * D] values tensor; dense: rows of D + 24 elements
    _check_exact(523, F, D, sparse_dtype, seed=7, dense_pitch=D + 24, sparse_pitch=(F + 5) * D, sparse_off=3 * D)


@pytest.mark.parametrize("F", [10, 26, 50, 100])
def test_random_normal_per_packing(F):
    from torchrec_b200.ops.interaction import DotInteractionFn

    B, D = 1000, 64
    torch.manual_seed(F)
    dense = (torch.randn(B, D, device=DEV) * 0.5).to(torch.bfloat16).requires_grad_(True)
    sparse = (torch.randn(B, F, D, device=DEV) * 0.5).to(torch.bfloat16).requires_grad_(True)
    out = DotInteractionFn.apply(dense, sparse)
    n = D + (F + 1) * F // 2
    d32 = dense.detach().float().requires_grad_(True)
    s32 = sparse.detach().float().requires_grad_(True)
    ref = _ref64(d32, s32)
    torch.testing.assert_close(out[:, :n].float(), ref, rtol=2e-2, atol=8e-2)
    assert float(out.detach()[:, n:].abs().sum()) == 0.0
    g = (torch.randn(B, out.shape[1], device=DEV) * 0.1).to(torch.bfloat16)
    g[:, n:] = 0
    out.backward(g)
    ref.backward(g[:, :n].float())
    tol_d = 0.03 * float(d32.grad.abs().max()) + 1e-2
    tol_s = 0.03 * float(s32.grad.abs().max()) + 1e-2
    assert float((dense.grad.float() - d32.grad).abs().max()) < tol_d
    assert float((sparse.grad.float() - s32.grad).abs().max()) < tol_s


@pytest.mark.parametrize("D,F", [(8, 26), (24, 26), (272, 26), (64, 128)])
def test_out_of_range_shapes_fall_back(D, F):
    from torchrec_b200.ops import _lib
    from torchrec_b200.ops import dense as _dense
    from torchrec_b200.ops import interaction as I

    B = 64
    gen = torch.Generator().manual_seed(1)
    d64, s64 = _dyadic(B, D, gen=gen), _dyadic(B, F, D, gen=gen)
    dense = d64.to(torch.bfloat16).to(DEV)
    sparse = s64.to(torch.bfloat16).to(DEV)
    assert not I.supported(dense, sparse)
    ld = _ceil8(D + (F + 1) * F // 2)
    out = torch.empty(B, ld, dtype=torch.bfloat16, device=DEV)
    code = _lib.lib().trb_interaction_fwd(_lib.ptr(dense), ctypes.c_int64(D), _lib.ptr(sparse), ctypes.c_int64(F * D), 0, _lib.ptr(out),
                                          ctypes.c_int64(ld), B, F, D, _lib.stream_ptr(DEV))
    assert code == -20
    gd = torch.empty_like(dense)
    gs = torch.empty_like(sparse)
    code = _lib.lib().trb_interaction_bwd(_lib.ptr(dense), ctypes.c_int64(D), _lib.ptr(sparse), ctypes.c_int64(F * D), 0, _lib.ptr(out),
                                          ctypes.c_int64(ld), _lib.ptr(gd), ctypes.c_int64(D), _lib.ptr(gs), ctypes.c_int64(F * D), 0, B, F, D,
                                          _lib.stream_ptr(DEV))
    assert code == -20
    _dense.set_dense_backend("wgmma")
    try:
        got = _dense.dot_interaction(dense, sparse)
    finally:
        _dense.set_dense_backend("torch")
    assert got.shape == (B, D + (F + 1) * F // 2)
    assert torch.equal(got.cpu(), _ref64(d64, s64).to(torch.bfloat16))


@pytest.fixture
def kernel_only(monkeypatch):
    """The eager interaction raises while the wgmma backend is on: the kernel must serve every interaction."""
    from torchrec_b200.ops import dense as _dense

    orig = _dense._triu_flat_index

    def guarded(n, device):
        if _dense.get_dense_backend() == "wgmma":
            raise AssertionError("dot interaction fell back to the eager path")
        return orig(n, device)

    monkeypatch.setattr(_dense, "_triu_flat_index", guarded)


def _ebc(D, F, rows, dev):
    from torchrec_b200.modules.embedding_configs import EmbeddingBagConfig
    from torchrec_b200.modules.embedding_modules import EmbeddingBagCollection

    return EmbeddingBagCollection([EmbeddingBagConfig(name=f"t{i}", embedding_dim=D, num_embeddings=rows, feature_names=[f"f{i}"]) for i in range(F)],
                                  device=dev)


@pytest.mark.parametrize("D,F", [(64, 26), (32, 40)])
def test_dlrm_wgmma_matches_torch(D, F, kernel_only):
    from torchrec_b200.models.dlrm import DLRM
    from torchrec_b200.ops import _lib
    from torchrec_b200.ops import dense as _dense
    from torchrec_b200.sparse import KeyedJaggedTensor

    torch.manual_seed(0)
    keys = [f"f{i}" for i in range(F)]
    m = DLRM(_ebc(D, F, 100, DEV), 13, [256, 128, D], [512, 256, 1], dense_device=DEV)
    B = 256
    kjt = KeyedJaggedTensor(keys=keys, values=torch.randint(0, 100, (F * B,), device=DEV), lengths=torch.ones(F * B, dtype=torch.int32, device=DEV))
    x = torch.randn(B, 13, device=DEV)
    ref = m(x, kjt)
    ref.sum().backward()
    gref = {n: p.grad.clone() for n, p in m.named_parameters() if p.grad is not None}
    m.zero_grad()
    _dense.set_dense_backend("wgmma")
    try:
        n0 = _lib.launch_count()
        out = m(x, kjt)
        out.sum().backward()
        assert _lib.launch_count() > n0
    finally:
        _dense.set_dense_backend("torch")
    assert float((out.float() - ref).abs().max()) < 0.05 * float(ref.abs().max()) + 0.02
    for n, p in m.named_parameters():
        if p.grad is None or "embedding_bags" in n:
            continue
        tol = 0.06 * float(gref[n].abs().max()) + 1e-2
        assert float((p.grad - gref[n]).abs().max()) < tol, n


def test_dlrm_dense_cuda_graphs_match_eager_d64(kernel_only):
    """capture_dense_graphs at D = 64, F = 26: training with the dense sub-modules replayed as CUDA graphs equals eager training."""
    from torchrec_b200.datasets.random import RandomRecDataset
    from torchrec_b200.models.dlrm import DLRM, DLRMTrain
    from torchrec_b200.ops import dense as _dense

    D, F = 64, 26
    _dense.set_dense_backend("wgmma")
    try:
        keys = [f"f{i}" for i in range(F)]

        def make():
            torch.manual_seed(0)
            return DLRMTrain(DLRM(_ebc(D, F, 500, DEV), 13, [64, D], [256, 64, 1], dense_device=DEV))

        a, b = make(), make()
        b.load_state_dict(a.state_dict())
        ds = RandomRecDataset(keys, 256, hash_sizes=[500] * F, ids_per_features=[1] * F, num_dense=13, manual_seed=3, num_generated_batches=4)
        batches = [x.to(DEV) for x in ds.batch_generator._generated_batches]
        with torch.no_grad():
            emb = b.model.sparse_arch(batches[0].sparse_features)
        b.model.capture_dense_graphs(batches[0].dense_features, emb)
        oa, ob = torch.optim.SGD(a.parameters(), lr=0.1), torch.optim.SGD(b.parameters(), lr=0.1)
        for i in range(4):
            la, _ = a(batches[i])
            lb, _ = b(batches[i])
            torch.testing.assert_close(lb, la, rtol=2e-2, atol=2e-3)
            for m, o, l in ((a, oa, la), (b, ob, lb)):
                o.zero_grad()
                l.backward()
                o.step()
        for (n, pa), (_, pb) in zip(a.named_parameters(), b.named_parameters()):
            torch.testing.assert_close(pb, pa, rtol=5e-2, atol=5e-3, msg=n)
    finally:
        _dense.set_dense_backend("torch")
