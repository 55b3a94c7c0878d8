"""wgmma dot-interaction forward/backward vs the PyTorch formulation (reference dlrm.py:210-222)."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _ref(dense, sparse):
    B, D = dense.shape
    F = sparse.shape[1]
    c = torch.cat((dense.unsqueeze(1), sparse), dim=1)
    z = torch.bmm(c, c.transpose(1, 2))
    ti = torch.triu_indices(F + 1, F + 1, offset=1, device=dense.device)
    return torch.cat((dense, z[:, ti[0], ti[1]]), dim=1)


@pytest.mark.parametrize("B,F", [(4, 26), (7, 26), (1000, 26), (513, 3), (64, 31), (5003, 26)])
@pytest.mark.parametrize("sparse_dtype", [torch.float32, torch.bfloat16])
def test_interaction_fwd_bwd(B, F, sparse_dtype):
    from torchrec_b200.ops.interaction import DotInteractionFn

    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    dense = (torch.randn(B, 128, device=dev) * 0.5).to(torch.bfloat16).requires_grad_(True)
    sparse = (torch.randn(B, F, 128, device=dev) * 0.5).to(sparse_dtype).requires_grad_(True)
    out = DotInteractionFn.apply(dense, sparse)
    n = 128 + (F + 1) * F // 2
    d32 = dense.detach().float().requires_grad_(True)
    s32 = sparse.detach().to(torch.bfloat16).float().requires_grad_(True)
    ref = _ref(d32, s32)
    torch.testing.assert_close(out[:, :n].float(), ref, rtol=2e-2, atol=8e-2)
    assert float(out[:, n:].abs().sum()) == 0.0
    g = (torch.randn(B, out.shape[1], device=dev) * 0.1).to(torch.bfloat16)
    g[:, n:] = 0
    out.backward(g)
    ref.backward(g[:, :n].float())
    tol_d = 0.03 * float(d32.grad.abs().max()) + 1e-2
    tol_s = 0.03 * float(s32.grad.abs().max()) + 1e-2
    assert float((dense.grad.float() - d32.grad).abs().max()) < tol_d
    assert float((sparse.grad.float() - s32.grad).abs().max()) < tol_s


def test_dlrm_with_wgmma_backend_matches_torch():
    from torchrec_b200.models.dlrm import DLRM
    from torchrec_b200.modules.embedding_configs import EmbeddingBagConfig
    from torchrec_b200.modules.embedding_modules import EmbeddingBagCollection
    from torchrec_b200.ops import dense as D
    from torchrec_b200.sparse import KeyedJaggedTensor

    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    keys = [f"f{i}" for i in range(26)]
    ebc = EmbeddingBagCollection([EmbeddingBagConfig(name=f"t{i}", embedding_dim=128, num_embeddings=100, feature_names=[k]) for i, k in enumerate(keys)], device=dev)
    m = DLRM(ebc, 13, [512, 256, 128], [1024, 512, 256, 1], dense_device=dev)
    B = 256
    kjt = KeyedJaggedTensor(keys=keys, values=torch.randint(0, 100, (26 * B,), device=dev), lengths=torch.ones(26 * B, dtype=torch.int32, device=dev))
    x = torch.randn(B, 13, device=dev)
    ref = m(x, kjt)
    ref.sum().backward()
    gref = {n: p.grad.clone() for n, p in m.named_parameters() if p.grad is not None}
    m.zero_grad()
    D.set_dense_backend("wgmma")
    try:
        out = m(x, kjt)
        out.sum().backward()
    finally:
        D.set_dense_backend("torch")
    assert float((out.float() - ref).abs().max()) < 0.05 * float(ref.abs().max()) + 0.02
    for n, p in m.named_parameters():
        if p.grad is None or "embedding_bags" in n:
            continue
        tol = 0.06 * float(gref[n].abs().max()) + 1e-2
        assert float((p.grad - gref[n]).abs().max()) < tol, n


@pytest.mark.gpu
def test_dlrm_dense_cuda_graphs_match_eager():
    """capture_dense_graphs: training with the dense sub-modules replayed as CUDA graphs equals eager training."""
    from torchrec_b200.models.dlrm import DLRM, DLRMTrain
    from torchrec_b200.datasets.random import RandomRecDataset
    from torchrec_b200.modules.embedding_configs import EmbeddingBagConfig
    from torchrec_b200.modules.embedding_modules import EmbeddingBagCollection
    from torchrec_b200.ops import dense as _dense

    dev = torch.device("cuda:0")
    _dense.set_dense_backend("wgmma")
    try:
        keys = [f"f{i}" for i in range(26)]

        def make():
            torch.manual_seed(0)
            ebc = EmbeddingBagCollection([EmbeddingBagConfig(name=f"t{i}", embedding_dim=128, num_embeddings=500, feature_names=[k]) for i, k in enumerate(keys)], device=dev)
            return DLRMTrain(DLRM(ebc, 13, [64, 128], [256, 64, 1], dense_device=dev))

        a, b = make(), make()
        b.load_state_dict(a.state_dict())
        ds = RandomRecDataset(keys, 256, hash_sizes=[500] * 26, ids_per_features=[1] * 26, num_dense=13, manual_seed=3, num_generated_batches=4)
        batches = [x.to(dev) for x in ds.batch_generator._generated_batches]
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
        # a batch of another size falls back to the eager modules
        small = RandomRecDataset(keys, 64, hash_sizes=[500] * 26, ids_per_features=[1] * 26, num_dense=13, manual_seed=4, num_generated_batches=1).batch_generator._generated_batches[0].to(dev)
        lb, _ = b(small)
        assert torch.isfinite(lb)
    finally:
        _dense.set_dense_backend("torch")
