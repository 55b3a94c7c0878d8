"""The composable per-group kernels / grouped lookups on an H100: CUDA TBE kernels vs the CPU reference path of the same classes."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _groups(kernel, fused):
    from torchrec_b200.modules.embedding_configs import DataType, PoolingType
    from torchrec_b200.parallel.embedding_types import EmbeddingComputeKernel as K
    from torchrec_b200.parallel.embedding_types import GroupedEmbeddingConfig, ShardedEmbeddingTable

    def tb(name, rows, dim, feats):
        return ShardedEmbeddingTable(num_embeddings=max(rows, 1), embedding_dim=dim, name=name, feature_names=feats, embedding_names=feats, compute_kernel=kernel,
                                     local_rows=rows, local_cols=dim)

    # an EMPTY shard (0 rows) in the middle: a rank the plan gave no rows keeps the feature layout (row-wise / table-row-wise shardings)
    tables = [tb("a", 64, 128, ["fa"]), tb("z", 0, 64, ["fz"]), tb("b", 100, 64, ["fb1", "fb2"])]
    return [GroupedEmbeddingConfig(DataType.FP32, PoolingType.SUM, False, False, kernel, tables, fused_params=fused)]


def _batch(dev, B=16, seed=0):
    from torchrec_b200.sparse import KeyedJaggedTensor

    g = torch.Generator().manual_seed(seed)
    lens = torch.randint(0, 5, (4 * B,), generator=g)
    lens[B : 2 * B] = 0  # nothing is ever routed to the empty shard
    hs = [64, 1, 100, 100]
    vals = torch.cat([torch.randint(0, hs[f], (int(lens[f * B : (f + 1) * B].sum()),), generator=g) for f in range(4)])
    return KeyedJaggedTensor.from_lengths_sync(["fa", "fz", "fb1", "fb2"], vals, lens).to(dev)


@pytest.mark.parametrize("optimizer", ["exact_sgd", "exact_row_wise_adagrad", "adam"])
def test_grouped_pooled_lookup_cuda_matches_cpu(optimizer):
    from torchrec_b200.parallel.embedding_lookup import GroupedPooledEmbeddingsLookup
    from torchrec_b200.parallel.embedding_types import EmbeddingComputeKernel as K

    fused = {"optimizer": optimizer, "learning_rate": 0.05}
    cpu = GroupedPooledEmbeddingsLookup(_groups(K.FUSED, fused), device=torch.device("cpu"))
    gpu = GroupedPooledEmbeddingsLookup(_groups(K.FUSED, fused), device=torch.device("cuda:0"))
    gpu.load_state_dict({k: v.cuda() for k, v in cpu.state_dict().items()})
    for step in range(3):
        b = _batch(torch.device("cpu"), seed=step)
        oc = cpu(b)
        og = gpu(b.to(torch.device("cuda:0")))
        torch.testing.assert_close(og.cpu(), oc, rtol=1e-5, atol=1e-5)
        w = torch.randn(oc.shape, generator=torch.Generator().manual_seed(100 + step))
        (oc * w).sum().backward()
        (og * w.cuda()).sum().backward()
    sc, sg = cpu.state_dict(), gpu.state_dict()
    for k in sc:
        torch.testing.assert_close(sg[k].cpu(), sc[k], rtol=2e-4, atol=2e-5, msg=lambda m: f"{optimizer} {k}: {m}")
    assert [type(o).__name__ for o in gpu.fused_optimizers()] == ["EmbeddingFusedOptimizer"]


def test_dense_and_sequence_kernels_cuda():
    from torchrec_b200.parallel.embedding_lookup import GroupedEmbeddingsLookup, GroupedPooledEmbeddingsLookup
    from torchrec_b200.parallel.embedding_types import EmbeddingComputeKernel as K

    dev = torch.device("cuda:0")
    dense_c = GroupedPooledEmbeddingsLookup(_groups(K.DENSE, None), device=torch.device("cpu"))
    dense_g = GroupedPooledEmbeddingsLookup(_groups(K.DENSE, None), device=dev)
    dense_g.load_state_dict({k: v.cuda() for k, v in dense_c.state_dict().items()})
    b = _batch(torch.device("cpu"))
    oc, og = dense_c(b), dense_g(b.to(dev))
    torch.testing.assert_close(og.cpu(), oc, rtol=1e-5, atol=1e-5)
    oc.sum().backward()
    og.sum().backward()
    (_, pc), = list(dense_c.named_parameters())
    (_, pg), = list(dense_g.named_parameters())
    torch.testing.assert_close(pg.grad.cpu(), pc.grad, rtol=1e-5, atol=1e-5)

    from torchrec_b200.modules.embedding_configs import DataType, PoolingType
    from torchrec_b200.parallel.embedding_types import GroupedEmbeddingConfig, ShardedEmbeddingTable

    t = ShardedEmbeddingTable(num_embeddings=50, embedding_dim=32, name="s", feature_names=["f"], embedding_names=["f"], compute_kernel=K.FUSED, local_rows=50, local_cols=32)
    g = [GroupedEmbeddingConfig(DataType.FP32, PoolingType.NONE, False, False, K.FUSED, [t], fused_params={"optimizer": "exact_sgd", "learning_rate": 0.1})]
    sc, sg = GroupedEmbeddingsLookup(g, device=torch.device("cpu")), GroupedEmbeddingsLookup(g, device=dev)
    sg.load_state_dict({k: v.cuda() for k, v in sc.state_dict().items()})
    from torchrec_b200.sparse import KeyedJaggedTensor

    kj = KeyedJaggedTensor.from_lengths_sync(["f"], torch.tensor([3, 7, 7, 49, 0]), torch.tensor([2, 0, 3]))
    rc, rg = sc(kj), sg(kj.to(dev))
    torch.testing.assert_close(rg.cpu(), rc)
    rc.sum().backward()
    rg.sum().backward()
    torch.testing.assert_close(sg.state_dict()["s.weight"].cpu(), sc.state_dict()["s.weight"], rtol=1e-5, atol=1e-6)
