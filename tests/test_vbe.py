"""Variable batch per feature, op layer on the CPU: padding to a uniform stride, the inverse-index expansion and its gradient
(``torchrec_b200/ops/vbe.py``), and which padding the sharded collection picks."""
import pytest
import torch

from torchrec_b200.ops import vbe as V
from torchrec_b200.sparse.jagged_tensor import KeyedJaggedTensor


def _vbe_kjt(sizes, max_len, seed, weighted=False, off_dtype=torch.int64, use_offsets=False):
    g = torch.Generator().manual_seed(seed)
    lengths = torch.cat([torch.randint(0, max_len + 1, (b,), generator=g) for b in sizes]) if sum(sizes) else torch.zeros(0, dtype=torch.int64)
    n = int(lengths.sum())
    values = torch.randint(0, 1000, (n,), generator=g)
    weights = torch.rand(n, generator=g) if weighted else None
    keys = [f"f{i}" for i in range(len(sizes))]
    if use_offsets:
        offsets = torch.cat([torch.zeros(1, dtype=torch.int64), lengths.cumsum(0)]).to(off_dtype)
        return KeyedJaggedTensor(keys=keys, values=values, weights=weights, offsets=offsets, stride_per_key_per_rank=[[b] for b in sizes])
    return KeyedJaggedTensor(keys=keys, values=values, weights=weights, lengths=lengths.to(off_dtype), stride_per_key_per_rank=[[b] for b in sizes])


def _pad_model(offsets, sizes, B):
    """Plain-python padding: bags u >= B_f of feature f are empty and start where the feature's values end."""
    out, base = [], 0
    for bf in sizes:
        for u in range(B):
            out.append(offsets[base + min(u, bf)])
        base += bf
    out.append(offsets[base])
    return out


@pytest.mark.parametrize("off_dtype", [torch.int32, torch.int64])
@pytest.mark.parametrize("use_offsets", [False, True])
@pytest.mark.parametrize("sizes,B", [([3, 0, 7, 7, 1], 7), ([2, 5], 9), ([0, 0], 4), ([4], 4)])
def test_pad_offsets_matches_python_model(sizes, B, off_dtype, use_offsets):
    kjt = _vbe_kjt(sizes, 3, seed=len(sizes) + B, weighted=True, off_dtype=off_dtype, use_offsets=use_offsets)
    padded = V.pad_offsets(kjt, B)
    assert padded.stride() == B and padded.keys() == kjt.keys() and not padded.variable_stride_per_key()
    assert padded.offsets().tolist() == _pad_model(kjt.offsets().tolist(), sizes, B)
    assert padded.offsets().dtype == kjt.offsets().dtype
    assert padded.values() is kjt.values() and padded.weights() is kjt.weights()
    # every feature keeps its bags, in order, followed by empty ones
    lengths = padded.lengths().view(len(sizes), B)
    pos = 0
    for f, bf in enumerate(sizes):
        assert lengths[f, :bf].tolist() == kjt.lengths()[pos : pos + bf].tolist() and int(lengths[f, bf:].sum()) == 0
        pos += bf


def test_pad_offsets_rejects_a_stride_below_a_feature():
    with pytest.raises(AssertionError):
        V.pad_offsets(_vbe_kjt([2, 5], 2, seed=0), 4)


def _expand_loop(pooled, keys, inv, names, dims):
    """float64 loop: out[b, cols(name)] = pooled[inv[row(feature), b], cols(name)]."""
    row = {k: i for i, k in enumerate(keys)}
    B = inv.shape[1]
    out = torch.zeros(B, sum(dims), dtype=torch.float64)
    c = 0
    for name, d in zip(names, dims):
        feat = name.split("@")[0]
        for b in range(B):
            src = int(inv[row[feat], b]) if feat in row else b
            out[b, c : c + d] = pooled[src, c : c + d].double()
        c += d
    return out


def _reduce_loop(grad, keys, inv, names, dims, S):
    row = {k: i for i, k in enumerate(keys)}
    out = torch.zeros(S, sum(dims), dtype=torch.float64)
    c = 0
    for name, d in zip(names, dims):
        feat = name.split("@")[0]
        for b in range(inv.shape[1]):
            src = int(inv[row[feat], b]) if feat in row else b
            out[src, c : c + d] += grad[b, c : c + d].double()
        c += d
    return out


@pytest.mark.parametrize("inv_dtype", [torch.int32, torch.int64])
def test_expand_cpu_forward_backward_vs_float64_loop(inv_dtype):
    g = torch.Generator().manual_seed(3)
    names, dims = ["a", "b@t1", "b@t2", "c"], [8, 4, 12, 16]
    keys = ["c", "a", "b"]  # inverse rows in another order than the features
    S, B = 5, 11
    inv = torch.randint(0, S, (3, B), generator=g).to(inv_dtype)
    pooled = torch.randn(S, sum(dims), generator=g, requires_grad=True)
    index = V.VbeIndex((keys, inv), names, dims, src_rows=S)
    out = V.vbe_expand(pooled, index)
    assert out.shape == (B, sum(dims))
    assert torch.equal(out.detach().double(), _expand_loop(pooled.detach(), keys, inv, names, dims))
    grad = torch.randn(B, sum(dims), generator=g)
    out.backward(grad)
    torch.testing.assert_close(pooled.grad.double(), _reduce_loop(grad, keys, inv, names, dims, S), rtol=1e-6, atol=1e-6)


def test_features_without_an_inverse_row_pass_through():
    g = torch.Generator().manual_seed(4)
    names, dims = ["a", "b", "c"], [4, 8, 4]
    B = 6
    inv = torch.randint(0, B, (1, B), generator=g)
    pooled = torch.randn(B, 16, generator=g, requires_grad=True)
    out = V.vbe_expand(pooled, V.VbeIndex((["b"], inv), names, dims, src_rows=B))
    assert torch.equal(out[:, :4], pooled[:, :4]) and torch.equal(out[:, 12:], pooled[:, 12:])
    assert torch.equal(out[:, 4:12], pooled[:, 4:12][inv[0]])
    out.sum().backward()
    assert torch.equal(pooled.grad[:, :4], torch.ones(B, 4))
    assert torch.equal(pooled.grad[:, 4:12].sum(1) / 8, torch.bincount(inv[0], minlength=B).float())


def test_column_table_maps_vectors_to_inverse_rows():
    index = V.VbeIndex((["b", "a"], torch.zeros(2, 3, dtype=torch.int64)), ["a", "x", "b@t", "a@u"], [8, 4, 16, 4], src_rows=3)
    t = index.col_table(4)  # fp32: 4 elements per 16-byte vector
    assert t.col_row.tolist() == [1, 1, -1, 0, 0, 0, 0, 1]
    assert t.row_vec_off.tolist() == [0, 4, 7] and t.row_vecs.tolist() == [3, 4, 5, 6, 0, 1, 7]
    assert t.max_nv == 4 and t.cols_vec == 8 and t.has_identity
    assert index.col_table(2) is None  # bf16: a 4-column block is half a vector
    assert index.col_table(4) is t
    # the owner of names and dims keeps the tables: a later batch's index with the same inverse keys finds them
    cache = {}
    a = V.VbeIndex((["b", "a"], torch.zeros(2, 3, dtype=torch.int64)), ["a", "x", "b@t", "a@u"], [8, 4, 16, 4], src_rows=3, tables=cache)
    b = V.VbeIndex((["b", "a"], torch.ones(2, 5, dtype=torch.int64)), ["a", "x", "b@t", "a@u"], [8, 4, 16, 4], src_rows=5, tables=cache)
    c = V.VbeIndex((["a", "b"], torch.ones(2, 5, dtype=torch.int64)), ["a", "x", "b@t", "a@u"], [8, 4, 16, 4], src_rows=5, tables=cache)
    assert a.col_table(4) is b.col_table(4) and c.col_table(4) is not a.col_table(4) and len(cache) == 2


def _sharded_cpu_ebc():
    from torchrec_b200.modules.embedding_configs import EmbeddingBagConfig
    from torchrec_b200.modules.embedding_modules import EmbeddingBagCollection
    from torchrec_b200.parallel import sharding_plan as sp
    from torchrec_b200.parallel.embeddingbag import EmbeddingBagCollectionSharder, ShardedEmbeddingBagCollection
    from torchrec_b200.parallel.types import ShardingEnv

    tables = [EmbeddingBagConfig(name="t0", embedding_dim=8, num_embeddings=40, feature_names=["f0"]),
              EmbeddingBagConfig(name="t1", embedding_dim=4, num_embeddings=30, feature_names=["f1"])]
    ebc = EmbeddingBagCollection(tables, device=torch.device("cpu"))
    plan = sp.construct_module_sharding_plan(ebc, {"t0": sp.table_wise(rank=0), "t1": sp.table_wise(rank=0)}, sharder=EmbeddingBagCollectionSharder(),
                                             world_size=1, local_size=1, device_type="cpu")
    env = ShardingEnv(world_size=1, rank=0, pg=None)
    return ebc, ShardedEmbeddingBagCollection(ebc, plan, env, device=torch.device("cpu"))


@pytest.mark.parametrize("B", [6, 2])
def test_sharded_collection_on_cpu_pads_to_the_largest_feature(B):
    """Off the device, and whenever a feature has more bags than the inverse indices are wide, the batch is padded to max_f B_f and
    takes the path it always took; the values equal the unsharded collection's."""
    gold, sharded = _sharded_cpu_ebc()
    g = torch.Generator().manual_seed(1)
    l0, l1 = torch.randint(1, 3, (2,), generator=g), torch.randint(0, 3, (3,), generator=g)
    n0, n1 = int(l0.sum()), int(l1.sum())
    kjt = KeyedJaggedTensor(keys=["f0", "f1"], values=torch.cat([torch.randint(0, 40, (n0,), generator=g), torch.randint(0, 30, (n1,), generator=g)]),
                            lengths=torch.cat([l0, l1]), stride_per_key_per_rank=[[2], [3]],
                            inverse_indices=(["f0", "f1"], torch.stack([torch.randint(0, 2, (B,), generator=g), torch.randint(0, 3, (B,), generator=g)])))
    ctx = sharded.create_context()
    padded = sharded._pad_vbe(ctx, kjt)
    assert padded.stride() == 3 and not ctx.vbe_full
    out = sharded(kjt).values()
    assert out.shape == (B, 12)
    torch.testing.assert_close(out, gold(kjt).values())
