"""Variable batch per feature on the device: the kernels of ``csrc/vbe.cu`` against models written here, and VBE batches through the
sharded collection's fused path (NVLink plane on one GPU: a single rank and 2 / 4 loopback ranks driven in lock step) against an
fp32 PyTorch reference of the unsharded collection fed the expanded batch."""
import types

import pytest
import torch

from torchrec_b200.modules.embedding_configs import EmbeddingBagConfig, PoolingType
from torchrec_b200.modules.embedding_modules import EmbeddingBagCollection
from torchrec_b200.ops import vbe as V
from torchrec_b200.ops.tbe import OptimType
from torchrec_b200.parallel import sharding_plan as sp
from torchrec_b200.parallel.embeddingbag import EmbeddingBagCollectionSharder, ShardedEmbeddingBagCollection
from torchrec_b200.parallel.engine import OptimizerSpec, ShardedLookupEngine
from torchrec_b200.parallel.sparse_plane import LoopbackGroup
from torchrec_b200.parallel.types import ShardingEnv
from torchrec_b200.sparse.jagged_tensor import KeyedJaggedTensor

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
LONG = 256  # VBE_LONG_SEG / VBE_SLICE of csrc/vbe.cu


# ---- pad_offsets ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("off_dtype", [torch.int32, torch.int64])
def test_pad_offsets_kernel_equals_cpu_model(off_dtype):
    g = torch.Generator().manual_seed(0)
    B = 300
    sizes = [B, 0, 1, 37, 256, 257, B, 0, 5]
    lengths = torch.cat([torch.randint(0, 4, (b,), generator=g) for b in sizes]).to(off_dtype)
    n = int(lengths.sum())
    values, weights = torch.randint(0, 99, (n,), generator=g), torch.rand(n, generator=g)
    keys = [f"f{i}" for i in range(len(sizes))]
    cpu = KeyedJaggedTensor(keys=keys, values=values, weights=weights, lengths=lengths, stride_per_key_per_rank=[[b] for b in sizes])
    gpu = KeyedJaggedTensor(keys=keys, values=values.to(DEV), weights=weights.to(DEV), lengths=lengths.to(DEV), stride_per_key_per_rank=[[b] for b in sizes])
    want, got = V.pad_offsets(cpu, B), V.pad_offsets(gpu, B)
    assert got.offsets().dtype == want.offsets().dtype and got.stride() == B
    assert torch.equal(got.offsets().cpu(), want.offsets())
    assert got.values() is gpu.values() and got.weights() is gpu.weights()


# ---- expand ---------------------------------------------------------------------------------------------------------------
NAMES = ["a", "b", "c@t1", "c@t2", "d", "e"]   # c feeds two tables; d has no inverse row
DIMS = [16, 64, 128, 256, 64, 128]
KEYS = ["e", "c", "a", "b"]                      # R = 4 < F = 5, rows in another order than the features


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("inv_dtype", [torch.int32, torch.int64])
def test_expand_kernel_is_a_bit_exact_gather(dtype, inv_dtype, monkeypatch):
    g = torch.Generator().manual_seed(1)
    B = 1000  # not a multiple of 32
    inv = torch.randint(0, B, (len(KEYS), B), generator=g).to(inv_dtype).to(DEV)
    pooled = torch.randn(B, sum(DIMS), generator=g).to(dtype).to(DEV)
    want = V.expand_eager(pooled, (KEYS, inv), NAMES, DIMS)
    monkeypatch.setattr(V, "expand_eager", _must_not_run)
    got = V.vbe_expand(pooled, V.VbeIndex((KEYS, inv), NAMES, DIMS, src_rows=B))
    assert got.dtype == dtype and torch.equal(got, want)


def test_expand_fewer_pooled_rows_than_samples(monkeypatch):
    g = torch.Generator().manual_seed(2)
    names, dims, keys = ["a", "b"], [32, 64], ["a", "b"]
    S, B = 37, 501
    inv = torch.randint(0, S, (2, B), generator=g).to(DEV)
    pooled = torch.randn(S, 96, generator=g).to(DEV)
    want = V.expand_eager(pooled, (keys, inv), names, dims)
    monkeypatch.setattr(V, "expand_eager", _must_not_run)
    assert torch.equal(V.vbe_expand(pooled, V.VbeIndex((keys, inv), names, dims, src_rows=S)), want)


def test_expand_index_out_of_range_gives_zeros():
    g = torch.Generator().manual_seed(3)
    B = 70
    inv = torch.randint(0, B, (len(KEYS), B), generator=g).to(DEV)
    inv[1, 5], inv[1, 6], inv[3, 69] = B, -1, 2**40   # row 1 = feature c, row 3 = feature b
    pooled = torch.randn(B, sum(DIMS), generator=g).to(DEV).requires_grad_()
    out = V.vbe_expand(pooled, V.VbeIndex((KEYS, inv), NAMES, DIMS, src_rows=B))
    ok = inv.clamp(0, B - 1)
    want = V.expand_eager(pooled.detach(), (KEYS, ok), NAMES, DIMS)
    c0, c1 = DIMS[0] + DIMS[1], DIMS[0] + DIMS[1] + DIMS[2] + DIMS[3]
    want[5:7, c0:c1] = 0
    want[69, DIMS[0] : DIMS[0] + DIMS[1]] = 0
    assert torch.equal(out.detach(), want)
    out.backward(torch.ones_like(out))   # the rejected samples belong to no segment
    assert float(pooled.grad[:, c0].sum()) == B - 2 and float(pooled.grad[:, DIMS[0]].sum()) == B - 1


def test_misaligned_columns_keep_the_eager_formulation():
    inv = torch.zeros(1, 8, dtype=torch.int64, device=DEV)
    index = V.VbeIndex((["a"], inv), ["a"], [12], src_rows=8)  # 12 bf16 columns = 24 bytes
    pooled = torch.randn(8, 12, device=DEV).bfloat16()
    assert index.kernels_serve(pooled) is None and index.kernels_serve(pooled.float()) is not None
    assert torch.equal(V.vbe_expand(pooled, index), pooled[:1].expand(8, 12))


def _must_not_run(*args, **kwargs):
    raise AssertionError("the eager path ran where the native VBE path was expected")


# ---- csr + reduce ---------------------------------------------------------------------------------------------------------
def _inv_from_lengths(lengths, n_bags, seed):
    """One inverse row: bag u is referenced by lengths[u] samples, at shuffled positions; bags >= len(lengths) by nobody."""
    g = torch.Generator().manual_seed(seed)
    row = torch.repeat_interleave(torch.arange(len(lengths)), torch.tensor(lengths))
    assert len(lengths) <= n_bags
    return row[torch.randperm(row.numel(), generator=g)]


def _fill(lengths, B):
    """Extend a list of segment lengths with length-1 segments up to B samples."""
    assert sum(lengths) <= B
    return list(lengths) + [1] * (B - sum(lengths))


def _segment_shapes():
    B = 4096
    g = torch.Generator().manual_seed(5)
    r18 = []
    while sum(r18) < B:
        r18.append(min(int(torch.randint(1, 9, (1,), generator=g)), B - sum(r18)))
    edge = [LONG - 1, LONG, LONG + 1, 2 * LONG - 1, 2 * LONG, 2 * LONG + 1, 0, 0, 3, 0]
    return {
        "identity": (B, B, [torch.arange(B)] * 3),
        "random_1_8": (B, B, [_inv_from_lengths(r18, B, 10 + r) for r in range(3)]),
        "hot_bag": (32768, 32768, [torch.zeros(32768, dtype=torch.int64), torch.full((32768,), 7), torch.zeros(32768, dtype=torch.int64)]),
        # 3 x 100 segments of 300 samples: more long segments than the card has SMs
        "many_long": (32768, 32768, [_inv_from_lengths(_fill([300] * 100, 32768), 32768, 20 + r) for r in range(3)]),
        "threshold": (B, B, [_inv_from_lengths(_fill(edge, B), B, 30 + r) for r in range(3)]),
        # fewer pooled rows than samples: bags 50..63 unreferenced, the second row's 8 bags all long
        "few_bags": (B, 64, [torch.randint(0, hi, (B,), generator=g) for hi in (50, 8, 50)]),
    }


_SHAPES = _segment_shapes()
R_NAMES, R_DIMS, R_KEYS = ["x", "y", "z", "w"], [64, 16, 128, 32], ["x", "y", "z"]   # w: identity when S == B


def _reduce_oracle(grad, keys, inv, names, dims, S):
    """float64: gpooled[u, cols(f)] = sum of grad[b, cols(f)] over the samples b with inv[r(f), b] == u."""
    row = {k: i for i, k in enumerate(keys)}
    out = torch.zeros(S, sum(dims), dtype=torch.float64, device=grad.device)
    c = 0
    for name, d in zip(names, dims):
        feat = name.split("@")[0]
        if feat in row:
            out[:, c : c + d].index_add_(0, inv[row[feat]].long(), grad[:, c : c + d].double())
        else:
            out[:, c : c + d] = grad[:, c : c + d].double()
        c += d
    return out


def _reduce(grad, index):
    pooled = torch.zeros(index.S, grad.shape[1], dtype=grad.dtype, device=grad.device, requires_grad=True)
    V.vbe_expand(pooled, index).backward(grad)
    return pooled.grad


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("shape", list(_SHAPES))
def test_reduce_is_bit_equal_to_float64_on_a_dyadic_grid(shape, dtype, monkeypatch):
    """Gradients are multiples of 1/4 in [-2, 2]: every partial sum is exact in fp32 whatever the order, so the result must equal the
    float64 sum rounded once to the output dtype."""
    monkeypatch.setattr(V, "expand_eager", _must_not_run)
    B, S, rows = _SHAPES[shape]
    names, dims = (R_NAMES, R_DIMS) if S == B else (R_NAMES[:3], R_DIMS[:3])
    inv = torch.stack(rows).to(DEV)
    g = torch.Generator().manual_seed(6)
    grad = (torch.randint(-8, 9, (B, sum(dims)), generator=g).float() / 4).to(dtype).to(DEV)
    got = _reduce(grad, V.VbeIndex((R_KEYS, inv), names, dims, src_rows=S))
    want = _reduce_oracle(grad, R_KEYS, inv, names, dims, S).to(dtype)
    assert got.dtype == dtype and torch.equal(got, want)
    referenced = torch.zeros(S, dtype=torch.bool, device=DEV).index_fill_(0, inv[1], True)
    assert float(got[:, dims[0] : dims[0] + dims[1]][~referenced].abs().sum()) == 0.0  # bags nobody references get zeros


def test_reduce_is_deterministic_and_within_the_fp32_bound():
    """Random-normal bf16 gradients, one bag referenced by every sample of every feature. Two calls on fresh buffers give the same
    bits. Bound: a sum of n terms accumulated in fp32 in any order is within (n - 1) * 2^-24 * sum|g| of the exact sum, and the
    rounding of the result to bf16 adds at most 2^-9 * |result|."""
    B = S = 32768
    names, dims, keys = [f"f{i}" for i in range(8)], [128] * 8, [f"f{i}" for i in range(8)]
    inv = torch.zeros(8, B, dtype=torch.int64, device=DEV)
    inv[1] = 5
    grad = torch.randn(B, sum(dims), generator=torch.Generator(device=DEV).manual_seed(7), device=DEV).bfloat16()
    a = _reduce(grad, V.VbeIndex((keys, inv), names, dims, src_rows=S))
    junk = torch.randn(B, sum(dims), device=DEV)  # move the allocator so the second call sees other buffers
    b = _reduce(grad.clone(), V.VbeIndex((keys, inv.clone()), names, dims, src_rows=S))
    del junk
    assert torch.equal(a, b)
    exact = _reduce_oracle(grad, keys, inv, names, dims, S)
    bound = (B - 1) * 2.0**-24 * _reduce_oracle(grad.abs(), keys, inv, names, dims, S) + 2.0**-9 * exact.abs()
    assert bool(((a.double() - exact).abs() <= bound).all())


@pytest.mark.parametrize("inv_dtype", [torch.int32, torch.int64])
def test_csr_segments_are_ascending_and_complete(inv_dtype):
    B, S, rows = _SHAPES["threshold"]
    inv = torch.stack(rows).to(inv_dtype).to(DEV)
    inv[2, 11] = S + 3  # an index outside [0, S) belongs to no segment
    index = V.VbeIndex((R_KEYS, inv), R_NAMES, R_DIMS, src_rows=S)
    seg_off, seg_b, lists = (t.cpu() for t in index.csr())
    R = inv.shape[0]
    assert seg_off[0] == 0 and int(seg_off[-1]) == R * B - 1 and bool((seg_off[1:] >= seg_off[:-1]).all())
    inv_c = inv.cpu().long()
    for r in range(R):
        lo, hi = int(seg_off[r * S]), int(seg_off[(r + 1) * S])
        bs = seg_b[lo:hi].long()
        valid = torch.arange(B)[(inv_c[r] >= 0) & (inv_c[r] < S)]
        assert torch.equal(bs.sort().values, valid)                      # every sample exactly once per row
        bag = torch.repeat_interleave(torch.arange(S), (seg_off[r * S + 1 : (r + 1) * S + 1] - seg_off[r * S : (r + 1) * S]).long())
        assert torch.equal(inv_c[r][bs], bag)                            # in the segment of the bag it references
        same = bag[1:] == bag[:-1]
        assert bool((bs[1:][same] > bs[:-1][same]).all())                # ascending inside a segment
    lens = seg_off[1:] - seg_off[:-1]
    assert int(lists[0]) == int((lens > LONG).sum()) and int(lists[1]) == int(((lens[lens > LONG] + LONG - 1) // LONG).sum())


def test_expand_and_reduce_replay_in_a_cuda_graph():
    g = torch.Generator().manual_seed(8)
    B = S = 2048
    names, dims, keys = R_NAMES, R_DIMS, R_KEYS

    def draw(seed):
        gg = torch.Generator().manual_seed(seed)
        rows = [_inv_from_lengths(_fill([700, 300, 1, 0, 9], B), B, seed + r) for r in range(3)]
        return torch.stack(rows).to(DEV), torch.randn(S, sum(dims), generator=gg).to(DEV), (torch.randint(-8, 9, (B, sum(dims)), generator=gg).float() / 4).to(DEV)

    inv, pooled, grad = draw(1)
    pooled.requires_grad_()
    tables = {}  # the static column table is built (a host-to-device copy) during warm-up, outside the capture

    def step():
        out = V.vbe_expand(pooled, V.VbeIndex((keys, inv), names, dims, src_rows=S, tables=tables))
        out.backward(grad)
        return out

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        step()
    torch.cuda.current_stream().wait_stream(side)
    pooled.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = step()
    for seed in (2, 3):
        inv2, pooled2, grad2 = draw(seed)
        with torch.no_grad():
            inv.copy_(inv2), pooled.copy_(pooled2), grad.copy_(grad2)
        graph.replay()
        assert torch.equal(out, V.expand_eager(pooled2, (keys, inv2), names, dims))
        assert torch.equal(pooled.grad, _reduce_oracle(grad2, keys, inv2, names, dims, S).float())


# ---- VBE batches through the sharded collection ---------------------------------------------------------------------------------
T_DIMS, T_ROWS = [128, 64, 128, 32, 256], [500, 37, 1201, 64, 90]
LR, EPS = 0.1, 1e-3


def _tables(pooling):
    return [EmbeddingBagConfig(name=f"t{i}", embedding_dim=d, num_embeddings=r, feature_names=[f"f{i}"] if i != 1 else ["f1", "f1b"], pooling=pooling)
            for i, (d, r) in enumerate(zip(T_DIMS, T_ROWS))]


def _plan(kind, tables, W):
    gens = {}
    for i, t in enumerate(tables):
        k = kind if kind != "mixed" else ["tw", "rw", "cw", "tw", "rw"][i % 5]
        if k == "tw":
            gens[t.name] = sp.table_wise(rank=i % W)
        elif k == "rw":
            gens[t.name] = sp.row_wise()
        else:
            gens[t.name] = sp.column_wise(ranks=[(i + j) % W for j in range(2)])
    return gens


def _vbe_batch(tables, B, max_len, weighted, seed, keep_one_full=True):
    """A VBE batch (device KJT with inverse indices over every feature) and the same batch expanded to B samples per feature as
    per-feature (values, lengths, weights) lists for the reference."""
    g = torch.Generator().manual_seed(seed)
    keys, lens, vals, wts, sizes, inv, expanded = [], [], [], [], [], [], []
    choices = [1, B // 8, B // 3, B]
    for t in tables:
        for fn in t.feature_names:
            bf = choices[int(torch.randint(0, len(choices), (1,), generator=g))]
            if keep_one_full and not keys:
                bf = B
            l = torch.randint(0, max_len + 1, (bf,), generator=g)
            v = torch.randint(0, t.num_embeddings, (int(l.sum()),), generator=g)
            w = torch.rand(v.numel(), generator=g)
            row = torch.randint(0, bf, (B,), generator=g)
            keys.append(fn), lens.append(l), vals.append(v), wts.append(w), sizes.append(bf), inv.append(row)
            off = torch.cat([torch.zeros(1, dtype=torch.int64), l.cumsum(0)])
            pos = torch.cat([torch.arange(int(off[u]), int(off[u + 1])) for u in row.tolist()]) if B else torch.zeros(0, dtype=torch.int64)
            expanded.append((v[pos].to(DEV), l[row].to(DEV), w[pos].to(DEV) if weighted else None))
    kjt = KeyedJaggedTensor(keys=keys, values=torch.cat(vals).to(DEV), lengths=torch.cat(lens).to(DEV), weights=torch.cat(wts).to(DEV) if weighted else None,
                            stride_per_key_per_rank=[[b] for b in sizes], inverse_indices=(keys, torch.stack(inv).to(DEV)))
    return kjt, expanded


class _Reference:
    """fp32 PyTorch model of the unsharded collection with row-wise Adagrad (state per row and column shard)."""

    def __init__(self, tables, full, col_shards, mean):
        self.tables, self.mean, self.col_shards = tables, mean, col_shards
        self.w = {k: v.clone() for k, v in full.items()}
        self.state = {t.name: torch.zeros(t.num_embeddings, len(col_shards[t.name]), device=DEV) for t in tables}

    def _features(self):
        return [(t, fi) for t in self.tables for fi in t.feature_names]

    def forward(self, expanded, B):
        outs = []
        for (t, _), (v, l, w) in zip(self._features(), expanded):
            rows = self.w[t.name][v] * (w.unsqueeze(1) if w is not None else 1.0)
            seg = torch.repeat_interleave(torch.arange(B, device=DEV), l)
            out = torch.zeros(B, t.embedding_dim, device=DEV).index_add_(0, seg, rows)
            outs.append(out / l.clamp(min=1).unsqueeze(1) if self.mean else out)
        return torch.cat(outs, 1)

    def update(self, batches, grads, scale):
        """One optimizer step from the (expanded batch, output gradient) of every rank."""
        B = grads[0].shape[0]
        gw = {t.name: torch.zeros_like(self.w[t.name]) for t in self.tables}
        for expanded, grad in zip(batches, grads):
            c = 0
            for (t, _), (v, l, w) in zip(self._features(), expanded):
                d = t.embedding_dim
                seg = torch.repeat_interleave(torch.arange(B, device=DEV), l)
                gr = grad[:, c : c + d][seg] * scale
                if w is not None:
                    gr = gr * w.unsqueeze(1)
                if self.mean:
                    gr = gr / l.clamp(min=1)[seg].unsqueeze(1)
                gw[t.name].index_add_(0, v, gr)
                c += d
        for t in self.tables:
            for k, (co, cn) in enumerate(self.col_shards[t.name]):
                gs = gw[t.name][:, co : co + cn]
                touched = gs.abs().sum(1) > 0
                self.state[t.name][:, k] += (gs * gs).sum(1) / cn
                step = (LR / (self.state[t.name][:, k].sqrt() + EPS)).unsqueeze(1) * gs
                self.w[t.name][:, co : co + cn] -= step * touched.unsqueeze(1)


def _check_tables(ref, tables, shard_views):
    for t in tables:
        got_w = torch.zeros_like(ref.w[t.name])
        got_s = torch.zeros_like(ref.state[t.name])
        for shard, wview, st, _tbe in shard_views:
            if shard.name == t.name:
                got_w[shard.row_off : shard.row_off + shard.rows, shard.col_off : shard.col_off + shard.cols] = wview
                k = [co for co, _ in ref.col_shards[t.name]].index(shard.col_off)
                got_s[shard.row_off : shard.row_off + shard.rows, k] = st["momentum1"]
        torch.testing.assert_close(got_w, ref.w[t.name], rtol=2e-4, atol=2e-5)
        torch.testing.assert_close(got_s, ref.state[t.name], rtol=2e-4, atol=1e-6)


@pytest.mark.parametrize("W", [1, 2, 4])
@pytest.mark.parametrize("kind", ["tw", "rw", "cw", "mixed"])
@pytest.mark.parametrize("weighted,mean", [(False, False), (True, False), (False, True)])
def test_vbe_through_the_plane_virtual_ranks(W, kind, weighted, mean, monkeypatch):
    """W virtual ranks in lock step, three training steps. Per rank and step: pad to B, route through the plane, lookup + output
    dist, MEAN divisor from the padded lengths, expansion; backward through the expansion's reduce into the gradient push and the
    fused row-wise Adagrad."""
    monkeypatch.setattr(V, "expand_eager", _must_not_run)
    torch.manual_seed(7)
    B, max_len = 48, 5
    tables = _tables(PoolingType.MEAN if mean else PoolingType.SUM)
    ebc = EmbeddingBagCollection(tables=tables, is_weighted=weighted, device=torch.device("cpu"))
    plan = sp.construct_module_sharding_plan(ebc, _plan(kind, tables, W), sharder=EmbeddingBagCollectionSharder(), world_size=W, local_size=W, device_type="cuda")
    full = {t.name: (torch.randn(t.num_embeddings, t.embedding_dim, device=DEV) * 0.1) for t in tables}
    names = [f for t in tables for f in t.feature_names]
    feature_table = [ti for ti, t in enumerate(tables) for _ in t.feature_names]
    emb_dims = [tables[ti].embedding_dim for ti in feature_table]
    total_cols = sum(emb_dims)
    group = LoopbackGroup(W, DEV)
    engines = []
    for r in range(W):
        eng = ShardedLookupEngine(tables, names, feature_table, plan, ShardingEnv.from_loopback(W, r, group), DEV, pooled=True, is_weighted=weighted,
                                  opt_specs={t.name: OptimizerSpec(optim=OptimType.EXACT_ROWWISE_ADAGRAD, lr=LR, eps=EPS) for t in tables}, output_dtype=torch.float32)
        for shard, wview, _st, _tbe in eng.local_shard_views():
            wview.copy_(full[shard.name][shard.row_off : shard.row_off + shard.rows, shard.col_off : shard.col_off + shard.cols])
        engines.append(eng)
    col_shards = {t.name: sorted({(s.col_off, s.cols) for s in engines[0]._table_shards[ti]}) for ti, t in enumerate(tables)}
    ref = _Reference(tables, full, col_shards, mean)
    # the sharded module's own MEAN divisor, run on what the method reads of the module
    module_view = [types.SimpleNamespace(_feature_names=names, _post_mean_feature=list(eng._post_mean_feature), _embedding_dims=emb_dims, _total_cols=total_cols)
                   for eng in engines]
    for step in range(3):
        batches = [_vbe_batch(tables, B, max_len, weighted, 100 * step + r) for r in range(W)]
        padded = [V.pad_offsets(kjt, B) for kjt, _ in batches]
        index = [V.VbeIndex(kjt.inverse_indices(), names, emb_dims, src_rows=B) for kjt, _ in batches]
        ids = [engines[r].plane_input_dist(padded[r], None, total_cols, capacity=len(names) * B * max_len) for r in range(W)]
        for r in range(W):
            ids[r].plane.forward_kernels(ids[r], 0)
        grads, leaves = [], []
        for r in range(W):
            pooled = ids[r].plane.forward_finish(0).clone().requires_grad_()
            vals = pooled
            if any(engines[r]._post_mean_feature):  # row-sharded MEAN features: divided by the PADDED batch's lengths before the expansion
                vals = pooled * ShardedEmbeddingBagCollection._mean_divisor(module_view[r], padded[r])
            out = V.vbe_expand(vals, index[r])
            torch.testing.assert_close(out, ref.forward(batches[r][1], B), rtol=1e-4, atol=1e-5)
            grads.append(torch.randn(B, total_cols, device=DEV))
            out.backward(grads[-1])
            leaves.append(pooled)
        if W == 1:  # a single rank has no inbox: the fused backward reads the gradient where autograd left it
            ids[0].plane.backward(ids[0], leaves[0].grad, 1.0)
        else:
            for r in range(W):
                ids[r].plane.backward_push(leaves[r].grad)
            for r in range(W):
                ids[r].plane.backward_apply(ids[r], 1.0 / W)
        torch.cuda.synchronize()
        assert all(int(i.plane.overflow.item()) == 0 for i in ids)
        ref.update([b for _, b in batches], grads, 1.0 / W)
    _check_tables(ref, tables, [v for eng in engines for v in eng.local_shard_views()])


def _sharded_module(kind, weighted, mean):
    from torchrec_b200.optim.apply_optimizer_in_backward import apply_optimizer_in_backward
    from torchrec_b200.optim.rowwise_adagrad import RowWiseAdagrad
    from torchrec_b200.parallel.model_parallel import DistributedModelParallel
    from torchrec_b200.parallel.types import ShardingPlan

    tables = _tables(PoolingType.MEAN if mean else PoolingType.SUM)
    ebc = EmbeddingBagCollection(tables=tables, is_weighted=weighted, device=torch.device("meta"))
    apply_optimizer_in_backward(RowWiseAdagrad, ebc.parameters(), {"lr": LR, "eps": EPS})
    plan = sp.construct_module_sharding_plan(ebc, _plan(kind, tables, 1), sharder=EmbeddingBagCollectionSharder(), world_size=1, local_size=1, device_type="cuda")

    class Wrap(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.ebc = ebc

        def forward(self, k):
            return self.ebc(k).values()

    dmp = DistributedModelParallel(Wrap(), device=DEV, plan=ShardingPlan({"ebc": plan}), sharders=[EmbeddingBagCollectionSharder()])
    sharded = dmp.module.ebc
    full = {t.name: (torch.randn(t.num_embeddings, t.embedding_dim, device=DEV) * 0.1) for t in tables}
    with torch.no_grad():
        for shard, wview, _st, _tbe in sharded._engine.local_shard_views():
            wview.copy_(full[shard.name][shard.row_off : shard.row_off + shard.rows, shard.col_off : shard.col_off + shard.cols])
    col_shards = {t.name: sorted({(s.col_off, s.cols) for s in sharded._engine._table_shards[ti]}) for ti, t in enumerate(tables)}
    return tables, dmp, sharded, _Reference(tables, full, col_shards, mean)


def _forbid_other_paths(monkeypatch):
    monkeypatch.setattr(V, "expand_eager", _must_not_run)
    monkeypatch.setattr(ShardedLookupEngine, "input_dist", _must_not_run)
    monkeypatch.setattr(ShardedLookupEngine, "input_dist_routed", _must_not_run)


@pytest.mark.parametrize("kind", ["tw", "rw", "cw", "mixed"])
@pytest.mark.parametrize("weighted,mean", [(False, False), (True, False), (False, True)])
def test_sharded_collection_trains_on_vbe_batches_through_the_fused_path(kind, weighted, mean, monkeypatch):
    """The sharded module itself on one rank: input dist on the plane, fused lookup + output dist, expansion, three steps of fused
    row-wise Adagrad. The eager expansion and the non-plane input dists raise."""
    _forbid_other_paths(monkeypatch)
    torch.manual_seed(11)
    B = 48
    tables, dmp, sharded, ref = _sharded_module(kind, weighted, mean)
    kjt, expanded = _vbe_batch(tables, B, 5, weighted, 1)
    for step in range(3):
        out = dmp(kjt)
        assert out.shape == (B, sum(t.embedding_dim * len(t.feature_names) for t in tables))
        torch.testing.assert_close(out, ref.forward(expanded, B), rtol=1e-4, atol=1e-5)
        grad = torch.randn(out.shape, device=DEV)
        out.backward(grad)
        ref.update([expanded], [grad], 1.0)
    torch.cuda.synchronize()
    _check_tables(ref, tables, sharded._engine.local_shard_views())


def test_feature_with_more_bags_than_samples_keeps_the_old_padding():
    tables, dmp, sharded, ref = _sharded_module("tw", False, False)
    B = 48
    kjt, _ = _vbe_batch(tables, B, 3, False, 2)
    keys, inv = kjt.inverse_indices()
    narrow = KeyedJaggedTensor(keys=kjt.keys(), values=kjt.values(), lengths=kjt.lengths(), stride_per_key_per_rank=kjt.stride_per_key_per_rank(),
                               inverse_indices=(keys, inv[:, :20].contiguous()))
    ctx = sharded.create_context()
    assert sharded._pad_vbe(ctx, narrow).stride() == B and not ctx.vbe_full   # B_f = 48 > 20 samples: padded to max_f B_f
    ctx = sharded.create_context()
    assert sharded._pad_vbe(ctx, kjt).stride() == B and ctx.vbe_full
    assert dmp(narrow).shape[0] == 20


def test_vbe_step_does_not_synchronise_the_host(monkeypatch):
    """After warm-up a VBE forward + backward through the sharded module issues no blocking host call (the per-feature batch sizes
    travel in a pinned, non-blocking copy)."""
    _forbid_other_paths(monkeypatch)
    tables, dmp, sharded, ref = _sharded_module("tw", False, False)
    B = 48
    kjt, _ = _vbe_batch(tables, B, 5, False, 3)
    grad = torch.randn(B, sum(t.embedding_dim * len(t.feature_names) for t in tables), device=DEV)
    for _ in range(4):
        dmp(kjt).backward(grad)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        dmp(kjt).backward(grad)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()


def test_context_built_on_a_side_stream_survives_until_the_backward(monkeypatch):
    """Pipelined training runs ``input_dist`` on a data-dist stream and forward + backward on the default stream after
    ``ctx.record_stream``. The context's expansion index (inverse indices, CSR) is allocated on the side stream; once recorded, the
    allocator must not hand its blocks to the side stream's next batches while the default stream still has the reduce queued. Here
    the default stream is kept busy, later batches' input dists run ahead on the side stream with the same allocation sizes, and
    the gradient of the first batch must still equal the oracle."""
    _forbid_other_paths(monkeypatch)
    tables, dmp, sharded, ref = _sharded_module("tw", False, False)
    B = 4096
    names, dims = sharded._embedding_names, sharded._embedding_dims
    base, _ = _vbe_batch(tables, B, 2, False, 50)

    def with_inverse(seed):  # the same bags every time (one id volume for the plane's regions), other inverse indices
        g = torch.Generator().manual_seed(seed)
        rows = torch.stack([torch.randint(0, bf, (B,), generator=g) for bf in base.stride_per_key()]).to(DEV)
        return KeyedJaggedTensor(keys=base.keys(), values=base.values(), lengths=base.lengths(), stride_per_key_per_rank=base.stride_per_key_per_rank(),
                                 inverse_indices=(base.keys(), rows))

    batches = [with_inverse(i) for i in range(3)]
    for seed in (7, 8):   # warm-up: plane buffers, capacity measurement, column table
        sharded(with_inverse(seed)).values().sum().backward()
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    cur = torch.cuda.current_stream()
    ctx = sharded.create_context()
    with torch.cuda.stream(side):
        dist = sharded.input_dist(ctx, batches[0]).wait().wait()
        done = torch.cuda.Event()
        done.record(side)
    assert ctx.vbe_full and ctx.vbe_index._csr is not None
    ctx.record_stream(cur)
    cur.wait_event(done)
    keys, inv = batches[0].inverse_indices()
    inv_copy = inv.clone()
    out = sharded.compute_and_output_dist(ctx, dist).wait().values()
    grad = (torch.randint(-8, 9, out.shape, device=DEV).float() / 4)
    pooled_grad = []
    out.grad_fn.register_hook(lambda gin, gout: pooled_grad.append(gin[0]))
    # keep the default stream busy so the host runs ahead of it, then queue the backward behind that work
    busy = torch.randn(4096, 4096, device=DEV)
    for _ in range(40):
        busy = busy @ busy * 1e-3
    out.backward(grad)
    del ctx, dist, out
    with torch.cuda.stream(side):   # later batches: same sizes, same stream, while reduce(0) may still be queued
        for kjt in batches[1:]:
            sharded.input_dist(sharded.create_context(), kjt).wait().wait()
    torch.cuda.synchronize()
    want = _reduce_oracle(grad, list(keys), inv_copy, names, dims, B).float()
    assert torch.equal(pooled_grad[0], want)
