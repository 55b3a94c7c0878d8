"""Quantized tables served from pinned host memory: zero-copy ``MANAGED`` lookups and ``MANAGED_CACHING`` lookups behind the HBM row
cache, bit-exact against a ``DEVICE`` module holding the same quantized bytes, plus the cache's bookkeeping, CUDA-graph capture and the
sharded modules planned with ``quant_uvm`` / ``quant_uvm_caching``."""
import numpy as np
import pytest
import torch

from torchrec_b200.ops.quant_tbe import QuantTableBatchedEmbeddingBags
from torchrec_b200.ops.tbe import EmbeddingLocation as EL
from torchrec_b200.types import DataType

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
FORMATS = {"FP32": [DataType.FP32], "FP16": [DataType.FP16], "BF16": [DataType.BF16], "INT8": [DataType.INT8], "INT4": [DataType.INT4],
           "INT2": [DataType.INT2], "FP8": [DataType.FP8], "mixed": [DataType.INT8, DataType.INT2, DataType.FP16, DataType.FP32]}
PLACEMENTS = {"managed": ([EL.MANAGED], 0.2), "cache0.01": ([EL.MANAGED_CACHING], 0.01), "cache0.25": ([EL.MANAGED_CACHING], 0.25),
              "cache1.0": ([EL.MANAGED_CACHING], 1.0), "mixed": ([EL.DEVICE, EL.MANAGED, EL.MANAGED_CACHING], 0.05)}
ROWS = [3000, 1200, 2500, 700]


def _specs(dts, dims):
    return [(f"t{i}", ROWS[i % len(ROWS)], dims[i % len(dims)], dts[i % len(dts)]) for i in range(4)]


def _pair(specs, locs, clf, pooling_mode=0, fmap=None, **kw):
    """A DEVICE module with random quantized rows and a placed module holding the same bytes."""
    ref = QuantTableBatchedEmbeddingBags(specs, fmap, pooling_mode=pooling_mode, device=DEV)
    g = torch.Generator().manual_seed(7)
    for t, (_, r, d, _) in enumerate(specs):
        ref.assign_from_float(t, torch.randn(r, d, generator=g))
    locations = [locs[t % len(locs)] for t in range(len(specs))]
    mod = QuantTableBatchedEmbeddingBags(specs, fmap, pooling_mode=pooling_mode, device=DEV, locations=locations, cache_load_factor=clf, **kw)
    for t, w in enumerate(ref.split_embedding_weights()):
        mod.split_embedding_weights()[t].copy_(w)
    mod.invalidate_cache()
    return ref, mod


def _batch(rng, B, rows_of_feature, max_len, idx_dtype, bad=True):
    """Zipf(1.05) ids (hot rows repeat within and across batches), a few out-of-range ids."""
    F = len(rows_of_feature)
    lengths = rng.integers(0, max_len + 1, size=F * B)
    vals = []
    for f, rows in enumerate(rows_of_feature):
        n = int(lengths[f * B : (f + 1) * B].sum())
        ids = (rng.zipf(1.05, size=n) - 1) % rows
        if bad and n > 4:
            ids[rng.integers(0, n, size=2)] = [-1, rows + 3]
        vals.append(ids)
    offsets = np.concatenate([[0], np.cumsum(lengths)])
    idx = torch.from_numpy(np.concatenate(vals)).to(idx_dtype).to(DEV)
    off = torch.from_numpy(offsets).to(idx_dtype).to(DEV)
    return idx, off


def _rows_of_feature(mod):
    return [mod.embedding_specs[t][1] for t in mod.feature_table_map]


@pytest.mark.parametrize("fmt", list(FORMATS))
@pytest.mark.parametrize("placement", list(PLACEMENTS))
def test_placed_lookup_bit_exact(fmt, placement):
    dts = FORMATS[fmt]
    locs, clf = PLACEMENTS[placement]
    rng = np.random.default_rng(11)
    for mode in ("sum", "mean", "weighted", "seq"):
        dims = [128] if mode == "seq" else [64, 128, 32]
        pooling = {"sum": 0, "weighted": 0, "mean": 1, "seq": 2}[mode]
        specs = _specs(dts, dims)
        fmap = [0, 1, 2, 3, 1]
        ref, mod = _pair(specs, locs, clf, pooling_mode=pooling, fmap=fmap)
        if fmt in ("FP8", "INT8", "INT4", "FP16", "BF16") and mode != "seq":
            assert mod._uniform_fmt >= 0  # the vector kernel
        rof = [specs[t][1] for t in fmap]
        for step in range(6):
            B = 4096 if step == 2 else 256  # batch 2: more distinct ids than the small caches hold
            idx, off = _batch(rng, B, rof, 3 if mode != "seq" else 2, torch.int64 if step % 2 else torch.int32)
            psw = torch.rand(idx.numel(), device=DEV) if mode == "weighted" else None
            want = ref(idx, off, psw, batch_size=B)
            got = mod(idx, off, psw, batch_size=B)
            assert torch.equal(got, want), (mode, step)


def test_host_tables_are_exact_pinned_and_stay_on_host():
    specs = [("a", 5000, 128, DataType.INT8), ("b", 3000, 64, DataType.FP8), ("c", 100, 32, DataType.FP16)]
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated(DEV)
    mod = QuantTableBatchedEmbeddingBags(specs, device=DEV, locations=[EL.MANAGED, EL.MANAGED_CACHING, EL.DEVICE], cache_load_factor=0.1)
    torch.cuda.synchronize()
    grew = torch.cuda.memory_allocated(DEV) - before
    for t in (0, 1):
        w = mod.split_embedding_weights()[t]
        assert not w.is_cuda and w.is_pinned()
        assert w.untyped_storage().nbytes() == specs[t][1] * mod._row_bytes[t]
    slots = mod.cache_slots[1]
    assert slots == 300
    device_table = 100 * mod._row_bytes[2]
    cache = slots * mod._row_bytes[1] + 4 * 3000
    metadata = slots * 9 + 2 * 8 * slots + 64 * 1024  # row_of_slot + ref, miss list + victims, small per-feature tensors
    assert grew <= device_table + cache + metadata
    mod.cuda()
    mod.to(DEV)
    for t in (0, 1):
        assert not mod.split_embedding_weights()[t].is_cuda
    ref, mod = _pair(specs, [EL.MANAGED, EL.MANAGED_CACHING, EL.DEVICE], 0.1)
    mod = mod.cuda()
    rng = np.random.default_rng(1)
    idx, off = _batch(rng, 64, _rows_of_feature(mod), 3, torch.int32)
    assert torch.equal(mod(idx, off), ref(idx, off))


def _valid(idx, off, mod, B, cached_t):
    n = 0
    o = off.cpu().long()
    ids = idx.cpu().long()
    for f, t in enumerate(mod.feature_table_map):
        if t != cached_t:
            continue
        seg = ids[o[f * B] : o[(f + 1) * B]]
        n += int(((seg >= 0) & (seg < mod.embedding_specs[t][1])).sum())
    return n


def test_cache_counts_hits_admissions_and_overflow():
    specs = [("a", 4000, 128, DataType.INT8), ("b", 500, 128, DataType.INT8)]
    ref, mod = _pair(specs, [EL.MANAGED_CACHING, EL.DEVICE], 1.0, max_admissions_per_call=64)
    rng = np.random.default_rng(3)
    B = 512
    idx, off = _batch(rng, B, _rows_of_feature(mod), 2, torch.int64)
    seg = idx[: int(off[B])]
    distinct = int(torch.unique(seg[(seg >= 0) & (seg < 4000)]).numel())
    assert distinct > 64  # more distinct ids than one call may admit: the miss list overflows
    prev = mod.cache_stats()["a"]
    admitted = []
    for _ in range(30):
        assert torch.equal(mod(idx, off), ref(idx, off))
        s = mod.cache_stats()["a"]
        d = {k: s[k] - prev[k] for k in ("lookups", "hits", "misses", "admissions")}
        assert d["hits"] + d["misses"] == d["lookups"] == _valid(idx, off, mod, B, 0)
        assert d["admissions"] <= min(64, s["slots"])
        admitted.append(d["admissions"])
        prev = s
        if d["hits"] == d["lookups"]:
            break
    assert admitted[0] == 64 and sum(admitted) == distinct  # rows left out of a full miss list are admitted by later calls
    assert prev["evictions"] == 0
    # the same batch again: every lookup hits
    mod(idx, off)
    s = mod.cache_stats()["a"]
    assert s["hits"] - prev["hits"] == s["lookups"] - prev["lookups"] > 0
    # a write after a forward invalidates the cache: the next output shows the new rows
    new = torch.randn(4000, 128, generator=torch.Generator().manual_seed(9))
    old_out = mod(idx, off)
    mod.assign_from_float(0, new)
    ref.assign_from_float(0, new)
    out = mod(idx, off)
    assert not torch.equal(out, old_out)
    assert torch.equal(out, ref(idx, off))


def test_small_cache_evicts_and_stays_exact():
    specs = [("a", 20000, 64, DataType.FP8)]
    ref, mod = _pair(specs, [EL.MANAGED_CACHING], 0.01)
    rng = np.random.default_rng(5)
    for step in range(8):
        idx, off = _batch(rng, 1024, [20000], 2, torch.int32)
        assert torch.equal(mod(idx, off), ref(idx, off))
        s = mod.cache_stats()["a"]
        assert s["admissions"] <= (step + 1) * s["slots"]
    assert s["evictions"] > 0 and 0 < s["hits"] < s["lookups"]
    assert int((mod._qc(0, "row_of_slot") >= 0).sum()) == s["slots"]


def test_forward_has_no_host_sync_and_graph_capture_matches_eager():
    specs = [("a", 6000, 128, DataType.FP8), ("b", 3000, 128, DataType.FP8), ("c", 800, 128, DataType.FP8)]
    ref, mod = _pair(specs, [EL.MANAGED_CACHING, EL.MANAGED, EL.DEVICE], 0.05)
    rng = np.random.default_rng(8)
    B, F = 256, 3

    def ids():
        return torch.cat([torch.from_numpy((rng.zipf(1.05, size=B) - 1) % r) for r in (6000, 3000, 800)]).to(DEV)

    off = torch.arange(F * B + 1, dtype=torch.int64, device=DEV)  # one id per bag: static offsets
    static = ids()
    mod(static, off)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = mod(static, off)
        out = mod(static, off)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert torch.equal(out, ref(static, off))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        mod(static, off)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        gout = mod(static, off)
    before = mod.cache_stats()["a"]
    for _ in range(5):
        new = ids()
        static.copy_(new)
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(gout, ref(new, off))
        assert torch.equal(gout, mod(new, off))
        torch.cuda.synchronize()  # a replay does not wait for the admission of an eager call
    after = mod.cache_stats()["a"]
    assert after["lookups"] - before["lookups"] == 10 * B and after["admissions"] > before["admissions"]


def _ebc_case(W):
    from torchrec_b200.inference.modules import quantize_inference_model
    from torchrec_b200.modules.embedding_configs import EmbeddingBagConfig
    from torchrec_b200.modules.embedding_modules import EmbeddingBagCollection

    tables = [EmbeddingBagConfig(name="a", embedding_dim=128, num_embeddings=3000, feature_names=["fa"]),
              EmbeddingBagConfig(name="b", embedding_dim=64, num_embeddings=5000, feature_names=["fb", "fb2"]),
              EmbeddingBagConfig(name="c", embedding_dim=128, num_embeddings=700, feature_names=["fc"])]

    class M(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.ebc = EmbeddingBagCollection(tables=tables)

    torch.manual_seed(0)
    return quantize_inference_model(M(), quantization_dtype=DataType.INT8, output_dtype=torch.float32).ebc


def _kjts(n, hs, B=128, seed=2):
    from torchrec_b200.sparse import KeyedJaggedTensor

    rng = np.random.default_rng(seed)
    keys = list(hs)
    out = []
    for _ in range(n):
        lens = torch.from_numpy(rng.integers(0, 4, size=len(keys) * B))
        vals = torch.cat([torch.from_numpy((rng.zipf(1.05, size=int(lens[i * B : (i + 1) * B].sum())) - 1) % hs[k]) for i, k in enumerate(keys)])
        out.append(KeyedJaggedTensor(keys=keys, values=vals, lengths=lens, stride=B).to(DEV))
    return out


@pytest.mark.parametrize("fused", [True, False])
def test_sharded_ebc_mixed_kernels_equal_all_quant(fused):
    from torchrec_b200.parallel import sharding_plan as sp
    from torchrec_b200.parallel.quant_embeddingbag import QuantEmbeddingBagCollectionSharder, ShardedQuantEmbeddingBagCollection
    from torchrec_b200.parallel.types import CacheParams, ShardingEnv

    W = 2 if torch.cuda.device_count() >= 2 else 1
    qebc = _ebc_case(W)

    def build(kernels):
        gens = {"a": sp.table_wise(rank=0, compute_kernel=kernels[0]), "b": sp.table_wise(rank=W - 1, compute_kernel=kernels[1]),
                "c": sp.table_wise(rank=0, compute_kernel=kernels[2])}
        plan = sp.construct_module_sharding_plan(qebc, gens, sharder=QuantEmbeddingBagCollectionSharder(), world_size=W, local_size=W, device_type="cuda")
        if kernels[1] == "quant_uvm_caching":
            plan["b"].cache_params = CacheParams(load_factor=0.02)
        return ShardedQuantEmbeddingBagCollection(qebc, plan, ShardingEnv.from_local(W, 0), device=DEV)

    base = build(["quant", "quant", "quant"])
    mixed = build(["quant_uvm", "quant_uvm_caching", "quant"])
    placed = [t for t in mixed._tbes if isinstance(t, QuantTableBatchedEmbeddingBags) and t._placed]
    assert placed and any(t._cached for t in placed)
    for t in placed:
        if t._cached:
            assert list(t.cache_slots.values()) == [100]
    for kjt in _kjts(5, {"fa": 3000, "fb": 5000, "fb2": 5000, "fc": 700}):
        if fused:
            want, got = base.forward_fused(kjt), mixed.forward_fused(kjt)
        else:
            run = lambda m: m.output_dist(None, m.compute(None, m.input_dist(None, kjt).wait().wait())).wait()
            want, got = run(base), run(mixed)
        assert torch.equal(got.values(), want.values())


def test_sharded_ec_mixed_kernels_equal_all_quant():
    from torchrec_b200.inference.modules import quantize_inference_model
    from torchrec_b200.modules.embedding_configs import EmbeddingConfig
    from torchrec_b200.modules.embedding_modules import EmbeddingCollection
    from torchrec_b200.parallel import sharding_plan as sp
    from torchrec_b200.parallel.quant_embedding import QuantEmbeddingCollectionSharder, ShardedQuantEmbeddingCollection
    from torchrec_b200.parallel.types import CacheParams, ShardingEnv

    W = 2 if torch.cuda.device_count() >= 2 else 1
    tables = [EmbeddingConfig(name="a", embedding_dim=64, num_embeddings=3000, feature_names=["fa"]),
              EmbeddingConfig(name="b", embedding_dim=64, num_embeddings=5000, feature_names=["fb"]),
              EmbeddingConfig(name="c", embedding_dim=64, num_embeddings=700, feature_names=["fc"])]

    class M(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.ec = EmbeddingCollection(tables=tables)

    torch.manual_seed(0)
    qec = quantize_inference_model(M(), quantization_dtype=DataType.INT8, output_dtype=torch.float32).ec

    def build(kernels):
        gens = {"a": sp.table_wise(rank=0, compute_kernel=kernels[0]), "b": sp.table_wise(rank=W - 1, compute_kernel=kernels[1]),
                "c": sp.table_wise(rank=0, compute_kernel=kernels[2])}
        plan = sp.construct_module_sharding_plan(qec, gens, sharder=QuantEmbeddingCollectionSharder(), world_size=W, local_size=W, device_type="cuda")
        if kernels[1] == "quant_uvm_caching":
            plan["b"].cache_params = CacheParams(load_factor=0.05)
        return ShardedQuantEmbeddingCollection(qec, plan, ShardingEnv.from_local(W, 0), device=DEV)

    base = build(["quant", "quant", "quant"])
    mixed = build(["quant_uvm", "quant_uvm_caching", "quant"])
    assert any(t._placed for t in mixed._tbes)
    for kjt in _kjts(5, {"fa": 3000, "fb": 5000, "fc": 700}):
        want, got = base(kjt), mixed(kjt)
        for k in want:
            assert torch.equal(got[k].values(), want[k].values())


def test_decomposed_quant_bag_mixed_kernels_equal_all_quant():
    from torchrec_b200.modules.embedding_configs import PoolingType
    from torchrec_b200.parallel.embedding_types import EmbeddingComputeKernel as K
    from torchrec_b200.parallel.embedding_types import GroupedEmbeddingConfig, ShardedEmbeddingTable
    from torchrec_b200.parallel.quant_embedding_kernel import QuantBatchedEmbeddingBag
    from torchrec_b200.sparse import KeyedJaggedTensor

    def config(kernels):
        ts = [ShardedEmbeddingTable(name=n, num_embeddings=r, embedding_dim=d, feature_names=[f"f{n}"], data_type=DataType.INT8, local_rows=r,
                                    local_cols=d, compute_kernel=k, fused_params={"cache_load_factor": 0.1} if k == K.QUANT_UVM_CACHING else None)
              for (n, r, d), k in zip([("a", 3000, 128), ("b", 5000, 64), ("c", 700, 32)], kernels)]
        return GroupedEmbeddingConfig(data_type=DataType.INT8, pooling=PoolingType.SUM, is_weighted=False, has_feature_processor=False,
                                      compute_kernel=kernels[0], embedding_tables=ts)

    base = QuantBatchedEmbeddingBag(config([K.QUANT] * 3), device=DEV)
    mixed = QuantBatchedEmbeddingBag(config([K.QUANT_UVM, K.QUANT_UVM_CACHING, K.QUANT]), device=DEV)
    assert mixed.emb_module.locations == [EL.MANAGED, EL.MANAGED_CACHING, EL.DEVICE]
    assert mixed.emb_module.cache_slots == {1: 500}
    g = torch.Generator().manual_seed(3)
    for t, (_, r, d, _) in enumerate(base.emb_module.embedding_specs):
        w = torch.randn(r, d, generator=g)
        base.emb_module.assign_from_float(t, w)
        mixed.emb_module.assign_from_float(t, w)
    for kjt in _kjts(5, {"fa": 3000, "fb": 5000, "fc": 700}):
        kjt = KeyedJaggedTensor(keys=kjt.keys(), values=kjt.values(), lengths=kjt.lengths(), stride=kjt.stride())
        assert torch.equal(mixed(kjt), base(kjt))
