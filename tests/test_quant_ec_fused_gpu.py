"""The fused sequence path of ShardedQuantEmbeddingCollection (kjt_route with per-id output positions + quantized sequence lookups
storing into one flat output on the first device) against the decomposed input_dist / compute / output_dist of the same module
(bit-equal) and against the unsharded quantized module (close). One-GPU plans put several row and column shards of one table on
cuda:0, so row routing runs with a single device; the two-GPU case skips on one GPU."""
import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
D = 64
ROWS = {"a": 300, "b": 1000, "c": 77, "d": 500}
FEATURES = {"a": ["fa"], "b": ["fb", "fb2"], "c": ["fc"], "d": ["fd"]}
KEYS = ["fb2", "fa", "fd", "fc", "fb"]
HASH = {"fa": 300, "fb": 1000, "fb2": 1000, "fc": 77, "fd": 500}


def _qec(fmt, out_dtype, need_indices=False):
    from torchrec_b200.inference.modules import quantize_inference_model
    from torchrec_b200.modules.embedding_configs import EmbeddingConfig
    from torchrec_b200.modules.embedding_modules import EmbeddingCollection
    from torchrec_b200.types import DataType

    tables = [EmbeddingConfig(name=t, embedding_dim=D, num_embeddings=r, feature_names=FEATURES[t]) for t, r in ROWS.items()]

    class M(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.ec = EmbeddingCollection(tables=tables, need_indices=need_indices)

    torch.manual_seed(0)
    if fmt == "mixed":  # four row formats, mixed inside every (rank, width) group
        per = {"a": DataType.INT8, "b": DataType.FP8, "c": DataType.INT4, "d": DataType.INT2}
        return quantize_inference_model(M(), quantization_dtype=DataType.INT8, per_table_weight_dtype=per, output_dtype=out_dtype).ec
    return quantize_inference_model(M(), quantization_dtype=getattr(DataType, fmt), output_dtype=out_dtype).ec


def _ps(kind, shards, kernel="quant"):
    """shards: (rank, row_off, col_off, rows, cols)"""
    from torchrec_b200.parallel.types import CacheParams, EnumerableShardingSpec, ParameterSharding, ShardMetadata

    spec = EnumerableShardingSpec([ShardMetadata(shard_sizes=[r, c], shard_offsets=[ro, co], placement=f"rank:{k}/cuda:{k}") for k, ro, co, r, c in shards])
    ps = ParameterSharding(sharding_type=kind, compute_kernel=kernel, ranks=[s[0] for s in shards], sharding_spec=spec)
    if kernel == "quant_uvm_caching":
        ps.cache_params = CacheParams(load_factor=0.05)
    return ps


def _tw(t, k=0, kernel="quant"):
    return _ps("table_wise", [(k, 0, 0, ROWS[t], D)], kernel)


def _cw(t, ks=(0, 0), kernel="quant"):
    return _ps("column_wise", [(k, 0, i * D // len(ks), ROWS[t], D // len(ks)) for i, k in enumerate(ks)], kernel)


def _rw(t, cuts, ks=None, kernel="quant"):
    edges = [0] + list(cuts) + [ROWS[t]]
    ks = ks or [0] * (len(edges) - 1)
    return _ps("row_wise", [(k, lo, 0, hi - lo, D) for k, lo, hi in zip(ks, edges[:-1], edges[1:])], kernel)


def _grid(t, cuts, ks=None, kernel="quant"):
    edges = [0] + list(cuts) + [ROWS[t]]
    cells = [(lo, hi, c) for c in (0, D // 2) for lo, hi in zip(edges[:-1], edges[1:])]
    ks = ks or [0] * len(cells)
    return _ps("table_row_wise", [(k, lo, c, hi - lo, D // 2) for k, (lo, hi, c) in zip(ks, cells)], kernel)


def _ragged(t, cut, halves_first, ks=(0, 0, 0), kernel="quant"):
    """rows [0, cut) and [cut, rows): one of the two in column halves, the other whole width"""
    R, h = ROWS[t], D // 2
    if halves_first:
        cells = [(0, 0, cut, h), (0, h, cut, h), (cut, 0, R - cut, D)]
    else:
        cells = [(0, 0, cut, D), (cut, 0, R - cut, h), (cut, h, R - cut, h)]
    return _ps("table_row_wise", [(k, ro, co, r, c) for k, (ro, co, r, c) in zip(ks, cells)], kernel)


PLANS = {
    "tw": lambda: {t: _tw(t) for t in ROWS},
    "cw": lambda: {"a": _cw("a"), "b": _cw("b"), "c": _tw("c"), "d": _cw("d")},
    "rw": lambda: {"a": _rw("a", [100, 200]), "b": _rw("b", [250, 500, 750]), "c": _rw("c", [40]), "d": _rw("d", [10])},
    "twrw": lambda: {"a": _grid("a", [150]), "b": _grid("b", [100, 900]), "c": _tw("c"), "d": _grid("d", [333])},
    "mixed": lambda: {"a": _rw("a", [100, 200]), "b": _cw("b"), "c": _tw("c"), "d": _grid("d", [250])},
    # row shards cut into different column slices
    "ragged": lambda: {"a": _ragged("a", 150, halves_first=True), "b": _cw("b"), "c": _tw("c"), "d": _ragged("d", 100, halves_first=False)},
}


def _sharded(qec, plan):
    from torchrec_b200.parallel.quant_embedding import ShardedQuantEmbeddingCollection
    from torchrec_b200.parallel.types import ShardingEnv

    W = 1 + max(s.placement.rank() if hasattr(s.placement, "rank") else int(str(s.placement).split("/")[0].split(":")[1])
                for ps in plan.values() for s in ps.sharding_spec.shards)
    return ShardedQuantEmbeddingCollection(qec, plan, ShardingEnv.from_local(W, 0), device=DEV)


def _kjt(g, B, idx_dtype, empty_key=None, bad=True, long=False):
    """long: 10-60 ids per bag (the route's warp-per-bag writer); otherwise 0-5 (its thread-per-bag writer)"""
    from torchrec_b200.sparse import KeyedJaggedTensor

    lens = torch.randint(10, 61, (len(KEYS) * B,), generator=g) if long else torch.randint(0, 6, (len(KEYS) * B,), generator=g)
    lens[torch.rand(lens.shape, generator=g) < 0.2] = 0  # empty bags
    if empty_key is not None:
        i = KEYS.index(empty_key)
        lens[i * B : (i + 1) * B] = 0
    vals = []
    for i, k in enumerate(KEYS):
        n = int(lens[i * B : (i + 1) * B].sum())
        v = torch.randint(0, HASH[k], (n,), generator=g)
        if bad and n > 2:  # a negative and an out-of-range id
            v[0], v[-1] = -3, HASH[k] + 17
        vals.append(v)
    return KeyedJaggedTensor(keys=KEYS, values=torch.cat(vals).to(idx_dtype), lengths=lens.to(idx_dtype), stride=B)


def _decomposed(m, kjt):
    ctx = m.create_context()
    return m.output_dist(ctx, m.compute(ctx, m.input_dist(ctx, kjt).wait().wait())).wait()


def _assert_equal(got, want):
    assert list(got) == list(want)
    for k in want:
        assert torch.equal(got[k].values(), want[k].values()), k
        assert torch.equal(got[k].lengths(), want[k].lengths()), k
        gw, ww = got[k].weights_or_none(), want[k].weights_or_none()
        assert (gw is None) == (ww is None) and (gw is None or torch.equal(gw, ww)), k


@pytest.mark.parametrize("out_dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("kind", list(PLANS))
@pytest.mark.parametrize("fmt", ["FP8", "INT8", "INT4", "INT2", "FP16", "mixed"])
def test_fused_equals_decomposed_and_unsharded(fmt, kind, out_dtype):
    need_indices = out_dtype == torch.float32
    qec = _qec(fmt, out_dtype, need_indices)
    m = _sharded(qec, PLANS[kind]())
    g = torch.Generator().manual_seed(7)
    for step, (B, long) in enumerate(((33, False), (7, False), (64, False), (1, False), (24, True))):  # batches that grow and shrink
        kjt = _kjt(g, B, torch.int64 if step % 2 else torch.int32, empty_key="fd" if step in (1, 4) else None, long=long)
        got = m(kjt.to(DEV))
        _assert_equal(got, _decomposed(m, kjt.to(DEV)))
        ref = qec(kjt)  # unsharded quantized module on the CPU reference path
        assert set(got) == set(ref)
        # shards of a table's columns are re-quantised with their own row scales; 2-bit rows re-quantised on a coarser grid differ by
        # up to a third of a step, so they are compared to the unsharded module only where a shard holds whole rows
        sliced = kind in ("cw", "twrw", "mixed", "ragged")
        if (fmt in ("INT2", "mixed")) and sliced:
            continue
        tol = 2e-2 if fmt == "INT4" and kind != "tw" else 2e-3
        for k in ref:
            torch.testing.assert_close(got[k].values().cpu().float(), ref[k].values().float(), rtol=tol, atol=tol * 5)
    assert int(m._plane().overflow.item()) == 0


@pytest.mark.parametrize("kind", ["rw", "mixed"])
def test_host_placed_and_cached_shards_next_to_hbm_shards(kind):
    qec = _qec("INT8", torch.float32, need_indices=True)
    kernels = {"rw": {"a": "quant_uvm", "b": "quant_uvm_caching", "c": "quant", "d": "quant_uvm_caching"},
               "mixed": {"a": "quant_uvm_caching", "b": "quant_uvm", "c": "quant", "d": "quant_uvm"}}[kind]
    plan_hbm = PLANS[kind]()
    plan = {}
    for t, ps in plan_hbm.items():
        shards = [(0, s.shard_offsets[0], s.shard_offsets[1], s.shard_sizes[0], s.shard_sizes[1]) for s in ps.sharding_spec.shards]
        plan[t] = _ps(ps.sharding_type, shards, kernels[t])
    base, placed = _sharded(qec, plan_hbm), _sharded(qec, plan)
    assert any(t._placed for t in placed._tbes) and any(t._placed and t._cached for t in placed._tbes)
    g = torch.Generator().manual_seed(3)
    for step in range(5):  # later calls hit the rows the earlier ones admitted
        kjt = _kjt(g, 48, torch.int64 if step % 2 else torch.int32, long=step == 4).to(DEV)
        got = placed(kjt)
        _assert_equal(got, _decomposed(placed, kjt))
        _assert_equal(got, base(kjt))
    stats = [s for t in placed._tbes if t._placed for s in t.cache_stats().values()]
    assert sum(s["lookups"] for s in stats) > 0 and sum(s["hits"] for s in stats) > 0
    assert int(placed._plane().overflow.item()) == 0


def test_no_host_sync_when_length_per_key_is_cached():
    m = _sharded(_qec("INT8", torch.float32, need_indices=True), PLANS["mixed"]())
    g = torch.Generator().manual_seed(5)
    kjts = [_kjt(g, 40, torch.int64).to(DEV) for _ in range(3)]
    for k in kjts:
        k.length_per_key()  # cached on the batch
    want = [_decomposed(m, k) for k in kjts]
    m(kjts[0])  # builds the plane and its buffers
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        got = [m(k) for k in kjts]  # new lengths per key: the feature bases are copied again
    finally:
        torch.cuda.set_sync_debug_mode(0)
    for a, b in zip(got, want):
        _assert_equal(a, b)


def test_cuda_graph_replay_equals_eager():
    m = _sharded(_qec("FP8", torch.bfloat16), PLANS["twrw"]())
    kjt = _kjt(torch.Generator().manual_seed(9), 64, torch.int32).to(DEV)
    kjt.length_per_key()
    want = _decomposed(m, kjt)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        m(kjt)  # warm-up: plane, buffers and feature bases of this batch
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = m(kjt)
    for k in out:
        out[k].values().fill_(7)
    graph.replay()
    _assert_equal(out, want)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
@pytest.mark.parametrize("fmt", ["INT8", "mixed"])
def test_two_gpus(fmt):
    qec = _qec(fmt, torch.float32, need_indices=True)
    plan = {"a": _rw("a", [100, 200], ks=[0, 1, 1]), "b": _cw("b", ks=(1, 0)), "c": _tw("c", k=1), "d": _ragged("d", 250, False, ks=(1, 0, 1))}
    m = _sharded(qec, plan)
    g = torch.Generator().manual_seed(11)
    for B, long in ((16, False), (64, False), (5, False), (24, True), (40, False)):
        kjt = _kjt(g, B, torch.int64, long=long)
        got = m(kjt.to(DEV))
        _assert_equal(got, _decomposed(m, kjt.to(DEV)))
    assert int(m._plane().overflow.item()) == 0


def test_calls_from_different_streams():
    """Calls issued on alternating streams with no ordering between them: the plane orders the reuse of its buffers itself."""
    m = _sharded(_qec("INT8", torch.float32, need_indices=True), PLANS["ragged"]())
    g = torch.Generator().manual_seed(13)
    kjts = [_kjt(g, B, torch.int64, long=B == 32).to(DEV) for B in (40, 40, 32, 8)]
    kjts.append(kjts[0])  # the same lengths per key again: the feature bases are kept
    want = [_decomposed(m, k) for k in kjts]
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    got = []
    for i, k in enumerate(kjts):
        if i % 2:
            with torch.cuda.stream(side):
                got.append(m(k))
        else:
            got.append(m(k))
    torch.cuda.synchronize()
    for a, b in zip(got, want):
        _assert_equal(a, b)
