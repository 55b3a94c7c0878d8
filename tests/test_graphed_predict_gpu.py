"""Graphed serving on one H100: the ingest kernel (``csrc/serve_ingest.cu``) against a PyTorch construction of the same tensors, and
``GraphedPredictor`` replays against the eager predictor (bit-equal on the batch padded to the bucket, close on the batch itself) for
quantized DLRMs with a bf16 or FP8 dense arch, a weighted collection, host-resident cached tables, and behind ``InferenceServer``."""
import threading

import numpy as np
import pytest
import torch

from torchrec_b200.inference.graphed import GraphedPredictor, pack_slab
from torchrec_b200.inference.server import batch_views
from torchrec_b200.sparse import KeyedJaggedTensor

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
SENT_I, SENT_F = -777, -3.5


def _request(rng, B, F1, F2, nf, max_len, rows=1000):
    dense = rng.standard_normal((B, nf)).astype(np.float32) if nf else None
    idl = ids = None
    if F1:
        l1 = rng.integers(0, max_len + 1, size=F1 * B).astype(np.int32)
        idl = (l1, rng.integers(0, rows, size=int(l1.sum())).astype(np.int64))
    if F2:
        l2 = rng.integers(0, max_len + 1, size=F2 * B).astype(np.int32)
        ids = (l2, rng.integers(0, rows, size=int(l2.sum())).astype(np.int64), rng.random(int(l2.sum())).astype(np.float32))
    return dense, idl, ids


def _pad_lengths(l, F, B, B_cap):
    out = np.zeros(F * B_cap, dtype=np.int64)
    for f in range(F):
        out[f * B_cap : f * B_cap + B] = l[f * B : (f + 1) * B]
    return out


# ---- the ingest kernel -------------------------------------------------------------------------------------------------------
def _ingest_case(B, B_cap, nnz_cap, F1, F2, nf, max_len, seed, shift=0, over=None):
    from torchrec_b200.ops import serve
    from torchrec_b200.inference.graphed import pack_desc

    rng = np.random.default_rng(seed)
    dense, idl, ids = _request(rng, B, F1, F2, nf, max_len)
    slab, d = pack_slab(B, dense, idl, ids, F1, F2)
    fields = pack_desc(d)
    if over == "B":
        fields[0] = B_cap + 1
    slab_dev = torch.zeros(slab.numel() + 64, dtype=torch.uint8, device=DEV)
    slab_dev[shift : shift + slab.numel()].copy_(slab)
    desc = torch.from_numpy(fields).to(DEV)
    buf = serve.IngestBuffers.allocate(B_cap, nnz_cap, nf, F1, F2, torch.int32 if seed % 2 else torch.int64, DEV)
    for t in (buf.dense, buf.idl_values, buf.idl_lengths, buf.idl_offsets, buf.ids_values, buf.ids_lengths, buf.ids_offsets, buf.ids_weights):
        if t is not None:
            t.fill_(SENT_F if t.is_floating_point() else SENT_I)
    err = torch.zeros(1, dtype=torch.int32, device=DEV)
    serve.ingest(slab_dev[shift:], desc, buf, nf, F1, F2, err)
    torch.cuda.synchronize()
    return dense, idl, ids, buf, int(err[0])


@pytest.mark.parametrize("case", [
    dict(B=37, B_cap=64, nnz_cap=2000, F1=5, F2=3, nf=13, max_len=4, seed=1),    # random B below capacity
    dict(B=64, B_cap=64, nnz_cap=None, F1=4, F2=2, nf=7, max_len=3, seed=2),     # B and nnz exactly at capacity
    dict(B=10, B_cap=16, nnz_cap=50, F1=3, F2=2, nf=13, max_len=0, seed=3),      # a batch without ids
    dict(B=29, B_cap=32, nnz_cap=800, F1=6, F2=0, nf=13, max_len=5, seed=4),     # only id_list
    dict(B=5, B_cap=8, nnz_cap=300, F1=0, F2=4, nf=13, max_len=7, seed=5),       # only id_score_list
    dict(B=33, B_cap=40, nnz_cap=999, F1=3, F2=3, nf=0, max_len=3, seed=6),      # no dense features
    dict(B=1, B_cap=2048, nnz_cap=5000, F1=26, F2=1, nf=13, max_len=2, seed=7),  # one sample in the largest bucket
    dict(B=700, B_cap=2048, nnz_cap=40001, F1=26, F2=0, nf=13, max_len=2, seed=8),  # several scan tiles
    dict(B=20, B_cap=24, nnz_cap=600, F1=3, F2=2, nf=5, max_len=4, seed=9, shift=8),  # sections not 16-byte aligned: element-wise copies
])
def test_ingest_matches_torch(case):
    case = dict(case)
    B, B_cap, F1, F2, nf = case["B"], case["B_cap"], case["F1"], case["F2"], case["nf"]
    if case["nnz_cap"] is None:  # exactly at capacity: the bigger list fills the bucket
        rng = np.random.default_rng(case["seed"])
        _, idl, ids = _request(rng, B, F1, F2, nf, case["max_len"])
        case["nnz_cap"] = max(len(idl[1]), len(ids[1]))
    dense, idl, ids, buf, err = _ingest_case(**case)
    assert err == 0
    if nf:
        want = np.zeros((B_cap, nf), dtype=np.float32)
        want[:B] = dense
        assert np.array_equal(buf.dense.cpu().numpy(), want)  # padded rows are zero
    for lst, F, lens, offs, vals, wts in ((idl, F1, buf.idl_lengths, buf.idl_offsets, buf.idl_values, None),
                                          (ids, F2, buf.ids_lengths, buf.ids_offsets, buf.ids_values, buf.ids_weights)):
        if not F:
            assert lens is None
            continue
        pl = _pad_lengths(lst[0], F, B, B_cap)
        assert np.array_equal(lens.cpu().numpy(), pl)  # padded bags are empty: every feature keeps stride B_cap
        assert np.array_equal(offs.cpu().long().numpy(), np.concatenate([[0], np.cumsum(pl)]))
        n = len(lst[1])
        v = vals.cpu().numpy()
        assert np.array_equal(v[:n], lst[1]) and (v[n:] == SENT_I).all()  # nothing past nnz written
        if wts is not None:
            w = wts.cpu().numpy()
            assert np.array_equal(w[:n], lst[2]) and (w[n:] == SENT_F).all()


@pytest.mark.parametrize("over", ["B", "nnz"])
def test_ingest_over_capacity_raises_flag_and_writes_nothing(over):
    kw = dict(B=30, B_cap=32, nnz_cap=10, F1=3, F2=2, nf=13, max_len=3, seed=11, over=over)
    if over == "B":
        kw["nnz_cap"] = 1000
    dense, idl, ids, buf, err = _ingest_case(**kw)
    assert err == 1
    for t in (buf.dense, buf.idl_values, buf.idl_lengths, buf.idl_offsets, buf.ids_values, buf.ids_lengths, buf.ids_offsets, buf.ids_weights):
        x = t.cpu()
        assert (x == (SENT_F if x.is_floating_point() else SENT_I)).all()


# ---- models ------------------------------------------------------------------------------------------------------------------
ROWS = [3000, 5000, 700, 1500]


def _shard(qebc, kernels, load_factor=0.02):
    from torchrec_b200.parallel import sharding_plan as sp
    from torchrec_b200.parallel.quant_embeddingbag import QuantEmbeddingBagCollectionSharder, ShardedQuantEmbeddingBagCollection
    from torchrec_b200.parallel.types import CacheParams, ShardingEnv

    names = [c.name for c in qebc.embedding_bag_configs()]
    gens = {n: sp.table_wise(rank=0, compute_kernel=kernels.get(n, "quant")) for n in names}
    plan = sp.construct_module_sharding_plan(qebc, gens, sharder=QuantEmbeddingBagCollectionSharder(), world_size=1, local_size=1, device_type="cuda")
    for n in names:
        if kernels.get(n) == "quant_uvm_caching":
            plan[n].cache_params = CacheParams(load_factor=load_factor)
    return ShardedQuantEmbeddingBagCollection(qebc, plan, ShardingEnv.from_local(1, 0), device=DEV)


def _dlrm(dense_kind, kernels=None):
    """Quantized DLRM: INT8, FP8 and INT4 tables and a MEAN-pooled INT8 table, one GPU; bf16 (wgmma) or FP8 dense arch."""
    from torchrec_b200.inference.modules import quantize_dense, quantize_inference_model
    from torchrec_b200.models.dlrm import DLRM
    from torchrec_b200.modules.embedding_configs import EmbeddingBagConfig, PoolingType
    from torchrec_b200.modules.embedding_modules import EmbeddingBagCollection
    from torchrec_b200.types import DataType

    torch.manual_seed(0)
    keys = [f"f{i}" for i in range(4)]
    tables = [EmbeddingBagConfig(name=f"t{i}", embedding_dim=64, num_embeddings=ROWS[i], feature_names=[keys[i]],
                                 pooling=PoolingType.MEAN if i == 3 else PoolingType.SUM) for i in range(4)]
    model = DLRM(EmbeddingBagCollection(tables), 13, [128, 64], [256, 128, 1], dense_device=DEV).eval()
    q = quantize_inference_model(model, per_table_weight_dtype={"t0": DataType.INT8, "t1": DataType.FP8, "t2": DataType.INT4, "t3": DataType.INT8},
                                 output_dtype=torch.float32)
    q.sparse_arch.embedding_bag_collection = _shard(q.sparse_arch.embedding_bag_collection, kernels or {})
    if dense_kind == "fp8":
        q = quantize_dense(q, torch.float8_e4m3fn)

    def predict(dense, kjt, _wkjt):
        return q(dense, kjt).sigmoid().reshape(-1)

    predict.model = q
    return keys, predict


class _Weighted(torch.nn.Module):
    """id_list collection + weighted (id_score_list) collection + a linear head."""

    def __init__(self):
        from torchrec_b200.inference.modules import quantize_inference_model
        from torchrec_b200.modules.embedding_configs import EmbeddingBagConfig
        from torchrec_b200.modules.embedding_modules import EmbeddingBagCollection

        super().__init__()
        torch.manual_seed(1)
        self.ebc = EmbeddingBagCollection([EmbeddingBagConfig(name=f"a{i}", embedding_dim=32, num_embeddings=ROWS[i], feature_names=[f"a{i}"]) for i in range(2)])
        self.webc = EmbeddingBagCollection([EmbeddingBagConfig(name=f"w{i}", embedding_dim=32, num_embeddings=ROWS[i + 2], feature_names=[f"w{i}"])
                                            for i in range(2)], is_weighted=True)
        quantize_inference_model(self, output_dtype=torch.float32)
        self.ebc, self.webc = _shard(self.ebc, {}), _shard(self.webc, {})
        self.head = torch.nn.Linear(13 + 4 * 32, 2, device=DEV)

    def forward(self, dense, kjt, wkjt):
        return torch.sigmoid(self.head(torch.cat([dense, self.ebc(kjt).values(), self.webc(wkjt).values()], 1)))


@pytest.fixture
def wgmma():
    from torchrec_b200.ops import dense as _dense

    prev = _dense.get_dense_backend()
    _dense.set_dense_backend("wgmma")
    yield
    _dense.set_dense_backend(prev)


def _padded(gp, dense, idl, ids, B, B_cap):
    """The batch padded to B_cap exactly as the ingest kernel pads it, as eager inputs."""
    x = torch.zeros(B_cap, gp.num_float, device=DEV)
    x[:B] = torch.from_numpy(dense)
    kjt = wkjt = None
    if idl is not None:
        kjt = KeyedJaggedTensor(keys=gp.id_list_keys, values=torch.from_numpy(idl[1]).to(DEV),
                                lengths=torch.from_numpy(_pad_lengths(idl[0], gp.F_idl, B, B_cap)).int().to(DEV), stride=B_cap)
    if ids is not None:
        wkjt = KeyedJaggedTensor(keys=gp.id_score_list_keys, values=torch.from_numpy(ids[1]).to(DEV),
                                 lengths=torch.from_numpy(_pad_lengths(ids[0], gp.F_ids, B, B_cap)).int().to(DEV),
                                 weights=torch.from_numpy(ids[2]).to(DEV), stride=B_cap)
    return x, kjt, wkjt


def _check(gp, predict, rng, B, max_len, tol, rows=min(ROWS)):
    dense, idl, ids = _request(rng, B, gp.F_idl, gp.F_ids, gp.num_float, max_len, rows)
    slab, d = pack_slab(B, dense, idl, ids, gp.F_idl, gp.F_ids)
    i = gp.bucket_for(d)
    with torch.inference_mode():
        got = gp.run(slab.to(DEV), d).clone()
        if i is not None:
            B_cap = gp.buckets[i][0]
            pad = predict(*_padded(gp, dense, idl, ids, B, B_cap))[:B]
            assert torch.equal(got, pad), (B, B_cap)  # the graph computes exactly what eager computes on the padded batch
        want = predict(*batch_views(slab.to(DEV), d, gp.id_list_keys, gp.id_score_list_keys))
    assert got.shape == want.shape
    assert float((got - want).abs().max()) < tol  # GEMM tiling may change with M
    return i


TOL = {"bf16": 5e-3, "fp8": 0.02}


@pytest.mark.parametrize("dense_kind", ["bf16", "fp8"])
def test_graph_equals_eager_padded_and_close_unpadded(wgmma, dense_kind):
    keys, predict = _dlrm(dense_kind)
    gp = GraphedPredictor(predict, [(16, 400), (128, 3000)], num_float=13, id_list_keys=keys, device=DEV, buffer_bytes=1 << 20, max_batch_size=256)
    gp.capture()
    rng = np.random.default_rng(0)
    used = [_check(gp, predict, rng, B, 4, TOL[dense_kind]) for B in (1, 7, 16, 17, 100, 128, 200)]
    assert used == [0, 0, 0, 1, 1, 1, None]


def test_weighted_collection_graph(wgmma):
    m = _Weighted()
    gp = GraphedPredictor(m, [(32, 500)], num_float=13, id_list_keys=["a0", "a1"], id_score_list_keys=["w0", "w1"], buffer_bytes=1 << 20,
                          max_batch_size=64)
    assert gp.device == DEV
    gp.capture()
    rng = np.random.default_rng(1)
    for B in (1, 9, 32, 50):
        _check(gp, m, rng, B, 5, 1e-5)


def test_one_bucket_many_batches(wgmma):
    keys, predict = _dlrm("bf16")
    gp = GraphedPredictor(predict, [(64, 2000)], num_float=13, id_list_keys=keys, device=DEV, buffer_bytes=1 << 20, max_batch_size=64)
    gp.capture()
    rng = np.random.default_rng(2)
    # large then small batches: stale rows or ids left by a bigger batch would show up in the next one
    for step in range(20):
        B = int(rng.integers(1, 65)) if step % 3 else 64
        assert _check(gp, predict, rng, B, int(rng.integers(0, 6)), TOL["bf16"]) == 0


def test_cached_host_tables_across_admissions(wgmma):
    keys, predict = _dlrm("bf16", kernels={"t0": "quant_uvm_caching", "t1": "quant_uvm", "t3": "quant_uvm_caching"})
    gp = GraphedPredictor(predict, [(128, 3000)], num_float=13, id_list_keys=keys, device=DEV, buffer_bytes=1 << 20, max_batch_size=128)
    gp.capture()
    rng = np.random.default_rng(3)
    for _ in range(8):  # every call misses rows and admits some: results must not depend on what the cache holds
        _check(gp, predict, rng, int(rng.integers(32, 129)), 4, TOL["bf16"], rows=1500)


def test_run_does_not_sync_the_host(wgmma):
    keys, predict = _dlrm("fp8")
    gp = GraphedPredictor(predict, [(64, 1000)], num_float=13, id_list_keys=keys, device=DEV, buffer_bytes=1 << 20, max_batch_size=64)
    gp.capture()
    rng = np.random.default_rng(4)
    batches = []
    for B in (3, 64, 20):
        dense, idl, _ = _request(rng, B, 4, 0, 13, 3)
        slab, d = pack_slab(B, dense, idl, None, 4, 0)
        batches.append((slab.pin_memory(), d))
    outs = []
    with torch.inference_mode():
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            for slab, d in batches:
                gp.slab[: d.total_bytes].copy_(slab[: d.total_bytes], non_blocking=True)
                outs.append(gp.run(gp.slab, d).clone())
        finally:
            torch.cuda.set_sync_debug_mode(0)
        torch.cuda.synchronize()
        for (slab, d), o in zip(batches, outs):
            want = predict(*batch_views(slab.to(DEV), d, keys, ()))
            assert float((o - want).abs().max()) < TOL["fp8"]
    assert not gp.ingest_failed()


def test_inference_server_with_graphed_predictor(wgmma):
    from torchrec_b200.inference.server import InferenceServer, ServerConfig

    keys, predict = _dlrm("bf16")
    cfg = ServerConfig(max_batch_size=256, batching_interval_ms=2.0, buffer_bytes=1 << 20)
    gp = GraphedPredictor(predict, [16, 64], num_float=13, id_list_keys=keys, device=DEV, buffer_bytes=cfg.buffer_bytes, max_batch_size=cfg.max_batch_size)
    gp.capture()
    srv = InferenceServer([gp], [DEV], id_list_keys=keys, config=cfg)
    rng = np.random.default_rng(5)
    reqs = [(B,) + _request(rng, B, 4, 0, 13, 3)[:2] for B in [int(x) for x in rng.integers(1, 40, size=40)] + [120, 200, 3]]
    results = [None] * len(reqs)

    def client(i):
        B, dense, idl = reqs[i]
        results[i] = srv.predict(B, dense, idl, timeout_s=60.0)

    try:
        threads = [threading.Thread(target=client, args=(i,)) for i in range(len(reqs))]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
        assert srv.stats()["batches"] >= 1
    finally:
        srv.shutdown()
    with torch.inference_mode():
        for (B, dense, idl), got in zip(reqs, results):
            kjt = KeyedJaggedTensor(keys=keys, values=torch.from_numpy(idl[1]).to(DEV), lengths=torch.from_numpy(idl[0]).to(DEV), stride=B)
            want = predict(torch.from_numpy(dense).to(DEV), kjt, None).float().reshape(B, -1).cpu().numpy()
            assert got.shape == want.shape
            assert np.abs(got - want).max() < TOL["bf16"]


def _cache_is_consistent(tbe):
    """Every cached row owns its slot: two rows mapped to one slot means an admission raced another one."""
    for c in range(len(tbe._cached)):
        sor, ros = tbe._qc(c, "slot_of_row").long().cpu(), tbe._qc(c, "row_of_slot").long().cpu()
        rows = torch.nonzero(sor >= 0).flatten()
        if not torch.equal(ros[sor[rows]], rows):
            return False
    return True


def test_replay_right_after_eager_admission(wgmma):
    from torchrec_b200.ops.quant_tbe import QuantTableBatchedEmbeddingBags

    keys, predict = _dlrm("bf16", kernels={"t0": "quant_uvm_caching", "t1": "quant_uvm_caching"})
    gp = GraphedPredictor(predict, [(32, 1000)], num_float=13, id_list_keys=keys, device=DEV, buffer_bytes=1 << 20, max_batch_size=512)
    gp.capture()
    tbes = [m for m in predict.model.modules() if isinstance(m, QuantTableBatchedEmbeddingBags) and m._placed and m._cached]
    assert tbes and {id(t) for t in tbes} == {id(t) for t in gp._cached_tbes}
    rng = np.random.default_rng(6)
    calls = []
    with torch.inference_mode():
        for step in range(6):
            # an over-bucket batch runs eagerly and leaves its admission pending on a side stream; the replay follows at once
            for B, max_len in ((int(rng.integers(300, 513)), 6), (int(rng.integers(1, 33)), 4)):
                dense, idl, _ = _request(rng, B, 4, 0, 13, max_len, rows=min(ROWS))
                slab, d = pack_slab(B, dense, idl, None, 4, 0)
                slab_dev = slab.to(DEV)
                calls.append((gp.bucket_for(d), B, dense, idl, slab_dev, d, gp.run(slab_dev, d).clone()))
        torch.cuda.synchronize()
        assert all(_cache_is_consistent(t) for t in tbes)
        assert [c[0] for c in calls] == [None, 0] * 6
        for i, B, dense, idl, slab_dev, d, got in calls:
            if i is None:
                want = predict(*batch_views(slab_dev, d, keys, ()))
                assert float((got - want).abs().max()) < TOL["bf16"]
            else:
                assert torch.equal(got, predict(*_padded(gp, dense, idl, None, B, 32))[:B])
    assert all(_cache_is_consistent(t) for t in tbes)


def test_dlrm_predict_module_constructor(wgmma):
    from torchrec_b200.inference.dlrm_predict import DLRMPredictModule

    keys, predict = _dlrm("fp8")
    pm = DLRMPredictModule(predict.model, keys, device="cuda:0")
    gp = GraphedPredictor(pm, [64], num_float=13, buffer_bytes=1 << 20, max_batch_size=64)
    assert gp.device == DEV and gp.id_list_keys == keys
    gp.capture()
    rng = np.random.default_rng(7)
    for B in (5, 64):
        dense, idl, _ = _request(rng, B, 4, 0, 13, 3)
        slab, d = pack_slab(B, dense, idl, None, 4, 0)
        with torch.inference_mode():
            got = gp.run(slab.to(DEV), d).cpu()
        want = pm({"float_features": torch.from_numpy(dense).to(DEV), "id_list_features.lengths": torch.from_numpy(idl[0]).to(DEV),
                   "id_list_features.values": torch.from_numpy(idl[1]).to(DEV)})["default"]
        torch.cuda.synchronize()
        assert float((got - want).abs().max()) < TOL["fp8"]


def test_rejected_batch_reaches_flag_and_server(wgmma):
    from torchrec_b200.inference.server import InferenceServer, ServerConfig

    keys, predict = _dlrm("fp8")
    cfg = ServerConfig(max_batch_size=64, buffer_bytes=1 << 20)
    gp = GraphedPredictor(predict, [64], num_float=13, id_list_keys=keys, device=DEV, buffer_bytes=cfg.buffer_bytes, max_batch_size=64)
    gp.capture()
    rng = np.random.default_rng(8)
    dense, idl, _ = _request(rng, 16, 4, 0, 13, 3)
    slab, d = pack_slab(16, dense, idl, None, 4, 0)
    assert not gp.ingest_failed()
    bad = slab.clone()
    bad[d.idl_lengths_off : d.idl_lengths_off + 4].view(torch.int32)[0] += 5  # lengths no longer sum to the id count
    with torch.inference_mode():
        gp.run(bad.to(DEV), d)
        torch.cuda.synchronize()
        assert gp.ingest_failed()  # the kernel wrote the flag into mapped host memory
        assert not gp.ingest_failed()  # reading clears it
        gp.run(slab.to(DEV), d)
        torch.cuda.synchronize()
        assert not gp.ingest_failed()
    # a server with larger batches or other keys than the predictor was built for is refused
    with pytest.raises(ValueError):
        InferenceServer([gp], [DEV], id_list_keys=keys, config=ServerConfig(max_batch_size=128, buffer_bytes=1 << 20))
    with pytest.raises(ValueError):
        InferenceServer([gp], [DEV], id_list_keys=keys[::-1], config=cfg)
    srv = InferenceServer([gp], [DEV], id_list_keys=keys, config=cfg)
    try:
        stream = torch.cuda.Stream(DEV)
        with torch.inference_mode(), torch.cuda.stream(stream):
            with pytest.raises(RuntimeError, match="rejected"):
                srv._run_graphed(0, bad.pin_memory(), d, stream)
            ok = srv._run_graphed(0, slab.pin_memory(), d, stream)
        kjt = KeyedJaggedTensor(keys=keys, values=torch.from_numpy(idl[1]).to(DEV), lengths=torch.from_numpy(idl[0]).to(DEV), stride=16)
        with torch.inference_mode():
            want = predict(torch.from_numpy(dense).to(DEV), kjt, None).reshape(16, 1).cpu()
        assert float((ok - want).abs().max()) < TOL["fp8"]
    finally:
        srv.shutdown()
