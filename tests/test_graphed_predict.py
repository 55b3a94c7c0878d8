"""Host logic of the graphed predictor (``inference/graphed.py``): bucket choice, the ingest descriptor, the slab layout and the eager
path for batches no bucket holds. The device side is in test_graphed_predict_gpu.py."""
import numpy as np
import pytest
import torch

from torchrec_b200.inference.graphed import (DESC_FIELDS, GraphedPredictor, choose_bucket, normalize_buckets, pack_desc, pack_slab,
                                             slab_bytes_for)
from torchrec_b200.inference.server import InferenceServer, ServerConfig, _BatchDesc, batch_views

BUCKETS = [(16, 100), (64, 400), (64, 1000), (256, 2000)]


@pytest.mark.parametrize("B,n1,n2,want", [
    (1, 0, 0, 0), (16, 100, 100, 0), (16, 101, 0, 1), (17, 0, 0, 1), (16, 0, 101, 1), (64, 400, 400, 1), (64, 401, 0, 2),
    (64, 1000, 1000, 2), (65, 0, 0, 3), (1, 1001, 0, 3), (256, 2000, 2000, 3), (257, 0, 0, None), (1, 2001, 0, None), (1, 0, 2001, None),
])
def test_choose_bucket_edges(B, n1, n2, want):
    assert choose_bucket(BUCKETS, B, n1, n2) == want


def test_normalize_buckets_defaults_and_validation():
    assert normalize_buckets([64, (16, 10), 64, (16, 10)], 1 << 20) == [(16, 10), (64, (1 << 20) // 8)]
    with pytest.raises(ValueError):
        normalize_buckets([], 1 << 20)
    with pytest.raises(ValueError):
        normalize_buckets([(0, 10)], 1 << 20)
    with pytest.raises(ValueError):
        normalize_buckets([(4, -1)], 1 << 20)


def test_desc_fields_are_batch_desc_fields_and_pack_in_order():
    names = [f for f, _ in _BatchDesc._fields_]
    assert all(f in names for f in DESC_FIELDS)
    d = _BatchDesc()
    for i, f in enumerate(DESC_FIELDS):
        setattr(d, f, 1000 * i + 7 if f != "dense_off" else -1)
    got = pack_desc(d)
    assert got.dtype == np.int64 and got.tolist() == [1000 * i + 7 if f != "dense_off" else -1 for i, f in enumerate(DESC_FIELDS)]
    # the kernel's descriptor enum (csrc/serve_ingest.cu) lists the same fields in the same order
    import os
    import re

    src = open(os.path.join(os.path.dirname(__file__), "..", "torchrec_b200", "ops", "csrc", "serve_ingest.cu")).read()
    enum = re.search(r"enum : int \{(.*?)\};", src, re.S).group(1)
    ids = [t.strip().split("=")[0].strip() for t in enum.split(",") if t.strip()]
    assert ids == ["D_B", "D_NUM_FLOAT", "D_F_IDL", "D_F_IDS", "D_DENSE_OFF", "D_IDL_LEN_OFF", "D_IDL_VAL_OFF", "D_IDL_NNZ", "D_IDS_LEN_OFF",
                   "D_IDS_VAL_OFF", "D_IDS_WGT_OFF", "D_IDS_NNZ", "D_TOTAL_BYTES", "D_FIELDS"]
    assert len(ids) - 1 == len(DESC_FIELDS)


def _request(rng, B, F1, F2, nf=3, max_len=3):
    dense = rng.standard_normal((B, nf)).astype(np.float32) if nf else None
    l1 = rng.integers(0, max_len + 1, size=F1 * B).astype(np.int32)
    v1 = rng.integers(0, 50, size=int(l1.sum())).astype(np.int64)
    l2 = rng.integers(0, max_len + 1, size=F2 * B).astype(np.int32)
    v2 = rng.integers(0, 50, size=int(l2.sum())).astype(np.int64)
    w2 = rng.random(int(l2.sum())).astype(np.float32)
    return dense, (l1, v1), (l2, v2, w2)


def test_pack_slab_matches_views_and_layout():
    rng = np.random.default_rng(0)
    B, F1, F2 = 5, 2, 3
    dense, idl, ids = _request(rng, B, F1, F2)
    slab, d = pack_slab(B, dense, idl, ids, F1, F2)
    assert d.total_bytes == slab_bytes_for(B, 3, F1, F2, len(idl[1]), len(ids[1]))
    for f in ("dense_off", "idl_lengths_off", "idl_values_off", "ids_lengths_off", "ids_values_off", "ids_weights_off"):
        assert getattr(d, f) % 16 == 0
    x, kjt, wkjt = batch_views(slab, d, ["a", "b"], ["c", "d", "e"])
    assert np.array_equal(x.numpy(), dense)
    assert np.array_equal(kjt.lengths().numpy(), idl[0]) and np.array_equal(kjt.values().numpy(), idl[1])
    assert np.array_equal(wkjt.lengths().numpy(), ids[0]) and np.array_equal(wkjt.values().numpy(), ids[1])
    assert np.array_equal(wkjt.weights().numpy(), ids[2])
    # absent sections: offset -1, no bytes
    slab, d = pack_slab(B, None, idl)
    assert d.dense_off == -1 and d.ids_values_off == -1 and d.num_float == 0 and d.id_score_features == 0


def _keys(n, p):
    return [f"{p}{i}" for i in range(n)]


def _cpu_predict():
    torch.manual_seed(0)
    lin = torch.nn.Linear(3 + 2, 1)

    def predict(dense, kjt, wkjt):
        s1 = torch.zeros(dense.shape[0]).index_add_(0, torch.repeat_interleave(torch.arange(kjt.stride()).repeat(2), kjt.lengths().long()),
                                                    kjt.values().float())
        s2 = torch.zeros(dense.shape[0]).index_add_(0, torch.repeat_interleave(torch.arange(wkjt.stride()).repeat(3), wkjt.lengths().long()),
                                                    wkjt.weights())
        return lin(torch.cat([dense, s1[:, None], s2[:, None]], 1)).squeeze(1)

    return predict


def test_eager_path_for_batches_no_bucket_holds():
    predict = _cpu_predict()
    gp = GraphedPredictor(predict, [(4, 20), (8, 40)], num_float=3, id_list_keys=_keys(2, "a"), id_score_list_keys=_keys(3, "c"),
                          device=torch.device("cpu"), buffer_bytes=1 << 16, max_batch_size=64)
    rng = np.random.default_rng(1)
    for B, max_len, eager in ((9, 1, True), (2, 30, True), (64, 3, True), (4, 1, False)):
        dense, idl, ids = _request(rng, B, 2, 3, max_len=max_len)
        slab, d = pack_slab(B, dense, idl, ids, 2, 3)
        assert (gp.bucket_for(d) is None) == eager
        if eager:
            got = gp.run(slab, d)
            assert torch.equal(got, predict(*batch_views(slab, d, _keys(2, "a"), _keys(3, "c"))))
        else:
            with pytest.raises(RuntimeError, match="before capture"):
                gp.run(slab, d)
    # other feature counts than the graphs were built for go eager too
    dense, idl, _ = _request(rng, 2, 2, 0)
    _, d = pack_slab(2, dense, idl, None, 2, 0)
    assert gp.bucket_for(d) is None
    # beyond the server's largest batch: refused
    dense, idl, ids = _request(rng, 65, 2, 3, max_len=0)
    slab, d = pack_slab(65, dense, idl, ids, 2, 3)
    with pytest.raises(ValueError):
        gp.run(slab, d)
    with pytest.raises(RuntimeError):
        gp.capture()


def test_bucket_larger_than_slab_and_uncaptured_server_refused():
    with pytest.raises(ValueError):
        GraphedPredictor(_cpu_predict(), [4096], num_float=13, id_list_keys=_keys(26, "f"), device=torch.device("cpu"), buffer_bytes=1 << 16)
    gp = GraphedPredictor(_cpu_predict(), [4], num_float=3, id_list_keys=_keys(2, "a"), id_score_list_keys=_keys(3, "c"), device=torch.device("cpu"))
    with pytest.raises(ValueError):
        InferenceServer([gp], [torch.device("cpu")], id_list_keys=_keys(2, "a"), id_score_list_keys=_keys(3, "c"), config=ServerConfig())


def test_modules_of_callables():
    from torchrec_b200.inference.graphed import modules_of

    lin = torch.nn.Linear(2, 1)

    def closure(dense, kjt, wkjt):
        return lin(dense)

    assert modules_of(lin) == [lin]
    assert modules_of(lin.forward) == [lin]
    assert modules_of(closure) == [lin]
    assert modules_of(len) == []


def _quant_model(ec: bool):
    from torchrec_b200.inference.modules import quantize_inference_model
    from torchrec_b200.modules.embedding_configs import EmbeddingBagConfig, EmbeddingConfig
    from torchrec_b200.modules.embedding_modules import EmbeddingBagCollection, EmbeddingCollection

    class M(torch.nn.Module):
        def __init__(self):
            super().__init__()
            if ec:
                self.ec = EmbeddingCollection(tables=[EmbeddingConfig(name="s", embedding_dim=8, num_embeddings=50, feature_names=["s"])])
            self.ebc = EmbeddingBagCollection([EmbeddingBagConfig(name=f"t{i}", embedding_dim=8, num_embeddings=100 + i, feature_names=[f"f{i}"])
                                               for i in range(4)])

        def forward(self, dense, kjt, wkjt):
            return self.ebc(kjt).values().sum(1)

    torch.manual_seed(0)
    return quantize_inference_model(M())


def test_out_of_scope_modules_are_refused():
    from torchrec_b200.inference.modules import shard_quant_model

    keys = [f"f{i}" for i in range(4)]
    with pytest.raises(ValueError, match="sequence"):
        GraphedPredictor(_quant_model(ec=True), [4], num_float=0, id_list_keys=keys, device=torch.device("cpu"))
    GraphedPredictor(_quant_model(ec=False), [4], num_float=0, id_list_keys=keys, device=torch.device("cpu"))
    sharded, _ = shard_quant_model(_quant_model(ec=False), world_size=2, compute_device="cpu", sharding_device="cpu")
    ebc = sharded.ebc
    assert sum(1 for units in ebc._rank_meta if units) == 2  # the planner spread the tables over both ranks
    with pytest.raises(ValueError, match="spans devices"):
        GraphedPredictor(sharded, [4], num_float=0, id_list_keys=keys, device=torch.device("cpu"))
