"""FP8 wire of the NVLink sparse plane on ONE GPU (``LoopbackGroup``: W virtual ranks, every "peer" buffer local).

Two sets of virtual ranks get the same weights and batches: one without quantized-comms codecs, one with the FP8 row-wise codecs of
``QCommsConfig(forward_precision=FP8, backward_precision=FP8)``. The FP8 set must produce, bit for bit, what the portable path's codec
kernels (``get_qcomm_codec(FP8)``) make of the plain set's values: decode(encode(pooled rows)) on the directly written columns,
the plain values on the row-sharded (staged) columns, and the plain update from decode(encode(gradient)).
"""
import gc

import pytest
import torch

from torchrec_b200.modules.embedding_configs import EmbeddingBagConfig, PoolingType
from torchrec_b200.modules.embedding_modules import EmbeddingBagCollection
from torchrec_b200.ops.tbe import OptimType
from torchrec_b200.parallel import sharding_plan as sp
from torchrec_b200.parallel.embeddingbag import EmbeddingBagCollectionSharder
from torchrec_b200.parallel.engine import OptimizerSpec, ShardedLookupEngine
from torchrec_b200.parallel.qcomm_codec import CommType, QCommsConfig, get_qcomm_codec, get_qcomm_codecs, get_qcomm_codecs_registry
from torchrec_b200.parallel.sparse_plane import LoopbackGroup
from torchrec_b200.parallel.types import CommOp, ShardingEnv
from torchrec_b200.sparse.jagged_tensor import KeyedJaggedTensor

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
DIMS = [128, 64, 128, 32, 256]
ROWS = [500, 37, 1201, 64, 90]


def _fp8(R=32):
    return get_qcomm_codecs(QCommsConfig(forward_precision=CommType.FP8, backward_precision=CommType.FP8, fp8_quantize_dim=R))


def _tables(dims, rows, pooling):
    return [EmbeddingBagConfig(name=f"t{i}", embedding_dim=d, num_embeddings=r, feature_names=[f"f{i}"] if i != 1 else ["f1", "f1b"], pooling=pooling)
            for i, (d, r) in enumerate(zip(dims, rows))]


def _plan(kind, tables, W):
    gens = {}
    for i, t in enumerate(tables):
        k = kind if kind != "mixed" else ["tw", "rw", "cw", "tw", "rw"][i % 5]
        if k == "tw":
            gens[t.name] = sp.table_wise(rank=i % W)
        elif k == "rw":
            gens[t.name] = sp.row_wise()
        elif k == "cw":
            gens[t.name] = sp.column_wise(ranks=[(i + j) % W for j in range(2 if t.embedding_dim % 64 == 0 else 1)])
    return gens


def _kjt(tables, B, maxL, weighted, seed):
    g = torch.Generator().manual_seed(seed)
    keys, lens, vals = [], [], []
    for ti, t in enumerate(tables):
        for fn in t.feature_names:
            keys.append(fn)
            l = torch.ones(B, dtype=torch.int64) if ti == 0 else torch.randint(0, maxL + 1, (B,), generator=g)
            lens.append(l)
            vals.append(torch.randint(0, t.num_embeddings, (int(l.sum()),), generator=g))
    values = torch.cat(vals)
    w = torch.rand(values.numel(), generator=g) if weighted else None
    return KeyedJaggedTensor(keys=keys, values=values.to(DEV), lengths=torch.cat(lens).to(DEV), weights=w.to(DEV) if w is not None else None, stride=B)


class _Ranks:
    """W virtual ranks of one sharded module over one LoopbackGroup."""

    def __init__(self, W, kind, weighted, mean, out_dtype, codecs, optim=OptimType.EXACT_ROWWISE_ADAGRAD, dims=DIMS, rows=ROWS, B=64, seed=7):
        torch.manual_seed(seed)
        self.W, self.B = W, B
        self.tables = tables = _tables(dims, rows, PoolingType.MEAN if mean else PoolingType.SUM)
        ebc = EmbeddingBagCollection(tables=tables, is_weighted=weighted, device=torch.device("cpu"))
        plan = sp.construct_module_sharding_plan(ebc, _plan(kind, tables, W), sharder=EmbeddingBagCollectionSharder(), world_size=W, local_size=W, device_type="cuda")
        full = {t.name: torch.randn(t.num_embeddings, t.embedding_dim, device=DEV) * 0.1 for t in tables}
        self.feature_names = [f for t in tables for f in t.feature_names]
        feature_table = [ti for ti, t in enumerate(tables) for _ in t.feature_names]
        self.total_cols = sum(tables[ti].embedding_dim for ti in feature_table)
        self.group = LoopbackGroup(W, DEV)
        self.engines = []
        for r in range(W):
            eng = ShardedLookupEngine(tables, self.feature_names, feature_table, plan, ShardingEnv.from_loopback(W, r, self.group), DEV, pooled=True,
                                      is_weighted=weighted, opt_specs={t.name: OptimizerSpec(optim=optim, lr=0.1, eps=1e-3) for t in tables},
                                      output_dtype=out_dtype, qcomm_codecs=codecs)
            for shard, wview, _st, _tbe in eng.local_shard_views():
                wview.copy_(full[shard.name][shard.row_off : shard.row_off + shard.rows, shard.col_off : shard.col_off + shard.cols])
            self.engines.append(eng)
        self.weighted = weighted

    def input_dist(self, kjts):
        self.ids = [self.engines[r].plane_input_dist(kjts[r], None, self.total_cols, capacity=6 * self.B * 5) for r in range(self.W)]
        self.planes = [i.plane for i in self.ids]

    def forward(self, out_slot=0):
        for r in range(self.W):
            self.planes[r].forward_kernels(self.ids[r], out_slot)
        return [self.planes[r].forward_finish(out_slot) for r in range(self.W)]

    def backward(self, grads, split=False):
        for r in range(self.W):
            self.planes[r].backward_push(grads[r])
        if split:
            for r in range(self.W):
                self.planes[r].prepare_backward(self.ids[r].slot, fork=(r % 2 == 0))
        for r in range(self.W):
            self.planes[r].backward_apply(self.ids[r], 1.0 / self.W, want_psw=self.weighted)

    def state(self):
        out = []
        for eng in self.engines:
            for shard, w, st, _tbe in eng.local_shard_views():
                out.append((shard.name, shard.row_off, shard.col_off, w.clone(), {k: v.clone() for k, v in st.items()}))
        return out

    def direct_mask(self):
        """Output columns the forward carries as FP8: those of tables that are not row-sharded."""
        eng = self.engines[0]
        base = [0]
        for ti in [ti for ti, t in enumerate(self.tables) for _ in t.feature_names]:
            base.append(base[-1] + self.tables[ti].embedding_dim)
        m = torch.zeros(self.total_cols, dtype=torch.bool, device=DEV)
        for u in eng._units:
            if not eng._table_row_sharded[u.shard.table_idx]:
                c = base[u.feature] + u.shard.col_off
                m[c : c + u.shard.cols] = True
        return m


def _roundtrip(x, wire_dtype, R=32):
    """What the portable path's FP8 codec makes of ``x``: decode(encode(x)) per group of R consecutive columns, cast to the wire dtype."""
    codec = get_qcomm_codec(CommType.FP8, None, R)
    return codec.decode(codec.encode(x.float().contiguous())).view(x.shape).to(wire_dtype)


def _same_state(a, b):
    assert len(a) == len(b)
    for (n, ro, co, w1, s1), (_, _, _, w2, s2) in zip(a, b):
        assert torch.equal(w1, w2), f"weights of {n} rows {ro} cols {co} differ"
        for k in s1:
            assert torch.equal(s1[k], s2[k]), f"state {k} of {n} differs"


@pytest.fixture(autouse=True)
def _collect():
    yield
    gc.collect()


@pytest.mark.parametrize("W", [2, 4, 8])
@pytest.mark.parametrize("kind", ["tw", "cw", "mixed"])
@pytest.mark.parametrize("weighted,mean", [(False, False), (True, False), (False, True)])
@pytest.mark.parametrize("out_dtype", [torch.bfloat16, torch.float32])
def test_fp8_forward_and_backward_are_bit_exact(W, kind, weighted, mean, out_dtype):
    B = 64 if W != 4 else 48
    plain = _Ranks(W, kind, weighted, mean, out_dtype, None, B=B)
    q = _Ranks(W, kind, weighted, mean, out_dtype, _fp8(), B=B)
    kjts = [_kjt(plain.tables, B, 5, weighted, 100 + r) for r in range(W)]
    plain.input_dist(kjts)
    q.input_dist(kjts)
    assert all(p.wire_format == {"fwd": ("fp8", 32), "bwd": ("fp8", 32)} for p in q.planes)
    assert all(p.wire_format == {"fwd": None, "bwd": None} for p in plain.planes)
    direct = q.direct_mask()
    assert bool(direct.any())
    for slot in (1, 0):  # an eval slot first, then the training slot the backward follows
        ref = [o.clone() for o in plain.forward(slot)]
        got = [o.clone() for o in q.forward(slot)]
        for r in range(W):
            expect = torch.where(direct, _roundtrip(ref[r], out_dtype), ref[r])
            assert torch.equal(got[r], expect), f"rank {r} out slot {slot}"
    grads = [torch.randn(B, plain.total_cols, device=DEV) for _ in range(W)]
    q.backward(grads, split=(W == 4))
    plain.backward([_roundtrip(g, out_dtype) for g in grads], split=(W == 4))
    torch.cuda.synchronize()
    _same_state(q.state(), plain.state())
    if weighted:
        for pq, pp in zip(q.planes, plain.planes):
            assert torch.equal(pq.psw_grad_buf, pp.psw_grad_buf)


@pytest.mark.parametrize("grad_dtype", [torch.bfloat16, torch.float32])
def test_fp8_backward_adam_bf16_gradients(grad_dtype):
    W, B = 4, 64
    plain = _Ranks(W, "mixed", False, False, torch.bfloat16, None, optim=OptimType.ADAM)
    q = _Ranks(W, "mixed", False, False, torch.bfloat16, _fp8(), optim=OptimType.ADAM)
    kjts = [_kjt(plain.tables, B, 4, False, 7 + r) for r in range(W)]
    plain.input_dist(kjts)
    q.input_dist(kjts)
    plain.forward()
    q.forward()
    grads = [torch.randn(B, plain.total_cols, device=DEV).to(grad_dtype) for _ in range(W)]
    q.backward(grads, split=True)
    plain.backward([_roundtrip(g, torch.bfloat16) for g in grads], split=True)
    torch.cuda.synchronize()
    _same_state(q.state(), plain.state())


@pytest.mark.parametrize("case", ["misaligned", "int8", "bf16", "one_rank"])
def test_fallback_is_the_plain_plane(case):
    dims, W, codecs = DIMS, 2, _fp8()
    if case == "misaligned":
        dims = [48] + DIMS[1:]  # a 48-wide table at R = 32
    elif case == "int8":
        codecs = get_qcomm_codecs(QCommsConfig(forward_precision=CommType.INT8, backward_precision=CommType.INT8))
    elif case == "bf16":
        codecs = get_qcomm_codecs(QCommsConfig(forward_precision=CommType.BF16, backward_precision=CommType.BF16))
    else:
        W = 1
    B = 64
    plain = _Ranks(W, "mixed" if W > 1 else "tw", False, False, torch.bfloat16, None, dims=dims)
    q = _Ranks(W, "mixed" if W > 1 else "tw", False, False, torch.bfloat16, codecs, dims=dims)
    kjts = [_kjt(plain.tables, B, 4, False, 11 + r) for r in range(W)]
    plain.input_dist(kjts)
    q.input_dist(kjts)
    for pq, pp in zip(q.planes, plain.planes):
        assert pq.wire_format == {"fwd": None, "bwd": None}
        assert pq.buf.nbytes == pp.buf.nbytes
    for a, b in zip(q.forward(), plain.forward()):
        assert torch.equal(a, b)
    grads = [torch.randn(B, plain.total_cols, device=DEV) for _ in range(W)]
    if W == 1:  # one rank reads the gradient in place: no push, no inbox
        q.planes[0].backward(q.ids[0], grads[0], 1.0)
        plain.planes[0].backward(plain.ids[0], grads[0], 1.0)
    else:
        q.backward(grads)
        plain.backward(grads)
    torch.cuda.synchronize()
    _same_state(q.state(), plain.state())


def test_registry_codecs_select_fp8():
    """What ``EmbeddingBagCollectionSharder(qcomm_codecs_registry=...)`` hands the engine: the pooled all-to-all codecs."""
    reg = get_qcomm_codecs_registry(QCommsConfig(forward_precision=CommType.FP8, backward_precision=CommType.FP8))
    q = _Ranks(2, "tw", False, False, torch.bfloat16, reg[CommOp.POOLED_EMBEDDINGS_ALL_TO_ALL.name])
    q.input_dist([_kjt(q.tables, 64, 3, False, r) for r in range(2)])
    assert all(p.wire_format == {"fwd": ("fp8", 32), "bwd": ("fp8", 32)} for p in q.planes)


def _step(ranks, kjts, grads):
    ranks.input_dist(kjts)
    outs = ranks.forward()
    ranks.backward(grads)
    return outs


def test_fp8_step_replays_as_a_cuda_graph_without_host_sync():
    W, B = 2, 64
    eager = _Ranks(W, "mixed", False, False, torch.bfloat16, _fp8())
    graphed = _Ranks(W, "mixed", False, False, torch.bfloat16, _fp8())
    kjts1 = [_kjt(eager.tables, B, 3, False, 40 + r) for r in range(W)]
    # batch 2: the same bag lengths, new ids (every table has at least 37 rows); it is copied into batch 1's tensors before the replay
    kjts2 = [KeyedJaggedTensor(keys=k.keys(), values=(k.values() * 7 + 1) % 37, lengths=k.lengths().clone(), stride=B) for k in kjts1]
    grads = [torch.randn(B, eager.total_cols, device=DEV) for _ in range(W)]
    _step(eager, kjts1, grads)
    out_eager = [o.clone() for o in _step(eager, kjts2, grads)]

    static = [KeyedJaggedTensor(keys=k.keys(), values=k.values().clone(), lengths=k.lengths().clone(), stride=B) for k in kjts1]
    _step(graphed, static, grads)  # warm-up: the plane, its tables and every lazy allocation exist now
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        outs = _step(graphed, static, grads)
    for k, new in zip(static, kjts2):
        k.values().copy_(new.values())
    graph.replay()
    torch.cuda.synchronize()
    for a, b in zip(outs, out_eager):
        assert torch.equal(a, b)
    _same_state(graphed.state(), eager.state())
    # one more eager FP8 step under the sync checker: nothing on the step's path blocks the host
    torch.cuda.set_sync_debug_mode("error")
    try:
        _step(eager, kjts2, grads)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
