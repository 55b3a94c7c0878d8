"""Host side of the fused sequence path of ShardedQuantEmbeddingCollection: the unit table (route rows, edge rules, group slices) and the
feature bases of the flat output. Pure functions of the plan and the batch, no GPU needed."""
import pytest
import torch

from torchrec_b200.parallel.engine import TableShard
from torchrec_b200.parallel.quant_embedding import INT64_MAX, feature_bases, sequence_units


def _sh(ti, rank, row_off, rows, col_off, cols):
    return TableShard(ti, f"t{ti}", rank, row_off, col_off, rows, cols)


# table 0: 100 x 64, 4 row shards of 25 rows, two on each rank; table 1: 50 x 64 in two column halves on rank 0 / 1;
# table 2: 30 x 32 whole on rank 1; table 3: 40 x 64, grid: two column halves x row shards [0, 10) [10, 40)
ROWS = {0: 100, 1: 50, 2: 30, 3: 40}
DIM = {"a": 64, "b": 64, "b2": 64, "c": 32, "d": 64}
GROUPS = [
    (0, [("a", 0, _sh(0, 0, 0, 25, 0, 64)), ("a", 0, _sh(0, 0, 25, 25, 0, 64))]),
    (0, [("b", 1, _sh(1, 0, 0, 50, 0, 32)), ("b2", 1, _sh(1, 0, 0, 50, 0, 32)), ("d", 3, _sh(3, 0, 0, 10, 0, 32)),
         ("d", 3, _sh(3, 0, 10, 30, 32, 32))]),
    (1, [("b", 1, _sh(1, 1, 0, 50, 32, 32)), ("b2", 1, _sh(1, 1, 0, 50, 32, 32)), ("c", 2, _sh(2, 1, 0, 30, 0, 32)),
         ("d", 3, _sh(3, 1, 10, 30, 0, 32)), ("d", 3, _sh(3, 1, 0, 10, 32, 32))]),
    (1, [("a", 0, _sh(0, 1, 50, 25, 0, 64)), ("a", 0, _sh(0, 1, 75, 25, 0, 64))]),
]


def _takes(t, u, i):
    """Does unit u take id i (kjt_route.cu: a whole-row unit forwards every id, the others follow route_take with the edge rule)?"""
    lo, hi, e = t.row_lo[u], t.row_hi[u], t.edge[u]
    if (lo, hi) == (0, INT64_MAX):
        return True
    return lo <= i < hi or ((e & 1) and i < lo) or ((e & 2) and i >= hi)


def test_unit_order_slots_and_group_slices():
    t = sequence_units(GROUPS, ROWS, DIM)
    assert t.feature == [f for _, us in GROUPS for f, _, _ in us]
    assert t.rank == [0] * 6 + [1] * 7
    assert t.slot == list(range(6)) + list(range(7))
    assert t.dest_ustart == [0, 6, 13]
    assert t.group_slice == [(0, 2), (2, 6), (6, 11), (11, 13)]
    assert t.col == [0, 0, 0, 0, 0, 32, 32, 32, 0, 0, 32, 0, 0]
    assert t.dim == [64, 64, 64, 64, 64, 64, 64, 64, 32, 64, 64, 64, 64]


def test_row_ranges_and_edge_flags():
    t = sequence_units(GROUPS, ROWS, DIM)
    # table 0, four row shards: first keeps ids below, last keeps ids above, the inner ones only their rows
    a = [u for u, f in enumerate(t.feature) if f == "a"]
    assert [(t.row_lo[u], t.row_hi[u], t.edge[u]) for u in a] == [(0, 25, 1), (25, 50, 0), (50, 75, 0), (75, 100, 2)]
    # whole-row units (column shards, table-wise) take every id
    for u, f in enumerate(t.feature):
        if f in ("b", "b2", "c"):
            assert (t.row_lo[u], t.row_hi[u], t.edge[u]) == (0, INT64_MAX, 0)
    # grid: each column slice has its own first / last row shard
    d = [u for u, f in enumerate(t.feature) if f == "d"]
    assert sorted((t.col[u], t.row_lo[u], t.row_hi[u], t.edge[u]) for u in d) == [(0, 0, 10, 1), (0, 10, 40, 2), (32, 0, 10, 1), (32, 10, 40, 2)]


# the same shards, all on one device: row and column shards of one table share a (rank, width) group
ONE_DEVICE = [(0, GROUPS[0][1] + GROUPS[3][1]), (0, GROUPS[1][1] + GROUPS[2][1])]
# row shards cut into different column slices: table 0 rows [0, 40) in two column halves, rows [40, 100) whole width; table 3 rows
# [0, 10) whole width, rows [10, 40) in column halves on two ranks
RAGGED = [
    (0, [("a", 0, _sh(0, 0, 0, 40, 0, 32)), ("a", 0, _sh(0, 0, 0, 40, 32, 32)), ("d", 3, _sh(3, 0, 10, 30, 0, 32))]),
    (0, [("a", 0, _sh(0, 0, 40, 60, 0, 64)), ("d", 3, _sh(3, 0, 0, 10, 0, 64))]),
    (1, [("d", 3, _sh(3, 1, 10, 30, 32, 32))]),
]


def test_ragged_row_shards_route_each_id_to_its_own_rectangle():
    t = sequence_units(RAGGED, ROWS, DIM)
    assert [(t.row_lo[u], t.row_hi[u], t.edge[u]) for u in range(len(t.feature))] == [
        (0, 40, 1), (0, 40, 1), (10, 40, 2), (40, 100, 2), (0, 10, 1), (10, 40, 2)]


@pytest.mark.parametrize("groups", [GROUPS, ONE_DEVICE, RAGGED])
def test_every_feature_column_covered_once_per_id(groups):
    t = sequence_units(groups, ROWS, DIM)
    cols = [sh.cols for _, us in groups for _, _, sh in us]
    tables = {f: ti for _, us in groups for f, ti, _ in us}
    for f, ti in tables.items():
        for i in [-7, -1] + list(range(ROWS[ti])) + [ROWS[ti], ROWS[ti] + 1000]:
            hits = [0] * DIM[f]
            for u in range(len(t.feature)):
                if t.feature[u] == f and _takes(t, u, i):
                    for c in range(t.col[u], t.col[u] + cols[u]):
                        hits[c] += 1
            assert hits == [1] * DIM[f], (f, i)


def test_representatives_bound_the_routed_ids():
    t = sequence_units(ONE_DEVICE, ROWS, DIM)
    # the 4 row shards of "a" (one column slice) receive each id once: one representative; the two row shards of each column half of
    # "d" likewise; every column half of "b" / "b2" receives every id
    halves = [("b", 0), ("b", 32), ("b2", 0), ("b2", 32), ("c", 0), ("d", 0), ("d", 32)]
    assert [t.feature[u] for u in t.group_reps[0]] == ["a"]
    assert sorted((t.feature[u], t.col[u]) for u in t.group_reps[1]) == halves
    assert sorted((t.feature[u], t.col[u]) for u in t.dev_reps[0]) == [("a", 0)] + halves
    t = sequence_units(GROUPS, ROWS, DIM)
    assert sorted((t.feature[u], t.col[u]) for u in t.dev_reps[1]) == [("a", 0), ("b", 32), ("b2", 32), ("c", 0), ("d", 0), ("d", 32)]


@pytest.mark.parametrize("bad", ["gap", "overlap", "outside"])
def test_shards_that_do_not_tile_the_table_are_refused(bad):
    a = {"gap": [_sh(0, 0, 0, 25, 0, 64), _sh(0, 0, 50, 50, 0, 64)],
         "overlap": [_sh(0, 0, 0, 60, 0, 64), _sh(0, 0, 50, 50, 0, 64)],
         "outside": [_sh(0, 0, 0, 50, 0, 64), _sh(0, 0, 50, 60, 0, 64)]}[bad]
    with pytest.raises(ValueError, match="do not tile"):
        sequence_units([(0, [("a", 0, sh) for sh in a])], ROWS, DIM)


def test_feature_bases_follow_input_key_order():
    bases, total = feature_bases(["c", "x", "a", "b"], [3, 9, 0, 5], {"a": 64, "b": 32, "c": 16})
    assert bases == {"c": 0, "a": 48, "b": 48}
    assert total == 48 + 5 * 32


def test_unit_table_of_a_sharded_module_matches_its_groups():
    from torchrec_b200.inference.modules import quantize_inference_model
    from torchrec_b200.modules.embedding_configs import EmbeddingConfig
    from torchrec_b200.modules.embedding_modules import EmbeddingCollection
    from torchrec_b200.parallel.quant_embedding import ShardedQuantEmbeddingCollection
    from torchrec_b200.parallel.types import EnumerableShardingSpec, ParameterSharding, ShardingEnv, ShardMetadata
    from torchrec_b200.types import DataType

    tables = [EmbeddingConfig(name="t0", embedding_dim=64, num_embeddings=100, feature_names=["a"]),
              EmbeddingConfig(name="t1", embedding_dim=64, num_embeddings=50, feature_names=["b", "b2"])]

    class M(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.ec = EmbeddingCollection(tables=tables)

    qec = quantize_inference_model(M(), quantization_dtype=DataType.INT8).ec

    def ps(kind, shards):
        spec = EnumerableShardingSpec([ShardMetadata(shard_sizes=[r, c], shard_offsets=[ro, co], placement="rank:0/cuda:0") for ro, co, r, c in shards])
        return ParameterSharding(sharding_type=kind, compute_kernel="quant", ranks=[0] * len(shards), sharding_spec=spec)

    plan = {"t0": ps("row_wise", [(0, 0, 30, 64), (30, 0, 30, 64), (60, 0, 40, 64)]), "t1": ps("column_wise", [(0, 0, 50, 32), (0, 32, 50, 32)])}
    m = ShardedQuantEmbeddingCollection(qec, plan, ShardingEnv.from_local(1, 0), device=torch.device("cpu"))
    t = sequence_units(m._group_units, {0: 100, 1: 50}, m._feature_dim)
    assert [t.feature[u0:u1] for u0, u1 in t.group_slice] == [g[1] for g in m._groups]
    assert [t.col[u0:u1] for u0, u1 in t.group_slice] == [g[2] for g in m._groups]
    a = [u for u, f in enumerate(t.feature) if f == "a"]
    assert [(t.row_lo[u], t.row_hi[u], t.edge[u]) for u in a] == [(0, 30, 1), (30, 60, 0), (60, 100, 2)]
