"""Placed quantized tables without a GPU: the CPU reference path serves every location, and the planner's HBM / DDR estimate of a
``quant_uvm_caching`` shard is what the module allocates for its cache (rows + 4-byte slot map) and its host table."""
import math

import pytest
import torch

from torchrec_b200.ops.quant_tbe import QuantTableBatchedEmbeddingBags
from torchrec_b200.ops.tbe import EmbeddingLocation as EL
from torchrec_b200.types import DataType

SPECS = [("a", 300, 64, DataType.INT8), ("b", 200, 32, DataType.INT2), ("c", 150, 64, DataType.FP8), ("d", 90, 32, DataType.FP16)]


@pytest.mark.parametrize("pooling_mode", [0, 1])
@pytest.mark.parametrize("weighted", [False, True])
def test_cpu_reference_path_serves_every_location(pooling_mode, weighted):
    g = torch.Generator().manual_seed(0)
    weights = [torch.randn(r, d, generator=g) for _, r, d, _ in SPECS]
    B, F = 16, len(SPECS)
    lengths = torch.randint(0, 4, (F * B,), generator=g)
    offsets = torch.cat([torch.zeros(1, dtype=torch.int64), lengths.cumsum(0)])
    ids = torch.cat([torch.randint(-2, r + 2, (int(lengths[f * B : (f + 1) * B].sum()),), generator=g) for f, (_, r, _, _) in enumerate(SPECS)])
    psw = torch.rand(ids.numel(), generator=g) if weighted else None
    outs = []
    for locs in ([EL.DEVICE] * F, [EL.MANAGED] * F, [EL.MANAGED_CACHING] * F, [EL.DEVICE, EL.MANAGED, EL.MANAGED_CACHING, EL.MANAGED]):
        m = QuantTableBatchedEmbeddingBags(SPECS, pooling_mode=pooling_mode, locations=locs, cache_load_factor=0.1)
        for t, w in enumerate(weights):
            m.assign_from_float(t, w)
        outs.append(m(ids, offsets, psw, batch_size=B))
    for o in outs[1:]:
        assert torch.equal(o, outs[0])


def test_sequence_cpu_reference_path_serves_every_location():
    specs = [("a", 100, 32, DataType.INT4), ("b", 60, 32, DataType.FP8)]
    g = torch.Generator().manual_seed(1)
    weights = [torch.randn(r, d, generator=g) for _, r, d, _ in specs]
    ids = torch.tensor([3, 99, -1, 5, 59, 60, 0], dtype=torch.int32)
    offsets = torch.tensor([0, 2, 3, 5, 7], dtype=torch.int32)
    outs = []
    for locs in ([EL.DEVICE] * 2, [EL.MANAGED_CACHING, EL.MANAGED]):
        m = QuantTableBatchedEmbeddingBags(specs, pooling_mode=2, locations=locs)
        for t, w in enumerate(weights):
            m.assign_from_float(t, w)
        outs.append(m(ids, offsets, batch_size=2))
    assert torch.equal(outs[0], outs[1])


def test_all_device_module_is_unchanged():
    m = QuantTableBatchedEmbeddingBags(SPECS)
    assert not m._placed
    assert sorted(n for n, _ in m.named_buffers()) == ["feat_col", "feat_dim", "feat_fmt", "feat_rb", "feat_rows", "feat_woff", "weights"]
    assert m.weights.numel() == sum(r * m._row_bytes[t] for t, (_, r, _, _) in enumerate(SPECS))


@pytest.mark.parametrize("rows,clf", [(10000, 0.2), (4096, 0.05), (777, 1.0)])
def test_planner_estimate_matches_cache_allocation(rows, clf):
    from torchrec_b200.parallel.planner.shard_estimators import calculate_shard_storages
    from torchrec_b200.parallel.quant_embeddingbag import QuantEmbeddingBagCollectionSharder

    dim = 128
    m = QuantTableBatchedEmbeddingBags([("t", rows, dim, DataType.INT8)], locations=[EL.MANAGED_CACHING], cache_load_factor=clf)
    rb = m._row_bytes[0]
    table = torch.empty(rows, rb, dtype=torch.uint8, device="meta")  # the quantized table as the module stores it
    st = calculate_shard_storages(QuantEmbeddingBagCollectionSharder(), "table_wise", table, "cuda", "quant_uvm_caching", [[rows, rb]],
                                  batch_sizes=[0], world_size=1, local_world_size=1, input_lengths=[0.0], num_poolings=[0.0], caching_ratio=clf,
                                  is_pooled=True, is_inference=True)[0]
    cache_bytes = m._qc(0, "cache").numel() + 4 * m._qc(0, "slot_of_row").numel()
    assert m.cache_slots[0] == math.ceil(rows * clf)
    assert abs(st.hbm - cache_bytes) < rb  # the planner budgets load_factor * bytes; the module rounds up to whole rows
    assert st.ddr == m.split_embedding_weights()[0].numel() == rows * rb
