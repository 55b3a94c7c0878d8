"""Planner unit tests (no process group needed; mirrors the reference's planner/tests strategy)."""
import pytest
import torch

from torchrec_b200.modules.embedding_configs import EmbeddingBagConfig
from torchrec_b200.modules.embedding_modules import EmbeddingBagCollection
from torchrec_b200.parallel.embeddingbag import EmbeddingBagCollectionSharder
from torchrec_b200.parallel.planner import (
    DynamicProgrammingProposer,
    EmbeddingEnumerator,
    EmbeddingShardingPlanner,
    GreedyPerfPartitioner,
    MemoryBalancedPartitioner,
    ParameterConstraints,
    PlannerError,
    Topology,
)
from torchrec_b200.parallel.types import ShardingType


class Model(torch.nn.Module):
    def __init__(self, tables):
        super().__init__()
        self.sparse = EmbeddingBagCollection(tables, device=torch.device("meta"))


def _tables(n=6, rows=100_000, dim=128):
    return [EmbeddingBagConfig(name=f"t{i}", embedding_dim=dim, num_embeddings=rows * (i + 1), feature_names=[f"f{i}"]) for i in range(n)]


def test_enumerator_lists_all_sharding_types_single_domain():
    topo = Topology(world_size=8, compute_device="cuda")
    opts = EmbeddingEnumerator(topo, batch_size=512).enumerate(Model(_tables(2, dim=256)), [EmbeddingBagCollectionSharder()])
    types = {o.sharding_type for o in opts if o.name == "t0"}
    # single NVLink domain: TWRW / TWCW / GRID collapse onto RW / CW
    assert {"data_parallel", "table_wise", "row_wise", "column_wise"} <= types
    assert "table_row_wise" not in types and "grid_shard" not in types
    for o in opts:
        for s in o.shards:
            assert s.storage is not None and s.perf is not None and s.perf.total >= 0
    rw = [o for o in opts if o.name == "t0" and o.sharding_type == "row_wise"][0]
    assert sum(s.size[0] for s in rw.shards) == 100_000


def test_enumerator_multi_host_adds_hierarchical_types():
    topo = Topology(world_size=16, local_world_size=8, compute_device="cuda")
    opts = EmbeddingEnumerator(topo, batch_size=512).enumerate(Model(_tables(1, dim=512)), [EmbeddingBagCollectionSharder()])
    types = {o.sharding_type for o in opts}
    assert {"table_row_wise", "table_column_wise", "grid_shard"} <= types


def test_planner_balances_and_respects_constraints():
    topo = Topology(world_size=4, compute_device="cuda")
    constraints = {"t0": ParameterConstraints(sharding_types=["row_wise"]), "t1": ParameterConstraints(sharding_types=["column_wise"], min_partition=64)}
    planner = EmbeddingShardingPlanner(topology=topo, batch_size=1024, constraints=constraints)
    plan = planner.plan(Model(_tables()), [EmbeddingBagCollectionSharder()])
    mp = plan.plan["sparse"]
    assert mp["t0"].sharding_type == "row_wise" and len(mp["t0"].ranks) == 4
    assert mp["t1"].sharding_type == "column_wise" and len(mp["t1"].sharding_spec.shards) == 2
    used = set(r for ps in mp.values() for r in ps.ranks)
    assert used == {0, 1, 2, 3}
    assert any("Planner Statistics" in l for l in planner._stats[0]._stats_table)


def test_planner_insufficient_storage_raises():
    topo = Topology(world_size=2, compute_device="cuda", hbm_cap=64 * 1024 * 1024)
    cons = {f"t{i}": ParameterConstraints(compute_kernels=["fused"]) for i in range(4)}  # no host-offloaded (UVM) options
    planner = EmbeddingShardingPlanner(topology=topo, batch_size=512, constraints=cons)
    with pytest.raises(PlannerError):
        planner.plan(Model(_tables(4, rows=10_000_000)), [EmbeddingBagCollectionSharder()])


def test_big_table_forces_row_wise_when_it_does_not_fit_one_gpu():
    topo = Topology(world_size=8, compute_device="cuda", hbm_cap=8 * 1024**3)
    tables = [EmbeddingBagConfig(name="big", embedding_dim=128, num_embeddings=40_000_000, feature_names=["f"])]  # 20 GB fp32
    cons = {"big": ParameterConstraints(compute_kernels=["fused"])}
    plan = EmbeddingShardingPlanner(topology=topo, batch_size=512, constraints=cons).plan(Model(tables), [EmbeddingBagCollectionSharder()])
    assert plan.plan["sparse"]["big"].sharding_type in ("row_wise", "column_wise")


def test_partitioners_and_dp_proposer():
    topo = Topology(world_size=4, compute_device="cuda")
    m = Model(_tables())
    for part in (GreedyPerfPartitioner(), MemoryBalancedPartitioner()):
        plan = EmbeddingShardingPlanner(topology=topo, batch_size=512, partitioner=part, proposer=DynamicProgrammingProposer()).plan(m, [EmbeddingBagCollectionSharder()])
        assert set(plan.plan["sparse"].keys()) == {f"t{i}" for i in range(6)}


def test_sharding_route_facade():
    from torchrec_b200.modules.embedding_configs import EmbeddingBagConfig
    from torchrec_b200.modules.embedding_modules import EmbeddingBagCollection
    from torchrec_b200.parallel import sharding_plan as sp
    from torchrec_b200.parallel.embeddingbag import EmbeddingBagCollectionSharder
    from torchrec_b200.parallel.sharding import all_routes, describe, units_for

    assert {r.sharding_type for r in all_routes()} == {"data_parallel", "table_wise", "column_wise", "table_column_wise", "row_wise", "table_row_wise", "grid_shard"}
    assert "sum" in describe("row_wise").combine and describe("column_wise").reference_module.endswith("cw_sharding.py")
    cfg = EmbeddingBagConfig(name="t", embedding_dim=16, num_embeddings=100, feature_names=["f"])
    ebc = EmbeddingBagCollection([cfg], device="meta")
    plan = sp.construct_module_sharding_plan(ebc, {"t": sp.row_wise()}, sharder=EmbeddingBagCollectionSharder(), world_size=4, local_size=4, device_type="cpu")
    shards = units_for(0, cfg, plan["t"])
    assert [s.rank for s in shards] == [0, 1, 2, 3] and sum(s.rows for s in shards) == 100 and all(s.cols == 16 for s in shards)


def test_annotation_estimator_and_shard_estimators():
    """The annotation-driven estimator package: evaluators per sharding type, config overrides through decorators, factory; functional storage helpers."""
    import torch

    from torchrec_b200.parallel.planner import constants as K
    from torchrec_b200.parallel.planner.estimator import (
        EmbeddingPerfEstimatorFactory, HardwarePerfConfig, ShardPerfContext, compute_block_usage_penalty, forward_compute, get_embedding_perf_sharding_evaluator,
        get_forward_compute, hbm_mem_bw, intra_host_bw, supported_sharding_types)
    from torchrec_b200.parallel.planner.shard_estimators import EmbeddingOffloadStats, calculate_pipeline_io_cost, calculate_shard_storages
    from torchrec_b200.parallel.planner.types import PlannerError
    from torchrec_b200.parallel.types import PipelineType

    def ctx(st, W=8, L=8, cols=128, rows=1_000_000, n_row=1):
        return ShardPerfContext(sharding_type=st, compute_kernel="fused", compute_device="cuda", world_size=W, local_world_size=L, batch_sizes=[2048], input_lengths=[20.0],
                                num_poolings=[1.0], hash_size=rows, emb_dim=cols, shard_rows=rows // n_row, shard_cols=cols, num_row_shards=n_row, table_data_type_size=4.0,
                                output_data_type_size=4.0, fwd_a2a_comm_data_type_size=4.0, bwd_a2a_comm_data_type_size=4.0, fwd_sr_comm_data_type_size=4.0,
                                bwd_sr_comm_data_type_size=4.0, is_pooled=True, device_bw=K.HBM_MEM_BW, comms_bw=K.INTRA_NODE_BANDWIDTH)

    tw = get_embedding_perf_sharding_evaluator("table_wise").evaluate(ctx("table_wise"))
    rw = get_embedding_perf_sharding_evaluator("row_wise").evaluate(ctx("row_wise", n_row=8))
    dp = get_embedding_perf_sharding_evaluator("data_parallel").evaluate(ctx("data_parallel"))
    assert rw.fwd_compute < tw.fwd_compute            # 1/8 of the ids per shard
    assert dp.input_dist_comms == 0 and dp.fwd_comms == 0 and dp.bwd_comms > tw.bwd_comms   # whole-table all-reduce
    inf = get_embedding_perf_sharding_evaluator("table_wise", is_inference=True).evaluate(ctx("table_wise"))
    assert inf.bwd_compute == 0 and inf.bwd_comms == 0 and inf.fwd_compute == tw.fwd_compute
    two_hosts = get_embedding_perf_sharding_evaluator("table_row_wise").evaluate(ctx("table_row_wise", W=16, L=8, n_row=8))
    one_host = get_embedding_perf_sharding_evaluator("table_row_wise").evaluate(ctx("table_row_wise", W=8, L=8, n_row=8))
    assert two_hosts.fwd_comms > one_host.fwd_comms
    assert compute_block_usage_penalty(128) == 1.0 and compute_block_usage_penalty(64) == K.HALF_BLOCK_PENALTY and compute_block_usage_penalty(16) == K.QUARTER_BLOCK_PENALTY

    @hbm_mem_bw(1.0e6)
    @intra_host_bw(2.0e5)
    @supported_sharding_types("table_wise", "row_wise")
    class Slow(HardwarePerfConfig):
        name = "slow"

        @forward_compute(sharding_type="row_wise")
        def rw_fwd(self, c):
            return 123.0

    cfg = Slow()
    assert cfg.hbm_mem_bw == 1.0e6 and HardwarePerfConfig.hbm_mem_bw == K.HBM_MEM_BW
    assert get_forward_compute(cfg, "row_wise") is not None and get_forward_compute(cfg, "table_wise") is None
    assert get_embedding_perf_sharding_evaluator("row_wise", cfg).evaluate(ctx("row_wise", n_row=8)).fwd_compute == 123.0
    with pytest.raises(PlannerError):
        get_embedding_perf_sharding_evaluator("grid_shard", cfg)
    assert EmbeddingPerfEstimatorFactory.available() == ["gb200", "h100"]
    assert EmbeddingPerfEstimatorFactory.get_config("gb200").hbm_to_ddr_mem_bw > K.HBM_TO_DDR_MEM_BW

    # functional storage helpers
    assert calculate_pipeline_io_cost(100, 50, 0, PipelineType.TRAIN_SPARSE_DIST, None) == 200
    assert calculate_pipeline_io_cost(100, 50, 10, PipelineType.TRAIN_PREFETCH_SPARSE_DIST, 6, count_ephemeral_storage_cost=True) == 300 + 20 + 50
    assert calculate_pipeline_io_cost(100, 50, 0, PipelineType.NONE, None) == 150 and calculate_pipeline_io_cost(1, 1, 1, PipelineType.NONE, None, is_inference=True) == 0
    t = torch.empty(1000, 64)
    st = calculate_shard_storages(None, "row_wise", t, "cuda", "fused", [[250, 64]] * 4, [32], 4, 4, [10.0], [1.0], 0.2, True)
    assert len(st) == 4 and st[0].hbm >= 250 * 64 * 4 + 250 * 4 and st[0].ddr == 0
    st_uvm = calculate_shard_storages(None, "table_wise", t, "cuda", "fused_uvm_caching", [[1000, 64]], [32], 4, 4, [10.0], [1.0], 0.25, True)
    assert st_uvm[0].ddr >= 1000 * 64 * 4 and st_uvm[0].hbm < st_uvm[0].ddr

    stats = EmbeddingOffloadStats(cacheability=0.3, expected_lookups=1000, mrc_hist_counts=torch.tensor([50.0, 30.0, 15.0, 5.0]), height=300)
    assert stats.expected_miss_rate(0.0) == 1.0 and abs(stats.expected_miss_rate(1.0) - 0.05) < 1e-6
    assert stats.expected_miss_rate(0.2) > stats.expected_miss_rate(0.6)


def test_perf_model_matches_measured_fused_kernels():
    """The planner's table-wise lookup costs for the DLRM headline plan against what the kernels measured on one H100 80GB HBM3
    (``tools/kernel_bench.py``, the busiest rank of the W = 8 job: 4 tables x 262144 one-hot samples, fp32 rows -> bf16, row-wise
    Adagrad): forward 0.297 ms, backward 0.776 ms. The NVLink half (fused lookup + output dist) needs 8 GPUs to measure and is not
    asserted."""
    import torch

    from torchrec_b200.modules.embedding_configs import EmbeddingBagConfig
    from torchrec_b200.modules.embedding_modules import EmbeddingBagCollection
    from torchrec_b200.parallel.embeddingbag import EmbeddingBagCollectionSharder
    from torchrec_b200.parallel.planner import EmbeddingShardingPlanner, Topology
    from torchrec_b200.parallel.planner.types import ParameterConstraints

    hashes = [39884406, 39043, 17289, 7420, 20263, 3, 7120, 1543, 63, 38532951, 2953546, 403346, 10, 2208, 11938, 155, 4, 976, 14, 39979771, 25641295, 39664984,
              585935, 12972, 108, 36]
    tables = [EmbeddingBagConfig(name=f"t{i}", embedding_dim=128, num_embeddings=h, feature_names=[f"f{i}"]) for i, h in enumerate(hashes)]

    class M(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.ebc = EmbeddingBagCollection(tables=tables, device=torch.device("meta"))

    W, fwd_ms, bwd_ms = 8, 0.297, 0.776
    planner = EmbeddingShardingPlanner(topology=Topology(world_size=W, local_world_size=W, compute_device="cuda"), batch_size=32768,
                                       constraints={t.name: ParameterConstraints(sharding_types=["table_wise"], compute_kernels=["fused"]) for t in tables})
    planner.plan(M(), [EmbeddingBagCollectionSharder(fused_params={"output_dtype": torch.bfloat16})])
    per = {}
    for so in planner._best_plan:
        for sh in so.shards:
            d = per.setdefault(sh.rank, [0.0, 0.0, 0])
            d[0] += sh.perf.fwd_compute
            d[1] += sh.perf.bwd_compute
            d[2] += 1
    fc, bc, n_tables = max(per.values(), key=lambda d: d[0])
    assert n_tables == 4, per  # the measured shape: the busiest rank looks up 4 tables for the global batch
    assert fc == pytest.approx(fwd_ms, rel=0.25), (fc, fwd_ms)
    assert bc == pytest.approx(bwd_ms, rel=0.25), (bc, bwd_ms)


def test_plan_loader_topology_factory_and_planner_helpers():
    """A stored plan is re-used (no search) when the planner inputs hash to the stored context, refused otherwise; topology from the
    trainer / hardware / kernel layers; validators; small search / formatting helpers."""
    from typing import Dict, Optional

    from torchrec_b200.modules.embedding_configs import EmbeddingBagConfig
    from torchrec_b200.modules.embedding_modules import EmbeddingBagCollection
    from torchrec_b200.parallel.embeddingbag import EmbeddingBagCollectionSharder
    from torchrec_b200.parallel.planner import EmbeddingShardingPlanner, Topology
    from torchrec_b200.parallel.planner.partitioners import OrderedDeviceHardware
    from torchrec_b200.parallel.planner.perf_models import NoopStorageModel
    from torchrec_b200.parallel.planner.planners import extract_plan, validate_compute_kernels, validate_modules_inclusion_in_sharding_plan, validate_rank_assignment
    from torchrec_b200.parallel.planner.stats import round_to_one_sigfig
    from torchrec_b200.parallel.planner.types import (CriticalPathEstimate, HardwareConfig, KernelConfig, PlanLoader, PlannerError, PlannerErrorType, ShardingOption,
                                                      TopologyFactory, TrainerConfig, hash_sha256_str, hash_sha256_to_int, round_to_nearest)
    from torchrec_b200.parallel.planner.utils import LuusJaakolaSearch, build_sharder_data, extract_comm_data_type_size, get_num_poolings, is_prefetch_pipelined, mb_to_bytes
    from torchrec_b200.parallel.types import ShardingPlan

    class Model(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.ebc = EmbeddingBagCollection([EmbeddingBagConfig(name=f"t{i}", embedding_dim=16, num_embeddings=1000 * (i + 1), feature_names=[f"f{i}"]) for i in range(4)],
                                              device=torch.device("meta"))

    def planner(loader=None, batch_size=64):
        return EmbeddingShardingPlanner(topology=Topology(world_size=4, local_world_size=4, compute_device="cuda"), batch_size=batch_size, plan_loader=loader)

    sharders = [EmbeddingBagCollectionSharder()]
    first = planner()
    plan_a = first.plan(Model(), sharders)
    stored = {so.storage_hash(): so for so in first.best_plan}
    ctx_hash = first.hash_planner_context_inputs_str()
    assert len(stored) == 4 and isinstance(first.hash_planner_context_inputs(), int) and len(ctx_hash) == 64

    class Loader(PlanLoader):
        def __init__(self, options: Optional[Dict[int, ShardingOption]], ctx: Optional[str]):
            self.options, self.ctx, self.loads = options, ctx, 0

        def load(self):
            self.loads += 1
            return self.options

        def plan_context_hash(self):
            return self.ctx

        def get_plan_id(self):
            return "stored-1"

    loader = Loader(stored, ctx_hash)
    second = planner(loader)
    plan_b = second.plan(Model(), sharders)
    assert loader.loads == 1 and second._num_proposals == 0, "the stored plan is used as is"
    for name, ps in plan_a.plan["ebc"].items():
        other = plan_b.plan["ebc"][name]
        assert (ps.sharding_type, ps.compute_kernel, ps.ranks) == (other.sharding_type, other.compute_kernel, other.ranks)
    with pytest.raises(PlannerError) as e:
        planner(Loader(stored, ctx_hash), batch_size=128).plan(Model(), sharders)  # other inputs: the stored plan is not trusted
    assert e.value.error_type == PlannerErrorType.PLANNER_INPUT_CONTEXT_MISMATCH
    with pytest.raises(PlannerError) as e:
        planner(Loader({**stored, 12345: next(iter(stored.values()))}, None)).plan(Model(), sharders)  # an option the search space does not have
    assert e.value.error_type == PlannerErrorType.PLAN_LOADING_FAILED
    assert planner(Loader(None, None)).plan(Model(), sharders).plan["ebc"].keys() == plan_a.plan["ebc"].keys()  # nothing stored: normal search
    assert len(extract_plan(list(first._enumerator.last_stored_search_space), stored)) == 4
    # validators
    validate_rank_assignment(plan_a, Topology(world_size=4, compute_device="cuda"))
    with pytest.raises(PlannerError):
        validate_rank_assignment(plan_a, Topology(world_size=1, compute_device="cuda"))
    validate_compute_kernels(first.best_plan)
    bad = first.best_plan[0]
    bad.compute_kernel = "warp_drive"
    with pytest.raises(PlannerError) as e:
        validate_compute_kernels([bad])
    assert e.value.error_type == PlannerErrorType.INVALID_COMPUTE_KERNEL
    validate_modules_inclusion_in_sharding_plan(plan_a, Model(), sharders)
    with pytest.raises(PlannerError) as e:
        validate_modules_inclusion_in_sharding_plan(ShardingPlan({}), Model(), sharders)
    assert e.value.error_type == PlannerErrorType.MISSING_MODULE_IN_PLAN
    # topology from layers: trainer > hardware > defaults; dry run; bandwidths only from hardware when asked
    hw = HardwareConfig(hbm_cap_bytes=180 * 2**30, ddr_cap_bytes=2**40, intra_host_bw=7.0, hbm_mem_bw=9.0, additional_params={"gen": "h100"})
    t = TopologyFactory.create_topology(TrainerConfig(world_size=16, local_world_size=8, hbm_cap_bytes=100 * 2**30), hw, KernelConfig(use_hardware_based_bandwidth=True))
    assert (t.world_size, t.local_world_size, t.devices[3].storage.hbm, t.devices[3].storage.ddr) == (16, 8, 100 * 2**30, 2**40)
    assert t.comms_bandwidths.intra_host_bw == 7.0 and t.hbm_mem_bw == 9.0 and hw.get_param("gen") == "h100" and not hw.has_param("x")
    t2 = TopologyFactory.create_topology(TrainerConfig(world_size=2, is_dry_run=True, dry_run_hbm_bytes=5 * 2**30), hw)
    assert t2.devices[0].storage.hbm == 5 * 2**30 and t2.comms_bandwidths.intra_host_bw != 7.0
    with pytest.raises(ValueError):
        TopologyFactory.create_topology(TrainerConfig())
    with pytest.raises(ValueError):
        TopologyFactory.create_topology(TrainerConfig(world_size=2, pod_size=4))
    with pytest.raises(ValueError):
        TopologyFactory.create_topology(TrainerConfig(world_size=2), kernel_config=KernelConfig(compute_device="tpu"))
    # helpers
    assert CriticalPathEstimate(1.5, 2.0).total() == 3.5 and round_to_nearest(149 * 2**30, 100 * 2**30) == 100 * 2**30
    assert hash_sha256_to_int([1, "a"]) == int(hash_sha256_str([1, "a"]), 16)
    assert round_to_one_sigfig(0.0342) == "0.03" and round_to_one_sigfig(1234) == "1000" and mb_to_bytes(1.5) == 1572864
    s = LuusJaakolaSearch(0, 10, 80, left_cost=(0 - 3.3) ** 2)
    y = s.next(0.0)
    while y is not None:
        assert 0 <= y <= 10
        y = s.next((y - 3.3) ** 2)
    assert abs(s.best()[0] - 3.3) < 0.5
    s.shrink_right(2.0)
    assert s.right == 2.0 and s.best()[0] <= 2.0
    so = second.best_plan[0]
    data = build_sharder_data(sharders[0])
    assert data.storage_usage_type.value == "base" and extract_comm_data_type_size(so, data) == (4, 4, 4, 4) and not is_prefetch_pipelined(so, data)
    assert get_num_poolings(None, so) == [1.0] * len(so.input_lengths)
    assert NoopStorageModel(Topology(world_size=4, compute_device="cuda")).rate(second.best_plan) > 0
    devs = Topology(world_size=4, local_world_size=2, compute_device="cuda").devices
    order = sorted(OrderedDeviceHardware(d, 2) for d in devs)
    assert [o.device.rank for o in order] == [0, 2, 1, 3]  # equal load: local rank 0 of every host first


def test_row_wise_shards_on_bucket_boundaries():
    """``num_buckets``: whole buckets per rank (reference example: 10 rows, 4 ranks, 5 buckets -> 4, 2, 2, 2 rows)."""
    from torchrec_b200.parallel.sharding_plan import calculate_shard_sizes_and_offsets

    sizes, offs = calculate_shard_sizes_and_offsets(torch.empty(10, 4, device="meta"), 4, 4, "row_wise", num_buckets=5)
    assert sizes == [[4, 4], [2, 4], [2, 4], [2, 4]] and offs == [[0, 0], [4, 0], [6, 0], [8, 0]]
    sizes, _ = calculate_shard_sizes_and_offsets(torch.empty(10, 4, device="meta"), 4, 4, "row_wise")
    assert [s[0] for s in sizes] == [3, 3, 3, 1]
    with pytest.raises(AssertionError):
        calculate_shard_sizes_and_offsets(torch.empty(10, 4, device="meta"), 4, 4, "row_wise", num_buckets=3)
