"""Device-side prefetch of the fused_uvm_caching training cache: residency against a plain-Python model of the victim policy, results
against an uncached table, no host synchronisation, the overflow error, and the prefetch pipeline."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


class PolicyModel:
    """One table's cache: victims are the lowest (score, slot) among the slots the batch does not use; the k-th missing row (ascending)
    takes the k-th victim (ascending slot); LRU scores are the batch tick, LFU scores count uses (1 on admission)."""

    def __init__(self, cache_rows, lfu):
        self.C, self.lfu = cache_rows, lfu
        self.slot_of_row = {}
        self.row_of_slot = [-1] * cache_rows
        self.score = [0] * cache_rows
        self.stamp = [0] * cache_rows

    def prefetch(self, ids, tick):
        ids = sorted(set(ids))
        if len(ids) > self.C:
            return False
        misses = []
        for r in ids:
            s = self.slot_of_row.get(r)
            if s is None:
                misses.append(r)
                continue
            self.score[s] = self.score[s] + 1 if self.lfu else tick
            self.stamp[s] = tick
        cand = sorted((s for s in range(self.C) if self.stamp[s] < tick), key=lambda s: (self.score[s], s))
        for r, s in zip(misses, sorted(cand[: len(misses)])):
            old = self.row_of_slot[s]
            if old >= 0:
                del self.slot_of_row[old]
            self.slot_of_row[r] = s
            self.row_of_slot[s] = r
            self.score[s] = 1 if self.lfu else tick
            self.stamp[s] = tick
        return True


def _batch(rng, rows_of_feature, B, max_len, dist, empty=()):
    lengths, ids = [], []
    for f, R in enumerate(rows_of_feature):
        ln = np.zeros(B, dtype=np.int64) if f in empty else rng.integers(0, max_len + 1, B)
        k = int(ln.sum())
        x = (rng.zipf(1.15, k) - 1) % R if dist == "zipf" else rng.integers(0, R, k)
        lengths.append(ln)
        ids.append(x)
    lengths = np.concatenate(lengths)
    return np.concatenate(ids), np.concatenate([[0], np.cumsum(lengths)])


def _ids_per_table(idx, off, fmap, B, T):
    per = [[] for _ in range(T)]
    for f, t in enumerate(fmap):
        per[t].extend(idx[off[f * B] : off[(f + 1) * B]].tolist())
    return per


@pytest.mark.parametrize("algo", ["lru", "lfu"])
@pytest.mark.parametrize("wdtype,opt", [(torch.float32, "rowwise_adagrad"), (torch.float16, "adam"), (torch.float32, "adam"), (torch.float16, "rowwise_adagrad")])
@pytest.mark.parametrize("dist", ["zipf", "uniform"])
def test_residency_and_training_match(algo, wdtype, opt, dist):
    from torchrec_b200.ops.tbe import OptimType, PoolingMode, TableBatchedEmbeddingBags
    from torchrec_b200.ops.uvm import UvmCachedEmbeddingBags

    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    specs, fmap = [(3000, 16), (900, 36), (5000, 128)], [0, 1, 1, 2, 0]
    optim = {"rowwise_adagrad": OptimType.EXACT_ROWWISE_ADAGRAD, "adam": OptimType.ADAM}[opt]
    kw = dict(pooling_mode=PoolingMode.SUM, optimizer=optim, learning_rate=0.05, eps=1e-3, weights_precision=wdtype)
    full = TableBatchedEmbeddingBags(specs, fmap, device=dev, **kw)
    cached = UvmCachedEmbeddingBags(specs, fmap, cache_load_factor=0.0, cache_algorithm=algo, min_cache_rows=96, device=dev, **kw)
    cache_rows = cached.cache_rows
    with torch.no_grad():
        for w_c, w_f in zip(cached.split_embedding_weights(), full.split_embedding_weights()):
            w_c.copy_(w_f.cpu())
    cached.load_rows_changed()
    models = [PolicyModel(c, algo == "lfu") for c in cache_rows]
    rng = np.random.default_rng(7)
    g = torch.Generator().manual_seed(1)
    B = 8
    rows_of_feature = [specs[t][0] for t in fmap]
    # fp16 rows: the cached and the uncached update agree to fp16 resolution, not bit for bit
    tol = {} if wdtype == torch.float32 else dict(rtol=1e-2, atol=1e-3)
    tick = 0
    for step in range(30):
        if step == 10:  # a batch that needs exactly cache_rows[0] rows of table 0
            need = cache_rows[0]
            a = rng.permutation(specs[0][0])[:need]
            idx0, off0 = _batch(rng, rows_of_feature, B, 2, dist, empty=(0, 4))
            lens = np.diff(off0)
            lens[0:B] = 0
            lens[0] = need
            per_f = [idx0[off0[f * B] : off0[(f + 1) * B]] for f in range(len(fmap))]
            per_f[0] = a
            idx = np.concatenate(per_f)
            off = np.concatenate([[0], np.cumsum(lens)])
        else:
            idx, off = _batch(rng, rows_of_feature, B, 3, dist, empty=(2,) if step % 4 == 1 else ())
        idx_d = torch.from_numpy(idx).to(dev)
        off_d = torch.from_numpy(off).to(dev)
        cached.prefetch(idx_d, off_d, B)
        tick += 1
        for t, ids in enumerate(_ids_per_table(idx, off, fmap, B, len(specs))):
            assert models[t].prefetch(ids, tick)
            got = cached.row_of_slot[t].cpu().tolist()
            assert got == models[t].row_of_slot, f"step {step} table {t}"
            want_res = sorted(models[t].slot_of_row)
            assert sorted(r for r in got if r >= 0) == want_res
        o_f = full(idx_d, off_d, None, batch_size=B)
        o_c = cached(idx_d, off_d, None, batch_size=B)
        torch.testing.assert_close(o_c, o_f, **tol)
        gout = torch.randn(o_f.shape, generator=g).to(dev)
        o_f.backward(gout)
        o_c.backward(gout)
    st = cached.stats
    assert st["evictions"] > 0 and st["hits"] > 0 and st["misses"] >= st["evictions"]
    for w_c, w_f in zip(cached.split_embedding_weights(), full.split_embedding_weights()):
        torch.testing.assert_close(w_c, w_f.cpu(), **tol)
    for s_c, s_f in zip(cached.split_optimizer_states(), full.split_optimizer_states()):
        for k in s_f:
            torch.testing.assert_close(s_c[k], s_f[k].cpu(), **tol)


def _small_cache(algo="lru"):
    from torchrec_b200.ops.tbe import OptimType, PoolingMode
    from torchrec_b200.ops.uvm import UvmCachedEmbeddingBags

    kw = dict(pooling_mode=PoolingMode.SUM, optimizer=OptimType.EXACT_ROWWISE_ADAGRAD, learning_rate=0.1, eps=1e-3)
    return UvmCachedEmbeddingBags([(400, 8), (300, 16)], [0, 1], cache_load_factor=0.0, cache_algorithm=algo, min_cache_rows=40,
                                  device=torch.device("cuda:0"), **kw)


def test_prefetch_and_forward_do_not_synchronize():
    dev = torch.device("cuda:0")
    cached = _small_cache()
    B = 16
    batches = []
    g = torch.Generator().manual_seed(3)
    for _ in range(6):
        idx = torch.cat([torch.randint(0, 400, (B,), generator=g), torch.randint(0, 300, (B,), generator=g)]).to(dev)
        batches.append((idx, torch.arange(0, 2 * B + 1, device=dev)))
    cached.prefetch(*batches[0], B)  # first call builds the device-side table descriptors
    cached(*batches[0], None, batch_size=B)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for idx, off in batches[1:]:
            cached.prefetch(idx, off, B)
            cached(idx, off, None, batch_size=B)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert cached.stats["misses"] > 0


def test_overflow_raises_and_leaves_cache_unchanged():
    dev = torch.device("cuda:0")
    cached = _small_cache()
    B = 8
    ok_idx = torch.cat([torch.arange(B), torch.arange(B)]).to(dev)
    off = torch.tensor([0, B, 2 * B], device=dev)
    cached.prefetch(ok_idx, off, 1)
    torch.cuda.synchronize()
    state = lambda: (cached._slot_of_row, cached._row_of_slot, cached.score[1], cached.cache.weights, cached.cache.state1)
    before = [x.clone() for x in state()]
    big = torch.cat([torch.arange(B), torch.arange(50)]).to(dev)  # table 0: resident rows only; table 1 has 40 slots
    off_big = torch.tensor([0, B, B + 50], device=dev)
    cached.prefetch(big, off_big, 1)
    torch.cuda.synchronize()
    with pytest.raises(RuntimeError, match="table 1 holds 40 rows but the batch needs 50 distinct rows"):
        cached(big, off_big, None, batch_size=1)
    for a, b in zip(before, state()):
        assert torch.equal(a, b)
    cached.prefetch(big, off_big, 1)
    with pytest.raises(RuntimeError, match="table 1"):
        cached.stats


def test_prefetch_pipeline_with_evicting_cache_matches_plain_loop():
    from torchrec_b200.datasets.random import RandomRecDataset
    from torchrec_b200.models.dlrm import DLRM, DLRMTrain
    from torchrec_b200.modules.embedding_configs import EmbeddingBagConfig
    from torchrec_b200.modules.embedding_modules import EmbeddingBagCollection
    from torchrec_b200.optim.apply_optimizer_in_backward import apply_optimizer_in_backward
    from torchrec_b200.optim.keyed import CombinedOptimizer, KeyedOptimizerWrapper
    from torchrec_b200.optim.optimizers import in_backward_optimizer_filter
    from torchrec_b200.optim.rowwise_adagrad import RowWiseAdagrad
    from torchrec_b200.ops.uvm import UvmCachedEmbeddingBags
    from torchrec_b200.parallel import sharding_plan as sp
    from torchrec_b200.parallel import train_pipeline as tp
    from torchrec_b200.parallel.embeddingbag import EmbeddingBagCollectionSharder
    from torchrec_b200.parallel.model_parallel import DistributedModelParallel
    from torchrec_b200.parallel.types import CacheParams, ShardingPlan

    dev = torch.device("cuda:0")
    keys, hashes = ["f0", "f1"], [40000, 100]

    def build():
        torch.manual_seed(0)
        tables = [EmbeddingBagConfig(name=f"t{i}", embedding_dim=32, num_embeddings=h, feature_names=[keys[i]]) for i, h in enumerate(hashes)]
        ebc = EmbeddingBagCollection(tables, device=torch.device("meta"))
        apply_optimizer_in_backward(RowWiseAdagrad, ebc.parameters(), {"lr": 0.05})
        model = DLRMTrain(DLRM(ebc, 13, [32, 32], [32, 1], dense_device=dev))
        plan = sp.construct_module_sharding_plan(ebc, {"t0": sp.table_wise(rank=0, compute_kernel="fused_uvm_caching"), "t1": sp.table_wise(rank=0)},
                                                 sharder=EmbeddingBagCollectionSharder(), world_size=1, local_size=1, device_type="cuda")
        plan["t0"].cache_params = CacheParams(load_factor=0.01)
        dmp = DistributedModelParallel(model, device=dev, plan=ShardingPlan({"model.sparse_arch.embedding_bag_collection": plan}),
                                       sharders=[EmbeddingBagCollectionSharder()])
        eng = dmp.module.model.sparse_arch.embedding_bag_collection._engine
        with torch.no_grad():
            gen = torch.Generator().manual_seed(11)
            for _, w, _st, _tbe in eng.local_shard_views():
                w.copy_((torch.randn(w.shape, generator=gen) * 0.1).to(w.device))
            for tbe in eng._tbes:
                if isinstance(tbe, UvmCachedEmbeddingBags):
                    tbe.load_rows_changed()
            for p in dmp.parameters():
                if p.requires_grad:
                    p.copy_((torch.randn(p.shape, generator=gen) * 0.05).to(p.device))
        dense_opt = KeyedOptimizerWrapper(dict(in_backward_optimizer_filter(dmp.named_parameters())), lambda p: torch.optim.SGD(p, lr=0.05))
        return dmp, CombinedOptimizer([dmp.fused_optimizer, dense_opt]), eng

    dmp_a, opt_a, eng_a = build()
    dmp_b, opt_b, eng_b = build()
    cached = [t for t in eng_b._tbes if isinstance(t, UvmCachedEmbeddingBags)]
    assert len(cached) == 1
    n = 12
    ds = RandomRecDataset(keys, 128, hash_sizes=hashes, ids_per_features=[3, 1], num_dense=13, manual_seed=8, num_generated_batches=n, num_batches=n, pin_memory=True)
    host = list(iter(ds))
    ref = []
    for b in host:
        b = b.to(dev)
        opt_a.zero_grad()
        loss, _ = dmp_a(b)
        loss.backward()
        opt_a.step()
        ref.append(float(loss))
    pipe = tp.PrefetchTrainPipelineSparseDist(dmp_b, opt_b, dev)
    it = iter(host)
    got = []
    while True:
        try:
            got.append(float(pipe.progress(it)[0]))
        except StopIteration:
            break
    torch.cuda.synchronize()
    assert cached[0].stats["evictions"] > 0
    assert got == pytest.approx(ref, rel=2e-4, abs=1e-5)
    wa = torch.cat([w.flatten().float().cpu() for _, w, _s, _t in eng_a.local_shard_views()])
    wb = torch.cat([w.flatten().float().cpu() for _, w, _s, _t in eng_b.local_shard_views()])
    torch.testing.assert_close(wb, wa, rtol=2e-4, atol=1e-6)


def test_back_to_back_prefetches_report_the_later_overflow():
    """The overflow of a prefetch issued while an earlier one is still pending is raised by ``stats`` at the latest."""
    dev = torch.device("cuda:0")
    cached = _small_cache()
    ok = torch.cat([torch.arange(8), torch.arange(8)]).to(dev)
    off = torch.tensor([0, 8, 16], device=dev)
    big = torch.cat([torch.arange(8), torch.arange(50)]).to(dev)
    off_big = torch.tensor([0, 8, 58], device=dev)
    cached.prefetch(ok, off, 1)
    cached.prefetch(big, off_big, 1)
    try:
        cached(big, off_big, None, batch_size=1)
    except RuntimeError as e:  # the forward may already see it
        assert "table 1" in str(e)
        return
    with pytest.raises(RuntimeError, match="table 1 holds 40 rows but the batch needs 50 distinct rows"):
        cached.stats


class ProtectingModel(PolicyModel):
    """PolicyModel whose victims also exclude the slots stamped at or after ``protect_from`` (a batch still in flight)."""

    def prefetch(self, ids, tick, protect_from=None):
        pf = tick if protect_from is None else protect_from
        ids = sorted(set(ids))
        misses = []
        for r in ids:
            s = self.slot_of_row.get(r)
            if s is None:
                misses.append(r)
                continue
            self.score[s] = self.score[s] + 1 if self.lfu else tick
            self.stamp[s] = tick
        cand = sorted((s for s in range(self.C) if self.stamp[s] < pf), key=lambda s: (self.score[s], s))
        for r, s in zip(misses, sorted(cand[: len(misses)])):
            old = self.row_of_slot[s]
            if old >= 0:
                del self.slot_of_row[old]
            self.slot_of_row[r] = s
            self.row_of_slot[s] = r
            self.score[s] = 1 if self.lfu else tick
            self.stamp[s] = tick
        return True


@pytest.mark.parametrize("algo", ["lru", "lfu"])
@pytest.mark.parametrize("start_tick", [0, 5000, 5_000_000])
@pytest.mark.parametrize("side_stream", [False, True])
def test_residency_at_large_ticks_and_with_an_in_flight_batch(algo, start_tick, side_stream):
    """Ticks past 2^11 and 2^22 (5000, 5M) run the second and third digit passes of the victim select; on a side stream the prefetch also spares
    the slots of the batch whose lookup ran last on the main stream. Residency must follow the model in both cases."""
    dev = torch.device("cuda:0")
    cached = _small_cache(algo)
    cached._tick = start_tick
    models = [ProtectingModel(c, algo == "lfu") for c in cached.cache_rows]
    side = torch.cuda.Stream(dev)
    rng = np.random.default_rng(11)
    B = 4
    tick, lookup_tick = start_tick, None
    for step in range(25):
        idx, off = _batch(rng, [400, 300], B, 4, "zipf" if step % 2 else "uniform")
        idx_d, off_d = torch.from_numpy(idx).to(dev), torch.from_numpy(off).to(dev)
        if side_stream:
            side.wait_stream(torch.cuda.current_stream(dev))
            with torch.cuda.stream(side):
                cached.prefetch(idx_d, off_d, B)
        else:
            cached.prefetch(idx_d, off_d, B)
        tick += 1
        pf = min(tick, lookup_tick) if (side_stream and lookup_tick is not None) else tick
        for t, ids in enumerate(_ids_per_table(idx, off, [0, 1], B, 2)):
            models[t].prefetch(ids, tick, pf)
        torch.cuda.synchronize()
        for t in range(2):
            assert cached.row_of_slot[t].cpu().tolist() == models[t].row_of_slot, f"step {step} table {t}"
        cached(idx_d, off_d, None, batch_size=B).sum().backward()
        lookup_tick = tick
    assert cached.stats["evictions"] > 0


@pytest.mark.parametrize("backend", ["dram", "ssd"])
def test_key_value_tables_train_on_cuda(backend, tmp_path):
    """Key-value tables on the GPU, DRAM store (rows moved zero-copy by the prefetch kernels) and SSD store (rows moved by the store's
    staging path from the device-side victim lists), against a dense table that holds the same rows."""
    from torchrec_b200.ops.kv_tbe import KeyValueEmbeddingBags
    from torchrec_b200.ops.tbe import OptimType, TableBatchedEmbeddingBags

    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    D, B = 16, 12
    kw = dict(optimizer=OptimType.EXACT_ROWWISE_ADAGRAD, learning_rate=0.1, eps=1e-3)
    # 60 + 50 keys over stores of 64 rows and caches of 16 rows: every step evicts
    kv = KeyValueEmbeddingBags([(1 << 12, D), (1 << 12, D)], [0, 1], store_rows=[64, 64], backend=backend, ssd_storage_directory=str(tmp_path / "kv"),
                               cache_load_factor=0.25, min_cache_rows=16, device=dev, **kw)
    g = torch.Generator().manual_seed(4)
    pools = [torch.randint(1 << 33, 1 << 39, (60,), generator=g), torch.randint(1 << 20, 1 << 38, (50,), generator=g)]
    dense = TableBatchedEmbeddingBags([(60, D), (50, D)], [0, 1], device=dev, **kw)
    for f in range(2):
        kv._keys_to_slots(f, pools[f].to(dev))
        keys_f, rows_f = kv.key_value_snapshot(f)
        order = (keys_f.unsqueeze(1) == pools[f].unsqueeze(0)).long().argmax(1)
        with torch.no_grad():
            dense.split_embedding_weights()[f][order.to(dev)] = rows_f.to(dev)
    for step in range(8):
        lengths = torch.randint(0, 2, (2 * B,), generator=g)
        vals = torch.cat([pool[torch.randint(0, pool.numel(), (int(lengths[f * B : (f + 1) * B].sum()),), generator=g)] for f, pool in enumerate(pools)])
        off = torch.cat([torch.zeros(1, dtype=torch.int64), lengths.cumsum(0)])
        pos = vals.clone()
        bounds = [int(off[0]), int(off[B]), int(off[2 * B])]
        for f in range(2):
            seg = vals[bounds[f] : bounds[f + 1]]
            pos[bounds[f] : bounds[f + 1]] = (seg.unsqueeze(1) == pools[f].unsqueeze(0)).long().argmax(1)
        out_kv = kv(vals.to(dev), off.to(dev), batch_size=B)
        out_d = dense(pos.to(dev), off.to(dev), batch_size=B)
        torch.testing.assert_close(out_kv, out_d, rtol=1e-5, atol=1e-6)
        gr = torch.randn(out_kv.shape, generator=g).to(dev)
        out_kv.backward(gr)
        out_d.backward(gr)
    assert kv.stats["evictions"] > 0
    for f in range(2):
        keys_f, rows_f = kv.key_value_snapshot(f)
        order = (keys_f.unsqueeze(1) == pools[f].unsqueeze(0)).long().argmax(1)
        torch.testing.assert_close(rows_f.to(dev), dense.split_embedding_weights()[f][order.to(dev)], rtol=1e-5, atol=1e-6)
    kv.close()
