"""Software-managed HBM cache over host-resident embedding tables (compute kernel FUSED_UVM_CACHING).

Parity: fbgemm's UVM + LRU/LFU cache inside SplitTableBatchedEmbeddingBagsCodegen (``prefetch`` / ``flush`` /
``cache_load_factor``; reference call sites distributed/embedding_lookup.py:714-767, batched_embedding_kernel.py).

Design (GPU-first, not a port of the 32-way set-associative lxu cache): the table-batched kernels ALWAYS run on a
device-resident cache table and see *slot* ids; a direct map ``slot_of_row`` (int32 per row, in HBM: 4 B/row) translates
ids -> slots, so the cache is fully associative and there are no conflict misses. ``prefetch`` (on a side stream, one
batch ahead) makes every id of the batch resident: victims are the least-recently / least-frequently used slots, their
rows AND optimizer state go back to pinned host memory and the missing rows come in. On CUDA the whole prefetch of all
tables is one sequence of kernels (``csrc/uvm_cache.cu``) that never waits on the device; the CPU emulation keeps a
host loop. Host tables the GPU cannot address (the SSD store of ``kv_tbe``) keep the device-side bookkeeping, but their rows
move through ``_move`` after reading the victim lists back. Forward and the fused backward+optimizer then touch HBM only.

Victim policy: per table, the victims are the ``n_miss`` slots with the lowest score (LRU: tick of the last batch that used
the slot; LFU: use count) among the slots the batch does not use, ties to the lower slot index; the k-th missing row
(ascending id) takes the k-th victim (ascending slot). A prefetch issued on another stream than the last lookup also spares
the slots of that lookup's batch, whose forward / backward may still run: under ``PrefetchTrainPipelineSparseDist`` the
cache must hold the distinct rows of two consecutive batches, and residency there differs from the single-stream policy.

Overflow: a table whose batch needs more distinct rows than it has slots moves nothing and leaves its cache state as it
was. When the rows fit but the slots left after sparing the in-flight batch do not, the hit scores and hit / miss counts of
the batch are already updated, but still no row moves. Either raises ``RuntimeError`` at the next ``prefetch`` / ``forward``
(once the prefetch has run), or at the latest in ``flush`` / ``stats``, which wait for it."""
from __future__ import annotations

import ctypes
import math
from typing import Dict, List, Optional, Sequence, Tuple

import torch
from torch import nn

from . import _lib
from .tbe import _OPT_STATE, _OPT_STATE_NAMES, EmbeddingLocation, OptimType, PoolingMode, TableBatchedEmbeddingBags


def row_copy(dst: torch.Tensor, dst_idx: Optional[torch.Tensor], src: torch.Tensor, src_idx: Optional[torch.Tensor], n: int, row_bytes: int, device: torch.device) -> None:
    """dst[dst_idx[i]] = src[src_idx[i]] for rows of ``row_bytes``; either side may be pinned host memory."""
    if n == 0:
        return
    if device.type != "cuda":
        d = dst.view(torch.uint8).view(-1, row_bytes)
        s = src.view(torch.uint8).view(-1, row_bytes)
        di = dst_idx.long() if dst_idx is not None else torch.arange(n)
        si = src_idx.long() if src_idx is not None else torch.arange(n)
        d[di] = s[si]
        return
    L = _lib.lib()
    code = L.trb_row_copy(_lib.ptr(dst), _lib.ptr(dst_idx), _lib.ptr(src), _lib.ptr(src_idx), ctypes.c_int64(n), ctypes.c_int64(row_bytes), _lib.stream_ptr(device))
    _lib.check(code, "trb_row_copy")


class _PrefetchArgs(ctypes.Structure):
    """``UvmPrefetchArgs`` of csrc/uvm_cache.cu."""
    _fields_ = [(n, ctypes.c_void_p) for n in ("indices", "offsets", "table_of_feature", "row_base", "slot_base", "host_elem_base", "cache_elem_base", "dim",
                                               "slot_of_row", "row_of_slot", "score", "stamp", "host_w", "cache_w", "host_s1", "cache_s1", "host_s2", "cache_s2",
                                               "stats", "overflow", "workspace")] + \
              [(n, ctypes.c_int64) for n in ("workspace_bytes", "n", "total_rows", "idx64", "off64", "B", "F", "T", "w_bytes", "s1_kind", "s2_kind", "tick",
                                             "protect_from", "lfu", "move_rows")]


class UvmCachedEmbeddingBags(nn.Module):
    """Drop-in for ``TableBatchedEmbeddingBags`` whose tables live in pinned host memory behind an HBM cache.

    cache_load_factor: fraction of every table's rows kept in HBM (at least ``min_cache_rows``).
    cache_algorithm: "lru" | "lfu"."""

    is_cached = True

    def __init__(self, embedding_specs: Sequence[Tuple[int, int]], feature_table_map: Optional[Sequence[int]] = None, cache_load_factor: float = 0.2,
                 cache_algorithm: str = "lru", min_cache_rows: int = 1024, device: Optional[torch.device] = None, **tbe_kwargs) -> None:
        super().__init__()
        self.device = torch.device(device) if device is not None else torch.device("cpu")
        self.embedding_specs = [(int(r), int(d)) for r, d in embedding_specs]
        self.feature_table_map = list(feature_table_map) if feature_table_map is not None else list(range(len(self.embedding_specs)))
        self.cache_algorithm = cache_algorithm
        self.cache_rows = [min(r, max(min_cache_rows, int(math.ceil(r * cache_load_factor)))) for r, _ in self.embedding_specs]
        self.location = EmbeddingLocation.MANAGED_CACHING
        tbe_kwargs.pop("location", None)
        # the kernels run on the cache table
        self.cache = TableBatchedEmbeddingBags([(c, d) for c, (_, d) in zip(self.cache_rows, self.embedding_specs)], self.feature_table_map, device=self.device,
                                               location=EmbeddingLocation.DEVICE if self.device.type == "cuda" else EmbeddingLocation.HOST, **tbe_kwargs)
        pin = self.device.type == "cuda"
        wdtype = self.cache.weights.dtype
        total = sum(r * d for r, d in self.embedding_specs)
        self.total_rows = sum(r for r, _ in self.embedding_specs)
        self.host_weights = torch.empty(total, dtype=wdtype, pin_memory=pin)
        k1, k2 = _OPT_STATE[self.cache.opt_code]
        mk = lambda kind: None if kind is None else torch.zeros(self.total_rows if kind == "row" else total, dtype=torch.float32, pin_memory=pin)
        self.host_state1, self.host_state2 = mk(k1), mk(k2)
        self._kinds = (k1, k2)
        # id <-> slot maps (HBM), recency / frequency per slot: one flat buffer each, a view per table
        slots_total = sum(self.cache_rows)
        self._slot_of_row = torch.full((self.total_rows,), -1, dtype=torch.int32, device=self.device)
        self._row_of_slot = torch.full((slots_total,), -1, dtype=torch.int64, device=self.device)
        self._score = torch.zeros(slots_total, dtype=torch.int64, device=self.device)
        self._stamp = torch.zeros(slots_total, dtype=torch.int64, device=self.device)  # tick of the last batch that used the slot
        self.slot_of_row = list(torch.split(self._slot_of_row, [r for r, _ in self.embedding_specs]))
        self.row_of_slot = list(torch.split(self._row_of_slot, self.cache_rows))
        self.score = list(torch.split(self._score, self.cache_rows))
        self._tick = 0
        self._prefetched: Optional[Tuple[int, int]] = None
        self._host_stats = {"hits": 0, "misses": 0, "evictions": 0}
        T = len(self.embedding_specs)
        self._stats_dev = torch.zeros(T, 3, dtype=torch.int64, device=self.device) if self.device.type == "cuda" else None
        self._overflow = torch.zeros(T, dtype=torch.int32, pin_memory=pin)  # mapped host memory: the prefetch kernels write it
        self._overflow_event: Optional[torch.cuda.Event] = None
        self._last: Optional[Tuple[torch.cuda.Event, torch.cuda.Stream]] = None  # last prefetch / lookup that touched the cache state
        self._prefetch_tick = 0       # tick of the batch `_prefetched` names
        self._lookup: Optional[Tuple[int, torch.cuda.Stream]] = None  # (tick, stream) of the last lookup's batch
        # host init (the cache starts empty)
        o = 0
        for r, d in self.embedding_specs:
            b = math.sqrt(1.0 / r)
            self.host_weights[o : o + r * d].copy_(torch.empty(r * d, dtype=torch.float32).uniform_(-b, b))
            o += r * d

    # ---- delegation of the TBE surface the sharding engine uses ---------------------------------------------------------
    def __getattr__(self, name: str):
        try:
            return super().__getattr__(name)
        except AttributeError:
            if name in ("opt_code", "hyper_host", "hyper_dev", "_dummy", "weight_decay_mode", "pooling_mode", "output_dtype", "table_names", "_state_kinds"):
                return getattr(self._modules["cache"], name)
            raise

    @property
    def weights(self) -> torch.Tensor:
        return self.host_weights

    @property
    def state1(self) -> Optional[torch.Tensor]:
        return self.host_state1

    @property
    def state2(self) -> Optional[torch.Tensor]:
        return self.host_state2

    def set_learning_rate(self, lr: float) -> None:
        self.cache.set_learning_rate(lr)

    def get_learning_rate(self) -> float:
        return self.cache.get_learning_rate()

    def set_optimizer_step(self, step: int) -> None:
        self.cache.set_optimizer_step(step)

    def _pre_update(self) -> None:
        self.cache._pre_update()

    @torch.no_grad()
    def init_parameters(self, init_ranges: Optional[Sequence[Tuple[float, float]]] = None) -> None:
        self.flush(invalidate=True)
        for t, w in enumerate(self.split_embedding_weights(flush=False)):
            rows = self.embedding_specs[t][0]
            lo, hi = init_ranges[t] if init_ranges is not None else (-math.sqrt(1.0 / rows), math.sqrt(1.0 / rows))
            w.copy_(torch.empty(w.shape, dtype=torch.float32).uniform_(lo, hi))

    # ---- host <-> cache row movement --------------------------------------------------------------------------------------
    def _bases(self, t: int) -> Tuple[int, int, int, int]:
        """(host element offset, host row offset, cache element offset, cache row offset) of table t."""
        he = sum(r * d for r, d in self.embedding_specs[:t])
        hr = sum(r for r, _ in self.embedding_specs[:t])
        ce = sum(c * d for c, (_, d) in zip(self.cache_rows[:t], self.embedding_specs[:t]))
        cr = sum(self.cache_rows[:t])
        return he, hr, ce, cr

    def _move(self, t: int, rows: torch.Tensor, slots: torch.Tensor, to_host: bool) -> None:
        n = rows.numel()
        if n == 0:
            return
        he, hr, ce, cr = self._bases(t)
        D = self.embedding_specs[t][1]
        esz = self.host_weights.element_size()
        pairs = [(self.host_weights, he * esz, self.cache.weights, ce * esz, D * esz)]
        for kind, hs, cs in ((self._kinds[0], self.host_state1, self.cache.state1), (self._kinds[1], self.host_state2, self.cache.state2)):
            if kind == "row":
                pairs.append((hs, hr * 4, cs, cr * 4, 4))
            elif kind == "elem":
                pairs.append((hs, he * 4, cs, ce * 4, D * 4))
        rows = rows.to(torch.int64).contiguous()
        slots = slots.to(torch.int64).contiguous()
        for host, hoff, cache, coff, rb in pairs:
            hb = host.view(torch.uint8)[hoff:]
            cb = cache.view(torch.uint8)[coff:]
            if to_host:
                row_copy(hb, rows, cb, slots, n, rb, self.device)
            else:
                row_copy(cb, slots, hb, rows, n, rb, self.device)

    # ---- counters and errors of the device-side prefetch ------------------------------------------------------------------------
    @property
    def stats(self) -> Dict[str, int]:
        """Cumulative ``hits`` / ``misses`` / ``evictions`` over distinct rows per batch (on CUDA read from device counters here)."""
        if self._stats_dev is None:
            return dict(self._host_stats)
        self._after_last(torch.cuda.current_stream(self.device))
        self._check_overflow(wait=True)
        h, m, e = self._stats_dev.sum(0).tolist()
        return {"hits": int(h), "misses": int(m), "evictions": int(e)}

    def _check_overflow(self, wait: bool = False) -> None:
        """Raise for an overflowing prefetch. The flags are sticky and any set flag is final, so without ``wait`` they are read as they
        stand (a prefetch still running reports at a later call); ``wait`` first waits for the latest prefetch, which covers all earlier."""
        if wait and self._overflow_event is not None:
            self._overflow_event.synchronize()
            self._overflow_event = None
        bad = self._overflow.nonzero(as_tuple=True)[0]
        if bad.numel():
            t = int(bad[0])
            need = int(self._overflow[t])
            self._overflow.zero_()
            if need > 0:
                raise RuntimeError(f"UVM cache of table {t} holds {self.cache_rows[t]} rows but the batch needs {need} distinct rows; raise cache_load_factor")
            raise RuntimeError(f"UVM cache of table {t} holds {self.cache_rows[t]} rows, too few for the prefetched batch and the batch still in flight "
                               "on another stream (a prefetch pipeline keeps the rows of two consecutive batches resident); raise cache_load_factor")

    def _after_last(self, stream) -> None:
        """Order ``stream`` after the last prefetch / lookup when that ran on another stream (device-side wait)."""
        if self._last is not None and self._last[1] != stream:
            stream.wait_event(self._last[0])

    def _mark(self, stream) -> None:
        ev = torch.cuda.Event()
        ev.record(stream)
        self._last = (ev, stream)

    def _dev_tables(self) -> Dict[str, torch.Tensor]:
        tab = self.__dict__.get("_dev_tab")
        if tab is None:
            rows = [r for r, _ in self.embedding_specs]
            dims = [d for _, d in self.embedding_specs]
            cum = lambda xs: [sum(xs[:i]) for i in range(len(xs) + 1)]
            mk = lambda xs, dt=torch.int64: torch.tensor(xs, dtype=dt, device=self.device)
            tab = {"tof": mk(self.feature_table_map, torch.int32), "row_base": mk(cum(rows)), "slot_base": mk(cum(self.cache_rows)),
                   "host_elem": mk(cum([r * d for r, d in self.embedding_specs])[:-1]),
                   "cache_elem": mk(cum([c * d for c, d in zip(self.cache_rows, dims)])[:-1]), "dim": mk(dims)}
            self.__dict__["_dev_tab"] = tab
        return tab

    def _prefetch_cuda(self, indices: torch.Tensor, offsets: torch.Tensor, B: int) -> None:
        self._check_overflow()
        # host tables the GPU cannot address (an SSD-backed key-value store): the kernels only update the maps, `_move` moves the rows
        zero_copy = all(t is None or t.is_pinned() for t in (self.host_weights, self.host_state1, self.host_state2))
        stream = torch.cuda.current_stream(self.device)
        self._after_last(stream)
        protect_from = self._tick
        if self._lookup is not None and self._lookup[1] != stream:
            protect_from = min(protect_from, self._lookup[0])  # that lookup's forward / backward may still use its slots
        idx, off = indices.contiguous(), offsets.contiguous()
        idx.record_stream(stream)
        off.record_stream(stream)
        tab = self._dev_tables()
        L = _lib.lib()
        L.trb_uvm_prefetch_ws_bytes.restype = ctypes.c_int64
        T = len(self.embedding_specs)
        ws = torch.empty(int(L.trb_uvm_prefetch_ws_bytes(ctypes.c_int64(idx.numel()), ctypes.c_int64(T), ctypes.c_int64(self.total_rows))), dtype=torch.uint8,
                         device=self.device)
        kind = {None: 0, "row": 1, "elem": 2}
        p = lambda t: t.data_ptr() if t is not None else 0
        a = _PrefetchArgs(p(idx), p(off), p(tab["tof"]), p(tab["row_base"]), p(tab["slot_base"]), p(tab["host_elem"]), p(tab["cache_elem"]), p(tab["dim"]),
                          p(self._slot_of_row), p(self._row_of_slot), p(self._score), p(self._stamp), p(self.host_weights), p(self.cache.weights),
                          p(self.host_state1), p(self.cache.state1), p(self.host_state2), p(self.cache.state2), p(self._stats_dev), p(self._overflow),
                          p(ws), ws.numel(), idx.numel(), self.total_rows, int(idx.dtype == torch.int64), int(off.dtype == torch.int64), B,
                          len(self.feature_table_map), T, self.host_weights.element_size(), kind[self._kinds[0]], kind[self._kinds[1]], self._tick,
                          protect_from, int(self.cache_algorithm == "lfu"), int(zero_copy))
        _lib.check(L.trb_uvm_prefetch(ctypes.byref(a), _lib.stream_ptr(self.device)), "trb_uvm_prefetch")
        self._mark(stream)
        self._overflow_event = self._last[0]
        if not zero_copy:
            self._move_listed_rows(ws, idx.numel())

    def _move_listed_rows(self, ws: torch.Tensor, n: int) -> None:
        """Row movement of a prefetch that ran with ``move_rows = 0``: read the victim / old-row / missing-row lists back (a host wait,
        which a store on SSD needs anyway) and move the rows of every table through ``_move``: write-back first, then the fill."""
        T = len(self.embedding_specs)
        lay = (ctypes.c_int64 * 6)()
        _lib.check(_lib.lib().trb_uvm_prefetch_ws_layout(ctypes.c_int64(n), ctypes.c_int64(T), ctypes.c_int64(self.total_rows), lay), "trb_uvm_prefetch_ws_layout")
        o_sel, o_base, o_take, o_victim, o_old, o_miss = list(lay)
        view = lambda off, cnt, dt: ws[off : off + cnt * torch.empty(0, dtype=dt).element_size()].view(dt)
        n_sel = int(view(o_sel, 1, torch.int32))
        if n_sel == 0:
            return
        miss_base = view(o_base, T + 1, torch.int64).tolist()
        take = view(o_take, T, torch.int32).tolist()
        victim, old, miss = view(o_victim, n_sel, torch.int64), view(o_old, n_sel, torch.int64), view(o_miss, n_sel, torch.int64)
        slot_base = self._dev_tables()["slot_base"].tolist()
        row_base = self._dev_tables()["row_base"].tolist()
        for t in range(T):
            lo, hi = miss_base[t], miss_base[t + 1]
            if not take[t] or hi == lo:
                continue
            slots = victim[lo:hi] - slot_base[t]
            prev = old[lo:hi]
            live = prev >= 0
            self._move(t, prev[live], slots[live], to_host=True)
            self._move(t, miss[lo:hi] - row_base[t], slots, to_host=False)

    # ---- prefetch: make every id of the batch resident --------------------------------------------------------------------------
    @torch.no_grad()
    def prefetch(self, indices: torch.Tensor, offsets: torch.Tensor, batch_size: Optional[int] = None) -> None:
        F = len(self.feature_table_map)
        B = batch_size if batch_size is not None else (offsets.numel() - 1) // max(F, 1)
        self._tick += 1
        if self.device.type == "cuda":
            self._prefetch_cuda(indices, offsets, B)
            self._prefetched = (indices.data_ptr(), int(indices.numel()))
            self._prefetch_tick = self._tick
            return
        bounds = offsets[torch.arange(0, F + 1, device=offsets.device) * B].tolist()
        per_table: Dict[int, List[torch.Tensor]] = {}
        for f, t in enumerate(self.feature_table_map):
            lo, hi = int(bounds[f]), int(bounds[f + 1])
            if hi > lo:
                per_table.setdefault(t, []).append(indices[lo:hi])
        for t, parts in per_table.items():
            rows_t = self.embedding_specs[t][0]
            ids = torch.unique(torch.cat(parts).long())
            ids = ids[(ids >= 0) & (ids < rows_t)]
            if ids.numel() > self.cache_rows[t]:
                raise RuntimeError(f"UVM cache of table {t} holds {self.cache_rows[t]} rows but the batch needs {ids.numel()} distinct rows; raise cache_load_factor")
            slots = self.slot_of_row[t][ids].long()
            hit = slots >= 0
            score = self.score[t]
            if self.cache_algorithm == "lfu":
                score[slots[hit]] += 1
            else:
                score[slots[hit]] = self._tick
            miss_ids = ids[~hit]
            n_miss = int(miss_ids.numel())
            self._host_stats["hits"] += int(hit.sum())
            self._host_stats["misses"] += n_miss
            if n_miss == 0:
                continue
            # victims: lowest score among slots NOT used by this batch
            protect = torch.zeros_like(score, dtype=torch.bool)
            protect[slots[hit]] = True
            cand = torch.where(protect, torch.full_like(score, torch.iinfo(torch.int64).max), score)
            victims = torch.topk(cand, n_miss, largest=False).indices
            old_rows = self.row_of_slot[t][victims]
            live = old_rows >= 0
            if bool(live.any()):
                self._move(t, old_rows[live], victims[live], to_host=True)
                self.slot_of_row[t][old_rows[live]] = -1
                self._host_stats["evictions"] += int(live.sum())
            self._move(t, miss_ids, victims, to_host=False)
            self.slot_of_row[t][miss_ids] = victims.to(torch.int32)
            self.row_of_slot[t][victims] = miss_ids
            score[victims] = self._tick if self.cache_algorithm != "lfu" else 1
        self._prefetched = (indices.data_ptr(), int(indices.numel()))
        self._prefetch_tick = self._tick

    @torch.no_grad()
    def translate(self, indices: torch.Tensor, offsets: torch.Tensor, batch_size: int) -> torch.Tensor:
        """ids -> cache slots (prefetches first unless ``prefetch`` already ran for these very indices)."""
        if self._prefetched != (indices.data_ptr(), int(indices.numel())):
            self.prefetch(indices, offsets, batch_size)
        self._prefetched = None
        F = len(self.feature_table_map)
        if self.device.type == "cuda":
            stream = torch.cuda.current_stream(self.device)
            self._check_overflow()
            self._after_last(stream)  # the prefetch of this batch may have run on the pipeline's prefetch stream
            self._lookup = (self._prefetch_tick, stream)
            self._mark(stream)
        if indices.is_cuda and _lib.use_cuda_kernels(indices) and indices.numel() > 0:
            # one launch, no host read: per-feature start positions gathered on the device, direct maps addressed through a pointer table
            tab = self.__dict__.get("_translate_tab")
            if tab is None or tab[2] != indices.device:
                ptrs = torch.tensor([self.slot_of_row[t].data_ptr() for t in self.feature_table_map], dtype=torch.int64, device=indices.device)
                rows = torch.tensor([self.embedding_specs[t][0] for t in self.feature_table_map], dtype=torch.int64, device=indices.device)
                pick = torch.arange(0, F + 1, device=indices.device) * 1
                tab = (ptrs, rows, indices.device, pick)
                self.__dict__["_translate_tab"] = tab
            bounds_dev = offsets[tab[3] * batch_size].to(torch.int64)
            idx = indices.contiguous()
            out = torch.empty_like(idx)
            code = _lib.lib().trb_cache_translate(_lib.ptr(idx), int(idx.dtype == torch.int64), _lib.ptr(bounds_dev), F, _lib.ptr(tab[0]), _lib.ptr(tab[1]), _lib.ptr(out),
                                                  ctypes.c_int64(idx.numel()), _lib.stream_ptr(idx.device))
            _lib.check(code, "trb_cache_translate")
            return out
        bounds = offsets[torch.arange(0, F + 1, device=offsets.device) * batch_size].tolist()
        out = indices.clone()
        for f, t in enumerate(self.feature_table_map):
            lo, hi = int(bounds[f]), int(bounds[f + 1])
            if hi > lo:
                ids = indices[lo:hi].long()
                ok = (ids >= 0) & (ids < self.embedding_specs[t][0])
                sl = self.slot_of_row[t][ids.clamp(0, self.embedding_specs[t][0] - 1)].to(indices.dtype)
                out[lo:hi] = torch.where(ok, sl, torch.full_like(sl, -1))
        return out

    def forward(self, indices: torch.Tensor, offsets: torch.Tensor, per_sample_weights: Optional[torch.Tensor] = None, batch_size: Optional[int] = None) -> torch.Tensor:
        F = len(self.feature_table_map)
        B = batch_size if batch_size is not None else (offsets.numel() - 1) // max(F, 1)
        return self.cache(self.translate(indices, offsets, B), offsets, per_sample_weights, batch_size=B)

    # ---- flush / views -----------------------------------------------------------------------------------------------------------
    @torch.no_grad()
    def flush(self, invalidate: bool = False) -> None:
        """Write every cached row (+ state) back to the host tables (before state_dict / checkpoint)."""
        if self.device.type == "cuda":
            self._after_last(torch.cuda.current_stream(self.device))
            self._check_overflow(wait=True)
        for t in range(len(self.embedding_specs)):
            slots = (self.row_of_slot[t] >= 0).nonzero(as_tuple=True)[0]
            if slots.numel():
                self._move(t, self.row_of_slot[t][slots], slots, to_host=True)
            if invalidate:
                self.slot_of_row[t].fill_(-1)
                self.row_of_slot[t].fill_(-1)
                self.score[t].zero_()
        if invalidate:
            self._stamp.zero_()
        if self.device.type == "cuda":
            torch.cuda.current_stream(self.device).synchronize()

    def split_embedding_weights(self, flush: bool = True) -> List[torch.Tensor]:
        if flush:
            self.flush()
        out, o = [], 0
        for r, d in self.embedding_specs:
            out.append(self.host_weights[o : o + r * d].view(r, d))
            o += r * d
        return out

    def split_optimizer_states(self) -> List[Dict[str, torch.Tensor]]:
        self.flush()
        names = _OPT_STATE_NAMES.get(self.cache.opt_code, (None, None))
        res: List[Dict[str, torch.Tensor]] = []
        eo = ro = 0
        for r, d in self.embedding_specs:
            st: Dict[str, torch.Tensor] = {}
            for buf, kind, name in ((self.host_state1, self._kinds[0], names[0]), (self.host_state2, self._kinds[1], names[1])):
                if buf is None or name is None:
                    continue
                st[name] = buf[ro : ro + r] if kind == "row" else buf[eo : eo + r * d].view(r, d)
            res.append(st)
            eo += r * d
            ro += r
        return res

    def load_rows_changed(self) -> None:
        """Call after writing into the host tables directly (load_state_dict): drops the now stale cache content."""
        if self.device.type == "cuda":
            self._after_last(torch.cuda.current_stream(self.device))
        for t in range(len(self.embedding_specs)):
            self.slot_of_row[t].fill_(-1)
            self.row_of_slot[t].fill_(-1)
            self.score[t].zero_()
        self._stamp.zero_()


# ---- unified-memory tensor helpers (fbgemm ``new_unified_tensor`` / ``is_uvm_tensor``, SURVEY 2.4b) ----------------------------
_UVM_TENSORS: "weakref.WeakValueDictionary[int, torch.Tensor]" = None  # type: ignore[assignment]


def new_unified_tensor(like: torch.Tensor, sizes: Sequence[int], is_host_mapped: bool = True) -> torch.Tensor:
    """A tensor of ``like``'s dtype that both the host and the GPU of ``like`` can address: pinned host memory mapped into the
    device address space (zero-copy, what ``EmbeddingLocation.MANAGED`` tables use). On a CPU-only box it is plain host memory."""
    global _UVM_TENSORS
    import weakref

    if _UVM_TENSORS is None:
        _UVM_TENSORS = weakref.WeakValueDictionary()
    t = torch.empty(tuple(sizes), dtype=like.dtype, device="cpu", pin_memory=torch.cuda.is_available())
    _UVM_TENSORS[t.data_ptr()] = t
    return t


def is_uvm_tensor(t: torch.Tensor) -> bool:
    """True for tensors made by :func:`new_unified_tensor` (or views sharing their base pointer)."""
    return _UVM_TENSORS is not None and t.device.type == "cpu" and t.data_ptr() in _UVM_TENSORS
