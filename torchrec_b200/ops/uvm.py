"""Software-managed HBM cache over host-resident embedding tables (compute kernel FUSED_UVM_CACHING).

Parity: fbgemm's UVM + LRU/LFU cache inside SplitTableBatchedEmbeddingBagsCodegen (``prefetch`` / ``flush`` /
``cache_load_factor``; reference call sites distributed/embedding_lookup.py:714-767, batched_embedding_kernel.py).

Design (GPU-first, not a port of the 32-way set-associative lxu cache): the table-batched kernels ALWAYS run on a
device-resident cache table and see *slot* ids; a direct map ``slot_of_row`` (int32 per row, in HBM: 4 B/row) translates
ids -> slots, so the cache is fully associative and there are no conflict misses. ``prefetch`` (on a side stream, one
batch ahead) makes every id of the batch resident: victims are the least-recently / least-frequently used slots, their
rows AND optimizer state go back to pinned host memory and the missing rows come in — both through one zero-copy row
mover kernel (``trb_row_copy``). Forward and the fused backward+optimizer then touch HBM only."""
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
        # id <-> slot maps (HBM), recency / frequency per slot
        self.slot_of_row = [torch.full((r,), -1, dtype=torch.int32, device=self.device) for r, _ in self.embedding_specs]
        self.row_of_slot = [torch.full((c,), -1, dtype=torch.int64, device=self.device) for c in self.cache_rows]
        self.score = [torch.zeros(c, dtype=torch.int64, device=self.device) for c in self.cache_rows]
        self._tick = 0
        self._prefetched: Optional[Tuple[int, int]] = None
        self.stats = {"hits": 0, "misses": 0, "evictions": 0}
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

    # ---- prefetch: make every id of the batch resident --------------------------------------------------------------------------
    @torch.no_grad()
    def prefetch(self, indices: torch.Tensor, offsets: torch.Tensor, batch_size: Optional[int] = None) -> None:
        F = len(self.feature_table_map)
        B = batch_size if batch_size is not None else (offsets.numel() - 1) // max(F, 1)
        self._tick += 1
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
            self.stats["hits"] += int(hit.sum())
            self.stats["misses"] += n_miss
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
                self.stats["evictions"] += int(live.sum())
            self._move(t, miss_ids, victims, to_host=False)
            self.slot_of_row[t][miss_ids] = victims.to(torch.int32)
            self.row_of_slot[t][victims] = miss_ids
            score[victims] = self._tick if self.cache_algorithm != "lfu" else 1
        self._prefetched = (indices.data_ptr(), int(indices.numel()))

    @torch.no_grad()
    def translate(self, indices: torch.Tensor, offsets: torch.Tensor, batch_size: int) -> torch.Tensor:
        """ids -> cache slots (prefetches first unless ``prefetch`` already ran for these very indices)."""
        if self._prefetched != (indices.data_ptr(), int(indices.numel())):
            self.prefetch(indices, offsets, batch_size)
        self._prefetched = None
        F = len(self.feature_table_map)
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
        for t in range(len(self.embedding_specs)):
            slots = (self.row_of_slot[t] >= 0).nonzero(as_tuple=True)[0]
            if slots.numel():
                self._move(t, self.row_of_slot[t][slots], slots, to_host=True)
            if invalidate:
                self.slot_of_row[t].fill_(-1)
                self.row_of_slot[t].fill_(-1)
                self.score[t].zero_()
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
        for t in range(len(self.embedding_specs)):
            self.slot_of_row[t].fill_(-1)
            self.row_of_slot[t].fill_(-1)
            self.score[t].zero_()


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
