"""Key-value ("virtual") embedding tables: rows addressed by arbitrary 64-bit keys, materialised on first touch, stored in DRAM or on
SSD behind the HBM row cache (compute kernels KEY_VALUE / DRAM_VIRTUAL_TABLE / SSD_VIRTUAL_TABLE).

Parity: the reference's ``KeyValueEmbedding(Bag)`` / ``ZeroCollisionKeyValueEmbedding(Bag)`` over fbgemm's ``SSDTableBatchedEmbeddingBags``
(RocksDB / DRAM KV backends, L1 HBM cache + L2 cache; reference distributed/batched_embedding_kernel.py:1917-2508, 3127-3700).

Three tiers, each with the mechanism that fits it on an H100 node:

    HBM   the row cache of ``UvmCachedEmbeddingBags``: the table-batched lookup / fused optimizer kernels only ever touch cache slots
    store ``store_rows`` row slots per table holding weights + optimizer state,
            backend "dram"  pinned host memory: rows move with the zero-copy row-mover kernel (PCIe reads / writes issued by the GPU)
            backend "ssd"   one memory-mapped file per state tensor under ``ssd_storage_directory``: rows move through a pinned staging
                            buffer (host gather from the page cache / SSD, then one H2D copy); survives the process (reopen = resume)
    keys  native id map (``csrc/dynemb``: partitioned open-addressing hash map with LRU / LFU / mixed eviction records): key -> store
          slot; a key seen for the first time gets a slot and a deterministic fresh row (uniform init seeded by the key, zero state);
          when the store is full the coldest keys are evicted (their rows are forgotten, like the reference's TTL / count eviction).

The table size the user declares (``num_embeddings``) is only the width of the key space: memory is ``store_rows`` rows.
"""
from __future__ import annotations

import math
import os
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from .uvm import UvmCachedEmbeddingBags, row_copy


def _s64(x: int) -> int:
    """A 64-bit constant as the signed integer with the same bit pattern (int64 tensor arithmetic wraps modulo 2^64)."""
    return x - (1 << 64) if x >= (1 << 63) else x


class KeyValueEmbeddingBags(UvmCachedEmbeddingBags):
    is_cached = True
    is_key_value = True

    def __init__(self, embedding_specs: Sequence[Tuple[int, int]], feature_table_map: Optional[Sequence[int]] = None, store_rows: Optional[Sequence[int]] = None,
                 backend: str = "dram", ssd_storage_directory: Optional[str] = None, cache_load_factor: float = 0.2, eviction: str = "mixed_lru_lfu",
                 device: Optional[torch.device] = None, init_seed: int = 0, **tbe_kwargs) -> None:
        from ..dynamic_embedding.id_transformer import IDTransformer

        self.key_space = [int(r) for r, _ in embedding_specs]
        dims = [int(d) for _, d in embedding_specs]
        if store_rows is None:  # default: a store as large as the declared table, capped so that an "infinite" key space stays finite
            store_rows = [min(r, 1 << 24) for r in self.key_space]
        self.store_rows = [int(s) for s in store_rows]
        self.backend = backend
        self._ssd_dir = ssd_storage_directory
        self._init_seed = int(init_seed)
        # the parent manages (store slot <-> HBM slot); we feed it store slots instead of raw ids
        super().__init__([(s, d) for s, d in zip(self.store_rows, dims)], feature_table_map, cache_load_factor=cache_load_factor, device=device, **tbe_kwargs)
        self.id_maps = [IDTransformer(s, eviction_config={"type": eviction}) for s in self.store_rows]
        self.kv_stats = {"inserted": 0, "store_evictions": 0}
        if backend == "ssd":
            self._to_ssd()
        elif backend != "dram":
            raise ValueError(f"unknown key-value backend {backend!r} (dram | ssd)")

    # ---- SSD backend ---------------------------------------------------------------------------------------------------------------
    def _to_ssd(self) -> None:
        d = self._ssd_dir or os.path.join(os.environ.get("TMPDIR", "/tmp"), f"trb200_kv_{os.getpid()}_{id(self):x}")
        os.makedirs(d, exist_ok=True)
        self._ssd_dir = d

        def remap(name: str, t: Optional[torch.Tensor]) -> Optional[torch.Tensor]:
            if t is None:
                return None
            path = os.path.join(d, f"{name}.bin")
            fresh = not os.path.exists(path) or os.path.getsize(path) != t.numel() * t.element_size()
            npdt = {torch.float32: np.float32, torch.float16: np.float16}.get(t.dtype)
            if npdt is None:  # bf16 rows: stored as their 16-bit patterns
                mm = np.memmap(path, dtype=np.int16, mode="w+" if fresh else "r+", shape=(t.numel(),))
                out = torch.from_numpy(mm).view(torch.bfloat16)
            else:
                mm = np.memmap(path, dtype=npdt, mode="w+" if fresh else "r+", shape=(t.numel(),))
                out = torch.from_numpy(mm)
            if fresh:
                out.copy_(t)
            self._mmaps.append(mm)
            return out

        self._mmaps: List[np.memmap] = []
        self.host_weights = remap("weights", self.host_weights)
        self.host_state1 = remap("state1", self.host_state1)
        self.host_state2 = remap("state2", self.host_state2)
        self._staging: Dict[int, torch.Tensor] = {}

    def _stage(self, nbytes: int) -> torch.Tensor:
        buf = self._staging.get(0)
        if buf is None or buf.numel() < nbytes:
            buf = self._staging[0] = torch.empty(int(nbytes * 1.5) + 4096, dtype=torch.uint8, pin_memory=self.device.type == "cuda")
        return buf

    def _move(self, t: int, rows: torch.Tensor, slots: torch.Tensor, to_host: bool) -> None:
        if self.backend != "ssd":
            return super()._move(t, rows, slots, to_host)
        n = rows.numel()
        if n == 0:
            return
        he, hr, ce, cr = self._bases(t)
        D = self.embedding_specs[t][1]
        rows_c = rows.to("cpu", torch.int64)
        slots_d = slots.to(self.device, torch.int64)
        triples = [(self.host_weights, he, self.cache.weights, ce, D)]
        for kind, hs, cs in ((self._kinds[0], self.host_state1, self.cache.state1), (self._kinds[1], self.host_state2, self.cache.state2)):
            if kind == "row":
                triples.append((hs, hr, cs, cr, 1))
            elif kind == "elem":
                triples.append((hs, he, cs, ce, D))
        for host, hoff, cache, coff, width in triples:
            hview = host[hoff : hoff + self.store_rows[t] * width].view(self.store_rows[t], width)
            cview = cache[coff : coff + self.cache_rows[t] * width].view(self.cache_rows[t], width)
            if to_host:
                hview[rows_c] = cview[slots_d].to("cpu")            # D2H of the victims, scatter into the mapped file
            else:
                stage = self._stage(n * width * host.element_size()).view(host.dtype)[: n * width].view(n, width)
                torch.index_select(hview, 0, rows_c, out=stage)    # host gather (page cache / SSD reads) into pinned memory
                cview[slots_d] = stage.to(self.device, non_blocking=True)
        if self.device.type == "cuda":
            torch.cuda.current_stream(self.device).synchronize()    # the staging buffer is reused by the next move

    # ---- keys -> store slots ---------------------------------------------------------------------------------------------------------
    @torch.no_grad()
    def _fresh_rows(self, t: int, keys: torch.Tensor, slots: torch.Tensor) -> None:
        """First touch of ``keys``: deterministic uniform init (seeded by the key, so every rank / restart agrees), zero optimizer state."""
        he, hr, _, _ = self._bases(t)
        D = self.embedding_specs[t][1]
        bound = math.sqrt(1.0 / max(self.key_space[t], 1))
        k = keys.to(torch.int64)
        # counter-based generator: splitmix-style hash of (seed, key, column) -> uniform in [-bound, bound)
        col = torch.arange(D, dtype=torch.int64).unsqueeze(0)
        c1, c2, c3 = _s64(0x9E3779B97F4A7C15), _s64(0xBF58476D1CE4E5B9), _s64(0x94D049BB133111EB)
        x = (k.unsqueeze(1) * c1 + col * c2 + (self._init_seed * 0x94D049BB133111EB) % (1 << 62)) & 0x7FFFFFFFFFFFFFFF
        x = ((x ^ (x >> 30)) * c2) & 0x7FFFFFFFFFFFFFFF
        x = ((x ^ (x >> 27)) * c3) & 0x7FFFFFFFFFFFFFFF
        u = ((x ^ (x >> 31)) & 0xFFFFFF).to(torch.float32) / float(1 << 24)
        w = (u * 2.0 - 1.0) * bound
        s = slots.to(torch.int64)
        self.host_weights[he : he + self.store_rows[t] * D].view(self.store_rows[t], D)[s] = w.to(self.host_weights.dtype)
        for kind, hs in ((self._kinds[0], self.host_state1), (self._kinds[1], self.host_state2)):
            if kind == "row":
                hs[hr : hr + self.store_rows[t]][s] = 0
            elif kind == "elem":
                hs[he : he + self.store_rows[t] * D].view(self.store_rows[t], D)[s] = 0

    @torch.no_grad()
    def _keys_to_slots(self, t: int, keys: torch.Tensor) -> torch.Tensor:
        idm = self.id_maps[t]
        k_cpu = keys.detach().to("cpu", torch.int64)
        slots, ok, fetch = idm.transform(k_cpu)
        if not ok:
            # store full: forget the coldest keys (their slots may be cached in HBM: drop those cache entries without write-back), retry
            need = int((slots < 0).sum())
            victims = idm.evict(max(need, 1))
            if victims.numel():
                vs = victims[:, 1].to(self.device, torch.int64)
                hb = self.slot_of_row[t][vs].long()
                live = hb >= 0
                if bool(live.any()):
                    self.row_of_slot[t][hb[live]] = -1
                    self.score[t][hb[live]] = 0
                    self.slot_of_row[t][vs[live]] = -1
                self.kv_stats["store_evictions"] += int(victims.shape[0])
            slots2, ok2, fetch2 = idm.transform(k_cpu)
            if not ok2:
                raise RuntimeError(f"key-value table {t}: one batch needs more distinct keys than the store holds ({self.store_rows[t]} rows); raise store_rows")
            slots, fetch = slots2, torch.cat([fetch, fetch2]) if fetch.numel() else fetch2
        if fetch.numel():
            self._fresh_rows(t, fetch[:, 0], fetch[:, 1])
            self.kv_stats["inserted"] += int(fetch.shape[0])
        return slots.to(keys.device)

    def _translate_keys(self, indices: torch.Tensor, offsets: torch.Tensor, B: int) -> torch.Tensor:
        """Per table: unique keys -> store slots (native hash map), scattered back to the positions of the batch."""
        F = len(self.feature_table_map)
        bounds = offsets[torch.arange(0, F + 1, device=offsets.device) * B].tolist()
        out = indices.clone()
        by_table: Dict[int, List[Tuple[int, int]]] = {}
        for f, t in enumerate(self.feature_table_map):
            lo, hi = int(bounds[f]), int(bounds[f + 1])
            if hi > lo:
                by_table.setdefault(t, []).append((lo, hi))
        for t, spans in by_table.items():
            ids = torch.cat([indices[lo:hi] for lo, hi in spans]).long()
            uniq, inv = torch.unique(ids, return_inverse=True)
            valid = uniq >= 0
            slots_u = torch.full_like(uniq, -1)
            if bool(valid.any()):
                slots_u[valid] = self._keys_to_slots(t, uniq[valid]).to(uniq.dtype)
            mapped = slots_u[inv].to(indices.dtype)
            p = 0
            for lo, hi in spans:
                out[lo:hi] = mapped[p : p + hi - lo]
                p += hi - lo
        return out

    # ---- TBE surface -----------------------------------------------------------------------------------------------------------------
    @torch.no_grad()
    def prefetch(self, indices: torch.Tensor, offsets: torch.Tensor, batch_size: Optional[int] = None) -> None:
        F = len(self.feature_table_map)
        B = batch_size if batch_size is not None else (offsets.numel() - 1) // max(F, 1)
        slots = self._translate_keys(indices, offsets, B)
        self._kv_cached = (indices.data_ptr(), int(indices.numel()), slots)
        UvmCachedEmbeddingBags.prefetch(self, slots, offsets, B)

    @torch.no_grad()
    def translate(self, indices: torch.Tensor, offsets: torch.Tensor, batch_size: int) -> torch.Tensor:
        kc = self.__dict__.get("_kv_cached")
        if kc is not None and kc[0] == indices.data_ptr() and kc[1] == int(indices.numel()):
            slots = kc[2]
        else:
            slots = self._translate_keys(indices, offsets, batch_size)
        self._kv_cached = None
        # the parent's cache logic works on store slots; its own `prefetch` must be used here (ours expects keys)
        if self._prefetched != (slots.data_ptr(), int(slots.numel())):
            UvmCachedEmbeddingBags.prefetch(self, slots, offsets, batch_size)
        return UvmCachedEmbeddingBags.translate(self, slots, offsets, batch_size)

    # ---- checkpoint view ---------------------------------------------------------------------------------------------------------------
    def key_value_snapshot(self, t: int) -> Tuple[torch.Tensor, torch.Tensor]:
        """(keys [n], rows [n, D]) of every key the table currently stores (cache flushed first): the sparse checkpoint of a virtual table."""
        self.flush()
        triples = self.id_maps[t].save()
        keys, slots = triples[:, 0], triples[:, 1]
        he, _, _, _ = self._bases(t)
        D = self.embedding_specs[t][1]
        rows = self.host_weights[he : he + self.store_rows[t] * D].view(self.store_rows[t], D)[slots]
        return keys, rows.clone()

    def close(self) -> None:
        """Flush the HBM cache and the mapped files (SSD backend)."""
        self.flush()
        for mm in getattr(self, "_mmaps", []):
            mm.flush()
