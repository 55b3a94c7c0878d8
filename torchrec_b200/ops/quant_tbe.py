"""Inference table-batched embedding over quantized rows (``csrc/tbe_quant.cu``).

Replaces fbgemm ``IntNBitTableBatchedEmbeddingBagsCodegen`` (reference quant/embedding_modules.py:425-442).
Row formats: FP32, FP16, BF16, INT8 / INT4 / INT2 (row-wise, fused fp16 scale+bias tail) and
block-scaled FP8 (e4m3 + one fp16 scale per 32 elements).

Tables are placed per table (``locations``): ``DEVICE`` rows live in HBM; ``MANAGED`` rows live in pinned host memory and are read
zero-copy by the lookup kernel; ``MANAGED_CACHING`` rows live in pinned host memory behind an HBM row cache of
``cache_load_factor * rows`` slots. A cache miss is served from host memory by the same kernel, so results never depend on what the
cache holds; the missed rows are admitted afterwards on a side stream (``trb_qcache_admit``)."""
from __future__ import annotations

import ctypes
import math
from typing import Dict, List, Optional, Sequence, Tuple, Union

import torch
import torch.nn as nn

from ..types import DataType
from . import _lib
from . import jagged as J
from .tbe import EmbeddingLocation

FMT = {DataType.FP32: 0, DataType.FP16: 1, DataType.BF16: 2, DataType.INT8: 3, DataType.INT4: 4, DataType.INT2: 5, DataType.FP8: 6}
_BITS = {DataType.INT8: 8, DataType.INT4: 4, DataType.INT2: 2}
FP8_BLOCK = 32


def row_bytes(dim: int, data_type: DataType, row_alignment: int = 16) -> int:
    if data_type == DataType.FP32:
        n = dim * 4
    elif data_type in (DataType.FP16, DataType.BF16):
        n = dim * 2
    elif data_type in _BITS:
        n = (dim * _BITS[data_type] + 7) // 8 + 4
    elif data_type == DataType.FP8:
        n = dim + (dim // FP8_BLOCK) * 2
    else:
        raise ValueError(data_type)
    return (n + row_alignment - 1) // row_alignment * row_alignment


def quantize_rows(weight: torch.Tensor, data_type: DataType, row_alignment: int = 16) -> torch.Tensor:
    """fp32 [rows, dim] -> uint8 [rows, row_bytes] in the kernel's row format."""
    rows, dim = weight.shape
    rb = row_bytes(dim, data_type, row_alignment)
    out = torch.zeros(rows, rb, dtype=torch.uint8, device=weight.device)
    w = weight.float()
    if data_type == DataType.FP32:
        out[:, : dim * 4] = w.contiguous().view(torch.uint8).view(rows, dim * 4)
    elif data_type == DataType.FP16:
        out[:, : dim * 2] = w.half().contiguous().view(torch.uint8).view(rows, dim * 2)
    elif data_type == DataType.BF16:
        out[:, : dim * 2] = w.bfloat16().contiguous().view(torch.uint8).view(rows, dim * 2)
    elif data_type in _BITS:
        q = J.fused_nbit_rowwise_quantize(w, _BITS[data_type])
        out[:, : q.shape[1]] = q
    elif data_type == DataType.FP8:
        assert dim % FP8_BLOCK == 0, f"block-scaled fp8 needs dim % {FP8_BLOCK} == 0"
        blocks = w.view(rows, dim // FP8_BLOCK, FP8_BLOCK)
        amax = blocks.abs().amax(dim=2, keepdim=True).clamp(min=1e-12)
        scale = (amax / 448.0).half().float().clamp(min=6e-8)
        q = (blocks / scale).to(torch.float8_e4m3fn).view(torch.uint8).view(rows, dim)
        out[:, :dim] = q
        out[:, dim : dim + (dim // FP8_BLOCK) * 2] = scale.half().contiguous().view(torch.uint8).view(rows, (dim // FP8_BLOCK) * 2)
    else:
        raise ValueError(data_type)
    return out


def dequantize_rows(q: torch.Tensor, dim: int, data_type: DataType) -> torch.Tensor:
    rows = q.shape[0]
    if data_type == DataType.FP32:
        return q[:, : dim * 4].contiguous().view(torch.float32).view(rows, dim)
    if data_type == DataType.FP16:
        return q[:, : dim * 2].contiguous().view(torch.float16).view(rows, dim).float()
    if data_type == DataType.BF16:
        return q[:, : dim * 2].contiguous().view(torch.bfloat16).view(rows, dim).float()
    if data_type in _BITS:
        return J.fused_nbit_rowwise_dequantize(q, _BITS[data_type], dim)
    if data_type == DataType.FP8:
        vals = q[:, :dim].contiguous().view(torch.float8_e4m3fn).float().view(rows, dim // FP8_BLOCK, FP8_BLOCK)
        scale = q[:, dim : dim + (dim // FP8_BLOCK) * 2].contiguous().view(torch.float16).float().view(rows, dim // FP8_BLOCK, 1)
        return (vals * scale).view(rows, dim)
    raise ValueError(data_type)


def host_zeros(nbytes: int) -> torch.Tensor:
    """Zeroed uint8 host tensor of exactly ``nbytes`` bytes, pinned (and device-addressable through UVA) when CUDA is available.
    PyTorch's caching pinned allocator would round the allocation up to a power of two."""
    if nbytes == 0 or not torch.cuda.is_available():
        return torch.zeros(nbytes, dtype=torch.uint8)
    p = ctypes.c_void_p()
    _lib.check(_lib.lib().trb_host_alloc(ctypes.c_int64(nbytes), ctypes.byref(p)), "trb_host_alloc")

    class _PinnedHostBuffer(ctypes.c_uint8 * nbytes):
        """The allocation as a buffer object: ``torch.frombuffer`` holds it while any tensor uses the memory, and the memory is freed
        with the last such tensor."""

        def __del__(self) -> None:
            _lib.lib().trb_host_free(ctypes.c_void_p(ctypes.addressof(self)))

    return torch.frombuffer(_PinnedHostBuffer.from_address(p.value), dtype=torch.uint8)


_PLACEMENTS = (EmbeddingLocation.DEVICE, EmbeddingLocation.MANAGED, EmbeddingLocation.MANAGED_CACHING)
# device-side per-table cache state: the buffers of cached table c are named f"_qc{c}_{name}"
_QC_BUFFERS = ("cache", "slot_of_row", "row_of_slot", "ref", "miss", "victim", "ctr", "state")


class QuantTableBatchedEmbeddingBags(nn.Module):
    """Inference TBE: ``embedding_specs`` = [(name, rows, dim, DataType)]; HBM tables live in one uint8 buffer (``weights``).

    ``locations`` (per table, default all ``EmbeddingLocation.DEVICE``) puts tables in pinned host memory (``MANAGED``) or in pinned
    host memory behind an HBM row cache (``MANAGED_CACHING``, ``cache_load_factor`` of the rows, per table or one value for all). At
    most ``max_admissions_per_call`` missed rows per cached table are admitted after each lookup; the others are admitted by later calls."""

    def __init__(self, embedding_specs: Sequence[Tuple[str, int, int, DataType]], feature_table_map: Optional[Sequence[int]] = None,
                 pooling_mode: int = 0, output_dtype: torch.dtype = torch.float32, device: Optional[torch.device] = None, row_alignment: int = 16,
                 locations: Optional[Sequence[EmbeddingLocation]] = None, cache_load_factor: Union[float, Sequence[float]] = 0.2,
                 max_admissions_per_call: int = 8192) -> None:
        super().__init__()
        device = torch.device(device) if device is not None else torch.device("cpu")
        self.embedding_specs = list(embedding_specs)
        self.feature_table_map = list(feature_table_map) if feature_table_map is not None else list(range(len(self.embedding_specs)))
        self.pooling_mode = pooling_mode  # 0 sum, 1 mean, 2 none
        self.output_dtype = output_dtype
        self.row_alignment = row_alignment
        self._row_bytes = [row_bytes(d, dt, row_alignment) for _, _, d, dt in self.embedding_specs]
        T = len(self.embedding_specs)
        self.locations = [EmbeddingLocation(int(l)) for l in locations] if locations is not None else [EmbeddingLocation.DEVICE] * T
        if len(self.locations) != T or any(l not in _PLACEMENTS for l in self.locations):
            raise ValueError(f"locations: one of DEVICE / MANAGED / MANAGED_CACHING per table, got {self.locations}")
        clf = list(cache_load_factor) if isinstance(cache_load_factor, (list, tuple)) else [float(cache_load_factor)] * T
        self.cache_load_factor = [float(x) for x in clf]
        self._placed = any(l != EmbeddingLocation.DEVICE for l in self.locations)
        offs, o = [], 0
        for (_, r, _, _), rb, loc in zip(self.embedding_specs, self._row_bytes, self.locations):
            offs.append(o)
            if loc == EmbeddingLocation.DEVICE:
                o += r * rb
        self._table_off = offs
        self.register_buffer("weights", torch.zeros(o, dtype=torch.uint8, device=device), persistent=False)
        # host tables are plain attributes, not buffers: .to() / .cuda() leave them in host memory
        self._host_tables: List[Optional[torch.Tensor]] = [
            host_zeros(r * rb).view(r, rb) if loc != EmbeddingLocation.DEVICE and device.type != "meta" else None
            for (_, r, _, _), rb, loc in zip(self.embedding_specs, self._row_bytes, self.locations)]
        fm = self.feature_table_map
        mk64 = lambda x: torch.tensor(x, dtype=torch.int64, device=device)
        mk32 = lambda x: torch.tensor(x, dtype=torch.int32, device=device)
        self._h_dim = [self.embedding_specs[t][2] for t in fm]
        cols, c = [], 0
        for d in self._h_dim:
            cols.append(c)
            c += d
        self._h_col, self.total_cols = cols, c
        if device.type != "meta":
            self.register_buffer("feat_woff", mk64([offs[t] for t in fm]), persistent=False)
            self.register_buffer("feat_rows", mk64([self.embedding_specs[t][1] for t in fm]), persistent=False)
            self.register_buffer("feat_dim", mk32(self._h_dim), persistent=False)
            self.register_buffer("feat_col", mk32(cols), persistent=False)
            self.register_buffer("feat_fmt", mk32([FMT[self.embedding_specs[t][3]] for t in fm]), persistent=False)
            self.register_buffer("feat_rb", mk32([self._row_bytes[t] for t in fm]), persistent=False)
        self.max_dim = max(self._h_dim) if self._h_dim else 0
        fmts = {FMT[dt] for _, _, _, dt in self.embedding_specs}
        # one row format for the whole launch + rows made of whole 16-byte vectors -> the vector kernel (tbe_quant.cu: qtbe_fwd_vec_kernel);
        # elements per vector: 16 for the 8-bit formats, 8 for fp16 / bf16, 32 for int4
        epv = {FMT[DataType.INT8]: 16, FMT[DataType.FP8]: 16, FMT[DataType.FP16]: 8, FMT[DataType.BF16]: 8, FMT[DataType.INT4]: 32}
        one = next(iter(fmts)) if len(fmts) == 1 else -1
        aligned = one in epv and all(d % epv[one] == 0 for d in self._h_dim) and all(rb % 16 == 0 for rb in self._row_bytes)
        self._uniform_fmt = one if aligned else -1
        if self._placed:
            self._init_placement(device, max_admissions_per_call)

    # ---- placement ----------------------------------------------------------------------------------------------------------------------
    def _init_placement(self, device: torch.device, max_admissions_per_call: int) -> None:
        self._cached = [t for t, l in enumerate(self.locations) if l == EmbeddingLocation.MANAGED_CACHING]
        self.cache_slots: Dict[int, int] = {}
        self._adm_event: Optional[torch.cuda.Event] = None
        self._side_stream: Optional[torch.cuda.Stream] = None
        self._cap_max = 0
        if device.type == "meta":
            return
        ctab = {t: c for c, t in enumerate(self._cached)}
        self.register_buffer("feat_ctab", torch.tensor([ctab.get(t, -1) for t in self.feature_table_map], dtype=torch.int32, device=device),
                             persistent=False)
        self.register_buffer("no_slot", torch.full((1,), -1, dtype=torch.int32, device=device), persistent=False)
        for c, t in enumerate(self._cached):
            _, rows, _, _ = self.embedding_specs[t]
            rb = self._row_bytes[t]
            if rb % 16:
                raise ValueError(f"table {self.embedding_specs[t][0]}: cached rows are copied in 16-byte vectors, row_alignment must make rows a "
                                 f"multiple of 16 bytes (got {rb})")
            slots = max(1, min(rows, int(math.ceil(rows * self.cache_load_factor[t]))))
            cap = min(slots, max_admissions_per_call)
            self.cache_slots[t] = slots
            self._cap_max = max(self._cap_max, cap)
            bufs = {
                "cache": torch.zeros(slots, rb, dtype=torch.uint8, device=device),
                "slot_of_row": torch.full((rows,), -1, dtype=torch.int32, device=device),
                "row_of_slot": torch.full((slots,), -1, dtype=torch.int64, device=device),
                "ref": torch.zeros(slots, dtype=torch.uint8, device=device),
                "miss": torch.zeros(cap, dtype=torch.int64, device=device),
                "victim": torch.zeros(cap, dtype=torch.int64, device=device),
                "ctr": torch.zeros(2, dtype=torch.int32, device=device),
                "state": torch.zeros(5, dtype=torch.int64, device=device),  # CLOCK hand, lookups, hits, admissions, evictions
            }
            for k in _QC_BUFFERS:
                self.register_buffer(f"_qc{c}_{k}", bufs[k], persistent=False)
        self._refresh_placement()

    def _qc(self, c: int, name: str) -> torch.Tensor:
        return getattr(self, f"_qc{c}_{name}")

    def _refresh_placement(self) -> None:
        """Absolute row bases and cache descriptors (they hold addresses, so they are rebuilt whenever the buffers move)."""
        dev = self.weights.device
        base = [self._host_tables[t].data_ptr() if l != EmbeddingLocation.DEVICE else self.weights.data_ptr() + self._table_off[t]
                for t, l in enumerate(self.locations)]
        self.feat_base = torch.tensor([base[t] for t in self.feature_table_map], dtype=torch.int64, device=dev)
        words = []
        for c, t in enumerate(self._cached):  # field order of QCacheTab (csrc/tbe_quant.cu)
            q = lambda k: self._qc(c, k).data_ptr()
            st = q("state")
            words.append([q("slot_of_row"), q("row_of_slot"), q("ref"), q("cache"), self._host_tables[t].data_ptr(), q("miss"), q("victim"),
                          q("ctr"), st, st + 8, self.cache_slots[t], self._qc(c, "miss").numel(), self._row_bytes[t]])
        self.cache_tabs = torch.tensor(words, dtype=torch.int64, device=dev) if words else None

    def _apply(self, fn, recurse: bool = True):
        super()._apply(fn, recurse)
        if self._placed and hasattr(self, "feat_ctab"):
            self._refresh_placement()
        return self

    def _wait_admission(self) -> None:
        """Order the current stream after the last admission (the next lookup, a cache reset and a weight write need it)."""
        ev = self._adm_event
        self._adm_event = None
        if ev is not None and not torch.cuda.is_current_stream_capturing():
            # (a graph capture starts after a device synchronize, so a capture never has to wait for an eager admission)
            torch.cuda.current_stream(self.weights.device).wait_event(ev)

    def _admit(self) -> None:
        """Admit the rows the lookup just missed. Eagerly it runs on a side stream, so the pooled output is not held up; inside a CUDA
        graph capture it runs on the capturing stream and becomes part of the graph."""
        L = _lib.lib()
        dev = self.weights.device
        args = (_lib.ptr(self.cache_tabs), len(self._cached), ctypes.c_int64(self._cap_max))
        if torch.cuda.is_current_stream_capturing():
            _lib.check(L.trb_qcache_admit(*args, _lib.stream_ptr(dev)), "trb_qcache_admit")
            return
        main = torch.cuda.current_stream(dev)
        if self._side_stream is None:
            self._side_stream = torch.cuda.Stream(device=dev)
        side = self._side_stream
        side.wait_stream(main)
        with torch.cuda.stream(side):
            _lib.check(L.trb_qcache_admit(*args, ctypes.c_void_p(side.cuda_stream)), "trb_qcache_admit")
        ev = torch.cuda.Event()
        ev.record(side)
        self._adm_event = ev

    @torch.no_grad()
    def invalidate_cache(self, table_idx: Optional[int] = None) -> None:
        """Empty the HBM row cache of one table (or of every cached table); every write to a cached table's rows must call this."""
        if not self._placed or not hasattr(self, "feat_ctab"):
            return
        if self.weights.is_cuda:
            self._wait_admission()
        for c, t in enumerate(self._cached):
            if table_idx is not None and t != table_idx:
                continue
            self._qc(c, "slot_of_row").fill_(-1)
            self._qc(c, "row_of_slot").fill_(-1)
            self._qc(c, "ref").zero_()
            self._qc(c, "ctr").zero_()
            self._qc(c, "state")[0].zero_()

    def cache_stats(self) -> Dict[str, Dict[str, int]]:
        """Per cached table: lookups, hits, misses, admissions, evictions since construction. Synchronizes with the device."""
        out: Dict[str, Dict[str, int]] = {}
        if not self._placed or not self._cached:
            return out
        if self._adm_event is not None:
            self._adm_event.synchronize()
        for c, t in enumerate(self._cached):
            _, lookups, hits, adm, ev = (int(x) for x in self._qc(c, "state").tolist())
            out[self.embedding_specs[t][0]] = {"lookups": lookups, "hits": hits, "misses": lookups - hits, "admissions": adm, "evictions": ev,
                                               "slots": self.cache_slots[t]}
        return out

    def split_embedding_weights(self) -> List[torch.Tensor]:
        """Per table uint8 [rows, row_bytes] views (host tables: the pinned host tensor itself). A write through a view of a cached
        table must be followed by ``invalidate_cache``."""
        if self._placed:
            return [self.weights[o : o + r * rb].view(r, rb) if h is None else h
                    for (_, r, _, _), rb, o, h in zip(self.embedding_specs, self._row_bytes, self._table_off, self._host_tables)]
        return [self.weights[o : o + r * rb].view(r, rb) for (_, r, _, _), rb, o in zip(self.embedding_specs, self._row_bytes, self._table_off)]

    @torch.no_grad()
    def assign_from_float(self, table_idx: int, weight: torch.Tensor) -> None:
        name, rows, dim, dt = self.embedding_specs[table_idx]
        dst = self.split_embedding_weights()[table_idx]
        if self._placed:
            self.invalidate_cache(table_idx)
        dst.copy_(quantize_rows(weight.to(self.weights.device), dt, self.row_alignment))

    def dequantized_table(self, table_idx: int) -> torch.Tensor:
        _, _, dim, dt = self.embedding_specs[table_idx]
        return dequantize_rows(self.split_embedding_weights()[table_idx], dim, dt)

    def forward(self, indices: torch.Tensor, offsets: torch.Tensor, per_sample_weights: Optional[torch.Tensor] = None, batch_size: Optional[int] = None) -> torch.Tensor:
        F = len(self.feature_table_map)
        B = batch_size if batch_size is not None else (offsets.numel() - 1) // max(F, 1)
        pooled = self.pooling_mode != 2
        if not _lib.use_cuda_kernels(self.weights):
            return self._ref_forward(indices, offsets, per_sample_weights, B, pooled)
        n = indices.numel()
        if pooled:
            out = torch.empty(B, self.total_cols, dtype=self.output_dtype, device=self.weights.device)
            stride = self.total_cols
        else:
            D = self._h_dim[0]
            out = torch.empty(n, D, dtype=self.output_dtype, device=self.weights.device)
            stride = D
        L = _lib.lib()
        if self._placed:
            self._wait_admission()
            code = L.trb_qtbe_fwd_placed(_lib.ptr(self.feat_base), _lib.ptr(self.feat_ctab), _lib.ptr(self.cache_tabs), _lib.ptr(self.no_slot),
                                         _lib.ptr(self.feat_rows), _lib.ptr(self.feat_dim), _lib.ptr(self.feat_col), _lib.ptr(self.feat_fmt),
                                         _lib.ptr(self.feat_rb), _lib.ptr(indices), 1 if indices.dtype == torch.int64 else 0, _lib.ptr(offsets),
                                         1 if offsets.dtype == torch.int64 else 0, _lib.ptr(per_sample_weights), _lib.ptr(out),
                                         _lib.dtype_code(self.output_dtype), ctypes.c_int64(stride), B, F, self.max_dim, int(self.pooling_mode == 1),
                                         int(pooled), ctypes.c_int64(n), int(self._uniform_fmt), _lib.stream_ptr(self.weights.device))
            _lib.check(code, "trb_qtbe_fwd_placed")
            if self._cached:
                self._admit()
            return out
        code = L.trb_qtbe_fwd_ex(_lib.ptr(self.weights), _lib.ptr(self.feat_woff), _lib.ptr(self.feat_rows), _lib.ptr(self.feat_dim), _lib.ptr(self.feat_col),
                              _lib.ptr(self.feat_fmt), _lib.ptr(self.feat_rb), _lib.ptr(indices), 1 if indices.dtype == torch.int64 else 0,
                              _lib.ptr(offsets), 1 if offsets.dtype == torch.int64 else 0, _lib.ptr(per_sample_weights), _lib.ptr(out),
                              _lib.dtype_code(self.output_dtype), ctypes.c_int64(stride), B, F, self.max_dim, int(self.pooling_mode == 1), int(pooled),
                              ctypes.c_int64(n), int(self._uniform_fmt), _lib.stream_ptr(self.weights.device))
        _lib.check(code, "trb_qtbe_fwd_ex")
        return out

    def forward_scatter(self, indices: torch.Tensor, offsets: torch.Tensor, pos: torch.Tensor, B: int, out: torch.Tensor, feat_obase: torch.Tensor,
                        feat_ostride: torch.Tensor, feat_col: torch.Tensor, bound: int) -> None:
        """Sequence lookup over routed ids (``trb_qtbe_seq_scatter``). ``offsets`` (int32 / int64, ``F * B + 1`` entries, the first need
        not be 0) slice ``indices`` and ``pos`` (int32, the position of each id inside its feature's values). The row of routed id k of
        feature f is stored at ``out + feat_obase[f] + pos[k] * feat_ostride[f] + feat_col[f]`` (int64 / int32 / int32, one entry per
        feature; ``out`` may live on another device with peer access enabled). ``bound`` >= the number of routed ids. Placed tables wait
        for the last admission first and admit the rows this lookup missed afterwards."""
        L = _lib.lib()
        F = len(self.feature_table_map)
        if self._placed:
            self._wait_admission()
            where = [None, None, _lib.ptr(self.feat_base), _lib.ptr(self.feat_ctab), _lib.ptr(self.cache_tabs), _lib.ptr(self.no_slot)]
        else:
            where = [_lib.ptr(self.weights), _lib.ptr(self.feat_woff), None, None, None, None]
        code = L.trb_qtbe_seq_scatter(*where, _lib.ptr(self.feat_rows), _lib.ptr(self.feat_dim), _lib.ptr(feat_col), _lib.ptr(self.feat_fmt),
                                      _lib.ptr(self.feat_rb), _lib.ptr(feat_obase), _lib.ptr(feat_ostride), _lib.ptr(indices),
                                      int(indices.dtype == torch.int64), _lib.ptr(offsets), int(offsets.dtype == torch.int64), _lib.ptr(pos), _lib.ptr(out),
                                      _lib.dtype_code(self.output_dtype), B, F, ctypes.c_int64(bound), int(self._uniform_fmt),
                                      _lib.stream_ptr(self.weights.device))
        _lib.check(code, "trb_qtbe_seq_scatter")
        if self._placed and self._cached:
            self._admit()

    def _ref_forward(self, indices, offsets, psw, B: int, pooled: bool) -> torch.Tensor:
        offsets = offsets.long()
        indices = indices.long()
        F = len(self.feature_table_map)
        if not pooled:
            D = self._h_dim[0]
            out = torch.zeros(indices.numel(), D, dtype=torch.float32, device=indices.device)
        else:
            out = torch.zeros(B, self.total_cols, dtype=torch.float32, device=indices.device)
        tables = {t: self.dequantized_table(t) for t in set(self.feature_table_map)}
        for f, t in enumerate(self.feature_table_map):
            tab = tables[t]
            off = offsets[f * B : (f + 1) * B + 1]
            lo, hi = int(off[0]), int(off[-1])
            idx = indices[lo:hi]
            valid = (idx >= 0) & (idx < tab.shape[0])
            vals = tab[torch.where(valid, idx, torch.zeros_like(idx))] * valid.unsqueeze(1)
            if not pooled:
                out[lo:hi] = vals
                continue
            if psw is not None:
                vals = vals * psw[lo:hi].float().unsqueeze(1)
            lengths = off[1:] - off[:-1]
            seg = torch.repeat_interleave(torch.arange(B, device=indices.device), lengths)
            pooled_v = torch.zeros(B, tab.shape[1], device=indices.device).index_add_(0, seg, vals)
            if self.pooling_mode == 1:
                pooled_v = pooled_v / lengths.clamp(min=1).unsqueeze(1)
            out[:, self._h_col[f] : self._h_col[f] + tab.shape[1]] = pooled_v
        return out.to(self.output_dtype)
