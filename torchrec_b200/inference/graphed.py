"""Serve predictions from captured CUDA graphs.

A serving batch is small and the device side of a prediction is cheap, so an eager predict call is bound by its host time: KJT
construction, the lookup's ctypes launches, every dense layer, the interaction and the over arch issued one by one. ``GraphedPredictor``
captures ingest + predict once per bucket ``(B_cap, nnz_cap)`` and replays the smallest bucket that holds each batch:

* ``ops/csrc/serve_ingest.cu`` turns the device copy of the server's batch slab into the bucket's static inputs (dense rows padded
  with zeros, key-major lengths / offsets of stride ``B_cap`` whose padded bags are empty, values and weights), reading every size
  from a small device descriptor, so one graph serves every batch that fits;
* the KJTs inside the graph carry both lengths and offsets and a fixed stride, so nothing on the captured path reads the device;
* a batch larger than every bucket runs the wrapped callable eagerly on the same slab. A replay after it first waits for the HBM row
  cache admission that eager call left on its side stream, so the graph's lookups and admissions never overlap it.

Scope: predict callables whose tables all live on one device (``shard_quant_model(world_size=1)``: HBM, ``quant_uvm`` and
``quant_uvm_caching`` tables, bf16 or FP8 dense arch). The modules a callable runs are found from the callable itself (a module, a
bound method's owner, or the modules its closure and globals reference). A module spread over several devices (the W > 1 inference
plane) or holding a sequence (EC) collection, whose outputs need ``length_per_key()``, is refused with ``ValueError``: serve it with
the plain callable, which the server runs eagerly.

Example::

    gp = GraphedPredictor(DLRMPredictModule(sharded, keys), buckets=[64, 256, 2048], num_float=13)
    gp.capture()
    server = InferenceServer([gp], [torch.device("cuda:0")], id_list_keys=keys)
"""
from __future__ import annotations

import inspect
from typing import Any, Callable, List, Optional, Sequence, Tuple, Union

import numpy as np
import torch

from ..sparse.jagged_tensor import KeyedJaggedTensor
from .server import ServerConfig, _BatchDesc, batch_views

# Field order of the ingest descriptor (``csrc/serve_ingest.cu``: D_*), all int64; names are those of the server's batch descriptor.
DESC_FIELDS = ("batch_size", "num_float", "id_list_features", "id_score_features", "dense_off", "idl_lengths_off", "idl_values_off", "idl_num_values",
               "ids_lengths_off", "ids_values_off", "ids_weights_off", "ids_num_values", "total_bytes")

Bucket = Tuple[int, int]


def pack_desc(d: Any) -> np.ndarray:
    """The ingest descriptor of one batch: the ``DESC_FIELDS`` of a server batch descriptor (``server._BatchDesc``) as int64."""
    return np.array([int(getattr(d, f)) for f in DESC_FIELDS], dtype=np.int64)


def _align16(x: int) -> int:
    return (x + 15) & ~15


def slab_bytes_for(B: int, num_float: int, F_idl: int, F_ids: int, nnz_idl: int = 0, nnz_ids: int = 0) -> int:
    """Bytes of the server's slab for a batch of ``B`` samples (``csrc/serving``: every section 16-byte aligned)."""
    return (_align16(B * num_float * 4) + _align16(B * F_idl * 4) + _align16(nnz_idl * 8) + _align16(B * F_ids * 4) + _align16(nnz_ids * 8)
            + _align16(nnz_ids * 4))


def pack_slab(B: int, dense: Optional[np.ndarray] = None, id_list: Optional[Tuple[np.ndarray, np.ndarray]] = None,
              id_score_list: Optional[Tuple[np.ndarray, np.ndarray, np.ndarray]] = None, num_id_list_features: int = 0,
              num_id_score_features: int = 0) -> Tuple[torch.Tensor, _BatchDesc]:
    """One batch in the serving core's slab layout (``csrc/serving``) and its descriptor, built on the host: the input of ``run`` without
    a server, for tests and latency measurements. Lists are ``(lengths int32 [F * B] key-major, values int64[, weights fp32])``."""
    d = _BatchDesc()
    d.batch_size, d.num_requests = B, 1
    parts: List[Tuple[str, np.ndarray]] = []
    if dense is not None:
        d.num_float = dense.shape[1]
        parts.append(("dense_off", np.ascontiguousarray(dense, dtype=np.float32)))
    if id_list is not None:
        d.id_list_features = num_id_list_features
        d.idl_num_values = len(id_list[1])
        parts += [("idl_lengths_off", np.ascontiguousarray(id_list[0], dtype=np.int32)), ("idl_values_off", np.ascontiguousarray(id_list[1], dtype=np.int64))]
    if id_score_list is not None:
        d.id_score_features = num_id_score_features
        d.ids_num_values = len(id_score_list[1])
        parts += [("ids_lengths_off", np.ascontiguousarray(id_score_list[0], dtype=np.int32)), ("ids_values_off", np.ascontiguousarray(id_score_list[1], dtype=np.int64)),
                  ("ids_weights_off", np.ascontiguousarray(id_score_list[2], dtype=np.float32))]
    for f in ("dense_off", "idl_lengths_off", "idl_values_off", "ids_lengths_off", "ids_values_off", "ids_weights_off"):
        setattr(d, f, -1)
    off = 0
    for f, a in parts:
        setattr(d, f, off)
        off = _align16(off + a.nbytes)
    d.total_bytes = off
    slab = np.zeros(max(off, 16), dtype=np.uint8)
    for f, a in parts:
        o = getattr(d, f)
        slab[o : o + a.nbytes] = a.view(np.uint8).reshape(-1)
    return torch.from_numpy(slab), d


def normalize_buckets(buckets: Sequence[Union[int, Bucket]], buffer_bytes: int) -> List[Bucket]:
    """``B_cap`` or ``(B_cap, nnz_cap)`` entries -> sorted, de-duplicated ``(B_cap, nnz_cap)``. A bare ``B_cap`` gets the most ids a slab of
    ``buffer_bytes`` can carry (``buffer_bytes // 8``), so every batch the server forms with ``B <= B_cap`` fits that bucket."""
    out = set()
    for b in buckets:
        B_cap, nnz_cap = (int(b), buffer_bytes // 8) if isinstance(b, (int, np.integer)) else (int(b[0]), int(b[1]))
        if B_cap < 1 or nnz_cap < 0:
            raise ValueError(f"bucket {b!r}: need B_cap >= 1 and nnz_cap >= 0")
        out.add((B_cap, nnz_cap))
    if not out:
        raise ValueError("GraphedPredictor needs at least one bucket")
    return sorted(out)


def choose_bucket(buckets: Sequence[Bucket], B: int, nnz_idl: int, nnz_ids: int) -> Optional[int]:
    """Index of the smallest bucket (``buckets`` sorted by ``B_cap``, then ``nnz_cap``) holding ``B`` samples and the ids of both lists;
    None when no bucket holds the batch."""
    for i, (B_cap, nnz_cap) in enumerate(buckets):
        if B <= B_cap and nnz_idl <= nnz_cap and nnz_ids <= nnz_cap:
            return i
    return None


def _dlrm_predict_fn(pm: torch.nn.Module) -> Callable:
    model = pm.predict_module

    def predict(dense, kjt, _wkjt):
        return model(dense, kjt).sigmoid().reshape(-1)

    return predict


def modules_of(fn: Any) -> List[torch.nn.Module]:
    """The modules a predict callable runs: the callable itself, the owner of a bound method, or the modules its closure and globals
    reference."""
    if isinstance(fn, torch.nn.Module):
        return [fn]
    owner = getattr(fn, "__self__", None)
    if isinstance(owner, torch.nn.Module):
        return [owner]
    try:
        cv = inspect.getclosurevars(fn)
    except TypeError:
        return []
    return [v for v in list(cv.nonlocals.values()) + list(cv.globals.values()) if isinstance(v, torch.nn.Module)]


def check_single_device(modules: Sequence[torch.nn.Module], device: torch.device) -> None:
    """Raise ``ValueError`` for what a graph of one device cannot serve: tensors or shards on another CUDA device, and sequence (EC)
    collections."""
    from ..parallel.quant_embedding import ShardedQuantEmbeddingCollection
    from ..parallel.quant_embeddingbag import ShardedQuantEmbeddingBagCollection, _dev
    from ..quant.embedding_modules import EmbeddingCollection as QuantEmbeddingCollection

    for top in modules:
        for m in top.modules():
            if isinstance(m, (ShardedQuantEmbeddingCollection, QuantEmbeddingCollection)):
                raise ValueError(f"{type(m).__name__}: sequence collections need length_per_key() of every batch and are served eagerly")
            if isinstance(m, ShardedQuantEmbeddingBagCollection):
                ranks = [r for r, units in enumerate(m._rank_meta) if units]
                if len(ranks) > 1 or any(_dev(m._device_type, r) != device for r in ranks):
                    raise ValueError(f"a sharded collection on ranks {ranks} spans devices other than {device} and is served eagerly")
        for t in list(top.parameters()) + list(top.buffers()):
            if t.is_cuda and t.device != device:
                raise ValueError(f"a tensor of the predict module lives on {t.device}, not {device}: multi-device models are served eagerly")


class GraphedPredictor:
    """``predict_fn(dense [B, num_float] | None, id_list KJT | None, id_score_list KJT | None) -> Tensor [B] or [B, P]`` (the server
    executor's contract) or a ``DLRMPredictModule``, replayed from one CUDA graph per bucket.

    ``buckets``: ``B_cap`` or ``(B_cap, nnz_cap)`` entries (see ``normalize_buckets``). ``buffer_bytes`` and ``max_batch_size`` are the
    server's (``ServerConfig``): the device slab holds ``buffer_bytes``, and ``capture`` warms the callable up at the largest batch a
    slab can carry, so a later eager batch does not regrow buffers the graphs have captured. ``run`` returns a view of the graph's
    static output, valid until the next ``run``."""

    def __init__(self, predict_fn: Union[Callable, torch.nn.Module], buckets: Sequence[Union[int, Bucket]], num_float: int,
                 id_list_keys: Optional[Sequence[str]] = None, id_score_list_keys: Sequence[str] = (), device: Optional[torch.device] = None,
                 buffer_bytes: int = ServerConfig.buffer_bytes, max_batch_size: int = ServerConfig.max_batch_size) -> None:
        from .dlrm_predict import DLRMPredictModule

        if isinstance(predict_fn, DLRMPredictModule):
            if id_list_keys is None:
                id_list_keys = predict_fn.id_list_features_keys
            if device is None:
                device = predict_fn._device or next(predict_fn.predict_module.parameters()).device
            predict_fn = _dlrm_predict_fn(predict_fn)
        if device is None and isinstance(predict_fn, torch.nn.Module):
            device = next(predict_fn.parameters()).device
        self.predict_fn = predict_fn
        self.device = torch.device(device) if device is not None else torch.device("cuda")
        if self.device.type == "cuda" and self.device.index is None and torch.cuda.is_available():
            self.device = torch.device("cuda", torch.cuda.current_device())
        self._modules = modules_of(predict_fn)
        check_single_device(self._modules, self.device)
        self.num_float = int(num_float)
        self.id_list_keys = list(id_list_keys or [])
        self.id_score_list_keys = list(id_score_list_keys)
        self.F_idl, self.F_ids = len(self.id_list_keys), len(self.id_score_list_keys)
        self.buffer_bytes = int(buffer_bytes)
        self.max_batch_size = int(max_batch_size)
        self.buckets = normalize_buckets(buckets, self.buffer_bytes)
        for B_cap, _ in self.buckets:
            if slab_bytes_for(B_cap, self.num_float, self.F_idl, self.F_ids) > self.buffer_bytes:
                raise ValueError(f"bucket B_cap={B_cap}: its dense rows and lengths alone exceed the {self.buffer_bytes}-byte slab")
        self.offsets_dtype = torch.int64 if max(n for _, n in self.buckets) >= 2**31 else torch.int32
        self.slab: Optional[torch.Tensor] = None  # device copy of the batch slab: the graphs' input
        self._graphs: List[torch.cuda.CUDAGraph] = []
        self._outs: List[torch.Tensor] = []
        self._launches: List[int] = []

    # ---- host logic ------------------------------------------------------------------------------------------------------------
    def bucket_for(self, d: Any) -> Optional[int]:
        """The bucket a batch descriptor replays, or None for the eager path (no bucket holds it, or its feature counts differ)."""
        if (d.num_float, d.id_list_features, d.id_score_features) != (self.num_float, self.F_idl, self.F_ids):
            return None
        return choose_bucket(self.buckets, d.batch_size, d.idl_num_values if self.F_idl else 0, d.ids_num_values if self.F_ids else 0)

    def _eager(self, slab_dev: torch.Tensor, d: Any) -> torch.Tensor:
        return self.predict_fn(*batch_views(slab_dev, d, self.id_list_keys, self.id_score_list_keys))

    @property
    def captured(self) -> bool:
        return bool(self._graphs)

    # ---- device side -----------------------------------------------------------------------------------------------------------
    def _static_inputs(self, buf) -> Tuple[Optional[torch.Tensor], Optional[KeyedJaggedTensor], Optional[KeyedJaggedTensor]]:
        B_cap = buf.B_cap
        kjt = wkjt = None
        if self.F_idl:
            kjt = KeyedJaggedTensor(keys=self.id_list_keys, values=buf.idl_values, lengths=buf.idl_lengths, offsets=buf.idl_offsets, stride=B_cap)
        if self.F_ids:
            wkjt = KeyedJaggedTensor(keys=self.id_score_list_keys, values=buf.ids_values, lengths=buf.ids_lengths, offsets=buf.ids_offsets,
                                     weights=buf.ids_weights, stride=B_cap)
        return buf.dense, kjt, wkjt

    def _ingest(self, buf) -> None:
        from ..ops import serve as _serve

        _serve.ingest(self.slab, self._desc, buf, self.num_float, self.F_idl, self.F_ids, self._error)

    def _empty_batch_desc(self, B: int) -> np.ndarray:
        """Descriptor of ``B`` samples with zero dense rows and empty bags: an all-zero slab holds that batch in any layout."""
        nf, F1, F2 = self.num_float, self.F_idl, self.F_ids
        _, d = pack_slab(B, np.zeros((B, nf), dtype=np.float32) if nf else None, (np.zeros(F1 * B), np.zeros(0)) if F1 else None,
                         (np.zeros(F2 * B), np.zeros(0), np.zeros(0)) if F2 else None, F1, F2)
        return pack_desc(d)

    def _set_desc(self, fields: np.ndarray) -> None:
        host = torch.empty(len(DESC_FIELDS), dtype=torch.int64, pin_memory=True)  # the caching host allocator keeps it until the copy ran
        host.numpy()[:] = fields
        self._desc.copy_(host, non_blocking=True)

    def capture(self, num_warmup_iters: int = 2) -> "GraphedPredictor":
        """Warm every bucket up eagerly (lookup workspaces, GEMM weight casts and module loads happen outside capture), warm the
        callable up at the largest batch a slab can carry, then capture ingest + predict once per bucket on a private stream into one
        shared memory pool."""
        from ..ops import _lib
        from ..ops.serve import IngestBuffers

        if self.device.type != "cuda":
            raise RuntimeError("GraphedPredictor.capture needs a CUDA device")
        dev = self.device
        B_max, nnz_max = max(b for b, _ in self.buckets), max(n for _, n in self.buckets)
        with torch.cuda.device(dev), torch.inference_mode(False):  # static buffers are ordinary tensors: callers may write them
            self.slab = torch.zeros(self.buffer_bytes, dtype=torch.uint8, device=dev)
            self._desc = torch.zeros(len(DESC_FIELDS), dtype=torch.int64, device=dev)
            self._error = torch.zeros(1, dtype=torch.int32, pin_memory=True)  # mapped host memory: the kernel writes it, the host reads it
            # graphs never run concurrently, so the buckets share one set of buffers sized for the largest
            shared = IngestBuffers.allocate(B_max, nnz_max, self.num_float, self.F_idl, self.F_ids, self.offsets_dtype, dev)
            bufs = [shared.view(B_cap, nnz_cap) for B_cap, nnz_cap in self.buckets]
        with torch.cuda.device(dev), torch.inference_mode():
            torch.cuda.synchronize(dev)
            stream = torch.cuda.Stream(dev)
            stream.wait_stream(torch.cuda.current_stream(dev))
            with torch.cuda.stream(stream):
                # eager, at the largest batch the server can hand over (a slab holds at most buffer_bytes // 8 ids): buffers that grow with
                # the batch reach their final size before any graph captures their addresses
                self._warmup_eager(max(self.max_batch_size, B_max), max(self.buffer_bytes // 8, nnz_max) if self.F_idl or self.F_ids else 0)
                for buf in bufs:
                    self._set_desc(self._empty_batch_desc(buf.B_cap))
                    for _ in range(num_warmup_iters):
                        self._ingest(buf)
                        self.predict_fn(*self._static_inputs(buf))
            torch.cuda.synchronize(dev)
            pool = torch.cuda.graph_pool_handle()
            graphs, outs, launches = [], [], []
            for buf in bufs:
                g = torch.cuda.CUDAGraph()
                n0 = _lib.launch_count()
                with torch.cuda.graph(g, pool=pool, stream=stream):
                    self._ingest(buf)
                    out = self.predict_fn(*self._static_inputs(buf))
                graphs.append(g)
                outs.append(out)
                launches.append(_lib.launch_count() - n0)
            torch.cuda.synchronize(dev)
        self._bufs, self._graphs, self._outs, self._launches = bufs, graphs, outs, launches
        self._cached_tbes = self._find_cached_tbes()
        if int(self._error[0]):
            raise RuntimeError("serve_ingest rejected a warm-up batch")
        return self

    def _find_cached_tbes(self) -> list:
        """Tables behind an HBM row cache: their eager calls admit rows on a side stream that a replay must wait for."""
        from ..ops.quant_tbe import QuantTableBatchedEmbeddingBags

        seen = {}
        for top in self._modules:
            for m in top.modules():
                if isinstance(m, QuantTableBatchedEmbeddingBags) and m._placed and m._cached:
                    seen[id(m)] = m
        return list(seen.values())

    def _warmup_eager(self, B: int, nnz: int) -> None:
        """One eager call on empty bags whose value tensors hold ``nnz`` ids (lookup buffers are sized from the value count)."""
        dev = self.device
        dense = torch.zeros(B, self.num_float, device=dev) if self.num_float else None
        kjt = wkjt = None
        if self.F_idl:
            kjt = KeyedJaggedTensor(keys=self.id_list_keys, values=torch.zeros(nnz, dtype=torch.int64, device=dev),
                                    lengths=torch.zeros(self.F_idl * B, dtype=torch.int32, device=dev), stride=B)
        if self.F_ids:
            wkjt = KeyedJaggedTensor(keys=self.id_score_list_keys, values=torch.zeros(nnz, dtype=torch.int64, device=dev),
                                     lengths=torch.zeros(self.F_ids * B, dtype=torch.int32, device=dev),
                                     weights=torch.zeros(nnz, dtype=torch.float32, device=dev), stride=B)
        self.predict_fn(dense, kjt, wkjt)

    def ingest_failed(self) -> bool:
        """True when an ingest launch has rejected its batch since the last call (reads the flag without a device sync: call it after the
        batch's output has been synchronised). Clears the flag."""
        if self.slab is None or not int(self._error[0]):
            return False
        self._error.zero_()
        return True

    def run(self, slab_dev: torch.Tensor, d: Any) -> torch.Tensor:
        """Predict the batch described by ``d`` (a server batch descriptor) whose slab is on the device in ``slab_dev``: the smallest
        bucket holding it is replayed (``slab_dev`` is copied into the graphs' slab unless it is that slab); a batch no bucket holds runs
        the callable eagerly on ``slab_dev``. Returns the first ``B`` rows of the output; no host synchronisation."""
        B = int(d.batch_size)
        if B > max(self.max_batch_size, self.buckets[-1][0]):
            raise ValueError(f"batch of {B} samples exceeds max_batch_size={self.max_batch_size}")
        i = self.bucket_for(d)
        with torch.inference_mode():
            if i is None:
                return self._eager(slab_dev, d)
            if not self._graphs:
                raise RuntimeError("GraphedPredictor.run before capture()")
            n = int(d.total_bytes)
            if slab_dev.data_ptr() != self.slab.data_ptr():
                self.slab[:n].copy_(slab_dev[:n], non_blocking=True)
            self._set_desc(pack_desc(d))
            for tbe in self._cached_tbes:  # a replay runs no Python: order it after an admission an eager call left pending
                tbe._wait_admission()
            self._graphs[i].replay()
            if self._launches[i]:
                from ..ops import _lib

                _lib.add_launches(self._launches[i])
            return self._outs[i][:B]
