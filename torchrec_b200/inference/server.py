"""Inference server: native batching core (csrc/serving) + per-GPU executor threads + optional gRPC front end.

Parity: reference torchrec/inference/server.cpp (gRPC ``Predictor.Predict``), inference_legacy BatchingQueue / GPUExecutor /
ResultSplit / ResourceManager, protos/predictor.proto. The C++ core coalesces requests into ONE pinned slab per batch
(dense | lengths | values | weights, KJT key-major layout); the executor issues one H2D copy per batch, runs the predict
module (quantized sharded model, ``inference/modules.py``) on its own CUDA stream and hands the predictions back to C++,
which splits them per request."""
from __future__ import annotations

import ctypes
import threading
import time
from dataclasses import dataclass
from typing import Callable, Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from ..csrc import build as _native
from ..sparse.jagged_tensor import KeyedJaggedTensor


class _BatchDesc(ctypes.Structure):
    _fields_ = [("batch_id", ctypes.c_int64), ("buffer_index", ctypes.c_int32), ("batch_size", ctypes.c_int32), ("num_requests", ctypes.c_int32),
                ("num_float", ctypes.c_int32), ("id_list_features", ctypes.c_int32), ("id_score_features", ctypes.c_int32), ("dense_off", ctypes.c_int64),
                ("idl_lengths_off", ctypes.c_int64), ("idl_values_off", ctypes.c_int64), ("idl_num_values", ctypes.c_int64), ("ids_lengths_off", ctypes.c_int64),
                ("ids_values_off", ctypes.c_int64), ("ids_weights_off", ctypes.c_int64), ("ids_num_values", ctypes.c_int64), ("total_bytes", ctypes.c_int64),
                ("oldest_wait_us", ctypes.c_int64)]


_LIB = None


def _lib():
    global _LIB
    if _LIB is None:
        L = _native.load("serving")
        vp, i64, i32 = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int32
        L.trb_srv_create.restype = vp
        L.trb_srv_create.argtypes = [i32, i64, i32, i32, i32, i64]
        L.trb_srv_destroy.argtypes = [vp]
        L.trb_srv_shutdown.argtypes = [vp]
        L.trb_srv_add_buffer.argtypes = [vp, vp, i64]
        L.trb_srv_submit.restype = i64
        L.trb_srv_submit.argtypes = [vp, i32, i32, vp, i32, vp, vp, i64, i32, vp, vp, vp, i64]
        L.trb_srv_pop_batch.restype = ctypes.c_int
        L.trb_srv_pop_batch.argtypes = [vp, ctypes.c_int, i64, ctypes.POINTER(_BatchDesc)]
        L.trb_srv_complete.restype = ctypes.c_int
        L.trb_srv_complete.argtypes = [vp, i64, vp, i32, ctypes.c_int]
        L.trb_srv_wait.restype = ctypes.c_int
        L.trb_srv_wait.argtypes = [vp, i64, vp, i64, i64, ctypes.POINTER(i64)]
        L.trb_srv_stats.argtypes = [vp, ctypes.POINTER(i64)]
        _LIB = L
    return _LIB


def batch_views(buf: torch.Tensor, d: "_BatchDesc", id_list_keys: Sequence[str], id_score_list_keys: Sequence[str]):
    """``(dense [B, num_float] | None, id_list KJT | None, id_score_list KJT | None)`` as views of one batch slab ``buf`` (host or device)."""
    B = d.batch_size

    def view(off, n, dtype, esz):
        return buf[off : off + n * esz].view(dtype)

    dense = view(d.dense_off, B * d.num_float, torch.float32, 4).view(B, d.num_float) if d.num_float else None
    kjt = wkjt = None
    if d.id_list_features:
        kjt = KeyedJaggedTensor(keys=id_list_keys, values=view(d.idl_values_off, d.idl_num_values, torch.int64, 8),
                                lengths=view(d.idl_lengths_off, B * d.id_list_features, torch.int32, 4), stride=B)
    if d.id_score_features:
        wkjt = KeyedJaggedTensor(keys=id_score_list_keys, values=view(d.ids_values_off, d.ids_num_values, torch.int64, 8),
                                 lengths=view(d.ids_lengths_off, B * d.id_score_features, torch.int32, 4),
                                 weights=view(d.ids_weights_off, d.ids_num_values, torch.float32, 4), stride=B)
    return dense, kjt, wkjt


@dataclass
class ServerConfig:
    max_batch_size: int = 2048
    batching_interval_ms: float = 1.0
    max_outstanding_per_gpu: int = 2
    batching_threads: int = 2
    num_buffers_per_gpu: int = 4
    buffer_bytes: int = 16 << 20
    max_queue_requests: int = 1 << 16
    outputs_per_sample: int = 1


class InferenceServer:
    """``predict_fn(dense [B, num_float] | None, id_list KJT | None, id_score_list KJT | None) -> Tensor [B] or [B, P]``,
    one callable per device. A captured ``inference.graphed.GraphedPredictor`` may stand in for a callable: its batches replay a CUDA
    graph from the predictor's static device slab."""

    def __init__(self, predict_fns: Sequence[Callable], devices: Sequence[torch.device], id_list_keys: Sequence[str] = (), id_score_list_keys: Sequence[str] = (),
                 config: Optional[ServerConfig] = None) -> None:
        from .graphed import GraphedPredictor

        assert len(predict_fns) == len(devices) and len(devices) >= 1
        self.cfg = config or ServerConfig()
        self.devices = [torch.device(d) for d in devices]
        self.predict_fns = list(predict_fns)
        self._graphed = [isinstance(fn, GraphedPredictor) for fn in self.predict_fns]
        for fn, dev, g in zip(self.predict_fns, self.devices, self._graphed):
            if g and (dev.type != "cuda" or not fn.captured or fn.device != dev or fn.buffer_bytes < self.cfg.buffer_bytes
                      or fn.max_batch_size < self.cfg.max_batch_size or fn.id_list_keys != list(id_list_keys)
                      or fn.id_score_list_keys != list(id_score_list_keys)):
                raise ValueError(f"a GraphedPredictor serves the CUDA device it was captured on, after capture(), with the server's keys, a slab "
                                 f"of at least buffer_bytes={self.cfg.buffer_bytes} and max_batch_size >= {self.cfg.max_batch_size} (got device "
                                 f"{dev}, captured={fn.captured}, {fn.device}, {fn.buffer_bytes} bytes, max_batch_size={fn.max_batch_size}, "
                                 f"keys {fn.id_list_keys} / {fn.id_score_list_keys})")
        self._out_host: List[Optional[torch.Tensor]] = [None] * len(self.devices)
        self.id_list_keys, self.id_score_list_keys = list(id_list_keys), list(id_score_list_keys)
        L = _lib()
        self._h = L.trb_srv_create(self.cfg.max_batch_size, int(self.cfg.batching_interval_ms * 1000), len(self.devices), self.cfg.max_outstanding_per_gpu,
                                   self.cfg.batching_threads, self.cfg.max_queue_requests)
        pin = torch.cuda.is_available()
        self._slabs = [torch.empty(self.cfg.buffer_bytes, dtype=torch.uint8, pin_memory=pin) for _ in range(self.cfg.num_buffers_per_gpu * len(self.devices))]
        for s in self._slabs:
            L.trb_srv_add_buffer(self._h, s.data_ptr(), s.numel())
        self._stop = False
        self._threads = [threading.Thread(target=self._executor, args=(i,), daemon=True, name=f"trb-exec-{i}") for i in range(len(self.devices))]
        for t in self._threads:
            t.start()

    # ---- client API --------------------------------------------------------------------------------------------
    def submit(self, batch_size: int, dense: Optional[np.ndarray] = None, id_list: Optional[Tuple[np.ndarray, np.ndarray]] = None,
               id_score_list: Optional[Tuple[np.ndarray, np.ndarray, np.ndarray]] = None) -> int:
        """id_list = (lengths int32 [F*B] key-major, values int64); id_score_list adds float32 weights. Returns a request id."""
        def p(a):
            return a.ctypes.data_as(ctypes.c_void_p) if a is not None else None

        d = np.ascontiguousarray(dense, dtype=np.float32) if dense is not None else None
        nf = d.shape[1] if d is not None else 0
        l1 = v1 = l2 = v2 = w2 = None
        if id_list is not None:
            l1, v1 = np.ascontiguousarray(id_list[0], dtype=np.int32), np.ascontiguousarray(id_list[1], dtype=np.int64)
            assert l1.size == len(self.id_list_keys) * batch_size and int(l1.sum()) == v1.size
        if id_score_list is not None:
            l2, v2, w2 = (np.ascontiguousarray(id_score_list[0], dtype=np.int32), np.ascontiguousarray(id_score_list[1], dtype=np.int64),
                          np.ascontiguousarray(id_score_list[2], dtype=np.float32))
            assert l2.size == len(self.id_score_list_keys) * batch_size and int(l2.sum()) == v2.size == w2.size
        rid = _lib().trb_srv_submit(self._h, batch_size, nf, p(d), len(self.id_list_keys) if l1 is not None else 0, p(l1), p(v1), v1.size if v1 is not None else 0,
                                    len(self.id_score_list_keys) if l2 is not None else 0, p(l2), p(v2), p(w2), v2.size if v2 is not None else 0)
        if rid < 0:
            raise RuntimeError("inference server intake queue is full")
        return rid

    def wait(self, request_id: int, batch_size: int, timeout_s: float = 10.0) -> np.ndarray:
        out = np.empty(batch_size * self.cfg.outputs_per_sample, dtype=np.float32)
        n = ctypes.c_int64(0)
        rc = _lib().trb_srv_wait(self._h, request_id, out.ctypes.data_as(ctypes.c_void_p), out.size, int(timeout_s * 1e6), ctypes.byref(n))
        if rc == 1:
            raise TimeoutError(f"request {request_id} timed out")
        if rc != 0:
            raise RuntimeError(f"request {request_id} failed with status {rc}")
        return out[: n.value].reshape(batch_size, -1)

    def predict(self, batch_size: int, dense=None, id_list=None, id_score_list=None, timeout_s: float = 10.0) -> np.ndarray:
        return self.wait(self.submit(batch_size, dense, id_list, id_score_list), batch_size, timeout_s)

    def stats(self) -> Dict[str, int]:
        a = (ctypes.c_int64 * 8)()
        _lib().trb_srv_stats(self._h, a)
        names = ["requests", "batches", "samples", "rejected", "timeouts", "queue_us_sum", "queue_us_max", "exec_us_sum"]
        return dict(zip(names, list(a)))

    # ---- executor ------------------------------------------------------------------------------------------------
    def _tensors(self, slab: torch.Tensor, d: _BatchDesc, dev: torch.device):
        host = slab[: d.total_bytes]
        buf = host.to(dev, non_blocking=True) if dev.type == "cuda" else host  # ONE copy per batch
        return batch_views(buf, d, self.id_list_keys, self.id_score_list_keys)

    def _run_graphed(self, gpu: int, slab: torch.Tensor, d: _BatchDesc, stream) -> torch.Tensor:
        """A ``GraphedPredictor``: the slab goes into its static device slab (the one H2D copy), the result back through a pinned buffer."""
        gp = self.predict_fns[gpu]
        n = d.total_bytes
        gp.slab[:n].copy_(slab[:n], non_blocking=True)
        out = gp.run(gp.slab, d).reshape(d.batch_size, -1)
        if self._out_host[gpu] is None or self._out_host[gpu].numel() < out.numel():
            self._out_host[gpu] = torch.empty(max(out.numel(), self.cfg.max_batch_size * self.cfg.outputs_per_sample), dtype=torch.float32, pin_memory=True)
        res = self._out_host[gpu][: out.numel()].view(out.shape)
        res.copy_(out, non_blocking=True)
        stream.synchronize()
        if gp.ingest_failed():
            raise RuntimeError("serve_ingest rejected the batch")
        return res

    def _executor(self, gpu: int) -> None:
        L = _lib()
        dev = self.devices[gpu]
        stream = torch.cuda.Stream(dev) if dev.type == "cuda" else None
        graphed = self._graphed[gpu]
        d = _BatchDesc()
        while not self._stop:
            rc = L.trb_srv_pop_batch(self._h, gpu, 50_000, ctypes.byref(d))
            if rc == 2:
                return
            if rc != 0:
                continue
            try:
                with torch.inference_mode():
                    if graphed:
                        with torch.cuda.stream(stream):
                            out = self._run_graphed(gpu, self._slabs[d.buffer_index], d, stream)
                    elif stream is not None:
                        with torch.cuda.stream(stream):
                            out = self.predict_fns[gpu](*self._tensors(self._slabs[d.buffer_index], d, dev))
                            out = out.float().reshape(d.batch_size, -1).cpu()
                    else:
                        out = self.predict_fns[gpu](*self._tensors(self._slabs[d.buffer_index], d, dev)).float().reshape(d.batch_size, -1).contiguous()
                L.trb_srv_complete(self._h, d.batch_id, out.data_ptr(), out.shape[1], 0)
            except Exception:  # the failure goes to every request of the batch; the server keeps running
                import traceback

                traceback.print_exc()
                L.trb_srv_complete(self._h, d.batch_id, None, 0, -5)

    def shutdown(self) -> None:
        if self._h:
            self._stop = True
            _lib().trb_srv_shutdown(self._h)
            for t in self._threads:
                t.join(timeout=2)
            _lib().trb_srv_destroy(self._h)
            self._h = None

    def __del__(self) -> None:
        try:
            self.shutdown()
        except Exception:
            pass


# ---- gRPC front end (wire-compatible with the reference's predictor.proto) ----------------------------------------------
def _proto_classes():
    """Build the predictor.proto message classes at runtime (no protoc in the image)."""
    from google.protobuf import descriptor_pb2, descriptor_pool, message_factory

    fd = descriptor_pb2.FileDescriptorProto(name="trb_predictor.proto", package="predictor", syntax="proto3")
    T = descriptor_pb2.FieldDescriptorProto

    def msg(name, fields):
        m = fd.message_type.add(name=name)
        for i, (fname, ftype, tname, label) in enumerate(fields, 1):
            f = m.field.add(name=fname, number=i, type=ftype, label=label)
            if tname:
                f.type_name = tname
        return m

    O, R = T.LABEL_OPTIONAL, T.LABEL_REPEATED
    msg("SparseFeatures", [("num_features", T.TYPE_INT32, None, O), ("lengths", T.TYPE_BYTES, None, O), ("values", T.TYPE_BYTES, None, O), ("weights", T.TYPE_BYTES, None, O)])
    msg("FloatFeatures", [("num_features", T.TYPE_INT32, None, O), ("values", T.TYPE_BYTES, None, O)])
    msg("PredictionRequest", [("batch_size", T.TYPE_INT32, None, O), ("float_features", T.TYPE_MESSAGE, ".predictor.FloatFeatures", O),
                              ("id_list_features", T.TYPE_MESSAGE, ".predictor.SparseFeatures", O), ("id_score_list_features", T.TYPE_MESSAGE, ".predictor.SparseFeatures", O),
                              ("embedding_features", T.TYPE_MESSAGE, ".predictor.FloatFeatures", O), ("unary_features", T.TYPE_MESSAGE, ".predictor.SparseFeatures", O)])
    msg("FloatVec", [("data", T.TYPE_FLOAT, None, R)])
    resp = msg("PredictionResponse", [("predictions", T.TYPE_MESSAGE, ".predictor.PredictionResponse.PredictionsEntry", R)])
    entry = resp.nested_type.add(name="PredictionsEntry")
    entry.options.map_entry = True
    entry.field.add(name="key", number=1, type=T.TYPE_STRING, label=O)
    entry.field.add(name="value", number=2, type=T.TYPE_MESSAGE, label=O, type_name=".predictor.FloatVec")
    pool = descriptor_pool.DescriptorPool()
    pool.Add(fd)
    get = lambda n: message_factory.GetMessageClass(pool.FindMessageTypeByName(f"predictor.{n}"))
    return get("PredictionRequest"), get("PredictionResponse")


_PROTO = None


def proto_classes():
    global _PROTO
    if _PROTO is None:
        _PROTO = _proto_classes()
    return _PROTO


def serve_grpc(server: InferenceServer, port: int = 50051, task_name: str = "default", max_workers: int = 16):
    """Start a gRPC ``predictor.Predictor/Predict`` endpoint in front of ``server``. Returns the grpc server object."""
    from concurrent import futures

    import grpc

    Req, Resp = proto_classes()

    def predict(request, context):
        B = request.batch_size
        dense = None
        if request.float_features.num_features:
            dense = np.frombuffer(request.float_features.values, dtype=np.float32).reshape(B, request.float_features.num_features)
        idl = ids = None
        if request.id_list_features.num_features:
            s = request.id_list_features
            idl = (np.frombuffer(s.lengths, dtype=np.int32), np.frombuffer(s.values, dtype=np.int64))
        if request.id_score_list_features.num_features:
            s = request.id_score_list_features
            ids = (np.frombuffer(s.lengths, dtype=np.int32), np.frombuffer(s.values, dtype=np.int64), np.frombuffer(s.weights, dtype=np.float32))
        out = server.predict(B, dense, idl, ids)
        resp = Resp()
        resp.predictions[task_name].data.extend(out.reshape(-1).tolist())
        return resp

    handler = grpc.method_handlers_generic_handler("predictor.Predictor", {
        "Predict": grpc.unary_unary_rpc_method_handler(predict, request_deserializer=Req.FromString, response_serializer=lambda m: m.SerializeToString())})
    g = grpc.server(futures.ThreadPoolExecutor(max_workers=max_workers))
    g.add_generic_rpc_handlers((handler,))
    bound = g.add_insecure_port(f"127.0.0.1:{port}")
    g.start()
    g.bound_port = bound  # type: ignore[attr-defined]
    return g


class PredictorClient:
    """Minimal client of the ``predictor.Predictor`` service (reference inference/client.py)."""

    def __init__(self, target: str) -> None:
        import grpc

        Req, Resp = proto_classes()
        self._Req = Req
        self._channel = grpc.insecure_channel(target)
        self._call = self._channel.unary_unary("/predictor.Predictor/Predict", request_serializer=lambda m: m.SerializeToString(), response_deserializer=Resp.FromString)

    def predict(self, batch_size: int, dense: Optional[np.ndarray] = None, id_list: Optional[Tuple[np.ndarray, np.ndarray]] = None, num_id_list_features: int = 0,
                timeout: float = 10.0) -> Dict[str, np.ndarray]:
        r = self._Req(batch_size=batch_size)
        if dense is not None:
            r.float_features.num_features = dense.shape[1]
            r.float_features.values = np.ascontiguousarray(dense, dtype=np.float32).tobytes()
        if id_list is not None:
            r.id_list_features.num_features = num_id_list_features
            r.id_list_features.lengths = np.ascontiguousarray(id_list[0], dtype=np.int32).tobytes()
            r.id_list_features.values = np.ascontiguousarray(id_list[1], dtype=np.int64).tobytes()
        resp = self._call(r, timeout=timeout)
        return {k: np.asarray(v.data, dtype=np.float32) for k, v in resp.predictions.items()}

    def close(self) -> None:
        self._channel.close()


# ---- native (C++) network front: csrc/serving/net_front.cpp -------------------------------------------------------------------------
class NativeFront:
    """Handle of the C++ TCP front started by ``serve_native``: ``port``, ``stats()``, ``stop()``."""

    def __init__(self, handle: int, port: int) -> None:
        self._h, self.port = handle, port

    def stats(self) -> Dict[str, int]:
        a = (ctypes.c_int64 * 3)()
        _lib().trb_srv_listen_stats(ctypes.c_void_p(self._h), a)
        return {"served": a[0], "malformed": a[1], "refused": a[2]}

    def stop(self) -> None:
        if self._h:
            _lib().trb_srv_listen_stop(ctypes.c_void_p(self._h))
            self._h = 0

    def __del__(self) -> None:
        try:
            self.stop()
        except Exception:
            pass


def serve_native(server: InferenceServer, port: int = 0, task_name: str = "default", max_connections: int = 64, timeout_s: float = 10.0) -> NativeFront:
    """Start the C++ network front on 127.0.0.1 (``port=0``: any free port). Sockets, request parsing (the ``predictor.PredictionRequest``
    protobuf wire format, read by hand), intake into the batching queue and response encoding all run on C++ threads; Python only executes
    the model on the executor threads. Frames are ``uint32 little-endian length + message bytes`` (grpc++ is not available in this image:
    the gRPC front ``serve_grpc`` speaks HTTP/2 through the Python grpc runtime instead). Stop the front before shutting the server down."""
    L = _lib()
    L.trb_srv_listen.restype = ctypes.c_void_p
    L.trb_srv_listen.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_char_p, ctypes.c_int, ctypes.c_int, ctypes.c_int64, ctypes.POINTER(ctypes.c_int)]
    L.trb_srv_listen_stop.argtypes = [ctypes.c_void_p]
    L.trb_srv_listen_stats.argtypes = [ctypes.c_void_p, ctypes.POINTER(ctypes.c_int64)]
    bound = ctypes.c_int(0)
    h = L.trb_srv_listen(server._h, int(port), task_name.encode(), int(server.cfg.outputs_per_sample), int(max_connections), int(timeout_s * 1e6), ctypes.byref(bound))
    if not h:
        raise RuntimeError(f"cannot listen on 127.0.0.1:{port}")
    return NativeFront(h, bound.value)


class NativePredictorClient:
    """Client of the native front: the same ``predictor`` protobuf messages as the gRPC client, framed with a 4-byte length."""

    def __init__(self, host: str, port: int, timeout: float = 10.0) -> None:
        import socket

        self._Req, self._Resp = proto_classes()
        self._sock = socket.create_connection((host, port), timeout=timeout)
        self._sock.setsockopt(socket.IPPROTO_TCP, socket.TCP_NODELAY, 1)

    def _recv(self, n: int) -> bytes:
        chunks = []
        while n:
            c = self._sock.recv(n)
            if not c:
                raise ConnectionError("native front closed the connection")
            chunks.append(c)
            n -= len(c)
        return b"".join(chunks)

    def predict_raw(self, payload: bytes) -> bytes:
        self._sock.sendall(len(payload).to_bytes(4, "little") + payload)
        n = int.from_bytes(self._recv(4), "little")
        return self._recv(n)

    def predict(self, batch_size: int, dense: Optional[np.ndarray] = None, id_list: Optional[Tuple[np.ndarray, np.ndarray]] = None, num_id_list_features: int = 0,
                id_score_list: Optional[Tuple[np.ndarray, np.ndarray, np.ndarray]] = None, num_id_score_list_features: int = 0) -> Dict[str, np.ndarray]:
        r = self._Req(batch_size=batch_size)
        if dense is not None:
            r.float_features.num_features = dense.shape[1]
            r.float_features.values = np.ascontiguousarray(dense, dtype=np.float32).tobytes()
        if id_list is not None:
            r.id_list_features.num_features = num_id_list_features
            r.id_list_features.lengths = np.ascontiguousarray(id_list[0], dtype=np.int32).tobytes()
            r.id_list_features.values = np.ascontiguousarray(id_list[1], dtype=np.int64).tobytes()
        if id_score_list is not None:
            r.id_score_list_features.num_features = num_id_score_list_features
            r.id_score_list_features.lengths = np.ascontiguousarray(id_score_list[0], dtype=np.int32).tobytes()
            r.id_score_list_features.values = np.ascontiguousarray(id_score_list[1], dtype=np.int64).tobytes()
            r.id_score_list_features.weights = np.ascontiguousarray(id_score_list[2], dtype=np.float32).tobytes()
        raw = self.predict_raw(r.SerializeToString())
        resp = self._Resp.FromString(raw)
        if not resp.predictions:
            raise RuntimeError(f"native front reported a failed request ({raw.hex()})")
        return {k: np.asarray(v.data, dtype=np.float32) for k, v in resp.predictions.items()}

    def close(self) -> None:
        self._sock.close()
