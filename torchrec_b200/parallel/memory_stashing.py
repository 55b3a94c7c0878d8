"""Memory stashing: park embedding weights / optimizer state in pinned host memory while they are not needed and bring
them back just in time (reference torchrec/distributed/memory_stashing.py:38-800).

On an 80 GB H100 this is what lets the *dense* part of a step borrow the HBM of tables it does not touch (e.g. the
optimizer state between its use in the backward of step i and step i+1, or tables of a frozen tower). A stash is an async
D2H copy on the ``d2h`` stream followed by freeing the device storage in place (``untyped_storage().resize_(0)`` — every
view, including the table-batched kernel's parameter views, keeps pointing at the same storage object); a restore
re-allocates the storage and copies back on the ``h2d`` stream. ``await_restore`` makes the compute stream wait."""
from __future__ import annotations

import threading
from concurrent.futures import Future, ThreadPoolExecutor
from typing import Any, Callable, Dict, List, Optional, Tuple

import torch
from torch import nn


class _Stash:
    def __init__(self, tensor: torch.Tensor) -> None:
        self.tensor = tensor
        self.nbytes = tensor.untyped_storage().nbytes()
        self.host: Optional[torch.Tensor] = None
        self.event: Optional[torch.cuda.Event] = None
        self.stashed = False


class MemoryStashingManager:
    _h2d: Optional["torch.cuda.Stream"] = None
    _d2h: Optional["torch.cuda.Stream"] = None
    _pool: Optional[ThreadPoolExecutor] = None
    _stashes: Dict[str, List[_Stash]] = {}
    _delay = False
    _pending: List[Callable[[], None]] = []
    _lock = threading.Lock()

    # ---- configuration ------------------------------------------------------------------------------------------
    @classmethod
    def set_streams(cls, h2d_stream: Optional["torch.cuda.Stream"] = None, d2h_stream: Optional["torch.cuda.Stream"] = None) -> None:
        cls._h2d, cls._d2h = h2d_stream, d2h_stream

    @classmethod
    def h2d_stream(cls):
        if cls._h2d is None and torch.cuda.is_available():
            cls._h2d = torch.cuda.Stream()
        return cls._h2d

    @classmethod
    def d2h_stream(cls):
        if cls._d2h is None and torch.cuda.is_available():
            cls._d2h = torch.cuda.Stream()
        return cls._d2h

    @classmethod
    def is_enabled(cls) -> bool:
        return True

    @classmethod
    def set_delay_stash(cls, delay: bool) -> None:
        """Delay mode queues stashes until ``execute_pending_stashes`` (e.g. fired from a backward-injection hook)."""
        cls._delay = delay

    @classmethod
    def execute_pending_stashes(cls) -> None:
        with cls._lock:
            todo, cls._pending = cls._pending, []
        for fn in todo:
            fn()

    @classmethod
    def thread_submit(cls, fn: Callable[..., Any], *args: Any, **kwargs: Any) -> Future:
        if cls._pool is None:
            cls._pool = ThreadPoolExecutor(max_workers=2, thread_name_prefix="trb-stash")
        return cls._pool.submit(fn, *args, **kwargs)

    @classmethod
    def reset(cls) -> None:
        for key in list(cls._stashes):
            cls._restore(key)
        cls._stashes, cls._pending, cls._delay = {}, [], False

    # ---- core ---------------------------------------------------------------------------------------------------
    @classmethod
    def _stash_tensors(cls, key: str, tensors: List[torch.Tensor]) -> None:
        def run() -> None:
            out: List[_Stash] = []
            for t in tensors:
                if t is None or t.numel() == 0 or t.untyped_storage().nbytes() == 0:
                    continue
                s = _Stash(t)
                flat = torch.empty(0, dtype=torch.uint8, device=t.device).set_(t.untyped_storage(), 0, (s.nbytes,), (1,))
                if t.is_cuda:
                    s.host = torch.empty(s.nbytes, dtype=torch.uint8, pin_memory=True)
                    stream = cls.d2h_stream()
                    stream.wait_stream(torch.cuda.current_stream(t.device))
                    with torch.cuda.stream(stream):
                        s.host.copy_(flat, non_blocking=True)
                        s.event = torch.cuda.Event()
                        s.event.record(stream)
                    s.event.synchronize()  # the storage may only be released once the copy has left the device
                else:
                    s.host = flat.clone()
                t.untyped_storage().resize_(0)
                s.stashed = True
                out.append(s)
            cls._stashes.setdefault(key, []).extend(out)

        if cls._delay:
            with cls._lock:
                cls._pending.append(run)
        else:
            run()

    @classmethod
    def _restore(cls, key: str) -> None:
        for s in cls._stashes.pop(key, []):
            if not s.stashed:
                continue
            t = s.tensor
            t.untyped_storage().resize_(s.nbytes)
            flat = torch.empty(0, dtype=torch.uint8, device=t.device).set_(t.untyped_storage(), 0, (s.nbytes,), (1,))
            if t.is_cuda:
                stream = cls.h2d_stream()
                with torch.cuda.stream(stream):
                    flat.copy_(s.host, non_blocking=True)
                torch.cuda.current_stream(t.device).wait_stream(stream)  # await_restore
            else:
                flat.copy_(s.host)
            s.stashed = False

    @staticmethod
    def _engines(model: nn.Module):
        for m in model.modules():
            eng = getattr(m, "engine", None)
            if eng is not None and hasattr(eng, "_tbes"):
                yield eng

    # ---- public API ----------------------------------------------------------------------------------------------
    @classmethod
    def stash_embedding_weights(cls, model: nn.Module, key: str = "embedding_weights") -> int:
        ts = [tbe.weights.data for eng in cls._engines(model) for tbe in eng._tbes]
        cls._stash_tensors(key, ts)
        return sum(t.numel() * t.element_size() for t in ts)

    @classmethod
    def restore_embedding_weights(cls, key: str = "embedding_weights") -> None:
        cls._restore(key)

    @classmethod
    def stash_optimizer_state(cls, model: nn.Module, key: str = "optimizer_state") -> int:
        ts = [st for eng in cls._engines(model) for tbe in eng._tbes for st in (tbe.state1, tbe.state2) if st is not None]
        cls._stash_tensors(key, ts)
        return sum(t.numel() * t.element_size() for t in ts)

    @classmethod
    def restore_optimizer_state(cls, key: str = "optimizer_state") -> None:
        cls._restore(key)

    @classmethod
    def stash_tensors(cls, key: str, tensors: List[torch.Tensor]) -> None:
        """Generic entry (activations, caches)."""
        cls._stash_tensors(key, tensors)

    @classmethod
    def restore_tensors(cls, key: str) -> None:
        cls._restore(key)

    @classmethod
    def stash_optimizer_state_threaded(cls, model: nn.Module) -> "Future[int]":
        return cls.thread_submit(cls.stash_optimizer_state, model)

    @classmethod
    def restore_optimizer_state_threaded(cls) -> "Future[None]":
        return cls.thread_submit(cls.restore_optimizer_state)

    @classmethod
    def restore_embedding_weights_threaded(cls) -> "Future[None]":
        return cls.thread_submit(cls.restore_embedding_weights)

    @classmethod
    def stashed_bytes(cls) -> int:
        return sum(s.nbytes for v in cls._stashes.values() for s in v if s.stashed)
