"""ctypes loader for the sm_90a kernel library (``torchrec_b200/ops/_lib/libtrb200_ops.so``).

The CUDA path is the product: on a machine with a GPU a missing / unloadable library raises
immediately (no silent PyTorch fallback). On a CPU-only machine every op runs its PyTorch
reference implementation (used by the gloo unit tests).
"""
from __future__ import annotations

import ctypes
import os
import threading
from typing import Optional, Sequence

import torch

_LOCK = threading.Lock()
_LIB: Optional[ctypes.CDLL] = None
_TRIED = False

F32, F16, BF16, U8, I32, I64, FP8 = 0, 1, 2, 3, 4, 5, 6

_DTYPE_CODE = {
    torch.float32: F32,
    torch.float16: F16,
    torch.bfloat16: BF16,
    torch.uint8: U8,
    torch.int32: I32,
    torch.int64: I64,
}


def dtype_code(dt: torch.dtype) -> int:
    return _DTYPE_CODE[dt]


class KernelLibraryError(RuntimeError):
    pass


def _load() -> Optional[ctypes.CDLL]:
    global _LIB, _TRIED
    if _TRIED:
        return _LIB
    with _LOCK:
        if _TRIED:
            return _LIB
        from . import build as _build

        path = _build.lib_path()
        if not os.path.exists(path) and os.environ.get("TRB200_NO_AUTOBUILD", "0") != "1":
            try:
                _build.build()
            except Exception as e:  # pragma: no cover - depends on toolchain
                if torch.cuda.is_available():
                    raise KernelLibraryError(f"cannot build the sm_90a kernel library: {e}") from e
        if os.path.exists(path):
            try:
                _LIB = ctypes.CDLL(path, mode=ctypes.RTLD_GLOBAL)
            except OSError as e:
                if torch.cuda.is_available():
                    raise KernelLibraryError(f"cannot load {path}: {e}") from e
                _LIB = None
        elif torch.cuda.is_available():
            raise KernelLibraryError(
                f"{path} is missing; run `python -m torchrec_b200.ops.build` (the CUDA path has no fallback)"
            )
        _TRIED = True
        return _LIB


def lib() -> ctypes.CDLL:
    """Return the loaded kernel library or raise (used by every CUDA code path)."""
    l = _load()
    if l is None:
        raise KernelLibraryError("torchrec_b200 kernel library is not available")
    return l


def available() -> bool:
    try:
        return _load() is not None
    except KernelLibraryError:
        return False


def use_cuda_kernels(*tensors: torch.Tensor) -> bool:
    """True when the tensors live on a CUDA device (then the native kernel MUST be used)."""
    for t in tensors:
        if t is not None and t.is_cuda:
            lib()  # raises loudly if the extension is missing on a GPU box
            return True
    return False


def ptr(t: Optional[torch.Tensor]) -> ctypes.c_void_p:
    if t is None:
        return ctypes.c_void_p(0)
    return ctypes.c_void_p(t.data_ptr())


_raw_stream = getattr(torch._C, "_cuda_getCurrentRawStream", None)


def stream_ptr(device: Optional[torch.device] = None) -> ctypes.c_void_p:
    """cudaStream_t of the current stream of ``device``. ~30 calls per train step: use the raw C accessor (no Stream object,
    no device-index normalisation in Python) when this torch build has it."""
    if _raw_stream is not None:
        idx = device.index if device is not None and device.index is not None else torch.cuda.current_device()
        return ctypes.c_void_p(_raw_stream(idx))
    return ctypes.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def ptr_array(ptrs: Sequence[int]):
    arr = (ctypes.c_void_p * len(ptrs))()
    for i, p in enumerate(ptrs):
        arr[i] = p
    return arr


def check(code: int, what: str) -> None:
    if code != 0:
        if code > 0:
            raise KernelLibraryError(f"{what}: CUDA error {code}")
        raise KernelLibraryError(f"{what}: library error {code}")


def launch_count() -> int:
    l = _load()
    if l is None:
        return 0
    l.trb_launch_count.restype = ctypes.c_ulonglong
    return int(l.trb_launch_count())


def launch_count_add(n: int) -> None:
    l = _load()
    if l is not None:
        l.trb_launch_count_add(ctypes.c_ulonglong(n))


def add_launches(n: int) -> None:
    """Account for native kernels replayed by a CUDA graph (the host-side launch counter only sees the capture)."""
    if n > 0 and available():
        lib().trb_launch_count_add(ctypes.c_ulonglong(int(n)))
