"""NVLink peer-memory groups: symmetric buffers + device-side barrier for the fused collectives.

One process per GPU; every rank allocates the same buffer (``cudaMalloc`` in ``csrc/peer_mem.cu``),
exports a CUDA IPC handle, and maps the peers' buffers. Kernels then receive the table of peer
pointers and move data with plain loads/stores over NVSwitch — no NCCL call on the hot path.
NCCL (the process group) is only used to exchange the 64-byte IPC handles.
"""
from __future__ import annotations

import ctypes
import os
import socket
from typing import Dict, List, Optional, Sequence, Tuple

import torch
import torch.distributed as dist

from ..ops import _lib


class _RawArray:
    def __init__(self, ptr: int, nbytes: int) -> None:
        self.__cuda_array_interface__ = {"shape": (nbytes,), "typestr": "|u1", "data": (ptr, False), "version": 3, "strides": None}


def tensor_from_ptr(ptr: int, nbytes: int, device: torch.device) -> torch.Tensor:
    """uint8 tensor aliasing raw device memory (local or peer-mapped)."""
    return torch.as_tensor(_RawArray(ptr, nbytes), device=device)


class SymmetricBuffer:
    """Same-size buffer on every rank; ``ptrs[r]`` is rank r's buffer mapped into this process."""

    def __init__(self, nbytes: int, local_ptr: int, ptrs: List[int], device: torch.device) -> None:
        self.nbytes = nbytes
        self.local_ptr = local_ptr
        self.ptrs = ptrs
        self.device = device
        self._bytes = tensor_from_ptr(local_ptr, nbytes, device)

    def local(self, dtype: torch.dtype, shape: Sequence[int], byte_offset: int = 0) -> torch.Tensor:
        n = 1
        for s in shape:
            n *= s
        nb = n * torch.empty(0, dtype=dtype).element_size()
        return self._bytes[byte_offset : byte_offset + nb].view(dtype).view(*shape)

    def peer_ptrs(self, byte_offset: int = 0) -> List[int]:
        return [p + byte_offset for p in self.ptrs]


class PeerGroup:
    """All ranks of one NVLink domain (one host). Collective construction."""

    _CACHE: Dict[int, "PeerGroup"] = {}

    def __init__(self, pg: dist.ProcessGroup, device: torch.device) -> None:
        self.pg = pg
        self.device = device
        self.world = dist.get_world_size(pg)
        self.rank = dist.get_rank(pg)
        self._lib = _lib.lib()
        self._lib.trb_set_device(device.index if device.index is not None else torch.cuda.current_device())
        self._buffers: List[SymmetricBuffer] = []
        # one signal pad (uint32 flags[W]) + epoch counter per barrier *channel*: collectives that may be in
        # flight concurrently on different streams (input dist vs lookup/output dist) use different channels
        self.N_CHANNELS = 4
        self._pad = self.alloc(256 * self.N_CHANNELS)
        self._epoch = torch.zeros(self.N_CHANNELS, dtype=torch.int32, device=device)
        self._pad_ptr_arrs = [_lib.ptr_array([p + 256 * c for p in self._pad.ptrs]) for c in range(self.N_CHANNELS)]
        for c in range(self.N_CHANNELS):
            self.barrier(c)
        torch.cuda.synchronize(device)

    @staticmethod
    def supported(pg: Optional[dist.ProcessGroup], device: torch.device) -> bool:
        """True when the fused NVLink path can be used: CUDA, NCCL group, <= 16 ranks on ONE host."""
        if os.environ.get("TRB_TRANSPORT", "auto") == "nccl":
            return False
        if pg is None or device.type != "cuda" or not dist.is_initialized():
            return False
        W = dist.get_world_size(pg)
        if W < 2 or W > 16:
            return False
        if dist.get_backend(pg) not in ("nccl", "cpu:gloo,cuda:nccl"):
            return False
        key = id(pg)
        if key in PeerGroup._SUPPORT:
            return PeerGroup._SUPPORT[key]
        info = [None] * W
        dist.all_gather_object(info, (socket.gethostname(), device.index), group=pg)
        ok = len({h for h, _ in info}) == 1 and len({d for _, d in info}) == W
        if ok:
            L = _lib.lib()
            me = device.index if device.index is not None else torch.cuda.current_device()
            ok = all(d == me or L.trb_can_access_peer(me, d) for _, d in info)
        flags = [None] * W
        dist.all_gather_object(flags, bool(ok), group=pg)
        ok = all(flags)
        PeerGroup._SUPPORT[key] = ok
        return ok

    _SUPPORT: Dict[int, bool] = {}

    @staticmethod
    def get(pg: dist.ProcessGroup, device: torch.device) -> "PeerGroup":
        key = id(pg)
        if key not in PeerGroup._CACHE:
            PeerGroup._CACHE[key] = PeerGroup(pg, device)
        return PeerGroup._CACHE[key]

    def alloc(self, nbytes: int) -> SymmetricBuffer:
        """Collective: allocate ``nbytes`` (zeroed) on every rank and map all peers."""
        nbytes = (int(nbytes) + 255) // 256 * 256
        ptr = ctypes.c_void_p(0)
        _lib.check(self._lib.trb_peer_alloc(ctypes.byref(ptr), ctypes.c_size_t(nbytes)), "trb_peer_alloc")
        handle = ctypes.create_string_buffer(64)
        _lib.check(self._lib.trb_ipc_get_handle(ptr, handle), "trb_ipc_get_handle")
        handles: List[Optional[bytes]] = [None] * self.world
        dist.all_gather_object(handles, bytes(handle.raw), group=self.pg)
        ptrs: List[int] = []
        for r, h in enumerate(handles):
            if r == self.rank:
                ptrs.append(int(ptr.value))
                continue
            out = ctypes.c_void_p(0)
            hb = ctypes.create_string_buffer(h, 64)
            _lib.check(self._lib.trb_ipc_open_handle(hb, ctypes.byref(out)), f"trb_ipc_open_handle(rank {r})")
            ptrs.append(int(out.value))
        buf = SymmetricBuffer(nbytes, int(ptr.value), ptrs, self.device)
        self._buffers.append(buf)
        dist.barrier(group=self.pg)
        return buf

    def barrier(self, channel: int = 0) -> None:
        """Device-side barrier of all ranks on the current stream (graph capturable)."""
        code = self._lib.trb_barrier(self._pad_ptr_arrs[channel], self.world, self.rank, ctypes.c_void_p(self._epoch.data_ptr() + 4 * channel),
                                     _lib.stream_ptr(self.device))
        _lib.check(code, "trb_barrier")


def cast_copy(src: torch.Tensor, dst: torch.Tensor, scale: float = 1.0) -> None:
    """dst[r, c] = cast(src[r, c] * scale) for 2-D row-major tensors (native kernel)."""
    assert src.dim() == 2 and dst.shape == src.shape and src.stride(1) == 1 and dst.stride(1) == 1
    L = _lib.lib()
    code = L.trb_cast_copy(_lib.ptr(src), _lib.dtype_code(src.dtype), _lib.ptr(dst), _lib.dtype_code(dst.dtype), ctypes.c_int64(src.shape[0]),
                           src.shape[1], ctypes.c_int64(src.stride(0)), ctypes.c_int64(dst.stride(0)), ctypes.c_float(scale), _lib.stream_ptr(src.device))
    _lib.check(code, "trb_cast_copy")


def staging_reduce(staging: torch.Tensor, out: torch.Tensor, col_mask: torch.Tensor, W: int) -> None:
    """out[b, c] = sum over ranks j with bit j of col_mask[c] set of staging[j, b, c]."""
    Wd, B, C = staging.shape
    L = _lib.lib()
    code = L.trb_staging_reduce(_lib.ptr(staging), _lib.dtype_code(staging.dtype), _lib.ptr(out), _lib.dtype_code(out.dtype), _lib.ptr(col_mask), B, C,
                                ctypes.c_int64(staging.stride(1)), ctypes.c_int64(out.stride(0)), ctypes.c_int64(staging.stride(0)), W,
                                _lib.stream_ptr(out.device))
    _lib.check(code, "trb_staging_reduce")


def grad_push(src: torch.Tensor, chunks: torch.Tensor, dst_ptrs: List[int], dst_dtype: torch.dtype, dst_pitch: int, row_base: int, scale: float = 1.0, vec: int = 4) -> None:
    """Scatter column chunks of ``src [B_local, cols]`` into the owners' gradient inboxes (native kernel ``trb_grad_push``).
    ``chunks``: int32 ``[n, 3]`` rows of (destination rank, source column, destination column), ``vec`` (4 or 8) elements per chunk."""
    assert src.dim() == 2 and src.stride(1) == 1 and chunks.dtype == torch.int32 and chunks.is_contiguous()
    L = _lib.lib()
    code = L.trb_grad_push(_lib.ptr(src), _lib.dtype_code(src.dtype), ctypes.c_int64(src.stride(0)), _lib.ptr(chunks), chunks.shape[0], int(vec), _lib.ptr_array(dst_ptrs), len(dst_ptrs),
                           _lib.dtype_code(dst_dtype), ctypes.c_int64(dst_pitch), ctypes.c_int64(row_base), src.shape[0], ctypes.c_float(scale), _lib.stream_ptr(src.device))
    _lib.check(code, "trb_grad_push")


def grad_push_fp8(src: torch.Tensor, chunks: torch.Tensor, row_dim: int, dst_ptrs: List[int], scale_ptrs: List[int], dst_pitch: int, scale_pitch: int,
                  row_base: int) -> None:
    """FP8 variant of ``grad_push`` (native kernel ``trb_grad_push_fp8``): every chunk is a group of ``row_dim`` columns, stored as e4m3
    payload into ``dst_ptrs`` (uint8 rows of ``dst_pitch`` bytes) and one fp32 scale into ``scale_ptrs`` (rows of ``scale_pitch`` scales)."""
    assert src.dim() == 2 and src.stride(1) == 1 and chunks.dtype == torch.int32 and chunks.is_contiguous()
    L = _lib.lib()
    code = L.trb_grad_push_fp8(_lib.ptr(src), _lib.dtype_code(src.dtype), ctypes.c_int64(src.stride(0)), _lib.ptr(chunks), chunks.shape[0], int(row_dim),
                               _lib.ptr_array(dst_ptrs), _lib.ptr_array(scale_ptrs), len(dst_ptrs), ctypes.c_int64(dst_pitch), ctypes.c_int64(scale_pitch),
                               ctypes.c_int64(row_base), src.shape[0], _lib.stream_ptr(src.device))
    _lib.check(code, "trb_grad_push_fp8")


def fp8_wire_decode(payload_ptr: int, pay_pitch: int, scale_ptr: int, scale_pitch: int, row_dim: int, cols: torch.Tensor, rows: int, out: torch.Tensor) -> None:
    """``out[r, c : c + 16]`` = FP8 payload + scales decoded to ``out.dtype``, for every 16-column chunk start ``c`` in ``cols`` (int32)."""
    assert out.stride(1) == 1 and cols.dtype == torch.int32
    L = _lib.lib()
    code = L.trb_fp8_wire_decode(ctypes.c_void_p(payload_ptr), ctypes.c_int64(pay_pitch), ctypes.c_void_p(scale_ptr), ctypes.c_int64(scale_pitch), int(row_dim),
                                 _lib.ptr(cols), cols.numel(), ctypes.c_int64(rows), _lib.ptr(out), _lib.dtype_code(out.dtype), ctypes.c_int64(out.stride(0)),
                                 _lib.stream_ptr(out.device))
    _lib.check(code, "trb_fp8_wire_decode")
