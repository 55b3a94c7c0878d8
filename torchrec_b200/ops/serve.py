"""Launcher of ``csrc/serve_ingest.cu``: one server batch slab, already on the device, into the static inputs of a graph bucket.

``ingest`` takes the device copy of the slab the batching core packed, a device descriptor of the batch (``inference/graphed.py:
pack_desc``) and the bucket's buffers (``IngestBuffers``), and fills the buffers in one launch whose shape depends on the bucket only,
so it can be captured in a CUDA graph and replayed for every batch that fits. There is no CPU implementation: the buffers feed a CUDA
graph."""
from __future__ import annotations

import ctypes
from dataclasses import dataclass
from typing import Optional

import torch

from . import _lib


@dataclass
class IngestBuffers:
    """Static inputs of one bucket ``(B_cap, nnz_cap)``. A list with no features, and ``dense`` without float features, are None."""

    B_cap: int
    nnz_cap: int
    dense: Optional[torch.Tensor]        # fp32 [B_cap, num_float]
    idl_lengths: Optional[torch.Tensor]  # int32 [F1 * B_cap]
    idl_offsets: Optional[torch.Tensor]  # int32 / int64 [F1 * B_cap + 1]
    idl_values: Optional[torch.Tensor]   # int64 [nnz_cap]
    ids_lengths: Optional[torch.Tensor]
    ids_offsets: Optional[torch.Tensor]
    ids_values: Optional[torch.Tensor]
    ids_weights: Optional[torch.Tensor]  # fp32 [nnz_cap]

    @staticmethod
    def allocate(B_cap: int, nnz_cap: int, num_float: int, F_idl: int, F_ids: int, offsets_dtype: torch.dtype, device: torch.device) -> "IngestBuffers":
        def lists(F: int, weighted: bool):
            if not F:
                return None, None, None, None
            return (torch.zeros(F * B_cap, dtype=torch.int32, device=device), torch.zeros(F * B_cap + 1, dtype=offsets_dtype, device=device),
                    torch.zeros(nnz_cap, dtype=torch.int64, device=device), torch.zeros(nnz_cap, dtype=torch.float32, device=device) if weighted else None)

        l1, o1, v1, _ = lists(F_idl, False)
        l2, o2, v2, w2 = lists(F_ids, True)
        dense = torch.zeros(B_cap, num_float, dtype=torch.float32, device=device) if num_float else None
        return IngestBuffers(B_cap, nnz_cap, dense, l1, o1, v1, l2, o2, v2, w2)

    def view(self, B_cap: int, nnz_cap: int) -> "IngestBuffers":
        """The buffers of a smaller bucket in the front of these (buckets whose graphs never run at the same time share storage)."""
        assert B_cap <= self.B_cap and nnz_cap <= self.nnz_cap

        def front(t: Optional[torch.Tensor], n: int) -> Optional[torch.Tensor]:
            return t[:n] if t is not None else None

        F1 = self.idl_lengths.numel() // self.B_cap if self.idl_lengths is not None else 0
        F2 = self.ids_lengths.numel() // self.B_cap if self.ids_lengths is not None else 0
        return IngestBuffers(B_cap, nnz_cap, self.dense[:B_cap] if self.dense is not None else None, front(self.idl_lengths, F1 * B_cap),
                             front(self.idl_offsets, F1 * B_cap + 1), front(self.idl_values, nnz_cap), front(self.ids_lengths, F2 * B_cap),
                             front(self.ids_offsets, F2 * B_cap + 1), front(self.ids_values, nnz_cap), front(self.ids_weights, nnz_cap))


def desc_fields() -> int:
    return int(_lib.lib().trb_serve_ingest_desc_fields())


def ingest(slab: torch.Tensor, desc: torch.Tensor, buf: IngestBuffers, num_float: int, F_idl: int, F_ids: int, error: torch.Tensor) -> None:
    """Fill ``buf`` from the batch described by ``desc`` (device int64 ``[desc_fields()]``) in ``slab`` (device uint8). A batch that does
    not fit the bucket sets ``error[0] = 1`` (int32, device or pinned host memory) and writes nothing; the flag is never cleared here."""
    assert slab.is_cuda and slab.dtype == torch.uint8 and desc.is_cuda and desc.dtype == torch.int64, "ingest runs on the device"
    offsets = buf.idl_offsets if buf.idl_offsets is not None else buf.ids_offsets
    off64 = int(offsets is not None and offsets.dtype == torch.int64)
    code = _lib.lib().trb_serve_ingest(
        _lib.ptr(slab), ctypes.c_int64(slab.numel()), _lib.ptr(desc), int(buf.B_cap), ctypes.c_int64(buf.nnz_cap), int(num_float), int(F_idl), int(F_ids),
        _lib.ptr(buf.dense), _lib.ptr(buf.idl_lengths), _lib.ptr(buf.idl_offsets), _lib.ptr(buf.idl_values), _lib.ptr(buf.ids_lengths),
        _lib.ptr(buf.ids_offsets), _lib.ptr(buf.ids_values), _lib.ptr(buf.ids_weights), off64, _lib.ptr(error), _lib.stream_ptr(slab.device))
    _lib.check(code, "trb_serve_ingest")
