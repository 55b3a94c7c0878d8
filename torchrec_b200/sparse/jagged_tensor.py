"""Jagged data types: ``JaggedTensor``, ``KeyedJaggedTensor`` (KJT), ``KeyedTensor`` (KT).

Same user contract as the reference (torchrec/sparse/jagged_tensor.py:634,1909,3503): KJT stores a
multi-feature ragged batch with key-major values and ``[F x B]`` lengths, lazily caches
``length_per_key`` / ``offset_per_key``, supports variable batch per feature (VBE) through
``stride_per_key_per_rank`` + ``inverse_indices``, and exposes the ``dist_*`` hooks the input
all-to-all uses. The implementation is new: all jagged math goes through
``torchrec_b200.ops.jagged`` (sm_90a kernels on CUDA, PyTorch on CPU).
"""
from __future__ import annotations

import abc
import operator
from typing import Any, Dict, List, Optional, Sequence, Tuple, Union

import torch
from torch.utils._pytree import register_pytree_node

from ..ops import jagged as J
from ..streamable import Pipelineable


def _cumsum_list(xs: Sequence[int]) -> List[int]:
    out, c = [0], 0
    for x in xs:
        c += int(x)
        out.append(c)
    return out


def _to_offsets(lengths: torch.Tensor) -> torch.Tensor:
    return J.asynchronous_complete_cumsum(lengths.view(-1))


def _to_lengths(offsets: torch.Tensor) -> torch.Tensor:
    return offsets[1:] - offsets[:-1]


def _maybe_compute_lengths(lengths: Optional[torch.Tensor], offsets: Optional[torch.Tensor]) -> torch.Tensor:
    if lengths is None:
        assert offsets is not None
        lengths = _to_lengths(offsets)
    return lengths


def _maybe_compute_offsets(lengths: Optional[torch.Tensor], offsets: Optional[torch.Tensor]) -> torch.Tensor:
    if offsets is None:
        assert lengths is not None
        offsets = _to_offsets(lengths)
    return offsets


def _get_weights_or_throw(weights: Optional[torch.Tensor]) -> torch.Tensor:
    assert weights is not None, "This (Keyed)JaggedTensor doesn't have weights."
    return weights


def _get_lengths_offset_per_key_or_throw(x: Optional[List[int]]) -> List[int]:
    assert x is not None, "This (Keyed)JaggedTensor doesn't have lengths_offset_per_key."
    return x


def _get_stride_per_key_or_throw(x: Optional[List[int]]) -> List[int]:
    assert x is not None, "This (Keyed)JaggedTensor doesn't have stride_per_key."
    return x


def _get_inverse_indices_or_throw(x: Optional[Tuple[List[str], torch.Tensor]]) -> Tuple[List[str], torch.Tensor]:
    assert x is not None, "This KJT doesn't have inverse indices."
    return x


def _assert_offsets_or_lengths_is_provided(offsets, lengths) -> None:
    assert offsets is not None or lengths is not None, "Must provide lengths or offsets"


def _sum_by_splits(values: List[int], splits: List[int]) -> List[int]:
    out, i = [], 0
    for s in splits:
        out.append(sum(values[i : i + s]))
        i += s
    return out


def _pin_and_move(t: torch.Tensor, device: torch.device) -> torch.Tensor:
    if t.device == device:
        return t
    if device.type == "cuda" and t.device.type == "cpu":
        return t.pin_memory().to(device, non_blocking=True)
    return t.to(device)


# ---------------------------------------------------------------------------------------------
class JaggedTensorMeta(abc.ABCMeta, torch.fx._symbolic_trace.ProxyableClassMeta):
    """Constructing a JaggedTensor / KeyedJaggedTensor / KeyedTensor from fx proxies inside a symbolic trace records a node instead of
    failing (reference jagged_tensor.py:630). Outside a trace construction is the plain one (one module-flag read per call)."""

    def __call__(cls, *args, **kwargs):
        if not torch.fx._symbolic_trace._is_fx_tracing_flag:
            return type.__call__(cls, *args, **kwargs)
        return torch.fx._symbolic_trace.ProxyableClassMeta.__call__(cls, *args, **kwargs)


class JaggedTensor(Pipelineable, metaclass=JaggedTensorMeta):
    """A tensor with one jagged dimension: ``values`` [sum L (, D)] + ``lengths`` / ``offsets`` [B]."""

    _fields = ["_values", "_weights", "_lengths", "_offsets"]

    def __init__(
        self,
        values: torch.Tensor,
        weights: Optional[torch.Tensor] = None,
        lengths: Optional[torch.Tensor] = None,
        offsets: Optional[torch.Tensor] = None,
    ) -> None:
        self._values = values
        self._weights = weights
        _assert_offsets_or_lengths_is_provided(offsets, lengths)
        if offsets is not None:
            assert offsets.dim() == 1, "offsets must be 1-D"
        if lengths is not None:
            assert lengths.dim() == 1, "lengths must be 1-D"
        self._lengths = lengths
        self._offsets = offsets

    @staticmethod
    def empty(is_weighted: bool = False, device: Optional[torch.device] = None, values_dtype: Optional[torch.dtype] = None,
              weights_dtype: Optional[torch.dtype] = None, lengths_dtype: torch.dtype = torch.int32) -> "JaggedTensor":
        weights = torch.empty(0, dtype=weights_dtype, device=device) if is_weighted else None
        return JaggedTensor(
            values=torch.empty(0, dtype=values_dtype, device=device),
            offsets=torch.empty(0, dtype=lengths_dtype, device=device),
            lengths=torch.empty(0, dtype=lengths_dtype, device=device),
            weights=weights,
        )

    @staticmethod
    def from_dense_lengths(values: torch.Tensor, lengths: torch.Tensor, weights: Optional[torch.Tensor] = None) -> "JaggedTensor":
        """Build from a padded ``[B, N(, D)]`` tensor and per-row lengths."""
        mask = torch.arange(values.size(1), device=values.device).view(1, -1) < lengths.view(-1, 1)
        return JaggedTensor(values=values[mask], weights=weights[mask] if weights is not None else None, lengths=lengths)

    @staticmethod
    def from_dense(values: List[torch.Tensor], weights: Optional[List[torch.Tensor]] = None) -> "JaggedTensor":
        lengths = torch.tensor([v.size(0) for v in values], dtype=torch.int32, device=values[0].device if values else None)
        return JaggedTensor(
            values=torch.cat(values, 0),
            weights=torch.cat(weights, 0) if weights is not None else None,
            lengths=lengths,
            offsets=_to_offsets(lengths),
        )

    def to_dense(self) -> List[torch.Tensor]:
        off = self.offsets().tolist()
        return [self._values[off[i] : off[i + 1]] for i in range(len(off) - 1)]

    def to_dense_weights(self) -> Optional[List[torch.Tensor]]:
        if self._weights is None:
            return None
        off = self.offsets().tolist()
        return [self._weights[off[i] : off[i + 1]] for i in range(len(off) - 1)]

    def to_padded_dense(self, desired_length: Optional[int] = None, padding_value: float = 0.0) -> torch.Tensor:
        if desired_length is None:
            desired_length = int(self.lengths().max()) if self.lengths().numel() else 0
        return J.jagged_to_padded_dense(self._values, [self.offsets()], [desired_length], padding_value)

    def to_padded_dense_weights(self, desired_length: Optional[int] = None, padding_value: float = 0.0) -> Optional[torch.Tensor]:
        if self._weights is None:
            return None
        if desired_length is None:
            desired_length = int(self.lengths().max()) if self.lengths().numel() else 0
        return J.jagged_to_padded_dense(self._weights, [self.offsets()], [desired_length], padding_value)

    def device(self) -> torch.device:
        return self._values.device

    def lengths(self) -> torch.Tensor:
        self._lengths = _maybe_compute_lengths(self._lengths, self._offsets)
        return self._lengths

    def lengths_or_none(self) -> Optional[torch.Tensor]:
        return self._lengths

    def offsets(self) -> torch.Tensor:
        self._offsets = _maybe_compute_offsets(self._lengths, self._offsets)
        return self._offsets

    def offsets_or_none(self) -> Optional[torch.Tensor]:
        return self._offsets

    def values(self) -> torch.Tensor:
        return self._values

    def weights(self) -> torch.Tensor:
        return _get_weights_or_throw(self._weights)

    def weights_or_none(self) -> Optional[torch.Tensor]:
        return self._weights

    def to(self, device: torch.device, non_blocking: bool = False) -> "JaggedTensor":
        mv = lambda t: None if t is None else t.to(device, non_blocking=non_blocking)
        return JaggedTensor(values=mv(self._values), weights=mv(self._weights), lengths=mv(self._lengths), offsets=mv(self._offsets))

    def record_stream(self, stream: torch.Stream) -> None:
        for t in (self._values, self._weights, self._lengths, self._offsets):
            if t is not None and t.is_cuda:
                t.record_stream(stream)

    def __str__(self) -> str:
        off = self.offsets().tolist()
        vals = self._values.tolist()
        rows = [vals[off[i] : off[i + 1]] for i in range(len(off) - 1)]
        s = "JaggedTensor({\n    " + repr(rows) + "\n"
        if self._weights is not None:
            w = self._weights.tolist()
            s += '    "weights": ' + repr([w[off[i] : off[i + 1]] for i in range(len(off) - 1)]) + "\n"
        return s + "})\n"


def _jt_flatten(t: JaggedTensor):
    return [getattr(t, a) for a in JaggedTensor._fields], None


def _jt_unflatten(values, context) -> JaggedTensor:
    return JaggedTensor(*values)


register_pytree_node(JaggedTensor, _jt_flatten, _jt_unflatten, serialized_type_name="torchrec_b200.sparse.JaggedTensor")


# ---------------------------------------------------------------------------------------------
def _permute_tensor_by_segments(tensor: torch.Tensor, segment_sizes: torch.Tensor, recat: torch.Tensor,
                                weights: Optional[torch.Tensor] = None, output_size: Optional[int] = None):
    lengths, values, w = J.permute_1D_sparse_data(recat, segment_sizes, tensor, weights, output_size)
    return values, w


_PERM_INDEX_CACHE: Dict[Tuple[Tuple[int, ...], str], torch.Tensor] = {}


def _perm_index_tensor(indices: List[int], device: torch.device) -> torch.Tensor:
    """int32 device copy of a key permutation, cached per (permutation, device): ``torch.tensor(list, device="cuda")`` is a
    pageable H2D copy followed by a stream synchronize, i.e. one full host/GPU sync per KJT permute in a train step."""
    key = (tuple(indices), str(device))
    t = _PERM_INDEX_CACHE.get(key)
    if t is None:
        if len(_PERM_INDEX_CACHE) > 4096:
            _PERM_INDEX_CACHE.clear()
        with torch.inference_mode(False):  # cached: a serving call under inference_mode must not poison later training calls
            t = _PERM_INDEX_CACHE[key] = torch.tensor(indices, dtype=torch.int32, device=device)
    return t


class KeyedJaggedTensor(Pipelineable, metaclass=JaggedTensorMeta):
    """Multi-feature jagged batch (see module docstring). Layout: values are key-major; lengths are
    ``[F * B]`` (or a per-key variable batch when ``stride_per_key_per_rank`` is given)."""

    _fields = ["_values", "_weights", "_lengths", "_offsets"]

    def __init__(
        self,
        keys: List[str],
        values: torch.Tensor,
        weights: Optional[torch.Tensor] = None,
        lengths: Optional[torch.Tensor] = None,
        offsets: Optional[torch.Tensor] = None,
        stride: Optional[int] = None,
        stride_per_key_per_rank: Optional[Union[torch.Tensor, List[List[int]]]] = None,
        stride_per_rank: Optional[List[int]] = None,
        stride_per_key: Optional[List[int]] = None,
        length_per_key: Optional[List[int]] = None,
        lengths_offset_per_key: Optional[List[int]] = None,
        offset_per_key: Optional[List[int]] = None,
        index_per_key: Optional[Dict[str, int]] = None,
        jt_dict: Optional[Dict[str, JaggedTensor]] = None,
        inverse_indices: Optional[Tuple[List[str], torch.Tensor]] = None,
    ) -> None:
        self._keys: List[str] = list(keys)
        self._values = values
        self._weights = weights
        if offsets is not None:
            assert offsets.dim() == 1
        if lengths is not None:
            assert lengths.dim() == 1
        self._lengths = lengths
        self._offsets = offsets
        self._stride_per_key_per_rank: Optional[torch.Tensor] = None
        self._stride_per_rank = stride_per_rank
        self._variable_stride_per_key = False
        if stride_per_key_per_rank is not None:
            spkpr = stride_per_key_per_rank if isinstance(stride_per_key_per_rank, torch.Tensor) else torch.tensor(
                stride_per_key_per_rank, dtype=torch.int64).view(len(keys), -1) if len(stride_per_key_per_rank) else torch.zeros(0, 0, dtype=torch.int64)
            self._stride_per_key_per_rank = spkpr.cpu()
            self._variable_stride_per_key = True
        self._stride: Optional[int] = stride
        self._length_per_key = length_per_key
        self._offset_per_key = offset_per_key
        self._index_per_key = index_per_key
        self._jt_dict = jt_dict
        self._inverse_indices = inverse_indices
        self._lengths_offset_per_key: Optional[List[int]] = lengths_offset_per_key
        self._stride_per_key: Optional[List[int]] = stride_per_key  # pre-computed caches handed over by a caller that already has them

    # ---- constructors -----------------------------------------------------------------------
    @staticmethod
    def from_offsets_sync(keys, values, offsets, weights=None, stride=None, stride_per_key_per_rank=None, inverse_indices=None) -> "KeyedJaggedTensor":
        return KeyedJaggedTensor(keys=keys, values=values, weights=weights, offsets=offsets, stride=stride,
                                 stride_per_key_per_rank=stride_per_key_per_rank, inverse_indices=inverse_indices).sync()

    @staticmethod
    def from_lengths_sync(keys, values, lengths, weights=None, stride=None, stride_per_key_per_rank=None, inverse_indices=None) -> "KeyedJaggedTensor":
        return KeyedJaggedTensor(keys=keys, values=values, weights=weights, lengths=lengths, stride=stride,
                                 stride_per_key_per_rank=stride_per_key_per_rank, inverse_indices=inverse_indices).sync()

    @staticmethod
    def concat(kjt_list: List["KeyedJaggedTensor"]) -> "KeyedJaggedTensor":
        if len(kjt_list) == 0:
            raise ValueError("Can't concat empty KJT list")
        is_weighted = kjt_list[0].weights_or_none() is not None
        has_length_per_key = True
        length_per_key: List[int] = []
        keys: List[str] = []
        value_list, weight_list, length_list = [], [], []
        stride_per_key_per_rank: List[List[int]] = []
        variable = kjt_list[0].variable_stride_per_key()
        stride = None
        for kjt in kjt_list:
            assert (kjt.weights_or_none() is not None) == is_weighted, "Can't merge weighted KJT with unweighted KJT"
            assert kjt.variable_stride_per_key() == variable
            if kjt._length_per_key is None:
                has_length_per_key = False
            if has_length_per_key:
                length_per_key += kjt._length_per_key
            keys += kjt.keys()
            value_list.append(kjt.values())
            if is_weighted:
                weight_list.append(kjt.weights())
            length_list.append(kjt.lengths())
            if variable:
                stride_per_key_per_rank += kjt.stride_per_key_per_rank()
            else:
                if stride is None:
                    stride = kjt.stride()
                assert stride == kjt.stride(), "Can only merge KJTs of the same stride"
        return KeyedJaggedTensor(
            keys=keys,
            values=torch.cat(value_list, 0),
            weights=torch.cat(weight_list, 0) if is_weighted else None,
            lengths=torch.cat(length_list, 0),
            stride=None if variable else stride,
            stride_per_key_per_rank=stride_per_key_per_rank if variable else None,
            length_per_key=length_per_key if has_length_per_key else None,
        )

    @staticmethod
    def empty(is_weighted: bool = False, device: Optional[torch.device] = None, values_dtype=None, weights_dtype=None, lengths_dtype=torch.int32) -> "KeyedJaggedTensor":
        weights = torch.empty(0, dtype=weights_dtype, device=device) if is_weighted else None
        return KeyedJaggedTensor(keys=[], values=torch.empty(0, dtype=values_dtype, device=device), weights=weights,
                                 lengths=torch.empty(0, dtype=lengths_dtype, device=device), stride=0)

    @staticmethod
    def empty_like(kjt: "KeyedJaggedTensor") -> "KeyedJaggedTensor":
        return KeyedJaggedTensor(
            keys=[], values=torch.empty(0, device=kjt.device(), dtype=kjt.values().dtype),
            weights=None if kjt.weights_or_none() is None else torch.empty(0, device=kjt.device(), dtype=kjt.weights().dtype),
            lengths=torch.empty(0, device=kjt.device(), dtype=kjt.lengths().dtype),
            stride=None if kjt.variable_stride_per_key() else kjt.stride(),
            stride_per_key_per_rank=[] if kjt.variable_stride_per_key() else None,
        )

    @staticmethod
    def from_jt_dict(jt_dict: Dict[str, JaggedTensor]) -> "KeyedJaggedTensor":
        keys = list(jt_dict.keys())
        if not keys:
            return KeyedJaggedTensor.empty()
        jts = [jt_dict[k] for k in keys]
        strides = [jt.lengths().numel() for jt in jts]
        weighted = jts[0].weights_or_none() is not None
        return KeyedJaggedTensor(
            keys=keys,
            values=torch.cat([jt.values() for jt in jts]),
            weights=torch.cat([jt.weights() for jt in jts]) if weighted else None,
            lengths=torch.cat([jt.lengths() for jt in jts]),
            stride=strides[0] if len(set(strides)) == 1 else None,
            stride_per_key_per_rank=None if len(set(strides)) == 1 else [[s] for s in strides],
        ).sync()

    # ---- cached metadata ---------------------------------------------------------------------
    def sync(self) -> "KeyedJaggedTensor":
        if not torch.jit.is_scripting():
            self.length_per_key()
            self.offset_per_key()
        return self

    def unsync(self) -> "KeyedJaggedTensor":
        self._length_per_key = None
        self._offset_per_key = None
        return self

    def device(self) -> torch.device:
        return self._values.device

    def lengths(self) -> torch.Tensor:
        self._lengths = _maybe_compute_lengths(self._lengths, self._offsets)
        return self._lengths

    def lengths_or_none(self) -> Optional[torch.Tensor]:
        return self._lengths

    def offsets(self) -> torch.Tensor:
        self._offsets = _maybe_compute_offsets(self._lengths, self._offsets)
        return self._offsets

    def offsets_or_none(self) -> Optional[torch.Tensor]:
        return self._offsets

    def keys(self) -> List[str]:
        return self._keys

    def values(self) -> torch.Tensor:
        return self._values

    def weights(self) -> torch.Tensor:
        return _get_weights_or_throw(self._weights)

    def weights_or_none(self) -> Optional[torch.Tensor]:
        return self._weights

    def stride(self) -> int:
        if self._stride is None:
            if self._variable_stride_per_key:
                spk = self.stride_per_key()
                self._stride = max(spk) if spk else 0
            elif self._stride_per_rank is not None:
                self._stride = sum(self._stride_per_rank)
            else:
                n = len(self._keys)
                if n == 0:
                    self._stride = 0
                elif self._offsets is not None and self._offsets.numel() > 0:
                    self._stride = (self._offsets.numel() - 1) // n
                elif self._lengths is not None:
                    self._stride = self._lengths.numel() // n
                else:
                    self._stride = 0
        return self._stride

    def stride_per_key(self) -> List[int]:
        if self._stride_per_key is not None:
            return self._stride_per_key
        if self._stride_per_key_per_rank is not None:
            return self._stride_per_key_per_rank.sum(dim=1).tolist() if self._stride_per_key_per_rank.numel() else []
        return [self.stride()] * len(self._keys)

    def stride_per_key_per_rank(self) -> List[List[int]]:
        if self._stride_per_key_per_rank is None:
            return []
        return self._stride_per_key_per_rank.tolist()

    def variable_stride_per_key(self) -> bool:
        return self._variable_stride_per_key

    def inverse_indices(self) -> Tuple[List[str], torch.Tensor]:
        return _get_inverse_indices_or_throw(self._inverse_indices)

    def inverse_indices_or_none(self) -> Optional[Tuple[List[str], torch.Tensor]]:
        return self._inverse_indices

    def _key_indices(self) -> Dict[str, int]:
        if self._index_per_key is None:
            self._index_per_key = {k: i for i, k in enumerate(self._keys)}
        return self._index_per_key

    def lengths_offset_per_key(self) -> List[int]:
        if self._lengths_offset_per_key is None:
            self._lengths_offset_per_key = _cumsum_list(self.stride_per_key())
        return self._lengths_offset_per_key

    def length_per_key(self) -> List[int]:
        """Number of values of each key — reads the device once and caches (host sync point, as in
        the reference jagged_tensor.py:1382-1391)."""
        if self._length_per_key is None:
            if len(self._keys) == 0:
                self._length_per_key = []
            elif self._variable_stride_per_key:
                lo = self.lengths_offset_per_key()
                csum = torch.cat([self.lengths().new_zeros(1), torch.cumsum(self.lengths(), 0)])
                tot = csum[torch.tensor(lo, device=csum.device)]
                self._length_per_key = (tot[1:] - tot[:-1]).tolist()
            else:
                self._length_per_key = self.lengths().view(len(self._keys), -1).sum(dim=1).tolist()
        return self._length_per_key

    def length_per_key_or_none(self) -> Optional[List[int]]:
        return self._length_per_key

    def offset_per_key(self) -> List[int]:
        if self._offset_per_key is None:
            self._offset_per_key = _cumsum_list(self.length_per_key())
        return self._offset_per_key

    def offset_per_key_or_none(self) -> Optional[List[int]]:
        return self._offset_per_key

    # ---- structure ops -----------------------------------------------------------------------
    def split(self, segments: List[int]) -> List["KeyedJaggedTensor"]:
        """Split by consecutive groups of keys (views into the same storage)."""
        split_list: List[KeyedJaggedTensor] = []
        start = 0
        start_offset = 0
        _length_per_key = self.length_per_key()
        _offset_per_key = self.offset_per_key()
        lo = self.lengths_offset_per_key()
        for segment in segments:
            end = start + segment
            end_offset = _offset_per_key[end]
            keys = self._keys[start:end]
            spkpr = None
            if self._variable_stride_per_key:
                spkpr = self._stride_per_key_per_rank[start:end]
            if segment == 0:
                split_list.append(KeyedJaggedTensor(
                    keys=keys, values=self._values[:0], weights=None if self._weights is None else self._weights[:0],
                    lengths=self.lengths()[:0], stride=None if spkpr is not None else self.stride(),
                    stride_per_key_per_rank=spkpr, stride_per_rank=self._stride_per_rank, length_per_key=[], offset_per_key=None))
            else:
                split_list.append(KeyedJaggedTensor(
                    keys=keys,
                    values=self._values[start_offset:end_offset],
                    weights=None if self._weights is None else self._weights[start_offset:end_offset],
                    lengths=self.lengths()[lo[start] : lo[end]],
                    stride=None if spkpr is not None else self.stride(),
                    stride_per_key_per_rank=spkpr,
                    stride_per_rank=self._stride_per_rank,
                    length_per_key=_length_per_key[start:end],
                    offset_per_key=None,
                    inverse_indices=None,
                ))
            start = end
            start_offset = end_offset
        return split_list

    def permute(self, indices: List[int], indices_tensor: Optional[torch.Tensor] = None) -> "KeyedJaggedTensor":
        """Reorder / select / repeat keys. Parity: jagged_tensor.py:2816-2925."""
        if indices_tensor is None:
            indices_tensor = _perm_index_tensor(indices, self.device())
        length_per_key = self.length_per_key()
        permuted_keys = [self._keys[i] for i in indices]
        permuted_length_per_key = [length_per_key[i] for i in indices]
        total = sum(permuted_length_per_key)
        spkpr = None
        if self._variable_stride_per_key:
            spkpr = self._stride_per_key_per_rank[torch.tensor(indices, dtype=torch.long)] if len(indices) else self._stride_per_key_per_rank[:0]
            lo = self.lengths_offset_per_key()
            seg_sizes = torch.tensor(self.stride_per_key(), device=self.device(), dtype=torch.int64)
            lengths64 = self.lengths()
            # segments = the per-key runs of `lengths` (stride_per_key entries each); the permuted lengths are the op's VALUES output
            _, out_lengths, _ = J.permute_1D_sparse_data(indices_tensor, seg_sizes, lengths64, None, sum(self.stride_per_key()[i] for i in indices))
            vals_seg = torch.tensor(length_per_key, device=self.device(), dtype=torch.int64)
            _, values, weights = J.permute_1D_sparse_data(indices_tensor, vals_seg, self._values, self._weights, total)
            permuted_lengths = out_lengths
        else:
            F = len(self._keys)
            lengths2d = self.lengths().view(F, -1) if F > 0 else self.lengths().view(0, 0)
            permuted_lengths, values, weights = J.permute_2D_sparse_data(indices_tensor, lengths2d, self._values, self._weights, total)
            permuted_lengths = permuted_lengths.reshape(-1)
        return KeyedJaggedTensor(
            keys=permuted_keys, values=values, weights=weights, lengths=permuted_lengths,
            stride=None if spkpr is not None else self._stride, stride_per_key_per_rank=spkpr,
            stride_per_rank=self._stride_per_rank if spkpr is None else None,
            length_per_key=permuted_length_per_key if len(permuted_keys) > 0 else None,
            inverse_indices=self._inverse_indices,
        )

    def flatten_lengths(self) -> "KeyedJaggedTensor":
        return KeyedJaggedTensor(keys=self._keys, values=self._values, weights=self._weights, lengths=self.lengths().view(-1),
                                 stride=self._stride, stride_per_key_per_rank=self._stride_per_key_per_rank if self._variable_stride_per_key else None,
                                 length_per_key=self._length_per_key, offset_per_key=self._offset_per_key)

    def __getitem__(self, key: str) -> JaggedTensor:
        offset_per_key = self.offset_per_key()
        index = self._key_indices()[key]
        start, end = offset_per_key[index], offset_per_key[index + 1]
        lo = self.lengths_offset_per_key()
        return JaggedTensor(
            values=self._values[start:end],
            weights=None if self._weights is None else self._weights[start:end],
            lengths=self.lengths()[lo[index] : lo[index + 1]],
            offsets=None,
        )

    def to_dict(self) -> Dict[str, JaggedTensor]:
        if self._jt_dict is None:
            self._jt_dict = {k: self[k] for k in self._keys}
        return self._jt_dict

    def record_stream(self, stream: torch.Stream) -> None:
        for t in (self._values, self._weights, self._lengths, self._offsets):
            if t is not None and t.is_cuda:
                t.record_stream(stream)
        if self._inverse_indices is not None and self._inverse_indices[1].is_cuda:
            self._inverse_indices[1].record_stream(stream)

    def to(self, device: torch.device, non_blocking: bool = False, dtype: Optional[torch.dtype] = None) -> "KeyedJaggedTensor":
        mv = lambda t: None if t is None else t.to(device, non_blocking=non_blocking)
        weights = self._weights
        if weights is not None and dtype is not None:
            weights = weights.to(dtype)
        inv = self._inverse_indices
        if inv is not None:
            inv = (inv[0], inv[1].to(device, non_blocking=non_blocking))
        return KeyedJaggedTensor(
            keys=self._keys, values=mv(self._values), weights=mv(weights), lengths=mv(self._lengths), offsets=mv(self._offsets),
            stride=self._stride, stride_per_key_per_rank=self._stride_per_key_per_rank if self._variable_stride_per_key else None,
            stride_per_rank=self._stride_per_rank, length_per_key=self._length_per_key, offset_per_key=self._offset_per_key,
            index_per_key=self._index_per_key, jt_dict=None, inverse_indices=inv,
        )

    def pin_memory(self) -> "KeyedJaggedTensor":
        pm = lambda t: None if t is None else t.pin_memory()
        inv = self._inverse_indices
        if inv is not None:
            inv = (inv[0], inv[1].pin_memory())
        return KeyedJaggedTensor(
            keys=self._keys, values=pm(self._values), weights=pm(self._weights), lengths=pm(self._lengths), offsets=pm(self._offsets),
            stride=self._stride, stride_per_key_per_rank=self._stride_per_key_per_rank if self._variable_stride_per_key else None,
            stride_per_rank=self._stride_per_rank, length_per_key=self._length_per_key, offset_per_key=self._offset_per_key,
            index_per_key=self._index_per_key, jt_dict=None, inverse_indices=inv,
        )

    # ---- input-dist hooks (reference jagged_tensor.py:3180-3380) ---------------------------------
    def dist_labels(self) -> List[str]:
        labels = ["lengths", "values"]
        if self.variable_stride_per_key():
            labels.append("strides")
        if self.weights_or_none() is not None:
            labels.append("weights")
        return labels

    def dist_splits(self, key_splits: List[int]) -> List[List[int]]:
        batch_size_per_split = _sum_by_splits(self.stride_per_key(), key_splits)
        length_per_split = _sum_by_splits(self.length_per_key(), key_splits)
        splits = [batch_size_per_split, length_per_split]
        if self.variable_stride_per_key():
            splits.append(key_splits)
        if self.weights_or_none() is not None:
            splits.append(length_per_split)
        return splits

    def dist_tensors(self) -> List[torch.Tensor]:
        tensors = [self.lengths(), self.values()]
        if self.variable_stride_per_key():
            strides = _pin_and_move(torch.tensor(self.stride_per_key(), dtype=torch.int64), self.device())
            tensors.append(strides)
        if self.weights_or_none() is not None:
            tensors.append(self.weights())
        return tensors

    @staticmethod
    def dist_init(
        keys: List[str],
        tensors: List[torch.Tensor],
        variable_stride_per_key: bool,
        num_workers: int,
        recat: Optional[torch.Tensor],
        stride_per_rank: Optional[List[int]],
        stagger: int = 1,
    ) -> "KeyedJaggedTensor":
        """Rebuild the local KJT from all-to-all received buffers (rank-major) by a recat permute
        into key-major order."""
        assert len(tensors) in (2, 3, 4)
        lengths, values = tensors[0], tensors[1]
        stride_per_rank_per_key = tensors[2] if variable_stride_per_key else None
        weights = tensors[-1] if (variable_stride_per_key and len(tensors) == 4) or (not variable_stride_per_key and len(tensors) == 3) else None
        if variable_stride_per_key:
            assert stride_per_rank_per_key is not None
            spkpr_t = stride_per_rank_per_key.view(num_workers, len(keys)).T.cpu()
            if stagger > 1:
                local_world = num_workers // stagger
                order = torch.arange(num_workers).view(stagger, local_world).T.reshape(-1)
                # strides arrive in staggered rank order; restore plain rank order for metadata
                spkpr_t = spkpr_t[:, torch.argsort(order)] if False else spkpr_t
            if recat is not None and recat.numel() > 0:
                seg = stride_per_rank_per_key.to(torch.int64)
                lengths_csum = torch.cat([lengths.new_zeros(1, dtype=torch.int64), torch.cumsum(lengths.to(torch.int64), 0)])
                seg_off = torch.cat([seg.new_zeros(1), torch.cumsum(seg, 0)])
                val_seg = lengths_csum[seg_off[1:]] - lengths_csum[seg_off[:-1]]
                _, new_lengths, _ = J.permute_1D_sparse_data(recat, seg, lengths, None, lengths.numel())  # (segment sizes, permuted ENTRIES, weights)
                _, values, weights = J.permute_1D_sparse_data(recat, val_seg, values, weights, values.numel())
                lengths = new_lengths
            return KeyedJaggedTensor(keys=keys, values=values, weights=weights, lengths=lengths, stride_per_key_per_rank=spkpr_t)
        assert stride_per_rank is not None
        single_batch_per_rank = all(s == stride_per_rank[0] for s in stride_per_rank)
        if recat is not None and recat.numel() > 0:
            if single_batch_per_rank:
                stride = stride_per_rank[0]
                lengths, values, weights = J.permute_2D_sparse_data(recat, lengths.view(-1, stride), values, weights, values.numel())
                lengths = lengths.reshape(-1)
            else:
                # uneven batch per rank: segments of [rank][key] with per-rank stride
                nk = len(keys)
                seg = torch.tensor([s for s in stride_per_rank for _ in range(nk)], device=lengths.device, dtype=torch.int64)
                lengths_csum = torch.cat([lengths.new_zeros(1, dtype=torch.int64), torch.cumsum(lengths.to(torch.int64), 0)])
                seg_off = torch.cat([seg.new_zeros(1), torch.cumsum(seg, 0)])
                val_seg = lengths_csum[seg_off[1:]] - lengths_csum[seg_off[:-1]]
                _, new_lengths, _ = J.permute_1D_sparse_data(recat, seg, lengths, None, lengths.numel())  # (segment sizes, permuted ENTRIES, weights)
                _, values, weights = J.permute_1D_sparse_data(recat, val_seg, values, weights, values.numel())
                lengths = new_lengths
        return KeyedJaggedTensor(keys=keys, values=values, weights=weights, lengths=lengths,
                                 stride=sum(stride_per_rank), stride_per_rank=stride_per_rank)

    def __str__(self) -> str:
        if len(self._keys) == 0 or (self._offsets is None and self._lengths is None):
            return "KeyedJaggedTensor()\n"
        s = "KeyedJaggedTensor({\n"
        for k in self._keys:
            jt = self[k]
            off = jt.offsets().tolist()
            vals = jt.values().tolist()
            s += f'    "{k}": ' + repr([vals[off[i] : off[i + 1]] for i in range(len(off) - 1)]) + ",\n"
        return s + "})\n"


def _kjt_flatten(t: KeyedJaggedTensor):
    ctx = (t._keys, t._stride_per_key_per_rank if t._variable_stride_per_key else None, t._stride, t._stride_per_rank)
    return [getattr(t, a) for a in KeyedJaggedTensor._fields], ctx


def _kjt_unflatten(values, context) -> KeyedJaggedTensor:
    keys, spkpr, stride, spr = context
    return KeyedJaggedTensor(keys, *values, stride=stride if spkpr is None else None, stride_per_key_per_rank=spkpr, stride_per_rank=spr)


register_pytree_node(KeyedJaggedTensor, _kjt_flatten, _kjt_unflatten, serialized_type_name="torchrec_b200.sparse.KeyedJaggedTensor")


def flatten_kjt_list(kjt_arr: List[KeyedJaggedTensor]):
    flat, ctxs = [], []
    for k in kjt_arr:
        f, c = _kjt_flatten(k)
        flat.extend(f)
        ctxs.append(c)
    return flat, ctxs


def unflatten_kjt_list(values, contexts) -> List[KeyedJaggedTensor]:
    n = len(KeyedJaggedTensor._fields)
    return [_kjt_unflatten(values[i * n : (i + 1) * n], c) for i, c in enumerate(contexts)]


# ---------------------------------------------------------------------------------------------
class KeyedTensor(Pipelineable, metaclass=JaggedTensorMeta):
    """Dense tensor whose ``key_dim`` is a concatenation of per-key blocks ([B, sum(D)] for pooled
    embeddings). Parity: jagged_tensor.py:3503-3770."""

    def __init__(
        self,
        keys: List[str],
        length_per_key: List[int],
        values: torch.Tensor,
        key_dim: int = 1,
        offset_per_key: Optional[List[int]] = None,
        index_per_key: Optional[Dict[str, int]] = None,
    ) -> None:
        self._keys = list(keys)
        self._length_per_key = list(length_per_key)
        self._values = values
        self._key_dim = key_dim
        self._offset_per_key = offset_per_key
        self._index_per_key = index_per_key

    @staticmethod
    def from_tensor_list(keys: List[str], tensors: List[torch.Tensor], key_dim: int = 1, cat_dim: int = 1) -> "KeyedTensor":
        length_per_key = [t.shape[key_dim] for t in tensors]
        return KeyedTensor(keys=keys, length_per_key=length_per_key, values=torch.cat(tensors, dim=cat_dim), key_dim=key_dim)

    def keys(self) -> List[str]:
        return self._keys

    def values(self) -> torch.Tensor:
        return self._values

    def key_dim(self) -> int:
        return self._key_dim

    def device(self) -> torch.device:
        return self._values.device

    def offset_per_key(self) -> List[int]:
        if self._offset_per_key is None:
            self._offset_per_key = _cumsum_list(self._length_per_key)
        return self._offset_per_key

    def length_per_key(self) -> List[int]:
        return self._length_per_key

    def _key_indices(self) -> Dict[str, int]:
        if self._index_per_key is None:
            self._index_per_key = {k: i for i, k in enumerate(self._keys)}
        return self._index_per_key

    def __getitem__(self, key: str) -> torch.Tensor:
        i = self._key_indices()[key]
        off = self.offset_per_key()
        return self._values.narrow(self._key_dim, off[i], self._length_per_key[i])

    def to_dict(self) -> Dict[str, torch.Tensor]:
        off = self.offset_per_key()
        return {k: self._values.narrow(self._key_dim, off[i], self._length_per_key[i]) for i, k in enumerate(self._keys)}

    @staticmethod
    def regroup(keyed_tensors: List["KeyedTensor"], groups: List[List[str]]) -> List[torch.Tensor]:
        return regroup_kts(keyed_tensors, groups)

    @staticmethod
    def regroup_as_dict(keyed_tensors: List["KeyedTensor"], groups: List[List[str]], keys: List[str]) -> Dict[str, torch.Tensor]:
        assert len(groups) == len(keys), "Groups and keys should have same length"
        return dict(zip(keys, regroup_kts(keyed_tensors, groups)))

    def record_stream(self, stream: torch.Stream) -> None:
        if self._values.is_cuda:
            self._values.record_stream(stream)

    def to(self, device: torch.device, non_blocking: bool = False) -> "KeyedTensor":
        return KeyedTensor(keys=self._keys, length_per_key=self._length_per_key, values=self._values.to(device, non_blocking=non_blocking),
                           key_dim=self._key_dim, offset_per_key=self._offset_per_key, index_per_key=self._index_per_key)

    def __str__(self) -> str:
        if len(self._keys) == 0:
            return "KeyedTensor()\n"
        return "KeyedTensor({\n" + "".join(f'    "{k}": {self[k].tolist()!r},\n' for k in self._keys) + "})\n"


def regroup_kts(keyed_tensors: List[KeyedTensor], groups: List[List[str]]) -> List[torch.Tensor]:
    """Gather the column blocks named in each group from several KTs into one tensor per group
    (replaces fbgemm.regroup_keyed_tensor / permute_multi_embedding, jagged_tensor.py:264-304)."""
    assert len(keyed_tensors) > 0
    key_dim = keyed_tensors[0].key_dim()
    where: Dict[str, Tuple[int, int, int]] = {}
    for ti, kt in enumerate(keyed_tensors):
        off = kt.offset_per_key()
        for ki, k in enumerate(kt.keys()):
            if k not in where:
                where[k] = (ti, off[ki], kt.length_per_key()[ki])
    out = []
    for group in groups:
        parts = []
        for k in group:
            ti, o, l = where[k]
            parts.append(keyed_tensors[ti].values().narrow(key_dim, o, l))
        out.append(torch.cat(parts, dim=key_dim) if parts else keyed_tensors[0].values().narrow(key_dim, 0, 0))
    return out


def permute_multi_embedding(keyed_tensors: List[KeyedTensor], groups: List[List[str]]) -> List[torch.Tensor]:
    return regroup_kts(keyed_tensors, groups)


def _kt_flatten(t: KeyedTensor):
    return [t._values], (t._keys, t._length_per_key, t._key_dim)


def _kt_unflatten(values, context) -> KeyedTensor:
    keys, lpk, kd = context
    return KeyedTensor(keys, lpk, values[0], kd)


register_pytree_node(KeyedTensor, _kt_flatten, _kt_unflatten, serialized_type_name="torchrec_b200.sparse.KeyedTensor")


def jt_is_equal(jt_1: "JaggedTensor", jt_2: "JaggedTensor") -> bool:
    """Same values, weights, lengths and offsets (an optional field must be present on both sides or on neither)."""
    if not isinstance(jt_1, JaggedTensor) or not isinstance(jt_2, JaggedTensor):
        return False
    if jt_1.values().shape != jt_2.values().shape or not torch.allclose(jt_1.values(), jt_2.values()):
        return False
    wa, wb = jt_1.weights_or_none(), jt_2.weights_or_none()
    if (wa is None) != (wb is None) or (wa is not None and (wa.shape != wb.shape or not torch.allclose(wa, wb))):
        return False
    return torch.equal(jt_1.lengths(), jt_2.lengths()) and torch.equal(jt_1.offsets(), jt_2.offsets())


def kjt_is_equal(kjt_1: "KeyedJaggedTensor", kjt_2: "KeyedJaggedTensor") -> bool:
    a, b = kjt_1, kjt_2
    if a.keys() != b.keys():
        return False
    if not torch.equal(a.values(), b.values()) or not torch.equal(a.lengths(), b.lengths()):
        return False
    wa, wb = a.weights_or_none(), b.weights_or_none()
    if (wa is None) != (wb is None):
        return False
    return wa is None or torch.allclose(wa, wb)


class ComputeKJTToJTDict(torch.nn.Module):
    """Module form of ``kjt.to_dict()`` (reference jagged_tensor.py:1703)."""

    def forward(self, keyed_jagged_tensor: KeyedJaggedTensor) -> Dict[str, JaggedTensor]:
        return keyed_jagged_tensor.to_dict()


class ComputeJTDictToKJT(torch.nn.Module):
    def forward(self, jt_dict: Dict[str, JaggedTensor]) -> KeyedJaggedTensor:
        return KeyedJaggedTensor.from_jt_dict(jt_dict)
