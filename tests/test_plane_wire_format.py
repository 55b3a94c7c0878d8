"""Which wire the NVLink sparse plane picks for each direction from the user's quantized-comms codecs (CPU: pure selection rules)."""
import pytest

from torchrec_b200.parallel.qcomm_codec import CommType, QCommsConfig, get_qcomm_codec, get_qcomm_codecs, get_qcomm_codecs_registry
from torchrec_b200.parallel.sparse_plane import select_wire_format
from torchrec_b200.parallel.types import CommOp, QuantizedCommCodecs

FP8 = get_qcomm_codecs(QCommsConfig(forward_precision=CommType.FP8, backward_precision=CommType.FP8, fp8_quantize_dim=32))
# three 128-wide direct units side by side; the push serves them at inbox columns 0, 128 (rank 0) and 0 (rank 1)
DIRECT = [(0, 128), (128, 128), (256, 128)]
PUSH = [(0, 0, 128), (128, 128, 128), (256, 0, 128)]


def test_aligned_layout_is_fp8_both_ways():
    fmt, why = select_wire_format(4, DIRECT, PUSH, FP8)
    assert fmt == {"fwd": ("fp8", 32), "bwd": ("fp8", 32)} and why == []


def test_row_dims_per_direction():
    codecs = get_qcomm_codecs(QCommsConfig(forward_precision=CommType.FP8, backward_precision=CommType.FP8, fp8_quantize_dim=128, fp8_quantize_dim_bwd=64))
    fmt, _ = select_wire_format(2, DIRECT, PUSH, codecs)
    assert fmt == {"fwd": ("fp8", 128), "bwd": ("fp8", 64)}
    fwd_only = get_qcomm_codecs(QCommsConfig(forward_precision=CommType.FP8, backward_precision=CommType.BF16, fp8_quantize_dim=32))
    assert select_wire_format(2, DIRECT, PUSH, fwd_only)[0] == {"fwd": ("fp8", 32), "bwd": None}


def test_misaligned_column_block_keeps_the_wire_dtype():
    # a 48-wide table at R = 32: both directions see it
    fmt, why = select_wire_format(2, [(0, 48), (48, 128)], [(0, 0, 48), (48, 0, 128)], FP8)
    assert fmt == {"fwd": None, "bwd": None} and len(why) == 2 and all("48" in w for w in why)
    # a 32-wide block at an offset that is not a multiple of R = 64
    codecs = get_qcomm_codecs(QCommsConfig(forward_precision=CommType.FP8, backward_precision=CommType.FP8, fp8_quantize_dim=64))
    fmt, _ = select_wire_format(2, [(0, 64), (96, 64)], [(0, 0, 64), (96, 64, 64)], codecs)
    assert fmt == {"fwd": None, "bwd": None}


def test_staged_columns_do_not_count_for_the_forward():
    # a row-sharded 48-wide table is summed at the destination: it is not a direct column, but its gradient is pushed
    fmt, why = select_wire_format(2, DIRECT, PUSH + [(384, 128, 48)], FP8)
    assert fmt == {"fwd": ("fp8", 32), "bwd": None} and len(why) == 1 and why[0].startswith("bwd")
    # only row-sharded tables: nothing to quantize forward, the push still is
    assert select_wire_format(2, [], PUSH, FP8)[0] == {"fwd": None, "bwd": ("fp8", 32)}


@pytest.mark.parametrize("kind", [CommType.FP32, CommType.FP16, CommType.BF16, CommType.INT8, CommType.MX4])
def test_other_codecs_keep_the_wire_dtype(kind):
    codecs = get_qcomm_codecs(QCommsConfig(forward_precision=kind, backward_precision=kind))
    assert select_wire_format(4, DIRECT, PUSH, codecs) == ({"fwd": None, "bwd": None}, [])
    assert get_qcomm_codec(kind, None, 32).fp8_row_dim is None


def test_no_codec_and_one_rank():
    assert select_wire_format(4, DIRECT, PUSH, None) == ({"fwd": None, "bwd": None}, [])
    assert select_wire_format(4, DIRECT, PUSH, QuantizedCommCodecs()) == ({"fwd": None, "bwd": None}, [])
    assert select_wire_format(1, DIRECT, PUSH, FP8) == ({"fwd": None, "bwd": None}, [])


@pytest.mark.parametrize("row_dim", [48, 96, 256])
def test_unsupported_row_dim(row_dim):
    codecs = get_qcomm_codecs(QCommsConfig(forward_precision=CommType.FP8, backward_precision=CommType.FP8, fp8_quantize_dim=row_dim))
    fmt, why = select_wire_format(2, [(0, 768)], [(0, 0, 768)], codecs)
    assert fmt == {"fwd": None, "bwd": None} and len(why) == 2


def test_registry_codecs_of_the_pooled_all_to_all():
    reg = get_qcomm_codecs_registry(QCommsConfig(forward_precision=CommType.FP8, backward_precision=CommType.FP8))
    codecs = reg[CommOp.POOLED_EMBEDDINGS_ALL_TO_ALL.name]
    assert codecs.forward.fp8_row_dim == 32 and codecs.backward.fp8_row_dim == 32
    assert select_wire_format(8, DIRECT, PUSH, codecs)[0] == {"fwd": ("fp8", 32), "bwd": ("fp8", 32)}
    # the reduce-scatter codecs never carry FP8
    rs = reg[CommOp.POOLED_EMBEDDINGS_REDUCE_SCATTER.name]
    assert select_wire_format(8, DIRECT, PUSH, rs)[0] == {"fwd": None, "bwd": None}
