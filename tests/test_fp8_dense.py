"""FP8 dense inference on CPU: the number format (ops/fp8_dense.py), the emulation, the module swap of quantize_dense and the
DLRM predict factory with ``dense_dtype``."""
import math

import pytest
import torch
from torch import nn

from torchrec_b200.inference.modules import quantize_dense
from torchrec_b200.models.dlrm import DLRM, DLRM_DCN
from torchrec_b200.modules.crossnet import LowRankCrossNet
from torchrec_b200.modules.embedding_configs import EmbeddingBagConfig
from torchrec_b200.modules.embedding_modules import EmbeddingBagCollection
from torchrec_b200.modules.mlp import MLP, Perceptron
from torchrec_b200.ops import fp8_dense as F8
from torchrec_b200.quant.dense_modules import Fp8Linear, Fp8LowRankCrossNet, Fp8MLP
from torchrec_b200.sparse import KeyedJaggedTensor


def _scale_by_definition(amax: float) -> float:
    """Smallest power of two s (>= 2^-126) with amax <= 448 s; 1 for 0 (float64 search)."""
    if amax == 0.0:
        return 1.0
    k = -126
    while amax > 448.0 * 2.0 ** k:
        k += 1
    return 2.0 ** k


def test_scale_rule_powers_of_two():
    vals = [0.0, 448.0, 449.0, 224.0, 224.0001, 1.0, 1e-30, 1e-45, 3.0e38, 56.0, 57.0, 0.4375, 448.0 * 2.0 ** -20]
    g = torch.Generator().manual_seed(0)
    vals += (torch.rand(200, generator=g, dtype=torch.float64) * 10.0 ** torch.randint(-20, 20, (200,), generator=g)).tolist()
    amax = torch.tensor(vals, dtype=torch.float32)
    s = F8.pow2_scale(amax)
    for a, sv in zip(amax.tolist(), s.tolist()):
        assert sv == _scale_by_definition(a), (a, sv)
        m, _ = math.frexp(sv)
        assert m == 0.5  # exact power of two


def _rows(M, K, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(M, K, generator=g)
    x *= 10.0 ** torch.randint(-6, 6, (M, 1), generator=g).float()  # mixed row magnitudes
    return x


def test_quantize_rows_reference_blocks():
    M, K = 9, 200  # a full block and a partial one (72 values, padded to 208 columns)
    x = _rows(M, K)
    x[3] = 0.0  # zero row
    x[4, :128] = 0.0  # zero block
    x[5, 7] = 448.0  # block whose amax is exactly 448: scale 1, value kept exactly
    x[5, :128].clamp_(-448.0, 448.0)
    x[6, 150] = -448.0
    x[6, 128:].clamp_(-448.0, 448.0)
    q, s = F8.quantize_rows_reference(x)
    assert q.dtype == torch.float8_e4m3fn and q.shape == (M, 208) and s.shape == (2, 128)
    assert bool((q[:, K:].float() == 0).all())
    assert bool((s[:, M:] == 1).all())
    sb = F8.row_block_scales(s, M)
    assert sb.shape == (M, 2)
    assert bool((sb[3] == 1).all()) and float(sb[4, 0]) == 1.0
    assert float(sb[5, 0]) == 1.0 and float(q[5, 7].float()) == 448.0
    assert float(sb[6, 1]) == 1.0 and float(q[6, 150].float()) == -448.0
    for r in range(M):
        for b in range(2):
            blk = x[r, 128 * b : min(K, 128 * (b + 1))]
            assert float(sb[r, b]) == _scale_by_definition(float(blk.abs().max()))
    # error of one e4m3 rounding: half an ulp (2^-4 relative) for normals, 2^-10 s for subnormals
    deq = F8.dequantize(q, s, K)
    bound = torch.maximum(x.abs() * 2.0 ** -4, sb.repeat_interleave(128, 1)[:, :K] * 2.0 ** -10)
    assert bool(((deq - x).abs() <= bound).all())


def test_quantize_weight_channel_scales():
    w = _rows(24, 13, seed=1)
    q, s = F8.quantize_weight(w)
    assert q.shape == (24, 16) and s.shape == (24,)
    for n in range(24):
        assert float(s[n]) == _scale_by_definition(float(w[n].abs().max()))
    assert bool((q[:, 13:].float() == 0).all())
    deq = F8.dequantize(q, s)[:, :13]
    assert bool(((deq - w).abs() <= torch.maximum(w.abs() * 2.0 ** -4, s[:, None] * 2.0 ** -10)).all())


def test_emulation_matches_formula():
    M, K, N = 5, 300, 32
    xq, sa = F8.quantize_rows_reference(_rows(M, K, seed=2))
    wq, sw = F8.quantize_weight(torch.randn(N, K))
    bias = torch.randn(N)
    ref = F8.gemm_fp8_reference(xq, sa, wq, sw, bias, F8.ACT_RELU)
    # hand-written: out[m, n] = relu(sw[n] * sum_kb sa[m, kb] * sum_{k in kb} a[m, k] w[n, k] + bias[n])
    a, w = xq.double(), wq.double()
    sab = F8.row_block_scales(sa, M).double()
    for m in range(M):
        for n in range(N):
            acc = 0.0
            for kb in range(sab.shape[1]):
                acc += float(sab[m, kb]) * sum(float(a[m, k]) * float(w[n, k]) for k in range(128 * kb, min(xq.shape[1], 128 * (kb + 1))))
            want = max(0.0, float(sw[n]) * acc + float(bias[n]))
            assert abs(float(ref[m, n]) - want) <= 1e-9 * (1.0 + abs(want))
    # the CPU path of gemm_fp8 (fp32 emulation) agrees with the oracle up to fp32 / bf16 rounding
    got = F8.gemm_fp8(xq, sa, wq, sw, bias, F8.ACT_RELU)
    assert got.dtype == torch.bfloat16
    assert torch.allclose(got.double(), ref, rtol=2 ** -7, atol=1e-3 * float(ref.abs().max()))
    gq, gs = F8.gemm_fp8(xq, sa, wq, sw, bias, F8.ACT_RELU, out_fp8=True)
    assert gq.dtype == torch.float8_e4m3fn and gs.shape == (1, 128)
    assert torch.allclose(F8.dequantize(gq, gs).double(), ref, rtol=2 ** -3, atol=1e-3 * float(ref.abs().max()))


def test_fp8_mlp_swaps_only_eligible_layers():
    torch.manual_seed(0)
    mlp = MLP(20, [32, 24, 48, 16])  # 24 % 16 != 0: that layer stays a Perceptron
    f = Fp8MLP.from_float(mlp)
    kinds = [type(l) for l in f._mlp]
    assert kinds == [Fp8Linear, Perceptron, Fp8Linear, Fp8Linear]
    assert f._mlp[1] is mlp._mlp[1]
    x = torch.randn(7, 20)
    ref = mlp(x).detach()
    out = f(x)
    assert out.dtype == torch.bfloat16 and out.shape == ref.shape
    assert float((out.float() - ref).norm() / ref.norm()) < 0.1
    # a producer's zero-padded input columns are accepted
    out_pad = f(torch.nn.functional.pad(x, (0, 4)))
    assert torch.equal(out_pad, out)
    # sigmoid layers are not fused by the fp8 epilogue: such an MLP is left alone
    sig = MLP(16, [32, 16], activation="sigmoid")
    assert not Fp8MLP.eligible(sig)
    assert quantize_dense(nn.Sequential(sig), torch.float8_e4m3fn)[0] is sig


def _ebc(keys, dim):
    return EmbeddingBagCollection([EmbeddingBagConfig(name=f"t_{k}", embedding_dim=dim, num_embeddings=40 + 3 * i, feature_names=[k]) for i, k in enumerate(keys)])


def _kjt(keys, B, seed=0):
    g = torch.Generator().manual_seed(seed)
    lengths = torch.randint(1, 3, (len(keys) * B,), generator=g)
    return KeyedJaggedTensor(keys=keys, values=torch.randint(0, 40, (int(lengths.sum()),), generator=g), lengths=lengths)


def test_quantize_dense_dlrm_and_dcn():
    torch.manual_seed(0)
    keys = ["a", "b", "c"]
    dlrm = DLRM(_ebc(keys, 16), 5, [32, 16], [48, 32, 1]).eval()
    dcn = DLRM_DCN(_ebc(keys, 16), 5, [32, 16], [48, 32, 1], dcn_num_layers=2, dcn_low_rank_dim=16).eval()
    x, kjt = torch.rand(6, 5), _kjt(keys, 6)
    for model in (dlrm, dcn):
        ref = model(x, kjt).detach()
        ebc = model.sparse_arch.embedding_bag_collection
        head = model.over_arch.model[1]
        q = quantize_dense(model, torch.float8_e4m3fn)
        assert q is model
        assert isinstance(model.dense_arch.model, Fp8MLP) and isinstance(model.over_arch.model[0], Fp8MLP)
        assert model.over_arch.model[1] is head and type(head) is nn.Linear and head.weight.dtype == torch.float32
        assert model.sparse_arch.embedding_bag_collection is ebc
        if model is dcn:
            assert isinstance(model.inter_arch.crossnet, Fp8LowRankCrossNet)
        assert not any(isinstance(m, (MLP, LowRankCrossNet)) for m in model.modules())
        out = model(x, kjt)
        assert out.shape == ref.shape and bool(torch.isfinite(out).all())
        # FP8 dense arch against the fp32 model: a few e4m3 roundings (2^-4 relative each) per layer, on logits of order 0.1 - 1
        assert float((out.float() - ref).abs().max()) < 0.1 * (1.0 + float(ref.abs().max()))


def test_crossnet_ineligible_rank_untouched():
    cn = LowRankCrossNet(32, 2, low_rank=8)
    holder = nn.Sequential(cn)
    assert quantize_dense(holder, torch.float8_e4m3fn)[0] is cn


def test_fp8_state_dict_round_trip(tmp_path):
    torch.manual_seed(0)
    mlp_a, mlp_b = MLP(40, [32, 16]), MLP(40, [32, 16])
    fa, fb = Fp8MLP.from_float(mlp_a), Fp8MLP.from_float(mlp_b)
    sd = fa.state_dict()
    assert sd["_mlp.0.weight"].dtype == torch.float8_e4m3fn and sd["_mlp.0.weight_scale"].dtype == torch.float32
    torch.save(sd, tmp_path / "fp8.pt")
    fb.load_state_dict(torch.load(tmp_path / "fp8.pt"))
    x = torch.randn(3, 40)
    assert torch.equal(fa(x), fb(x))
    ca, cb = Fp8LowRankCrossNet.from_float(LowRankCrossNet(32, 2, 16)), Fp8LowRankCrossNet.from_float(LowRankCrossNet(32, 2, 16))
    cb.load_state_dict(ca.state_dict())
    y = torch.randn(3, 32)
    assert torch.equal(ca(y), cb(y))


def test_quantize_dense_half_unchanged():
    mlp = MLP(8, [16, 16])
    out = quantize_dense(nn.Sequential(mlp), torch.bfloat16)
    assert out[0] is mlp and mlp._mlp[0]._linear.weight.dtype == torch.bfloat16


def test_dlrm_predict_factory_dense_dtype():
    from torchrec_b200.inference.dlrm_predict import DLRMModelConfig, DLRMPredictFactory, create_training_batch

    keys = ["cat_0", "cat_1", "cat_2"]
    kw = dict(dense_arch_layer_sizes=[32, 16], dense_in_features=4, embedding_dim=16, id_list_features_keys=keys, num_embeddings_per_feature=[50, 60, 70],
              num_embeddings=100, over_arch_layer_sizes=[32, 1])
    assert DLRMModelConfig(**kw).dense_dtype is None
    factory = DLRMPredictFactory(DLRMModelConfig(**kw, dense_dtype=torch.float8_e4m3fn))
    module = factory.create_predict_module(world_size=1, device="cpu")
    assert sum(isinstance(m, Fp8MLP) for m in module.predict_module.modules()) == 2
    batch = create_training_batch(4, keys, 50, batch_size=6, ids_per_feature=2)
    out = module({"float_features": batch.dense_features, "id_list_features.lengths": batch.sparse_features.lengths(),
                  "id_list_features.values": batch.sparse_features.values()})
    assert out["default"].shape == (6,) and bool(((out["default"] >= 0) & (out["default"] <= 1)).all())
    plain = DLRMPredictFactory(DLRMModelConfig(**kw)).create_predict_module(world_size=1, device="cpu")
    assert not any(isinstance(m, Fp8MLP) for m in plain.predict_module.modules())
