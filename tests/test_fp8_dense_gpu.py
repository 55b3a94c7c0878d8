"""FP8 dense inference on the H100: the quantize kernel against its CPU mirror (bit for bit), the e4m3 wgmma GEMM against the
float64 oracle on the same quantized operands, the FP8 modules and DLRM / DLRM-DCN predict modules against their CPU emulation, and a
CUDA-graph replay of the FP8 dense forward."""
import copy
import gc

import pytest
import torch

from torchrec_b200.inference.dlrm_predict import DLRMPredictModule
from torchrec_b200.inference.modules import quantize_dense
from torchrec_b200.models.dlrm import DLRM, DLRM_DCN
from torchrec_b200.modules.crossnet import LowRankCrossNet
from torchrec_b200.modules.embedding_configs import EmbeddingBagConfig
from torchrec_b200.modules.embedding_modules import EmbeddingBagCollection
from torchrec_b200.modules.mlp import MLP
from torchrec_b200.ops import fp8_dense as F8
from torchrec_b200.quant.dense_modules import Fp8LowRankCrossNet, Fp8MLP
from torchrec_b200.sparse import KeyedJaggedTensor

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)


@pytest.fixture(autouse=True)
def _collect_after_test():
    # The models and the CUDA graph built here sit in reference cycles: collect them now, so that their release does not happen in
    # a garbage-collector pass inside a later test's stream capture
    yield
    gc.collect()
    torch.cuda.synchronize()

# (N, K) of the DLRM benchmark's top MLP and of the DLRM-DCN cross net at low rank 512
SHAPES = [(1024, 480), (1024, 1024), (512, 1024), (256, 512), (512, 3456), (3456, 512)]


def _rows(M, K, seed, dtype=torch.float32):
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(M, K, generator=g, device=DEV)
    x *= 10.0 ** torch.randint(-6, 6, (M, 1), generator=g, device=DEV).float()  # mixed row magnitudes
    x[:: 5] = 0.0  # rows of zeros
    return x.to(dtype)


@pytest.mark.parametrize("K", [13, 127, 128, 480, 3456])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_quantize_rows_bit_exact(K, dtype):
    M = 257
    x = _rows(M, K, seed=K, dtype=dtype)
    q, s = F8.quantize_rows(x)
    rq, rs = F8.quantize_rows_reference(x.cpu())
    assert q.shape == rq.shape and s.shape == rs.shape
    assert torch.equal(q.cpu().view(torch.uint8), rq.view(torch.uint8))
    assert torch.equal(s.cpu(), rs)
    # any row pitch: a column slice of a wider matrix
    wide = _rows(M, K + 7, seed=K + 1, dtype=dtype)
    q2, s2 = F8.quantize_rows(wide[:, 3 : 3 + K])
    rq2, rs2 = F8.quantize_rows_reference(wide[:, 3 : 3 + K].cpu())
    assert torch.equal(q2.cpu().view(torch.uint8), rq2.view(torch.uint8)) and torch.equal(s2.cpu(), rs2)


def _operands(M, N, K, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(M, K, generator=g, device=DEV, dtype=torch.float32).to(torch.bfloat16)
    w = torch.randn(N, K, generator=g, device=DEV) * K ** -0.5
    bias = torch.randn(N, generator=g, device=DEV)
    aq, sa = F8.quantize_rows(x)
    wq, sw = F8.quantize_weight(w)
    return aq, sa, wq, sw, bias


def _tolerance(aq, sa, wq, sw, ref):
    # |out - ref| <= 2^-8 |ref| + 2^-10 sum_k |a_k w_k|: 2^-8 covers the bf16 rounding of the output (half an ulp is 2^-9 relative) and the
    # fp32 promotion arithmetic; the 2^-10 term covers the tensor core's reduced-precision accumulation of fp8 products inside a
    # K-block, whose error scales with the sum of the magnitudes of the products, not with the (possibly cancelling) result.
    mag = F8.gemm_fp8_reference(aq.float().abs().to(F8.E4M3), sa, wq.float().abs().to(F8.E4M3), sw)
    return 2.0 ** -8 * ref.abs() + 2.0 ** -10 * mag


@pytest.mark.parametrize("M", [1, 7, 129, 4096])
@pytest.mark.parametrize("N,K", SHAPES)
def test_gemm_bf16_out_vs_oracle(M, N, K):
    aq, sa, wq, sw, bias = _operands(M, N, K, seed=M * 7 + N + K)
    for use_bias in (False, True):
        for act in (F8.ACT_NONE, F8.ACT_RELU):
            b = bias if use_bias else None
            out = F8.gemm_fp8(aq, sa, wq, sw, b, act)
            ref = F8.gemm_fp8_reference(aq, sa, wq, sw, b, act)
            assert out.dtype == torch.bfloat16 and out.shape == (M, N)
            err = (out.double() - ref).abs()
            tol = _tolerance(aq, sa, wq, sw, ref)
            assert bool((err <= tol).all()), (use_bias, act, float((err - tol).max()))


@pytest.mark.parametrize("M", [1, 7, 129, 4096])
@pytest.mark.parametrize("N,K", SHAPES)
def test_gemm_fp8_out_vs_oracle(M, N, K):
    aq, sa, wq, sw, bias = _operands(M, N, K, seed=M * 11 + N + K)
    for act in (F8.ACT_NONE, F8.ACT_RELU):
        q, s = F8.gemm_fp8(aq, sa, wq, sw, bias, act, out_fp8=True)
        assert q.dtype == F8.E4M3 and q.shape == (M, N) and s.shape == ((N + 127) // 128, (M + 127) // 128 * 128)
        sb = F8.row_block_scales(s, M)
        mant, _ = torch.frexp(sb)
        assert bool((mant == 0.5).all()), "every output scale is a power of two"
        ref = F8.gemm_fp8_reference(aq, sa, wq, sw, bias, act)
        tol = _tolerance(aq, sa, wq, sw, ref)
        sfull = sb.double().repeat_interleave(128, dim=1)[:, :N]
        # the kernel rounds its fp32 value (within `tol` of ref) once to e4m3 at the block scale: half an ulp is at most 2^-4 of the
        # value for e4m3 normals and 2^-10 s for subnormals
        bound = 2.0 ** -4 * (ref.abs() + tol) + 2.0 ** -10 * sfull + tol
        err = (F8.dequantize(q, s).double() - ref).abs()
        assert bool((err <= bound).all()), (act, float((err - bound).max()))
        assert bool((q.float().abs() <= 448).all())


def _assert_close(got, want, rel):
    got, want = got.float().cpu(), want.float().cpu()
    assert got.shape == want.shape
    scale = float(want.abs().max()) + 1e-6
    assert float((got - want).abs().max()) <= rel * scale, float((got - want).abs().max()) / scale


def test_fp8_mlp_and_crossnet_cuda_vs_cpu_emulation():
    torch.manual_seed(0)
    mlp = MLP(479, [1024, 1024, 512, 256])
    f_cpu = Fp8MLP.from_float(mlp)
    f_gpu = copy.deepcopy(f_cpu).to(DEV)
    x = torch.rand(300, 479)
    # Tolerance: both run the same quantized chain; fp32 summation order differs, so an intermediate value next to an e4m3 rounding
    # boundary can land one ulp apart, which moves the output by a small fraction of its range
    _assert_close(f_gpu(x.to(DEV)), f_cpu(x), 0.03)
    # a producer's zero-padded bf16 columns
    xp = torch.nn.functional.pad(x, (0, 1)).to(torch.bfloat16)
    _assert_close(f_gpu(xp.to(DEV)), f_cpu(xp), 0.03)
    cn = LowRankCrossNet(3456, 3, 512)
    c_cpu = Fp8LowRankCrossNet.from_float(cn)
    c_gpu = copy.deepcopy(c_cpu).to(DEV)
    y = torch.randn(200, 3456)
    _assert_close(c_gpu(y.to(DEV)), c_cpu(y), 0.03)


def _models():
    torch.manual_seed(0)
    keys = [f"f{i}" for i in range(26)]

    def ebc():
        return EmbeddingBagCollection([EmbeddingBagConfig(name=f"t_{k}", embedding_dim=128, num_embeddings=1000 + i, feature_names=[k]) for i, k in enumerate(keys)])

    dlrm = DLRM(ebc(), 13, [512, 256, 128], [1024, 1024, 512, 256, 1]).eval()
    dcn = DLRM_DCN(ebc(), 13, [512, 256, 128], [1024, 1024, 512, 256, 1], dcn_num_layers=3, dcn_low_rank_dim=512).eval()
    return keys, {"dlrm": dlrm, "dcn": dcn}


def _batch(keys, B, seed=0):
    g = torch.Generator().manual_seed(seed)
    lengths = torch.ones(len(keys) * B, dtype=torch.int32)
    return {"float_features": torch.rand(B, 13, generator=g), "id_list_features.lengths": lengths,
            "id_list_features.values": torch.randint(0, 1000, (len(keys) * B,), generator=g)}


@pytest.mark.parametrize("name", ["dlrm", "dcn"])
def test_predict_module_fp8_vs_cpu_emulation_and_fp32(name):
    keys, models = _models()
    fp32 = models[name]
    batch = _batch(keys, 512)
    ref32 = DLRMPredictModule(copy.deepcopy(fp32), keys, device="cpu")(batch)["default"]
    emu = DLRMPredictModule(quantize_dense(copy.deepcopy(fp32), torch.float8_e4m3fn), keys, device="cpu")
    gpu = DLRMPredictModule(quantize_dense(copy.deepcopy(fp32).to(DEV), torch.float8_e4m3fn), keys, device="cuda:0")
    assert sum(isinstance(m, (Fp8MLP, Fp8LowRankCrossNet)) for m in gpu.predict_module.modules()) == (3 if name == "dcn" else 2)
    out_emu = emu(batch)["default"]
    out_gpu = gpu({k: v.to(DEV) for k, v in batch.items()})["default"]
    # probabilities: the same quantized chain on both sides (see test_fp8_mlp_and_crossnet_cuda_vs_cpu_emulation)
    assert float((out_gpu - out_emu).abs().max()) < 0.01
    # sanity against the fp32 model: every FP8 layer adds roundings of up to 2^-4 relative to its inputs, weights and outputs; through
    # 7 layers (10 with the cross net) that stays well inside 0.1 on a probability
    assert float((out_gpu - ref32).abs().max()) < 0.1


@pytest.mark.parametrize("name", ["dlrm", "dcn"])
def test_fp8_dense_forward_cuda_graph_replay(name):
    keys, models = _models()
    model = quantize_dense(models[name].to(DEV), torch.float8_e4m3fn)
    batch = _batch(keys, 1024, seed=1)
    dense = batch["float_features"].to(DEV)
    kjt = KeyedJaggedTensor(keys=keys, lengths=batch["id_list_features.lengths"].to(DEV), values=batch["id_list_features.values"].to(DEV))

    def dense_forward(x, emb):
        return model.over_arch(model.inter_arch(dense_features=model.dense_arch(x), sparse_features=emb))

    with torch.inference_mode():
        emb = model.sparse_arch(kjt)
        eager = dense_forward(dense, emb).clone()
        static_x, static_emb = dense.clone(), emb.clone()
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            dense_forward(static_x, static_emb)  # warm-up outside the capture
        torch.cuda.current_stream().wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            static_out = dense_forward(static_x, static_emb)
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(static_out, eager)
        # new inputs through the same graph
        x2 = torch.rand_like(dense)
        static_x.copy_(x2)
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(static_out, dense_forward(x2, emb))
