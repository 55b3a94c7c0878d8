"""FP8 dense inference against bf16 on the GPU at hand.

    python tools/fp8_dense_bench.py [--rounds 3] [--iters 20] [--rows 100000] [--out results.jsonl]

GEMM section: for M in {2048, 8192, 32768} and (N, K) in the DLRM benchmark's top-MLP shapes and the DLRM-DCN cross net at low rank 512
((1024, 480), (1024, 1024), (512, 1024), (256, 512), (512, 3456), (3456, 512)) it times, in the same process and alternating round by
round, (a) the FP8 GEMM with a bf16 output including the quantization of its bf16 input, (b) the FP8 GEMM alone on quantized operands and
(c) the bf16 wgmma GEMM (``gemm_bf16``), all with an fp32 bias. Rates are 2 M N K over the median time of a round.

Predict section: ms per batch of the forward of a DLRM and a DLRM-DCN (3 cross layers, rank 512) predict module with the benchmark's
dense arch (512, 256, 128) and over arch (1024, 1024, 512, 256, 1), 26 FP8 tables of dimension 128, at batch 512, 4096 and 32768, with
the dense arch in FP8 (``quantize_dense(..., torch.float8_e4m3fn)``) or on the bf16 wgmma kernels (fp32 weights, bf16 operands).

Every line is one JSON object and carries the card name, its power limit and the SM clock read in the same run."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from torchrec_b200.ops import dense as _dense  # noqa: E402
from torchrec_b200.ops import fp8_dense as F8  # noqa: E402
from torchrec_b200.ops.gemm import gemm_bf16_tn  # noqa: E402

GEMM_MS = [2048, 8192, 32768]
GEMM_NK = [(1024, 480), (1024, 1024), (512, 1024), (256, 512), (512, 3456), (3456, 512)]
BATCHES = [512, 4096, 32768]


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True, check=True).stdout
    name, power, sm, sm_max = q.strip().splitlines()[0].split(", ")
    return {"gpu": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max}


def time_ms(fn, iters: int) -> float:
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / iters


def median(xs):
    s = sorted(xs)
    return s[len(s) // 2]


def gemm_section(args, info, emit) -> None:
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(0)
    for M in GEMM_MS:
        for N, K in GEMM_NK:
            x = torch.randn(M, K, generator=g, device=dev).to(torch.bfloat16)
            w = torch.randn(N, K, generator=g, device=dev) * K ** -0.5
            bias = torch.randn(N, generator=g, device=dev)
            wq, sw = F8.quantize_weight(w)
            xq, sa = F8.quantize_rows(x)
            Kp8 = (K + 7) // 8 * 8
            xb = torch.nn.functional.pad(x, (0, Kp8 - K)) if Kp8 != K else x
            wb = torch.nn.functional.pad(w.to(torch.bfloat16), (0, Kp8 - K)) if Kp8 != K else w.to(torch.bfloat16)
            cases = {
                "fp8_with_quantize": lambda: F8.gemm_fp8(*F8.quantize_rows(x), wq, sw, bias),
                "fp8_gemm_only": lambda: F8.gemm_fp8(xq, sa, wq, sw, bias),
                "bf16": lambda: gemm_bf16_tn(xb, wb, bias),
            }
            for fn in cases.values():  # warm-up of every case (module load, tensor-map encoding paths)
                fn()
            torch.cuda.synchronize()
            times = {k: [] for k in cases}
            for _ in range(args.rounds):
                for k, fn in cases.items():
                    times[k].append(time_ms(fn, args.iters))
            flop = 2.0 * M * N * K
            row = {"section": "gemm", "M": M, "N": N, "K": K, **info}
            for k, ts in times.items():
                ms = median(ts)
                row[f"{k}_ms"] = round(ms, 5)
                row[f"{k}_tflops"] = round(flop / (ms * 1e-3) / 1e12, 1)
            row["speedup_fp8_with_quantize_vs_bf16"] = round(row["bf16_ms"] / row["fp8_with_quantize_ms"], 3)
            emit(row)


def predict_models(rows: int):
    from torchrec_b200.inference.modules import quantize_inference_model, shard_quant_model
    from torchrec_b200.models.dlrm import DLRM, DLRM_DCN
    from torchrec_b200.modules.embedding_configs import EmbeddingBagConfig
    from torchrec_b200.modules.embedding_modules import EmbeddingBagCollection
    from torchrec_b200.types import DataType

    keys = [f"f{i}" for i in range(26)]
    out = {}
    for name in ("dlrm", "dcn"):
        torch.manual_seed(0)
        ebc = EmbeddingBagCollection([EmbeddingBagConfig(name=f"t_{k}", embedding_dim=128, num_embeddings=rows, feature_names=[k]) for k in keys])
        if name == "dlrm":
            model = DLRM(ebc, 13, [512, 256, 128], [1024, 1024, 512, 256, 1])
        else:
            model = DLRM_DCN(ebc, 13, [512, 256, 128], [1024, 1024, 512, 256, 1], dcn_num_layers=3, dcn_low_rank_dim=512)
        model.eval()
        model = quantize_inference_model(model, quantization_dtype=DataType.FP8)
        sharded, _ = shard_quant_model(model, world_size=1, compute_device="cuda", sharding_device="cpu")
        out[name] = sharded.to(torch.device("cuda", 0))
    return keys, out


def predict_section(args, info, emit) -> None:
    from torchrec_b200.inference.modules import quantize_dense
    from torchrec_b200.sparse import KeyedJaggedTensor

    from torchrec_b200.modules.crossnet import LowRankCrossNet
    from torchrec_b200.modules.mlp import MLP

    dev = torch.device("cuda", 0)
    keys, models = predict_models(args.rows)
    for name, model in models.items():
        # one model, its dense modules switched between the float form (bf16 wgmma) and the FP8 form: the tables are shared
        swaps = [(parent, cname, child, quantize_dense(torch.nn.Sequential(child), torch.float8_e4m3fn)[0])
                 for parent in list(model.modules()) for cname, child in list(parent.named_children()) if isinstance(child, (MLP, LowRankCrossNet))]

        def use(fp8: bool, model=model, swaps=swaps):
            for parent, cname, flt, f8 in swaps:
                setattr(parent, cname, f8 if fp8 else flt)
            return model

        variants = {"bf16": lambda *a, use=use: use(False)(*a), "fp8": lambda *a, use=use: use(True)(*a)}
        for B in BATCHES:
            g = torch.Generator(device=dev).manual_seed(B)
            dense = torch.rand(B, 13, generator=g, device=dev)
            kjt = KeyedJaggedTensor(keys=keys, lengths=torch.ones(len(keys) * B, dtype=torch.int32, device=dev),
                                    values=torch.randint(0, args.rows, (len(keys) * B,), generator=g, device=dev))
            with torch.inference_mode():
                for m in variants.values():
                    m(dense, kjt)
                torch.cuda.synchronize()
                times = {k: [] for k in variants}
                for _ in range(args.rounds):
                    for k, m in variants.items():
                        times[k].append(time_ms(lambda: m(dense, kjt), args.iters))
            row = {"section": "predict", "model": name, "batch": B, "tables": "FP8 (26 x %d rows x 128)" % args.rows, **info}
            for k, ts in times.items():
                row[f"{k}_dense_ms"] = round(median(ts), 4)
            row["speedup_fp8_vs_bf16"] = round(row["bf16_dense_ms"] / row["fp8_dense_ms"], 3)
            emit(row)


def main() -> None:
    p = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    p.add_argument("--rounds", type=int, default=3, help="alternating rounds per case; the median round is reported")
    p.add_argument("--iters", type=int, default=20, help="calls per timed round")
    p.add_argument("--rows", type=int, default=100_000, help="rows per embedding table of the predict modules")
    p.add_argument("--sections", type=str, default="gemm,predict")
    p.add_argument("--out", type=str, default="", help="also append the JSON lines to this file")
    args = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("fp8_dense_bench.py measures on a GPU; none is visible")
    torch.cuda.set_device(0)
    _dense.set_dense_backend("wgmma")
    info = card()

    def emit(row: dict) -> None:
        line = json.dumps(row)
        print(line, flush=True)
        if args.out:
            with open(args.out, "a") as f:
                f.write(line + "\n")

    sections = args.sections.split(",")
    if "gemm" in sections:
        gemm_section(args, info, emit)
    if "predict" in sections:
        predict_section(args, info, emit)
    emit({"section": "card_after", **card()})


if __name__ == "__main__":
    main()
