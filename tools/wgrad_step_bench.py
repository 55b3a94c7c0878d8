"""The seven weight-gradient GEMMs of the one-GPU DLRM training step (batch 32768), run as ``LinearActFn.backward`` runs them:
the split plan, the memset of the fp32 output, the GEMM and, for the 479- and 13-wide inputs, the copy that drops the padding
column(s). CUDA-event time per wgrad (median of 20, L2 flushed before each) on seeded inputs. The step replays these launches from a
CUDA graph, so each timed call is enqueued behind a sleeping kernel: the events then bracket device time only, not the host time of
the Python launcher.

    python tools/wgrad_step_bench.py [--save DIR]                    # time the kernel library of this source tree
    python tools/wgrad_step_bench.py --trees OLD NEW [--rounds 3]    # alternate two source trees (each built), one process per
                                                                     # round and tree; reads the card name and power limit too

``--trees`` also reports how far each tree's gradients are from the first round of the first tree, relative to the largest
gradient magnitude: the split-K reductions add in a nondeterministic order, so two runs of one build differ as well."""
import argparse
import json
import os
import subprocess
import sys
import tempfile

M = 32768
# (name, n_out, n_in): gw [n_out, n_in] = gy^T [n_out, M] . x [M, n_in]; bottom MLP 13-512-256-128, top MLP 479-1024-1024-512-256
WGRADS = [("bot0", 512, 13), ("bot1", 256, 512), ("bot2", 128, 256), ("top0", 1024, 479), ("top1", 1024, 1024), ("top2", 512, 1024),
          ("top3", 256, 512)]


def _run_tree(tree, save_dir):
    import torch

    from torchrec_b200.ops import gemm

    assert os.path.abspath(gemm.__file__).startswith(os.path.abspath(tree) + os.sep), gemm.__file__
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(2024)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    res = {}
    for name, n_out, n_in in WGRADS:
        Kp = (n_in + 7) // 8 * 8
        gy = (torch.randn(M, n_out, device=dev, generator=g) * 0.3).to(torch.bfloat16)
        xb = torch.zeros(M, Kp, dtype=torch.bfloat16, device=dev)
        xb[:, :n_in] = (torch.randn(M, n_in, device=dev, generator=g) * 0.3).to(torch.bfloat16)
        split, tile_n = gemm._wgrad_plan(n_out, Kp, M, sms)

        def wgrad():  # LinearActFn.backward's wgrad()
            w = gemm.gemm_bf16(gy, xb, a_mn=True, b_mn=True, out_dtype=torch.float32, split_k=split, tile_n=tile_n)[:, :n_in]
            return w.contiguous() if (w.stride(1) != 1 or w.shape[1] != w.stride(0)) else w

        for _ in range(10):
            wgrad()
        ts = []
        for _ in range(20):
            torch.cuda._sleep(1_000_000)  # ~0.5 ms: the host enqueues the flush, both events and the wgrad meanwhile
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            wgrad()
            e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1) * 1e3)
        res[name] = {"us": sorted(ts)[len(ts) // 2], "split": split}
        if save_dir:
            torch.save(wgrad().cpu(), os.path.join(save_dir, name + ".pt"))
    return res


def _print_one(res):
    print("| wgrad | n_out x n_in | split | us | TFLOP/s |\n|---|---|---|---|---|")
    for name, n_out, n_in in WGRADS:
        r = res[name]
        print(f"| {name} | {n_out} x {n_in} | {r['split']} | {r['us']:.1f} | {2 * M * n_out * n_in / r['us'] / 1e6:.0f} |")
    print(f"\ntotal: {sum(r['us'] for r in res.values()):.1f} us")


def _alternate(trees, rounds):
    import torch

    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    print(f"# {smi.stdout.strip()}  (name, power limit, max SM clock)\n")
    runs = {t: [] for t in trees}
    with tempfile.TemporaryDirectory() as tmp:
        for r in range(rounds):
            for i, t in enumerate(trees):
                d = os.path.join(tmp, f"{i}_{r}")
                os.makedirs(d)
                cmd = [sys.executable, os.path.abspath(__file__), "--tree", os.path.abspath(t), "--save", d, "--json"]
                out = subprocess.run(cmd, capture_output=True, text=True, check=True).stdout
                runs[t].append((json.loads(out.strip().splitlines()[-1]), d))
        med = lambda xs: sorted(xs)[len(xs) // 2]
        head = " | ".join(f"tree {i} split | tree {i} us (rounds) | tree {i} TFLOP/s" for i in range(len(trees)))
        print(f"| wgrad | n_out x n_in | {head} |\n|---|---|" + "---|---|---|" * len(trees))
        tot = [0.0] * len(trees)
        for name, n_out, n_in in WGRADS:
            cells = []
            for i, t in enumerate(trees):
                us = [res[name]["us"] for res, _ in runs[t]]
                tot[i] += med(us)
                cells.append(f"{runs[t][0][0][name]['split']} | {med(us):.1f} ({', '.join(f'{u:.1f}' for u in us)}) | {2 * M * n_out * n_in / med(us) / 1e6:.0f}")
            print(f"| {name} | {n_out} x {n_in} | " + " | ".join(cells) + " |")
        print("\ntotal of medians: " + ", ".join(f"tree {i} ({t}) {tot[i]:.1f} us" for i, t in enumerate(trees)))
        print("\n| wgrad | " + " | ".join(f"tree {i} round {r}" for i in range(len(trees)) for r in range(rounds)) + " |")
        print("|---|" + "---|" * (len(trees) * rounds))
        ref_dir = runs[trees[0]][0][1]
        for name, _, _ in WGRADS:
            ref = torch.load(os.path.join(ref_dir, name + ".pt"))
            scale = ref.abs().max().item()
            cells = []
            for t in trees:
                for _, d in runs[t]:
                    x = torch.load(os.path.join(d, name + ".pt"))
                    cells.append("shape!" if x.shape != ref.shape else f"{(x - ref).abs().max().item() / scale:.2e}")
            print(f"| {name} | " + " | ".join(cells) + " |")
        print("\n(max |gw - gw of tree 0, round 0| / max |gw of tree 0, round 0|)")


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--tree", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))), help="source tree whose kernel library is timed")
    ap.add_argument("--save", default="")
    ap.add_argument("--json", action="store_true")
    ap.add_argument("--trees", nargs="+", default=None)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if args.trees:
        _alternate(args.trees, args.rounds)
    else:
        sys.path.insert(0, args.tree)
        res = _run_tree(args.tree, args.save)
        print(json.dumps(res) if args.json else "", end="\n" if args.json else "")
        if not args.json:
            _print_one(res)
