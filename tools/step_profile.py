"""Per-kernel CUDA time of the step ``bench.py`` times, through torch.profiler (works under torchrun; ncu must not wrap multi-rank
commands). The model is built and prepared as in ``bench.main``: dense CUDA graphs captured (unless ``--cuda-graphs 0``), then
``init_data_parallel``. Prints rank 0's table (us per step).

    python tools/step_profile.py --gpus 1 [--steps 6]
    torchrun --nproc-per-node 2 tools/step_profile.py --gpus 2 [--steps 6]
"""
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402


def main() -> None:
    args = bench.parse_args()
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    device = torch.device(f"cuda:{int(os.environ.get('LOCAL_RANK', 0))}")
    torch.cuda.set_device(device)
    if world > 1:
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        dist.init_process_group("nccl", device_id=device)
    from torchrec_b200.datasets.random import RandomRecDataset

    torch.manual_seed(0)
    dmp, opt, keys, hashes, ids_per_feature, num_dense, _backend, _info = bench.build_ours(args, device, rank, world)
    ds = RandomRecDataset(keys, args.batch_size, hash_sizes=hashes, ids_per_features=ids_per_feature, num_dense=num_dense,
                          manual_seed=1234 + rank, num_generated_batches=4)
    batches = [b.to(device) for b in ds.batch_generator._generated_batches]
    inner = getattr(dmp.module, "model", None)
    if args.cuda_graphs != 0 and hasattr(inner, "capture_dense_graphs"):
        with torch.no_grad():
            sample_emb = inner.sparse_arch(batches[0].sparse_features)
        inner.capture_dense_graphs(batches[0].dense_features, sample_emb)
        inner.overlap_sparse_dense = bool(args.overlap_sparse)
        torch.cuda.synchronize()
    dmp.init_data_parallel()

    def step(b):
        opt.zero_grad()
        loss, _ = dmp(b)
        loss.backward()
        opt.step()

    for i in range(5):
        step(batches[i % 4])
    torch.cuda.synchronize()
    if world > 1:
        dist.barrier()
    n = max(2, min(args.steps, 6))
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA, torch.profiler.ProfilerActivity.CPU]) as prof:
        for i in range(n):
            step(batches[i % 4])
        torch.cuda.synchronize()
    if rank == 0:
        rows = []
        for e in prof.key_averages():
            t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)
            if t and e.device_type == torch.autograd.DeviceType.CUDA:
                rows.append((t / n, e.count / n, e.key[:110]))
        rows.sort(reverse=True)
        tot = sum(r[0] for r in rows)
        print(f"# rank 0 kernel time per step at {world} GPU(s): {tot:.0f} us\n\n| us/step | launches/step | kernel |\n|---|---|---|")
        for t, c, k in rows[:40]:
            print(f"| {t:.1f} | {c:.1f} | `{k}` |")
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
