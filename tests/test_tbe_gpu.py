"""Numerics of the sm_90a TBE kernels vs the fp32 PyTorch reference implementation."""
import pytest
import torch

from torchrec_b200.ops import tbe as T

pytestmark = pytest.mark.gpu


def _inputs(F, B, rows, maxL, device, seed=0, idx_dtype=torch.int64, hot=False):
    g = torch.Generator().manual_seed(seed)
    lengths = torch.randint(0, maxL + 1, (F * B,), generator=g)
    offsets = torch.cat([torch.zeros(1, dtype=torch.int64), lengths.cumsum(0)])
    idx = []
    for f in range(F):
        n = int(lengths[f * B : (f + 1) * B].sum())
        hi = 3 if (hot and f == 0) else rows[f]
        idx.append(torch.randint(0, hi, (n,), generator=g))
    indices = torch.cat(idx).to(idx_dtype)
    psw = torch.rand(indices.numel(), generator=g)
    return indices.to(device), offsets.to(device), psw.to(device)


@pytest.mark.parametrize("dim", [16, 64, 128, 256, 1024])
@pytest.mark.parametrize("wdtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("weighted", [False, True])
def test_pooled_forward(dim, wdtype, weighted):
    dev = torch.device("cuda:0")
    specs = [(100, dim), (57, dim), (1000, dim)]
    fmap = [0, 1, 1, 2]
    B = 33
    meta_g = T.TbeMeta.build([r for r, _ in specs], [d for _, d in specs], fmap, dev)
    meta_c = T.TbeMeta.build([r for r, _ in specs], [d for _, d in specs], fmap, torch.device("cpu"))
    w = (torch.randn(sum(r * d for r, d in specs)) * 0.1).to(wdtype)
    idx, off, psw = _inputs(4, B, [100, 57, 57, 1000], 5, dev, idx_dtype=torch.int32 if dim == 64 else torch.int64)
    for mean in (False, True):
        out = T.pooled_forward(meta_g, w.to(dev), idx, off, psw if weighted else None, B, mean, torch.float32)
        ref = T._ref_pooled_forward(meta_c, w.float(), idx.cpu(), off.cpu(), psw.cpu() if weighted else None, B, mean, torch.float32)
        torch.testing.assert_close(out.cpu(), ref, rtol=1e-4, atol=1e-4)
    out_bf = T.pooled_forward(meta_g, w.to(dev), idx, off, None, B, False, torch.bfloat16)
    ref = T._ref_pooled_forward(meta_c, w.float(), idx.cpu(), off.cpu(), None, B, False, torch.float32)
    torch.testing.assert_close(out_bf.float().cpu(), ref, rtol=2e-2, atol=2e-2)


@pytest.mark.parametrize("opt", [T.OptimType.EXACT_SGD, T.OptimType.EXACT_ROWWISE_ADAGRAD, T.OptimType.EXACT_ADAGRAD, T.OptimType.ADAM,
                                 T.OptimType.PARTIAL_ROWWISE_ADAM, T.OptimType.LAMB, T.OptimType.LARS_SGD, T.OptimType.NONE, T.OptimType.LION])
@pytest.mark.parametrize("dim", [32, 128, 512])
def test_fused_backward_matches_reference(opt, dim):
    dev = torch.device("cuda:0")
    specs = [(50, dim), (3, dim), (400, dim)]
    fmap = [0, 1, 2, 2]
    B = 300  # many duplicates on the 3-row table -> runs spanning several 32-wide chunks
    torch.manual_seed(1)
    cpu = T.TableBatchedEmbeddingBags(specs, fmap, optimizer=opt, learning_rate=0.05, eps=1e-3, weight_decay=0.01 if opt == T.OptimType.LAMB else 0.0)
    gpu = T.TableBatchedEmbeddingBags(specs, fmap, optimizer=opt, learning_rate=0.05, eps=1e-3, weight_decay=0.01 if opt == T.OptimType.LAMB else 0.0, device=dev)
    gpu.weights.data.copy_(cpu.weights.data)
    for step in range(2):
        idx, off, psw = _inputs(4, B, [50, 3, 400, 400], 4, dev, seed=step, hot=True)
        proj = torch.randn(B, 4 * dim)
        og = gpu(idx, off, psw)
        oc = cpu(idx.cpu(), off.cpu(), psw.cpu())
        torch.testing.assert_close(og.cpu(), oc, rtol=1e-4, atol=1e-4)
        (og * proj.to(dev)).sum().backward()
        (oc * proj).sum().backward()
        if opt == T.OptimType.NONE:
            torch.testing.assert_close(gpu.weights.grad.cpu(), cpu.weights.grad, rtol=2e-4, atol=2e-4)
            gpu.weights.grad = None
            cpu.weights.grad = None
        elif opt == T.OptimType.LION:
            # sign() is discontinuous: a gradient sum that differs in the last ulp (different reduction order) may flip an
            # element whose pre-sign value is ~0 -> allow a tiny fraction of 2*lr outliers
            bad = ((gpu.weights.cpu() - cpu.weights).abs() > 2e-4).float().mean()
            assert float(bad) < 5e-3, float(bad)
            gpu.weights.data.copy_(cpu.weights.data)
            gpu.state1.copy_(cpu.state1)
        else:
            torch.testing.assert_close(gpu.weights.cpu(), cpu.weights, rtol=2e-4, atol=2e-4)
            if gpu.state1 is not None:
                torch.testing.assert_close(gpu.state1.cpu(), cpu.state1, rtol=2e-4, atol=1e-5)


def test_bf16_tables_and_grads():
    dev = torch.device("cuda:0")
    specs = [(64, 128)]
    cpu = T.TableBatchedEmbeddingBags(specs, [0], optimizer=T.OptimType.EXACT_SGD, learning_rate=0.1)
    gpu = T.TableBatchedEmbeddingBags(specs, [0], optimizer=T.OptimType.EXACT_SGD, learning_rate=0.1, weights_precision=torch.bfloat16,
                                      output_dtype=torch.bfloat16, device=dev)
    cpu.weights.data.copy_(gpu.weights.data.float().cpu())
    idx, off, _ = _inputs(1, 40, [64], 3, dev)
    og = gpu(idx, off)
    oc = cpu(idx.cpu(), off.cpu())
    torch.testing.assert_close(og.float().cpu(), oc, rtol=2e-2, atol=2e-2)
    og.sum().backward()
    oc.sum().backward()
    torch.testing.assert_close(gpu.weights.float().cpu(), cpu.weights, rtol=2e-2, atol=2e-2)


def test_sequence_forward_backward():
    dev = torch.device("cuda:0")
    specs = [(30, 64), (40, 64)]
    cpu = T.TableBatchedEmbeddingBags(specs, [0, 1, 1], pooling_mode=T.PoolingMode.NONE, optimizer=T.OptimType.EXACT_ROWWISE_ADAGRAD, learning_rate=0.1)
    gpu = T.TableBatchedEmbeddingBags(specs, [0, 1, 1], pooling_mode=T.PoolingMode.NONE, optimizer=T.OptimType.EXACT_ROWWISE_ADAGRAD, learning_rate=0.1, device=dev)
    gpu.weights.data.copy_(cpu.weights.data)
    idx, off, _ = _inputs(3, 17, [30, 40, 40], 4, dev)
    og = gpu(idx, off)
    oc = cpu(idx.cpu(), off.cpu())
    torch.testing.assert_close(og.cpu(), oc)
    proj = torch.randn_like(oc)
    (og * proj.to(dev)).sum().backward()
    (oc * proj).sum().backward()
    torch.testing.assert_close(gpu.weights.cpu(), cpu.weights, rtol=1e-4, atol=1e-5)


def test_large_keys_64bit_path_and_launch_counter():
    from torchrec_b200.ops import _lib

    dev = torch.device("cuda:0")
    n0 = _lib.launch_count()
    specs = [(1 << 20, 32)]
    gpu = T.TableBatchedEmbeddingBags(specs, [0], optimizer=T.OptimType.EXACT_SGD, learning_rate=1.0, device=dev)
    w0 = gpu.weights.clone()
    idx = torch.tensor([5, 5, 7, (1 << 20) - 1], device=dev)
    off = torch.tensor([0, 2, 4], device=dev)
    out = gpu(idx, off)
    out.sum().backward()
    torch.cuda.synchronize()
    d = (gpu.weights - w0).view(-1, 32)
    assert torch.allclose(d[5], torch.full((32,), -2.0, device=dev))
    assert torch.allclose(d[7], torch.full((32,), -1.0, device=dev))
    assert float(d.abs().sum()) == pytest.approx(32 * 4.0)
    assert _lib.launch_count() > n0


@pytest.mark.gpu
def test_psw_grad_matches_reference():
    """Per-sample-weight gradient kernel vs autograd of F.embedding_bag."""
    import torch.nn.functional as F

    dev = torch.device("cuda:0")
    torch.manual_seed(3)
    from torchrec_b200.ops.tbe import OptimType, PoolingMode, TableBatchedEmbeddingBags

    B = 37
    t = TableBatchedEmbeddingBags([(100, 16), (50, 128)], [0, 1, 1], pooling_mode=PoolingMode.SUM, optimizer=OptimType.EXACT_SGD, learning_rate=0.0, device=dev)
    t.init_parameters([(-1, 1), (-1, 1)])
    lengths = torch.randint(0, 5, (3 * B,), device=dev)
    off = torch.cat([lengths.new_zeros(1), lengths.cumsum(0)])
    n = int(off[-1])
    rows = torch.tensor([100, 50, 50], device=dev).repeat_interleave(B).repeat_interleave(lengths)
    idx = (torch.rand(n, device=dev) * rows).long()
    psw = torch.rand(n, device=dev, requires_grad=True)
    out = t(idx, off, psw, batch_size=B)
    gout = torch.randn_like(out)
    (out * gout).sum().backward()
    ws = t.split_embedding_weights()
    psw2 = psw.detach().clone().requires_grad_()
    refs = []
    for f, tb in enumerate([0, 1, 1]):
        lo, hi = int(off[f * B]), int(off[(f + 1) * B])
        o = off[f * B : (f + 1) * B] - lo
        refs.append(F.embedding_bag(idx[lo:hi], ws[tb].float(), o, mode="sum", per_sample_weights=psw2[lo:hi]))
    ref = torch.cat(refs, 1)
    torch.testing.assert_close(out.float(), ref, atol=1e-4, rtol=1e-4)
    (ref * gout).sum().backward()
    torch.testing.assert_close(psw.grad, psw2.grad, atol=1e-4, rtol=1e-4)


@pytest.mark.gpu
@pytest.mark.parametrize("opt", [T.OptimType.EXACT_SGD, T.OptimType.EXACT_ROWWISE_ADAGRAD])
@pytest.mark.parametrize("dim,gdtype", [(128, torch.bfloat16), (64, torch.float32), (256, torch.float32)])
def test_fused_backward_unique_rows_fast_path(opt, dim, gdtype):
    """Large tables -> (almost) all ids distinct: exercises the one-hot forward and the unique-rows backward fast paths,
    mixed with a tiny table whose chunks take the generic walk."""
    dev = torch.device("cuda:0")
    specs = [(200_000, dim), (7, dim), (150_000, dim)]
    fmap = [0, 1, 2]
    B = 1000
    torch.manual_seed(5)
    cpu = T.TableBatchedEmbeddingBags(specs, fmap, optimizer=opt, learning_rate=0.05, eps=1e-3)
    gpu = T.TableBatchedEmbeddingBags(specs, fmap, optimizer=opt, learning_rate=0.05, eps=1e-3, device=dev, output_dtype=gdtype)
    gpu.weights.data.copy_(cpu.weights.data)
    g = torch.Generator().manual_seed(0)
    for step in range(2):
        idx = torch.cat([torch.randint(0, r, (B,), generator=g) for r, _ in specs])
        off = torch.arange(0, 3 * B + 1)
        og = gpu(idx.to(dev), off.to(dev), None, batch_size=B)
        oc = cpu(idx, off, None, batch_size=B)
        torch.testing.assert_close(og.float().cpu(), oc, rtol=2e-2 if gdtype == torch.bfloat16 else 1e-5, atol=2e-2 if gdtype == torch.bfloat16 else 1e-5)
        proj = torch.randn(B, 3 * dim, generator=g)
        og.backward(proj.to(dev).to(gdtype))
        oc.backward(proj.to(gdtype).float())
        torch.testing.assert_close(gpu.weights.cpu(), cpu.weights, rtol=1e-4, atol=1e-5)
        if gpu.state1 is not None:
            torch.testing.assert_close(gpu.state1.cpu(), cpu.state1, rtol=1e-4, atol=1e-6)


@pytest.mark.gpu
@pytest.mark.parametrize("vec", [4, 8])
@pytest.mark.parametrize("sdtype", [torch.bfloat16, torch.float32])
def test_grad_push_kernel_single_gpu(vec, sdtype):
    """The NVLink gradient scatter with both 'ranks' mapped to local buffers: checks the chunk addressing, scaling and casting."""
    from torchrec_b200.parallel.p2p import grad_push

    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    B, W = 37, 2
    widths = [16, 8, 24, 8]          # unit widths; units 0,2 -> rank 0, units 1,3 -> rank 1
    owner = [0, 1, 0, 1]
    src_cols = [0, 16, 24, 48]
    src = torch.randn(B, 56, device=dev).to(sdtype)
    pitch = 40
    inbox = [torch.zeros(W * B, pitch, dtype=torch.bfloat16, device=dev) for _ in range(W)]
    chunks, dst_c = [], [0, 0]
    for u, (w, r, sc) in enumerate(zip(widths, owner, src_cols)):
        for k in range(0, w, vec):
            chunks.append([r, sc + k, dst_c[r] + k])
        dst_c[r] += w
    ct = torch.tensor(chunks, dtype=torch.int32, device=dev)
    my_rank = 1
    grad_push(src, ct, [t.data_ptr() for t in inbox], torch.bfloat16, pitch, my_rank * B, 0.5, vec)
    torch.cuda.synchronize()
    exp0 = torch.cat([src[:, 0:16], src[:, 24:48]], 1).float() * 0.5
    exp1 = torch.cat([src[:, 16:24], src[:, 48:56]], 1).float() * 0.5
    torch.testing.assert_close(inbox[0][B : 2 * B, :40].float(), exp0.to(torch.bfloat16).float(), rtol=1e-2, atol=1e-2)
    torch.testing.assert_close(inbox[1][B : 2 * B, :16].float(), exp1.to(torch.bfloat16).float(), rtol=1e-2, atol=1e-2)
    assert float(inbox[0][:B].abs().sum()) == 0.0 and float(inbox[1][B:, 16:].abs().sum()) == 0.0


@pytest.mark.parametrize("wdtype,ulp", [(torch.bfloat16, 2.0**-7), (torch.float16, 2.0**-10)])
def test_stochastic_rounding_kernel_is_unbiased(wdtype, ulp):
    """Low-precision tables: an update of ulp/16 per step is lost by round-to-nearest and kept in expectation by the kernel's
    stochastic rounding (reproducible for a given sr_seed)."""
    dev = torch.device("cuda:0")

    def run(sr: bool, seed: int = 7):
        tbe = T.TableBatchedEmbeddingBags([(256, 128)], optimizer=T.OptimType.EXACT_SGD, learning_rate=1.0, weights_precision=wdtype, output_dtype=torch.float32,
                                          stochastic_rounding=sr, sr_seed=seed, device=dev)
        with torch.no_grad():
            tbe.weights.fill_(1.0)
        idx, off = torch.arange(256, device=dev), torch.arange(257, device=dev)
        g = torch.full((256, 128), -ulp / 16, device=dev)
        for _ in range(32):
            tbe(idx, off).backward(g)
        return tbe.weights.float().cpu()

    assert torch.equal(run(False), torch.ones(256 * 128))
    w = run(True)
    assert abs(w.mean().item() - (1.0 + 2 * ulp)) < 0.05 * ulp          # 32 steps x ulp/16 = 2 ulp on average
    assert set(w.unique().tolist()) <= {1.0 + k * ulp for k in range(0, 20)} and w.unique().numel() >= 3  # Binomial(32, 1/16) steps up
    assert torch.equal(w, run(True))                                      # same seed, same noise
    assert not torch.equal(w, run(True, seed=8))
