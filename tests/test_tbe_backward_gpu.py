"""Fused embedding backward (csrc/tbe_bwd.cu) and per-sample-weight gradient (csrc/tbe_psw_grad.cu) against a float64 oracle.

The oracle lives in this file and is written from the optimizer definitions (the semantics of ``apply_row`` in tbe_bwd.cu, including
the order of clipping and weight decay). It does not use ``tbe._ref_*``: those are the library's own CPU path.

Exact comparisons. Gradients are drawn from the dyadic grid k / 64 (|k| <= 64) and per-sample weights from {0.5, 1, 2}, so every
gradient term is j / 128 with |j| <= 256. A sum of N such terms is an integer multiple of 1/128 below 256 N / 128 in magnitude; it is
exact in fp32 while 256 N <= 2^24, i.e. for N <= 65536 occurrences of one row. Every case keeps the occurrences of a row below that
bound (the largest run is 30 000), so each partial sum the kernels form is exact and the summed gradient does not depend on the
summation order. Weights are drawn from the grid j / 2^14 (|j| <= 1024) and learning rates of exact tests are powers of two, so
``w - lr * g`` is exact in float64 and its single rounding to fp32 is what ``fmaf`` returns. Then:
  * OptimType.NONE: the dense gradient equals the float64 sum (torch.equal);
  * EXACT_SGD: the weights equal the float64 update rounded to fp32 once, then to the table dtype (bf16 / fp16 tables without
    stochastic rounding round the fp32 result to nearest).

Tolerances. Where the optimizer itself rounds (Adagrad, Adam, LAMB, LARS, Lion) the bound is derived from fp32 rounding, unit
roundoff u = 2^-24. A row reduction (sum of g^2 over D, norms) is a per-lane sum of 4 * MAXV terms followed by a 5-level shuffle tree,
so its relative error is at most (4 * MAXV + 6) u (all terms non-negative). Each further operation of the update (scaling, add, sqrt,
division, the final fma) adds at most a few u relative to its operands. Every updated value x therefore satisfies
    |x_kernel - x_oracle| <= c * k * u * (|x_before| + |x_after - x_before|),   c = 4 * MAXV + 40,
at step k (k scales the error carried in through state from earlier steps). MEAN pooling divides by the bag length in fp32 and then
accumulates with one rounding per term, so a summed gradient of cnt terms is within (cnt + 2) u sum|term| of the exact sum. These
bounds are below 1e-4 of the update, while one dropped or doubled gradient piece (at least 1/128 in some element) moves a summed
gradient by more than 1e-3 of its size in every case here.
"""
import pytest
import torch

from torchrec_b200.ops import tbe as T

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
U = 2.0 ** -24
O = T.OptimType
NONE, SGD, RWADA, ADAGRAD, LARS, LION = 8, 0, 1, 2, 7, 9
WD_NONE, WD_L2, WD_DECOUPLE = 0, 1, 2
DTYPE_PAIRS = [(torch.float32, torch.float32), (torch.float32, torch.bfloat16), (torch.bfloat16, torch.float32),
               (torch.bfloat16, torch.bfloat16), (torch.float16, torch.float32), (torch.float16, torch.bfloat16)]


# ---- inputs ---------------------------------------------------------------------------------------------------------------------
def _dyadic_grad(gen, shape, dtype):
    return (torch.randint(-64, 65, shape, generator=gen).double() / 64).to(dtype).to(DEV)


def _dyadic_weights(gen, n, dtype):
    return (torch.randint(-1024, 1025, (n,), generator=gen).double() / 16384).to(dtype).to(DEV)


def _dyadic_psw(gen, n):
    return torch.tensor([0.5, 1.0, 2.0])[torch.randint(0, 3, (n,), generator=gen)].to(DEV)


def _batch(ids_per_feature, B, gen, idx_dtype=torch.int64, empty_frac=0.1, shuffle=True):
    """Split each feature's ids into B bags of random lengths (about ``empty_frac`` of them empty)."""
    vals, lens = [], []
    for ids in ids_per_feature:
        n = ids.numel()
        if shuffle:
            ids = ids[torch.randperm(n, generator=gen)]
        cuts = torch.sort(torch.randint(0, n + 1, (B - 1,), generator=gen)).values
        lengths = torch.cat([torch.zeros(1, dtype=torch.int64), cuts, torch.tensor([n])]).diff()
        for j in torch.nonzero(torch.rand(B - 1, generator=gen) < empty_frac).flatten().tolist():
            lengths[j + 1] += lengths[j]
            lengths[j] = 0
        vals.append(ids)
        lens.append(lengths)
    offsets = torch.cat([torch.zeros(1, dtype=torch.int64), torch.cat(lens).cumsum(0)])
    return torch.cat(vals).to(idx_dtype).to(DEV), offsets.to(idx_dtype).to(DEV)


def _states(opt, weights, total_rows):
    kinds = T._OPT_STATE[opt]
    return [None if k is None else torch.zeros(total_rows if k == "row" else weights.numel(), dtype=torch.float32, device=DEV) for k in kinds]


def _maxv(max_dim):
    return 1 if max_dim <= 128 else (4 if max_dim <= 512 else 16)


# ---- float64 oracle -------------------------------------------------------------------------------------------------------------
def _pooled_terms(meta, idx, off, psw, grad, B, mean):
    """Per feature: valid row ids and their gradient terms grad[bag] * psw (/ L for MEAN), float64."""
    idx, off = idx.long(), off.long()
    out = []
    for f in range(meta.num_features):
        D, rows, col = meta.h_dim[f], meta.h_rows[f], meta.h_col[f]
        o = off[f * B : (f + 1) * B + 1]
        lengths = o[1:] - o[:-1]
        lo, hi = int(o[0]), int(o[-1])
        bag = torch.repeat_interleave(torch.arange(B, device=DEV), lengths, output_size=hi - lo)
        s = torch.ones(hi - lo, dtype=torch.float64, device=DEV)
        if psw is not None:
            s = s * psw[lo:hi].double()
        if mean:
            s = s / lengths[bag].clamp(min=1).double()
        ids = idx[lo:hi]
        ok = (ids >= 0) & (ids < rows)
        out.append((f, ids[ok], grad[bag[ok], col : col + D].double() * s[ok, None]))
    return out


def _seq_terms(meta, idx, off, grad, B):
    idx, off = idx.long(), off.long()
    first, out = int(off[0]), []
    for f in range(meta.num_features):
        lo, hi = int(off[f * B]), int(off[(f + 1) * B])
        ids = idx[lo:hi]
        ok = (ids >= 0) & (ids < meta.h_rows[f])
        out.append((f, ids[ok], grad[lo - first : hi - first].double()[ok]))
    return out


def _row_sums(meta, terms):
    """Sum the terms per unique (table, row) with index_add_ in float64; also the sum of |term| and the count."""
    groups = {}
    for f, ids, g in terms:
        grp = groups.setdefault(meta.h_woff[f], (f, [], []))
        grp[1].append(ids)
        grp[2].append(g)
    res = []
    for f, ids_l, g_l in groups.values():
        ids, g = torch.cat(ids_l), torch.cat(g_l)
        if ids.numel() == 0:
            continue
        rows, inv = torch.unique(ids, return_inverse=True)
        D = meta.h_dim[f]
        gs = torch.zeros(rows.numel(), D, dtype=torch.float64, device=DEV).index_add_(0, inv, g)
        gabs = torch.zeros_like(gs).index_add_(0, inv, g.abs())
        cnt = torch.bincount(inv, minlength=rows.numel()).double()
        res.append(dict(f=f, rows=rows, g=gs, gabs=gabs, cnt=cnt))
    return res


def _assert_exact_fp32(sums):
    for r in sums:
        assert torch.equal(r["g"], r["g"].float().double()), "test inputs break the exact-sum bound"


class Oracle:
    """float64 copy of a TBE's flat weights and optimizer state, updated from the optimizer definitions, with the accumulated fp32
    error bound of every element (see the module docstring)."""

    def __init__(self, meta, weights, states, opt, wd_mode, hyper):
        self.meta, self.opt, self.wdm = meta, opt, wd_mode
        self.hp = torch.tensor(hyper, dtype=torch.float32).double().tolist()  # the kernel reads fp32 hyper-parameters
        self.w = weights.double().clone()
        self.s = [None if s is None else s.double().clone() for s in states]
        self.tol_w = torch.zeros_like(self.w)
        self.tol_s = [None if s is None else torch.zeros_like(s) for s in self.s]
        self.c = 4 * _maxv(meta.max_dim) + 40
        self.k = 0

    def _set(self, i, index, new):
        old = self.s[i][index]
        self.tol_s[i][index] += self.c * self.k * U * (old.abs() + (new - old).abs())
        self.s[i][index] = new

    def step(self, sums, mean=False):
        assert not mean or self.opt in (SGD, NONE), "the MEAN bound is derived for SGD and the dense gradient only"
        self.k += 1
        lr, eps, b1, b2, wd, step, maxg, mom = self.hp
        opt, wdm = self.opt, self.wdm
        S1, S2 = self.s
        for r in sums:
            f, rows = r["f"], r["rows"]
            D = self.meta.h_dim[f]
            key = self.meta.h_rowbase[f] + rows
            e = self.meta.h_woff[f] + rows[:, None] * D + torch.arange(D, device=DEV)
            g = r["g"]
            gerr = (r["cnt"][:, None] + 2) * U * r["gabs"] if mean else torch.zeros_like(g)
            if maxg > 0:
                g = g.clamp(-maxg, maxg)
            if opt == NONE:
                S1[e] += g
                self.tol_s[0][e] += gerr
                continue
            w_old = self.w[e]
            w = w_old.clone()
            if wdm == WD_L2:
                g = g + wd * w
            if wdm == WD_DECOUPLE and opt in (SGD, RWADA, ADAGRAD, LARS):
                w = w * (1 - lr * wd)
            if opt == SGD:
                w = w - lr * g
            elif opt == RWADA:
                ns = S1[key] + (g * g).sum(1) / D
                self._set(0, key, ns)
                w = w - (lr / (ns.sqrt() + eps))[:, None] * g
            elif opt == ADAGRAD:
                ns = S1[e] + g * g
                self._set(0, e, ns)
                w = w - lr * g / (ns.sqrt() + eps)
            elif opt in (3, 4, 5, 6):
                m = b1 * S1[e] + (1 - b1) * g
                self._set(0, e, m)
                if opt in (4, 6):
                    vr = b2 * S2[key] + (1 - b2) * (g * g).sum(1) / D
                    self._set(1, key, vr)
                    v = vr[:, None].expand_as(g)
                else:
                    v = b2 * S2[e] + (1 - b2) * g * g
                    self._set(1, e, v)
                upd = (m / (1 - b1**step)) / ((v / (1 - b2**step)).sqrt() + eps)
                if opt in (5, 6) or wdm == WD_DECOUPLE:
                    upd = upd + wd * w
                if opt in (5, 6):
                    un, wn = upd.norm(dim=1), w.norm(dim=1)
                    upd = upd * torch.where((un > 0) & (wn > 0), wn / un, torch.ones_like(un))[:, None]
                w = w - lr * upd
            elif opt == LION:
                m = S1[e]
                u = torch.sign(b1 * m + (1 - b1) * g)
                if wdm == WD_DECOUPLE:
                    u = u + wd * w
                w = w - lr * u
                self._set(0, e, b2 * m + (1 - b2) * g)
            elif opt == LARS:
                eta = mom if mom > 0 else 0.001
                gn, wn = g.norm(dim=1), w.norm(dim=1)
                ratio = torch.where((gn > 0) & (wn > 0), eta * wn / (gn + wd * wn + eps), torch.ones_like(gn))
                w = w - lr * ratio[:, None] * g
            self.tol_w[e] += self.c * self.k * U * (w_old.abs() + (w - w_old).abs()) + lr * gerr
            self.w[e] = w

    def assert_weights(self, w, exact, what="weights", allow_frac=0.0):
        if exact:
            exp = self.w.float().to(w.dtype)
            bad = w != exp
            assert not bad.any(), f"{what}: {int(bad.sum())} of {w.numel()} elements differ from the exactly rounded update"
            self.w = exp.double()  # the next step starts from the stored (rounded) rows
            return
        _assert_within(w, self.w, self.tol_w, w.dtype, what, allow_frac)

    def assert_state(self, i, s, exact=False, what=None, allow_frac=0.0):
        what = what or f"state{i + 1}"
        if exact:
            bad = s != self.s[i].float()
            assert not bad.any(), f"{what}: {int(bad.sum())} of {s.numel()} elements differ from the exact sum"
            return
        _assert_within(s, self.s[i], self.tol_s[i], s.dtype, what, allow_frac)


def _assert_within(x, ref64, tol, dtype, what, allow_frac=0.0):
    if dtype in (torch.bfloat16, torch.float16):  # the stored value is additionally rounded to nearest in the table dtype
        tol = tol + ref64.abs() * (2.0 ** -8 if dtype == torch.bfloat16 else 2.0 ** -11)
    err = (x.double() - ref64).abs()
    bad = err > tol
    frac = float(bad.double().mean())
    assert frac <= allow_frac, (f"{what}: {int(bad.sum())} of {x.numel()} elements outside the fp32 bound, worst |err| - bound = "
                                f"{float((err - tol).max()):.3e}")


def _kernel_step(meta, w, states, opt, wdm, hyper, idx, off, psw, grad, B, mean, seq=False):
    hdev = torch.tensor(hyper, dtype=torch.float32, device=DEV)
    s1, s2 = states
    if seq:
        T.sequence_backward(meta, w, s1, s2, hdev, hyper, opt, wdm, idx, off, B, grad)
    else:
        T.fused_backward(meta, w, s1, s2, hdev, hyper, opt, wdm, idx, off, psw, B, mean, grad=grad)


def _hyper(lr=2.0 ** -4, eps=1e-3, b1=0.9, b2=0.999, wd=0.0, step=0.0, maxg=0.0, momentum=0.0):
    return [lr, eps, b1, b2, wd, step, maxg, momentum]


def _check_one_step(meta, weights, opt, idx, off, psw, grad, B, mean=False, hyper=None, seq=False):
    """One backward from a fresh state: NONE and EXACT_SGD compare exactly, other optimizers within the fp32 bound."""
    hyper = hyper or _hyper()
    states = _states(opt, weights, meta.total_rows)
    if opt == NONE:
        states[0] = torch.zeros(weights.numel(), dtype=torch.float32, device=DEV)
    oracle = Oracle(meta, weights, states, opt, WD_NONE, hyper)
    terms = _seq_terms(meta, idx, off, grad, B) if seq else _pooled_terms(meta, idx, off, psw, grad, B, mean)
    sums = _row_sums(meta, terms)
    if not mean:
        _assert_exact_fp32(sums)
    oracle.step(sums, mean)
    _kernel_step(meta, weights, states, opt, WD_NONE, hyper, idx, off, psw, grad, B, mean, seq)
    torch.cuda.synchronize()
    exact = not mean and opt in (NONE, SGD)
    if opt == NONE:
        oracle.assert_state(0, states[0], exact=exact, what="dense gradient")
    else:
        oracle.assert_weights(weights, exact)
        for i, s in enumerate(states):
            if s is not None:
                oracle.assert_state(i, s)


# ---- a. hot-row spans -----------------------------------------------------------------------------------------------------------
SPAN_COUNTS = [1, 31, 32, 33, 64, 65, 767, 768, 769, 800, 4096, 30000]
N_COLD = 7  # rows 0..6 once each: every run of the hot rows (sorted after them) starts off a multiple of 32
INVALID = [-1, -5]  # with rows and rows + 9 (added per table): invalid ids sort last


def _span_ids(rows, counts, n_cold, gen, n_invalid):
    ids = [torch.arange(n_cold)]
    ids += [torch.full((c,), n_cold + i, dtype=torch.int64) for i, c in enumerate(counts)]
    bad = torch.tensor(INVALID + [rows, rows + 9])
    ids.append(bad[torch.randint(0, bad.numel(), (n_invalid,), generator=gen)])
    starts = (torch.tensor([n_cold] + counts[:-1]).cumsum(0)).tolist()
    return torch.cat(ids), starts


@pytest.mark.parametrize("opt", [NONE, SGD, RWADA])
@pytest.mark.parametrize("gdtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("idx_dtype", [torch.int32, torch.int64])
def test_hot_row_spans(opt, gdtype, idx_dtype):
    """Runs of 1 .. 30 000 occurrences of one row, each starting off a 32-position chunk boundary: the chunk walk, the warp span
    combine (<= 24 chunks) and the block-wide long-span kernel (> 768 occurrences). 70 invalid ids fill the last chunks (at least one
    chunk holds invalid ids only) and make the position count odd."""
    gen = torch.Generator().manual_seed(11)
    rows, D, B = 64, 128, 1024
    ids, starts = _span_ids(rows, SPAN_COUNTS, N_COLD, gen, 70)
    assert all(s % 32 != 0 for s in starts) and ids.numel() % 32 != 0 and max(SPAN_COUNTS) <= 65536
    meta = T.TbeMeta.build([rows], [D], [0], DEV)
    idx, off = _batch([ids], B, gen, idx_dtype)
    psw = _dyadic_psw(gen, idx.numel())
    grad = _dyadic_grad(gen, (B, D), gdtype)
    w = _dyadic_weights(gen, rows * D, torch.float32)
    _check_one_step(meta, w, opt, idx, off, psw, grad, B)


@pytest.mark.parametrize("opt", [NONE, SGD, RWADA])
def test_more_long_spans_than_sms(opt):
    """200 rows x 800 occurrences: more long spans than the H100 has SMs, so the long-span kernel's grid-stride loop runs."""
    gen = torch.Generator().manual_seed(12)
    rows, D, B = 256, 32, 2048
    ids, _ = _span_ids(rows, [800] * 200, 13, gen, 45)
    assert 200 > torch.cuda.get_device_properties(DEV).multi_processor_count
    meta = T.TbeMeta.build([rows], [D], [0], DEV)
    idx, off = _batch([ids], B, gen)
    grad = _dyadic_grad(gen, (B, D), torch.float32)
    w = _dyadic_weights(gen, rows * D, torch.float32)
    _check_one_step(meta, w, opt, idx, off, _dyadic_psw(gen, idx.numel()), grad, B)


# ---- b. embedding dims ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dims", [[4], [128], [132], [512], [516], [1024], [2048], [8, 512], [4, 2048]], ids=lambda d: "x".join(map(str, d)))
@pytest.mark.parametrize("opt", [NONE, SGD, RWADA])
def test_dims(dims, opt):
    """Every instantiation (D <= 128, <= 512, <= 2048) and the walk / no-walk split. In mixed-dim TBEs the narrow table runs through
    the wide table's instantiation. The widest table has hot rows with long runs (800 and 1500 occurrences)."""
    gen = torch.Generator().manual_seed(sum(dims))
    rows, B = 3000, 256
    meta = T.TbeMeta.build([rows] * len(dims), dims, list(range(len(dims))), DEV)
    feats = []
    for t in range(len(dims)):
        ids = [torch.randint(0, rows, (2000,), generator=gen), torch.full((100,), 17, dtype=torch.int64), torch.tensor([-1, rows, rows + 1])]
        if t == len(dims) - 1:
            ids += [torch.full((800,), 5, dtype=torch.int64), torch.full((1500,), 2999, dtype=torch.int64)]
        feats.append(torch.cat(ids))
    idx, off = _batch(feats, B, gen)
    grad = _dyadic_grad(gen, (B, meta.total_cols), torch.float32)
    w = _dyadic_weights(gen, sum(rows * d for d in dims), torch.float32)
    _check_one_step(meta, w, opt, idx, off, _dyadic_psw(gen, idx.numel()), grad, B)


def test_too_wide_rows_fail_before_any_update():
    """D = 2052 is wider than any instantiation: the backward raises and leaves every row and the dense gradient as they were."""
    gen = torch.Generator().manual_seed(9)
    meta = T.TbeMeta.build([50, 20], [8, 2052], [0, 1], DEV)
    idx, off = _batch([torch.randint(0, 50, (200,), generator=gen), torch.randint(0, 20, (200,), generator=gen)], 16, gen)
    grad = _dyadic_grad(gen, (16, meta.total_cols), torch.float32)
    for opt in (SGD, NONE):
        w = _dyadic_weights(gen, 50 * 8 + 20 * 2052, torch.float32)
        w0 = w.clone()
        states = [torch.zeros_like(w), None] if opt == NONE else [None, None]
        with pytest.raises(Exception, match="library error -2"):
            _kernel_step(meta, w, states, opt, WD_NONE, _hyper(), idx, off, None, grad, 16, False)
        torch.cuda.synchronize()
        assert torch.equal(w, w0) and (states[0] is None or not states[0].any())


# ---- c. multi-row walk kernel vs the generic walk -------------------------------------------------------------------------------
@pytest.mark.parametrize("opt", [SGD, RWADA])
@pytest.mark.parametrize("D", [4, 64, 128, 132, 512])
def test_walk_kernel_matches_generic_walk(opt, D):
    """SGD and row-wise Adagrad take tbe_bwd_walk_kernel. A max_gradient far above every gradient changes no value but sends every
    chunk to the generic walk instead (random fp32 gradients and per-sample weights, so a different summation order would show).
    SGD must give the same bits. Row-wise Adagrad's square sum may be contracted into a different fma chain in the two kernels: it
    differs by at most 2 (4 MAXV + 6) u relative (two bounds of the reduction error), which moves the multiplier lr / (sqrt(ns) + eps)
    by less than 16 u relative, so the stored weights differ by at most 32 u |update| plus one rounding step of the table dtype, and
    the row state by 32 u relative."""
    rows = 40_000
    for wdt, gdt in [(torch.float32, torch.float32), (torch.float32, torch.bfloat16), (torch.bfloat16, torch.float32), (torch.bfloat16, torch.bfloat16)]:
        gen = torch.Generator().manual_seed(D)
        meta = T.TbeMeta.build([rows, 5], [D, D], [0, 1, 0], DEV)
        B = 512
        feats = [torch.cat([torch.randint(0, rows, (1500,), generator=gen), torch.full((40,), 7, dtype=torch.int64)]),
                 torch.randint(0, 5, (600,), generator=gen),
                 torch.cat([torch.randint(0, rows, (1500,), generator=gen), torch.full((900,), 3, dtype=torch.int64)])]
        idx, off = _batch(feats, B, gen)
        psw = torch.rand(idx.numel(), generator=gen).to(DEV)
        w = (torch.randn((rows + 5) * D, generator=gen) * 0.1).to(wdt).to(DEV)
        states = _states(opt, w, meta.total_rows)
        for step in range(2):
            grad = torch.randn(B, 3 * D, generator=gen).to(gdt).to(DEV)
            w_prev, w_g, st_g = w.clone(), w.clone(), [None if s is None else s.clone() for s in states]
            _kernel_step(meta, w, states, opt, WD_NONE, _hyper(lr=0.05), idx, off, psw, grad, B, False)
            _kernel_step(meta, w_g, st_g, opt, WD_NONE, _hyper(lr=0.05, maxg=3e38), idx, off, psw, grad, B, False)
            torch.cuda.synchronize()
            where = f"{wdt} table, {gdt} gradient, step {step}"
            assert not torch.equal(w, w_prev), f"{where}: nothing was updated"
            if opt == SGD:
                nd = int((w != w_g).sum())
                assert nd == 0, f"{where}: {nd} weights differ between the walk and the generic walk"
                continue
            step_ulp = 2.0 ** -7 if wdt == torch.bfloat16 else 2.0 ** -23
            bound = 32 * U * (w_g.double() - w_prev.double()).abs() + step_ulp * w_g.double().abs()
            err = (w.double() - w_g.double()).abs()
            assert bool((err <= bound).all()), f"{where}: weights differ by up to {float((err - bound).max()):.3e} beyond the bound"
            s_err = (states[0].double() - st_g[0].double()).abs()
            assert bool((s_err <= 32 * U * st_g[0].double().abs()).all()), f"{where}: row states differ beyond 32 u"
            w.copy_(w_g)  # both runs continue from the same state
            states[0].copy_(st_g[0])


# ---- d. optimizer options -------------------------------------------------------------------------------------------------------
OPT_CASES = [(o, wdm, 0.0) for o in (O.EXACT_SGD, O.EXACT_ROWWISE_ADAGRAD, O.EXACT_ADAGRAD, O.ADAM, O.PARTIAL_ROWWISE_ADAM, O.LAMB,
                                      O.PARTIAL_ROWWISE_LAMB, O.LARS_SGD, O.LION) for wdm in (WD_NONE, WD_L2, WD_DECOUPLE)]
OPT_CASES += [(O.ADAMW, WD_NONE, 0.0), (O.LARS_SGD, WD_NONE, 0.02), (O.LARS_SGD, WD_L2, 0.02), (O.NONE, WD_NONE, 0.0)]


@pytest.mark.parametrize("clip", [False, True])
@pytest.mark.parametrize("opt,wdm,momentum", OPT_CASES, ids=lambda v: str(v))
def test_optimizer_options(opt, wdm, momentum, clip):
    """Three steps through the module, so optimizer state feeds back into later updates; ``clip`` sets max_gradient below the largest
    summed gradient. Mixed dims 8 / 132 / 64 share the D <= 512 instantiation; a 3-row table makes runs cross chunks."""
    gen = torch.Generator().manual_seed(21)
    specs, fmap, B = [(40, 8), (3, 132), (300, 64)], [0, 1, 2, 2], 300
    maxg = 1.5 if clip else 0.0
    tbe = T.TableBatchedEmbeddingBags(specs, fmap, optimizer=opt, learning_rate=0.05, eps=1e-3, weight_decay=0.01, weight_decay_mode=T.WeightDecayMode(wdm),
                                      max_gradient=maxg, momentum=momentum, device=DEV)
    with torch.no_grad():
        tbe.weights.copy_(_dyadic_weights(gen, tbe.weights.numel(), torch.float32))
    code = tbe.opt_code
    oracle = Oracle(tbe.meta, tbe.weights.detach(), [tbe.state1, tbe.state2], code, int(tbe.weight_decay_mode), tbe.hyper_host)
    lion = code == LION
    largest = 0.0
    for step in range(3):
        feats = [torch.randint(0, r, (B * 3,), generator=gen) for r in (40, 3, 300, 300)]
        idx, off = _batch(feats, B, gen)
        psw = _dyadic_psw(gen, idx.numel())
        grad = _dyadic_grad(gen, (B, tbe.meta.total_cols), torch.float32)
        out = tbe(idx, off, psw)
        out.backward(grad)
        torch.cuda.synchronize()
        sums = _row_sums(tbe.meta, _pooled_terms(tbe.meta, idx, off, psw, grad, B, False))
        _assert_exact_fp32(sums)
        largest = max(largest, max(float(r["g"].abs().max()) for r in sums))
        oracle.hp[T.HP_STEP] = tbe.hyper_host[T.HP_STEP]
        if code == NONE:
            oracle.s[0], oracle.tol_s[0] = torch.zeros_like(oracle.w), torch.zeros_like(oracle.w)
            oracle.step(sums)
            oracle.assert_state(0, tbe.weights.grad.view(-1), exact=True, what="dense gradient")
            tbe.weights.grad = None
            continue
        oracle.step(sums)
        # sign() is discontinuous: a pre-sign value within rounding of 0 may flip (2 lr in one element), and the flip reaches the
        # momentum through L2 decay
        allow = 5e-3 if lion else 0.0
        oracle.assert_weights(tbe.weights, exact=False, what=f"weights after step {step + 1}", allow_frac=allow)
        for i, s in enumerate((tbe.state1, tbe.state2)):
            if s is not None:
                oracle.assert_state(i, s, what=f"state{i + 1} after step {step + 1}", allow_frac=allow)
    if clip:
        assert largest > maxg, "max_gradient must clip something"


# ---- e. pooling and per-sample weights ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("opt", [NONE, SGD])
@pytest.mark.parametrize("mean", [False, True])
@pytest.mark.parametrize("weighted", [False, True])
def test_pooling_and_weights(opt, mean, weighted):
    """SUM / MEAN with and without per-sample weights, a third of the bags empty, invalid ids (-1, rows, rows + 9) in the first
    table, so an id equal to its table's row count must not reach row 0 of the next table."""
    gen = torch.Generator().manual_seed(31 + 2 * mean + weighted)
    specs, B = [(500, 64), (7, 32), (900, 128)], 200
    meta = T.TbeMeta.build([r for r, _ in specs], [d for _, d in specs], [0, 1, 2], DEV)
    feats = [torch.cat([torch.randint(0, 500, (600,), generator=gen), torch.tensor([-1, 500, 500, 509])]),
             torch.randint(0, 7, (500,), generator=gen),
             torch.cat([torch.randint(0, 900, (400,), generator=gen), torch.tensor([900, -3])])]
    idx, off = _batch(feats, B, gen, empty_frac=0.33)
    psw = _dyadic_psw(gen, idx.numel()) if weighted else None
    grad = _dyadic_grad(gen, (B, meta.total_cols), torch.float32)
    w = _dyadic_weights(gen, sum(r * d for r, d in specs), torch.float32)
    _check_one_step(meta, w, opt, idx, off, psw, grad, B, mean=mean)


@pytest.mark.parametrize("opt", [NONE, SGD])
def test_mean_long_bags(opt):
    """MEAN over bags of hundreds of ids (1/L is inexact), on a 5-row table whose rows run over many chunks."""
    gen = torch.Generator().manual_seed(41)
    B, D = 32, 64
    meta = T.TbeMeta.build([5], [D], [0], DEV)
    idx, off = _batch([torch.randint(0, 5, (B * 300,), generator=gen)], B, gen, empty_frac=0.0)
    assert int((off[1:] - off[:-1]).max()) >= 300
    grad = _dyadic_grad(gen, (B, D), torch.float32)
    _check_one_step(meta, _dyadic_weights(gen, 5 * D, torch.float32), opt, idx, off, _dyadic_psw(gen, idx.numel()), grad, B, mean=True)


# ---- f. (table, output) dtype pairs ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("wdtype,odtype", DTYPE_PAIRS, ids=lambda d: str(d).replace("torch.", ""))
def test_dtype_pairs_train(wdtype, odtype):
    """Every (table, output) pair the forward accepts trains: the pooled output and the updated rows are exact (round to nearest)."""
    gen = torch.Generator().manual_seed(51)
    specs, fmap, B = [(100, 64), (6, 16)], [0, 1, 1], 128
    tbe = T.TableBatchedEmbeddingBags(specs, fmap, optimizer=O.EXACT_SGD, learning_rate=2.0 ** -4, weights_precision=wdtype, output_dtype=odtype,
                                      stochastic_rounding=False, device=DEV)
    with torch.no_grad():
        tbe.weights.copy_(_dyadic_weights(gen, tbe.weights.numel(), wdtype))
    oracle = Oracle(tbe.meta, tbe.weights.detach(), [None, None], SGD, WD_NONE, tbe.hyper_host)
    for _ in range(2):
        feats = [torch.randint(0, r, (B * 4,), generator=gen) for r in (100, 6, 6)]
        idx, off = _batch(feats, B, gen)
        psw = _dyadic_psw(gen, idx.numel())
        out = tbe(idx, off, psw)
        ref = torch.zeros(B, tbe.meta.total_cols, dtype=torch.float64, device=DEV)
        for f, ids, _ in _pooled_terms(tbe.meta, idx, off, psw, torch.zeros(B, tbe.meta.total_cols, device=DEV), B, False):
            lo, hi = int(off[f * B]), int(off[(f + 1) * B])
            bag = torch.repeat_interleave(torch.arange(B, device=DEV), (off[f * B + 1 : (f + 1) * B + 1] - off[f * B : (f + 1) * B]).long(), output_size=hi - lo)
            D, col = tbe.meta.h_dim[f], tbe.meta.h_col[f]
            rows = oracle.w[tbe.meta.h_woff[f] : tbe.meta.h_woff[f] + specs[fmap[f]][0] * D].view(-1, D)
            ref[:, col : col + D].index_add_(0, bag, rows[idx[lo:hi].long()] * psw[lo:hi].double()[:, None])
        assert torch.equal(out, ref.float().to(odtype)), "pooled forward is not the exactly rounded sum"
        grad = _dyadic_grad(gen, (B, tbe.meta.total_cols), odtype)
        out.backward(grad)
        torch.cuda.synchronize()
        sums = _row_sums(tbe.meta, _pooled_terms(tbe.meta, idx, off, psw, grad, B, False))
        _assert_exact_fp32(sums)
        oracle.step(sums)
        oracle.assert_weights(tbe.weights, exact=True)


# ---- g. 64-bit sort keys --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("opt", [NONE, SGD])
def test_64bit_keys(opt):
    """A first table that declares 2^32 rows (so keys need 64 bits) but is only touched below row 16, backed by a small buffer; the
    second table's rows start at global row 2^32. Both must be updated at the right rows and nowhere else."""
    gen = torch.Generator().manual_seed(61)
    D0, D1, rows1, touched, B = 8, 16, 40, 16, 64
    big = 1 << 32
    woff, rows, rowbase, dims = [0, touched * D0], [big, rows1], [0, big], [D0, D1]
    n_elem = touched * D0 + rows1 * D1
    i64 = lambda v: torch.tensor(v, dtype=torch.int64, device=DEV)
    meta = T.TbeMeta(i64(woff), i64(rows), i64(rowbase), torch.tensor(dims, dtype=torch.int32, device=DEV), torch.tensor([0, D0], dtype=torch.int32, device=DEV),
                     woff, rows, rowbase, dims, [0, D0], max(dims), big + rows1, D0 + D1, 2)
    # (no invalid id >= 2^32 in the first table: a wrong validity check would turn it into a row far outside the small buffer)
    feats = [torch.cat([torch.randint(0, touched, (300,), generator=gen), torch.tensor([-1, -4])]),
             torch.cat([torch.randint(0, rows1, (300,), generator=gen), torch.tensor([rows1, -2])])]
    # every valid id stays inside the buffer: a mistake in this test cannot make the kernel write outside it
    for f, ids in enumerate(feats):
        ok = ids[(ids >= 0) & (ids < rows[f])]
        assert woff[f] + (int(ok.max()) + 1) * dims[f] <= (woff[f + 1] if f + 1 < len(woff) else n_elem)
    assert meta.total_rows >= (1 << 32) - 1
    idx, off = _batch(feats, B, gen)
    grad = _dyadic_grad(gen, (B, D0 + D1), torch.float32)
    w = _dyadic_weights(gen, n_elem, torch.float32)
    _check_one_step(meta, w, opt, idx, off, _dyadic_psw(gen, idx.numel()), grad, B)


# ---- h. per-sample-weight gradient ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("wdtype,gdtype", DTYPE_PAIRS, ids=lambda d: str(d).replace("torch.", ""))
@pytest.mark.parametrize("mean", [False, True])
def test_psw_grad(wdtype, gdtype, mean):
    """d psw[i] = <grad[bag(i)], W[idx[i]]> (/ L for MEAN) against float64, per element within D u sum_j |w_j g_j| (+ 2 u for the
    final scaling); invalid ids give exactly 0. Bags of up to 2000 ids, dims 4, 2048 and 132 in one TBE."""
    gen = torch.Generator().manual_seed(71)
    specs, B = [(50, 4), (30, 2048), (70, 132)], 12
    meta = T.TbeMeta.build([r for r, _ in specs], [d for _, d in specs], [0, 1, 2], DEV)
    feats = []
    for r, _ in specs:
        ids = torch.randint(0, r, (B * 700,), generator=gen)
        bad = torch.rand(ids.numel(), generator=gen) < 0.05
        feats.append(torch.where(bad, torch.tensor([-1, r])[torch.randint(0, 2, (ids.numel(),), generator=gen)], ids))
    idx, off = _batch(feats, B, gen, empty_frac=0.2)
    assert int((off[1:] - off[:-1]).max()) >= 2000
    w = torch.randn(sum(r * d for r, d in specs), generator=gen).to(wdtype).to(DEV)
    grad = torch.randn(B, meta.total_cols, generator=gen).to(gdtype).to(DEV)
    out = T.psw_grad(meta, w, idx, off, B, mean, grad=grad)
    torch.cuda.synchronize()
    offl, idxl = off.long(), idx.long()
    for f in range(meta.num_features):
        D, rows, col, wo = meta.h_dim[f], meta.h_rows[f], meta.h_col[f], meta.h_woff[f]
        o = offl[f * B : (f + 1) * B + 1]
        lengths = o[1:] - o[:-1]
        lo, hi = int(o[0]), int(o[-1])
        bag = torch.repeat_interleave(torch.arange(B, device=DEV), lengths, output_size=hi - lo)
        ids = idxl[lo:hi]
        ok = (ids >= 0) & (ids < rows)
        prod = w[wo : wo + rows * D].view(rows, D)[ids.clamp(0, rows - 1)].double() * grad[bag, col : col + D].double()
        scale = 1.0 / lengths[bag].clamp(min=1).double() if mean else torch.ones_like(bag, dtype=torch.float64)
        ref = prod.sum(1) * scale * ok
        bound = (D * U * prod.abs().sum(1) + 2 * U * ref.abs()) * scale
        got = out[lo:hi].double()
        assert torch.equal(got[~ok], torch.zeros_like(got[~ok])), f"feature {f}: invalid ids must give 0"
        err = (got - ref).abs()
        assert bool((err <= bound).all()), f"feature {f} (D = {D}): worst |err| - bound = {float((err - bound).max()):.3e}"


# ---- i. sequence (unpooled) backward --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("opt", [NONE, SGD, RWADA])
@pytest.mark.parametrize("gdtype", [torch.float32, torch.bfloat16])
def test_sequence_backward_long_runs(opt, gdtype):
    """PoolingMode.NONE: one gradient row per position. Two features share a table, and its hot row occurs 1 700 times."""
    gen = torch.Generator().manual_seed(81)
    D, B = 64, 48
    meta = T.TbeMeta.build([30, 200], [D, D], [0, 1, 1], DEV)
    feats = [torch.cat([torch.randint(0, 30, (400,), generator=gen), torch.tensor([-1, 30])]),
             torch.cat([torch.randint(0, 200, (500,), generator=gen), torch.full((900,), 123, dtype=torch.int64)]),
             torch.cat([torch.full((800,), 123, dtype=torch.int64), torch.tensor([200, -7])])]
    idx, off = _batch(feats, B, gen)
    grad = _dyadic_grad(gen, (idx.numel(), D), gdtype)
    w = _dyadic_weights(gen, (30 + 200) * D, torch.float32)
    _check_one_step(meta, w, opt, idx, off, None, grad, B, seq=True)
