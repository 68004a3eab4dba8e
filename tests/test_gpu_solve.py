"""-m gpu: the triangular solve below the shared-memory limit, smk_chol_solve_* (chol_solve_kernel<T>, csrc/solve.cu), at
the shapes every Factor.solve caller runs it at, on the device's own factor of a GP covariance (helpers.gp_factor).

One CTA per (sample, group of RB right-hand sides) holds its group in shared memory (RB = 4 float32, 2 float64) and
walks the factor in diagonal blocks of NB (128 float32, 64 float64), applying the stored block inverses winv.  The
cases put N on both sides of every block edge up to Npad = 14 080, the largest size the kernel takes (226 KB of shared
memory in float32, 225 KB in float64); F on both sides of the group edges up to 1000; S = 1, 3 and 40 (the grid pass's
sample chunk); and the right-hand-side layouts of the callers:
  a   one y for every sample, y_stride = 0, mean subtracted (the grid pass, the time GP; F > 1 with ldy = N);
  b   per-sample y, y_stride = N, mean NULL (the refinement's K^-1 kx);
  c0  the pending fantasies, y_stride = F ldy, ldy = N, mean subtracted;
  c5  the same with ldy = N + 5, NaN in the gaps;
  d   the identity as F = N right-hand sides, mean NULL, alpha only (ML-II's K^-1), float64;
with all three outputs, alpha only, or alpha NULL (the forward pass only: sum_log_diag and quad).  The factors are
Matern52, D = 4, noise 1e-2, and one badly conditioned factor per dtype, SE, D = 2, N = 1000, noise ILL (1e-6 in float64;
1e-4 in float32, the smallest power of ten that keeps the device's float32 factor of that input positive definite: at
1e-5 it meets a non-positive pivot), so that the NB c term of the alpha bound is exercised.  Every output buffer starts
as NaN and is one element longer than the call may write.  The module takes about 100 s on an H100, most of it the
host references of the four N = 14 080 cases.

Bounds (helpers.check_solve), stated before running, per checked column:
  alpha         componentwise backward error <= max(32 x scipy's, 4 (N + NB c)), c the Skeel condition of the diagonal
                blocks;
  quad          within max(32 x scipy's own inconsistency, 4 N u) relative;
  sum_log_diag  within 4 N u sum |log L_ii|;
  padding rows of alpha exactly 0.
smk_chol_solve_gm_* runs on the same inputs and is held to the same bounds (the two sum in different orders, so they are
not compared bit for bit).  Worst measured fraction of each bound (record_property), H100 80GB HBM3 at a 700 W power
limit, both entries alike:
  alpha  0.013 (float64, N = 1); 5e-4 from N = 2 on; the badly conditioned cases 8e-7 (their NB c is large);
  quad   0.955 (float64, N = 1, where the bound is 4 u and the kernel multiplies by the stored 1 / L_11 instead of
         dividing); 0.18 from N = 2 on;
  sld    0.125 (float32, N = 1); 0.024 from N = 2 on;
  leading block of a joint factor: alpha 5e-5, quad 0.014, sld 0.010.
The public entry must advance smk_launch_count() by exactly 1 on every case: the shared-memory kernel ran, not the
global-memory solve (at N = 14 080 that is the 226 KB / 225 KB configuration).

Bitwise invariants (torch.equal), shared-memory entry unless noted:
  1. item s of a batch of 3 or 40 equals that sample solved alone;
  2. column f of an F-column call equals that column solved with F = 1, f at 0, RB - 1, RB and F - 1 (each right-hand
     side has its own accumulators, whatever its group); the same for smk_chol_solve_gm_* across its FB = 1 / 4 / 8
     groupings;
  3. NaN in the strict upper triangle of L, in the strict upper triangle of every winv block, in y past what is read
     and in the ldy gaps changes nothing;
  4. the forward-only call returns sum_log_diag and quad equal to the full call's, the alpha-only call alpha;
  5. both entries: under n_lead < N, NaN in rows >= n_lead of L and winv changes nothing (joint factors of
     n_lead = 63, 64, 65, 2040 observed and P = 3, 10 pending points).
Argument codes of both entries: every check runs before any launch.
"""
import functools

import numpy as np
import pytest

from tests.helpers import SOLVE_NB as NBS, Worst, check_solve, cur_stream, gp_factor, lib

pytestmark = pytest.mark.gpu

RB = {"f32": 4, "f64": 2}                # right-hand sides per CTA (SolveCfg<T>::RB)
ILL = {"f32": 1e-4, "f64": 1e-6}         # noise of the badly conditioned factor (SE, D = 2, N = 1000)


@pytest.fixture(scope="module")
def engs():
    import torch
    from spearmint_b200.engine import GPEIEngine
    return {"f32": GPEIEngine(dtype=torch.float32), "f64": GPEIEngine(dtype=torch.float64)}


_engs = {}


@pytest.fixture(scope="module", autouse=True)
def _bind(engs):
    _engs.update(engs)
    yield
    _factored.cache_clear()


@functools.lru_cache(maxsize=1)
def _factored(prec, N, S, seed, Ntot=None, ill=False):
    """(eng, A, winv, hb, y) of helpers.gp_factor: Matern52, D = 4, noise 1e-2, or SE, D = 2, noise ILL."""
    eng = _engs[prec]
    if ill:
        return (eng,) + gp_factor(eng, N, S, seed, Ntot, "SE", 2, ILL[prec])
    return (eng,) + gp_factor(eng, N, S, seed, Ntot)


def _run(entry, eng, N, S, F, L, winv, y, y_stride, ldy, mean, outs="all"):
    """One call with every output buffer NaN and one element longer than the call may write.  outs: "all", "alpha"
    (sum_log_diag and quad NULL) or "fwd" (alpha NULL).  Returns ((alpha [S][F][Npad], sld [S], quad [S][F]), None for
    a NULL output; the launches counted)."""
    import torch
    from spearmint_b200.engine import check, fn, ptr
    Npad = L.shape[-1]

    def buf(n, on):
        return torch.full((n + 1,), float("nan"), dtype=eng.dtype, device=eng.device) if on else None

    bufs = (buf(S * F * Npad, outs != "fwd"), buf(S, outs != "alpha"), buf(S * F, outs != "alpha"))
    n0 = lib().smk_launch_count()
    check(fn(entry, eng.dtype)(N, Npad, S, F, ptr(L), ptr(winv), ptr(y), y_stride, ldy, ptr(mean),
                               *[ptr(b) for b in bufs], cur_stream()), entry)
    launches = lib().smk_launch_count() - n0
    out = []
    for b, shape, what in zip(bufs, ((S, F, Npad), (S,), (S, F)), ("alpha", "sum_log_diag", "quad")):
        if b is not None:
            assert bool(torch.isnan(b[-1])), "%s wrote past the end of %s" % (entry, what)
            b = b[:-1].view(shape)
        out.append(b)
    return tuple(out), launches


def _same(a, b):
    import torch
    return all((x is None and y is None) or torch.equal(x, y) for x, y in zip(a, b))


def _rhs(eng, layout, N, S, F, y, hb, seed):
    """The right-hand sides of a layout: (y on the device, the same with NaN in every element the solve must not read,
    y_stride, ldy, mean or None).  y: the standardised observations of the factor."""
    rs = np.random.RandomState(seed)
    ldy = N + 5 if layout == "c5" else N
    mean = hb.mean if layout in ("a", "c0", "c5") else None
    if layout == "a":
        h, y_stride = np.tile(y[:N], (F, 1)) + (0.1 * rs.randn(F, N) if F > 1 else 0.0), 0
    elif layout == "b":
        h, y_stride = rs.randn(S, N), N
    elif layout == "d":
        h, y_stride = np.eye(N), 0
    else:
        h, y_stride = np.zeros((S, F, ldy)), F * ldy
        h[:, :, :N] = y[:N] + 0.3 * rs.randn(S, F, N)
    h = h.reshape(-1)
    clean = np.concatenate([h, np.zeros(7)])            # 7 elements past the last one any sample reads
    read = np.zeros(clean.shape, dtype=bool)
    for s in range(S if y_stride else 1):
        for f in range(F):
            read[s * y_stride + f * ldy:s * y_stride + f * ldy + N] = True
    poisoned = np.where(read, clean, np.nan)
    return eng.to_dev(clean), eng.to_dev(poisoned), y_stride, ldy, mean


def _cols(F, rb):
    """Columns held to the reference: every one of a small F, else both ends of the first two groups, of a middle group
    and of the last two."""
    if F <= 3 * rb:
        return list(range(F))
    m, last = F // 2 // rb * rb, (F - 1) // rb * rb
    return sorted({0, rb - 1, rb, 2 * rb - 1, m, m + rb - 1, last - 1, last, F - 1})


# (prec, N, F, S, layout, outs, ill): every N, F and S of the module docstring at least once, the layouts and output
# combinations spread over them
CASES = [("f32", 1, 1, 1, "a", "all", False), ("f32", 2, 2, 1, "c0", "all", False),
         ("f32", 127, 3, 3, "c5", "alpha", False), ("f32", 128, 4, 1, "a", "all", False),
         ("f32", 129, 5, 3, "c5", "all", False), ("f32", 255, 1, 3, "b", "fwd", False),
         ("f32", 256, 8, 1, "a", "alpha", False), ("f32", 257, 9, 3, "c0", "fwd", False),
         ("f32", 1000, 3, 1, "a", "all", True),
         ("f32", 2047, 1, 40, "a", "all", False), ("f32", 2047, 1, 3, "b", "all", False),
         ("f32", 2047, 101, 1, "c5", "all", False), ("f32", 4097, 1000, 1, "c0", "alpha", False),
         ("f32", 14080, 1, 1, "a", "all", False), ("f32", 14080, 5, 1, "c5", "fwd", False),
         ("f64", 1, 2, 1, "a", "all", False), ("f64", 63, 3, 3, "c5", "all", False),
         ("f64", 64, 1, 1, "b", "all", False), ("f64", 64, 64, 1, "d", "alpha", False),
         ("f64", 65, 100, 1, "c0", "all", False), ("f64", 65, 65, 1, "d", "alpha", False),
         ("f64", 127, 101, 1, "a", "alpha", False), ("f64", 128, 1, 3, "b", "fwd", False),
         ("f64", 129, 3, 1, "c5", "fwd", False), ("f64", 191, 2, 3, "a", "all", False),
         ("f64", 1000, 3, 1, "a", "all", True),
         ("f64", 1025, 101, 1, "c5", "all", False), ("f64", 1025, 1025, 1, "d", "alpha", False),
         ("f64", 4097, 3, 1, "c0", "all", False), ("f64", 4097, 4097, 1, "d", "alpha", False),
         ("f64", 14080, 1, 1, "a", "all", False), ("f64", 14080, 3, 1, "c5", "alpha", False)]


def _id(c):
    return "%s-N%d-F%d-S%d-%s-%s%s" % (c[0], c[1], c[2], c[3], c[4], c[5], "-ill" if c[6] else "")


@pytest.mark.parametrize("prec,N,F,S,layout,outs,ill", CASES, ids=[_id(c) for c in CASES])
def test_solve_shapes(record_property, prec, N, F, S, layout, outs, ill):
    import torch
    eng, A, winv, hb, y = _factored(prec, N, S, N % 97, None, ill)
    Npad, nb, rb = A.shape[-1], NBS[prec], RB[prec]
    assert Npad <= 14080
    yd, yd_nan, y_stride, ldy, mean = _rhs(eng, layout, N, S, F, y, hb, N + F)
    call = functools.partial(_run, N=N, S=S, F=F, y_stride=y_stride, ldy=ldy, mean=mean)

    full, n = call("smk_chol_solve", eng, L=A, winv=winv, y=yd)
    assert n == 1, "smk_chol_solve took %d launches: not the shared-memory kernel" % n
    gm, _ = call("smk_chol_solve_gm", eng, L=A, winv=winv, y=yd)
    if outs != "all":                               # 4. alpha only / forward only: the same bits as the full call
        part, n = call("smk_chol_solve", eng, L=A, winv=winv, y=yd, outs=outs)
        assert n == 1
        want = (full[0], None, None) if outs == "alpha" else (None, full[1], full[2])
        assert _same(part, want), "the %s call differs from the full call" % outs

    # 3. NaN where the solve must not read
    Lp, Wp = A.clone(), winv.clone()
    Lp.masked_fill_(torch.ones((Npad, Npad), dtype=torch.bool, device=A.device).triu_(1), float("nan"))
    Wp.masked_fill_(torch.ones((nb, nb), dtype=torch.bool, device=A.device).triu_(1), float("nan"))
    poisoned, _ = call("smk_chol_solve", eng, L=Lp, winv=Wp, y=yd_nan)
    assert _same(poisoned, full), "NaN outside the system reached the result"
    del Lp, Wp, poisoned

    # 1. batch items alone
    for s in sorted({0, 1, S - 1}) if S > 1 else []:
        one, _ = _run("smk_chol_solve", eng, N, 1, F, A[s:s + 1], winv[s:s + 1], yd[s * y_stride:], y_stride, ldy,
                      None if mean is None else mean[s:s + 1])
        assert _same(one, tuple(None if t is None else t[s:s + 1] for t in full)), "item %d of %d" % (s, S)

    # 2. columns alone, both entries
    for f in sorted({0, rb - 1, rb, F - 1} & set(range(F))) if F > 1 else []:
        for entry, ref in (("smk_chol_solve", full), ("smk_chol_solve_gm", gm)):
            one, _ = call(entry, eng, L=A, winv=winv, y=yd[f * ldy:], F=1)
            assert torch.equal(one[0][:, 0], ref[0][:, f]), "%s: column %d of %d" % (entry, f, F)
            if ref[2] is not None:
                assert torch.equal(one[1], ref[1]) and torch.equal(one[2][:, 0], ref[2][:, f]), (entry, f)

    # accuracy of both entries against scipy on the device's L
    W = Worst(record_property)
    cols = _cols(F, rb)
    yh = yd.cpu().numpy()
    mh = None if mean is None else mean.cpu().numpy()
    for tag, (alpha, sld, quad) in (("smem", full), ("gm", gm)):
        a = alpha.cpu().numpy()
        assert not np.any(a[:, :, N:]), "%s: padding of alpha" % tag
    for s in sorted({0, S // 2, S - 1}):
        Lh = np.tril(A[s, :N, :N].cpu().numpy())
        Wh = winv[s].cpu().numpy()
        b = np.stack([yh[s * y_stride + f * ldy:s * y_stride + f * ldy + N] for f in cols], axis=1)
        if mh is not None:
            b = b - mh[s]                           # element type: the device forms y - mean the same way
        for tag, (alpha, sld, quad) in (("smem", full), ("gm", gm)):
            fr = check_solve(prec, Lh, Wh, b, alpha[s][cols][:, :N].T.cpu().numpy(),
                             None if quad is None else quad[s][cols].cpu().numpy(),
                             None if sld is None else float(sld[s]), "%s %s N=%d F=%d s=%d" % (tag, prec, N, F, s))
            for k, v in fr.items():
                W("%s_%s" % (tag, k), v)
        del Lh
    W.flush()


@pytest.mark.parametrize("prec", ["f32", "f64"])
@pytest.mark.parametrize("n_lead", [63, 64, 65, 2040])
@pytest.mark.parametrize("P", [3, 10])
def test_leading_block_ignores_rows_past_n_lead(record_property, prec, n_lead, P):
    """5. The observed block of a joint factor of n_lead + P points (pending points' observed solve), mean subtracted,
    both entries: within the bounds against the leading block, padding exactly 0, and the same bits after rows >= n_lead
    of L and of winv are set to NaN."""
    eng, A, winv, hb, y = _factored(prec, n_lead, 2, 11, n_lead + P)
    nb = NBS[prec]
    yd = eng.to_dev(y[:n_lead])
    Ap, Wp = A.clone(), winv.clone()
    Ap[:, n_lead:, :] = float("nan")
    b0, r0 = divmod(n_lead, nb)
    Wp[:, b0, r0:, :] = float("nan")
    Wp[:, b0 + 1:] = float("nan")
    W = Worst(record_property)
    mh = hb.mean.cpu().numpy()
    for entry in ("smk_chol_solve", "smk_chol_solve_gm"):
        lead, n = _run(entry, eng, n_lead, 2, 1, A, winv, yd, 0, n_lead, hb.mean)
        if entry == "smk_chol_solve":
            assert n == 1
        assert _same(lead, _run(entry, eng, n_lead, 2, 1, Ap, Wp, yd, 0, n_lead, hb.mean)[0]), \
            "%s: rows >= n_lead reached the result" % entry
        alpha, sld, quad = (t.cpu().numpy() for t in lead)
        assert not np.any(alpha[:, :, n_lead:]), "%s: padding of alpha" % entry
        for s in range(2):
            Ll = np.tril(A[s, :n_lead, :n_lead].cpu().numpy())
            b = (yd.cpu().numpy() - mh[s])[:, None]
            fr = check_solve(prec, Ll, winv[s].cpu().numpy(), b, alpha[s][:, :n_lead].T, quad[s], sld[s],
                             "%s %s lead %d + %d s=%d" % (entry, prec, n_lead, P, s))
            for k, v in fr.items():
                W("%s_%s" % ("gm" if entry.endswith("_gm") else "smem", k), v)
    W.flush()


@pytest.mark.parametrize("prec", ["f32", "f64"])
@pytest.mark.parametrize("entry", ["smk_chol_solve", "smk_chol_solve_gm"])
def test_argument_codes(engs, prec, entry):
    """Every argument code of both entries, each returned before any launch, on valid small buffers; alpha NULL is
    refused by the global-memory entry (-11, alpha is its working vector) and accepted by the public one below the
    limit (the forward pass only)."""
    import torch
    from spearmint_b200.engine import fn, ptr
    eng = engs[prec]
    N, Npad, S, F, nb = 100, 128, 2, 3, NBS[prec]
    dev, dt = eng.device, eng.dtype
    L = torch.eye(Npad, dtype=dt, device=dev).repeat(S, 1, 1)
    winv = torch.eye(nb, dtype=dt, device=dev).repeat(S, Npad // nb, 1, 1)
    y = torch.ones((F * N,), dtype=dt, device=dev)
    alpha = torch.zeros((S, F, Npad), dtype=dt, device=dev)
    sld = torch.zeros((S,), dtype=dt, device=dev)
    quad = torch.zeros((S, F), dtype=dt, device=dev)
    good = dict(N=N, Npad=Npad, S=S, F=F, L=ptr(L), winv=ptr(winv), y=ptr(y), y_stride=0, ldy=N, mean=None,
                alpha=ptr(alpha), sld=ptr(sld), quad=ptr(quad))
    order = ["N", "Npad", "S", "F", "L", "winv", "y", "y_stride", "ldy", "mean", "alpha", "sld", "quad"]
    f = fn(entry, dt)

    def rc(**kw):
        a = dict(good, **kw)
        n0 = lib().smk_launch_count()
        r = f(*[a[k] for k in order], cur_stream())
        return r, lib().smk_launch_count() - n0

    r, n = rc()
    assert r == 0 and (n == 1 if entry == "smk_chol_solve" else n > 1)
    bad = [(-1, dict(N=0)), (-1, dict(N=-5)), (-2, dict(Npad=64)), (-2, dict(Npad=192)), (-3, dict(S=0)),
           (-4, dict(F=0)), (-5, dict(L=None)), (-6, dict(winv=None)), (-7, dict(y=None)), (-9, dict(ldy=N - 1))]
    if entry == "smk_chol_solve_gm":
        bad += [(-11, dict(alpha=None)), (-3, dict(S=65536))]
    for code, kw in bad:
        assert rc(**kw) == (code, 0), (entry, kw)
    if entry == "smk_chol_solve":
        assert rc(alpha=None) == (0, 1)
    torch.cuda.synchronize()
