"""Both ends of the EI grid pass at the shapes it runs them at: the covariance build that feeds every factorisation, the
cross mean of the fantasies and of the time GP, the EI sweeps that turn the moments into EI, the column sum and the
top-k selection that decide what next() proposes, and the constrained chooser's probability of feasibility with its two
helpers.  Each kernel is compared with a float64 evaluation of its own device operands (the float32-rounded inputs
promoted to double), so that a bound measures the kernel's arithmetic and not the input rounding.  Every output buffer
starts as NaN (or another sentinel), so an element no kernel writes shows up, and so does one it should have left alone.

Several outputs are single roundings or fixed-order sums; those are checked bit for bit against the same operations on
the host.  The other bounds are a-priori, derived in the docstrings in units of u = 2^-24 (float32) or 2^-53 (float64);
the worst measured ratio to each bound is recorded with record_property and quoted in the test's docstring.
"""
import math

import numpy as np
import pytest
import scipy.special as sps

from tests.helpers import U32, U64, Worst, check_rows, cur_stream, frac, gen_bound, kern, lib, same

gpu = pytest.mark.gpu

KINDS4 = ("SE", "ARDSE", "Matern32", "Matern52")
TINY = 2.0 ** -1074                 # the smallest double denormal
SQ2PI = math.sqrt(2.0 * math.pi)


def _c128(n):
    return (n + 127) // 128 * 128


def _tdt(prec):
    import torch
    return torch.float64 if prec == "f64" else torch.float32


def _dev(a, dt):
    import torch
    return torch.as_tensor(np.ascontiguousarray(a), dtype=dt, device="cuda")


def _nan(shape, dt):
    import torch
    return torch.full(shape, float("nan"), dtype=dt, device="cuda")


def _h(t):
    """Device tensor -> host float64 (the device values promoted exactly)."""
    return None if t is None else t.double().cpu().numpy()


def _pad(a, ld):
    """a [..., n] embedded in [..., ld] with NaN past n."""
    out = np.full(a.shape[:-1] + (ld,), np.nan)
    out[..., :a.shape[-1]] = a
    return out


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


def _api():
    from spearmint_b200._lib import KINDS, check, fn, ptr
    lib()
    return KINDS, check, fn, ptr


# ==================================================================================================== 1. EI sweep
SWEEP_S = (1, 2, 3, 4, 5, 8, 40)
SWEEP_F = (1, 2, 3, 4, 5, 7, 8, 100)
SWEEP_M = (1, 255, 257)


def _moments(rs, S, F, M):
    """float64 moments aimed at where the sweep can go wrong: u = (best - mu) / s dense in [-4.05, -3.95] around the
    float32 / double switch (30 %), spread over [-37, 10] (55 %) and in the deep tail [-40, -37] where phi(u) is denormal
    (15 %); s from 1e-6 to 1e3; 6 % of the variances 0, -0.0 or -1e-4 (the tensor-core path produces negative var by
    design); log_time from -5 to 5.  Returns mu [S][F][M], var [S][M], best [S][F], log_time [S][M]."""
    sd = 10.0 ** rs.uniform(-6.0, 3.0, (S, M))
    pick = rs.rand(S, F, M)
    u = np.where(pick < 0.3, rs.uniform(-4.05, -3.95, pick.shape),
                 np.where(pick < 0.85, rs.uniform(-37.0, 10.0, pick.shape), rs.uniform(-40.0, -37.0, pick.shape)))
    best = rs.randn(S, F)
    mu = best[:, :, None] - u * sd[:, None, :]
    var = sd * sd
    bad = rs.rand(S, M) < 0.06
    var[bad] = np.array([0.0, -0.0, -1e-4])[rs.randint(0, 3, int(bad.sum()))]
    return mu, var, best, rs.uniform(-5.0, 5.0, (S, M))


def _sweep(prec, M, S, F, ops, ldm, ei=True, start=None, want_max=False, lt=False, weighted=False):
    """One smk_ei_sweep_* (or _weighted_*) call with NaN-filled ei [S][ldm]; ei_sum starts as `start` (host [ldm]).
    Returns host (ei, ei_sum, ei_max as uint64 bits)."""
    import torch
    _, check, fn, ptr = _api()
    e = _nan((S, ldm), torch.float64) if ei else None
    es = None if start is None else _dev(start, torch.float64)
    em = torch.full((S,), 0x5EED, dtype=torch.int64, device="cuda") if want_max else None
    name = "smk_ei_sweep_weighted" if weighted else "smk_ei_sweep"
    extra = ops["w"] if weighted else (ops["lt"] if lt else None)
    check(fn(name, _tdt(prec))(M, S, F, ptr(ops["mu"]), ptr(ops["var"]), ldm, ptr(ops["best"]), ptr(extra), ptr(e),
                               ptr(es), ptr(em), cur_stream()), name)
    return (_h(e), _h(es), None if em is None else em.cpu().numpy().view(np.uint64))


def _ei_ref(b, m, v, f32):
    """Host EI of one sample: b [F], m [F][n], v [n] (device values in float64).  Returns per-fantasy EI [F][n] by the
    reference's formula s (u Phi(u) + phi(u)) (OPT:551-555; max(best - mu, 0) where var <= 0), the magnitude T [F][n]
    (below), the per-fantasy bound [F][n] and the float32-branch mask [F][n] of ei_one_f32.

    Bound of one term, derived for each evaluator and summed over the two (kernel and host), relative to the magnitude
    of the terms that cancel, T = s (|u| Phi(u) + phi(u)) (not to EI, which is T / u^2 in the tail).  One ulp is up to
    2 u relative.
      Phi = 0.5 erfc(-u / sqrt 2): erfc 5 ulp (10 u); the argument carries 1.5 u (one product, the rounded constant),
          which moves erfc(x) by |d ln erfc / d ln x| <= 2 x^2 + 2 = u^2 + 2 times that: (13 + 1.5 u^2) u relative;
      phi = exp(-u^2 / 2) / sqrt(2 pi): exp 1 ulp (2 u), the constant and its product 1.5 u, the rounded argument
          u^2 / 2 u: (3.5 + 0.5 u^2) u relative;
      the products u Phi, s (.) and the sum: 3 u of T; u itself (two roundings) moves EI by s Phi |du| <= 3 u T.
    Per evaluator 22.5 + 2 u^2, both: (46 + 4 u^2) u64 T.
    float32 branch (v > 0 and the float32 u > -4; the host predicts it exactly, the float32 operations being IEEE):
      s = sqrtf(v), best - mu and the division: 3 u32 T; erfcf 4 ulp (8 u32) and the argument's 1.6 u32 (u^2 + 2);
      expf 2 ulp (4 u32), the constant and its product 1.5 u32, the argument u^2 / 2 u32; fmaf and s (.): 2 u32 T.
      Total (22 + 2.2 u^2) u32 T, plus the host's (23 + 2 u^2) u64 T.
    Below u = -37 phi(u) and Phi(u) are denormal and lose their relative accuracy: each evaluator adds at most
    (8 |u| + 8) s denormal ulps (erfc's few ulps times |u|, the sum and the products), and one more for the rounding of
    the result to the denormal grid.
    scipy's ndtr returns 0 below u = -37.7 (it stops where exp(-u^2 / 2) would be denormal), so the host takes
    Phi(u) = 0.5 erfcx(-u / sqrt 2) exp(-u^2 / 2) below u = -37: erfcx to a few ulp, the same argument analysis."""
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        pos = v > 0
        s = np.sqrt(np.where(pos, v, 1.0))[None, :]
        u = (b[:, None] - m) / s
        Phi = _ndtr(u)
        phi = np.exp(-u ** 2 / 2.0) / SQ2PI
        e = np.where(pos, s * (u * Phi + phi), np.maximum(b[:, None] - m, 0.0))
        T = np.where(pos, s * (np.abs(u) * Phi + phi), 0.0)
        C = (46.0 + 4.0 * u * u) * U64
        br32 = np.zeros(m.shape, dtype=bool)
        if f32:
            f = np.float32
            fu = (f(b)[:, None] - m.astype(f)) / np.sqrt(v.astype(f))[None, :]
            br32 = pos[None, :] & (fu > f(-4.0))
            C = np.where(br32, (22.0 + 2.2 * u * u) * U32 + (23.0 + 2.0 * u * u) * U64, C)
        B = np.where(pos, C * T + 2.0 * ((8.0 * np.abs(u) + 8.0) * s + 1.0) * TINY, 0.0)
    return e, T, B, br32 & pos[None, :]


def _ndtr(x):
    """Phi(x) in float64, down to the denormal range (scipy's ndtr underflows to 0 below -37.7)."""
    with np.errstate(over="ignore", under="ignore"):
        return np.where(x < -37.0, 0.5 * sps.erfcx(-x / math.sqrt(2.0)) * np.exp(-x * x / 2.0), sps.ndtr(x))


def _check_ei(W, tag, prec, F, h, ei, cols, lt):
    """ei [S][ldm] (device) against the host reference on the candidates cols, every sample.
      mean over F: the kernel's F - 1 additions and the division, the host's pairwise sum: (2 F + 1) / F u64 sum_f T_f;
      log_time: exp 1 ulp (2 u) and the division (u), on both sides: 6 u64 |ref|, the rest divided by exp(log_time),
          and one denormal ulp for the division's rounding;
      var <= 0 without log_time: max(best - mu, 0) summed in f order, then / F, exactly."""
    S = ei.shape[0]
    for s in range(S):
        v = h["var"][s, cols]
        e, T, B, br32 = _ei_ref(h["best"][s], h["mu"][s][:, cols], v, prec == "f32")
        ref = e.sum(0) / F
        bound = B.sum(0) / F + (2.0 * F + 1.0) / F * U64 * T.sum(0)
        bad = ~(v > 0)
        if np.any(bad):                          # the kernel's fmax path, summed in f order like the kernel
            acc = np.zeros(int(bad.sum()))
            for f in range(F):
                acc = acc + np.maximum(h["best"][s, f] - h["mu"][s][f, cols[bad]], 0.0)
            ref[bad] = acc / F if F > 1 else acc
            bound[bad] = 0.0
        if lt:
            et = np.exp(h["lt"][s, cols])
            ref = ref / et
            bound = bound / et + 6.0 * U64 * np.abs(ref) + TINY
        got = ei[s, cols]
        W(tag + "_frac", frac(np.abs(got - ref), bound, "%s: EI of sample %d" % (tag, s)))
        assert np.all(got >= 0), "%s: negative EI in sample %d" % (tag, s)
        if prec == "f32" and F == 1 and not lt:
            # the switch sits at u = -4: on the float32 side every EI is a widened float32, on the double side (the
            # dense window [-4.05, -4]) none is (a double result lands on a float32 value with probability 2^-29)
            g = got[None, :]
            rep = np.float32(g).astype(np.float64) == g
            assert np.all(rep[br32]), "%s: a float32-branch EI is not a float32 value (sample %d)" % (tag, s)
            with np.errstate(invalid="ignore", divide="ignore"):
                u = (h["best"][s][:, None] - h["mu"][s][:, cols]) / np.sqrt(np.where(v > 0, v, 1.0))[None, :]
            win = (v > 0)[None, :] & ~br32 & (u > -4.05) & (g > 0)
            assert not np.any(rep[win]), "%s: a double-branch EI next to u = -4 is a float32 value" % tag


def _seq_sum(start, ei, M):
    """start + sum_s ei[s] in s order (the kernel's per-thread total), over j < M."""
    t = np.zeros(M)
    for s in range(ei.shape[0]):
        t = t + ei[s, :M]
    return start[:M] + t


def _max_bits(ei, M):
    mx = ei[:, :M].max(1)
    return np.where(mx > 0, _bits(mx), np.uint64(0))


def _sweep_case(W, tag, prec, S, F, M, ldm, rs, cols=None, lt_cases=(False, True), data=None):
    """The four calls of one shape (with ei and ei_sum, with ei_max too, ei only, ei_max only) and their invariants on
    every entry, then the accuracy on the candidates cols (default all)."""
    dt = _tdt(prec)
    mu, var, best, lt = _moments(rs, S, F, M) if data is None else data
    ops = {"mu": _dev(_pad(mu, ldm), dt), "var": _dev(_pad(var, ldm), dt), "best": _dev(best, dt),
           "lt": _dev(_pad(lt, ldm), dt)}
    h = {k: _h(t) for k, t in ops.items()}
    start = _pad(np.where(rs.rand(M) < 0.2, 0.0, 10.0 ** rs.uniform(-3, 3, M)), ldm)
    for with_lt in lt_cases:
        t = "%s_lt" % tag if with_lt else tag
        e1, s1, _ = _sweep(prec, M, S, F, ops, ldm, start=start, lt=with_lt)
        e2, s2, m2 = _sweep(prec, M, S, F, ops, ldm, start=start, want_max=True, lt=with_lt)
        e3, _, _ = _sweep(prec, M, S, F, ops, ldm, lt=with_lt)
        _, _, m4 = _sweep(prec, M, S, F, ops, ldm, ei=False, want_max=True, lt=with_lt)
        assert np.all(np.isfinite(e1[:, :M])), "%s: unwritten ei entries j < M" % t
        assert np.all(np.isnan(e1[:, M:])), "%s: ei entries j >= M were written (ldm = %d)" % (t, ldm)
        assert same(e2, e1) and same(e3, e1), "%s: ei differs with ei_max or without ei_sum" % t
        assert same(s1[:M], _seq_sum(start, e1, M)), "%s: ei_sum != start + sum_s ei[s] in s order" % t
        assert np.all(np.isnan(s1[M:])), "%s: ei_sum entries j >= M were written" % t
        assert same(s2, s1), "%s: ei_sum differs with ei_max" % t
        assert np.array_equal(m2, _max_bits(e1, M)), "%s: ei_max is not the bits of max_j ei" % t
        assert np.array_equal(m4, m2), "%s: ei_max differs without ei / ei_sum" % t
        _check_ei(W, t, prec, F, h, e1, np.arange(M) if cols is None else cols, with_lt)
    return ops, h, start


@gpu
@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_ei_sweep_shapes(record_property, prec):
    """smk_ei_sweep_* at S in {1, 2, 3, 4, 5, 8, 40} x F in {1, 2, 3, 4, 5, 7, 8, 100} x M in {1, 255, 257}, ldm =
    ceil128(M) + 128, with and without log_time: both sides of the 4-wide unrolls over samples (F = 1) and fantasies
    (F > 1) and their tails.  Exact on every entry: ei the same bits with and without ei_max and ei_sum; ei_sum = start
    + sum_s ei[s] in s order; ei_max the bits of max_j ei; entries j >= M untouched.  Accuracy: _ei_ref / _check_ei.
    Worst measured on an H100 80 GB HBM3 (SXM, 700 W power limit), as a fraction of the bound, float32 / float64: 0.5 / 0.5
    without log_time, 0.56 / 1.0 with it; the largest are single denormal ulps in the deep tail, where the bound is
    a denormal ulp or two.  Regression: ei_one returned EI a few denormal ulps below zero for u < -37.5."""
    W = Worst(record_property)
    rs = np.random.RandomState(11 if prec == "f32" else 12)
    for S in SWEEP_S:
        for F in SWEEP_F:
            for M in SWEEP_M:
                _sweep_case(W, "sweep", prec, S, F, M, _c128(M) + 128, rs)
    W.flush()


@gpu
@pytest.mark.parametrize("prec", ["f32", "f64"])
@pytest.mark.parametrize("S,F", [(40, 1), (4, 100)])
def test_ei_sweep_at_size(record_property, prec, S, F):
    """M = 100 010 (the headline grid plus the jitter cloud), ldm = ceil128(M) and ceil128(M) + 128, with and without
    log_time.  The exact invariants on every entry; the accuracy on the first and the last 256-thread block and 20 000
    random candidates.  Same bounds as test_ei_sweep_shapes.  Worst measured on an H100 80 GB HBM3 (SXM, 700 W power
    limit): 0.5 without log_time, 1.0 with it, in both precisions (single denormal ulps in the deep tail)."""
    W = Worst(record_property)
    M = 100010
    rs = np.random.RandomState(S * 1000 + F)
    data = _moments(rs, S, F, M)
    blk = (M - 1) // 256 * 256
    cols = np.unique(np.concatenate([np.arange(256), np.arange(blk, M), rs.choice(M, 20000, replace=False)]))
    for ldm in (_c128(M), _c128(M) + 128):
        _sweep_case(W, "at_size", prec, S, F, M, ldm, rs, cols=cols, data=data)
    W.flush()


# ==================================================================================================== 2. weighted, colsum
@gpu
@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_ei_sweep_weighted(prec):
    """smk_ei_sweep_weighted_* at the shapes of test_ei_sweep_shapes and at M = 100 010 (S = 4, F = 100), with w from 1
    down to 1e-300: the kernel forms ei_cand(...) * w, one rounding of the plain sweep's EI (the mean over the F
    fantasies first), so ei_w equals ei_plain * w (one float64 multiply on the host) bit for bit; ei_sum = start + sum_s
    ei_w[s] in s order; ei_max the bits of max_j ei_w; entries j >= M untouched."""
    rs = np.random.RandomState(21 if prec == "f32" else 22)
    cases = [(S, F, M) for S in SWEEP_S for F in SWEEP_F for M in SWEEP_M] + [(4, 100, 100010)]
    for S, F, M in cases:
        ldm = _c128(M) + 128
        t = "S%d F%d M%d" % (S, F, M)
        mu, var, best, lt = _moments(rs, S, F, M)
        w = 10.0 ** rs.uniform(-300, 0, (S, M))
        w[rs.rand(S, M) < 0.05] = 1.0
        dt = _tdt(prec)
        import torch
        ops = {"mu": _dev(_pad(mu, ldm), dt), "var": _dev(_pad(var, ldm), dt), "best": _dev(best, dt),
               "w": _dev(_pad(w, ldm), torch.float64)}
        start = _pad(10.0 ** rs.uniform(-3, 3, M), ldm)
        ep, _, _ = _sweep(prec, M, S, F, ops, ldm)
        ew, sw, mw = _sweep(prec, M, S, F, ops, ldm, start=start, want_max=True, weighted=True)
        ew3, _, _ = _sweep(prec, M, S, F, ops, ldm, weighted=True)
        assert np.all(np.isnan(ew[:, M:])) and np.all(np.isnan(sw[M:])), "%s: entries j >= M were written" % t
        assert same(ew[:, :M], ep[:, :M] * w), "%s: ei_w != ei_plain * w bit for bit" % t
        assert same(ew3, ew), "%s: ei_w differs without ei_sum / ei_max" % t
        assert same(sw[:M], _seq_sum(start, ew, M)), "%s: ei_sum != start + sum_s ei_w[s] in s order" % t
        assert np.array_equal(mw, _max_bits(ew, M)), "%s: ei_max is not the bits of max_j ei_w" % t


@gpu
@pytest.mark.parametrize("S", [1, 3, 40])
@pytest.mark.parametrize("M", [1, 255, 257, 100010])
def test_ei_colsum(S, M):
    """smk_ei_colsum (it sets the accuracy guard's scale): ei_sum[j] = start[j] + sum_s ei[s][j] in s order, bit for bit,
    at ldm = ceil128(M) + 128 with NaN past M in both ei and ei_sum (never read, never written)."""
    import torch
    _, check, _, ptr = _api()
    rs = np.random.RandomState(S + M)
    ldm = _c128(M) + 128
    ei = _pad(np.where(rs.rand(S, M) < 0.3, 0.0, 10.0 ** rs.uniform(-300, 3, (S, M))), ldm)
    start = _pad(10.0 ** rs.uniform(-3, 3, M), ldm)
    es, eid = _dev(start, torch.float64), _dev(ei, torch.float64)
    check(lib().smk_ei_colsum(M, S, ptr(eid), ldm, ptr(es), cur_stream()), "ei_colsum")
    got = es.cpu().numpy()
    assert same(got[:M], _seq_sum(start, ei, M)), "ei_sum != start + sum_s ei[s] in s order"
    assert np.all(np.isnan(got[M:])), "ei_sum entries j >= M were written"


# ==================================================================================================== 3. top-k
TOPK_M = (1, 2, 255, 256, 4095, 4096, 4097, 8191, 8192, 8193, 100010, 2 ** 20 + 3)
TOPK_K = (1, 2, 20, 255, 256)
PATTERNS = ("random", "equal", "ties", "last_slice", "zeros", "denormal", "neginf", "nan", "mostly_nan")


def _scores(pat, M, npdt, rs):
    """Score patterns: random; all equal; a few tied values with the maximum at indices 0, 4095, 4096, 8191 and M - 1
    (slice edges); the top values only in the last, partial 4096-slice; +-0.0 with some -1; denormals (1e-310 in float64,
    1e-40 in float32); half -inf; half NaN; all NaN but 100."""
    x = rs.rand(M)
    if pat == "equal":
        x[:] = 0.5
    elif pat == "ties":
        x = np.floor(rs.rand(M) * 20) / 20
        x[[i for i in (0, 4095, 4096, 8191, M - 1) if i < M]] = 1.0
    elif pat == "last_slice":
        x = 0.5 * x
        x[(M - 1) // 4096 * 4096:] += 1.0
    elif pat == "zeros":
        x = np.where(rs.rand(M) < 0.5, 0.0, -0.0)
        x[rs.rand(M) < 0.1] = -1.0
    elif pat == "denormal":
        x = x * (1e-310 if npdt == np.float64 else 1e-40)
    elif pat == "neginf":
        x[rs.rand(M) < 0.5] = -np.inf
    elif pat == "nan":
        x[rs.rand(M) < 0.5] = np.nan
    elif pat == "mostly_nan":
        keep = rs.choice(M, min(M, 100), replace=False)
        y = np.full(M, np.nan)
        y[keep] = x[keep]
        x = y
    return x.astype(npdt)


def _topk_order(score):
    """Non-NaN indices sorted by value descending, then by index ascending (the numpy first-max rule)."""
    idx = np.nonzero(~np.isnan(score))[0]
    return idx[np.lexsort((idx, -score[idx].astype(np.float64)))]


def _topk_expect(score, order, k):
    """The first k of order in ascending order; slots beyond the non-NaN count hold index -1 and value -inf (first)."""
    top = order[:k][::-1]
    ri = np.full(k, -1, dtype=np.int64)
    rv = np.full(k, -np.inf, dtype=score.dtype)
    ri[k - len(top):] = top
    rv[k - len(top):] = score[top]
    return ri, rv


def _topk(prec, M, k, score_d, ws_short=0):
    import torch
    _, _, fn, ptr = _api()
    nb = lib().smk_topk_workspace_bytes(M, k)
    ws = torch.empty((nb + 64,), dtype=torch.uint8, device="cuda")
    idx = torch.full((max(k, 1),), -77, dtype=torch.int32, device="cuda")
    val = _nan((max(k, 1),), _tdt(prec))
    rc = fn("smk_topk", _tdt(prec))(M, k, ptr(score_d), ptr(idx), ptr(val), ptr(ws), nb - ws_short, cur_stream())
    return rc, idx.cpu().numpy().astype(np.int64), val.cpu().numpy()


@gpu
@pytest.mark.parametrize("prec", ["f32", "f64"])
@pytest.mark.parametrize("M", TOPK_M)
def test_topk(prec, M):
    """smk_topk_* against the host order (value descending, index ascending; NaN never selected) for k in {1, 2, 20,
    255, 256, M} (k <= min(M, 256)) and every score pattern of _scores: the indices exactly, the values bit for bit
    (so +0.0 and -0.0 are told apart) and equal to score[idx].  Stage 1 sees a last slice with fewer entries than k at
    M = 4097 and 8193 (1 entry), and the stage-1 short-lists of several slices tie across slice boundaries.

    Contract when fewer than k scores are non-NaN: the missing slots are the first ones, with index -1 and value -inf
    (include/spearmint_b200.h).  The multi-round GPEIEngine.topk keeps it (test_engine_topk_multi_round).  Callers
    that can meet it: backend.top_mean_ei raises FloatingPointError on an index -1, the forest's argmax maps it to 0
    (numpy's argmax of all-NaN EI), and the accuracy guard's k = 1 call reads only the value; engine.tail_fix cannot
    meet it, since a NaN in the EI sum makes its max NaN and it returns before ranking."""
    npdt = np.float64 if prec == "f64" else np.float32
    rs = np.random.RandomState(M)
    ks = sorted({k for k in TOPK_K + (M,) if k <= min(M, 256)})
    for pat in PATTERNS:
        score = _scores(pat, M, npdt, rs)
        order = _topk_order(score)
        sd = _dev(score, _tdt(prec))
        for k in ks:
            rc, idx, val = _topk(prec, M, k, sd)
            assert rc == 0, "M %d k %d %s: rc %d" % (M, k, pat, rc)
            ri, rv = _topk_expect(score, order, k)
            assert np.array_equal(idx, ri), "M %d k %d %s: indices differ from the host order" % (M, k, pat)
            assert np.array_equal(val.view(np.uint32 if prec == "f32" else np.uint64),
                                  rv.view(np.uint32 if prec == "f32" else np.uint64)), \
                "M %d k %d %s: values differ from score[idx] bit for bit" % (M, k, pat)


@gpu
@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_topk_argument_codes(prec):
    """k = 257 (past kMaxK) and k > M give -2; a workspace one byte short of smk_topk_workspace_bytes gives -6."""
    sd = _dev(np.arange(300.0), _tdt(prec))
    assert _topk(prec, 300, 257, sd)[0] == -2
    assert _topk(prec, 10, 11, sd)[0] == -2
    assert _topk(prec, 300, 20, sd, ws_short=1)[0] == -6
    assert _topk(prec, 300, 20, sd)[0] == 0


@gpu
@pytest.mark.parametrize("M,k,pat", [
    (5000, 257, "ties"), (5000, 512, "ties"), (5000, 700, "ties"), (100010, 700, "ties"), (100010, 512, "random"),
    (800, 512, "nan400"), (800, 700, "neginf500"), (300, 300, "nan100"),
])
def test_engine_topk_multi_round(M, k, pat):
    """GPEIEngine.topk for k > 256 (several rounds, each masking what the earlier ones took) against the host order,
    with ties across the 256-entry round boundary (30 distinct values), and the contract of the single call when fewer
    than k scores are non-NaN (index -1, value -inf, first) or when the scores themselves hold -inf.

    Regression: the rounds used to mask taken entries with -inf, which a later round can select again: with 400 NaN
    scores of 800 and k = 512 the second round returned 112 of the first round's indices a second time (the chooser's
    top_mean_ei proposed duplicates), and with 500 genuine -inf scores the masked entries outranked them by index."""
    import torch
    from spearmint_b200.engine import GPEIEngine
    eng = GPEIEngine(dtype=torch.float64)
    rs = np.random.RandomState(M + k)
    score = np.floor(rs.rand(M) * 30) / 30 if pat == "ties" else rs.rand(M)
    if pat.startswith("nan"):
        score[rs.choice(M, int(pat[3:]), replace=False)] = np.nan
    if pat.startswith("neginf"):
        score[rs.choice(M, int(pat[6:]), replace=False)] = -np.inf
    idx, val = eng.topk(_dev(score, torch.float64), M, k)
    idx, val = idx.cpu().numpy().astype(np.int64), val.cpu().numpy()
    ri, rv = _topk_expect(score, _topk_order(score), k)
    assert np.array_equal(idx, ri), "indices differ from the host order"
    assert np.array_equal(_bits(val), _bits(rv)), "values differ from score[idx]"


# ==================================================================================================== 4. covariance build
COV_N = (1, 31, 32, 33, 127, 128, 129)
COV_D = (1, 31, 32, 33, 64, 65)


def _cov_ops(rs, N, D, S, dt):
    X = rs.rand(N, D)
    ils = 1.0 / rs.uniform(0.3, 2.0, (S, D))
    a2 = np.exp(0.25 * rs.randn(S))
    da = 10.0 ** rs.uniform(-4, -1, S)
    d = {"X": _dev(X, dt), "ils": _dev(ils, dt), "a2": _dev(a2, dt), "da": _dev(da, dt)}
    return d, {k: _h(t) for k, t in d.items()}


def _cov_ref(kind, h, Yh, s, rows, cols, u, self_diag, host_twice):
    """amp2 k(r2) [rows][cols] in float64 on the device operands, and the a-priori bound of each element: the
    SIMT-generator bound (helpers.gen_bound; the kernel scales both points, takes their difference and accumulates its
    square with fused multiply-adds, the form the bound covers) and, on the self case's diagonal, the rounding of
    amp2 fl(1e-6) + diag_add and of its sum with amp2 k(0) = amp2: u (amp2 1e-6 + |dg|) + u |val|.  host_twice (the
    float64 build): the host's float64 evaluation follows the same analysis, so its bound counts twice."""
    ils = h["ils"][s]
    Xs = h["X"][rows] * ils
    Ys = Yh[cols] * ils
    r2 = np.zeros((len(rows), len(cols)))
    for d in range(Xs.shape[1]):
        r2 += (Xs[:, d:d + 1] - Ys[None, :, d]) ** 2
    a2 = h["a2"][s]
    K = a2 * kern(kind, r2)
    nx, ny = np.sqrt((Xs * Xs).sum(1)), np.sqrt((Ys * Ys).sum(1))
    B = gen_bound(kind, r2, nx[:, None], ny[None, :], Xs.shape[1], a2, u)
    if self_diag:
        c = float(np.float32(1e-6)) if u == U32 else 1e-6
        dg = a2 * c + h["da"][s]
        on = rows[:, None] == cols[None, :]
        K = np.where(on, a2 + dg, K)
        B = B + np.where(on, u * (a2 * c + dg) + u * (a2 + dg), 0.0)
    return K, B * (2.0 if host_twice else 1.0)


@gpu
@pytest.mark.parametrize("prec", ["f32", "f64"])
@pytest.mark.parametrize("N", COV_N)
def test_cov_build_shapes(record_property, prec, N):
    """smk_cov_build_* (self and cross) and smk_cov_build_lower_* at N in {1, 31, 32, 33, 127, 128, 129} (the 32 x 32
    output-tile edges) x D in {1, 31, 32, 33, 64, 65} (the 32-wide D staging), the four kinds in turn, S = 40 every
    third case (else 1); self ld in {N, Npad, Npad + 128}, cross M in {1, 33, 1000} with ld in {M, ceil128(M) + 128}.
    Exact: the self build is bitwise symmetric and the identity on rows and columns [N, ld); the lower build equals the
    full one bit for bit on every 32-tile on or below the diagonal and leaves the strict-upper tiles as they were;
    the cross build leaves columns [M, ld) as they were.  Accuracy on samples 0 and S - 1: _cov_ref.
    Worst measured on an H100 80 GB HBM3 (SXM, 700 W power limit), as a fraction of the bound, float32 / float64: self 0.14 /
    0.072, cross 0.11 / 0.052."""
    import torch
    KINDS, check, fn, ptr = _api()
    dt = _tdt(prec)
    u = U32 if prec == "f32" else U64
    W = Worst(record_property)
    rs = np.random.RandomState(N + (0 if prec == "f32" else 1000))
    st = cur_stream()
    for i, D in enumerate(COV_D):
        c = COV_N.index(N) * len(COV_D) + i
        kind, S = KINDS4[c % 4], (40 if c % 3 == 0 else 1)
        Npad = _c128(N)
        ld = (N, Npad, Npad + 128)[(c // 2) % 3]
        M = (1, 33, 1000)[c % 3]
        ldc = (M, _c128(M) + 128)[(c // 3) % 2]
        t = "%s N%d D%d S%d ld%d" % (kind, N, D, S, ld)
        d, h = _cov_ops(rs, N, D, S, dt)
        full, low = _nan((S, ld, ld), dt), _nan((S, ld, ld), dt)
        check(fn("smk_cov_build", dt)(KINDS[kind], N, N, D, S, ptr(d["X"]), None, ptr(d["ils"]), ptr(d["a2"]),
                                      ptr(d["da"]), ptr(full), ld, st), "cov_build")
        check(fn("smk_cov_build_lower", dt)(KINDS[kind], N, D, S, ptr(d["X"]), ptr(d["ils"]), ptr(d["a2"]),
                                            ptr(d["da"]), ptr(low), ld, st), "cov_build_lower")
        Yd = _dev(rs.rand(M, D), dt)
        Yh = _h(Yd)
        cr = _nan((S, N, ldc), dt)
        check(fn("smk_cov_build", dt)(KINDS[kind], N, M, D, S, ptr(d["X"]), ptr(Yd), ptr(d["ils"]), ptr(d["a2"]),
                                      None, ptr(cr), ldc, st), "cov_build cross")
        full, low, cr = _h(full), _h(low), _h(cr)
        eye = np.eye(ld)
        ti, tj = np.arange(ld)[:, None] // 32, np.arange(ld)[None, :] // 32
        assert np.all(np.isfinite(full)), "%s: unwritten entries in the self build" % t
        assert np.array_equal(full, np.swapaxes(full, 1, 2)), "%s: the self build is not symmetric" % t
        assert np.array_equal(full[:, N:, :], np.broadcast_to(eye[N:], (S, ld - N, ld))), "%s: padding rows" % t
        assert np.array_equal(full[:, :, N:], np.broadcast_to(eye[:, N:], (S, ld, ld - N))), "%s: padding cols" % t
        assert same(low[:, ti >= tj], full[:, ti >= tj]), "%s: lower build != full build on its tiles" % t
        assert np.all(np.isnan(low[:, ti < tj])), "%s: lower build wrote a strict-upper tile" % t
        assert np.all(np.isfinite(cr[:, :, :M])) and np.all(np.isnan(cr[:, :, M:])), "%s: cross columns (M %d)" % (t, M)
        rows = np.arange(N)
        for s in sorted({0, S - 1}):
            K, B = _cov_ref(kind, h, h["X"], s, rows, rows, u, True, prec == "f64")
            W("self_frac", frac(np.abs(full[s, :N, :N] - K), B, "%s: self build, sample %d" % (t, s)))
            K, B = _cov_ref(kind, h, Yh, s, rows, np.arange(M), u, False, prec == "f64")
            W("cross_frac", frac(np.abs(cr[s, :, :M] - K), B, "%s: cross build M %d, sample %d" % (t, M, s)))
    W.flush()


@gpu
@pytest.mark.parametrize("prec,N,ld,lower", [("f32", 8192, 8192, False), ("f64", 4096, _c128(4097), True)])
def test_cov_build_at_size(record_property, prec, N, ld, lower):
    """The float32 self build at N = 8192, D = 32, S = 2 (the C5 configuration) and the float64 lower build of the
    headline log-likelihood (N = 4096 and the augmented row: ld = ceil128(4097)), Matern52, on helpers.check_rows.
    Exact on the whole matrix (on the device): nothing left unwritten, the self build symmetric, the lower build equal
    to the full one on its tiles and the strict-upper tiles untouched.  Same bound as test_cov_build_shapes.  Worst
    measured on an H100 80 GB HBM3 (SXM, 700 W power limit): 0.063 (float32), 0.035 (float64)."""
    import torch
    KINDS, check, fn, ptr = _api()
    dt = _tdt(prec)
    u = U32 if prec == "f32" else U64
    S, D, kind = 2, 32, "Matern52"
    rs = np.random.RandomState(N)
    d, h = _cov_ops(rs, N, D, S, dt)
    st = cur_stream()
    full = _nan((S, ld, ld), dt)
    check(fn("smk_cov_build", dt)(KINDS[kind], N, N, D, S, ptr(d["X"]), None, ptr(d["ils"]), ptr(d["a2"]),
                                  ptr(d["da"]), ptr(full), ld, st), "cov_build")
    assert not bool(torch.isnan(full).any()), "unwritten entries"
    assert torch.equal(full, full.transpose(1, 2)), "the self build is not symmetric"
    if lower:
        low = _nan((S, ld, ld), dt)
        check(fn("smk_cov_build_lower", dt)(KINDS[kind], N, D, S, ptr(d["X"]), ptr(d["ils"]), ptr(d["a2"]),
                                            ptr(d["da"]), ptr(low), ld, st), "cov_build_lower")
        t = torch.arange(ld, device="cuda") // 32
        on = (t[:, None] >= t[None, :]).expand(S, ld, ld)
        assert torch.equal(low[on], full[on]), "lower build != full build on its tiles"
        assert bool(torch.isnan(low[~on]).all()), "lower build wrote a strict-upper tile"
        del low
    rows = check_rows(N, ld, rs)
    W = Worst(record_property)
    for s in range(S):
        got = full[s][torch.as_tensor(rows, device="cuda")].double().cpu().numpy()
        r = rows[rows < N]
        eye = np.eye(ld)
        assert np.array_equal(got[rows >= N], eye[rows[rows >= N]]), "padding rows"
        assert np.array_equal(got[rows < N][:, N:], eye[r][:, N:]), "padding cols"
        K, B = _cov_ref(kind, h, h["X"], s, r, np.arange(N), u, True, prec == "f64")
        W("frac", frac(np.abs(got[rows < N][:, :N] - K), B, "sample %d" % s))
    W.flush()


# ==================================================================================================== 5. cross mean
CM_F = (1, 7, 8, 9, 16, 17, 100)
CM_N = (1, 7, 8, 9, 2047)
CM_M = (1, 33, 45, 97)
# the order raises the dynamic shared-memory attribute twice (float64 D >= 178, float32 D >= 364), then runs a small D
CM_D = {"f64": (1, 33, 177, 178, 200, 1, 33), "f32": (1, 33, 363, 364, 400, 1)}


@gpu
@pytest.mark.parametrize("prec", ["f64", "f32"])
def test_cross_mean_shapes(record_property, prec):
    """smk_cross_mean_* at F in {1, 7, 8, 9, 16, 17, 100} (the 8-wide F groups and their edges) for every D of CM_D in
    turn, N in {1, 7, 8, 9, 2047} (the 8 row-lanes), M ragged to the 32-candidate tile, S in {1, 40}, ldm = M + 5, alpha
    NaN past N (never read), mu NaN-filled (entries j >= M untouched).

    Bound of mu[s][f][j] = sum_n alpha_fn amp2 k(x_n, c_j) + mean: sum_n |alpha_fn| times the generator bound of each
    element (helpers.gen_bound), plus the summation: each of the 8 lanes strided over n takes ceil(N / 8) rounded fused
    multiply-adds, their 8-way reduction 8 more, each at most u sum_n |alpha_fn k_jn|, and the final + mean u (|mu| +
    |mean|).  float64: the host's float64 evaluation follows the same analysis (its dot product N roundings), so the
    generator bound counts twice and N more roundings are added.  Worst measured on an H100 80 GB HBM3 (SXM, 700 W power
    limit): 0.23 (float32), 0.074 (float64)."""
    KINDS, check, fn, ptr = _api()
    dt = _tdt(prec)
    u = U32 if prec == "f32" else U64
    W = Worst(record_property)
    rs = np.random.RandomState(5 if prec == "f64" else 6)
    c = 0
    for D in CM_D[prec]:
        for F in CM_F:
            N, M, S = CM_N[c % 5], CM_M[c % 4], (40 if c % 6 == 0 else 1)
            kind = KINDS4[c % 4]
            c += 1
            t = "%s D%d F%d N%d M%d S%d" % (kind, D, F, N, M, S)
            Npad, ldm = _c128(N), M + 5
            d, h = _cov_ops(rs, N, D, S, dt)
            Cd = _dev(rs.rand(M, D), dt)
            mean = _dev(0.1 * rs.randn(S), dt)
            al = np.full((S, F, Npad), np.nan)
            al[:, :, :N] = rs.randn(S, F, N) * 10.0 ** rs.uniform(-1, 2, (S, F, 1))
            ald = _dev(al, dt)
            mu = _nan((S, F, ldm), dt)
            check(fn("smk_cross_mean", dt)(KINDS[kind], N, Npad, M, D, S, F, ptr(d["X"]), ptr(Cd), ptr(d["ils"]),
                                           ptr(d["a2"]), ptr(mean), ptr(ald), ptr(mu), ldm, cur_stream()), "cross_mean")
            mu = _h(mu)
            assert np.all(np.isfinite(mu[..., :M])) and np.all(np.isnan(mu[..., M:])), "%s: entries j >= M" % t
            Ch, mh, ah = _h(Cd), _h(mean), _h(ald)
            for s in sorted({0, S - 1}):
                K, B = _cov_ref(kind, h, Ch, s, np.arange(N), np.arange(M), u, False, False)   # [N][M]
                a = ah[s, :, :N]
                ref = a.dot(K) + mh[s]
                acc = np.abs(a).dot(np.abs(K))
                nsum = -(-N // 8) + 8 + (N if prec == "f64" else 0)
                bound = np.abs(a).dot(B) * (2.0 if prec == "f64" else 1.0) + u * (nsum * acc + np.abs(ref) +
                                                                                 abs(mh[s]))
                W("frac", frac(np.abs(mu[s, :, :M] - ref), bound, "%s: sample %d" % (t, s)))
    W.flush()


# ==================================================================================================== 6. feasibility
CP_D = (1, 7, 8, 9, 16, 17, 32)
CP_N = (1, 63, 64, 65, 4097)
CP_M = (1, 127, 128, 129, 10010)
CP_KINDS = ("SE", "Matern32", "Matern52")


def _cp_call(prec, kind, N, Npad, M, D, S, d, Cd, ta, gain, ldm, want_m):
    import torch
    KINDS, check, fn, ptr = _api()
    p = _nan((S, ldm), torch.float64)
    m = _nan((S, ldm), torch.float64) if want_m else None
    check(fn("smk_constraint_prob", _tdt(prec))(KINDS[kind], N, Npad, M, D, S, ptr(d["X"]), ptr(Cd), ptr(d["ils"]),
                                                ptr(d["a2"]), ptr(ta), ptr(gain), ptr(p), ptr(m), ldm, cur_stream()),
          "constraint_prob")
    return _h(p), _h(m)


@gpu
@pytest.mark.parametrize("prec", ["f32", "f64"])
@pytest.mark.parametrize("N", CP_N)
def test_constraint_prob_shapes(record_property, prec, N):
    """smk_constraint_prob_* at N in {1, 63, 64, 65, 4097} (the 64-observation tiles) x D in {1, 7, 8, 9, 16, 17, 32}
    (the 8-wide D staging), M in {1, 127, 128, 129, 10 010} (the 128-candidate tiles) in turn, the three instantiations
    (SE, shared with ARDSE; Matern32; Matern52), S = 40 every fourth case, ldm = M + 7, t_alpha with entries of both
    signs around 1e4 (K_c^-1 ff is like that) and NaN past N.

    m = amp2 sum_n k_n t_n (m_out), all in float64: the scaled points, the differences and their fused squares are the
    generator's form, so each k_n is within helpers.gen_bound (amp2 = 1, u64); the sum takes ceil(N / 16) rounded fused
    multiply-adds per thread and a 16-way reduction, each at most u64 sum |k_n t_n|, and amp2 v one rounding.  The host's
    float64 evaluation follows the same analysis (its dot product N roundings).  So, in u64 amp2 units:
    2 sum_n |t_n| gb_n + (N + ceil(N / 16) + 17) sum_n |k_n t_n|, and 2 u64 |m|: the cancellation is the whole point.
    p = 0.5 erfc(-gain m / sqrt 2) against Phi(gain m_dev) on the host (_ndtr: scipy's ndtr, and below -37, where ndtr
    underflows to 0, 0.5 erfcx(-x / sqrt 2) exp(-x^2 / 2)), m_dev the device's own m, with gain chosen so that gain m
    reaches -38 (p denormal).  The argument of erfc carries 2.5 u64 on each side (the products gain m and (.) / sqrt 2,
    the rounded constant), which erfc magnifies by |d ln erfc / d ln x| <= 2 x^2 + 2 = (gain m)^2 + 2; erfc itself is
    within 5 ulp (10 u64) on each side: (30 + 5 (gain m)^2) u64 p relative, which is about 7 200 u64 at gain m = -38,
    and 8 denormal ulps for the roundings of a denormal result.  The bound is formed as p ((30 + 5 g^2 m^2) u64): the
    product u64 p underflows below p = 2e-292 and would leave only the absolute term, which the gradual-underflow range
    -37.7 < gain m < -37.5 (p between 1e-310 and 2.2e-308, still 40-odd significant bits) then exceeds.  p is also the
    same bits with m_out NULL.  Entries j >= M untouched.
    Worst measured on an H100 80 GB HBM3 (SXM, 700 W power limit), float32 inputs / float64: m 0.040 / 0.034 of the
    bound, with sum |k t| up to 2.2e5 times |m|; p 0.39 / 0.42."""
    import torch
    dt = _tdt(prec)
    W = Worst(record_property)
    rs = np.random.RandomState(N + (7 if prec == "f64" else 0))
    Npad = _c128(N)
    for i, D in enumerate(CP_D):
        c = CP_N.index(N) * len(CP_D) + i
        M, kind, S = CP_M[c % 5], CP_KINDS[c % 3], (40 if c % 4 == 0 else 1)
        t = "%s N%d D%d M%d S%d" % (kind, N, D, M, S)
        ldm = M + 7
        d, h = _cov_ops(rs, N, D, S, dt)
        Cd = _dev(rs.rand(M, D), dt)
        ta = np.full((S, Npad), np.nan)
        ta[:, :N] = 1e4 * rs.randn(S, N)
        tad = _dev(ta, torch.float64)
        p1, m1 = _cp_call(prec, kind, N, Npad, M, D, S, d, Cd, tad, _dev(np.ones(S), torch.float64), ldm, True)
        assert np.all(np.isfinite(m1[:, :M])) and np.all(np.isnan(m1[:, M:])), "%s: m_out entries" % t
        gain = 38.0 / np.maximum(np.abs(m1[:, :M]).max(1), 1e-300)
        gd = _dev(gain, torch.float64)
        p2, m2 = _cp_call(prec, kind, N, Npad, M, D, S, d, Cd, tad, gd, ldm, True)
        p3, _ = _cp_call(prec, kind, N, Npad, M, D, S, d, Cd, tad, gd, ldm, False)
        assert same(m2, m1), "%s: m depends on gain" % t
        assert same(p3, p2), "%s: p differs with m_out NULL" % t
        assert np.all(np.isfinite(p2[:, :M])) and np.all(np.isnan(p2[:, M:])), "%s: p entries" % t
        gm = gain[:, None] * m2[:, :M]
        ref = _ndtr(gm)
        W("p_frac", frac(np.abs(p2[:, :M] - ref), ref * ((30.0 + 5.0 * gm * gm) * U64) + 8.0 * TINY, t + ": p"))
        Ch = _h(Cd)
        cols = np.arange(M) if M <= 1000 else np.unique(np.concatenate([
            np.arange(0, M, 128), np.arange(127, M, 128), [M - 1], rs.choice(M, 200, replace=False)]))
        for s in sorted({0, S - 1}):
            K, B = _cov_ref(kind, h, Ch, s, np.arange(N), cols, U64, False, False)    # [N][m], amp2 included
            a2 = h["a2"][s]
            tt = ta[s, :N]
            ref = tt.dot(K)
            bound = 2.0 * np.abs(tt).dot(B) + U64 * ((N + -(-N // 16) + 17) * np.abs(tt).dot(np.abs(K)) +
                                                     2.0 * np.abs(ref))
            W("m_frac", frac(np.abs(m2[s, cols] - ref), bound, "%s: m, sample %d" % (t, s)))
            W("m_cancel", float((np.abs(tt).dot(np.abs(K)) / np.maximum(np.abs(ref), 1e-300 * a2)).max()))
    W.flush()


@gpu
@pytest.mark.parametrize("N", [1, 31, 32, 33, 4097])
def test_lower_matvec(record_property, N):
    """smk_lower_matvec_f64: out = L z reads only the lower triangle of L [Npad][Npad] and rows < N: NaN in the strict
    upper triangle, in rows >= N and in z past N still give a finite out[:N], and out[N:] stays untouched.
    Bound: each lane sums ceil((row + 1) / 32) products with fused multiply-adds, then 5 shuffle levels: (ceil((row + 1)
    / 32) + 5) u64 sum_k |L_rk z_k|, against math.fsum (the exact sum, rounded once: + 1 u64).  Worst measured on an
    H100 80 GB HBM3 (SXM, 700 W power limit): 0.21."""
    import torch
    _, check, _, ptr = _api()
    rs = np.random.RandomState(N)
    Npad = _c128(N) + (128 if N == 33 else 0)
    L = rs.randn(Npad, Npad)
    L[np.triu_indices(Npad, 1)] = np.nan
    L[N:] = np.nan
    z = rs.randn(Npad)
    z[N:] = np.nan
    out = _nan((Npad,), torch.float64)
    Ld, zd = _dev(L, torch.float64), _dev(z, torch.float64)        # alive until the kernel has read them
    check(lib().smk_lower_matvec_f64(N, Npad, ptr(Ld), ptr(zd), ptr(out), cur_stream()), "lower_matvec")
    out = out.cpu().numpy()
    assert np.all(np.isfinite(out[:N])) and np.all(np.isnan(out[N:])), "out: rows >= N written or rows < N not"
    ref = np.array([math.fsum(L[r, :r + 1] * z[:r + 1]) for r in range(N)])
    mag = np.array([np.abs(L[r, :r + 1] * z[:r + 1]).sum() for r in range(N)])
    lev = -(-(np.arange(N) + 1) // 32) + 5 + 1
    W = Worst(record_property)
    W("frac", frac(np.abs(out[:N] - ref), lev * U64 * mag * 1.01, "lower_matvec"))
    W.flush()


@gpu
@pytest.mark.parametrize("prec", ["f32", "f64"])
@pytest.mark.parametrize("N,Npad", [(1, 128), (127, 128), (128, 256), (300, 384)])
def test_loglik_set_rhs_batched(prec, N, Npad):
    """smk_loglik_set_rhs_batched_*: row N of each item holds y[s][:N] exactly and A[s][N][N] = 1e30 (in the element
    type); every other entry keeps its sentinel, with ldy = N + 5.  Argument codes: Npad <= N and Npad % 128 != 0 give
    -2, ldy < N gives -5."""
    _, check, fn, ptr = _api()
    dt = _tdt(prec)
    S, ldy = 3, N + 5
    rs = np.random.RandomState(N)
    y = _dev(rs.randn(S, ldy), dt)
    A = _dev(np.full((S, Npad, Npad), -7.0), dt)
    f = fn("smk_loglik_set_rhs_batched", dt)
    check(f(N, Npad, S, ptr(y), ldy, ptr(A), cur_stream()), "loglik_set_rhs_batched")
    exp = np.full((S, Npad, Npad), -7.0)
    exp[:, N, :N] = _h(y)[:, :N]
    exp[:, N, N] = float(np.float32(1e30)) if prec == "f32" else 1e30
    assert same(_h(A), exp), "entries other than row N [0, N] changed, or row N is not y"
    assert f(N, N, S, ptr(y), ldy, ptr(A), cur_stream()) == -2
    assert f(N, Npad + 1, S, ptr(y), ldy, ptr(A), cur_stream()) == -2
    assert f(N, Npad, S, ptr(y), N - 1, ptr(A), cur_stream()) == -5
