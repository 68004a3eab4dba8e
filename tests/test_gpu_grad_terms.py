"""The two kernels of csrc/grad.cu at the shapes the choosers run them at, each against a float64 evaluation of its own
device inputs (X, the query points, inv_ls and amp2 as the device holds them, promoted; ls = 1 / inv_ls), and their
callers against the float64 oracle.

smk_ei_grad_terms_* forms OUT[f][d] = sum_n A[f][n] T[n][d] with A = (alpha rows, gamma row) and T = (gk, kx).
  * Per-element probe: row f of A one-hot at n_f gives OUT[f] = T[n_f] exactly (fma(0, t, a) = a).  Compared with
    oracle.gp_oracle.grad_kernel / cov at that row, within a bound stated per element: the device's r2 is a sum of D
    squares, off by at most e = 2 (D + 8) u sum_d (|x_d il_d| + |xq_d il_d|)^2 (this also covers the oracle's expanded
    r2 in float64); k and dk/dr2 are evaluated on the host at r2 - e and r2 + e, and their largest move plus
    (8 + 2 |argument of exp|) u of rounding is the bound, with 4 u (|x il| + |xq il|) on each difference x il - xq il.
    At a row equal to the query point the device's difference is not exactly 0: x il - xq il contracts to a fused
    multiply-add against the rounded xq il, so r2 = O(u^2) and gk = O(u |w| il |x il|) there, which that term covers.
  * Contraction: random A (padding columns n >= N NaN), against the float64 product with the probed reference T:
        |OUT - A T|_fd <= sum_n |A_fn| ((N + 2) u (|T_nd| + b_nd) + b_nd),   b the per-element bound above,
    i.e. the fma chain over n (N roundings) on top of each element's own error.
  * Bitwise: NaN padding changes nothing; a batch item equals its sample alone; query q of a Q = 3 call equals q alone;
    the first rows (and the gamma row) of an F-fantasy call equal those of an F = 100 and an F = 1 call.
smk_mll_grad_terms_*:
  * Per-pair probe: alpha = 0, K^-1 = -e_{j0 i0} puts the integrand of pair (i0, j0) alone in out, within the same kind
    of per-element bound (here e = 2 (D + 8) u sum_d ((x_i - x_j) il)^2 + 8 u (|x_i il|^2 + |x_j il|^2)).
  * Full sum with the device's alpha and K^-1 (ldk > N, columns >= N NaN), against a float64 sum built in blocks of rows.
    Bound: each term's own error (J = alpha_i alpha_j - K^-1_ji to 2 u (|alpha_i alpha_j| + |K^-1_ji|), the kernel
    factor as above) plus (5 + W + N) u64 sum |term|: the double sum is a 5-level warp tree and then W double atomics
    (W = warps of the grid) in whatever order they land -- the bound holds for every order -- and N u64 for the host's
    own sum.
The measured worst fraction of each bound is printed (-s).
"""
import numpy as np
import pytest

from oracle import gp_oracle as O
from tests.helpers import data as _data, synth_hypers as _hypers

U = {"f32": 2.0 ** -24, "f64": 2.0 ** -53}
U64 = 2.0 ** -53
S3, S5 = np.sqrt(3.0), np.sqrt(5.0)
KIND = "Matern52"


def _npad(N):
    return (N + 127) // 128 * 128


# ---------------------------------------------------------------------------------------------------- host references
def _k(kind, r2):
    """correlation and the argument of its exp at r2 >= 0"""
    if kind in ("SE", "ARDSE"):
        return np.exp(-0.5 * r2), 0.5 * r2
    r = np.sqrt(r2)
    if kind == "Matern32":
        return (1.0 + S3 * r) * np.exp(-S3 * r), S3 * r
    return (1.0 + S5 * r + (5.0 / 3.0) * r2) * np.exp(-S5 * r), S5 * r


def _w(kind, r2):
    """dk/dr2"""
    if kind in ("SE", "ARDSE"):
        return -0.5 * np.exp(-0.5 * r2)
    r = np.sqrt(r2)
    if kind == "Matern32":
        return -1.5 * np.exp(-S3 * r)
    return -(5.0 / 6.0) * np.exp(-S5 * r) * (1.0 + S5 * r)


def _moves(kind, r2, e):
    """largest |k(r2') - k(r2)| and |w(r2') - w(r2)| for r2' = max(r2 - e, 0), r2 + e"""
    k0, w0 = _k(kind, r2)[0], _w(kind, r2)
    dk = dw = 0.0
    for r in (np.maximum(r2 - e, 0.0), r2 + e):
        dk = np.maximum(dk, np.abs(_k(kind, r)[0] - k0))
        dw = np.maximum(dw, np.abs(_w(kind, r) - w0))
    return dk, dw


def terms_ref(kind, X, xq, il, a2, u):
    """T [N][D+1] = (gk, kx) at one query point from the oracle, and its per-element bound b [N][D+1]."""
    ls = 1.0 / il
    T = np.empty((X.shape[0], X.shape[1] + 1))
    T[:, :-1] = np.squeeze(O.grad_kernel(kind, ls, X, xq[None, :]), axis=1)
    T[:, -1] = O.cov(kind, a2, ls, X, xq[None, :])[:, 0]
    a, b = X * il, xq * il
    r2 = ((a - b) ** 2).sum(axis=1)
    e = 2.0 * (X.shape[1] + 8) * u * ((np.abs(a) + np.abs(b)) ** 2).sum(axis=1)
    dk, dw = _moves(kind, r2, e)
    k, arg = _k(kind, r2)
    w = _w(kind, r2)
    rnd = (8.0 + 2.0 * arg) * u
    B = np.empty_like(T)
    diff = a - b
    B[:, :-1] = (dw[:, None] * np.abs(2.0 * il * diff) + np.abs(w[:, None] * 2.0 * il) * 4.0 * u * (np.abs(a) + np.abs(b))
                 + rnd[:, None] * np.abs(T[:, :-1]))
    B[:, -1] = a2 * (dk + rnd * k) + 2.0 * u * np.abs(T[:, -1])
    return T, B


def contraction_bound(A, T, B, u):
    N = A.shape[1]
    return np.abs(A).dot((N + 2) * u * (np.abs(T) + B) + B)


def mll_pair_ref(kind, X, il, i, j, u):
    """(corr_ij + 1e-6 delta_ij, delta_ij, gcorr_ij^d X[i][d]) from the oracle, and the bound of each."""
    ls = 1.0 / il
    x1, x2 = X[[i]], X[[j]]
    ref = np.empty(X.shape[1] + 2)
    ref[0] = O.kernel(kind, ls, x1, x2)[0, 0] + (1e-6 if i == j else 0.0)
    ref[1] = 1.0 if i == j else 0.0
    ref[2:] = O.grad_kernel(kind, ls, x1, x2)[0, 0] * X[i]
    _, bnd, _ = _mll_block(kind, x1, x2, il, np.ones((1, 1)), np.zeros((1, 1)), np.array([[i == j]]), u)
    bnd[1] = 0.0
    return ref, bnd


def _mll_block(kind, Xi, Xj, il, J, dJ, diag, u):
    """One block of pairs (rows Xi, columns Xj): the sums over the block of the terms of out[D+2], of their error
    bounds, and of their magnitudes.  J, dJ [bi][bj]: the block of J and its bound; diag [bi][bj]: i == j."""
    D = Xi.shape[1]
    r2, ab = np.zeros(J.shape), np.zeros(J.shape)
    for d in range(D):
        df = (Xi[:, d][:, None] - Xj[:, d][None, :]) * il[d]
        r2 += df * df
        ab += (Xi[:, d][:, None] * il[d]) ** 2 + (Xj[:, d][None, :] * il[d]) ** 2
    e = 2.0 * (D + 8) * u * r2 + 8.0 * U64 * ab
    dk, dw = _moves(kind, r2, e)
    k, arg = _k(kind, r2)
    w = _w(kind, r2)
    c = k + 1e-6 * diag
    out, bnd, mag = np.zeros(D + 2), np.zeros(D + 2), np.zeros(D + 2)
    t = J * c
    out[0], mag[0] = t.sum(), np.abs(t).sum()
    bnd[0] = (dJ * np.abs(c) + np.abs(J) * (dk + (8.0 + 2.0 * arg) * u * k + u * np.abs(c))).sum()
    out[1], mag[1], bnd[1] = np.where(diag, J, 0.0).sum(), np.where(diag, np.abs(J), 0.0).sum(), np.where(diag, dJ, 0.0).sum()
    for d in range(D):
        h = 2.0 * (Xi[:, d][:, None] - Xj[:, d][None, :]) * il[d] * il[d] * Xi[:, d][:, None]
        t = J * w * h
        out[2 + d], mag[2 + d] = t.sum(), np.abs(t).sum()
        bnd[2 + d] = (dJ * np.abs(w * h) + np.abs(J) * (dw * np.abs(h) + 8.0 * u * np.abs(w * h))).sum()
    return out, bnd, mag


def mll_sum_ref(kind, X, il, alpha, Kinv, u, block=256):
    """float64 out[D+2] and its bound for one sample, in blocks of rows i (never an N x N x D array).  Kinv is read as
    the kernel reads it: J_ij = alpha_i alpha_j - Kinv[j][i]."""
    N, D = X.shape
    out, bnd, mag = np.zeros(D + 2), np.zeros(D + 2), np.zeros(D + 2)
    for i0 in range(0, N, block):
        i1 = min(N, i0 + block)
        aa = alpha[i0:i1, None] * alpha[None, :]
        Kt = Kinv[:, i0:i1].T
        diag = np.arange(i0, i1)[:, None] == np.arange(N)[None, :]
        o, b, m = _mll_block(kind, X[i0:i1], X, il, aa - Kt, 2.0 * u * (np.abs(aa) + np.abs(Kt)), diag, u)
        out, bnd, mag = out + o, bnd + b, mag + m
    W = ((N + 15) // 16) ** 2 * 8
    return out, bnd + (5 + W + N) * U64 * mag


def fg_from_terms(out, amp2, mean, bests, pending):
    """RefineContext.per_sample on the host: (f_s, g_s) from out [S][F+1][D+1] (float64)."""
    import scipy.stats as sps
    F, D = out.shape[1] - 1, out.shape[2] - 1
    m = out[:, :F, D] + mean[:, None]
    v = amp2 * (1 + O.JITTER) - out[:, F, D]
    s = np.sqrt(v)[:, None]
    u = (bests - m) / s
    cdf, pdf = sps.norm.cdf(u), sps.norm.pdf(u)
    ei = s * (u * cdf + pdf)
    g = 0.5 * amp2[:, None, None] * (out[:, :F, :D] * -cdf[:, :, None] - 2.0 * out[:, F, :D][:, None, :] *
                                     (0.5 * pdf / s)[:, :, None])
    if not pending:
        return -ei.sum(axis=1), g[:, 0, :]
    return -ei.mean(axis=1), g.mean(axis=1)


def test_host_references_match_oracle():
    """No GPU: the blocked ML-II sum and the (gk, kx) terms above reproduce oracle.gp_oracle.mll_value_grad and
    grad_optimize_ei at small N."""
    import scipy.linalg as spla
    for kind in ("ARDSE", "Matern32", "Matern52", "SE"):
        X, y, rs = _data(40, 4, 3)
        pt = np.concatenate([[0.2, np.log(1e-2)], np.log(rs.uniform(0.4, 1.5, 4))])
        amp2, noise, ls = np.exp(pt[0]), np.exp(pt[1]), np.exp(pt[2:])
        il = 1.0 / (np.ones(4) if kind == "SE" else ls)
        mean = float(np.mean(y))
        K = O.cov(kind, amp2, ls, X) + (noise + 1e-8) * np.eye(40)    # jitter_chol's first jitter
        cf = spla.cho_factor(K, lower=True)
        alpha, Kinv = spla.cho_solve(cf, y - mean), spla.cho_solve(cf, np.eye(40))
        out, bnd = mll_sum_ref(kind, X, il, alpha, Kinv, U64, block=7)
        g = np.concatenate([[0.5 * out[0] * amp2, 0.5 * out[1] * noise], -amp2 * out[2:]])
        np.testing.assert_allclose(-g, O.mll_value_grad(kind, pt, X, y, mean)[1], rtol=1e-9, atol=1e-12)
        assert np.all(bnd > 0) and np.all(np.isfinite(bnd))
        if kind == "SE":
            continue
        h = (mean, noise, amp2, ls)
        K = O.cov(kind, amp2, ls, X) + noise * np.eye(40)
        cf = spla.cho_factor(K, lower=True)
        x = rs.rand(4)
        T, B = terms_ref(kind, X, x, 1.0 / ls, amp2, U64)
        A = np.stack([spla.cho_solve(cf, y - mean), spla.cho_solve(cf, T[:, -1])])
        f, gr = fg_from_terms(A.dot(T)[None], np.array([amp2]), np.array([mean]), np.array([[y.min()]]), False)
        f_ref, g_ref = O.grad_optimize_ei(kind, h, x, X, np.zeros((0, 4)), y)
        np.testing.assert_allclose(f[0], f_ref, rtol=1e-10)
        np.testing.assert_allclose(gr[0], g_ref, rtol=1e-9, atol=1e-13)
        assert np.all(B >= 0) and np.all(contraction_bound(A, T, B, U64) > 0)


# ---------------------------------------------------------------------------------------------------- device plumbing
_ENGS = {}


def _eng(prec):
    import torch
    from spearmint_b200.engine import GPEIEngine
    if prec not in _ENGS:
        _ENGS[prec] = GPEIEngine(dtype=torch.float32 if prec == "f32" else torch.float64)
    return _ENGS[prec]


def _h(t):
    return t.double().cpu().numpy()


def _grad_terms(eng, kind, N, Npad, D, S, Q, F, X, xq, inv_ls, amp2, alpha, gamma, raw=False):
    import torch
    from spearmint_b200.engine import KINDS, check, fn, ptr
    out = torch.full((S, Q, F + 1, D + 1), float("nan"), dtype=eng.dtype, device=eng.device)
    rc = fn("smk_ei_grad_terms", eng.dtype)(KINDS[kind], N, Npad, D, S, Q, F, ptr(X), ptr(xq), ptr(inv_ls), ptr(amp2),
                                            ptr(alpha), ptr(gamma), ptr(out), eng.stream())
    if raw:
        torch.cuda.synchronize()
        return rc
    check(rc, "ei_grad_terms")
    return out


def _targets(N, n_eq):
    t = {c for c0 in range(0, N, 64) for c in (c0, min(N, c0 + 64) - 1)} | {N - 1, n_eq}
    return sorted(t)


# (kind, N, D, F, S, Q)
EI_CASES = [("Matern52", 1, 1, 1, 1, 1), ("Matern32", 63, 3, 2, 3, 3), ("ARDSE", 64, 8, 100, 1, 1),
            ("Matern52", 65, 9, 1, 3, 3), ("Matern32", 1000, 31, 63, 1, 1), ("Matern52", 1000, 31, 64, 3, 1),
            ("ARDSE", 2051, 32, 100, 3, 3), ("Matern52", 2051, 33, 2, 40, 1), ("Matern32", 8192, 32, 100, 3, 1),
            ("Matern52", 8192, 3, 1, 40, 3), ("ARDSE", 512, 32, 1000, 1, 1), ("Matern52", 65, 1, 1000, 3, 1),
            ("Matern32", 1000, 8, 1000, 1, 3)]
_WORST = {}


def _note(key, frac):
    _WORST[key] = max(_WORST.get(key, 0.0), float(frac))
    print("worst fraction so far, %s: %.3g" % (key, _WORST[key]))


def _frac(err, bnd, tag):
    err, bnd = np.asarray(err, dtype=float), np.asarray(bnd, dtype=float)
    assert err.shape == bnd.shape and np.all(np.isfinite(err)), tag
    bad = err > bnd
    assert not np.any(bad), "%s: %d elements over the bound, worst %.3g" % (
        tag, int(bad.sum()), float((err / np.maximum(bnd, 1e-300)).max()))
    return float((err / np.maximum(bnd, 1e-300)).max()) if err.size else 0.0


@pytest.mark.gpu
@pytest.mark.parametrize("prec", ["f32", "f64"])
@pytest.mark.parametrize("kind,N,D,F,S,Q", EI_CASES)
def test_ei_grad_terms(prec, kind, N, D, F, S, Q):
    import torch
    eng, u = _eng(prec), U[prec]
    Npad = _npad(N)
    X, _, rs = _data(N, D, N + 7 * D + F)
    hb = eng.hypers(_hypers(rs, S, D, 1e-2), kind)
    xq = rs.rand(Q, D)
    n_eq = N // 2
    xq[0] = X[n_eq]                                            # r = 0 at row n_eq, bit for bit
    Xd, xqd = eng.to_dev(X), eng.to_dev(xq)
    Xh, xqh, ilh, a2h = _h(Xd), _h(xqd), _h(hb.inv_ls), _h(hb.amp2)
    refs = [[terms_ref(kind, Xh, xqh[q], ilh[s], a2h[s], u) for q in range(Q)] for s in range(S)]

    # per-element probe: one-hot rows of A
    tg = _targets(N, n_eq)
    Fp = max(F, len(tg))
    rows = [tg[f % len(tg)] for f in range(Fp + Q)]
    ap = torch.zeros((S, Fp, Npad), dtype=eng.dtype, device=eng.device)
    gp = torch.zeros((S, Q, Npad), dtype=eng.dtype, device=eng.device)
    ap[:, torch.arange(Fp), torch.tensor(rows[:Fp])] = 1.0
    gp[:, torch.arange(Q), torch.tensor(rows[Fp:])] = 1.0
    out = _h(_grad_terms(eng, kind, N, Npad, D, S, Q, Fp, Xd, xqd, hb.inv_ls, hb.amp2, ap, gp))
    frac = 0.0
    for s in range(S):
        for q in range(Q):
            T, B = refs[s][q]
            idx = rows[:Fp] + [rows[Fp + q]]
            frac = max(frac, _frac(np.abs(out[s, q] - T[idx]), B[idx], "probe %s s=%d q=%d" % (prec, s, q)))
    _note("ei probe " + prec, frac)

    # contraction with random A, padding NaN, and the bitwise invariants
    al = rs.randn(S, F, Npad) * 10.0
    ga = rs.randn(S, Q, Npad)
    al[:, :, N:] = np.nan
    ga[:, :, N:] = np.nan
    ald, gad = eng.to_dev(al), eng.to_dev(ga)
    out_d = _grad_terms(eng, kind, N, Npad, D, S, Q, F, Xd, xqd, hb.inv_ls, hb.amp2, ald, gad)
    z_al, z_ga = ald.clone(), gad.clone()
    z_al[:, :, N:] = 0.0
    z_ga[:, :, N:] = 0.0
    assert torch.equal(out_d, _grad_terms(eng, kind, N, Npad, D, S, Q, F, Xd, xqd, hb.inv_ls, hb.amp2, z_al, z_ga))
    out = _h(out_d)
    Ah, Gh = _h(ald)[:, :, :N], _h(gad)[:, :, :N]
    frac = 0.0
    for s in range(S):
        for q in range(Q):
            T, B = refs[s][q]
            A = np.concatenate([Ah[s], Gh[s, q][None]])
            frac = max(frac, _frac(np.abs(out[s, q] - A.dot(T)), contraction_bound(A, T, B, u),
                                   "contraction %s s=%d q=%d" % (prec, s, q)))
    _note("ei contraction " + prec, frac)
    if S > 1:
        s = S - 1
        one = _grad_terms(eng, kind, N, Npad, D, 1, Q, F, Xd, xqd, hb.inv_ls[s:], hb.amp2[s:], ald[s:], gad[s:])
        assert torch.equal(one, out_d[s:]), "batch item"
    if Q > 1:
        q = Q - 1
        one = _grad_terms(eng, kind, N, Npad, D, S, 1, F, Xd, xqd[q:], hb.inv_ls, hb.amp2, ald,
                          gad[:, q:].contiguous())
        assert torch.equal(one, out_d[:, q:]), "query alone"
    for Fs in (1, 100):
        if Fs < F:
            part = _grad_terms(eng, kind, N, Npad, D, S, Q, Fs, Xd, xqd, hb.inv_ls, hb.amp2,
                               ald[:, :Fs].contiguous(), gad)
            assert torch.equal(part[:, :, :Fs], out_d[:, :, :Fs]), "rows f < %d" % Fs
            assert torch.equal(part[:, :, Fs], out_d[:, :, F]), "gamma row against F = %d" % Fs


@pytest.mark.gpu
@pytest.mark.parametrize("prec", ["f32", "f64"])
def test_ei_grad_terms_arguments(prec):
    """Every argument check returns its documented code; SE is rejected (-1) as the header states; no F returns an
    error, up to the largest D the staging takes (324 in float64, 712 in float32), one more being -4."""
    import torch
    from spearmint_b200.engine import KINDS
    eng = _eng(prec)
    dev, dt = eng.device, eng.dtype
    Dmax = 712 if prec == "f32" else 324
    N, Npad, S, Q = 100, 128, 2, 1

    def args(D, F):
        return (N, Npad, D, S, Q, F, torch.rand(N, D, dtype=dt, device=dev), torch.rand(Q, D, dtype=dt, device=dev),
                torch.ones(S, D, dtype=dt, device=dev), torch.ones(S, dtype=dt, device=dev),
                torch.randn(S, F, Npad, dtype=dt, device=dev), torch.randn(S, Q, Npad, dtype=dt, device=dev))
    for D, F in ((32, 400), (32, 5000), (1, 400), (1, 5000), (Dmax, 1), (Dmax, 63), (Dmax, 1000)):
        assert _grad_terms(eng, KIND, *args(D, F), raw=True) == 0, (D, F)
    assert _grad_terms(eng, KIND, *args(Dmax + 1, 63), raw=True) == -4
    a = list(args(32, 400))
    bad = [(0, 0, -2), (1, 99, -2), (2, 0, -4), (3, 0, -5), (4, 0, -6), (5, 0, -7)] + [(p, None, -8) for p in range(6, 12)]
    for pos, val, code in bad:
        b = list(a)
        b[pos] = val
        assert _grad_terms(eng, KIND, *b, raw=True) == code, (pos, val)
    from spearmint_b200.engine import fn, ptr
    f = fn("smk_ei_grad_terms", dt)
    ps = [ptr(t) for t in a[6:]]
    out = torch.empty(S, Q, 401, 33, dtype=dt, device=dev)
    for kind in (-1, 4, KINDS["SE"]):
        assert f(kind, *a[:6], *ps, ptr(out), eng.stream()) == -1
    assert f(KINDS[KIND], *a[:6], *ps, None, eng.stream()) == -8
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------------- ML-II kernel
MLL_CASES = [("f64", "Matern52", 1, 1, 1), ("f64", "SE", 17, 5, 3), ("f64", "ARDSE", 17, 9, 1),
             ("f64", "Matern32", 1000, 8, 3), ("f64", "Matern52", 1000, 17, 1), ("f64", "SE", 1000, 32, 1),
             ("f64", "ARDSE", 4096, 9, 1), ("f64", "Matern52", 4096, 32, 3),
             ("f32", "Matern32", 1, 5, 1), ("f32", "ARDSE", 17, 8, 3), ("f32", "Matern52", 1000, 9, 1),
             ("f32", "SE", 1000, 17, 3), ("f32", "Matern32", 4096, 32, 1), ("f32", "Matern52", 4096, 1, 1)]


def _mll(eng, kind, N, D, S, X, inv_ls, alpha, lda, Kinv, ldk):
    import torch
    from spearmint_b200.engine import KINDS, check, fn, ptr
    out = torch.full((S, D + 2), float("nan"), dtype=torch.float64, device=eng.device)
    check(fn("smk_mll_grad_terms", eng.dtype)(KINDS[kind], N, D, S, ptr(X), ptr(inv_ls), ptr(alpha), lda, ptr(Kinv),
                                              ldk, ptr(out), eng.stream()), "mll_grad_terms")
    return out.cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("prec,kind,N,D,S", MLL_CASES)
def test_mll_grad_terms(prec, kind, N, D, S):
    import torch
    eng, u = _eng(prec), U[prec]
    X, y, rs = _data(N, D, 31 * N + D)
    hs = _hypers(rs, S, D, 1e-2)
    hb = eng.hypers(hs, kind)
    Xd = eng.to_dev(X)
    Xh, ilh = _h(Xd), _h(hb.inv_ls)
    lda, ldk = N + 5, N + 3

    # per-pair probe, one pair per batch item
    l0 = (N - 1) // 16 * 16
    pairs = sorted({(0, 0), (N - 1, N - 1), (N - 1, l0), (l0, N - 1), (N // 2, N // 3), (min(1, N - 1), 0)})
    P = len(pairs)
    il_p = hb.inv_ls[[p % S for p in range(P)]].contiguous()
    alpha = torch.zeros((P, lda), dtype=eng.dtype, device=eng.device)
    Kinv = torch.zeros((P, N, ldk), dtype=eng.dtype, device=eng.device)
    for p, (i, j) in enumerate(pairs):
        Kinv[p, j, i] = -1.0
    out = _mll(eng, kind, N, D, P, Xd, il_p, alpha, lda, Kinv, ldk)
    del Kinv
    frac = 0.0
    for p, (i, j) in enumerate(pairs):
        ref, bnd = mll_pair_ref(kind, Xh, ilh[p % S], i, j, u)
        frac = max(frac, _frac(np.abs(out[p] - ref), bnd, "pair %s (%d, %d)" % (prec, i, j)))
    _note("mll pair " + prec, frac)

    # full sum with the device's own alpha and K^-1 (as GP.value_grad forms them), ldk > N, columns >= N NaN
    fac = eng.factor(kind, Xd, hb)
    fac.check_pd()
    a_t, _, _ = fac.solve(eng.to_dev(y), F=1)
    eye = torch.eye(N, dtype=eng.dtype, device=eng.device)
    k_t, _, _ = fac.solve(eye, F=N, y_stride=0, ldy=N, subtract_mean=False)
    alpha = torch.full((S, lda), float("nan"), dtype=eng.dtype, device=eng.device)
    alpha[:, :N] = a_t[:, 0, :N]
    Kinv = torch.full((S, N, ldk), float("nan"), dtype=eng.dtype, device=eng.device)
    Kinv[:, :, :N] = k_t[:, :, :N]
    del k_t
    out = _mll(eng, kind, N, D, S, Xd, hb.inv_ls, alpha, lda, Kinv, ldk)
    ah, frac = _h(alpha), 0.0
    for s in range(S):
        Kh = Kinv[s, :, :N].double().cpu().numpy()
        ref, bnd = mll_sum_ref(kind, Xh, ilh[s], ah[s, :N], Kh, u)
        frac = max(frac, _frac(np.abs(out[s] - ref), bnd, "sum %s s=%d" % (prec, s)))
    _note("mll sum " + prec, frac)


# ---------------------------------------------------------------------------------------------------- callers
def _assert_fg(f, g, f_ref, g_ref):
    """The refinement's tolerances (test_refine_value_grad_matches_reference)."""
    np.testing.assert_allclose(f, f_ref, rtol=1e-6)
    np.testing.assert_allclose(np.ravel(g), np.ravel(g_ref), rtol=1e-6, atol=1e-10 * max(1.0, np.abs(g_ref).max()))


def _points(X, y, rs):
    """a point of the jitter cloud around the incumbent, and a random one"""
    x0 = np.clip(X[np.argmin(y)] + 1e-3 * rs.randn(X.shape[1]), 0.0, 1.0)
    return [x0, rs.rand(X.shape[1])]


@pytest.mark.gpu
@pytest.mark.parametrize("N,S,F", [(2048, 10, 100), (4096, 3, 100), (512, 3, 1000)])
def test_refine_plain(N, S, F):
    """RefineContext.value_grad, D = 32, P = 3, against grad_optimize_ei_over_hypers; F = 1000 fantasies at N = 512."""
    X, y, rs = _data(N, 32, N + F)
    hs = _hypers(rs, S, 32, 1e-2)
    pend = rs.rand(3, 32)
    normals = rs.randn(3, F)
    ctx = _eng("f64").refine_context(KIND, hs, X, pend, y, normals)
    for x in _points(X, y, rs):
        f, g = ctx.value_grad(x)
        _assert_fg(f, g, *O.grad_optimize_ei_over_hypers(KIND, hs, x, X, pend, y, normals))


@pytest.mark.gpu
def test_refine_per_second():
    """The per-second refinement at the c4 shape: D = 8, N = 1024, S = 10."""
    N, D, S = 1024, 8, 10
    X, y, rs = _data(N, D, 4)
    hs = _hypers(rs, S, D, 1e-2)
    durs = np.log(1.0 + X[:, 0] + 0.1 * rs.rand(N))
    ths = [(float(np.mean(durs)), 1e-3, 1.0, rs.uniform(0.3, 2.0, D)) for _ in range(S)]
    ctx = _eng("f64").refine_context(KIND, hs, X, np.zeros((0, D)), y, None, ths, durs)
    for x in _points(X, y, rs):
        f, g = ctx.value_grad(x)
        _assert_fg(f, g, *O.grad_optimize_ei_per_s_over_hypers(KIND, hs, ths, x, X, y, durs))


@pytest.mark.gpu
def test_refine_constrained():
    """ConstrainedRefineContext, D = 32, N = 2048, P = 2, F = 100, against the constrained oracle."""
    from tests import constrained_oracle as CO
    N, D, S = 2048, 32, 2
    rs = np.random.RandomState(6)
    comp = rs.rand(N, D)
    yv = np.sin(3 * comp).sum(1)
    vals = (yv - yv.mean()) / yv.std()
    vals[comp[:, 0] + comp[:, 1] > 1.2] = np.inf
    labels = CO.labels_of(vals)
    hs = [(0.05 * rs.randn(), 1e-2, float(np.exp(0.2 * rs.randn())), rs.uniform(0.4, 2.0, D)) for _ in range(S)]
    chs = [(0.0, rs.uniform(0.5, 3.0), rs.uniform(0.5, 2.0), rs.uniform(0.3, 1.5, D)) for _ in range(S)]
    ff = np.where(labels > 0, 1.0, -1.0) + 0.3 * rs.randn(N)
    pend = rs.rand(2, D)
    normals = rs.randn(2, 100)
    ctx = _eng("f64").constrained_refine_context(KIND, hs, chs, ff, comp, labels, pend, vals, normals)
    for x in _points(comp, np.where(labels > 0, vals, 1e9), rs):
        f, g = ctx.value_grad(x)
        _assert_fg(f, g, *CO.grad_optimize_ei_over_hypers(KIND, hs, chs, ff, x, comp, labels, pend, vals, normals))


@pytest.mark.gpu
def test_next_with_500_fantasies(tmp_path):
    """GPEIOptChooserB200.next() with pending_samples=500 and two pending jobs runs through its refinement."""
    from spearmint_b200.chooser import GPEIOptChooserB200 as mod
    N, M, D = 512, 300, 32
    rs = np.random.RandomState(12)
    grid = rs.rand(N + M + 2, D)
    yv = np.sin(3 * grid[:N]).sum(1)
    values = np.zeros(grid.shape[0])
    values[:N] = (yv - yv.mean()) / yv.std()
    ch = mod.init(str(tmp_path), "mcmc_iters=2,burnin=0,pending_samples=500,use_multiprocessing=0")
    np.random.seed(3)
    ret = ch.next(grid, values, np.ones(grid.shape[0]), np.arange(N, N + M), np.arange(N + M, N + M + 2), np.arange(N))
    if isinstance(ret, tuple):
        assert ret[0] == M and np.all(np.isfinite(ret[1])) and np.all((ret[1] >= 0) & (ret[1] <= 1))
    else:
        assert N <= int(ret) < N + M


@pytest.mark.gpu
def test_mlii_value_grad_d32():
    """GP.value_grad at D = 32, N = 1024 against mll_value_grad, to 1e-7."""
    import torch
    from spearmint_b200.gp import GP
    N, D = 1024, 32
    X, y, rs = _data(N, D, 8)
    eng = _eng("f64")
    gp = GP(KIND, engine=eng)
    gp.real_init(D, y)
    pt = np.concatenate([[0.1, np.log(1e-2)], np.log(rs.uniform(0.5, 2.0, D))])
    eye = torch.eye(N, dtype=eng.dtype, device=eng.device)
    f, g = gp.value_grad(pt, eng.to_dev(X), eng.to_dev(y), eye, float(np.mean(y)))
    f_ref, g_ref = O.mll_value_grad(KIND, pt, X, y, float(np.mean(y)))
    np.testing.assert_allclose(f, f_ref, rtol=1e-7)
    np.testing.assert_allclose(g, g_ref, rtol=1e-7, atol=1e-8 * max(1.0, np.abs(g_ref).max()))


def _gamma(ctx, x):
    """gamma = K^-1 kx of RefineContext._terms, as the device forms it: [S][N]."""
    import torch
    from spearmint_b200.engine import KINDS, check, fn, ptr
    eng, fac = ctx.eng, ctx.prep.fac
    S, N, D = fac.hb.S, fac.N, fac.D
    xq = eng.to_dev(np.reshape(x, (1, D)))
    kx = torch.empty((S, 1, N), dtype=eng.dtype, device=eng.device)
    check(fn("smk_cov_build", eng.dtype)(KINDS[ctx.kind], 1, N, D, S, ptr(xq), ptr(fac.X), ptr(fac.hb.inv_ls),
                                         ptr(fac.hb.amp2), None, ptr(kx), N, eng.stream()), "cov_build")
    gamma, _, _ = fac.solve(kx, F=1, y_stride=N, ldy=N, subtract_mean=False)
    return _h(gamma)[:, 0, :N]


@pytest.mark.gpu
def test_refine_float32():
    """DeviceBackend(refine_dtype="float32") against the float64 refinement at N = 2048, D = 32, P = 3, F = 100.

    Bound, derived from the float32 solve on the device's own factor: with dA = A32 - A64 the difference of the
    (alpha, gamma) rows of the two builds, the float32 terms must lie within
        sum_n |dA_fn| |T_nd| + the contraction bound of the float32 kernel
    of A64 T (T the float64 terms at the float32 inputs).  Propagated to first order through func_m = OUT[f][D] + mean,
    func_v = amp2 (1 + 1e-6) - OUT[F][D] and EI, that gives the bound on f; it is asserted with a factor 2 and the
    measured (f, g) errors are printed."""
    import scipy.stats as sps
    from spearmint_b200.backend import DeviceBackend
    N, D, F, S = 2048, 32, 100, 3
    X, y, rs = _data(N, D, 21)
    hs = _hypers(rs, S, D, 1e-2)
    pend = rs.rand(3, D)
    normals = rs.randn(3, F)
    c64 = _eng("f64").refine_context(KIND, hs, X, pend, y, normals)
    c32 = DeviceBackend(refine_dtype="float32").refine_context(KIND, hs, X, pend, y, normals)
    assert c32.eng.dtype != c64.eng.dtype
    u = U["f32"]
    Nt = N + 3
    fe, ge = 0.0, 0.0
    for x in _points(X, y, rs):
        f32, g32 = c32.value_grad(x)
        f64, g64 = c64.value_grad(x)
        o32 = c32._terms(c32.prep.fac, c32.prep.alpha, F, x)
        a32, a64 = _h(c32.prep.alpha)[:, :, :Nt], _h(c64.prep.alpha)[:, :, :Nt]
        g_32, g_64 = _gamma(c32, x), _gamma(c64, x)
        Xh, ilh, a2h = _h(c32.prep.fac.X), _h(c32.hb.inv_ls), _h(c32.hb.amp2)
        df, fb = 0.0, 0.0
        for s in range(S):
            T, B = terms_ref(KIND, Xh, _h(c32.eng.to_dev(x)), ilh[s], a2h[s], u)
            A64 = np.concatenate([a64[s], g_64[s][None]])
            dA = np.concatenate([a32[s], g_32[s][None]]) - A64
            bo = np.abs(dA).dot(np.abs(T)) + contraction_bound(A64, T, B, u)
            _frac(np.abs(o32[s] - A64.dot(T)), bo, "float32 terms s=%d" % s)
            # first-order propagation to f (mean over the fantasies of EI's sensitivity to m and v)
            o = c64._terms(c64.prep.fac, c64.prep.alpha, F, x)[s]
            m = o[:F, D] + c64.hb.host_mean[s]
            v = c64.hb.host_amp2[s] * (1 + O.JITTER) - o[F, D]
            sd = np.sqrt(v)
            uu = (c64.prep.bests_host[s] - m) / sd
            fb += np.mean(sps.norm.cdf(uu) * bo[:F, D] + 0.5 * sps.norm.pdf(uu) / sd * bo[F, D])
        assert abs(f32 - f64) <= 2.0 * fb, (f32, f64, fb)
        fe = max(fe, abs(f32 - f64) / abs(f64))
        ge = max(ge, float(np.abs(g32 - g64).max() / np.abs(g64).max()))
        print("float32 refinement: |df| = %.3g (bound %.3g), |df|/|f| = %.3g, max|dg|/max|g| = %.3g"
              % (abs(f32 - f64), 2.0 * fb, abs(f32 - f64) / abs(f64), ge))
