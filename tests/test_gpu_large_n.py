"""-m gpu: the triangular solve above the shared-memory limit (smk_chol_solve_gm_*, csrc/solve.cu) and every caller of
Factor.solve at a size that needs it.

smk_chol_solve_* keeps one group of right-hand sides per CTA in shared memory up to Npad = 14 080 and calls
smk_chol_solve_gm_* above (float64 at Npad = 14 208 included: its right-hand sides would fill exactly 227 KB, with no
room for the kernel's static shared memory).  The kernel cases run smk_chol_solve_gm_* directly at N = 1 ... 20 000 on
the device's own factor of a GP covariance (built and factored as Factor does), F = 1, 3, 100 and once F = N.

Accuracy of alpha, per checked column b: the componentwise backward error of the two substitutions,
    max_i |b - L L^T alpha|_i / (u (|L| |L^T| |alpha|)_i),
evaluated in float64 on the device's L, against the same measure of scipy's solve_triangular (element type) on the same
L.  Bound, stated before running: max(32 x scipy's, 4 (N + NB c)), c = max_b || |W_b| |L_bb| ||_inf the Skeel condition
of the diagonal blocks, because the solve applies the stored block inverses W_b instead of substituting inside a block.
quad must agree with scipy's |L^-1 b|^2 within max(32 x scipy's own inconsistency |t|^2 - b.alpha, 4 N u) relative;
sum_log_diag with the float64 sum within 4 N u sum |log L_ii|.  Padding rows of alpha must be zero.

Bitwise invariants: the public entry above the limit equals smk_chol_solve_gm_*; a batch item equals the same sample
solved alone; rows >= N of a joint factor (L and winv) filled with NaN change nothing under n_lead (at n_lead = 2040 for
the shared-memory kernel as well; test_gpu_solve.py covers the sizes below the limit); one float32 batch
whose last item starts more than 2^31 elements in.

Callers at N = 14 209 (above both limits) against the float64 oracle: the float64 grid pass with 3 pending points
and per second (1e-6 of max EI, equal argmax), plain and constrained refinement
(f, g) (1e-6), the constrained grid pass, ML-II (f, g) (1e-7); and next() of each chooser.
"""
import functools

import numpy as np
import pytest

from tests.helpers import (SOLVE_NB as NBS, check_solve as _check_solve, cur_stream as _stream, data as _data,
                           gp_factor as _gp_factor)

pytestmark = pytest.mark.gpu

NLIM = {"f32": 14080, "f64": 14080}      # the largest Npad the shared-memory kernel takes
KIND = "Matern52"
NX = 14209                               # Npad = 14336


@pytest.fixture(scope="module")
def engs():
    import torch
    from spearmint_b200.engine import GPEIEngine
    return {"f32": GPEIEngine(dtype=torch.float32), "f64": GPEIEngine(dtype=torch.float64)}


# ---------------------------------------------------------------------------------------------------- device plumbing
@functools.lru_cache(maxsize=1)
def _factored(prec, N, S, seed, Ntot=None):
    """helpers.gp_factor (Matern52, D = 4, noise 1e-2) on the module's engine of prec: (eng, A, winv, hb, y)."""
    eng = _engs[prec]
    return (eng,) + _gp_factor(eng, N, S, seed, Ntot, KIND)


_engs = {}


@pytest.fixture(scope="module", autouse=True)
def _bind(engs):
    _engs.update(engs)
    yield
    _factored.cache_clear()


def _solve(entry, eng, N, Npad, S, F, L, winv, y, y_stride, ldy, mean, scalars=True):
    import torch
    from spearmint_b200.engine import check, fn, ptr
    nan = float("nan")
    alpha = torch.full((S, F, Npad), nan, dtype=eng.dtype, device=eng.device)
    sld = torch.full((S,), nan, dtype=eng.dtype, device=eng.device) if scalars else None
    quad = torch.full((S, F), nan, dtype=eng.dtype, device=eng.device) if scalars else None
    check(fn(entry, eng.dtype)(N, Npad, S, F, ptr(L), ptr(winv), ptr(y), y_stride, ldy, ptr(mean), ptr(alpha),
                               ptr(sld), ptr(quad), _stream()), entry)
    return alpha, sld, quad


def _same(a, b):
    import torch
    return all((x is None and y is None) or torch.equal(x, y) for x, y in zip(a, b))


def _cols(F):
    return list(range(F)) if F <= 6 else sorted({0, 1, F // 3, F // 2, F - 2, F - 1})


# ---------------------------------------------------------------------------------------------------- kernel cases
SMALL = [1, 127, 129, 2047, 4097]
KCASES = [(p, N, F, S) for p in ("f32", "f64") for N in SMALL for F, S in ((1, 1), (3, 3), (100, 1))]
KCASES += [(p, N, F, S) for p in ("f32", "f64")
           for N, F, S in ((14081, 1, 1), (14081, 3, 3), (14209, 1, 1), (14209, 3, 3), (16384, 100, 1), (20000, 1, 1))]


@pytest.mark.parametrize("prec,N,F,S", KCASES)
def test_solve_gm(prec, N, F, S):
    """smk_chol_solve_gm_* against scipy on the device's own L; per-sample y with ldy = N + 5 for F = 3 (mean NULL),
    one y shared by every sample otherwise (mean subtracted).  S = 3: item 1 equals the sample solved alone.  Npad above
    the limit: smk_chol_solve_* equals smk_chol_solve_gm_* bit for bit."""
    import torch
    eng, A, winv, hb, y = _factored(prec, N, S, N % 97)
    Npad = A.shape[-1]
    rs = np.random.RandomState(N + F)
    if F == 3:
        ldy = N + 5
        yh = rs.randn(S, F, ldy)
        y_stride, mean = F * ldy, None
    else:
        ldy, y_stride = N, 0
        yh = np.tile(y, (F, 1)) + (0.1 * rs.randn(F, N) if F > 1 else 0.0)
        mean = hb.mean
    yd = eng.to_dev(np.ascontiguousarray(yh))
    out = _solve("smk_chol_solve_gm", eng, N, Npad, S, F, A, winv, yd, y_stride, ldy, mean)
    if Npad > NLIM[prec]:
        assert _same(out, _solve("smk_chol_solve", eng, N, Npad, S, F, A, winv, yd, y_stride, ldy, mean))
    if S == 3:
        s = 1
        one = _solve("smk_chol_solve_gm", eng, N, Npad, 1, F, A[s:s + 1], winv[s:s + 1],
                     yd.view(-1)[s * y_stride:], y_stride, ldy, None if mean is None else mean[s:s + 1])
        assert _same(one, tuple(t[s:s + 1] for t in out))
    alpha, sld, quad = (t.cpu().numpy() for t in out)
    assert not np.any(alpha[:, :, N:]), "padding of alpha"
    ydt = yd.cpu().numpy().reshape(-1)
    mh = None if mean is None else mean.cpu().numpy()
    cols = _cols(F)
    for s in range(S):
        Lh = np.tril(A[s, :N, :N].cpu().numpy())
        W = winv[s].cpu().numpy()
        b = np.stack([ydt[s * y_stride + f * ldy:s * y_stride + f * ldy + N] for f in cols], axis=1)
        if mh is not None:
            b = b - mh[s]                       # element type: the device forms y - mean the same way
        _check_solve(prec, Lh, W, b, alpha[s][cols][:, :N].T, quad[s][cols], sld[s], "%s N=%d F=%d s=%d" % (prec, N, F, s))
        del Lh


def test_solve_gm_identity_rhs_at_size():
    """F = N right-hand sides (ML-II's K^-1), float64, N = 14 209: columns spread over the range against scipy."""
    import torch
    prec, N = "f64", NX
    eng, A, winv, hb, y = _factored(prec, N, 1, 3)
    Npad = A.shape[-1]
    eye = torch.eye(N, dtype=eng.dtype, device=eng.device)
    alpha, sld, quad = _solve("smk_chol_solve", eng, N, Npad, 1, N, A, winv, eye, 0, N, None, scalars=False)
    cols = [0, 1, 63, 64, 4097, N // 2, N - 65, N - 1]
    a = alpha[0][cols].cpu().numpy()
    assert not np.any(a[:, N:])
    Lh = np.tril(A[0, :N, :N].cpu().numpy())
    b = np.zeros((N, len(cols)))
    b[cols, range(len(cols))] = 1.0
    _check_solve(prec, Lh, winv[0].cpu().numpy(), b, a[:, :N].T, None, None, "f64 F=N")


@pytest.mark.parametrize("prec", ["f32", "f64"])
@pytest.mark.parametrize("n_lead,P,entry", [pytest.param(2040, 10, "smk_chol_solve_gm", id="2040-10"),
                                            pytest.param(2040, 10, "smk_chol_solve", id="2040-10-smem"),
                                            pytest.param(NX, 3, "smk_chol_solve", id="14209-3")])
def test_joint_factor_leading_block_and_fantasy_layout(prec, n_lead, P, entry):
    """A joint factor of n_lead + P points, solved by `entry` (at n_lead = 2040 both the global-memory entry and the
    public one, which runs the shared-memory kernel there; above the limit the public one runs the global-memory
    kernel).  (1) The fantasy layout: all N + P rows, F = 3, y_stride = F (N + P), ldy = N + P, mean NULL.  (2) n_lead:
    the leading block with the mean subtracted; then rows >= n_lead of L and of winv are set to NaN and the result must
    not change by a bit."""
    import torch
    Nt = n_lead + P
    eng, A, winv, hb, y = _factored(prec, n_lead, 2, 11, Nt)
    A, winv = A.clone(), winv.clone()
    S, Npad, nb, F = 2, A.shape[-1], NBS[prec], 3
    rs = np.random.RandomState(5)
    fant = rs.randn(S, F, Nt)
    fd = eng.to_dev(fant)
    out = _solve(entry, eng, Nt, Npad, S, F, A, winv, fd, F * Nt, Nt, None)
    yd = eng.to_dev(y[:n_lead])
    lead = _solve(entry, eng, n_lead, Npad, S, 1, A, winv, yd, 0, n_lead, hb.mean)
    # rows >= n_lead of the joint factor and of its block inverses: NaN
    A[:, n_lead:, :] = float("nan")
    b0, r0 = divmod(n_lead, nb)
    winv[:, b0, r0:, :] = float("nan")
    winv[:, b0 + 1:] = float("nan")
    assert _same(lead, _solve(entry, eng, n_lead, Npad, S, 1, A, winv, yd, 0, n_lead, hb.mean))
    alpha, sld, quad = (t.cpu().numpy() for t in out)
    la, lsld, lquad = (t.cpu().numpy() for t in lead)
    assert not np.any(alpha[:, :, Nt:]) and not np.any(la[:, :, n_lead:])
    mh = hb.mean.cpu().numpy()
    ydt = yd.cpu().numpy()
    fdt = fd.cpu().numpy()
    for s in range(S):
        _, A0, W0, _, _ = _factored(prec, n_lead, 2, 11, Nt)
        Lh = np.tril(A0[s, :Nt, :Nt].cpu().numpy())
        W = W0[s].cpu().numpy()
        _check_solve(prec, Lh, W, fdt[s].T, alpha[s][:, :Nt].T, quad[s], sld[s], "%s joint %d s=%d" % (prec, Nt, s))
        Ll = np.ascontiguousarray(Lh[:n_lead, :n_lead])
        del Lh
        _check_solve(prec, Ll, W, (ydt - mh[s])[:, None], la[s][:, :n_lead].T, lquad[s], lsld[s],
                     "%s lead %d s=%d" % (prec, n_lead, s))


def test_batch_offsets_beyond_2_31():
    """float32, S = 8 at N = 17 500: the last item starts 7 Npad^2 = 2.15e9 elements into the batch, past 2^31.  It
    equals itself solved alone and meets the accuracy bound."""
    prec, N, S = "f32", 17500, 8
    eng, A, winv, hb, y = _factored(prec, N, S, 8)
    assert (S - 1) * A.shape[-1] ** 2 > 2 ** 31
    yd = eng.to_dev(y)
    Npad = A.shape[-1]
    out = _solve("smk_chol_solve", eng, N, Npad, S, 1, A, winv, yd, 0, N, hb.mean)
    s = S - 1
    one = _solve("smk_chol_solve_gm", eng, N, Npad, 1, 1, A[s:], winv[s:], yd, 0, N, hb.mean[s:])
    assert _same(one, tuple(t[s:] for t in out))
    alpha, sld, quad = (t.cpu().numpy() for t in out)
    Lh = np.tril(A[s, :N, :N].cpu().numpy())
    b = (yd.cpu().numpy() - hb.mean.cpu().numpy()[s])[:, None]
    _check_solve(prec, Lh, winv[s].cpu().numpy(), b, alpha[s][:, :N].T, quad[s], sld[s], "f32 S=8 item 7")


# ---------------------------------------------------------------------------------------------------- callers
TOL = 5e-3


def _problem(N, M, S, D, seed=0):
    """D = 32 where a float32 grid pass runs: at N = 14 209 in a few dimensions the float32 factorisation of the
    grid pass itself loses positive definiteness, whatever the solve does."""
    X, y, rs = _data(N, D, seed)
    cand = rs.rand(M, D)
    k = min(10, M)
    cand[:k] = X[np.argmin(y)] + 1e-3 * rs.randn(k, D)
    hs = [(0.1 * rs.randn(), 1e-2, float(np.exp(0.25 * rs.randn())), rs.uniform(0.3, 2.0, D)) for _ in range(S)]
    return X, y, cand, hs, rs


def _assert_parity(ei, ref, tol=TOL):
    assert ei.shape == ref.shape and np.all(np.isfinite(ei))
    for s in range(ref.shape[1]):
        scale = ref[:, s].max()
        assert scale > 1e-8
        assert np.abs(ei[:, s] - ref[:, s]).max() <= tol * scale, s
    assert int(np.argmax(ei.mean(axis=1))) == int(np.argmax(ref.mean(axis=1)))


def test_grid_pass_with_pending_and_per_second(engs):
    """The float64 build, within 1e-6 of max EI: with pending points (the observed-block solve under n_lead and the
    fantasy solve of the joint factor) and per second (the time GP's solve), all above the limit.  The float32 grid pass
    runs the same solves; at this size its own precision (explicit inverse, float32 factor) is what limits it."""
    from oracle import gp_oracle as O
    X, y, cand, hs, rs = _problem(NX - 3, 256, 1, 32)
    pend = rs.rand(3, X.shape[1])
    normals = rs.randn(3, 4)
    ref = O.ei_over_hypers(KIND, hs, X, pend, cand, y, normals)
    _assert_parity(engs["f64"].ei_over_hypers(KIND, hs, X, pend, cand, y, normals), ref, 1e-6)
    X, y, cand, hs, rs = _problem(NX, 256, 1, 32, seed=1)
    durs = np.log(1.0 + X[:, 0])
    ths = [(float(np.mean(durs)), 1e-3, 1.0, rs.uniform(0.3, 2.0, X.shape[1]))]
    nopend = np.zeros((0, X.shape[1]))
    ref = np.stack([O.compute_ei_per_s(KIND, hs[0], ths[0], X, nopend, cand, y, durs)], axis=1)
    _assert_parity(engs["f64"].ei_over_hypers(KIND, hs, X, nopend, cand, y, None, ths, durs), ref, 1e-6)


def test_refinement_value_grad(engs):
    from oracle import gp_oracle as O
    X, y, cand, hs, rs = _problem(NX - 3, 2, 1, 3, seed=2)
    pend = rs.rand(3, X.shape[1])
    normals = rs.randn(3, 2)
    ctx = engs["f64"].refine_context(KIND, hs, X, pend, y, normals)
    for x in cand[:2]:
        f, g = ctx.value_grad(x)
        f_ref, g_ref = O.grad_optimize_ei_over_hypers(KIND, hs, x, X, pend, y, normals)
        np.testing.assert_allclose(f, f_ref, rtol=1e-6)
        np.testing.assert_allclose(g, np.ravel(g_ref), rtol=1e-6, atol=1e-10 * max(1.0, np.abs(g_ref).max()))


def _constrained_problem(N, M, S, D=32, seed=4):
    rs = np.random.RandomState(seed)
    comp, cand = rs.rand(N, D), rs.rand(M, D)
    yv = np.sin(3 * comp).sum(1)
    vals = (yv - yv.mean()) / yv.std()
    bad = comp[:, 0] + comp[:, 1] > 1.2
    vals[bad] = np.inf
    from tests import constrained_oracle as CO
    labels = CO.labels_of(vals)
    hs = [(0.05 * rs.randn(), 1e-2, float(np.exp(0.2 * rs.randn())), rs.uniform(0.4, 2.0, D)) for _ in range(S)]
    chs = [(0.0, rs.uniform(0.5, 3.0), rs.uniform(0.5, 2.0), rs.uniform(0.3, 1.5, D)) for _ in range(S)]
    ff = np.where(bad, -1.0, 1.0) + 0.3 * rs.randn(N)
    return hs, chs, ff, comp, labels, np.zeros((0, D)), cand, vals


def test_constrained_grid_pass_and_refinement(engs):
    """N = 14 209 complete points: the float64 classification factor's t_alpha solve and the refinement's three factor
    sets all run above the limit."""
    import torch
    from tests import constrained_oracle as CO
    hs, chs, ff, comp, labels, pend, cand, vals = _constrained_problem(NX, 256, 1)
    eng = engs["f32"]
    ref_m = CO.constraint_mean(KIND, chs[0], ff, comp, cand)
    p, m = eng.constraint_prob_device(KIND, chs, ff, comp, labels, eng.to_dev(cand), want_mean=True)
    torch.cuda.synchronize()
    m = m[0, :cand.shape[0]].cpu().numpy()
    assert np.abs(m - ref_m).max() <= 1e-4 * np.abs(ref_m).max()
    ref = CO.ei_over_hypers(KIND, hs, chs, ff, comp, labels, pend, cand, vals)
    ei = eng.constrained_ei_over_hypers(KIND, hs, chs, ff, comp, labels, pend, cand, vals)
    _assert_parity(ei, ref)
    ctx = engs["f64"].constrained_refine_context(KIND, hs, chs, ff, comp, labels, pend, vals)
    for x in cand[:2]:
        f, g = ctx.value_grad(x)
        f_ref, g_ref = CO.grad_optimize_ei_over_hypers(KIND, hs, chs, ff, x, comp, labels, pend, vals)
        np.testing.assert_allclose(f, f_ref, rtol=1e-6)
        np.testing.assert_allclose(np.ravel(g), np.ravel(g_ref), rtol=1e-6,
                                   atol=1e-10 * max(1.0, np.abs(g_ref).max()))


def test_mlii_value_grad(engs):
    import torch
    from oracle import gp_oracle as O
    from spearmint_b200.gp import GP
    X, y, _, _, _ = _problem(NX, 1, 1, 3, seed=5)
    eng = engs["f64"]
    gp = GP(KIND, engine=eng)
    gp.real_init(X.shape[1], y)
    pt = np.array([0.0, np.log(1e-2), 0.0, np.log(0.7), np.log(1.3)])
    eye = torch.eye(NX, dtype=eng.dtype, device=eng.device)
    f, g = gp.value_grad(pt, eng.to_dev(X), eng.to_dev(y), eye, float(np.mean(y)))
    f_ref, g_ref = O.mll_value_grad(KIND, pt, X, y, float(np.mean(y)))
    np.testing.assert_allclose(f, f_ref, rtol=1e-7)
    np.testing.assert_allclose(g, g_ref, rtol=1e-7, atol=1e-8 * max(1.0, np.abs(g_ref).max()))


@pytest.mark.parametrize("chooser", ["GPEIOptChooserB200", "GPEIperSecChooserB200", "GPEIChooserB200",
                                     "GPConstrainedEIChooserB200"])
def test_chooser_next_at_size(chooser, tmp_path):
    import importlib
    mod = importlib.import_module("spearmint_b200.chooser." + chooser)
    N, M, D = NX, 300, 32
    rs = np.random.RandomState(9)
    grid = rs.rand(N + M + 2, D)
    yv = np.sin(3 * grid[:N]).sum(1)
    values = np.zeros(grid.shape[0])
    values[:N] = (yv - yv.mean()) / yv.std()
    if chooser == "GPConstrainedEIChooserB200":
        values[:N][grid[:N, 0] + grid[:N, 1] > 1.2] = np.inf
    durations = np.ones(grid.shape[0])
    durations[:N] = 1.0 + grid[:N, 0]
    complete = np.arange(N)
    candidates = np.arange(N, N + M)
    pending = np.arange(N + M, N + M + 2)
    ch = mod.init(str(tmp_path), "mcmc_iters=2" if chooser == "GPEIChooserB200" else "mcmc_iters=2,burnin=0")
    np.random.seed(1)
    ret = ch.next(grid, values, durations, candidates, pending, complete)
    if isinstance(ret, tuple):
        assert ret[0] == M and np.all(np.isfinite(ret[1])) and np.all((ret[1] >= 0) & (ret[1] <= 1))
    else:
        assert int(ret) in set(candidates.tolist())
