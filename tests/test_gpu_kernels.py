"""-m gpu: every C-ABI entry point against the CPU oracle on seeded inputs (float64 build bit-tight,
float32 build within the stated fp64->fp32 tolerances)."""
import numpy as np
import pytest
import scipy.linalg as spla

from oracle import gp_oracle as O

pytestmark = pytest.mark.gpu

KINDS = ["SE", "ARDSE", "Matern32", "Matern52"]


@pytest.fixture(scope="module")
def engines():
    import torch
    from spearmint_b200.engine import GPEIEngine
    return {"f32": GPEIEngine(dtype=torch.float32), "f64": GPEIEngine(dtype=torch.float64)}


def _problem(D, N, M, S, seed, noise=1e-3):
    rs = np.random.RandomState(seed)
    X, Cd = rs.rand(N, D), rs.rand(M, D)
    y = np.sin(3 * X).sum(1) + 0.01 * rs.randn(N)
    y = (y - y.mean()) / y.std()
    hs = [(0.1 * rs.randn(), noise, float(np.exp(0.25 * rs.randn())), rs.uniform(0.3, 2.0, D)) for _ in range(S)]
    return X, Cd, y, hs


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("prec", ["f64", "f32"])
def test_cov_build(engines, kind, prec):
    eng = engines[prec]
    X, Cd, y, hs = _problem(5, 70, 45, 3, 1)
    hb = eng.hypers(hs, kind)
    Ks = eng.cov(kind, hb, eng.to_dev(X)).double().cpu().numpy()
    Kc = eng.cov(kind, hb, eng.to_dev(X), eng.to_dev(Cd)).double().cpu().numpy()
    tol = dict(rtol=1e-12, atol=1e-13) if prec == "f64" else dict(rtol=2e-5, atol=2e-6)
    for s, h in enumerate(hs):
        np.testing.assert_allclose(Ks[s], O.cov(kind, h[2], h[3], X), **tol)
        np.testing.assert_allclose(Kc[s], O.cov(kind, h[2], h[3], X, Cd), **tol)


@pytest.mark.parametrize("prec", ["f64", "f32"])
def test_cov_build_lower(engines, prec):
    """smk_cov_build_lower: the lower triangle (and the padded identity) bit-equal to the full build, the 32 x 32 tiles
    strictly above the diagonal left exactly as they were."""
    import torch
    from spearmint_b200.engine import KINDS as KIDS, check, fn, ptr
    eng = engines[prec]
    dt = eng.dtype
    N, D, S, ld = 150, 5, 2, 256
    X, Cd, y, hs = _problem(D, N, 4, S, 9)
    hb = eng.hypers(hs, "Matern52")
    Xd = eng.to_dev(X)
    full = torch.zeros((S, ld, ld), dtype=dt, device=eng.device)
    low = torch.full((S, ld, ld), -7.0, dtype=dt, device=eng.device)
    st = eng.stream()
    check(fn("smk_cov_build", dt)(KIDS["Matern52"], N, N, D, S, ptr(Xd), None, ptr(hb.inv_ls), ptr(hb.amp2), ptr(hb.noise),
                                  ptr(full), ld, st), "cov_build")
    check(fn("smk_cov_build_lower", dt)(KIDS["Matern52"], N, D, S, ptr(Xd), ptr(hb.inv_ls), ptr(hb.amp2), ptr(hb.noise),
                                        ptr(low), ld, st), "cov_build_lower")
    full, low = full.cpu().numpy(), low.cpu().numpy()
    ti, tj = np.arange(ld)[:, None] // 32, np.arange(ld)[None, :] // 32
    for s in range(S):
        assert np.array_equal(low[s][ti >= tj], full[s][ti >= tj])
        assert np.all(low[s][ti < tj] == -7.0)


@pytest.mark.parametrize("prec,N", [("f64", 64), ("f64", 200), ("f32", 128), ("f32", 300), ("f32", 700)])
def test_potrf_and_solve(engines, prec, N):
    import torch
    eng = engines[prec]
    X, Cd, y, hs = _problem(6, N, 10, 3, 2)
    hb = eng.hypers(hs, "Matern52")
    fac = eng.factor("Matern52", eng.to_dev(X), hb)
    fac.check_pd()
    L = fac.L.double().cpu().numpy()
    tol = 1e-11 if prec == "f64" else 3e-4
    yd = eng.to_dev(y)
    alpha, sld, quad = fac.solve(yd, F=1, want_logdet=True, want_quad=True)
    alpha = alpha.double().cpu().numpy()
    NB = eng.NB
    for s, h in enumerate(hs):
        K = O.cov("Matern52", h[2], h[3], X) + h[1] * np.eye(N)
        Lref = spla.cholesky(K, lower=True)
        Lg = np.tril(L[s, :N, :N])
        assert np.abs(Lg - Lref).max() <= tol * np.abs(Lref).max()
        # padding carries the identity
        pad = L[s, N:, N:]
        assert np.allclose(np.tril(pad), np.eye(pad.shape[0]))
        # diagonal-block inverses
        W = fac.winv[s].double().cpu().numpy()
        for b in range(min(2, fac.Npad // NB)):
            blk = np.tril(L[s, b * NB:(b + 1) * NB, b * NB:(b + 1) * NB])
            assert np.abs(W[b].dot(blk) - np.eye(NB)).max() < (1e-10 if prec == "f64" else 2e-3)
        a_ref = spla.cho_solve((Lref, True), y - h[0])
        assert np.abs(alpha[s, 0, :N] - a_ref).max() <= (1e-8 if prec == "f64" else 2e-2) * np.abs(a_ref).max()
        assert np.all(alpha[s, 0, N:] == 0)
        # float32 pivots carry eps * K_jj / pivot relative error (cancellation in K_jj - sum l^2); the float32 log-det is
        # not used by the product (the sampler's log-likelihood is the float64 build)
        np.testing.assert_allclose(float(sld[s]), np.sum(np.log(np.diag(Lref))), rtol=1e-10 if prec == "f64" else 2e-4)
        np.testing.assert_allclose(float(quad[s, 0]), (y - h[0]).dot(a_ref), rtol=1e-9 if prec == "f64" else 5e-3)


def test_potrf_reports_not_pd(engines):
    import torch
    eng = engines["f32"]
    X = np.random.RandomState(0).rand(40, 3)
    hb = eng.hypers([(0.0, -5.0, 1.0, np.ones(3))], "Matern52")   # negative "noise" -> indefinite
    fac = eng.factor("Matern52", eng.to_dev(X), hb)
    with pytest.raises(np.linalg.LinAlgError):
        fac.check_pd()


def test_solve_multiple_rhs_and_leading_block(engines):
    eng = engines["f64"]
    N, P, F = 90, 5, 7
    X, Cd, y, hs = _problem(4, N + P, 10, 2, 3)
    hb = eng.hypers(hs, "Matern52")
    fac = eng.factor("Matern52", eng.to_dev(X), hb)
    rs = np.random.RandomState(5)
    Y = rs.randn(2, F, N + P)
    a, _, q = fac.solve(eng.to_dev(Y), F=F, y_stride=F * (N + P), ldy=N + P, want_quad=True)
    a = a.cpu().numpy()
    al, _, _ = fac.solve(eng.to_dev(y[:N]), F=1, n_lead=N)
    al = al.cpu().numpy()
    for s, h in enumerate(hs):
        K = O.cov("Matern52", h[2], h[3], X) + h[1] * np.eye(N + P)
        ref = np.linalg.solve(K, (Y[s] - h[0]).T).T
        np.testing.assert_allclose(a[s, :, :N + P], ref, rtol=1e-8, atol=1e-9)
        ref_l = np.linalg.solve(K[:N, :N], y[:N] - h[0])
        np.testing.assert_allclose(al[s, 0, :N], ref_l, rtol=1e-8, atol=1e-9)
        assert np.all(al[s, 0, N:] == 0)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("prec,D,N,M", [("f64", 3, 50, 97), ("f64", 40, 130, 300), ("f32", 8, 200, 1000),
                                        ("f32", 1, 33, 130), ("f32", 33, 260, 515)])
def test_predict_moments(engines, kind, prec, D, N, M):
    eng = engines[prec]
    X, Cd, y, hs = _problem(D, N, M, 3, 4)
    hb = eng.hypers(hs, kind)
    fac = eng.factor(kind, eng.to_dev(X), hb)
    fac.check_pd()
    alpha, _, _ = fac.solve(eng.to_dev(y), F=1)
    mu, var, ldm = eng.predict(kind, fac, eng.to_dev(Cd), alpha)
    mu, var = mu.double().cpu().numpy()[:, :M], var.double().cpu().numpy()[:, :M]
    for s, h in enumerate(hs):
        m_ref, v_ref, _, _ = O.predict(kind, h, X, Cd, y)
        if prec == "f64":
            np.testing.assert_allclose(mu[s], m_ref, rtol=1e-8, atol=1e-9)
            np.testing.assert_allclose(var[s], v_ref, rtol=1e-7, atol=1e-9)
        else:
            # SURVEY 8c: mean rtol 1e-4.  The absolute floor is eps_fp32 * sum_i |Kx_i alpha_i| (fp32 rounding of
            # Kx itself): ~2e-4 for Matern, ~1e-3 for the far worse conditioned SE-type kernels (cond ~ N*amp2/noise
            # with a super-exponential spectrum).  EI-level parity is asserted separately in test_gpu_golden.py.
            floor = 1e-3 if kind in ("SE", "ARDSE") else 2e-4
            np.testing.assert_allclose(mu[s], m_ref, rtol=1e-4, atol=floor)
            np.testing.assert_allclose(var[s], v_ref, rtol=1e-3, atol=floor * h[2])


@pytest.mark.parametrize("prec", ["f64", "f32"])
def test_cross_mean(engines, prec):
    eng = engines[prec]
    D, N, M, F = 5, 77, 210, 11
    X, Cd, y, hs = _problem(D, N, M, 2, 6)
    hb = eng.hypers(hs, "Matern52")
    fac = eng.factor("Matern52", eng.to_dev(X), hb)
    rs = np.random.RandomState(7)
    A = rs.randn(2, F, fac.Npad)
    A[:, :, N:] = 0
    mu = eng.cross_mean("Matern52", fac, eng.to_dev(Cd), eng.to_dev(A), F).double().cpu().numpy()
    for s, h in enumerate(hs):
        Kx = O.cov("Matern52", h[2], h[3], X, Cd)
        ref = A[s, :, :N].dot(Kx) + h[0]
        np.testing.assert_allclose(mu[s, :, :M], ref, rtol=1e-9 if prec == "f64" else 2e-4,
                                   atol=1e-10 if prec == "f64" else 2e-4)


@pytest.mark.parametrize("F", [1, 6])
def test_ei_sweep(engines, F):
    import torch
    eng = engines["f32"]
    rs = np.random.RandomState(8)
    S, M = 5, 1000
    ldm = 1024
    mu = rs.randn(S, F, ldm).astype(np.float32)
    var = np.abs(rs.randn(S, ldm)).astype(np.float32) * 0.5 + 1e-4
    var[0, :10] *= 1e-4            # deep tail: u << 0
    mu[0, :, :10] += 3.0
    best = rs.randn(S, F).astype(np.float32) - 1.0
    lt = (0.3 * rs.randn(S, ldm)).astype(np.float32)
    for log_time in (None, lt):
        ei, ei_sum = eng.ei_sweep(M, S, F, torch.from_numpy(mu).cuda(), torch.from_numpy(var).cuda(), ldm,
                                  torch.from_numpy(best).cuda(),
                                  None if log_time is None else torch.from_numpy(log_time).cuda())
        ref = np.zeros((S, M))
        for s in range(S):
            sdev = np.sqrt(var[s, :M].astype(float))[:, None]
            e = O._ei_from_moments(best[s].astype(float)[None, :], mu[s, :, :M].astype(float).T, sdev).mean(axis=1)
            ref[s] = e / (np.exp(log_time[s, :M].astype(float)) if log_time is not None else 1.0)
        got = ei.double().cpu().numpy()[:, :M]
        # double storage.  float32 moments are evaluated in float32 where u > -4 (cancellation < 20x: ~1e-5 relative) and in
        # double in the tail (u*Phi(u)+phi(u) amplifies 1-ulp erfc/FMA differences by ~u^2 there): the deep-tail entries
        # [0, :10] must be double-exact, everything else float32-exact
        np.testing.assert_allclose(got, ref, rtol=4e-5, atol=1e-300)
        np.testing.assert_allclose(got[0, :10], ref[0, :10], rtol=1e-9, atol=1e-300)
        np.testing.assert_allclose(ei_sum.double().cpu().numpy()[:M], ref.sum(0), rtol=4e-5, atol=1e-300)
        e64, _ = engines["f64"].ei_sweep(M, S, F, torch.from_numpy(mu).double().cuda(), torch.from_numpy(var).double().cuda(),
                                         ldm, torch.from_numpy(best).double().cuda(),
                                         None if log_time is None else torch.from_numpy(log_time).double().cuda())
        np.testing.assert_allclose(e64.cpu().numpy()[:, :M], ref, rtol=1e-9, atol=1e-300)


@pytest.mark.parametrize("M,k", [(10, 3), (5000, 20), (100000, 20), (4097, 1)])
def test_topk_matches_numpy(engines, M, k):
    import torch
    eng = engines["f32"]
    rs = np.random.RandomState(9)
    score = rs.rand(M).astype(np.float32)
    score[rs.randint(0, M, size=max(1, M // 50))] = score.max()   # ties at the top -> first-max rule
    idx, val = eng.topk(torch.from_numpy(score).cuda(), M, k)
    idx, val = idx.cpu().numpy(), val.cpu().numpy()
    assert idx[-1] == int(np.argmax(score))
    order = np.lexsort((-np.arange(M), score))       # ascending score, ties: higher index first
    np.testing.assert_array_equal(idx, order[-k:])
    np.testing.assert_array_equal(val, score[idx])


# ------------------------------------------------------------------------------------------------ tensor-core predict
@pytest.mark.parametrize("D,N,M", [(6, 100, 128), (8, 300, 1000), (3, 520, 257), (40, 260, 200)])
def test_predict_tc_beta_and_moments(engines, D, N, M):
    """wgmma 3xFP16 path: the fp16 operand pack of L^-1 (scale + hi/lo), the dumped beta^T = Kx^T L^-T tile product
    (descriptor / swizzle / pipeline / un-scaling check) and the resulting moments, against the oracle."""
    import torch
    from spearmint_b200 import _lib
    eng = engines["f32"]
    X, Cd, y, hs = _problem(D, N, M, 2, 11)
    hb = eng.hypers(hs, "Matern52")
    fac = eng.factor("Matern52", eng.to_dev(X), hb)
    fac.check_pd()
    alpha, _, _ = fac.solve(eng.to_dev(y), F=1)
    hi, lo, Np = fac.linv()
    Mc = ((M + 127) // 128) * 128
    dbg = torch.zeros((hb.S, Mc, Np), dtype=torch.float32, device=eng.device)
    mu, var, ldm = eng.predict("Matern52", fac, eng.to_dev(Cd), alpha.view(hb.S, fac.Npad), impl="tc", dbg_beta=dbg)
    mu2, var2, _ = eng.predict("Matern52", fac, eng.to_dev(Cd), alpha.view(hb.S, fac.Npad), impl="simt")
    linv = (hi.double() + lo.double()).cpu().numpy()
    h16, l16, exps, _ = fac.linv16()
    exps = exps.cpu().numpy()[:hb.S]
    for s in range(hb.S):       # exact power-of-two scale into [2^14, 2^15), hi + lo reproduces the float32 inverse to 2^-21
        sc = np.abs(linv[s]).max() * 2.0 ** exps[s]
        assert 2.0 ** 14 / 1.0001 <= sc < 2.0 ** 15, (sc, exps[s])     # (the 1.00001 safety factor can land just below 2^14)
        rec = (h16[s].double() + l16[s].double()).cpu().numpy() * 2.0 ** -float(exps[s])
        assert np.abs(rec - linv[s]).max() <= 2.0 ** -21 * np.abs(linv[s]).max()
        big = np.abs(linv[s]) >= 2.0 ** -17 * np.abs(linv[s]).max()
        assert np.all(np.abs(rec - linv[s])[big] <= 2.0 ** -21 * np.abs(linv[s])[big])
    dbg, mu, var = dbg.double().cpu().numpy(), mu.double().cpu().numpy(), var.double().cpu().numpy()
    for s, h in enumerate(hs):
        m_ref, v_ref, L, _ = O.predict("Matern52", h, X, Cd, y)
        Linv_ref = spla.solve_triangular(L, np.eye(N), lower=True)
        # entrywise error of an explicit inverse ~ cond(L) * 2^-21 (sanity bound; beta / var below are what matters)
        assert np.abs(linv[s, :N, :N] - Linv_ref).max() <= 5e-3 * np.abs(Linv_ref).max()
        assert np.all(np.triu(linv[s], 1) == 0)
        beta_ref = spla.solve_triangular(L, O.cov("Matern52", h[2], h[3], X, Cd), lower=True)      # (N, M)
        got = dbg[s, :M, :N].T
        assert np.abs(got - beta_ref).max() <= 2e-3 * np.abs(beta_ref).max(), np.abs(got - beta_ref).max()
        assert np.all(dbg[s, :M, N:] == 0)
        floor = 1e-3 if D <= 3 else 2e-4      # eps_fp32 * sum|Kx alpha|: low-D / large-N problems are worse conditioned
        np.testing.assert_allclose(mu[s, :M], m_ref, rtol=1e-4, atol=floor)
        np.testing.assert_allclose(var[s, :M], v_ref, rtol=1e-3, atol=floor * h[2])
    # and against the SIMT kernel of the same library
    np.testing.assert_allclose(var[:, :M], var2.double().cpu().numpy()[:, :M], rtol=1e-3, atol=floor)
    np.testing.assert_allclose(mu[:, :M], mu2.double().cpu().numpy()[:, :M], rtol=1e-4, atol=floor)


@pytest.mark.parametrize("amp2,noise", [(3e-5, 1e-8), (2.5e3, 1.0), (1.0, 1e-6), (7e-3, 5e-2)])
def test_predict_tc_operand_scaling_range(engines, amp2, noise):
    """The fp16 operand scaling follows amp2 (cross-covariance) and max|L^-1| (which follows 1/sqrt(noise + 1e-6 amp2)):
    moments stay at float32 accuracy over a wide range of both."""
    eng = engines["f32"]
    D, N, M = 5, 300, 384
    X, Cd, y, _ = _problem(D, N, M, 1, 5)
    rs = np.random.RandomState(9)
    hs = [(0.0, noise, amp2, rs.uniform(0.3, 2.0, D)), (0.2, noise * 3, amp2 * 0.37, rs.uniform(0.3, 2.0, D))]
    y = y * np.sqrt(amp2)
    hb = eng.hypers(hs, "Matern52")
    fac = eng.factor("Matern52", eng.to_dev(X), hb)
    fac.check_pd()
    alpha, _, _ = fac.solve(eng.to_dev(y), F=1)
    mu, var, _ = eng.predict("Matern52", fac, eng.to_dev(Cd), alpha.view(hb.S, fac.Npad), impl="tc")
    mu, var = mu.double().cpu().numpy(), var.double().cpu().numpy()
    for s, h in enumerate(hs):
        m_ref, v_ref, _, _ = O.predict("Matern52", h, X, Cd, y)
        np.testing.assert_allclose(var[s, :M], v_ref, rtol=1e-3, atol=3e-4 * h[2])
        np.testing.assert_allclose(mu[s, :M], m_ref, rtol=1e-4, atol=1e-3 * np.sqrt(amp2))


# ---------------------------------------------------------------------------------- cross-covariance operand generators
def _kxt_pack(eng, impl, kind, X, Cd, hs, alpha_np):
    """Runs one generator (0 = packed SIMT, 1 = tensor core) and returns (K [S][M][N] float64, mu [S][M])."""
    import torch
    from spearmint_b200 import _lib
    from spearmint_b200.engine import ptr, check, KINDS as KCODE
    L = _lib.lib()
    hb = eng.hypers(hs, kind)
    N, D = X.shape
    M, S = Cd.shape[0], hb.S
    Np, Mc, ldm = L.smk_tc_np(N), ((M + 127) // 128) * 128, ((M + 127) // 128) * 128
    Xd, Cdev = eng.to_dev(X), eng.to_dev(Cd)
    alpha = torch.zeros((S, Np), dtype=torch.float32, device=eng.device)
    alpha[:, :N] = torch.from_numpy(alpha_np.astype(np.float32)).to(eng.device)
    h16 = torch.full((S, Mc, Np), float("nan"), dtype=torch.float16, device=eng.device)
    l16 = torch.full((S, Mc, Np), float("nan"), dtype=torch.float16, device=eng.device)
    mu = torch.zeros((S, ldm), dtype=torch.float32, device=eng.device)
    nb = L.smk_kxt_pack_workspace_bytes(Np, M, S)
    ws = torch.empty((nb,), dtype=torch.uint8, device=eng.device)
    rc = L.smk_kxt_pack_f16(impl, KCODE[kind], N, Np, M, D, S, ptr(Xd), ptr(Cdev), ptr(hb.inv_ls), ptr(hb.amp2),
                            ptr(hb.mean), ptr(alpha), Np, ptr(h16), ptr(l16), ptr(mu), ldm, ptr(ws), nb, eng.stream())
    if rc == -1:
        return None, None
    check(rc, "kxt_pack")
    torch.cuda.synchronize()
    ea = np.array([15 - np.frexp(np.float32(np.float32(h[2]) * np.float32(1.000001)) * np.float32(1.00001))[1] for h in hs])
    K = (h16.double() + l16.double()).cpu().numpy() * (2.0 ** -ea)[:, None, None]
    return K, mu.double().cpu().numpy()


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("D,N,M,S", [(32, 300, 200, 5), (8, 520, 257, 10), (1, 100, 64, 2), (3, 1000, 130, 40), (17, 129, 128, 33)])
def test_kxt_generators_match_oracle(engines, kind, D, N, M, S):
    """Both generator implementations against the float64 cross-covariance: every element of the operand (incl. zero
    padding of the observation axis) and the fused mean."""
    eng = engines["f32"]
    X, Cd, y, hs = _problem(D, N, M, S, 3)
    Cd[:5] = X[0] + 1e-3 * np.random.RandomState(0).randn(5, D)          # the jitter cloud around an observation
    rs = np.random.RandomState(4)
    alpha = rs.randn(S, N) * 3.0
    for impl in (0, 1):
        K, mu = _kxt_pack(eng, impl, kind, X, Cd, hs, alpha)
        assert K is not None
        assert np.isfinite(K[:, :M]).all()
        assert np.all(K[:, :M, N:] == 0)
        for s, h in enumerate(hs):
            Kref = O.cov(kind, h[2], h[3], X, Cd).T                       # (M, N)
            err = np.abs(K[s, :M, :N] - Kref).max()
            assert err <= 3e-6 * h[2], (impl, s, err)
            mref = Kref @ alpha[s] + h[0]
            np.testing.assert_allclose(mu[s, :M], mref, rtol=2e-5, atol=2e-5 * np.abs(Kref * alpha[s]).sum(1).max())


def test_kxt_tc_generator_declines_unsupported_shapes(engines):
    eng = engines["f32"]
    X, Cd, y, hs = _problem(40, 64, 64, 2, 3)
    K, _ = _kxt_pack(eng, 1, "Matern52", X, Cd, hs, np.zeros((2, 64)))
    assert K is None                                                      # D > 32: the SIMT generator handles it
    K, _ = _kxt_pack(eng, 0, "Matern52", X, Cd, hs, np.zeros((2, 64)))
    assert K is not None
