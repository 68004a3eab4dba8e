"""The factorisations of the EI grid pass at the block counts it runs them at, against LAPACK on the same input.

Four paths, each through its own C entry point:
  TC fused     smk_potrf_trtri_tc_f32: left-looking float32 Cholesky with the rank-(jb*128) update of every block-column
               pair on wgmma 3xTF32 (predict_tc_kernel mode 2) and the explicit inverse L^-1 one block step behind on a
               second stream (mode 3).  The float32 grid pass from N = 2048 on.
  TC two-call  smk_potrf_lower_batched_tc_f32, then smk_trtri_split_tc_f32 (SMK_FUSED_INVERSE=0, Factor.linv()).
  SIMT f32     smk_potrf_lower_batched_f32 (+ smk_trtri_split_f32): the float32 grid pass below N = 2048.
  SIMT f64     smk_potrf_lower_batched_f64 (NB = 64): pending-point conditionals, the deep-tail re-evaluation and the
               latent factors, at any N.
Inputs are built as Factor builds them: smk_cov_build into [S][Npad][Npad], i.e. the full symmetric matrix
amp2 (k + 1e-6 I) + noise I with the identity on the padding, Npad = ceil128(N).  The explicit inverse is [S][Np][Np]
with Np = ceil256(N): at an odd block count it is one block wider than the factor.

Mode 2 first runs at nblk = 3 (with ncols = 128: the last block column alone), with ncols = 256 from nblk = 4; mode 3 from
nblk = 2.  The cases cover nblk = 1 ... 10 with N in each residue class (N = 128 nblk - 1, N = 128 (nblk - 1) + 1 with
the last block almost all padding, N = 128 nblk), and the sizes the grid pass runs at: nblk = 16, 17, 32, 33 and 64.

What a stale block update looks like: a backward error many orders of magnitude above LAPACK's, or non-finite entries.
What a race or a cross-item dependency looks like: a bitwise invariant fails.  Each output tile is produced by one CTA in
a fixed k order, so a batch item equals the same matrix factored alone, the fused call equals the two-call sequence, and
the strict upper triangle (never read) cannot change the lower one.
"""
import functools

import numpy as np
import pytest
import scipy.linalg as spla

from tests.helpers import check_rows, ratio, sym
from tests.helpers import cov_inputs as _inputs, cur_stream as _stream, data as _data, factor_path as _factor
from tests.helpers import lib as _lib, synth_hypers as _hypers

gpu = pytest.mark.gpu

U32, U64 = 2.0 ** -24, 2.0 ** -53      # unit roundoffs
NB = 128                               # block size of the factor storage and of the float32 factorisations
NB64 = 64                              # diagonal-block size of the float64 factorisation
DENSE_MAX = 2048                       # above this N the backward errors are evaluated on a row subset


def _npad(N):
    return (N + NB - 1) // NB * NB


def _np(N):
    return (N + 255) // 256 * 256


# ---------------------------------------------------------------------------------------------------- device plumbing
@pytest.fixture(scope="module")
def engs():
    import torch
    from spearmint_b200.engine import GPEIEngine
    return {"f32": GPEIEngine(dtype=torch.float32), "f64": GPEIEngine(dtype=torch.float64)}


def _same(a, b, A, B):
    """The outputs of two calls (A, B: the factored matrices) are bitwise equal: lower L, winv, info, hi and lo."""
    import torch
    bad = [] if torch.equal(torch.tril(A), torch.tril(B)) else ["L"]
    bad += [k for k in ("winv", "hi", "lo") if k in a and not torch.equal(a[k], b[k])]
    return bad + ([] if np.array_equal(a["info"], b["info"]) else ["info"])


def _item(out, s):
    return {k: v[s:s + 1] for k, v in out.items()}


# ---------------------------------------------------------------------------------------------------- host references
def _potrf_lapack(Ah):
    f = spla.lapack.spotrf if Ah.dtype == np.float32 else spla.lapack.dpotrf
    Lr, info = f(Ah, lower=1, clean=1)
    return Lr, info


def _trtri_lapack(L):
    f = spla.lapack.strtri if L.dtype == np.float32 else spla.lapack.dtrtri
    X, info = f(L, lower=1)
    assert info == 0
    return X


def _check_factor(rec, tag, s, A_in, L, winv, N, rows, u):
    """Backward error of L against LAPACK's on the same input, every diagonal-block inverse, the padding.  Returns the
    host copy of L."""
    Npad, nb = L.shape[-1], winv.shape[-1]
    Ah = A_in[s].cpu().numpy()
    Lg = np.tril(L[s].cpu().numpy())
    Lref, linfo = _potrf_lapack(Ah)
    assert linfo == 0, "%s item %d: LAPACK cannot factor this input (info %d): it tests nothing" % (tag, s, linfo)
    r_gpu, r_lap = ratio(Lg, Ah, rows, u), ratio(Lref, Ah, rows, u)
    del Lref
    bound = max(32.0 * r_lap, 2.0 * N)
    rec("%s_s%d_L_ratio_gpu" % (tag, s), r_gpu)
    rec("%s_s%d_L_ratio_lapack" % (tag, s), r_lap)
    assert r_gpu <= bound, "%s item %d: backward error %.3g u|L||L^T| (LAPACK %.3g, bound %.3g)" % (tag, s, r_gpu, r_lap,
                                                                                                  bound)
    # rows N .. Npad-1 of L: the identity, zero to the left
    ref_pad = np.zeros((Npad - N, Npad), dtype=Lg.dtype)
    ref_pad[:, N:] = np.eye(Npad - N)
    assert np.array_equal(Lg[N:], ref_pad), "%s item %d: padding rows of L" % (tag, s)
    # every diagonal-block inverse W_b: |W_b L_bb - I| against LAPACK's trtri of the same L_bb
    W = winv[s].cpu().numpy()
    eye, br = np.eye(nb), np.arange(nb)
    worst = (0.0, 0.0)
    for b in range(Npad // nb):
        Lbb = Lg[b * nb:(b + 1) * nb, b * nb:(b + 1) * nb]
        assert np.all(np.triu(W[b], 1) == 0), "%s item %d: winv[%d] has entries above the diagonal" % (tag, s, b)
        r_w = ratio(W[b], eye, br, u, R=Lbb)
        r_ref = ratio(_trtri_lapack(Lbb), eye, br, u, R=Lbb)
        assert r_w <= max(32.0 * r_ref, 2.0 * nb), "%s item %d: winv[%d] residual %.3g u (trtri %.3g)" % (tag, s, b, r_w,
                                                                                                     r_ref)
        worst = max(worst, (r_w, r_ref))
    rec("%s_s%d_winv_ratio_gpu_trtri" % (tag, s), worst)
    return Lg


def _check_inverse(rec, tag, s, Lg, hi, lo, N, rows):
    """The explicit inverse X = hi + lo (exact in float64): structure, and the residual |L X - I| / (u |L||X|) of the
    forward substitution L X = I against LAPACK's strtri on the same float32 L.  Returns X."""
    Npad = Lg.shape[0]
    h, l = hi[s].cpu().numpy(), lo[s].cpu().numpy()
    assert np.all(np.triu(h, 1) == 0) and np.all(np.triu(l, 1) == 0), "%s item %d: inverse above the diagonal" % (tag, s)
    X = h.astype(np.float64) + l
    del h, l
    assert not np.any(X[Npad:]) and not np.any(X[:, Npad:]), "%s item %d: inverse rows / cols Npad:Np" % (tag, s)
    ref_pad = np.zeros((Npad - N, Npad))
    ref_pad[:, N:] = np.eye(Npad - N)
    assert np.array_equal(X[N:Npad, :Npad], ref_pad), "%s item %d: padding rows of the inverse" % (tag, s)
    Xs = X[:Npad, :Npad]
    eye = np.eye(Npad)
    r_gpu = ratio(Lg, eye, rows, U32, R=Xs)
    r_ref = ratio(Lg, eye, rows, U32, R=_trtri_lapack(Lg))
    bound = max(32.0 * r_ref, 2.0 * N)
    rec("%s_s%d_X_ratio_gpu" % (tag, s), r_gpu)
    rec("%s_s%d_X_ratio_strtri" % (tag, s), r_ref)
    rec("%s_s%d_XL_ratio_gpu" % (tag, s), ratio(Xs, eye, rows, U32, R=Lg))          # |X L - I|: recorded only
    assert r_gpu <= bound, "%s item %d: |L X - I| %.3g u|L||X| (strtri %.3g, bound %.3g)" % (tag, s, r_gpu, r_ref, bound)
    return X


def _check_linv_alpha(eng, rec, tag, X_all, hi, lo, hb, A_in, N, y, kappa_check):
    """smk_linv_alpha_f32 with ragged N and ld_alpha = Npad: tmp = X (y - mean) and alpha = X^T tmp, each against a float64
    evaluation of the device's own operands within 2 N u of the componentwise sums; alpha[N:] = 0; and once per size
    alpha against a float64 solve on the input within 10 kappa_1 u."""
    import torch
    from spearmint_b200.engine import check, ptr
    S, Np, Npad = hi.shape[0], hi.shape[-1], A_in.shape[-1]
    alpha = torch.full((S, Npad), float("nan"), dtype=torch.float32, device=eng.device)
    tmp = torch.full((S, Np), float("nan"), dtype=torch.float32, device=eng.device)
    yd = eng.to_dev(y)
    check(_lib().smk_linv_alpha_f32(N, Np, S, ptr(hi), ptr(lo), ptr(yd), ptr(hb.mean), ptr(alpha), Npad, ptr(tmp),
                                    _stream()), "linv_alpha")
    alpha, tmp = alpha.cpu().numpy().astype(np.float64), tmp.cpu().numpy().astype(np.float64)
    y32, mean32 = yd.cpu().numpy().astype(np.float64), hb.mean.cpu().numpy().astype(np.float64)
    for s, X in X_all.items():
        r = y32 - mean32[s]
        Xn = X[:N, :N]
        t_ref, t_abs = Xn.dot(r), np.abs(Xn).dot(np.abs(r))
        assert np.all(np.abs(tmp[s, :N] - t_ref) <= 2 * N * U32 * t_abs), "%s item %d: tmp" % (tag, s)
        assert not np.any(tmp[s, N:]), "%s item %d: tmp[N:]" % (tag, s)
        a_ref, a_abs = Xn.T.dot(tmp[s, :N]), np.abs(Xn).T.dot(np.abs(tmp[s, :N]))
        assert np.all(np.abs(alpha[s, :N] - a_ref) <= 2 * N * U32 * a_abs), "%s item %d: alpha" % (tag, s)
        assert not np.any(alpha[s, N:]), "%s item %d: alpha[N:ld_alpha]" % (tag, s)
        if kappa_check and s == min(X_all):
            K = A_in[s].cpu().numpy()[:N, :N].astype(np.float64)
            Lk, info = spla.lapack.dpotrf(K, lower=1, clean=1)
            assert info == 0
            rcond, info = spla.lapack.dpocon(Lk, np.abs(sym(K)).sum(axis=0).max(), uplo="L")
            assert info == 0
            del K
            exact = spla.cho_solve((Lk, True), r)
            err = np.linalg.norm(alpha[s, :N] - exact) / np.linalg.norm(exact)
            rec("%s_alpha_rel_err_kappa1u" % tag, (err, 1.0 / rcond * U32))
            assert err <= 10.0 / rcond * U32, "%s: alpha off by %.3g, kappa_1 u = %.3g" % (tag, err, U32 / rcond)


def _check_pack(eng, hi, lo, X_all, plant):
    """smk_linv_pack_f16: the per-sample scale puts max|hi + lo| in [2^14, 2^15), and (h16 + l16) 2^-e reproduces hi + lo
    to 2^-21 of that maximum.  plant: the largest entry of sample 0 is moved to its last element, which the grid-stride
    loops of the absmax and pack kernels reach in their last pass."""
    import torch
    from spearmint_b200.engine import check, ptr
    S, Np = hi.shape[0], hi.shape[-1]
    if plant:
        hi, lo = hi.clone(), lo.clone()
        top = float(2.0 ** np.ceil(np.log2(np.abs(X_all[0]).max())) * 2.0)      # exact in tf32, > every other entry
        hi[0, Np - 1, Np - 1], lo[0, Np - 1, Np - 1] = top, 0.0
        X_all = dict(X_all)
        X_all[0] = X_all[0].copy()
        X_all[0][Np - 1, Np - 1] = top
    h16 = torch.empty((S, Np, Np), dtype=torch.float16, device=eng.device)
    l16 = torch.empty((S, Np, Np), dtype=torch.float16, device=eng.device)
    exps = torch.full((2 * S,), -999, dtype=torch.int32, device=eng.device)
    check(_lib().smk_linv_pack_f16(Np, S, ptr(hi), ptr(lo), ptr(h16), ptr(l16), ptr(exps), _stream()), "linv_pack_f16")
    exps = exps.cpu().numpy()[:S]
    for s, X in X_all.items():
        m = np.abs(X).max()
        sc = m * 2.0 ** exps[s]
        assert 2.0 ** 14 / 1.0001 <= sc < 2.0 ** 15, ("scale", s, sc, exps[s], plant)   # 1.00001 safety factor
        back = (h16[s].double() + l16[s].double()).cpu().numpy() * 2.0 ** -float(exps[s])
        assert np.abs(back - X).max() <= 2.0 ** -21 * m, ("pack", s, plant)


# ---------------------------------------------------------------------------------------------------- 1. the factorisations
PROBLEMS = (("Matern52", 32), ("Matern52", 8), ("SE", 3))       # the bench's problem, the smooth D = 8 one, SE D = 3
NOISES = (1e-2, 1e-3, 1e-4)
SS = (1, 2, 3, 8)


def _small_cases(path, nblks):
    out, i = [], 0
    for nblk in nblks:
        for N in sorted({NB * nblk - 1, NB * (nblk - 1) + 1, NB * nblk}):
            kind, D = PROBLEMS[i % 3]
            noise, S = NOISES[(i // 3) % 3], SS[i % 4]
            out.append(pytest.param(N, kind, D, noise, S, id="nblk%02d-N%d-%s-D%d-noise%g-S%d" % (nblk, N, kind, D,
                                                                                                 noise, S)))
            i += 1
    return out


def _factor_case(engs, rec, path, N, kind, D, noise, S, seed, plant=False):
    """One case of one path: the batch against LAPACK item by item, then the bitwise invariants on the device."""
    import torch
    eng = engs["f64" if path == "simt64" else "f32"]
    u = U64 if path == "simt64" else U32
    Npad, Np = _npad(N), _np(N)
    X, y, rs = _data(N, D, seed)
    hb = eng.hypers(_hypers(rs, S, D, noise), kind)
    A_in = _inputs(eng, kind, X, hb, Npad)                        # the exact input, kept
    paths = ("fused", "two") if path == "tc" else (path,)
    A = A_in.clone()
    out = _factor(paths[0], A, Np)

    rows = np.arange(Npad) if N <= DENSE_MAX else check_rows(N, Npad, rs, nb=NB64 if path == "simt64" else NB)
    X_all = {}
    for s in range(S):
        Lg = _check_factor(rec, path, s, A_in, A, out["winv"], N, rows, u)
        assert out["info"][s] == 0
        if "hi" in out:
            X_all[s] = _check_inverse(rec, path, s, Lg, out["hi"], out["lo"], N, rows)
        del Lg
    if "hi" in out:
        _check_linv_alpha(eng, rec, path, X_all, out["hi"], out["lo"], hb, A_in, N, y, kappa_check=N >= 2048)
        if N >= 4096:
            _check_pack(eng, out["hi"], out["lo"], X_all, plant=False)
            _check_pack(eng, out["hi"], out["lo"], X_all, plant=True)
    del X_all

    # bitwise invariants: the second tensor-core path, a NaN / a zero strict upper triangle, each item alone
    upper = torch.triu(torch.ones((Npad, Npad), dtype=torch.bool, device=A.device), 1)
    for p in paths:
        if p != paths[0]:
            B = A_in.clone()
            bad = _same(out, _factor(p, B, Np), A, B)
            assert not bad, "%s differs from %s in %s" % (p, paths[0], bad)
        for fill in (float("nan"), 0.0):
            B = A_in.masked_fill(upper, fill)
            bad = _same(out, _factor(p, B, Np), A, B)
            assert not bad, "%s: a strict upper triangle of %s changed %s: it is read" % (p, fill, bad)
    del upper
    if S > 1:
        for s in range(S):
            B = A_in[s:s + 1].clone()
            bad = _same(_item(out, s), _factor(paths[0], B, Np), A[s:s + 1], B)
            assert not bad, "%s: batch item %d differs from the same matrix factored alone in %s" % (paths[0], s, bad)


@gpu
@pytest.mark.parametrize("N,kind,D,noise,S", _small_cases("tc", range(1, 11)))
def test_tc_block_counts_1_to_10(engs, record_property, N, kind, D, noise, S):
    """TC fused and TC two-call at nblk = 1 ... 10 (the engine runs them from nblk = 2; nblk = 1 works at the entry
    points), dense over the whole matrix.

    Bounds: the componentwise backward error of L at most max(32 x spotrf's, 2 N); each |W_b L_bb - I| at most
    max(32 x strtri's, 2 NB); |L X - I| of the explicit inverse at most max(32 x strtri's, 2 N).
    Worst ratio measured on an H100 80 GB HBM3 (SXM, 400 W power limit) over all items, in units of u, with the largest
    GPU / LAPACK quotient of one item in brackets:
      L    noise 1e-2: 340 against spotrf's 52 (8.0x)   1e-3: 296 against 57 (8.9x)   1e-4: 289 against 56 (7.4x)
      X    noise 1e-2: 75 against strtri's 14 (10.9x)   1e-3: 68 against 17 (9.3x)    1e-4: 70 against 12 (10.3x)
      W_b  10.1 against strtri's 6.9
    Above 32 x LAPACK only because of the 2 N floor, which it stays far below: the error of L grows about linearly with
    N, at 0.15 - 0.33 N u here and 0.16 N u at N = 8192 (test_factor_at_size), while LAPACK's stays near 30 u.  That is
    the signature of the truncating float32 accumulation of the tensor cores (guard.cu: about half an ulp of the running
    sum lost in the same direction per 16-wide k step of each of the three MMAs), not of a missing term: a skipped k
    chunk of mode 2 or 3 measures 1e3 u to 1.7e7 u or leaves non-finite entries.
    """
    _factor_case(engs, record_property, "tc", N, kind, D, noise, S, seed=N + 7 * S)


@gpu
@pytest.mark.parametrize("N,kind,D,noise,S", _small_cases("simt32", range(1, 11)))
def test_simt_f32_block_counts_1_to_10(engs, record_property, N, kind, D, noise, S):
    """SIMT f32 (smk_potrf_lower_batched_f32, then smk_trtri_split_f32) at nblk = 1 ... 10, dense.  Same bounds as the
    tensor-core chain.  Worst ratio measured on an H100 80 GB HBM3 (SXM, 400 W power limit), in units of u, with the
    largest GPU / LAPACK quotient of one item in brackets:
      L    noise 1e-2: 47 against spotrf's 54 (1.8x)    1e-3: 32 against 55 (1.2x)    1e-4: 48 against 64 (1.9x)
      X    noise 1e-2: 17 against strtri's 18 (9.1x)    1e-3: 16 against 10 (2.5x)    1e-4: 14 against 13 (2.3x)
      W_b  17.3 against strtri's 7.3
    A rank-NB instead of rank-2NB trailing update measures 1e12 u and more, or leaves non-finite entries.
    """
    _factor_case(engs, record_property, "simt32", N, kind, D, noise, S, seed=N + 11 * S)


@gpu
@pytest.mark.parametrize("N,kind,D,noise,S", _small_cases("simt64", range(1, 11)))
def test_simt_f64_block_counts_2_to_20(engs, record_property, N, kind, D, noise, S):
    """SIMT f64 (smk_potrf_lower_batched_f64, NB = 64) at Npad = 128 ... 1280, i.e. 2 ... 20 diagonal blocks, dense.
    Bounds as above with the float64 u and NB = 64.  Worst ratio measured on an H100 80 GB HBM3 (SXM, 400 W power
    limit), in units of u, with the largest GPU / LAPACK quotient of one item in brackets:
      L    noise 1e-2: 42 against dpotrf's 21 (2.7x)    1e-3: 46 against 27 (2.3x)    1e-4: 65 against 24 (4.4x)
      W_b  24.5 against dtrtri's 2.7
    """
    _factor_case(engs, record_property, "simt64", N, kind, D, noise, S, seed=N + 13 * S)


@gpu
@pytest.mark.parametrize("path,N,kind,D,noise,S", [
    pytest.param("tc", 2048, "Matern52", 32, 1e-3, 4, id="tc-nblk16-N2048-Matern52-D32-noise1e-3-S4"),
    pytest.param("tc", 2100, "Matern52", 8, 1e-2, 2, id="tc-nblk17-N2100-Matern52-D8-noise1e-2-S2"),
    pytest.param("tc", 4096, "Matern52", 32, 1e-4, 2, id="tc-nblk32-N4096-Matern52-D32-noise1e-4-S2"),
    pytest.param("tc", 4200, "SE", 3, 1e-2, 1, id="tc-nblk33-N4200-SE-D3-noise1e-2-S1"),
    pytest.param("tc", 8192, "Matern52", 32, 1e-3, 1, id="tc-nblk64-N8192-Matern52-D32-noise1e-3-S1"),
    pytest.param("simt32", 2047, "Matern52", 8, 1e-3, 3, id="simt32-nblk16-N2047-Matern52-D8-noise1e-3-S3"),
    pytest.param("simt64", 4096, "Matern52", 32, 1e-4, 2, id="simt64-nblk32-N4096-Matern52-D32-noise1e-4-S2"),
    pytest.param("simt64", 1600, "Matern52", 4, 1e-3, 6, id="simt64-nblk13-N1600-Matern52-D4-noise1e-3-S6"),
])
def test_factor_at_size(engs, record_property, path, N, kind, D, noise, S):
    """The sizes the grid pass runs at: N = 2048, 4096 and 8192 (16, 32 and 64 block columns), and N = 2100 and 4200
    (odd block counts: mode 2 with the last block column alone, and an inverse one block wider than the factor); the
    largest N of the SIMT f32 chain; the float64 factor at the headline size and at the latent-factor shape.  Above
    N = 2048 the backward errors are evaluated on a row subset (block edges, 32-piece edges of five blocks, the last 200
    rows, 300 random rows).  At N = 4096 and 8192 the fp16 operand pack is checked too, once with the largest entry
    planted in the last element of sample 0.  Same bounds as at nblk <= 10.  Worst ratio measured on an H100 80 GB HBM3
    (SXM, 400 W power limit), in units of u, L against LAPACK's potrf and X against strtri on the same L:
      tc      N = 2048, noise 1e-3: L 353 against 33, X 134 against 10
              N = 2100, noise 1e-2: L 461 against 42, X 120 against 13
              N = 4096, noise 1e-4: L 611 against 29, X 231 against 9
              N = 4200, noise 1e-2: L 782 against 49, X 192 against 6
              N = 8192, noise 1e-3: L 1330 against 29 (46x), X 388 against 10.5 (37x)
      simt32  N = 2047, noise 1e-3: L 16 against 47, X 20 against 16
      simt64  N = 4096, noise 1e-4: L 55 against 13 (4.7x)                N = 1600, noise 1e-3: L 51 against 25 (2.5x)
    The tensor-core chain exceeds 32 x LAPACK here; see test_tc_block_counts_1_to_10 for why, and why the 2 N floor is
    the bound that applies to it.
    """
    _factor_case(engs, record_property, path, N, kind, D, noise, S, seed=N + S)


@gpu
def test_fused_stable_across_calls(engs):
    """Fused at N = 4096, then at N = 640, then at N = 4096 again: identical bits.  The static second stream and the
    per-block event vector of smk_potrf_trtri_tc_f32 are reused between calls of different block counts."""
    eng = engs["f32"]

    def run(N, S, seed):
        X, y, rs = _data(N, 32, seed)
        A = _inputs(eng, "Matern52", X, eng.hypers(_hypers(rs, S, 32, 1e-3), "Matern52"), _npad(N))
        return A, _factor("fused", A, _np(N))

    A1, o1 = run(4096, 2, 1)
    _, o2 = run(640, 3, 2)
    A3, o3 = run(4096, 2, 1)
    assert np.all(o1["info"] == 0) and np.all(o2["info"] == 0)
    bad = _same(o1, o3, A1, A3)
    assert not bad, "the second fused call at N = 4096 differs in %s" % bad


# ---------------------------------------------------------------------------------------------------- 2. info
def _base(n, seed):
    """A well-conditioned SPD B = L0 L0^T of order n and its Cholesky factor L0 (lower, positive diagonal)."""
    rs = np.random.RandomState(seed)
    L0 = np.tril(rs.randn(n, n), -1) * (0.5 / np.sqrt(n)) + np.diag(1.0 + rs.rand(n))
    return L0.dot(L0.T), L0


@functools.lru_cache(maxsize=4)
def _planted(n, p, bad_item, dt):
    """[3][n][n] of element type dt: two SPD matrices and, in item bad_item, B with B[p, p] -= 2 L0[p, p]^2, whose p-th
    pivot is -L0[p, p]^2 while every leading minor of order <= p is unchanged."""
    mats = []
    for s in range(3):
        B, L0 = _base(n, 1000 * n + 17 * s)
        if s == bad_item:
            B[p, p] -= 2.0 * L0[p, p] ** 2
        mats.append(B.astype(dt))
    return np.stack(mats)


INFO_CASES = ([("tc", 2, p, i % 3) for i, p in enumerate((0, 127, 128, 255))]
              + [("tc", 5, p, i % 3) for i, p in enumerate((256, 383, 639))]
              + [("tc", 32, 3000, 1)]
              + [("simt32", 3, p, i % 3) for i, p in enumerate((40, 159, 383))]
              + [("simt32", 10, 1000, 1)]
              + [("simt64", 2, p, i % 3) for i, p in enumerate((63, 64, 200))]
              + [("simt64", 10, 700, 2)])
INFO_IDS = ["%s-nblk%d-p%d-item%d" % c for c in INFO_CASES]


@pytest.mark.parametrize("path,nblk,p,bad_item", INFO_CASES, ids=INFO_IDS)
def test_planted_pivot_fixture_lapack(path, nblk, p, bad_item):
    """The fixture of test_info_names_planted_pivot: LAPACK's spotrf / dpotrf stops at exactly the planted pivot, and
    factors the other items."""
    host = _planted(NB * nblk, p, bad_item, np.float64 if path == "simt64" else np.float32)
    for s in range(3):
        assert _potrf_lapack(host[s])[1] == (p + 1 if s == bad_item else 0), s


@gpu
@pytest.mark.parametrize("path,nblk,p,bad_item", INFO_CASES, ids=INFO_IDS)
def test_info_names_planted_pivot(engs, path, nblk, p, bad_item):
    """info of the item with the planted pivot is exactly p + 1, the others 0; the other items are bitwise equal to the
    same matrices factored alone, inverses included.  On the tensor-core chain both paths, which agree bit for bit."""
    import torch
    eng = engs["f64" if path == "simt64" else "f32"]
    host = _planted(NB * nblk, p, bad_item, np.float64 if path == "simt64" else np.float32)
    Np = _np(NB * nblk)
    paths = ("fused", "two") if path == "tc" else (path,)
    expect = [p + 1 if s == bad_item else 0 for s in range(3)]
    first = None
    for q in paths:
        A = torch.from_numpy(host).to(eng.device)
        out = _factor(q, A, Np)
        assert out["info"].tolist() == expect, (q, out["info"], expect)
        if first is None:
            first = (A, out)
        else:
            bad = _same(first[1], out, first[0], A)
            assert not bad, "%s differs from %s in %s" % (q, paths[0], bad)
        for s in range(3):
            if s == bad_item:
                continue
            B = torch.from_numpy(host[s:s + 1]).to(eng.device)
            bad = _same(_item(out, s), _factor(q, B, Np), A[s:s + 1], B)
            assert not bad, "%s: item %d differs from the same matrix factored alone in %s" % (q, s, bad)
