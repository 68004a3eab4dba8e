"""The predict stage of the EI grid pass at the row-group, block and chunk counts it runs at, each kernel against float64
evaluations of its own operands.

Two paths, each through its own C entry point:
  TC    smk_predict_tc_f32 (csrc/predict_tc.cu): the SIMT generator kxt_kernel writes the cross-covariance operand Kxt as a
        scaled fp16 (hi, lo) pair; predict_tc_kernel mode 0 forms beta^T = Kxt Linv^T on wgmma as 3 x FP16 products
        (lo.hi + hi.lo + hi.hi) with float32 accumulation over the lower-trapezoidal k range nk = (g+1) 256 / 32 of row
        group g, two groups (g, ngroups-1-g) per work item, and reduces |beta|^2 (and z . beta when z is given) per
        row-group pair; finish_var_kernel sums the pair partials.  With fantasies, mode 1 multiplies the same Kxt chunk
        by alpha_f^T (Fp = ceil256(F) rows, one group per item, full k range).  The float32 grid pass from N = 2048 on.
  SIMT  smk_predict_f32 / _f64 (csrc/predict.cu): the fused generator plus blocked substitution against L, with the
        finished beta blocks parked in a scratch slab per persistent block.  float32 below N = 2048; float64 at any N for
        the deep-tail re-evaluation and the guard's re-evaluation.
Inputs are built as Factor builds them: smk_cov_build, then smk_potrf_trtri_tc_f32, smk_linv_pack_f16 and
smk_linv_alpha_f32 (TC), or the SIMT factorisation and smk_chol_solve.  Every candidate set starts with the incumbent
itself, the 10-point jitter cloud around it (OPT:236-238) and the last observation: there var cancels down to the noise,
and there the largest EI sits.

Each stage is compared with a float64 evaluation of ITS OWN device inputs, so that a failure points at one kernel:
  generator  Kxt (smk_kxt_pack_f16 impl 0 runs the same kxt_kernel) against amp2 k(X, C) on the float32 operands;
  GEMM       the dumped beta^T against (Kxt hi + lo) 2^-ea (Linv16 hi + lo)^T 2^-eb, i.e. exactly the GEMM's operands;
  epilogue   var against amp2 (1 + 1e-6) - sum_i beta_dev^2, mu against amp2 sum_n alpha_n k_n + mean with the device's
             alpha, and with z the mean + z . beta_dev of the GEMM epilogue;
  mode 1     mu_f against Kx_dev alpha_f + mean, and against smk_cross_mean_f32 / _f64 on the same alpha_f.
The bounds are a-priori and stated next to each check; measured ratios are recorded with record_property and quoted in
the docstrings of the tests.

Unit roundoff u = 2^-24 (float32), 2^-53 (float64).
"""
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import scipy.linalg as spla

from tests.helpers import GEN_EVAL_U, U32, U64, Worst, cov_inputs, cur_stream, data, factor_path, gen_bound, lib, \
    synth_hypers
from tests.helpers import dkern as _dkern, frac as _frac, kern as _kern, same as _same

gpu = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BM, BN = 128, 256                  # candidate tile, row group of the tensor-core GEMM
PROBLEMS = (("Matern52", 32), ("Matern52", 8), ("SE", 3))       # the bench's problem, the smooth D = 8 one, SE D = 3
NOISES = (1e-2, 1e-3, 1e-4)


def _npad(N):
    return (N + 127) // 128 * 128


def _np(N):
    return (N + 255) // 256 * 256


def _ceil128(M):
    return (M + 127) // 128 * 128


def _gemm_u(Np):
    """A-priori bound of one entry of the 3 x FP16 GEMM, in units of u (|A||B|)_ci: the dropped lo.lo term (each lo is at
    most 2^-11 of its value, so 2^-22 = 4 u) plus the truncating float32 accumulation, which loses less than one ulp
    (2 u of the running sum, itself at most (|A||B|)_ci) per addition into the accumulator: 3 MMAs per 16-wide k step give
    3 Np / 16 of them, and the 16-wide reduction inside one MMA adds at most 4 more levels."""
    return 4.0 + 2.0 * (3.0 * Np / 16.0 + 4.0)


# ---------------------------------------------------------------------------------------------------- host references
def _kx_ref(P, C, s, tc_gen=False, u=U32):
    """amp2 k(X, C) [m][N] in float64 on the device's float32 operands, and the a-priori bound of each element.

    SIMT generator (kxt_kernel; the same form holds for the fused generators of predict.cu and cross_mean): the bound of
    helpers.gen_bound, whose GEN_EVAL_U = 24 u amp2 covers the evaluation (sqrt.approx and ex2.approx at most 2 ulp each,
    the rounding of their arguments at most 2.3 u of k, three roundings of the polynomial, the amp2 2^ea product) and
    the fp16 (hi, lo) pair (2^-22 = 4 u).
    Tensor-core generator (kxt_tc.cu): q_d = (x_d - c_d)^2 in the difference form (3 u), its fp16 pair (4 u), w = 1/ls^2
    and its pair (5 u), the dropped lo.lo term (4 u) and the truncating accumulation of 3 x 32 / 16 MMA steps plus 4
    levels (20 u): every term is non-negative, so r2 is off by at most 40 u r2."""
    Xs = P["X"] * P["ils"][s]                  # exact: products of two float32 values
    Cs = C * P["ils"][s]
    nx, nc = np.sqrt((Xs * Xs).sum(1)), np.sqrt((Cs * Cs).sum(1))
    r2 = np.zeros((C.shape[0], Xs.shape[0]))
    for d in range(Xs.shape[1]):               # the difference form: nothing cancels
        r2 += (Cs[:, d:d + 1] - Xs[None, :, d]) ** 2
    a2 = P["amp2"][s]
    K = a2 * _kern(P["kind"], r2)
    if tc_gen:
        gb = u * a2 * (GEN_EVAL_U + 1.01 * _dkern(P["kind"], r2) * 40.0 * r2)
    else:
        gb = gen_bound(P["kind"], r2, nc[:, None], nx[None, :], P["D"], a2, u)
    return K, gb


def _scale_exp(x):
    """scale_exp of tc_common.cuh on the host: 15 - e with x 1.00001 < 2^e, in float32 arithmetic."""
    return 15 - int(np.frexp(np.float32(np.float32(x) * np.float32(1.00001)))[1])


def _ea(a2):
    return _scale_exp(np.float32(np.float32(a2) * np.float32(1.000001)))


# ---------------------------------------------------------------------------------------------------- device plumbing
@pytest.fixture(scope="module")
def engs():
    import torch
    from spearmint_b200.engine import GPEIEngine
    return {"f32": GPEIEngine(dtype=torch.float32), "f64": GPEIEngine(dtype=torch.float64)}


def _setup(engs, path, kind, N, D, noise, S, seed):
    """Factors, inverse, operand pack and alpha exactly as the grid pass builds them.  path: "tc", "simt32", "simt64"."""
    import torch
    from spearmint_b200.engine import check, fn, ptr
    eng = engs["f64" if path == "simt64" else "f32"]
    L = lib()
    st = cur_stream()
    Npad, Np = _npad(N), _np(N)
    X, y, rs = data(N, D, seed)
    hs = synth_hypers(rs, S, D, noise)
    hb = eng.hypers(hs, kind)
    A = cov_inputs(eng, kind, X, hb, Npad)
    out = factor_path("fused" if path == "tc" else path, A, Np)
    assert np.all(out["info"] == 0), out["info"]
    Xd, yd = eng.to_dev(X), eng.to_dev(y)
    P = dict(path=path, eng=eng, kind=kind, N=N, D=D, S=S, Npad=Npad, Np=Np, hs=hs, hb=hb, A=A, winv=out["winv"],
             Xd=Xd, yd=yd, rs=rs, y=y, noise=noise, seed=seed)
    P["X"] = Xd.double().cpu().numpy()
    P["ils"] = hb.inv_ls.double().cpu().numpy()
    P["amp2"] = hb.amp2.double().cpu().numpy()
    P["mean"] = hb.mean.double().cpu().numpy()
    if path == "tc":
        hi, lo = out["hi"], out["lo"]
        h16 = torch.empty((S, Np, Np), dtype=torch.float16, device=eng.device)
        l16 = torch.empty((S, Np, Np), dtype=torch.float16, device=eng.device)
        exps = torch.full((2 * S,), -999, dtype=torch.int32, device=eng.device)
        check(L.smk_linv_pack_f16(Np, S, ptr(hi), ptr(lo), ptr(h16), ptr(l16), ptr(exps), st), "linv_pack_f16")
        alpha = torch.full((S, Npad), float("nan"), dtype=torch.float32, device=eng.device)
        z = torch.full((S, Np), float("nan"), dtype=torch.float32, device=eng.device)
        check(L.smk_linv_alpha_f32(N, Np, S, ptr(hi), ptr(lo), ptr(yd), ptr(hb.mean), ptr(alpha), Npad, ptr(z), st),
              "linv_alpha")
        P.update(hi=hi, lo=lo, h16=h16, l16=l16, exps_dev=exps, exps=exps.cpu().numpy()[:S].astype(int), z=z)
    else:
        alpha = torch.full((S, 1, Npad), float("nan"), dtype=eng.dtype, device=eng.device)
        check(fn("smk_chol_solve", eng.dtype)(N, Npad, S, 1, ptr(A), ptr(out["winv"]), ptr(yd), 0, N, ptr(hb.mean),
                                              ptr(alpha), None, None, st), "chol_solve")
        alpha = alpha.view(S, Npad)
    P["alpha"] = alpha
    P["alpha_h"] = alpha.double().cpu().numpy()
    return P


def _cands(P, M, seed):
    """The incumbent, the jitter cloud around it (OPT:236-238), the last observation, then uniform points; first M."""
    rs = np.random.RandomState(seed)
    X, D = P["X"], P["D"]
    inc = X[int(np.argmin(P["y"]))]
    C = np.vstack([inc[None, :], inc + 1e-3 * rs.randn(10, D), X[-1:], rs.rand(max(M - 12, 0), D)])[:M]
    Cd = P["eng"].to_dev(C)
    return Cd.double().cpu().numpy(), Cd


def _alpha_f(P, F, seed):
    """F fantasy right-hand sides [S][F][Npad] (float32, zero padding): the device's alpha plus perturbations of its size."""
    import torch
    rs = np.random.RandomState(seed)
    S, N, Npad = P["S"], P["N"], P["Npad"]
    a = np.zeros((S, F, Npad))
    for s in range(S):
        sc = np.abs(P["alpha_h"][s, :N]).max()
        a[s, :, :N] = P["alpha_h"][s, :N][None, :] + 0.3 * sc * rs.randn(F, N)
    t = torch.from_numpy(a).to(device=P["eng"].device, dtype=torch.float32)
    return t, t.double().cpu().numpy()


def _predict_tc(P, Cd, F=1, alpha_f=None, z=False, dbg=False, pregen=False, ldm=None, S=None, items=None):
    """One smk_predict_tc_f32 call with NaN-filled outputs at ldm = M + 3 (default).  items: a subset of the samples,
    run as a batch of their own.  Returns host float64 arrays mu [S][ldm], var [S][ldm], mu_f [S][F][ldm], dbg."""
    import torch
    from spearmint_b200.engine import KINDS, check, ptr
    L = lib()
    st = cur_stream()
    eng, hb = P["eng"], P["hb"]
    M = Cd.shape[0]
    N, D, Np, Npad = P["N"], P["D"], P["Np"], P["Npad"]
    sel = slice(None) if items is None else slice(items[0], items[1])
    h16, l16, alpha = P["h16"][sel], P["l16"][sel], P["alpha"][sel]
    exps = P["exps_dev"] if items is None else torch.cat([P["exps_dev"][sel], P["exps_dev"][sel]])
    hb = hb if items is None else hb.slice(items[0], items[1])
    zz = (P["z"][sel] if z else None)
    af = alpha_f[sel] if alpha_f is not None else None
    S = hb.S
    ldm = M + 3 if ldm is None else ldm
    mu = torch.full((S, ldm), float("nan"), dtype=torch.float32, device=eng.device)
    var = torch.full((S, ldm), float("nan"), dtype=torch.float32, device=eng.device)
    mu_f = torch.full((S, F, ldm), float("nan"), dtype=torch.float32, device=eng.device) if F > 1 else None
    db = torch.full((S, _ceil128(M), Np), float("nan"), dtype=torch.float32, device=eng.device) if dbg else None
    nb = L.smk_predict_tc_workspace_bytes(Np, M, S, F)
    ws = torch.empty((nb,), dtype=torch.uint8, device=eng.device)
    kc = KINDS[P["kind"]]
    if pregen:
        check(L.smk_predict_tc_pregen_f32(kc, N, Np, M, D, S, ptr(P["Xd"]), ptr(Cd), ptr(hb.inv_ls), ptr(hb.amp2), ptr(ws),
                                          nb, F, st), "predict_tc_pregen")
    check(L.smk_predict_tc_f32(kc, N, Np, M, D, S, ptr(P["Xd"]), ptr(Cd), ptr(hb.inv_ls), ptr(hb.amp2), ptr(hb.mean),
                               ptr(h16), ptr(l16), ptr(exps), ptr(alpha), Npad, ptr(mu), ptr(var), ldm, ptr(ws), nb,
                               ptr(db), F, ptr(af), ptr(mu_f), ptr(zz), 1 if pregen else 0, st), "predict_tc")
    r = {"mu": mu.double().cpu().numpy(), "var": var.double().cpu().numpy()}
    if mu_f is not None:
        r["mu_f"] = mu_f.double().cpu().numpy()
    if db is not None:
        r["dbg"] = db.double().cpu().numpy()
    return r


def _kxt(P, Cd, impl):
    """smk_kxt_pack_f16 (impl 0: kxt_kernel, the generator predict_tc runs; 1: the tensor-core generator): the operand
    [S][ceil128(M)][Np] as float64 (hi + lo) 2^-ea, and the fused mean [S][M]; None if impl 1 declines the shape."""
    import torch
    from spearmint_b200.engine import KINDS, check, ptr
    L = lib()
    eng, hb = P["eng"], P["hb"]
    M, S, N, Np = Cd.shape[0], P["S"], P["N"], P["Np"]
    Mc = _ceil128(M)
    h16 = torch.full((S, Mc, Np), float("nan"), dtype=torch.float16, device=eng.device)
    l16 = torch.full((S, Mc, Np), float("nan"), dtype=torch.float16, device=eng.device)
    mu = torch.full((S, M), float("nan"), dtype=torch.float32, device=eng.device)
    nb = L.smk_kxt_pack_workspace_bytes(Np, M, S)
    ws = torch.empty((nb,), dtype=torch.uint8, device=eng.device)
    rc = L.smk_kxt_pack_f16(impl, KINDS[P["kind"]], N, Np, M, P["D"], S, ptr(P["Xd"]), ptr(Cd), ptr(hb.inv_ls),
                            ptr(hb.amp2), ptr(hb.mean), ptr(P["alpha"]), P["Npad"], ptr(h16), ptr(l16), ptr(mu), M,
                            ptr(ws), nb, cur_stream())
    if rc == -1 and impl == 1:
        return None, None
    check(rc, "kxt_pack")
    ea = np.array([_ea(a) for a in P["amp2"]], dtype=np.float64)
    K = (h16.double() + l16.double()).cpu().numpy() * (2.0 ** -ea)[:, None, None]
    return K, mu.double().cpu().numpy()


def _subset(M, rs, chunk=None, extra=300):
    """Candidates the host references are evaluated on: the first 12 (incumbent, cloud, last observation), both edges of
    every 128-candidate tile and of every chunk, the last candidate and a few hundred random ones."""
    r = set(range(min(12, M))) | {M - 1}
    for t in range(0, M, BM):
        r |= {t, min(t + BM - 1, M - 1)}
    if chunk:
        for c in range(0, M, chunk):
            r |= {c, min(c + chunk - 1, M - 1)}
    r |= set(rs.choice(M, min(extra, M), replace=False).tolist())
    return np.array(sorted(r))


# ---------------------------------------------------------------------------------------------------- stage checks
def _check_generator(W, tag, K, Kref, gb, N, M, clamped):
    """K [Mc][Np] of one sample on the subset rows given by Kref [m][N]: every element within its bound, exact zeros on
    the observation padding n >= N (all rows), and the rows M .. Mc-1 of the ragged last tile: finite, and for kxt_kernel
    (clamped), which generates them from candidate M - 1, bit for bit the last candidate's row."""
    Kd, Ks = K
    W(tag + "_gen_frac", _frac(np.abs(Ks[:, :N] - Kref), gb, tag + ": generator"))
    assert not np.any(Kd[:, N:]), tag + ": the generator's observation padding n >= N is not zero"
    assert np.all(np.isfinite(Kd[M:])), tag + ": rows of the ragged last tile"
    if clamped:
        assert _same(Kd[M:], np.broadcast_to(Kd[M - 1], Kd[M:].shape)), tag + ": ragged-tile rows != candidate M - 1"


def _check_gemm(W, tag, dbg_rows, A_rows, B, Np):
    """beta^T rows against the float64 product of the GEMM's own operands; bound _gemm_u(Np) u (|A||B|)."""
    ref = A_rows.dot(B.T)
    den = np.abs(A_rows).dot(np.abs(B).T)
    err = np.abs(dbg_rows - ref)
    f = _frac(err, _gemm_u(Np) * U32 * den, tag + ": beta (mode 0 GEMM)")
    m = den > 0
    W(tag + "_gemm_u", float((err[m] / den[m]).max()) / U32 if np.any(m) else 0.0)
    W(tag + "_gemm_frac", f)


def _check_var(W, tag, var, dbg, a2f, Np):
    """var = fl(amp2 1.000001) - sum_i beta_i^2 with the dumped beta: the per-thread fused sums over 2 x 64 columns of a
    pair, 2 shuffle levels and npairs partials add at most (Np + 8) u sum beta^2, the final subtraction u |var|."""
    ssq = (dbg * dbg).sum(1)
    ref = a2f - ssq
    bound = U32 * ((Np + 8) * ssq + np.abs(ref))
    W(tag + "_var_frac", _frac(np.abs(var - ref), bound, tag + ": var from beta (epilogue)"))
    return ref


def _check_mu_alpha(W, tag, mu, Kref, gb, alpha, mean, N):
    """mu = amp2 sum_n alpha_n k_n + mean, alpha the device's own: the kernel values are within gb each, the N-term float32
    sum within (N + 20) u sum |alpha_n K_n|, the final fma and the mean within 2 u |mu|."""
    a = alpha[:N]
    ref = Kref.dot(a) + mean
    bound = np.abs(a)[None, :].dot(gb.T).ravel() + U32 * ((N + 20) * np.abs(Kref).dot(np.abs(a)) + 2 * np.abs(ref) +
                                                          np.abs(mean))
    W(tag + "_mu_frac", _frac(np.abs(mu - ref), bound, tag + ": mu = Kx alpha + mean"))


def _check_mu_z(W, tag, mu, dbg, z, mean, Np):
    """mu = mean + z . beta_dev, z the device's linv_alpha tmp: (Np + 8) u sum |z beta| for the sums, 2 u |mu| for the
    last additions."""
    ref = dbg.dot(z) + mean
    bound = U32 * ((Np + 8) * np.abs(dbg).dot(np.abs(z)) + 2 * np.abs(ref) + np.abs(mean))
    W(tag + "_muz_frac", _frac(np.abs(mu - ref), bound, tag + ": mu = mean + z . beta (GEMM epilogue)"))


def _check_mu_f(W, tag, mu_f, A_rows, af, mean, fexp, Np):
    """mode 1: mu_f[f][c] = sum_n Kx_dev[c][n] alpha_f[f][n] + mean.  The GEMM bound, plus the fp16 pair of alpha_f (4 u of
    each entry, or 2^-25 2^-fexp absolute where the scaled entry is subnormal in fp16), plus 2 u |mu_f|."""
    ref = af.dot(A_rows.T) + mean                                  # [F][m]
    absd = np.abs(af).dot(np.abs(A_rows).T)
    bound = (_gemm_u(Np) + 4.0) * U32 * absd + 2.0 ** -25 * 2.0 ** -fexp * np.abs(A_rows).sum(1)[None, :] + \
        U32 * (2 * np.abs(ref) + np.abs(mean))
    W(tag + "_muf_frac", _frac(np.abs(mu_f - ref), bound, tag + ": mu_f (mode 1 GEMM)"))
    return ref, bound


def _cross_mean(P, Cd, af_dev, F, f64):
    """smk_cross_mean_f32 / _f64 on the same alpha_f (the _f64 one on float64 copies of the float32 operands)."""
    import torch
    from spearmint_b200.engine import KINDS, check, fn, ptr
    eng = P["eng"]
    dt = torch.float64 if f64 else torch.float32
    hb = P["hb"]
    ops = [t.to(dt).contiguous() for t in (P["Xd"], Cd, hb.inv_ls, hb.amp2, hb.mean, af_dev)]   # alive until read back
    S, M = P["S"], Cd.shape[0]
    mu = torch.full((S, F, M), float("nan"), dtype=dt, device=eng.device)
    check(fn("smk_cross_mean", dt)(KINDS[P["kind"]], P["N"], P["Npad"], M, P["D"], S, F, *[ptr(t) for t in ops], ptr(mu),
                                   M, cur_stream()), "cross_mean")
    return mu.double().cpu().numpy()


def _tc_stages(W, P, C, Cd, sub, F, af_dev, af, samples=None, gen_impl=0, r=None):
    """Every stage of the tensor-core predict for the candidates Cd, checked on the rows sub.  Returns the outputs of the
    call without z (mu, var, mu_f, dbg) for the bitwise checks."""
    S, N, Np, M = P["S"], P["N"], P["Np"], Cd.shape[0]
    if r is None:
        r = _predict_tc(P, Cd, F=F, alpha_f=af_dev, dbg=True)
    rz = _predict_tc(P, Cd, F=F, alpha_f=af_dev, z=True, dbg=True)
    K, mu_gen = _kxt(P, Cd, gen_impl)
    for k in ("mu", "var", "mu_f"):
        if k in r:
            assert np.all(np.isfinite(r[k][..., :M])), "%s: unwritten or non-finite entries j < M" % k
            assert np.all(np.isnan(r[k][..., M:])), "%s: entries j >= M were written (ldm = M + 3)" % k
    if gen_impl == 0:                     # the z call runs the default generator
        assert _same(r["var"], rz["var"]) and _same(r["dbg"], rz["dbg"]), "z changed var or beta"
        if "mu_f" in r:
            assert _same(r["mu_f"], rz["mu_f"]), "z changed mu_f"
    B = None
    zh = P["z"].double().cpu().numpy()
    tc_gen = gen_impl == 1
    if F > 1:
        cm32, cm64 = _cross_mean(P, Cd, af_dev, F, False), _cross_mean(P, Cd, af_dev, F, True)
    for s in (range(S) if samples is None else samples):
        tag = "s%d" % s
        Kref, gb = _kx_ref(P, C[sub], s, tc_gen=tc_gen)
        A_rows = K[s][sub]
        _check_generator(W, "gen" if not tc_gen else "gen_tc", (K[s], A_rows), Kref, gb, N, M, clamped=not tc_gen)
        a2f = float(np.float32(np.float32(P["amp2"][s]) * np.float32(1.000001)))
        B = (P["h16"][s].double() + P["l16"][s].double()).cpu().numpy() * 2.0 ** -float(P["exps"][s])
        dbg = r["dbg"][s]
        assert np.all(np.isfinite(dbg)), "%s: beta dump not written everywhere" % tag
        _check_gemm(W, "tc", dbg[sub], A_rows, B, Np)
        del B
        assert not np.any(dbg[:M, N:]), "%s: beta rows i >= N are not exactly zero" % tag
        vref = _check_var(W, "tc", r["var"][s, :M], dbg[:M], a2f, Np)
        W("tc_neg_var_over_amp2", max(0.0, -r["var"][s, :M].min() / a2f))
        W("tc_neg_var_ref_over_amp2", max(0.0, -vref.min() / a2f))
        _check_mu_alpha(W, "tc" if not tc_gen else "tc_gen_tc", r["mu"][s, sub], Kref, gb, P["alpha_h"][s], P["mean"][s], N)
        _check_mu_alpha(W, "kxt" if not tc_gen else "kxt_tc", mu_gen[s, sub], Kref, gb, P["alpha_h"][s], P["mean"][s], N)
        _check_mu_z(W, "tc", rz["mu"][s, :M], rz["dbg"][s][:M], zh[s], P["mean"][s], Np)
        if F > 1:
            fexp = _scale_exp(np.abs(af[s, :, :N]).max())
            ref, bnd = _check_mu_f(W, "tc", r["mu_f"][s][:, sub], A_rows[:, :N], af[s, :, :N], P["mean"][s], fexp, Np)
            # the path below N = 2048 on the same alpha_f: cross_mean_f64 (float64 throughout) and cross_mean_f32
            a = af[s, :, :N]
            tgen = np.abs(a).dot(gb.T)                                          # [F][m]: generator error through alpha_f
            acc = np.abs(a).dot(np.abs(Kref).T)
            ref64 = a.dot(Kref.T) + P["mean"][s]
            b64 = tgen * (U64 / U32) + U64 * ((N + 20) * acc + 2 * np.abs(ref64) + abs(P["mean"][s]))
            W("cm64_vs_tc_frac", _frac(np.abs(r["mu_f"][s][:, sub] - cm64[s][:, sub]), bnd + tgen + b64,
                                       "%s: mu_f against cross_mean_f64" % tag))
            W("cm64_frac", _frac(np.abs(cm64[s][:, sub] - ref64), b64, "%s: cross_mean_f64" % tag))
            b32 = tgen + U32 * ((N + 20) * acc + 2 * np.abs(ref64) + abs(P["mean"][s]))
            W("cm32_frac", _frac(np.abs(cm32[s][:, sub] - ref64), b32, "%s: cross_mean_f32" % tag))
    return r, rz


# ---------------------------------------------------------------------------------------------------- 1. tensor-core path
def _small_cases():
    out, i = [], 0
    for g in range(1, 11):
        for N in sorted({256 * g - 1, 256 * (g - 1) + 1, 256 * g}):
            kind, D = PROBLEMS[i % 3]
            noise, S = NOISES[(i // 3) % 3], (1, 2, 3, 8)[i % 4]
            M, F = (1, 127, 128, 129, 1000)[i % 5], (2, 100, 256, 257)[(i // 2) % 4]
            out.append(pytest.param(N, kind, D, noise, S, M, F, id="g%02d-N%d-%s-D%d-noise%g-S%d-M%d-F%d" % (
                g, N, kind, D, noise, S, M, F)))
            i += 1
    return out


def _bitwise_tc(P, Cd, F, af_dev, r, S_items=True, perm_seed=0):
    """Permuting the candidates permutes every output; a batch item equals the same sample predicted alone."""
    M = Cd.shape[0]
    perm = np.random.RandomState(perm_seed).permutation(M)
    import torch
    rp = _predict_tc(P, Cd[torch.as_tensor(perm, device=Cd.device)].contiguous(), F=F, alpha_f=af_dev)
    for k in ("mu", "var", "mu_f"):
        if k in r:
            assert _same(rp[k][..., :M], r[k][..., :M][..., perm]), "%s: a permutation of the candidates" % k
    if S_items and P["S"] > 1:
        for s in sorted({0, P["S"] - 1}):
            ra = _predict_tc(P, Cd, F=F, alpha_f=af_dev, items=(s, s + 1))
            for k in ("mu", "var", "mu_f"):
                if k in r:
                    assert _same(ra[k][0], r[k][s]), "%s: batch item %d differs from the sample alone" % (k, s)


@gpu
@pytest.mark.parametrize("N,kind,D,noise,S,M,F", _small_cases())
def test_predict_tc_row_groups_1_to_10(engs, record_property, N, kind, D, noise, S, M, F):
    """predict_tc at 1 ... 10 row groups (N = 256 g - 1, 256 (g - 1) + 1 and 256 g: even and odd group counts, and an
    inverse one 128-block wider than the factor at odd block counts), M = 1 ... 1000 (one ragged tile, exact tiles, one
    candidate past a tile), S = 1 ... 8, F = 2 ... 257 fantasies (Fp = 512 at F = 257: two fantasy groups).  Every stage
    against float64 on its own operands, every candidate for var and the z mean, the subset rows for the rest; then
    the bitwise invariants (permutation, batch item alone, ldm = M + 3 with NaN-filled outputs).

    Bounds (units of u = 2^-24): generator 24 + |dk/dr2| times the r2 rounding bound (_kx_ref); GEMM 4 + 2 (3 Np / 16 +
    4) against (|Kx||Linv|)_ic (_gemm_u); var (Np + 8) sum beta^2 + |var|; mean and z mean (N + 20) and (Np + 8) against
    their sums of magnitudes; mu_f the GEMM bound + 4 against (|Kx||alpha_f|).
    Worst measured on an H100 80 GB HBM3 (SXM, 700 W power limit), as a fraction of the bound, at noise 1e-2 / 1e-3 /
    1e-4:
      generator 0.19 / 0.17 / 0.17          GEMM 0.090 / 0.073 / 0.068 (59 / 47 / 39 u)    var 0.028 / 0.065 / 0.045
      mu 0.0016 / 0.0022 / 0.0012           z mean 0.019 / 0.0065 / 0.0068                mu_f 0.048 / 0.052 / 0.086
      cross_mean_f32 0.013 / 0.0031 / 0.0025   cross_mean_f64 0.013 / 0.0052 / 0.0045
    var went negative, down to -1.3e-6, -1.2e-4 and -2.9e-4 amp2: the float64 value from the dumped beta is just as
    negative, so it is the inverse's error in beta, not the epilogue (include/spearmint_b200.h).
    """
    P = _setup(engs, "tc", kind, N, D, noise, S, seed=N + 7 * S)
    C, Cd = _cands(P, M, seed=N + 1)
    af_dev, af = _alpha_f(P, F, seed=N + 2)
    W = Worst(record_property)
    sub = np.arange(M) if M <= 400 else _subset(M, P["rs"])
    r, _ = _tc_stages(W, P, C, Cd, sub, F, af_dev, af)
    _bitwise_tc(P, Cd, F, af_dev, r)
    W.flush()


AT_SIZE = [
    pytest.param(2048, "Matern52", 32, 1e-3, 2, 2, id="g08-N2048-Matern52-D32-noise1e-3-S2"),
    pytest.param(2100, "Matern52", 8, 1e-2, 2, 100, id="g09-N2100-Matern52-D8-noise1e-2-S2-F100"),
    pytest.param(4096, "Matern52", 32, 1e-4, 2, 1, id="g16-N4096-Matern52-D32-noise1e-4-S2"),
    pytest.param(4200, "SE", 3, 1e-2, 1, 257, id="g17-N4200-SE-D3-noise1e-2-S1-F257"),
    pytest.param(8192, "Matern52", 32, 1e-3, 1, 1, id="g32-N8192-Matern52-D32-noise1e-3-S1"),
]


@gpu
@pytest.mark.parametrize("N,kind,D,noise,S,F", AT_SIZE)
def test_predict_tc_at_size(engs, record_property, N, kind, D, noise, S, F):
    """The sizes the grid pass runs at: 8, 9, 16, 17 and 32 row groups (4 to 16 row-group pairs), 4106 candidates (33
    tiles, the last one ragged), fantasies at 9 and 17 groups.  Stage checks on a candidate subset (both edges of every
    tile, the jitter cloud, 300 random ones), var and the z mean on every candidate, then the bitwise invariants.
    Same bounds as test_predict_tc_row_groups_1_to_10.  Worst measured on an H100 80 GB HBM3 (SXM, 700 W power limit),
    as a fraction of the bound, at noise 1e-2 / 1e-3 / 1e-4:
      generator 0.17 / 0.14 / 0.20          GEMM 0.049 / 0.061 / 0.046 (80 / 136 / 71 u; the bound is 3092 u at
      N = 8192)                             var 0.0059 / 0.0051 / 0.0026    mu 1.6e-4 / 2.1e-4 / 1.1e-4
      z mean 0.0017 / 0.0012 / 2.6e-4       mu_f 0.014 / 0.018              cross_mean_f32 4.0e-4 / 2.9e-4
    """
    P = _setup(engs, "tc", kind, N, D, noise, S, seed=N + S)
    C, Cd = _cands(P, 4106, seed=N + 1)
    af_dev, af = (None, None) if F == 1 else _alpha_f(P, F, seed=N + 2)
    W = Worst(record_property)
    r, _ = _tc_stages(W, P, C, Cd, _subset(4106, P["rs"]), F, af_dev, af)
    _bitwise_tc(P, Cd, F, af_dev, r)
    W.flush()


@gpu
def test_predict_tc_headline_samples(engs, record_property):
    """N = 4096 with S = 40 (the headline's Np and 8 row-group pairs with the full sample batch): stage checks on the
    first and the last sample, the other samples through the bitwise batch-item check.  Worst measured on an H100 80 GB
    HBM3 (SXM, 700 W power limit), as a fraction of the bound: generator 0.11, GEMM 0.050 (78 u), var 0.0020."""
    P = _setup(engs, "tc", "Matern52", 4096, 32, 1e-3, 40, seed=40)
    C, Cd = _cands(P, 1300, seed=41)
    W = Worst(record_property)
    r, _ = _tc_stages(W, P, C, Cd, _subset(1300, P["rs"], extra=150), 1, None, None, samples=(0, 39))
    _bitwise_tc(P, Cd, 1, None, r)
    W.flush()


@gpu
@pytest.mark.parametrize("N,S,M,F,budget_mb", [
    pytest.param(4096, 2, 1300, 100, 16, id="g16-N4096-S2-chunks512x2+276-F100"),
    pytest.param(2100, 3, 1500, 257, 8, id="g09-N2100-S3-chunks256x5+220-F257"),
])
def test_predict_tc_chunks(engs, record_property, monkeypatch, N, S, M, F, budget_mb):
    """Candidate chunking (SMK_TC_BUDGET_MB is read on every call): at least three chunks and a ragged tail, so c_begin
    is non-zero and the last chunk has fewer tiles.  mu, var and mu_f equal the single-chunk call bit for bit (each
    output row depends only on its own Kxt row and Linv, in a fixed order); the chunked call is also checked against
    float64 on the chunk-edge subset, through the stage bounds of the single-chunk call's operands."""
    P = _setup(engs, "tc", "Matern52", N, 32 if N == 4096 else 8, 1e-3, S, seed=N + 3)
    C, Cd = _cands(P, M, seed=N + 4)
    af_dev, af = _alpha_f(P, F, seed=N + 5)
    W = Worst(record_property)
    one = _predict_tc(P, Cd, F=F, alpha_f=af_dev, dbg=True)
    per_cand = S * P["Np"] * 4
    chunk = (budget_mb << 20) // per_cand // 128 * 128
    assert 3 <= -(-M // chunk) and M % chunk, "the budget does not give >= 3 chunks with a ragged tail"
    monkeypatch.setenv("SMK_TC_BUDGET_MB", str(budget_mb))
    many = _predict_tc(P, Cd, F=F, alpha_f=af_dev, dbg=True)
    manyz = _predict_tc(P, Cd, F=F, alpha_f=af_dev, z=True)
    monkeypatch.delenv("SMK_TC_BUDGET_MB")
    onez = _predict_tc(P, Cd, F=F, alpha_f=af_dev, z=True)
    for k in ("mu", "var", "mu_f"):
        assert _same(many[k], one[k]), "%s: chunked differs from one chunk" % k
        assert _same(manyz[k], onez[k]), "%s (z): chunked differs from one chunk" % k
    # the beta dump of a chunked call is [S][chunk][Np], and every chunk writes its rows from row 0: the last one is left
    last = (M - 1) // chunk * chunk
    dump = many["dbg"].reshape(-1)[:S * chunk * P["Np"]].reshape(S, chunk, P["Np"])
    assert _same(dump[:, :M - last], one["dbg"][:, last:M]), "dbg_beta of the last chunk"
    _tc_stages(W, P, C, Cd, _subset(M, P["rs"], chunk=chunk, extra=100), F, af_dev, af, r=one)
    W.flush()


@gpu
def test_predict_tc_pregenerated_chunk_0(engs):
    """With z, chunk 0 generated ahead by smk_predict_tc_pregen_f32 and picked up with pregenerated = 1 gives the same
    bits as a call without pre-generation, with and without fantasies."""
    P = _setup(engs, "tc", "Matern52", 2100, 20, 1e-3, 3, seed=5)
    C, Cd = _cands(P, 1000, seed=6)
    af_dev, _ = _alpha_f(P, 100, seed=7)
    for F, a in ((1, None), (100, af_dev)):
        base = _predict_tc(P, Cd, F=F, alpha_f=a, z=True)
        pre = _predict_tc(P, Cd, F=F, alpha_f=a, z=True, pregen=True)
        for k in base:
            assert _same(base[k], pre[k]), "F = %d: %s differs with the pre-generated chunk" % (F, k)


@gpu
def test_predict_tc_stable_across_calls(engs):
    """N = 4096, then N = 640, then N = 4096 again (static streams, events, the pre-generation state and the function
    attribute are reused between calls of different shapes): identical bits, with and without z and pre-generation."""
    def run(N, S, seed, M):
        P = _setup(engs, "tc", "Matern52", N, 32, 1e-3, S, seed=seed)
        C, Cd = _cands(P, M, seed=seed + 1)
        af_dev, _ = _alpha_f(P, 2, seed=seed + 2)
        return [_predict_tc(P, Cd, F=2, alpha_f=af_dev), _predict_tc(P, Cd, z=True, pregen=True)]

    a = run(4096, 2, 11, 700)
    run(640, 3, 12, 300)
    b = run(4096, 2, 11, 700)
    for x, y in zip(a, b):
        for k in x:
            assert _same(x[k], y[k]), "%s differs in the second call at N = 4096" % k


# ---------------------------------------------------------------------------------------------------- child processes
CHILD_CASE = dict(N=2100, kind="Matern52", D=8, noise=1e-3, S=3, M=1500, F=100, seed=2100)


def _run_child(env_extra, out):
    env = dict(os.environ)
    env.update(env_extra)
    cmd = [sys.executable, "-m", "tests.predict_child", out] + ["%s=%s" % kv for kv in sorted(CHILD_CASE.items())]
    r = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, "child failed (%d):\n%s\n%s" % (r.returncode, r.stdout[-3000:], r.stderr[-3000:])
    z = np.load(out)
    return {k: z[k] for k in z.files}


@gpu
def test_predict_tc_overlap_equals_default(engs, monkeypatch):
    """SMK_TC_OVERLAP=1 (two Kxt buffers, the generator of chunk i+1 on a second stream under the GEMM of chunk i; read
    once per process, so run in a child) gives the bits of the default single-buffer chunking, and of one chunk."""
    c = CHILD_CASE
    P = _setup(engs, "tc", c["kind"], c["N"], c["D"], c["noise"], c["S"], seed=c["seed"])
    C, Cd = _cands(P, c["M"], seed=c["seed"] + 1)
    af_dev, _ = _alpha_f(P, c["F"], seed=c["seed"] + 2)
    one = _predict_tc(P, Cd, F=c["F"], alpha_f=af_dev)
    monkeypatch.setenv("SMK_TC_BUDGET_MB", "8")
    many = _predict_tc(P, Cd, F=c["F"], alpha_f=af_dev)
    with tempfile.TemporaryDirectory() as d:
        ch = _run_child({"SMK_TC_OVERLAP": "1", "SMK_TC_BUDGET_MB": "8"}, os.path.join(d, "out.npz"))
    for k in ("mu", "var", "mu_f"):
        assert _same(ch[k], many[k]), "%s: overlap differs from the default chunking" % k
        assert _same(ch[k], one[k]), "%s: overlap differs from one chunk" % k


@gpu
def test_predict_tc_tensor_core_generator(engs, record_property):
    """SMK_KXT_IMPL=tc (the tensor-core generator inside predict_tc; read once per process, so run in a child, with
    SMK_KXT_TC_MIN_LANES=1 so that three samples take it): every stage check with the tensor-core generator's own bound
    (_kx_ref, tc_gen), its operand taken from smk_kxt_pack_f16 impl 1.  Worst measured on an H100 80 GB HBM3 (SXM,
    700 W power limit), as a fraction of the bound: generator 0.16, mu 2.5e-4, GEMM 0.052, var 0.0045, mu_f 0.015."""
    c = CHILD_CASE
    P = _setup(engs, "tc", c["kind"], c["N"], c["D"], c["noise"], c["S"], seed=c["seed"])
    C, Cd = _cands(P, c["M"], seed=c["seed"] + 1)
    af_dev, af = _alpha_f(P, c["F"], seed=c["seed"] + 2)
    with tempfile.TemporaryDirectory() as d:
        ch = _run_child({"SMK_KXT_IMPL": "tc", "SMK_KXT_TC_MIN_LANES": "1"}, os.path.join(d, "out.npz"))
    default = _predict_tc(P, Cd, F=c["F"], alpha_f=af_dev)
    assert not _same(ch["mu"], default["mu"]), "the child did not run the tensor-core generator"
    W = Worst(record_property)
    r = {k: ch[k] for k in ("mu", "var", "mu_f", "dbg")}
    _tc_stages(W, P, C, Cd, _subset(c["M"], P["rs"], extra=150), c["F"], af_dev, af, gen_impl=1, r=r)
    W.flush()


# ---------------------------------------------------------------------------------------------------- engine routing
@gpu
def test_ei_prepared_takes_mode_1_with_fantasies(engs, record_property):
    """N + P >= 2048 with F = 100 fantasies (pending_samples) through prepare / ei_prepared: the engine routes the
    fantasy means to mode 1 of the tensor-core GEMM; mu_f is checked against the float64 cross-covariance of the joint
    inputs times the engine's own alpha_f (GEMM + fp16 pair + generator bounds).  Worst measured on an H100 80 GB HBM3
    (SXM, 700 W power limit): 0.0063 of the bound."""
    eng = engs["f32"]
    N, P_, F, D, kind = 2000, 60, 100, 8, "Matern52"
    X, y, rs = data(N + P_, D, 77)
    comp, pend, vals = X[:N], X[N:], y[:N]
    hs = synth_hypers(rs, 2, D, 1e-3)
    normals = rs.randn(P_, F)
    cand = np.vstack([comp[np.argmin(vals)] + 1e-3 * rs.randn(10, D), rs.rand(990, D)])
    seen = []
    orig = eng.predict

    def spy(*a, **kw):
        out = orig(*a, **kw)
        seen.append((kw.get("impl"), kw.get("alpha_f"), out))
        return out

    eng.predict = spy
    try:
        prep = eng.prepare(kind, hs, comp, pend, vals, normals)
        Cd = eng.to_dev(cand)
        eng.ei_prepared(prep, Cd, True, None)
    finally:
        del eng.predict
    assert len(seen) == 1 and seen[0][0] == "tc" and seen[0][1] is not None, "mode 1 was not taken"
    mu_f = seen[0][2][3].double().cpu().numpy()
    fac = prep.fac
    Pd = dict(kind=kind, D=D, X=fac.X.double().cpu().numpy(), ils=prep.hb.inv_ls.double().cpu().numpy(),
              amp2=prep.hb.amp2.double().cpu().numpy())
    af = prep.alpha.double().cpu().numpy()
    C = Cd.double().cpu().numpy()
    Np, Nj = _np(N + P_), N + P_
    W = Worst(record_property)
    for s in range(2):
        Kref, gb = _kx_ref(Pd, C, s)
        a = af[s, :, :Nj]
        ref = a.dot(Kref.T) + float(prep.hb.mean[s])
        fexp = _scale_exp(np.abs(a).max())
        bound = (_gemm_u(Np) + 4.0) * U32 * np.abs(a).dot(np.abs(Kref).T) + np.abs(a).dot(gb.T) + \
            2.0 ** -25 * 2.0 ** -fexp * np.abs(Kref).sum(1)[None, :] * 1.01 + U32 * 3 * np.abs(ref)
        W("engine_muf_frac", _frac(np.abs(mu_f[s, :, :C.shape[0]] - ref), bound, "engine mu_f, sample %d" % s))
    W.flush()


# ---------------------------------------------------------------------------------------------------- 2. SIMT predict
def _simt_case(engs, record_property, prec, N, kind, D, noise, S, M, seed):
    """smk_predict_f32 / _f64 against float64 substitution on the device's own L.  Per candidate, the variance error must
    be at most max(32 x the error of scipy's solve_triangular in the kernel's precision on the same L and on Kx rounded
    to that precision, floor), floor = 2 (N + 8) u (amp2 + sum beta^2): the float sum of N squares and of the two
    rounded products per term of the substitution, each at most N + 8 sequential roundings of a sum bounded by
    amp2 + sum beta^2 (every candidate, on or off the data, has sum beta^2 <= amp2 (1 + 1e-6)).  The mean (no L) gets
    the generator bound of _check_mu_alpha with the kernel's u.  In float64 scipy's solve is the reference itself, so
    there the floor is the bound."""
    import torch
    from spearmint_b200.engine import KINDS, check, fn, ptr
    path = "simt64" if prec == "f64" else "simt32"
    u = U64 if prec == "f64" else U32
    P = _setup(engs, path, kind, N, D, noise, S, seed)
    eng = P["eng"]
    C, Cd = _cands(P, M, seed + 1)
    ldm = M + 3
    mu = torch.full((S, ldm), float("nan"), dtype=eng.dtype, device=eng.device)
    var = torch.full((S, ldm), float("nan"), dtype=eng.dtype, device=eng.device)
    nb = lib().smk_predict_workspace_bytes(eng.esize, P["Npad"])
    ws = torch.empty((nb,), dtype=torch.uint8, device=eng.device)
    check(fn("smk_predict", eng.dtype)(KINDS[kind], N, P["Npad"], M, D, S, ptr(P["Xd"]), ptr(Cd), ptr(P["hb"].inv_ls),
                                       ptr(P["hb"].amp2), ptr(P["hb"].mean), ptr(P["A"]), ptr(P["winv"]), ptr(P["alpha"]),
                                       ptr(mu), ptr(var), ldm, ptr(ws), nb, cur_stream()), "predict")
    mu, var = mu.double().cpu().numpy(), var.double().cpu().numpy()
    assert np.all(np.isfinite(mu[:, :M])) and np.all(np.isfinite(var[:, :M])), "unwritten entries j < M"
    assert np.all(np.isnan(mu[:, M:])) and np.all(np.isnan(var[:, M:])), "entries j >= M written (ldm = M + 3)"
    sub = np.arange(M) if M <= 400 else _subset(M, P["rs"])
    W = Worst(record_property)
    lt = np.float64 if prec == "f64" else np.float32
    for s in range(S):
        Kref, gb = _kx_ref(P, C[sub], s, u=u)
        Lh = np.tril(P["A"][s, :N, :N].double().cpu().numpy())
        beta = spla.solve_triangular(Lh, Kref.T, lower=True)
        ssq = (beta * beta).sum(0)
        a2f = float(lt(lt(P["amp2"][s]) * lt(1.000001)))
        vref = a2f - ssq
        bl = spla.solve_triangular(Lh.astype(lt), Kref.T.astype(lt), lower=True).astype(np.float64)
        err_lap = np.abs(a2f - (bl * bl).sum(0) - vref)
        floor = 2.0 * (N + 8) * u * (a2f + ssq)
        err = np.abs(var[s, sub] - vref)
        W("%s_var_frac" % prec, _frac(err, np.maximum(32.0 * err_lap.max(), floor), "%s var, sample %d" % (prec, s)))
        if prec == "f32":                  # in float64 LAPACK's solve is the reference itself: the floor applies
            W("f32_var_vs_lapack", float(err.max() / max(err_lap.max(), 1e-300)))
        a = P["alpha_h"][s, :N]
        ref = Kref.dot(a) + P["mean"][s]
        bound = np.abs(a)[None, :].dot(gb.T).ravel() + u * ((N + 20) * np.abs(Kref).dot(np.abs(a)) + 2 * np.abs(ref) +
                                                          abs(P["mean"][s]))
        W("%s_mu_frac" % prec, _frac(np.abs(mu[s, sub] - ref), bound, "%s mu, sample %d" % (prec, s)))
    W.flush()


SIMT_SMALL = [("f32", N, PROBLEMS[i % 3], NOISES[i % 3], (1, 2, 3)[i % 3], M)
              for i, (N, M) in enumerate([(127, 129), (129, 300), (383, 1000), (640, 128), (1280, 257), (1281, 700)])] + \
             [("f64", N, PROBLEMS[i % 3], NOISES[(i + 1) % 3], (2, 1, 3)[i % 3], M)
              for i, (N, M) in enumerate([(63, 100), (65, 129), (200, 300), (640, 256), (1000, 130)])]


@gpu
@pytest.mark.parametrize("prec,N,prob,noise,S,M", [
    pytest.param(*c, id="%s-N%d-%s-D%d-noise%g-S%d-M%d" % (c[0], c[1], c[2][0], c[2][1], c[3], c[4], c[5]))
    for c in SIMT_SMALL])
def test_predict_simt_block_counts(engs, record_property, prec, N, prob, noise, S, M):
    """SIMT f32 at 1 ... 11 blocks of 128, SIMT f64 at 1 ... 16 blocks of its 128-row factor storage: the blocked
    substitution with 1, 2 and many parked beta blocks.  Bounds: _simt_case.  Worst measured on an H100 80 GB HBM3
    (SXM, 700 W power limit), as a fraction of the bound, at noise 1e-2 / 1e-3 / 1e-4:
      f32  var 0.011 / 0.030 / 0.013 (at most 3.0 x scipy's strsm error)   mu 0.0035 / 0.0038 / 0.0011
      f64  var 0.014 / 0.047 / 0.027                                        mu 0.0021 / 0.0066 / 0.0065"""
    _simt_case(engs, record_property, prec, N, prob[0], prob[1], noise, S, M, seed=N + 17 * S)


@gpu
@pytest.mark.parametrize("prec,N,kind,D,noise,S,M", [
    pytest.param("f32", 2047, "Matern52", 8, 1e-3, 3, 1000, id="f32-N2047-Matern52-D8-noise1e-3-S3"),
    pytest.param("f64", 4096, "Matern52", 32, 1e-4, 1, 256, id="f64-N4096-Matern52-D32-noise1e-4-S1-tailfix"),
    pytest.param("f64", 8192, "Matern52", 32, 1e-3, 1, 256, id="f64-N8192-Matern52-D32-noise1e-3-S1-tailfix"),
])
def test_predict_simt_at_size(engs, record_property, prec, N, kind, D, noise, S, M):
    """The largest N of the float32 substitution chain (16 blocks), and the float64 re-evaluation shape of tail_fix (256
    candidates at N = 4096 and 8192: 32 and 64 blocks).  Bounds: _simt_case.  Worst measured on an H100 80 GB HBM3
    (SXM, 700 W power limit), as a fraction of the bound: f32 var 0.0021 (0.42 x strsm's error), mu 2.1e-4; f64 var
    0.0028 (noise 1e-3) and 0.0039 (1e-4), mu 4.8e-5 and 1.8e-4."""
    _simt_case(engs, record_property, prec, N, kind, D, noise, S, M, seed=N + S)


# ---------------------------------------------------------------------------------------------------- 3. the guard
def _guard_host(Lh, X, rows, N, amp2, noise):
    """guard.cu in float64 on the host: p = column i of L L^T, b_r = (X p)_r, the running sums after every 16-wide step
    of each row, t_r = -3 2^-24 run_r, and g = max_q (0.5 |sum b^2 - |L_i|^2| + |sum 2 b t|) / (noise + 1e-6 amp2).
    Also returns, per probe, p, sum b^2 and sum 2 b t with a-priori bounds on the device's float64 evaluation of each:
    the products of float32 values are exact in float64, and a sum of n terms is off by at most n 2^-53 times the sum
    of their magnitudes (so b_r by e_r = 2 N 2^-53 sum_j |X_rj p_j| + the error of p carried through |X|, each prefix
    sum of row r by the same e_r, and run_r by (N / 16 + 1) e_r)."""
    worst, scale, parts = 0.0, 0.0, []
    Xn = X[:N, :N]
    ax = np.abs(Xn)
    steps = np.arange(0, N, 16)
    for i in rows:
        p = Lh[:N, :i + 1].dot(Lh[i, :i + 1])
        terms = Xn * p[None, :]
        b = terms.sum(1)
        run = np.zeros(N)
        for r0 in range(0, N, 512):                      # prefix sums row block by row block
            cs = np.cumsum(terms[r0:r0 + 512], axis=1)
            rr = np.arange(r0, min(r0 + 512, N))
            idx = np.minimum(steps[None, :] + 15, rr[:, None])
            ok = steps[None, :] <= rr[:, None]
            run[rr] = np.where(ok, np.take_along_axis(cs, idx, axis=1), 0.0).sum(1)
        t = -3.0 * 5.9604644775390625e-08 * run
        acc, acc2, li = (b * b).sum(), (2.0 * b * t).sum(), (Lh[i, :i + 1] ** 2).sum()
        worst = max(worst, 0.5 * abs(acc - li) + abs(acc2))
        scale = max(scale, acc + li + abs(acc2))
        ep = 2.0 * N * U64 * np.abs(Lh[:N, :i + 1]).dot(np.abs(Lh[i, :i + 1]))          # error bound of p
        e = 2.0 * N * U64 * ax.dot(np.abs(p)) + ax.dot(ep)                               # ... of b_r and of each prefix
        eb = 2.0 * np.abs(b).dot(e) + N * U64 * acc
        et = 3.0 * 5.9604644775390625e-08 * (N / 16.0 + 1.0) * e                         # ... of t_r
        eb2 = 2.0 * (np.abs(t).dot(e) + np.abs(b).dot(et)) + N * U64 * np.abs(2.0 * b * t).sum()
        parts.append(dict(p=p, ep=ep, acc=acc, eacc=eb, acc2=acc2, eacc2=eb2))
    den = noise + 1e-6 * amp2
    return worst / den, scale / den, parts


@gpu
@pytest.mark.parametrize("N,kind,D,noise,S", [
    pytest.param(300, "Matern52", 8, 1e-3, 2, id="N300-Matern52-D8-noise1e-3-S2"),
    pytest.param(2100, "SE", 3, 1e-2, 2, id="N2100-SE-D3-noise1e-2-S2"),
    pytest.param(4200, "Matern52", 32, 1e-4, 1, id="N4200-Matern52-D32-noise1e-4-S1"),
])
def test_tc_guard_formula(engs, record_property, N, kind, D, noise, S):
    """smk_tc_guard_f32 against the host float64 evaluation of the same formula on the device's L, hi, lo and probe rows
    (row 0, the incumbent, a row of the last 128-block, row N - 1).  Bound: float32 rounding of g (u g) plus the
    float64 accumulation of the device, whose sums of up to N terms of magnitude up to the scale of the cancelling
    difference carry at most 4 N 2^-53 of that scale.
    Each part of g is also checked on its own, from the workspace the test owns (guard.cu: p [S][4][Np], then acc [S][8]
    doubles): p (column i of L L^T), sum_r b_r^2 (acc[s][q]) and the accumulation-bias term sum_r 2 b_r t_r (acc[s][4 + q],
    the running 16-wide sums of guard_bv_kernel), each within the bounds of _guard_host.  In these problems the
    bias term is 78 - 85 % of g, so a wrong running sum moves g by far more than its bound as well.
    Worst measured on an H100 80 GB HBM3 (SXM, 700 W power limit), as a fraction of the bound, at noise 1e-2 / 1e-3 /
    1e-4: g 0.23 / 0.27 / 0.088; p 0.0062 / 0.012 / 0.0013; sum b^2 5.8e-4 / 0.0017 / 0.0024; sum 2 b t 5.2e-6 /
    1.4e-4 / 6.9e-6."""
    import torch
    from spearmint_b200.engine import check, ptr
    P = _setup(engs, "tc", kind, N, D, noise, S, seed=N + 9)
    rows = [0, int(np.argmin(P["y"])), N - 1 - (N % 128) // 2, N - 1]
    assert rows[2] >= (N - 1) // 128 * 128
    eng = P["eng"]
    rows_d = torch.tensor(rows, dtype=torch.int32, device=eng.device)
    g = torch.full((S,), float("nan"), dtype=torch.float32, device=eng.device)
    nb = lib().smk_tc_guard_workspace_bytes(P["Np"], S)
    ws = torch.empty((nb,), dtype=torch.uint8, device=eng.device)
    check(lib().smk_tc_guard_f32(N, P["Npad"], P["Np"], S, ptr(P["A"]), ptr(P["hi"]), ptr(P["lo"]), ptr(P["hb"].amp2),
                                 ptr(P["hb"].noise), ptr(rows_d), ptr(g), ptr(ws), nb, cur_stream()), "tc_guard")
    g = g.double().cpu().numpy()
    wsd = ws.view(torch.float64).cpu().numpy()
    pdev = wsd[:S * 4 * P["Np"]].reshape(S, 4, P["Np"])
    accd = wsd[S * 4 * P["Np"]:S * 4 * P["Np"] + 8 * S].reshape(S, 8)
    noise32 = P["hb"].noise.double().cpu().numpy()
    W = Worst(record_property)
    for s in range(S):
        Lh = np.tril(P["A"][s].double().cpu().numpy())
        X = P["hi"][s].double().cpu().numpy() + P["lo"][s].double().cpu().numpy()
        ref, scale, parts = _guard_host(Lh, X, rows, N, P["amp2"][s], noise32[s])
        assert ref > 0
        for q, h in enumerate(parts):
            what = "guard, sample %d, probe row %d" % (s, rows[q])
            W("guard_p_frac", _frac(np.abs(pdev[s, q, :N] - h["p"]), h["ep"], what + ": p = column of L L^T"))
            W("guard_bb_frac", _frac(abs(accd[s, q] - h["acc"]), h["eacc"], what + ": sum b^2 (%.9g, host %.9g)" % (
                accd[s, q], h["acc"])))
            W("guard_bias_frac", _frac(abs(accd[s, 4 + q] - h["acc2"]), h["eacc2"], what + ": sum 2 b t (%.9g, host %.9g)"
                                       % (accd[s, 4 + q], h["acc2"])))
            W("guard_bias_share", abs(h["acc2"]) / (0.5 * abs(h["acc"] - (Lh[rows[q], :rows[q] + 1] ** 2).sum()) +
                                                   abs(h["acc2"])))
        bound = U32 * ref + 4 * N * U64 * scale
        W("guard_frac", _frac(abs(g[s] - ref), bound, "guard, sample %d (g %.6g, host %.6g)" % (s, g[s], ref)))
    W.flush()


# ---------------------------------------------------------------------------------------------------- host only
@pytest.mark.parametrize("kind", ["SE", "Matern32", "Matern52"])
def test_host_kernel_matches_oracle(kind):
    """The float64 kernel the checks above use is the oracle's (gp.py's) kernel."""
    from oracle import gp_oracle as O
    rs = np.random.RandomState(3)
    X, C, ls = rs.rand(40, 5), rs.rand(30, 5), rs.uniform(0.3, 2.0, 5)
    P = dict(kind=kind, D=5, X=X, ils=(1.0 / (np.ones(5) if kind == "SE" else ls))[None, :], amp2=np.array([1.7]))
    K, gb = _kx_ref(P, C, 0)
    np.testing.assert_allclose(K, O.cov(kind, 1.7, ls, X, C).T, rtol=1e-12, atol=1e-14)
    assert np.all(gb >= GEN_EVAL_U * U32 * 1.7)


def test_bound_check_rejects_scalars_and_arrays():
    """_frac fails on any entry above its bound, for a scalar as for an array (np.argwhere of a 0-d array finds nothing,
    so a scalar check built on it would always pass), and requires exactness where the bound is 0."""
    for err, bound in ((2.0, 1.0), (np.float64(2.0), np.float64(1.0)), (np.array([0.5, 2.0]), 1.0),
                       (np.array([[0.0, 1e-30]]), np.array([[1.0, 0.0]]))):
        with pytest.raises(AssertionError):
            _frac(err, bound, "violation")
    assert _frac(0.5, 1.0, "scalar") == 0.5
    assert _frac(np.array([0.25, 0.0]), np.array([1.0, 0.0]), "array") == 0.25
