"""Shared helpers of the tests: golden fixture loading, the inputs of the EI grid pass built as Factor builds them, the
host-side measures of a factorisation's and a triangular solve's error, and the float64 kernel references with their
a-priori bounds."""
import os

import numpy as np
import scipy.linalg as spla

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
U32, U64 = 2.0 ** -24, 2.0 ** -53          # unit roundoff of float32 and float64
GEN_EVAL_U = 24.0                          # kernel evaluation + scaling + fp16 pair of one generator element, units of u amp2

OPT_CASES = ["opt_branin2d", "opt_d8_m52", "opt_d8_m52_pend", "opt_d5_ardse", "opt_d4_m32_pend",
             "opt_d3_se", "opt_d1_m52"]
PSEC_CASES = ["psec_d4", "psec_d3_pend"]


def load(name):
    z = np.load(os.path.join(GOLDEN, name + ".npz"), allow_pickle=False)
    return {k: z[k] for k in z.files}


def hypers(g, prefix="hs"):
    """list of (mean, noise, amp2, ls) tuples, the reference's hyper_samples layout (OPT:628)."""
    return [(float(g[prefix + "_mean"][s]), float(g[prefix + "_noise"][s]), float(g[prefix + "_amp2"][s]),
             np.array(g[prefix + "_ls"][s], dtype=float)) for s in range(len(g[prefix + "_mean"]))]


def sets(g):
    grid, values = g["grid"], g["values"]
    comp = grid[g["complete"]]
    cand = grid[g["candidates"]]
    pend = grid[g["pending"]] if g["pending"].size else np.zeros((0, grid.shape[1]))
    return comp, pend, cand, values[g["complete"]]


# ---------------------------------------------------------------------------------------------------- factorisation checks
NB = 128                # block size of the factor storage (and of the float32 factorisations)


def sym(A):
    """The symmetric matrix whose lower triangle is A's."""
    return np.tril(A) + np.tril(A, -1).T


def ratio(L, A, rows, u, R=None):
    """Componentwise backward error of a product of a lower triangular L with R (default L^T) over the lower triangle
    of the given rows, in units of the unit roundoff u:
        max_{i in rows, j <= i}  |L R - A|_ij / (u (|L| |R|)_ij).
    Componentwise because the augmented pivot A[N, N] = 1e30 of the log-likelihood factor would make a normwise
    max(|L||L^T|) blind to every other entry.  |L L^T - A| <= gamma_{n+1} |L||L^T| holds for Cholesky in any summation
    order, so LAPACK stays below ~n; the same holds for |L X - I| of a triangular inverse X formed by substitution.
    An entry whose |L||R| is exactly 0 (padding) must be reproduced exactly.  Evaluated in float64."""
    L = np.asarray(L, dtype=np.float64)
    R = L.T if R is None else np.asarray(R, dtype=np.float64)
    Lr = L[rows]
    E = np.abs(Lr.dot(R) - A[rows])
    Dn = np.abs(Lr).dot(np.abs(R))
    low = np.arange(A.shape[1])[None, :] <= rows[:, None]
    if np.any(low & (Dn == 0) & (E != 0)) or not np.all(np.isfinite(E[low])):
        return np.inf
    m = low & (Dn > 0)
    return float((E[m] / Dn[m]).max() / u)


def data(N, D, seed):
    """Observations X [N][D] in the unit cube, standardised values y, and the RandomState that drew them."""
    rs = np.random.RandomState(seed)
    X = rs.rand(N, D)
    y = np.sin(3 * X).sum(1) + 0.01 * rs.randn(N)
    return X, (y - y.mean()) / (y.std() if N > 1 else 1.0), rs


def synth_hypers(rs, S, D, noise):
    """bench.synth's hyper-samples with the given noise."""
    return [(0.1 * rs.randn(), noise, float(np.exp(0.25 * rs.randn())), rs.uniform(0.3, 2.0, D)) for _ in range(S)]


def lib():
    from spearmint_b200 import _lib as L
    return L.lib()


def cur_stream():
    import ctypes
    import torch
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def cov_inputs(eng, kind, X, hb, Npad):
    """[S][Npad][Npad] as Factor builds it: smk_cov_build (full symmetric matrix, identity padding)."""
    import torch
    from spearmint_b200.engine import KINDS, check, fn, ptr
    N, D = X.shape
    A = torch.zeros((hb.S, Npad, Npad), dtype=eng.dtype, device=eng.device)
    check(fn("smk_cov_build", eng.dtype)(KINDS[kind], N, N, D, hb.S, ptr(eng.to_dev(X)), None, ptr(hb.inv_ls),
                                         ptr(hb.amp2), ptr(hb.noise), ptr(A), Npad, eng.stream()), "cov_build")
    return A


def factor_path(path, A, Np):
    """Factors A [S][Npad][Npad] in place by one path of the EI grid pass:
      fused   smk_potrf_trtri_tc_f32 (tensor-core Cholesky and explicit inverse in one pipelined call)
      two     smk_potrf_lower_batched_tc_f32, then smk_trtri_split_tc_f32
      simt32  smk_potrf_lower_batched_f32, then smk_trtri_split_f32
      simt64  smk_potrf_lower_batched_f64 (no inverse).
    Returns {"info" (host), "winv", and for the paths with an explicit inverse "hi", "lo" ([S][Np][Np])}.  Every output
    buffer starts as NaN, so an element no kernel writes shows up."""
    import torch
    from spearmint_b200.engine import check, fn, ptr
    L = lib()
    S, Npad, dt, dev = A.shape[0], A.shape[-1], A.dtype, A.device
    st = cur_stream()
    nb = NB if dt == torch.float32 else 64
    out = {"winv": torch.full((S, Npad // nb, nb, nb), float("nan"), dtype=dt, device=dev)}
    info = torch.full((S,), -1, dtype=torch.int32, device=dev)
    if path != "simt64":
        out["hi"] = torch.full((S, Np, Np), float("nan"), dtype=torch.float32, device=dev)
        out["lo"] = torch.full((S, Np, Np), float("nan"), dtype=torch.float32, device=dev)
    if path in ("fused", "two"):
        nb_p = 2 * S * Npad * Npad * 4
        ws = torch.empty((nb_p,), dtype=torch.uint8, device=dev)
        nb_t = L.smk_trtri_tc_workspace_bytes(Npad, Np, S)
        wt = torch.empty((nb_t,), dtype=torch.uint8, device=dev)
        if path == "fused":
            check(L.smk_potrf_trtri_tc_f32(Npad, Np, S, ptr(A), ptr(out["winv"]), ptr(info), ptr(ws), nb_p,
                                           ptr(out["hi"]), ptr(out["lo"]), ptr(wt), nb_t, st), "potrf_trtri_tc")
        else:
            check(L.smk_potrf_lower_batched_tc_f32(Npad, S, ptr(A), ptr(out["winv"]), ptr(info), ptr(ws), nb_p, st),
                  "potrf_tc")
            check(L.smk_trtri_split_tc_f32(Npad, Np, S, ptr(A), ptr(out["winv"]), ptr(out["hi"]), ptr(out["lo"]),
                                           ptr(wt), nb_t, st), "trtri_split_tc")
    else:
        check(fn("smk_potrf_lower_batched", dt)(Npad, S, ptr(A), ptr(out["winv"]), ptr(info), st), "potrf")
        if path == "simt32":
            nb_t = L.smk_trtri_workspace_bytes(Np, S)
            wt = torch.empty((nb_t,), dtype=torch.uint8, device=dev)
            check(L.smk_trtri_split_f32(Npad, Np, S, ptr(A), ptr(out["winv"]), ptr(out["hi"]), ptr(out["lo"]), ptr(wt),
                                        nb_t, st), "trtri_split")
    out["info"] = info.cpu().numpy()           # read back: nothing of this call is in flight afterwards
    return out


# ---------------------------------------------------------------------------------------------------- triangular solve
SOLVE_U = {"f32": U32, "f64": U64}
SOLVE_NB = {"f32": 128, "f64": 64}         # diagonal blocks of the factor and of winv (Cfg<T>::NB)


def gp_factor(eng, N, S, seed, Ntot=None, kind="Matern52", D=4, noise=1e-2):
    """The factor of amp2 (k + 1e-6 I) + noise I over Ntot >= N points (bench.synth's hyper-samples), as Factor builds it,
    by smk_potrf_lower_batched_*.  Returns (A (=L, lower), winv, hb, y [Ntot] standardised); every sample is checked
    positive definite (info == 0)."""
    import torch
    from spearmint_b200.engine import check, fn, ptr
    Ntot = Ntot or N
    X, y, rs = data(Ntot, D, seed)
    hb = eng.hypers(synth_hypers(rs, S, D, noise), kind)
    Npad, nb = (Ntot + 127) // 128 * 128, SOLVE_NB["f32" if eng.dtype == torch.float32 else "f64"]
    A = cov_inputs(eng, kind, X, hb, Npad)
    winv = torch.full((S, Npad // nb, nb, nb), float("nan"), dtype=eng.dtype, device=eng.device)
    info = torch.full((S,), -1, dtype=torch.int32, device=eng.device)
    check(fn("smk_potrf_lower_batched", eng.dtype)(Npad, S, ptr(A), ptr(winv), ptr(info), cur_stream()), "potrf")
    assert not np.any(info.cpu().numpy())
    return A, winv, hb, y


def lmul(Lh, x, trans, absval=False):
    """float64 L x or L^T x for the lower triangular host matrix Lh [N][N] (element type), in row chunks."""
    N = x.shape[0]
    out = np.zeros_like(x)
    for r0 in range(0, N, 2048):
        Lc = Lh[r0:r0 + 2048].astype(np.float64)
        if absval:
            Lc = np.abs(Lc)
        if trans:
            out += Lc.T.dot(x[r0:r0 + 2048])
        else:
            out[r0:r0 + 2048] = Lc.dot(x)
    return out


def berr(Lh, b, a, u):
    """max_i |b - L L^T a|_i / (u (|L||L^T||a|)_i) over the columns of b / a ([N][k], float64)."""
    r = np.abs(b - lmul(Lh, lmul(Lh, a, True), False))
    d = lmul(Lh, lmul(Lh, np.abs(a), True, True), False, True)
    if np.any((d == 0) & (r != 0)) or not np.all(np.isfinite(r)):
        return np.inf
    m = d > 0
    return float((r[m] / d[m]).max() / u)


def skeel_blocks(Lh, W, N, nb):
    """max over diagonal blocks of || |W_b| |L_bb| ||_inf on the rows < N."""
    c = 1.0
    for b in range((N + nb - 1) // nb):
        n = min(nb, N - b * nb)
        Lb = np.abs(Lh[b * nb:b * nb + n, b * nb:b * nb + n].astype(np.float64))
        Wb = np.abs(np.tril(W[b][:n, :n]).astype(np.float64))
        c = max(c, float(Wb.dot(Lb).sum(axis=1).max()))
    return c


def check_solve(prec, Lh, W, b, alpha, quad, sld, tag):
    """One sample of smk_chol_solve(_gm)_* against scipy on the device's own L (Lh [N][N], element type; W its winv).
    b [N][k] as the device forms it (element type); alpha [N][k] (device) or None; quad [k] or None; sld scalar or None.
    Bounds, stated before running:
      alpha: componentwise backward error of the two substitutions <= max(32 x scipy's, 4 (N + NB c)), c the Skeel
             condition of the diagonal blocks (the solve applies the stored block inverses W_b);
      quad:  relative to scipy's |L^-1 b|^2 within max(32 x scipy's own inconsistency |t|^2 - b.alpha, 4 N u);
      sld:   within 4 N u sum |log L_ii| of the float64 sum.
    Returns the measured fraction of each bound checked: {"alpha", "quad", "sld"}."""
    u, N, nb = SOLVE_U[prec], b.shape[0], SOLVE_NB[prec]
    t_sp = spla.solve_triangular(Lh, b, lower=True, check_finite=False)
    a_sp = spla.solve_triangular(Lh, t_sp, lower=True, trans="T", check_finite=False)
    b64 = b.astype(np.float64)
    out = {}
    if alpha is not None:
        r_gpu = berr(Lh, b64, alpha.astype(np.float64), u)
        r_sp = berr(Lh, b64, a_sp.astype(np.float64), u)
        bound = max(32.0 * r_sp, 4.0 * (N + nb * skeel_blocks(Lh, W, N, nb)))
        print("%s: backward error %.3g u (scipy %.3g u, bound %.3g u)" % (tag, r_gpu, r_sp, bound))
        assert r_gpu <= bound, "%s: backward error %.3g u (scipy %.3g, bound %.3g)" % (tag, r_gpu, r_sp, bound)
        out["alpha"] = r_gpu / bound
    if quad is not None:
        q_sp = (t_sp.astype(np.float64) ** 2).sum(axis=0)
        incons = np.abs(q_sp - (b64 * a_sp.astype(np.float64)).sum(axis=0)) / q_sp
        err = np.abs(quad - q_sp) / q_sp
        qb = np.maximum(32.0 * incons, 4.0 * N * u)
        assert np.all(err <= qb), (tag, err, incons)
        out["quad"] = float((err / qb).max())
    if sld is not None:
        d = np.log(np.diag(Lh).astype(np.float64))
        sb = 4.0 * N * u * np.abs(d).sum() + 1e-300
        assert abs(sld - d.sum()) <= sb, (tag, sld, d.sum())
        out["sld"] = abs(sld - d.sum()) / sb
    return out


# ---------------------------------------------------------------------------------------------------- kernel references
def kern(kind, r2):
    """k(r2) of the four kernel kinds (GP:87-127), in the precision of r2."""
    if kind in ("SE", "ARDSE"):
        return np.exp(-0.5 * r2)
    r = np.sqrt(r2)
    if kind == "Matern32":
        a = np.sqrt(3.0) * r
        return (1.0 + a) * np.exp(-a)
    a = np.sqrt(5.0) * r
    return (1.0 + a + (5.0 / 3.0) * r2) * np.exp(-a)


def dkern(kind, r2):
    """|dk / dr2|."""
    if kind in ("SE", "ARDSE"):
        return 0.5 * np.exp(-0.5 * r2)
    r = np.sqrt(r2)
    if kind == "Matern32":
        return 1.5 * np.exp(-np.sqrt(3.0) * r)
    return (5.0 / 6.0) * (1.0 + np.sqrt(5.0) * r) * np.exp(-np.sqrt(5.0) * r)


def gen_bound(kind, r2, nc, nx, D, a2, u, eval_u=GEN_EVAL_U):
    """A-priori bound of one element amp2 k(r2) of a SIMT generator that scales both points (c s, x s, rounded once each),
    takes their difference (rounded once) and accumulates its square over d with D fused multiply-adds: each difference
    is off by at most 2 u (|c s| + |x s|), its square by 4 u |Delta_d| (|c_d| + |x_d|) s_d, and the D fused multiply-adds
    add at most (D + 2) u r2.  By Cauchy-Schwarz the sum over d is at most 4 u sqrt(r2) (|c s| + |x s|) + (D + 2) u r2,
    which moves k by |dk/dr2| times that.  On top, eval_u u amp2 for the evaluation itself (sqrt and exp at most 2 ulp
    each, the rounding of their arguments at most 2.3 u of k, three roundings of the polynomial, the amp2 product; 24
    also covers the fp16 pair of the tensor-core operand).  nc, nx: the norms |c s|, |x s| broadcast against r2."""
    dr2 = 4.0 * np.sqrt(r2) * (nc + nx) + (D + 2.0) * r2
    return u * a2 * (eval_u + 1.01 * dkern(kind, r2) * dr2)


class Worst(object):
    """The largest value per key, recorded once at the end of a test."""

    def __init__(self, rec):
        self.rec, self.v = rec, {}

    def __call__(self, key, val):
        self.v[key] = max(self.v.get(key, 0.0), float(val))

    def flush(self):
        for k, v in sorted(self.v.items()):
            self.rec(k, v)


def same(a, b):
    """Bit for bit, NaN sentinels included."""
    return a.shape == b.shape and np.array_equal(a, b, equal_nan=True)


def frac(err, bound, what):
    """max err / bound, every entry within its bound (an entry whose bound is 0 must be exact)."""
    err = np.atleast_1d(np.asarray(err, dtype=np.float64))       # argwhere of a 0-d array finds nothing
    bound = np.broadcast_to(np.asarray(bound, dtype=np.float64), err.shape)
    assert np.all(np.isfinite(err)), "%s: non-finite entries" % what
    zero = bound == 0
    assert not np.any(err[zero]), "%s: an entry with a zero bound is not exact" % what
    f = float((err[~zero] / bound[~zero]).max()) if np.any(~zero) else 0.0
    bad = np.argwhere(err > bound)
    assert bad.size == 0, "%s: %d entries above the bound, first %s, worst %.3g x the bound" % (what, len(bad),
                                                                                              bad[0].tolist(), f)
    return f


def check_rows(N, Npad, rs, nb=NB):
    """Rows the backward error is evaluated on when a dense |L||L^T| costs too much on the host: the first and last row
    of every nb-block, every 32-piece boundary of a few blocks, the last 200 rows, row N (when it is a row of the matrix)
    and 300 random rows."""
    nblk = Npad // nb
    r = {b * nb for b in range(nblk)} | {b * nb + nb - 1 for b in range(nblk)}
    for b in {0, 1, nblk // 2, nblk - 2, nblk - 1}:
        r |= {b * nb + 32 * p + o for p in range(nb // 32) for o in (0, 31)}
    r |= set(range(Npad - 200, Npad)) | ({N} if N < Npad else set())
    r |= set(rs.choice(Npad, 300, replace=False).tolist())
    return np.array(sorted(r))
