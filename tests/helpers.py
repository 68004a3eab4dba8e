"""Shared helpers of the tests: golden fixture loading, and the host-side measures of a factorisation's error."""
import os

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")

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
