"""TEST INFRASTRUCTURE ONLY -- CPU (numpy/scipy, float64) restatement of the constrained-EI grid pass.

CONS = chooser/GPConstrainedEIChooser.py (relative to ``/root/reference/spearmint/spearmint``).  Pinned against the
reference itself through ``tests/golden/cons_*.npz`` (``tests/golden/make_golden_constrained.py``,
``tests/test_constrained_oracle.py``).  It builds on ``oracle/gp_oracle.py``; like it, only tests and
``__graft_entry__.smoke()`` import it, never the product path.

A constraint hyper-sample is the reference's tuple ``(constraint_mean, constraint_gain, constraint_amp2,
constraint_ls)`` (CONS:294-297, 460-463); ``ff`` is the latent vector of the classification GP over every complete
input.  ``labels[i] = 1`` marks a finite value that is not the user's violating value (CONS:219-232).
"""
import numpy as np
import scipy.linalg as spla
import scipy.stats as sps

from oracle import gp_oracle as G

CONSTRAINT_NOISE = 1e-3   # CONS:184


def labels_of(vals, bad_value=np.inf):
    """1 for a finite value that is not ``bad_value``, else 0 (CONS:219-232)."""
    vals = np.asarray(vals, dtype=float)
    return np.logical_and(vals != bad_value, np.isfinite(vals)).astype(float)


def is_vanilla(labels):
    """No mix of feasible and violating points: the reference skips the classification GP (CONS:816-817)."""
    labels = np.asarray(labels)
    return bool(np.all(labels > 0) or np.all(labels <= 0))


def constraint_mean(kind, chyper, ff, comp_all, cand, noise=CONSTRAINT_NOISE):
    """Latent mean k_c(cand, X_all)' K_c^-1 ff of the classification GP (CONS:819-839).  The constraint mean is not
    added (CONS:444 comments it out, the grid pass never uses it)."""
    _, _, amp2, ls = chyper
    K = G.cov(kind, amp2, ls, comp_all) + noise * np.eye(comp_all.shape[0])
    L = spla.cholesky(K, lower=True)
    t_alpha = spla.cho_solve((L, True), ff)
    return np.dot(G.cov(kind, amp2, ls, comp_all, cand).T, t_alpha)


def constraint_prob(kind, chyper, ff, comp_all, cand, labels, noise=CONSTRAINT_NOISE):
    """P(feasible) = Phi(gain m_c) at the candidates; Phi(gain * 1) everywhere in the vanilla case (CONS:816-842)."""
    gain = chyper[1]
    if is_vanilla(labels):
        return np.full(cand.shape[0], sps.norm.cdf(gain * 1.0))
    return sps.norm.cdf(gain * constraint_mean(kind, chyper, ff, comp_all, cand, noise))


def compute_constrained_ei(kind, hyper, chyper, ff, comp, labels, pend, cand, vals, normals=None,
                           noise=CONSTRAINT_NOISE):
    """GPConstrainedEIChooser.compute_constrained_ei for one pair of samples (CONS:806-940): the objective EI on the
    feasible points only (the pending branch is OPT's, with the fantasy normals ``normals`` (P,F)), times P(feasible)."""
    good = np.asarray(labels) > 0
    ei = G.compute_ei(kind, hyper, comp[good], pend, cand, np.asarray(vals)[good], normals)
    return ei * constraint_prob(kind, chyper, ff, comp, cand, labels, noise)


def ei_over_hypers(kind, hyper_samples, chyper_samples, ff, comp, labels, pend, cand, vals, normals=None,
                   noise=CONSTRAINT_NOISE):
    """(M,S) matrix, one column per (objective, constraint) sample pair (CONS:450-468).  ``normals`` (S,P,F): the
    reference draws a fresh fantasy block from the global RNG for every sample (CONS:910)."""
    out = np.zeros((cand.shape[0], len(hyper_samples)))
    for s, (h, ch) in enumerate(zip(hyper_samples, chyper_samples)):
        out[:, s] = compute_constrained_ei(kind, h, ch, ff, comp, labels, pend, cand, vals,
                                           None if normals is None else normals[s], noise)
    return out


# ----------------------------------------------------------------------------- classification-GP sampler pieces
def latent_loglik(kind, amp2, ls, ff, comp, noise=CONSTRAINT_NOISE):
    """-sum log diag chol K_c - 0.5 ff' K_c^-1 ff, K_c = amp2 (k + 1e-6 I) + noise I: the data term of the joint
    [amp2, ff] move (CONS:1176-1180)."""
    K = G.cov(kind, amp2, ls, comp) + noise * np.eye(comp.shape[0])
    L = spla.cholesky(K, lower=True)
    return -np.sum(np.log(np.diag(L))) - 0.5 * np.dot(ff, spla.cho_solve((L, True), ff))


def latent_factor(kind, amp2, ls, comp, noise):
    """Lower Cholesky factor of amp2 (k + 1e-6 I) + noise I (CONS:1019-1021 with noise 1e-6, CONS:1193-1197)."""
    return spla.cholesky(G.cov(kind, amp2, ls, comp) + noise * np.eye(comp.shape[0]), lower=True)


# ----------------------------------------------------------------------------- refinement objective
def grad_optimize_ei(kind, hyper, chyper, ff, x, comp, labels, pend, vals, normals=None, noise=CONSTRAINT_NOISE):
    """(f, g) of grad_optimize_ei_nopend (CONS:692-803) / grad_optimize_ei_pend (CONS:529-690) for one sample pair at
    one point x (1-D).  ``normals`` (P,F): the block the reference draws after npr.set_state(randomstate) (CONS:618)."""
    mean, nz, amp2, ls = hyper
    _, gain, camp2, cls = chyper
    labels = np.asarray(labels)
    good = labels > 0
    compg, valsg = comp[good], np.asarray(vals, dtype=float)[good]
    vanilla = is_vanilla(labels)
    best = np.min(valsg)
    x = np.reshape(x, (1, -1))
    if not vanilla:                                                                 # CONS:710-733 / 547-575
        Kc = G.cov(kind, camp2, cls, comp) + noise * np.eye(comp.shape[0])
        t_alpha = spla.cho_solve((spla.cholesky(Kc, lower=True), True), ff)
        mc = np.dot(G.cov(kind, camp2, cls, comp, x).T, t_alpha)
        pc = sps.norm.cdf(gain * mc)
        gc = np.dot(t_alpha, G.grad_kernel(kind, cls, comp, x)[:, 0, :])
        gc = 0.5 * camp2 * gain * gc * sps.norm.pdf(gain * mc)                      # CONS:795-799 / 682-686
    if pend.shape[0] == 0:
        K = G.cov(kind, amp2, ls, compg) + nz * np.eye(compg.shape[0])
        L = spla.cholesky(K, lower=True)
        Kf = G.cov(kind, amp2, ls, comp) + nz * np.eye(comp.shape[0])
        Lf = spla.cholesky(Kf, lower=True)                                          # CONS:745-746
        alpha = spla.cho_solve((L, True), valsg - mean)
        kxf = G.cov(kind, amp2, ls, comp, x)
        beta = spla.solve_triangular(Lf, kxf, lower=True)                           # CONS:751
        m = np.dot(G.cov(kind, amp2, ls, compg, x).T, alpha) + mean
        v = amp2 * (1 + G.JITTER) - np.sum(beta ** 2, axis=0)
        s = np.sqrt(v)
        u = (best - m) / s
        ei = s * (u * sps.norm.cdf(u) + sps.norm.pdf(u))
        gm = np.dot(alpha, G.grad_kernel(kind, ls, compg, x)[:, 0, :])
        gv = np.dot(-2 * spla.cho_solve((Lf, True), kxf)[:, 0], G.grad_kernel(kind, ls, comp, x)[:, 0, :])
        g = 0.5 * amp2 * (gm * -sps.norm.cdf(u) + gv * 0.5 * sps.norm.pdf(u) / s)   # CONS:786
        ei_tot = np.sum(ei)
    else:
        cp, Lj, fant, _ = G.fantasies(kind, hyper, compg, pend, valsg, normals)
        kx = G.cov(kind, amp2, ls, cp, x)
        alpha = spla.cho_solve((Lj, True), fant - mean)                             # (N+P, F)
        beta = spla.solve_triangular(Lj, kx, lower=True)
        m = np.dot(kx.T, alpha)[0] + mean                                           # (F,)
        v = amp2 * (1 + G.JITTER) - np.sum(beta ** 2)
        s = np.sqrt(v)
        u = (best - m) / s                                                          # best, not the fantasy bests (CONS:655)
        ei = s * (u * sps.norm.cdf(u) + sps.norm.pdf(u))
        gk = G.grad_kernel(kind, ls, cp, x)[:, 0, :]
        gm = np.dot(alpha.T, gk)                                                    # (F, D)
        gv = np.dot(-2 * spla.cho_solve((Lj, True), kx)[:, 0], gk)                  # (D,)
        g = np.sum(0.5 * amp2 * (gm * -sps.norm.cdf(u)[:, None] + gv[None, :] * (0.5 * sps.norm.pdf(u) / s)[:, None]),
                   axis=0)                                                          # CONS:675-677
        ei_tot = np.sum(ei)                                                         # summed over fantasies (CONS:660)
    if vanilla:
        return -ei_tot, g
    return float(-ei_tot * pc[0]), pc[0] * g + ei_tot * gc


def grad_optimize_ei_over_hypers(kind, hyper_samples, chyper_samples, ff, x, comp, labels, pend, vals, normals=None,
                                 noise=CONSTRAINT_NOISE):
    """Sum over the sample pairs (CONS:471-501)."""
    f, g = 0.0, 0.0
    for h, ch in zip(hyper_samples, chyper_samples):
        fs, gs = grad_optimize_ei(kind, h, ch, ff, x, comp, labels, pend, vals, normals, noise)
        f, g = f + fs, g + gs
    return float(f), np.ravel(g)
