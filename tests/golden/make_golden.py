#!/usr/bin/env python
"""Generates tests/golden/*.npz by EXECUTING the reference (through oracle/ref_shim.py).

Run in the build container only (needs /root/reference):
    python tests/golden/make_golden.py [name ...]        (no name: every case in CASES)
Each .npz holds the exact inputs handed to the reference and the outputs it produced
(float64), so the fixtures travel to the GPU box where the reference does not exist.
"""
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle import ref_shim  # noqa: E402

R = ref_shim.load()
gp, OPT, PSEC, GPEI, sobol = R["gp"], R["OPT"], R["PSEC"], R["GPEI"], R["sobol_lib"]
KINDS = ["SE", "ARDSE", "Matern32", "Matern52"]


def synth(D, N, M, P, seed):
    """SURVEY 8(d) synthetic problem on the reference's own Sobol grid."""
    G = N + M + P
    grid = sobol.i4_sobol_generate(D, G, 1).T
    perm = np.random.RandomState(seed).permutation(G)
    complete = np.sort(perm[:N])
    pending = np.sort(perm[N:N + P])
    candidates = np.sort(perm[N + P:])
    values = np.full(G, np.nan)
    y = np.sin(3 * grid[complete]).sum(1) + 0.01 * np.random.RandomState(seed + 1).randn(N)
    values[complete] = (y - y.mean()) / y.std()
    durations = np.full(G, np.nan)
    durations[complete] = 1.0 + grid[complete, 0]
    return grid, values, durations, candidates, pending, complete


def pack_hypers(hs):
    return (np.array([h[0] for h in hs]), np.array([h[1] for h in hs]),
            np.array([h[2] for h in hs]), np.vstack([h[3] for h in hs]))


def golden_kernels():
    rs = np.random.RandomState(11)
    out = {}
    for D in (1, 3, 8):
        x1, x2 = rs.rand(7, D), rs.rand(5, D)
        ls = rs.uniform(0.3, 2.0, D)
        out["D%d_x1" % D], out["D%d_x2" % D], out["D%d_ls" % D] = x1, x2, ls
        out["D%d_dist2_self" % D] = gp.dist2(ls, x1)
        out["D%d_dist2_cross" % D] = gp.dist2(ls, x1, x2)
        out["D%d_grad_dist2" % D] = gp.grad_dist2(ls, x1, x2)
        for k in KINDS:
            f = getattr(gp, k)
            out["D%d_%s_self" % (D, k)] = f(ls, x1)
            out["D%d_%s_cross" % (D, k)] = f(ls, x1, x2)
            gk = "ARDSE" if k == "SE" else k
            gls = np.ones_like(ls) if k == "SE" else ls
            out["D%d_%s_grad" % (D, k)] = getattr(gp, "grad_" + gk)(gls, x1, x2)
    np.savez_compressed(os.path.join(HERE, "kernels.npz"), **out)


def record_logprobs(mod):
    """Wrap the reference slice sampler so every logprob evaluation is recorded."""
    rec = []
    orig = mod.util.slice_sample

    def wrapped(init_x, logprob, **kw):
        def lp(x):
            v = logprob(x)
            rec.append((np.array(x, dtype=float).copy(), float(v)))
            return v
        return orig(init_x, lp, **kw)
    mod.util.slice_sample = wrapped
    return rec, (lambda: setattr(mod.util, "slice_sample", orig))


def golden_se(name, D, N, M, S, seed):
    """covar=SE: the reference's next() raises AttributeError (gp has no grad_SE, OPT:404), so only
    ei_over_hypers with injected hyper-samples is frozen."""
    grid, values, durations, candidates, pending, complete = synth(D, N, M, 0, seed)
    ch = OPT.init(tempfile.mkdtemp(), "covar=SE,mcmc_iters=%d,use_multiprocessing=0" % S)
    comp, cand, pend, vals = grid[complete], grid[candidates], grid[pending], values[complete]
    ch._real_init(D, vals)
    rs = np.random.RandomState(seed)
    hs = [(0.1 * rs.randn(), 1e-3, float(np.exp(0.25 * rs.randn())), rs.uniform(0.3, 2.0, D)) for _ in range(S)]
    ch.hyper_samples = hs
    overall = ch.ei_over_hypers(comp, pend, cand, vals)
    m, n, a, l = pack_hypers(hs)   # before next(): its burn-in appends to this very list
    raised = 0
    try:
        np.random.seed(seed)
        ch.next(grid, values, durations, candidates, pending, complete)
    except AttributeError:
        raised = 1
    np.savez_compressed(os.path.join(HERE, name + ".npz"), kind="SE", S=S, grid=grid, values=values,
                        durations=durations, candidates=candidates, pending=pending, complete=complete,
                        hs_mean=m, hs_noise=n, hs_amp2=a, hs_ls=l, overall_ei=overall,
                        normals=np.zeros((0, 100)), next_raises_attribute_error=raised)
    print(name, "max mean EI", overall.mean(1).max(), "next() raised AttributeError:", raised)


def golden_opt(name, D, N, M, P, kind, S, noiseless, seed, burnin=8, ngrad=3):
    """GPEIOptChooser: sampler draws, ei_over_hypers, grad_optimize_ei_over_hypers, next()."""
    grid, values, durations, candidates, pending, complete = synth(D, N, M, P, seed)
    d = tempfile.mkdtemp()
    args = "covar=%s,mcmc_iters=%d,burnin=%d,noiseless=%d,use_multiprocessing=0,grid_subset=5" % (
        kind, S, burnin, int(noiseless))
    ch = OPT.init(d, args)
    np.random.seed(seed)
    state0 = np.random.get_state()
    rec, undo = record_logprobs(OPT)
    ret = ch.next(grid, values, durations, candidates, pending, complete)
    undo()
    hs = list(ch.hyper_samples)
    comp, cand, pend = grid[complete], grid[candidates], grid[pending]
    vals = values[complete]
    # The fantasy normals the reference draws after npr.set_state(self.randomstate) (OPT:588-589)
    np.random.set_state(ch.randomstate)
    normals = np.random.randn(max(P, 1), ch.pending_samples)[:P]
    overall = ch.ei_over_hypers(comp, pend, cand, vals)
    rsg = np.random.RandomState(seed + 5)
    gpts = rsg.rand(ngrad, D)
    gf, gg = [], []
    for x in gpts:
        f, g = ch.grad_optimize_ei_over_hypers(x.copy(), comp, pend, vals)
        gf.append(np.atleast_1d(f).ravel()[0])
        gg.append(g)
    mean, noise, amp2, ls = pack_hypers(hs)
    # logprob records of the last few sampler calls (ls conditional has len D, joint has len 3)
    lp_x_ls = np.array([r[0] for r in rec if r[0].size == D and D != 3][-12:])
    lp_v_ls = np.array([r[1] for r in rec if r[0].size == D and D != 3][-12:])
    out = dict(kind=kind, noiseless=int(noiseless), seed=seed, burnin=burnin, S=S,
               grid=grid, values=values, durations=durations, candidates=candidates,
               pending=pending, complete=complete,
               hs_mean=mean, hs_noise=noise, hs_amp2=amp2, hs_ls=ls, normals=normals,
               overall_ei=overall, grad_pts=gpts, grad_f=np.array(gf), grad_g=np.array(gg),
               next_is_tuple=int(isinstance(ret, tuple)),
               next_index=int(ret[0] if isinstance(ret, tuple) else ret),
               next_point=(ret[1] if isinstance(ret, tuple) else np.zeros(0)),
               n_logprob_calls=len(rec), lp_x_ls=lp_x_ls, lp_v_ls=lp_v_ls,
               rng_key=state0[1], rng_pos=state0[2])
    np.savez_compressed(os.path.join(HERE, name + ".npz"), **out)
    print(name, "next ->", out["next_index"], out["next_is_tuple"], "max mean EI",
          overall.mean(1).max(), "logprob calls", len(rec))


def golden_logprob(name, D, N, kind, seed):
    """Joint-hyper and length-scale conditionals of the slice sampler with all state recorded."""
    grid, values, durations, candidates, pending, complete = synth(D, N, 40, 0, seed)
    comp, vals = grid[complete], values[complete]
    out = dict(kind=kind, comp=comp, vals=vals)
    for mode, noiseless in (("noisy", 0), ("noiseless", 1)):
        ch = OPT.init(tempfile.mkdtemp(), "covar=%s,mcmc_iters=2,burnin=2,noiseless=%d,"
                      "use_multiprocessing=0" % (kind, noiseless))
        ch._real_init(D, vals)
        np.random.seed(seed)
        recs = []
        orig = OPT.util.slice_sample

        def wrapped(init_x, logprob, **kw):
            state = (ch.mean, ch.noise, ch.amp2, ch.ls.copy())

            def lp(x):
                v = logprob(x)
                recs.append((np.array(x, float).copy(), float(v), state, bool(kw.get("compwise"))))
                return v
            return orig(init_x, lp, **kw)
        OPT.util.slice_sample = wrapped
        for _ in range(3):
            ch.sample_hypers(comp, vals)
        OPT.util.slice_sample = orig
        joint = [r for r in recs if not r[3]][:40]
        lsr = [r for r in recs if r[3]][:40]
        out[mode + "_joint_x"] = np.array([r[0] for r in joint])
        out[mode + "_joint_lp"] = np.array([r[1] for r in joint])
        out[mode + "_joint_ls"] = np.array([r[2][3] for r in joint])
        out[mode + "_ls_x"] = np.array([r[0] for r in lsr])
        out[mode + "_ls_lp"] = np.array([r[1] for r in lsr])
        out[mode + "_ls_state"] = np.array([[r[2][0], r[2][1], r[2][2]] for r in lsr])
    np.savez_compressed(os.path.join(HERE, name + ".npz"), **out)
    print(name, "joint", len(out["noisy_joint_lp"]), "ls", len(out["noisy_ls_lp"]))


def golden_psec(name, D, N, M, P, kind, S, seed, burnin=6, noiseless=False):
    grid, values, durations, candidates, pending, complete = synth(D, N, M, P, seed)
    ch = PSEC.init(tempfile.mkdtemp(), "covar=%s,mcmc_iters=%d,burnin=%d,grid_subset=4,noiseless=%d" % (
        kind, S, burnin, int(noiseless)))
    np.random.seed(seed)
    ret = ch.next(grid, values, durations, candidates, pending, complete)
    comp, cand, pend = grid[complete], grid[candidates], grid[pending]
    vals, durs = values[complete], np.log(durations[complete])
    hs, ths = list(ch.hyper_samples), list(ch.time_hyper_samples)
    # per-sample EI/s with explicit hypers (P=0 so no RNG involved)
    per = np.zeros((cand.shape[0], S))
    for s in range(S):
        (ch.mean, ch.noise, ch.amp2, ch.ls) = hs[s]
        (ch.time_mean, ch.time_noise, ch.time_amp2, ch.time_ls) = ths[s]
        per[:, s] = ch.compute_ei_per_s(comp, pend, cand, vals, durs)
    overall = ch.ei_over_hypers(comp, pend, cand, vals, durs)
    gpts = np.random.RandomState(seed + 5).rand(3, D)
    gf, gg = [], []
    for x in gpts:
        f, g = ch.grad_optimize_ei_over_hypers(x.copy(), comp, vals, durs, True)
        gf.append(f)
        gg.append(g)
    m, n, a, l = pack_hypers(hs)
    tm, tn, ta, tl = pack_hypers(ths)
    out = dict(kind=kind, S=S, seed=seed, burnin=burnin, noiseless=int(noiseless), grid=grid, values=values,
               durations=durations,
               candidates=candidates, pending=pending, complete=complete,
               hs_mean=m, hs_noise=n, hs_amp2=a, hs_ls=l,
               ths_mean=tm, ths_noise=tn, ths_amp2=ta, ths_ls=tl, n_time_samples=len(ths),
               per_sample_ei_per_s=per, overall_ei=overall,
               grad_pts=gpts, grad_f=np.array(gf), grad_g=np.array(gg),
               next_is_tuple=int(isinstance(ret, tuple)),
               next_index=int(ret[0] if isinstance(ret, tuple) else ret),
               next_point=(ret[1] if isinstance(ret, tuple) else np.zeros(0)))
    np.savez_compressed(os.path.join(HERE, name + ".npz"), **out)
    print(name, "next ->", out["next_index"], out["next_is_tuple"])


def golden_gpei(name, D, N, M, P, seed, noiseless=False):
    """GPEIChooser: the proposal; with ``noiseless`` also the hyper-parameters the chain ends on."""
    grid, values, durations, candidates, pending, complete = synth(D, N, M, P, seed)
    ch = GPEI.init(tempfile.mkdtemp(), "mcmc_iters=4" + (",noiseless=1" if noiseless else ""))
    np.random.seed(seed)
    ret = ch.next(grid, values, durations, candidates, pending, complete)
    out = dict(grid=grid, values=values, durations=durations, candidates=candidates, pending=pending,
               complete=complete, seed=seed, next_index=int(ret))
    if noiseless:
        out.update(noiseless=1, mean=ch.mean, noise=ch.noise, amp2=ch.amp2, ls=ch.ls)
    np.savez_compressed(os.path.join(HERE, name + ".npz"), **out)
    print(name, "next ->", int(ret))


CASES = {
    "kernels":            lambda n: golden_kernels(),
    #                                  name  D   N    M   P  kind        S noiseless seed
    "opt_branin2d":       lambda n: golden_opt(n, 2, 20, 300, 0, "Matern52", 4, False, 1),
    "opt_d8_m52":         lambda n: golden_opt(n, 8, 64, 400, 0, "Matern52", 4, True, 2),
    "opt_d8_m52_pend":    lambda n: golden_opt(n, 8, 48, 300, 3, "Matern52", 3, True, 3),
    "opt_d5_ardse":       lambda n: golden_opt(n, 5, 40, 300, 0, "ARDSE", 3, False, 4),
    "opt_d4_m32_pend":    lambda n: golden_opt(n, 4, 32, 200, 2, "Matern32", 3, False, 5),
    "opt_d3_se":          lambda n: golden_se(n, 3, 24, 200, 2, 6),
    "opt_d1_m52":         lambda n: golden_opt(n, 1, 12, 100, 1, "Matern52", 2, False, 7),
    "logprob_d6":         lambda n: golden_logprob(n, 6, 40, "Matern52", 8),
    "psec_d4":            lambda n: golden_psec(n, 4, 40, 300, 0, "Matern52", 3, 9),
    "psec_d3_pend":       lambda n: golden_psec(n, 3, 30, 200, 2, "Matern52", 2, 10),
    "psec_d3_noiseless":  lambda n: golden_psec(n, 3, 30, 200, 2, "Matern52", 2, 13, noiseless=True),
    "gpei_d3":            lambda n: golden_gpei(n, 3, 25, 200, 2, 12),
    "gpei_d3_noiseless":  lambda n: golden_gpei(n, 3, 25, 200, 2, 14, noiseless=True),
}


if __name__ == "__main__":
    for name in sys.argv[1:] or list(CASES):       # e.g. make_golden.py gpei_d3_noiseless
        CASES[name](name)
