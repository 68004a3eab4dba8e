#!/usr/bin/env python
"""Generates tests/golden/oracle_vs_reference.npz by EXECUTING the reference (through oracle/ref_shim.py) on the inputs
of tests/test_oracle_vs_reference.py: kernel matrices and log-probabilities for the four covariance kinds, compute_ei
with and without pending points (the fantasy normals the reference drew are stored), a Sobol block, and the ML-II
optimum of GP.optimize_hypers.  Every input is stored next to the output it produced.

Run where the reference tree exists (SPEARMINT_REFERENCE, see oracle/ref_shim.py):
    python tests/golden/make_golden_oracle_vs_reference.py
"""
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle import ref_shim  # noqa: E402

KINDS = ["SE", "ARDSE", "Matern32", "Matern52"]


def problem(seed, D=3, N=25, M=40):
    rs = np.random.RandomState(seed)
    comp, cand = rs.rand(N, D), rs.rand(M, D)
    y = np.sin(3 * comp).sum(1) + 0.05 * rs.randn(N)
    return comp, cand, (y - y.mean()) / y.std(), rs


def main():
    R = ref_shim.load()
    gp, OPT, sb = R["gp"], R["OPT"], R["sobol_lib"]
    out = {}

    comp, cand, vals, rs = problem(1)
    ls = rs.uniform(0.4, 1.8, comp.shape[1])
    out.update(k_comp=comp, k_cand=cand, k_vals=vals, k_ls=ls, k_mean=0.1, k_noise=2e-3, k_amp2=1.3)
    for kind in KINDS:
        f = getattr(gp, kind)
        g = gp.GP(kind)
        g.real_init(comp.shape[1], vals)
        g.ls, g.amp2, g.noise, g.mean = ls, 1.3, 2e-3, 0.1
        out["K_%s" % kind] = f(ls, comp)
        out["Kx_%s" % kind] = f(ls, comp, cand)
        out["logprob_%s" % kind] = np.float64(g.logprob(comp, vals))

    comp, cand, vals, rs = problem(2)
    with tempfile.TemporaryDirectory() as d:
        ch = OPT.init(d, "mcmc_iters=2,burnin=1,use_multiprocessing=0")
        ch.D = comp.shape[1]
        ch.randomstate = np.random.get_state()
        ch.mean, ch.noise, ch.amp2, ch.ls = 0.05, 1e-3, 0.9, rs.uniform(0.4, 1.8, ch.D)
        out.update(ei_comp=comp, ei_cand=cand, ei_vals=vals, ei_hyper=np.array([ch.mean, ch.noise, ch.amp2]), ei_ls=ch.ls)
        out["ei_nopend"] = ch.compute_ei(comp, np.zeros((0, ch.D)), cand, vals)
        pend = rs.rand(2, ch.D)
        np.random.set_state(ch.randomstate)
        out["ei_normals"] = np.random.randn(2, ch.pending_samples)     # what compute_ei draws after the same set_state
        out["ei_pend"] = pend
        out["ei_withpend"] = ch.compute_ei(comp, pend, cand, vals)

    out["sobol_6_50_2"] = sb.i4_sobol_generate(6, 50, 2)

    comp, cand, vals, rs = problem(3, D=2, N=20)
    g = gp.GP("Matern52")
    g.real_init(2, vals)
    g.optimize_hypers(comp, vals)
    out.update(ml_comp=comp, ml_vals=vals, ml_hyper=np.array([g.mean, g.noise, g.amp2]), ml_ls=np.asarray(g.ls))

    np.savez_compressed(os.path.join(HERE, "oracle_vs_reference.npz"), **out)


if __name__ == "__main__":
    main()
