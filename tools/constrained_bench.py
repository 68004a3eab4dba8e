#!/usr/bin/env python
"""Constrained-EI grid pass (CONS:450-468, 806-940) at the headline shape: D=32, N=4096 complete observations of which
about 10 % violate the constraint, M=100k candidates, S=40 sample pairs.  Prints one JSON line per repetition with the
wall time of a pass (device synchronised), candidates/s and the CUDA-event split:

    objective   cov_potrf + linv_alpha | chol_solve + predict   (the plain pass on the feasible points)
    constraint_factor                  float64 factor of the classification GP over all points + t_alpha = K_c^-1 ff
    constraint_prob                    the probability kernel (csrc/constraint.cu)
    ei_sweep                           the probability-weighted sweep

and, at the same shape, the plain grid pass over the feasible points for comparison.  ``--next W`` instead times
GPConstrainedEIChooserB200.next() at workload W (default c2: D=8, N=512, M=10k, S=10), steady state (burnin=0,
grid_subset=20), calls after a warm-up call.  The card's name, power limit and SM clock limit
are read in the same run.

    python tools/constrained_bench.py [--reps R] [--workload headline|c2|c3] [--next c2]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from spearmint_b200.engine import GPEIEngine  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:           # the numbers below are still device-timed; the card is then unnamed
        q = "nvidia-smi unavailable (%s)" % e
    return q


def problem(D, N, M, S):
    comp, cand, vals, hs = bench.synth(D, N, M, S)
    rs = np.random.RandomState(7)
    # the feasible region is a half-space; about 10 % of the observations fall outside it
    w = rs.randn(D)
    proj = comp.dot(w)
    bad = proj > np.quantile(proj, 0.9)
    vals = vals.copy()
    vals[bad] = np.inf
    labels = (~bad).astype(float)
    chs = [(0.0, rs.uniform(0.5, 3.0), float(np.exp(0.25 * rs.randn())), rs.uniform(0.3, 2.0, D)) for _ in range(S)]
    ff = np.where(bad, -1.0, 1.0) + 0.3 * rs.randn(N)
    return comp, cand, vals, labels, hs, chs, ff


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--workload", default="headline")
    ap.add_argument("--next", default=None, metavar="WORKLOAD", help="time next() of the plugin at this workload")
    a = ap.parse_args()
    if a.next:
        return bench_next(a.next, a.reps)
    D, N, M, S = bench.WORKLOADS[a.workload]
    comp, cand, vals, labels, hs, chs, ff = problem(D, N, M, S)
    pend = np.zeros((0, D))
    eng = GPEIEngine(dtype=torch.float32)
    info = dict(workload=a.workload, D=D, N=N, N_good=int(labels.sum()), M=M, S=S, card=card())
    args = ("Matern52", hs, chs, ff, comp, labels, pend, cand, vals)
    eng.constrained_ei_over_hypers_device(*args)          # warm-up: modules, buffers, the float64 helper engine
    eng.ei_over_hypers_device("Matern52", hs, comp[labels > 0], pend, cand, vals[labels > 0], want_matrix=False)
    torch.cuda.synchronize()
    for r in range(a.reps):
        eng.timers = {}
        t0 = time.perf_counter()
        _, ei_sum, _ = eng.constrained_ei_over_hypers_device(*args)
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        st = eng.stage_ms()
        eng.timers = None
        obj = sum(st.get(k, 0.0) for k in ("cov_potrf", "linv_alpha", "chol_solve", "predict"))
        t1 = time.perf_counter()
        eng.ei_over_hypers_device("Matern52", hs, comp[labels > 0], pend, cand, vals[labels > 0], want_matrix=False)
        torch.cuda.synchronize()
        plain = time.perf_counter() - t1
        print(json.dumps(dict(info, rep=r, ms=1e3 * dt, cand_per_s=M / dt, objective_ms=obj,
                              constraint_factor_ms=st.get("constraint_factor", 0.0),
                              constraint_prob_ms=st.get("constraint_prob", 0.0), ei_sweep_ms=st.get("ei_sweep", 0.0),
                              plain_pass_ms=1e3 * plain, argmax=int(torch.argmax(ei_sum[:M])))), flush=True)


def bench_next(workload, reps):
    import tempfile
    import numpy.random as npr
    from spearmint_b200.chooser import GPConstrainedEIChooserB200 as CB
    D, N, M, S = bench.WORKLOADS[workload]
    comp, cand, vals, labels, _, _, _ = problem(D, N, M, S)
    grid = np.vstack([comp, cand])
    values = np.r_[vals, np.zeros(M)]
    complete, candidates, pending = np.arange(N), np.arange(N, N + M), np.array([], dtype=int)
    with tempfile.TemporaryDirectory() as d:
        ch = CB.init(d, "mcmc_iters=%d,burnin=0,grid_subset=20" % S)
        npr.seed(0)
        for r in range(reps + 1):                  # call 0 warms up modules and buffers
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            ret = ch.next(grid, values, np.zeros(N + M), candidates, pending, complete)
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            if r:
                print(json.dumps(dict(workload=workload, D=D, N=N, N_good=int(labels.sum()), M=M, S=S, card=card(),
                                      rep=r, next_ms=1e3 * dt, proposal=ret if np.isscalar(ret) else int(ret[0]))),
                      flush=True)


if __name__ == "__main__":
    main()
