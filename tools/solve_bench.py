#!/usr/bin/env python
"""Timing of the triangular solve: the shared-memory kernel (smk_chol_solve_*, below the limit) against the global-memory
one (smk_chol_solve_gm_*, any size) at one N both run, the global-memory solve above the limit, and optionally one
GPEIOptChooserB200.next() above the limit with its phase split.  CUDA events around R back-to-back calls after a warm-up;
the card's name and power limit are read in the same process.  One JSON line per measurement.

Usage: python tools/solve_bench.py [--next]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:           # the timing does not depend on it; say so in the record
        q = "unknown (%s)" % e
    return q


def factor(eng, N, S, seed=0):
    import torch
    from spearmint_b200.engine import check, fn, ptr
    from tests.helpers import cov_inputs, cur_stream, data, synth_hypers
    X, y, rs = data(N, 8, seed)
    hb = eng.hypers(synth_hypers(rs, S, 8, 1e-2), "Matern52")
    Npad = (N + 127) // 128 * 128
    A = cov_inputs(eng, "Matern52", X, hb, Npad)
    winv = torch.empty((S, Npad // eng.NB, eng.NB, eng.NB), dtype=eng.dtype, device=eng.device)
    info = torch.empty((S,), dtype=torch.int32, device=eng.device)
    check(fn("smk_potrf_lower_batched", eng.dtype)(Npad, S, ptr(A), ptr(winv), ptr(info), cur_stream()), "potrf")
    return A, winv, hb, y


def time_solve(eng, entry, A, winv, hb, N, F, reps):
    import torch
    from spearmint_b200.engine import check, fn, ptr
    from tests.helpers import cur_stream
    S, Npad = A.shape[0], A.shape[-1]
    rs = np.random.RandomState(1)
    y = eng.to_dev(rs.randn(F, N))
    alpha = torch.empty((S, F, Npad), dtype=eng.dtype, device=eng.device)
    f = fn(entry, eng.dtype)

    def call():
        check(f(N, Npad, S, F, ptr(A), ptr(winv), ptr(y), 0, N, ptr(hb.mean), ptr(alpha), None, None, cur_stream()),
              entry)
    call()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        call()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps, alpha


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--next", action="store_true", help="also time one GPEIOptChooserB200.next() at N = 16384")
    ap.add_argument("--next-dims", type=int, default=8)
    ap.add_argument("--next-only", action="store_true")
    a = ap.parse_args()
    import torch
    from spearmint_b200.engine import GPEIEngine
    dev = card()
    print(json.dumps({"card": dev}), flush=True)
    for prec, dt in (() if a.next_only else (("f32", torch.float32), ("f64", torch.float64))):
        eng = GPEIEngine(dtype=dt)
        for N, S in ((8192, 1), (8192, 40)):
            A, winv, hb, _ = factor(eng, N, S)
            for F in (1, 100):
                reps = 5 if S * F >= 1000 else 20
                t_old, a_old = time_solve(eng, "smk_chol_solve", A, winv, hb, N, F, reps)
                t_new, a_new = time_solve(eng, "smk_chol_solve_gm", A, winv, hb, N, F, reps)
                rel = float(((a_new - a_old).abs().max() / a_old.abs().max()).item())
                print(json.dumps(dict(prec=prec, N=N, S=S, F=F, old_ms=round(t_old, 3), gm_ms=round(t_new, 3),
                                      max_rel_diff=rel, card=dev)), flush=True)
            del A, winv
            torch.cuda.empty_cache()
        for N, S, F in ((16384, 1, 1), (16384, 10, 1), (16384, 1, 100)):
            A, winv, hb, _ = factor(eng, N, S)
            t_new, _ = time_solve(eng, "smk_chol_solve", A, winv, hb, N, F, 5)
            print(json.dumps(dict(prec=prec, N=N, S=S, F=F, gm_ms=round(t_new, 3), card=dev)), flush=True)
            del A, winv
            torch.cuda.empty_cache()
    if a.next:
        sys.path.insert(0, os.path.join(ROOT, "tools"))
        import next_bench
        out = next_bench.run("gpu", a.next_dims, 16384, 10000, 10, 0, 1, 20)
        print(json.dumps(dict(next=out, D=a.next_dims, N=16384, M=10000, S=10, burnin=0, card=dev)), flush=True)


if __name__ == "__main__":
    main()
