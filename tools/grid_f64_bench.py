#!/usr/bin/env python
"""One grid pass three ways, alternated in one process: the production float32 chain, float64 with the prediction on
the SIMT kernel (smk_predict_f64, DFMA; f64_mma_min_n forced above N) and float64 with the prediction on the fp64 tensor
cores (smk_predict_mma_f64, DMMA).  Per workload and way: the median pass time over --reps, split into factorisation
(covariance + Cholesky + alpha), prediction and EI sweep; the prediction's achieved TFLOP/s from the algorithmic count
M S (N^2 + (3D + 25) N); and the largest |EI_dmma - EI_simt| / max EI per column with both argmaxes.  Then
chooser.next() wall time with grid_dtype=float64 at c2 and at the headline (steady state: burnin=0, two calls, the
second reported).  The card's name and power limit are read in the same process.

    python tools/grid_f64_bench.py [--workloads tiny,c2,c3,c4,headline,c5] [--reps 3] [--no-next]

Prints one JSON line per workload, then one for next(), then a summary line."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import bench  # noqa: E402

SUBSET_S = {"c5": 1}           # c5 with one hyper-sample


def card():
    import torch
    out = dict(name=torch.cuda.get_device_name(0))
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
        name, pl, clk = [x.strip() for x in q.split(",")]
        out.update(smi_name=name, power_limit=pl, max_sm_clock=clk)
    except Exception as e:                      # read-only query; report what is missing rather than guess
        out.update(power_limit="unavailable (%s)" % type(e).__name__)
    return out


def one_pass(eng, D, N, M, S, comp, cand, vals, hs, ths, durs, want_matrix=False):
    """One grid pass on `eng`; returns (ms, stage_ms, ei or None, argmax of the mean)."""
    import torch
    eng.timers = {}
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    ei, ei_sum, _ = eng.ei_over_hypers_device(bench.KIND, hs, comp, None, cand, vals, want_matrix=want_matrix,
                                              time_hyper_samples=ths, durs_log=durs)
    idx, _ = eng.topk(ei_sum, M, 1)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1)
    st = eng.stage_ms()
    eng.timers = None
    return ms, st, (ei[:, :M].double().cpu().numpy() if ei is not None else None), int(idx[0].item())


def split(st):
    fac = sum(v for k, v in st.items() if k in ("cov_potrf", "chol_solve", "linv_alpha"))
    return dict(factor_ms=fac, predict_ms=st.get("predict", 0.0), sweep_ms=st.get("ei_sweep", 0.0))


def workload(name, reps, backend):
    D, N, M, S = bench.WORKLOADS[name]
    S = SUBSET_S.get(name, S)
    comp, cand, vals, hs = bench.synth(D, N, M, S)
    hs = hs[:S]
    ths, durs = None, None
    if name in bench.PER_SECOND:
        durs, ths = bench.synth_time(D, comp, S)
    e32, e64 = backend.eng32, backend.eng64
    saved = e64.f64_mma_min_n
    ways = {"f32": (e32, None), "f64_simt": (e64, N + 1), "f64_dmma": (e64, 0)}
    res = {k: [] for k in ways}
    args = (D, N, M, S, comp, cand, vals, hs, ths, durs)
    try:
        for k, (eng, thr) in ways.items():          # warm-up of every shape
            if thr is not None:
                e64.f64_mma_min_n = thr
            one_pass(eng, *args)
        for _ in range(reps):
            for k, (eng, thr) in ways.items():
                if thr is not None:
                    e64.f64_mma_min_n = thr
                res[k].append(one_pass(eng, *args))
        # outputs: the two float64 predicts on the same inputs, and the oracle-free agreement of their EI
        e64.f64_mma_min_n = N + 1
        _, _, ei_s, am_s = one_pass(e64, *args, want_matrix=True)
        e64.f64_mma_min_n = 0
        _, _, ei_d, am_d = one_pass(e64, *args, want_matrix=True)
    finally:
        e64.f64_mma_min_n = saved
    flops = float(M) * S * (float(N) * N + (3.0 * D + 25.0) * N)
    out = dict(workload=name, D=D, N=N, M=M, S=S, per_second=ths is not None, predict_flops=flops,
               routed_to=e64.predict_kernel_for(N), f64_mma_min_n=saved)
    for k, runs in res.items():
        i = int(np.argsort([r[0] for r in runs])[len(runs) // 2])      # the median pass, with its own split
        ms, st, _, am = runs[i]
        sp = split(st)
        out[k] = dict(ms=ms, ms_all=[r[0] for r in runs], argmax=am,
                      predict_tflops=flops / (sp["predict_ms"] * 1e-3) / 1e12 if sp["predict_ms"] > 0 else None, **sp)
    rel = max(float(np.abs(ei_d[s] - ei_s[s]).max() / max(np.abs(ei_s[s]).max(), 1e-300)) for s in range(S))
    out["dmma_vs_simt"] = dict(max_rel_ei=rel, argmax_simt=am_s, argmax_dmma=am_d, same_argmax=am_s == am_d)
    out["dmma_speedup_predict"] = out["f64_simt"]["predict_ms"] / out["f64_dmma"]["predict_ms"]
    return out


def next_ms(name):
    import next_bench
    from spearmint_b200.backend import DeviceBackend
    D, N, M, S = bench.WORKLOADS[name]
    b = DeviceBackend(grid_dtype="float64")
    calls = next_bench.run("gpu", D, N, M, S, burnin=0, calls=2, grid_subset=20, backend=b)
    return dict(workload=name, D=D, N=N, M=M, S=S, grid_dtype="float64", ms_calls=[c["ms"] for c in calls],
                ret=[c["ret"] for c in calls], phase_ms=calls[-1]["phase_ms"])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="tiny,c2,c4,c3,headline,c5")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--no-next", action="store_true")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("grid_f64_bench: needs a CUDA device (H100, sm_90a)")
    from spearmint_b200.backend import DeviceBackend
    info = card()
    print(json.dumps(dict(card=info)), flush=True)
    backend = DeviceBackend()
    rows = []
    for w in a.workloads.split(","):
        t0 = time.perf_counter()
        r = workload(w, a.reps, backend)
        r["wall_s"] = time.perf_counter() - t0
        rows.append(r)
        print(json.dumps(r), flush=True)
    for e in (backend.eng32, backend.eng64):           # next() builds its own backend: give the pooled buffers back
        e.trim()
    del backend
    import gc
    gc.collect()
    torch.cuda.empty_cache()
    if not a.no_next:
        for w in ("c2", "headline"):
            print(json.dumps(dict(next=next_ms(w))), flush=True)
    print(json.dumps(dict(summary=[dict(workload=r["workload"], N=r["N"], routed_to=r["routed_to"],
                                        f32_ms=r["f32"]["ms"], simt_ms=r["f64_simt"]["ms"], dmma_ms=r["f64_dmma"]["ms"],
                                        simt_predict_tflops=r["f64_simt"]["predict_tflops"],
                                        dmma_predict_tflops=r["f64_dmma"]["predict_tflops"],
                                        dmma_vs_simt_max_rel_ei=r["dmma_vs_simt"]["max_rel_ei"])
                                   for r in rows], card=info)), flush=True)


if __name__ == "__main__":
    main()
