"""Random-forest EI on the GPU against the reference's CPU path (scikit-learn fit + per-tree predict, one thread).

    python tools/rf_bench.py [--out rf_bench.json] [--reps 3]

For (N, D, M) in (512, 8, 20 000) and (4096, 32, 100 000), T = 50 trees on Sobol inputs: the device fit
(smk_forest_fit_f64, host-to-device copies included), predict + EI (smk_forest_predict_ei_f64 + device argmax) and a
whole RandomForestEIChooserB200.next() are timed with CUDA events (median of --reps after one warm-up); the CPU column
is sklearn's RandomForestRegressor(n_jobs=1).fit and the reference's per-tree predict + mean / var + EI on the same
inputs and draws.  The outputs are compared: trees node for node, mean / var / EI, argmax.  The card's name and power
limit are read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import numpy.random as npr
import scipy.stats as sps
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import sobol_oracle  # noqa: E402
from spearmint_b200.backend import DeviceBackend  # noqa: E402
from spearmint_b200.chooser.RandomForestEIChooserB200 import RandomForestEIChooserB200  # noqa: E402
from spearmint_b200.forest import draws  # noqa: E402

SHAPES = ((512, 8, 20000), (4096, 32, 100000))
T = 50


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:                     # the name from torch at least
        q = "%s, power limit unknown (%s)" % (torch.cuda.get_device_name(), e)
    return q


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return float(np.median(ts)), ts


def run_shape(be, N, D, M, reps):
    G = sobol_oracle.i4_sobol_generate(D, N + M, 1).T.copy()
    X, C = G[:N], G[N:]
    y = np.sum((X - 0.37) ** 2, axis=1) + 0.3 * np.sin(7 * X[:, 0]) * np.cos(3 * X[:, -1])
    best = float(y.min())
    npr.seed(0)
    w, s = draws(T, N)
    res = {"N": N, "D": D, "M": M, "T": T}
    holder = {}

    def fit():
        holder["f"] = be.forest_fit(X, y, w, s, D)
    res["fit_ms"], res["fit_ms_all"] = timed(fit, reps)
    forest = holder["f"]
    counts = forest.node_count.cpu().numpy()
    res["nodes_per_tree_mean"] = float(counts.mean())
    res["fit_us_per_node"] = 1000.0 * res["fit_ms"] / float(counts.max())

    def pred():
        holder["i"] = be.forest_argmax_ei(forest, C, best)
    res["predict_ei_ms"], res["predict_ei_ms_all"] = timed(pred, reps)

    grid = G
    vals = np.concatenate([y, np.zeros(M)])
    ch = RandomForestEIChooserB200(backend=be)

    def nxt():
        holder["p"] = ch.next(grid, vals, None, np.arange(N, N + M), np.arange(0), np.arange(N))
    res["next_ms"], res["next_ms_all"] = timed(nxt, reps)

    # CPU path of the reference: sklearn fit + per-tree predict on one thread, the same draws
    try:
        from sklearn.ensemble import RandomForestRegressor
    except ImportError:
        res["cpu"] = "sklearn not installed: not measured"
        return res
    npr.seed(0)
    rf = RandomForestRegressor(n_estimators=T, max_features=1.0, n_jobs=1)
    t0 = time.perf_counter()
    rf.fit(X, y)
    res["cpu_fit_s"] = time.perf_counter() - t0
    t0 = time.perf_counter()
    allp = [e.predict(C) for e in rf.estimators_]
    m = sum(allp) / T
    v = np.var(allp, axis=0, ddof=1)
    sd = np.sqrt(v) + 0.0001
    u = (best - m) / sd
    ei = sd * (u * sps.norm.cdf(u) + sps.norm.pdf(u))
    res["cpu_predict_ei_s"] = time.perf_counter() - t0
    res["cpu_threads"] = 1
    out = forest.predict(C, best)
    dm, dv, de = (out[k].cpu().numpy() for k in ("mean", "var", "ei"))
    same = 0
    for t, est in enumerate(rf.estimators_):
        d, tr = forest.tree(t), est.tree_
        same += int(np.array_equal(d["feature"], tr.feature) and np.array_equal(d["left"], tr.children_left)
                    and np.array_equal(d["right"], tr.children_right) and np.array_equal(d["threshold"], tr.threshold))
    res["trees_structurally_equal"] = "%d/%d" % (same, T)
    res["max_rel_dmean"] = float(np.abs(dm - m).max() / np.abs(m).max())
    res["max_rel_dvar"] = float(np.abs(dv - v).max() / v.max())
    res["max_rel_dei"] = float(np.abs(de - ei).max() / ei.max())
    res["argmax_equal"] = bool(int(holder["i"]) == int(np.argmax(ei)))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("rf_bench needs a CUDA device")
    be = DeviceBackend()
    out = {"card": card(), "shapes": [run_shape(be, N, D, M, a.reps) for N, D, M in SHAPES]}
    txt = json.dumps(out, indent=1)
    print(txt)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write(txt)


if __name__ == "__main__":
    main()
