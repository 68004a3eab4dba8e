"""Runs the tensor-core predict of one test problem in a process of its own and writes mu, var, mu_f (and, for a
single-chunk call, the beta dump) to an .npz file.

    python -m tests.predict_child OUT.npz N=... kind=... D=... noise=... S=... M=... F=... seed=...

SMK_TC_OVERLAP and SMK_KXT_IMPL are read once per process (function-level statics of the library), so the tests of
those switches run the call here, with the switch in the environment, and compare the result with the parent's.
The problem is built by the same helpers as in tests/test_gpu_predict.py from the same seeds."""
import os
import sys

import numpy as np


def main(argv):
    import torch
    from spearmint_b200.engine import GPEIEngine
    from tests.test_gpu_predict import _alpha_f, _cands, _predict_tc, _setup
    out = argv[0]
    kw = dict(a.split("=", 1) for a in argv[1:])
    N, D, S, M, F, seed = (int(kw[k]) for k in ("N", "D", "S", "M", "F", "seed"))
    engs = {"f32": GPEIEngine(dtype=torch.float32)}
    P = _setup(engs, "tc", kw["kind"], N, D, float(kw["noise"]), S, seed=seed)
    _, Cd = _cands(P, M, seed=seed + 1)
    af_dev, _ = _alpha_f(P, F, seed=seed + 2)
    r = _predict_tc(P, Cd, F=F, alpha_f=af_dev, dbg=not os.environ.get("SMK_TC_BUDGET_MB"))
    torch.cuda.synchronize()
    np.savez(out, **r)


if __name__ == "__main__":
    main(sys.argv[1:])
