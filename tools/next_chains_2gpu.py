#!/usr/bin/env python
"""torchrun --nproc-per-node 2 tools/next_chains_2gpu.py : next() with mcmc_chains=4 (chains 0, 2 on rank 0, chains 1, 3
on rank 1, exchanged in one all-gather) must give every rank the proposal and hyper-samples of a single-GPU run with the
same K.  Each rank makes that single-GPU run on its own device before the process group exists."""
import os
import sys
import tempfile

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests.helpers import load  # noqa: E402

CASES = ("opt_d8_m52", "opt_d8_m52_pend", "opt_d5_ardse", "opt_branin2d")


def run_all():
    from spearmint_b200.backend import DeviceBackend
    from spearmint_b200.chooser import GPEIOptChooserB200 as mod
    out = {}
    for name in CASES:
        g = load(name)
        ch = mod.init(tempfile.mkdtemp(), "covar=%s,mcmc_iters=8,burnin=%d,noiseless=%d,grid_subset=5,mcmc_chains=4" % (
            str(g["kind"]), int(g["burnin"]), int(g["noiseless"])))
        ch._backend = DeviceBackend()
        np.random.seed(int(g["seed"]))
        ret = ch.next(g["grid"], g["values"], g["durations"], g["candidates"], g["pending"], g["complete"])
        pt = ret[1] if isinstance(ret, tuple) else g["grid"][ret]
        out[name] = (pt, np.vstack([np.hstack(h) for h in ch.hyper_samples]), np.random.get_state()[1].copy())
    return out


if __name__ == "__main__":
    rank, local = int(os.environ["RANK"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    import spearmint_b200.chains as chains
    import spearmint_b200.locker as lk
    from spearmint_b200.chooser import GPEIOptChooserB200 as mod
    mod.log = lk.log = chains.log = lambda *a: None
    single = run_all()
    dist.init_process_group("nccl", device_id=torch.device("cuda:%d" % local))
    multi = run_all()
    ok = True
    for name in CASES:
        (p1, h1, s1), (p2, h2, s2) = single[name], multi[name]
        # samples and RNG bitwise; the proposal within the grid pass's cross-rank summation order (tools/next_2gpu.py)
        good = float(np.abs(p1 - p2).max()) < 2e-4 and np.array_equal(h1, h2) and np.array_equal(s1, s2)
        ok = ok and good
        print("rank %d %s: proposal |d| %.1e, samples |d| %.1e, RNG %s: %s" % (
            rank, name, float(np.abs(p1 - p2).max()), float(np.abs(h1 - h2).max()),
            "same" if np.array_equal(s1, s2) else "differs", "OK" if good else "MISMATCH"))
    dist.barrier()
    dist.destroy_process_group()
    sys.exit(0 if ok else 1)
