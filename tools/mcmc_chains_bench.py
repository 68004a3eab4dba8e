#!/usr/bin/env python
"""Wall time of next()'s hyper-parameter MCMC (stats["phase_ms"]["mcmc"] of the SECOND call: no burn-in) of
GPEIOptChooserB200 with mcmc_chains = K, one JSON line per (shape, K), plus the card and its power limit.

    python tools/mcmc_chains_bench.py [--shapes 8x100x8,8x512x8,32x4096x40] [--chains 1,2,4,8] [--runs 3]
    torchrun --nproc-per-node W tools/mcmc_chains_bench.py --chains W        (chain c on rank c mod W)

Shapes are DxNxS (S = mcmc_iters, a multiple of every K).  The problem is tools/next_bench.problem (the smooth test
function of bench.py's workloads) with 2000 candidates; burnin=2 keeps the first call short (its time is not reported).
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from next_bench import problem  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True).stdout.strip().splitlines()
        return q[torch.cuda.current_device()] if q else None
    except OSError:
        return None


def mcmc_ms(D, N, S, K, runs, M=2000):
    from spearmint_b200.chooser import GPEIOptChooserB200 as mod
    import spearmint_b200.chains as chains
    import spearmint_b200.locker as lk
    mod.log = lk.log = chains.log = lambda *a: None
    grid, values, candidates, complete = problem(D, N, M)
    out = []
    for r in range(runs):
        ch = mod.init(tempfile.mkdtemp(), "mcmc_iters=%d,burnin=2,noiseless=1,grid_subset=5,mcmc_chains=%d" % (S, K))
        np.random.seed(r)
        for call in range(2):
            ch.next(grid, values, None, candidates, np.array([], dtype=int), complete)
        out.append(dict(ms=ch.stats["phase_ms"]["mcmc"], loglik_evals=ch.stats.get("loglik_evals"),
                        loglik_batches=ch.stats.get("loglik_batches"), rounds=ch.stats.get("chain_rounds")))
    return out


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="8x100x8,8x512x8,32x4096x40")
    ap.add_argument("--chains", default="1,2,4,8")
    ap.add_argument("--runs", type=int, default=3)
    a = ap.parse_args()
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if world > 1:
        local = int(os.environ["LOCAL_RANK"])
        torch.cuda.set_device(local)
        dist.init_process_group("nccl", device_id=torch.device("cuda:%d" % local))
    rank = dist.get_rank() if world > 1 else 0
    for shape in a.shapes.split(","):
        D, N, S = (int(v) for v in shape.split("x"))
        for K in (int(k) for k in a.chains.split(",")):
            res = mcmc_ms(D, N, S, K, a.runs)
            ms = sorted(r["ms"] for r in res)
            if rank == 0:
                print(json.dumps(dict(D=D, N=N, S=S, K=K, world=world, runs=a.runs, mcmc_ms_median=ms[len(ms) // 2],
                                      mcmc_ms=ms, card=card(), detail=res)), flush=True)
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()
