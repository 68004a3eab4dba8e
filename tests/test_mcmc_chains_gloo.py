"""CPU, world_size 2 over gloo: mcmc_chains=4 with chain c on rank c mod 2 gives every rank the hyper_samples, state
pickle and global RNG state of a single-process run; a non positive definite item in one rank's chain raises on both
ranks and the collectives stay aligned.  The log-likelihood is the oracle's."""
import os
import pickle
import sys

import numpy as np
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
K = 4


def _run(d, fail_after=None):
    """next() of GPEIOptChooserB200 with mcmc_chains=K on opt_d8_m52 -> (hyper_samples, pickle, RNG state)."""
    from spearmint_b200.chooser import GPEIOptChooserB200 as mod
    import spearmint_b200.chains as chains
    import spearmint_b200.locker as lk
    from tests.helpers import load
    from tests.oracle_backend import OracleBackend
    mod.log = lk.log = chains.log = lambda *a: None

    class ChainOracle(OracleBackend):
        def __init__(self):
            OracleBackend.__init__(self, batched=True)

        def loglik(self, kind, comp, vals, chains=1):
            inner = OracleBackend.loglik(self, kind, comp, vals)
            outer = self

            class Failing(object):
                def batch(self, items):
                    out = inner.batch(items)
                    if fail_after is not None and outer.batches > fail_after:
                        out[:] = np.nan
                    return out
            return Failing()

    g = load("opt_d8_m52")
    ch = mod.init(d, "covar=%s,mcmc_iters=8,burnin=3,noiseless=%d,grid_subset=3,mcmc_chains=%d" % (
        str(g["kind"]), int(g["noiseless"]), K))
    ch._backend = ChainOracle()
    np.random.seed(7)
    ch.next(g["grid"], g["values"], g["durations"], g["candidates"], g["pending"], g["complete"])
    with open(ch.state_pkl, "rb") as fh:
        st = fh.read()
    return [np.hstack(h) for h in ch.hyper_samples], st, np.random.get_state()


def _worker(rank, world, port, out, d):
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    res = _run(os.path.join(d, str(rank)))
    with open(out + ".%d" % rank, "wb") as fh:
        pickle.dump(res, fh)
    dist.barrier()
    dist.destroy_process_group()


def test_chains_over_two_ranks_match_one_process(tmp_path):
    for r in range(2):
        os.makedirs(str(tmp_path / str(r)))
    os.makedirs(str(tmp_path / "one"))
    out = str(tmp_path / "res")
    mp.spawn(_worker, args=(2, 29541, out, str(tmp_path)), nprocs=2, join=True)
    hs1, st1, rng1 = _run(str(tmp_path / "one"))
    for r in range(2):
        with open(out + ".%d" % r, "rb") as fh:
            hs, st, rng = pickle.load(fh)
        assert len(hs) == len(hs1) == 8
        for a, b in zip(hs, hs1):
            np.testing.assert_array_equal(a, b)
        p, p1 = pickle.loads(st), pickle.loads(st1)
        assert sorted(p) == sorted(p1)
        assert len(p["chains"]) == K
        for c, c1 in zip(p["chains"], p1["chains"]):
            np.testing.assert_array_equal(np.hstack(c[:4]), np.hstack(c1[:4]))
            assert np.array_equal(c[4][1], c1[4][1]) and c[4][2:] == c1[4][2:]
        np.testing.assert_array_equal(np.hstack([p["mean"], p["noise"], p["amp2"], p["ls"]]),
                                      np.hstack([p1["mean"], p1["noise"], p1["amp2"], p1["ls"]]))
        assert np.array_equal(rng[1], rng1[1]) and rng[2:] == rng1[2:]


def _worker_err(rank, world, port, out, d):
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from spearmint_b200 import parallel
    res = []
    try:                                       # rank 1's chains (1 and 3) meet a non positive definite matrix
        _run(os.path.join(d, str(rank)), fail_after=5 if rank == 1 else None)
        res.append("no-raise")
    except np.linalg.LinAlgError as e:
        res.append("raised:" + str(e))
    t = torch.ones(3)                          # and the next collective still lines up
    parallel.allreduce_sum_(t)
    res.append(float(t[0]))
    with open(out + ".%d" % rank, "w") as fh:
        fh.write(repr(res))
    dist.barrier()
    dist.destroy_process_group()


def test_non_pd_in_one_ranks_chain_raises_on_both(tmp_path):
    for r in range(2):
        os.makedirs(str(tmp_path / str(r)))
    out = str(tmp_path / "err")
    mp.spawn(_worker_err, args=(2, 29543, out, str(tmp_path)), nprocs=2, join=True)
    r0, r1 = eval(open(out + ".0").read()), eval(open(out + ".1").read())
    assert r0[0].startswith("raised:") and "another rank" in r0[0]
    assert r1[0].startswith("raised:") and "not positive definite" in r1[0] and "another rank" not in r1[0]
    assert r0[1] == 2.0 and r1[1] == 2.0
