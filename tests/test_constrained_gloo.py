"""CPU, world_size 2 over gloo: DeviceBackend.constrained_ei_matrix shards (objective, constraint) sample PAIRS over
ranks, with their per-sample fantasy normals, and reassembles the reference's constrained EI matrix
(tests/golden/cons_nan_pend_d3.npz: violations as NaN, pending points).  The per-rank compute is a stand-in engine that
evaluates the oracle on the host: this covers the sharding and exchange logic of the backend only."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASE = os.path.join(ROOT, "tests", "golden", "cons_nan_pend_d3.npz")


class _OracleEngine(object):
    device = torch.device("cpu")

    def __init__(self):
        self.pairs = []

    def constrained_ei_over_hypers_device(self, kind, hs, chs, ff, comp, labels, pend, cand, vals, normals=None):
        from tests import constrained_oracle as CO
        self.pairs.append((len(hs), None if normals is None else normals.shape))
        M = cand.shape[0]
        ei = CO.ei_over_hypers(kind, hs, chs, ff, comp, labels, pend, cand, vals, normals)
        out = torch.zeros((len(hs), (M + 127) // 128 * 128), dtype=torch.float64)
        out[:, :M] = torch.from_numpy(ei.T)
        return out, out.sum(0), M

    def tail_fix(self, *args, **kw):
        return False


def _worker(rank, world, port, out):
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from spearmint_b200.backend import DeviceBackend
    from tests.test_constrained_oracle import load_case
    z, hs, chs, normals = load_case(CASE)
    be = object.__new__(DeviceBackend)
    be.eng32 = _OracleEngine()
    ei = be.constrained_ei_matrix(str(z["kind"]), hs, chs, z["ff"], z["comp"], z["labels"], z["pend"], z["cand"],
                                  z["vals"], normals)
    np.save(out + ".%d.npy" % rank, ei)
    with open(out + ".%d.txt" % rank, "w") as fh:
        fh.write(repr(be.eng32.pairs))
    dist.barrier()
    dist.destroy_process_group()


def test_sharded_constrained_pass_reassembles_the_reference_matrix(tmp_path):
    out = str(tmp_path / "cons")
    mp.spawn(_worker, args=(2, 29541, out), nprocs=2, join=True)
    z = np.load(CASE)
    S, P, F = z["gain"].shape[0], z["pend"].shape[0], int(z["F"])
    assert S == 3 and P > 0
    for rank in (0, 1):
        np.testing.assert_allclose(np.load(out + ".%d.npy" % rank), z["ei"], rtol=1e-9, atol=1e-15)
    # rank 0 owns samples 0 and 2, rank 1 sample 1, each with its own fantasy block
    assert eval(open(out + ".0.txt").read()) == [(2, (2, P, F))]
    assert eval(open(out + ".1.txt").read()) == [(1, (1, P, F))]
