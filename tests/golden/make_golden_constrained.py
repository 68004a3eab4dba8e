"""Freezes the reference's constrained chooser into tests/golden/cons_*.npz.

    python tests/golden/make_golden_constrained.py

Runs chooser/GPConstrainedEIChooser.py (CONS) through oracle/ref_shim.py's py2->py3 rewrites.
  * cons_<case>.npz: with injected sample state (objective and constraint hyper-samples, the latent ff),
    ``ei_over_hypers`` (CONS:450-468) and ``pred_constraint_voilation`` (CONS:425-447) per constraint sample; the seed of
    the global RNG the pending fantasies are drawn from (CONS:910).
  * cons_next_<case>.npz: whole ``next()`` calls from a seeded global RNG, with multiprocessing.Pool replaced by a
    serial stand-in that saves and restores the RNG around each task (as the fork does): the proposal, both sample
    chains, ff_samples, the pickle, stdout and the RNG state afterwards; one case makes a second call after one more
    observation.
"""
import os
import pickle
import re
import sys
import tempfile
import types

import numpy as np
import numpy.random as npr

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from oracle import ref_shim  # noqa: E402

# name: (kind, D, N, M, S, P, F, violation, bad_fraction, seed)
CASES = {
    "cons_inf_d2": ("Matern52", 2, 30, 400, 3, 0, 0, "inf", 0.25, 11),
    "cons_nan_pend_d3": ("Matern52", 3, 40, 500, 3, 3, 5, "nan", 0.2, 12),
    "cons_vanilla": ("Matern52", 2, 24, 300, 3, 0, 0, "none", 0.0, 13),
    "cons_m32_badval": ("Matern32", 4, 50, 600, 4, 0, 0, "value", 0.3, 14),
}
BAD_VALUE = 99.0

# A py2 print statement whose format arguments continue on the following lines (CONS:301-306):
#     print 'Predicting ...' % (
#     a, b, c)
_PRINT2_RE = re.compile(r"^(\s*)print\s+('[^'\n]*'\s*%\s*\((?:\n[^\n]*?)+?\))[ \t]*$", re.M)


def load_constrained():
    """ref_shim.load() plus the CONS module.  CONS imports matplotlib for its optional 2-D plots (stubbed: never used
    here) and holds two print statements spanning several lines, which are joined into print(...) calls before the
    shim's common rewrites."""
    mods = ref_shim.load()
    if "matplotlib" not in sys.modules:
        mpl = types.ModuleType("matplotlib")
        mpl.pyplot = types.ModuleType("matplotlib.pyplot")
        sys.modules["matplotlib"], sys.modules["matplotlib.pyplot"] = mpl, mpl.pyplot
    path = os.path.join(ref_shim.REF_PKG, "chooser", "GPConstrainedEIChooser.py")
    with open(path, "r") as fh:
        src = ref_shim._py3(_PRINT2_RE.sub(lambda m: "%sprint(%s)" % (m.group(1), m.group(2)), fh.read()))
    mod = types.ModuleType("chooser.GPConstrainedEIChooser")
    mod.__file__ = path
    sys.modules[mod.__name__] = mod
    exec(compile(src, path, "exec"), mod.__dict__)
    return dict(mods, CONS=mod)


def branin(x):
    a, b = 15 * x[:, 0] - 5, 15 * x[:, 1]
    return (b - 5.1 / (4 * np.pi ** 2) * a ** 2 + 5 / np.pi * a - 6) ** 2 + 10 * (1 - 1 / (8 * np.pi)) * np.cos(a) + 10


def make_case(name, kind, D, N, M, S, P, F, violation, bad_fraction, seed):
    rs = np.random.RandomState(seed)
    comp, cand = rs.rand(N, D), rs.rand(M, D)
    pend = rs.rand(P, D)
    y = branin(comp[:, :2])
    y = (y - y.mean()) / y.std()
    bad = np.zeros(N, bool)
    if violation != "none":
        bad[rs.permutation(N)[:int(round(bad_fraction * N))]] = True
    vals = y.copy()
    vals[bad] = {"inf": np.inf, "nan": np.nan, "value": BAD_VALUE}.get(violation, 0.0)
    bad_value = BAD_VALUE if violation == "value" else np.inf
    hyper = dict(mean=0.1 * rs.randn(S), noise=rs.uniform(1e-3, 1e-2, S), amp2=rs.uniform(0.5, 2.0, S),
                 ls=rs.uniform(0.3, 1.5, (S, D)))
    chyper = dict(cmean=0.1 * rs.randn(S), gain=rs.uniform(0.5, 3.0, S), camp2=rs.uniform(0.5, 2.0, S),
                  cls=rs.uniform(0.3, 1.5, (S, D)))
    ff = np.where(bad, -1.0, 1.0) + 0.3 * rs.randn(N)

    R = load_constrained()
    with tempfile.TemporaryDirectory() as d:
        ch = R["CONS"].GPConstrainedEIChooser(d, covar=kind, mcmc_iters=S, pending_samples=max(F, 1),
                                              constraint_violating_value=bad_value)
        ch.hyper_samples = [(hyper["mean"][s], hyper["noise"][s], hyper["amp2"][s], hyper["ls"][s]) for s in range(S)]
        ch.constraint_hyper_samples = [(chyper["cmean"][s], chyper["gain"][s], chyper["camp2"][s], chyper["cls"][s])
                                       for s in range(S)]
        ch.ff = ff.copy()
        ch.constraint_noise = 1e-3          # what _real_init sets (CONS:184)
        labels = np.logical_and(vals != bad_value, np.isfinite(vals)).astype(float)   # CONS:219-232
        npr.seed(seed)
        ei = ch.ei_over_hypers(comp, pend, cand, vals, labels)
        prob = np.zeros((S, M))
        for s, h in enumerate(ch.constraint_hyper_samples):
            ch.constraint_mean, ch.constraint_gain, ch.constraint_amp2, ch.constraint_ls = h
            prob[s] = ch.pred_constraint_voilation(cand, comp, labels).ravel()
        # the refinement objective (CONS:471-803) at 3 points; with pending points its fantasies come from
        # npr.set_state(randomstate) (CONS:618): randomstate = RandomState(seed + 100)
        ch.randomstate = np.random.RandomState(seed + 100).get_state()
        fg_x = np.random.RandomState(seed + 200).rand(3, D)
        fg_f, fg_g = np.zeros(3), np.zeros((3, D))
        for i, x in enumerate(fg_x):
            f, g = ch.grad_optimize_ei_over_hypers(x, comp, pend, vals, labels)
            fg_f[i], fg_g[i] = np.ravel(f)[0], g
    np.savez_compressed(os.path.join(HERE, name + ".npz"), kind=kind, seed=seed, comp=comp, cand=cand, pend=pend,
                        vals=vals, labels=labels, bad_value=bad_value, ff=ff, F=F, ei=ei, prob=prob, fg_x=fg_x,
                        fg_f=fg_f, fg_g=fg_g, **hyper, **chyper)
    print(name, ei.shape, "max EI %.3g" % ei.mean(1).max(), "argmax", int(np.argmax(ei.mean(1))))


# ----------------------------------------------------------------------------- whole next() runs of the reference
class _SerialResult(object):
    def __init__(self, value):
        self.value = value

    def get(self, timeout=None):
        return self.value


class _SerialPool(object):
    """multiprocessing.Pool stand-in: runs each task at once in this process.  The global RNG state is saved and
    restored around the task, which is what the reference's fork does (a worker's draws never reach the parent)."""

    def __init__(self, processes=None):
        pass

    def apply_async(self, fn, args=()):
        state = npr.get_state()
        try:
            return _SerialResult(fn(*args))
        finally:
            npr.set_state(state)

    def close(self):
        pass


# name: (kind, D, N complete, P pending, M candidates, violation, options, seed, second call)
NEXT_CASES = {
    "cons_next_inf_d2": ("Matern52", 2, 14, 0, 40, "inf", "mcmc_iters=3,burnin=2,grid_subset=2", 21, False),
    "cons_next_nan_pend_d3": ("Matern52", 3, 16, 2, 40, "nan",
                              "mcmc_iters=2,burnin=2,grid_subset=2,pending_samples=4", 22, False),
    "cons_next_badval_m32": ("Matern32", 2, 14, 0, 40, "value",
                             "mcmc_iters=2,burnin=1,grid_subset=2,noiseless=1,constraint_violating_value=99.0", 23,
                             False),
    "cons_next_twocall": ("Matern52", 2, 12, 0, 40, "inf", "mcmc_iters=2,burnin=2,grid_subset=2", 24, True),
    "cons_next_vanilla": ("ARDSE", 2, 12, 0, 40, "none", "mcmc_iters=2,burnin=1,grid_subset=2", 25, False),
}


def _next_inputs(kind, D, N, P, M, violation, seed):
    rs = np.random.RandomState(seed)
    grid = rs.rand(N + 1 + P + M, D)
    y = branin(np.hstack([grid[:, :2], np.zeros((grid.shape[0], max(0, 2 - D)))])[:, :2])
    values = (y - y.mean()) / y.std()
    bad = grid[:, 0] + grid[:, 1] > (1.3 if violation != "none" else 9.0)
    values[bad] = {"inf": np.inf, "nan": np.nan, "value": BAD_VALUE, "none": 0.0}[violation]
    complete = np.arange(N)
    pending = np.arange(N + 1, N + 1 + P)
    candidates = np.arange(N + 1 + P, N + 1 + P + M)
    return grid, values, complete, pending, candidates


def _record(ch, out, prefix):
    S = len(ch.hyper_samples)
    out[prefix + "hs_mean"] = np.array([h[0] for h in ch.hyper_samples])
    out[prefix + "hs_noise"] = np.array([h[1] for h in ch.hyper_samples])
    out[prefix + "hs_amp2"] = np.array([h[2] for h in ch.hyper_samples])
    out[prefix + "hs_ls"] = np.vstack([h[3] for h in ch.hyper_samples]) if S else np.zeros((0, 0))
    chs = ch.constraint_hyper_samples
    out[prefix + "chs_mean"] = np.array([h[0] for h in chs], dtype=float)
    out[prefix + "chs_gain"] = np.array([h[1] for h in chs], dtype=float)
    out[prefix + "chs_amp2"] = np.array([h[2] for h in chs], dtype=float)
    out[prefix + "chs_ls"] = np.vstack([h[3] for h in chs])
    out[prefix + "ff_samples"] = np.vstack(ch.ff_samples)
    out[prefix + "ff"] = np.asarray(ch.ff)
    with open(ch.state_pkl, "rb") as fh:
        state = pickle.load(fh, encoding="latin1")
    out[prefix + "pkl_keys"] = np.array(sorted(state))
    for k in ("ls", "amp2", "noise", "mean", "constraint_ls", "constraint_amp2", "constraint_mean"):
        out[prefix + "pkl_" + k] = np.asarray(state[k], dtype=float)


def make_next_case(name, kind, D, N, P, M, violation, options, seed, second):
    import contextlib
    import io
    R = load_constrained()
    R["CONS"].multiprocessing = types.SimpleNamespace(Pool=_SerialPool)
    grid, values, complete, pending, candidates = _next_inputs(kind, D, N, P, M, violation, seed)
    out = dict(kind=kind, grid=grid, values=values, complete=complete, pending=pending, candidates=candidates,
               options=options, seed=seed, second=second)
    with tempfile.TemporaryDirectory() as d:
        args = R["util"].unpack_args("covar=%s,%s" % (kind, options))
        if "pending_samples" in args:          # an arg string leaves it a str, which npr.randn rejects (CONS:76, 910)
            args["pending_samples"] = int(args["pending_samples"])
        ch = R["CONS"].GPConstrainedEIChooser(d, **args)
        npr.seed(seed)
        calls = [(complete, pending)]
        if second:
            calls.append((np.arange(N + 1), pending))          # one more observation
        for c, (cpl, pnd) in enumerate(calls):
            buf = io.StringIO()
            with contextlib.redirect_stdout(buf):
                ret = ch.next(grid, values, np.zeros(grid.shape[0]), candidates, pnd, cpl)
            p = "call%d_" % c
            if isinstance(ret, tuple):
                out[p + "ret_index"], out[p + "ret_point"] = int(ret[0]), np.asarray(ret[1])
            else:
                out[p + "ret_index"], out[p + "ret_point"] = int(ret), np.zeros(0)
            out[p + "stdout"] = np.array(buf.getvalue())
            st = npr.get_state()
            out[p + "rng_after"] = np.r_[st[1][:8], st[2]].astype(np.int64)
            _record(ch, out, p)
    np.savez_compressed(os.path.join(HERE, name + ".npz"), **out)
    print(name, "proposal", out["call0_ret_index"], out["call0_ret_point"])


if __name__ == "__main__":
    for name, args in CASES.items():
        make_case(name, *args)
    for name, args in NEXT_CASES.items():
        make_next_case(name, *args)
