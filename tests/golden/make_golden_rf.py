"""Freezes the reference's random-forest chooser into tests/golden/rf_*.npz.

    python tests/golden/make_golden_rf.py

Runs chooser/RandomForestEIChooser.py (RF) through oracle/ref_shim.py's py2->py3 rewrites on scikit-learn 1.9, with four
more rewrites that let RF load and run there:
  * ``sklearn.externals.joblib`` (removed from sklearn) is stubbed with joblib's Parallel / delayed;
  * ``sklearn.ensemble.forest`` is aliased to ``sklearn.ensemble._forest``;
  * the defaults ``min_samples_split=1`` and ``max_features="auto"``, which sklearn now rejects, become 2 and 1.0 (the
    same trees: the sklearn of 2013 treated 1 as 2, and "auto" meant all features for a regressor);
  * ``np.vstack[comp,pend]`` / ``np.hstack[vals,vals_pend]`` (a TypeError on every numpy) become calls, so the pending
    case runs.
Each case seeds the global RNG, runs ``next()`` (twice for the two-call case) and stores the proposal, the RNG state
afterwards, mean / var / EI at the candidates of the last call (a subset for the large case) and, for the small cases,
the arrays of the first 5 trees of the last fit.  Inputs: tests/rf_cases.py.
"""
import os
import sys
import types

import numpy as np
import numpy.random as npr
import scipy.stats as sps

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from oracle import ref_shim  # noqa: E402
from tests import rf_cases  # noqa: E402


def load_rf():
    import joblib
    import sklearn.ensemble
    import sklearn.ensemble._forest
    mods = ref_shim.load()
    ext = types.ModuleType("sklearn.externals.joblib")
    ext.Parallel, ext.delayed = joblib.Parallel, joblib.delayed
    sys.modules["sklearn.externals.joblib"] = ext
    sys.modules["sklearn.ensemble.forest"] = sklearn.ensemble._forest
    sklearn.ensemble.forest = sklearn.ensemble._forest
    path = os.path.join(ref_shim.REF_PKG, "chooser", "RandomForestEIChooser.py")
    with open(path) as fh:
        src = ref_shim._py3(fh.read())
    for old, new in (("min_samples_split=1,", "min_samples_split=2,"), ('max_features="auto",', "max_features=1.0,"),
                     ("np.vstack[comp,pend]", "np.vstack([comp,pend])"),
                     ("np.hstack[vals,vals_pend]", "np.hstack([vals,vals_pend])")):
        assert old in src, old
        src = src.replace(old, new)
    mod = types.ModuleType("chooser.RandomForestEIChooser")
    mod.__file__ = path
    sys.modules[mod.__name__] = mod
    exec(compile(src, path, "exec"), mod.__dict__)
    return dict(mods, RF=mod)


def make_case(RF, name):
    D, N, M, P, kwargs, seed, calls = rf_cases.CASES[name]
    state = rf_cases.inputs(name)
    ch = RF.RandomForestEIChooser(**kwargs)
    npr.seed(seed)
    out = {}
    for c in range(calls):
        grid, values, complete, candidates, pending = state
        prop = ch.next(grid, values, None, candidates, pending, complete)
        st = npr.get_state()
        out["proposal_%d" % c] = np.int64(prop)
        out["rng_key_%d" % c], out["rng_pos_%d" % c] = st[1].copy(), np.int64(st[2])
        out["rng_gauss_%d" % c] = np.array([st[3], st[4]])
        if c + 1 < calls:
            state = rf_cases.second_call(*state, proposal=prop)
    grid, values, complete, candidates, pending = state
    cand = grid[candidates]
    m, v = ch.rf.predict(cand)
    best = np.min(values[complete])
    s = np.sqrt(v) + 0.0001
    u = (best - m) / s
    ei = s * (u * sps.norm.cdf(u) + sps.norm.pdf(u))
    if name in rf_cases.SMALL:
        for t, est in enumerate(ch.rf.estimators_[:5]):
            tr = est.tree_
            for k in ("feature", "threshold", "children_left", "children_right", "n_node_samples"):
                out["tree%d_%s" % (t, k)] = np.asarray(getattr(tr, k))
            out["tree%d_value" % t] = tr.value[:, 0, 0].copy()
        out.update(mean=m, var=v, ei=ei)
    else:
        idx = rf_cases.subset(cand.shape[0])
        idx = np.union1d(idx, [int(np.argmax(ei))])
        out.update(subset=idx, mean=m[idx], var=v[idx], ei=ei[idx])
    out["argmax"] = np.int64(np.argmax(ei))
    np.savez_compressed(os.path.join(HERE, name + ".npz"), **out)
    print(name, "proposal", [int(out["proposal_%d" % c]) for c in range(calls)], "max EI %.4g" % ei.max())


if __name__ == "__main__":
    mods = load_rf()
    names = sys.argv[1:] or list(rf_cases.CASES)
    for n in names:
        make_case(mods["RF"], n)
