"""GPU: the device random forest (csrc/forest.cu) -- trees node for node equal to the oracle's (and so to sklearn's) at the
golden sizes, mean / var / EI and proposals of the reference's goldens (tests/golden/rf_*.npz) up to N=4096 / D=32,
the predict kernel against a numpy traversal of the same device trees at M=100 000, and a fully grown N=16 384 forest."""
import os

import numpy as np
import numpy.random as npr
import pytest
import torch

from tests import rf_cases
from tests import rf_oracle as O

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
KEYS = (("feature", "feature"), ("threshold", "threshold"), ("left", "children_left"), ("right", "children_right"),
        ("n_node_samples", "n_node_samples"))


class Recording(object):
    """DeviceBackend that keeps every fit's inputs and the last device forest."""

    def __init__(self):
        from spearmint_b200.backend import DeviceBackend
        self.be = DeviceBackend()
        self.fits, self.forest = [], None

    def forest_fit(self, X, y, weights, rand_r_states, max_features, max_depth=None, min_samples_split=2):
        self.fits.append((np.array(X), np.array(y), weights, rand_r_states, max_features, max_depth, min_samples_split))
        self.forest = self.be.forest_fit(X, y, weights, rand_r_states, max_features, max_depth, min_samples_split)
        return self.forest

    def forest_predict(self, forest, X):
        return self.be.forest_predict(forest, X)

    def forest_argmax_ei(self, forest, cand, best):
        return self.be.forest_argmax_ei(forest, cand, best)


def _run(name):
    from spearmint_b200.chooser.RandomForestEIChooserB200 import RandomForestEIChooserB200
    g = np.load(os.path.join(GOLDEN, name + ".npz"))
    D, N, M, P, kwargs, seed, calls = rf_cases.CASES[name]
    state = rf_cases.inputs(name)
    rec = Recording()
    ch = RandomForestEIChooserB200(backend=rec, **kwargs)
    npr.seed(seed)
    for c in range(calls):
        grid, values, complete, candidates, pending = state
        p = ch.next(grid, values, None, candidates, pending, complete)
        st = npr.get_state()
        assert p == int(g["proposal_%d" % c]), (name, c)
        assert np.array_equal(st[1], g["rng_key_%d" % c]) and st[2] == int(g["rng_pos_%d" % c])
        if c + 1 < calls:
            state = rf_cases.second_call(*state, proposal=p)
    return g, rec, state


def _check_moments(g, rec, state, idx=None):
    grid, values, complete, candidates, pending = state
    cand = grid[candidates] if idx is None else grid[candidates][idx]
    out = rec.forest.predict(cand, float(np.min(values[complete])))
    m, v, e = (out[k].cpu().numpy() for k in ("mean", "var", "ei"))
    assert np.abs(m - g["mean"]).max() <= 1e-12 * np.abs(g["mean"]).max()
    assert np.abs(v - g["var"]).max() <= 1e-12 * g["var"].max()
    assert np.abs(e - g["ei"]).max() <= 1e-9 * g["ei"].max()


@pytest.mark.parametrize("name", rf_cases.SMALL)
def test_golden_small_trees_and_proposal(name):
    g, rec, state = _run(name)
    X, y, w, s, mf, md, mss = rec.fits[-1]
    ref = O.fit(X, y, w, s, mf, md, mss)
    for t, tr in enumerate(ref):
        dev = rec.forest.tree(t)
        for ours, theirs in KEYS:
            np.testing.assert_array_equal(dev[ours], getattr(tr, theirs), err_msg="%s tree %d %s" % (name, t, ours))
        np.testing.assert_allclose(dev["value"], tr.value, rtol=1e-13, atol=0, err_msg="%s tree %d" % (name, t))
        if t < 5:
            for ours, theirs in KEYS:
                np.testing.assert_array_equal(dev[ours], g["tree%d_%s" % (t, theirs)])
            np.testing.assert_allclose(dev["value"], g["tree%d_value" % t], rtol=1e-13, atol=0)
    _check_moments(g, rec, state)


def test_golden_n4096_d32():
    g, rec, state = _run("rf_d32_n4096")
    _check_moments(g, rec, state, g["subset"])


def _grown(N, D, T, seed, fn=np.sin):
    from spearmint_b200.backend import DeviceBackend
    from spearmint_b200.forest import draws
    from oracle import sobol_oracle
    X = sobol_oracle.i4_sobol_generate(D, N, 1 + seed).T.copy()
    y = fn(4 * X).sum(1)
    npr.seed(seed)
    w, s = draws(T, N)
    return X, y, w, DeviceBackend().forest_fit(X, y, w, s, D)


def test_predict_kernel_matches_numpy_traversal_at_100k():
    X, y, w, forest = _grown(1000, 8, 50, 1)
    C = np.random.RandomState(2).rand(100000, 8)
    out = forest.predict(C, best=float(y.min()))
    allp = []
    for t in range(50):
        tr = forest.tree(t)
        ot = O.Tree()
        ot.feature, ot.threshold = tr["feature"].astype(np.int64), tr["threshold"]
        ot.children_left, ot.children_right = tr["left"].astype(np.int64), tr["right"].astype(np.int64)
        ot.value = tr["value"]
        allp.append(ot.predict(C))
    allp = np.array(allp)
    m = sum(allp) / 50
    v = np.var(allp, axis=0, ddof=1)
    assert np.abs(out["mean"].cpu().numpy() - m).max() <= 1e-12 * np.abs(m).max()
    assert np.abs(out["var"].cpu().numpy() - v).max() <= 1e-12 * v.max()
    e = O.ei(m, v, float(y.min()))
    assert np.abs(out["ei"].cpu().numpy() - e).max() <= 1e-9 * e.max()


def test_fully_grown_n16384_d32():
    N, D, T = 16384, 32, 50
    X, y, w, forest = _grown(N, D, T, 3, fn=np.cos)
    torch.cuda.synchronize()
    counts = forest.node_count.cpu().numpy()
    for t in range(T):
        n_in = int(np.count_nonzero(w[t]))
        assert 1 <= counts[t] <= 2 * n_in - 1
        tr = forest.tree(t)
        ot = O.Tree()
        ot.feature, ot.threshold = tr["feature"].astype(np.int64), tr["threshold"]
        ot.children_left, ot.children_right = tr["left"].astype(np.int64), tr["right"].astype(np.int64)
        ot.value = tr["value"]
        inbag = np.nonzero(w[t])[0]
        np.testing.assert_allclose(ot.predict(X[inbag]), y[inbag], rtol=1e-14, atol=1e-15)
        assert tr["n_node_samples"][0] == n_in
