"""CPU: the random-forest oracle (tests/rf_oracle.py) grows scikit-learn 1.9's trees node for node from the host draws of
spearmint_b200.forest.draws, and reproduces the reference chooser's goldens (tests/golden/rf_*.npz)."""
import os

import numpy as np
import numpy.random as npr
import pytest

from spearmint_b200.chooser.RandomForestEIChooserB200 import RandomForestEIChooserB200, resolve_max_features
from spearmint_b200.forest import draws
from tests import rf_cases
from tests import rf_oracle as O

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
TREE_KEYS = (("feature", "feature"), ("threshold", "threshold"), ("children_left", "children_left"),
             ("children_right", "children_right"), ("n_node_samples", "n_node_samples"))


def _same_tree(tree, arrays):
    """tree: oracle Tree; arrays: dict in sklearn's names.  Structure exactly, value to rtol 1e-13."""
    for k, _ in TREE_KEYS:
        np.testing.assert_array_equal(getattr(tree, k), arrays[k], err_msg=k)
    np.testing.assert_allclose(tree.value, arrays["value"], rtol=1e-13, atol=0)


@pytest.mark.parametrize("N", [2, 3, 50, 300])
@pytest.mark.parametrize("D", [1, 2, 8])
@pytest.mark.parametrize("max_features", [1.0, "sqrt", 3])
@pytest.mark.parametrize("max_depth", [None, 4])
def test_trees_equal_sklearn(N, D, max_features, max_depth):
    ens = pytest.importorskip("sklearn.ensemble")
    if max_features == 3 and D < 3:
        pytest.skip("sklearn rejects max_features > n_features")
    for seed in range(2):
        rs = np.random.RandomState(1000 * N + 10 * D + seed)
        X = rs.rand(N, D)
        y = np.sin(5 * X).sum(1) + 0.1 * rs.randn(N)
        npr.seed(seed)
        before = npr.get_state()
        rf = ens.RandomForestRegressor(n_estimators=6, max_features=max_features, max_depth=max_depth, n_jobs=1)
        rf.fit(X, y)
        after = npr.get_state()
        npr.set_state(before)
        weights, states = draws(6, N)
        ours = npr.get_state()
        assert np.array_equal(ours[1], after[1]) and ours[2] == after[2]     # the global RNG ends where sklearn's does
        forest = O.fit(X, y, weights, states, resolve_max_features(max_features, D), max_depth)
        for tree, est in zip(forest, rf.estimators_):
            t = est.tree_
            _same_tree(tree, dict({k: getattr(t, k) for k, _ in TREE_KEYS}, value=t.value[:, 0, 0]))
        m, v = O.predict(forest, X)
        allp = np.array([e.predict(X) for e in rf.estimators_])
        np.testing.assert_array_equal(m, sum(allp) / 6)
        np.testing.assert_array_equal(v, np.var(allp, axis=0, ddof=1))


def test_random_state_gives_the_same_forest_and_leaves_the_global_rng():
    npr.seed(5)
    before = npr.get_state()
    w1, s1 = draws(4, 40, random_state=7)
    w2, s2 = draws(4, 40, random_state=7)
    after = npr.get_state()
    assert np.array_equal(w1, w2) and np.array_equal(s1, s2)
    assert np.array_equal(before[1], after[1]) and before[2] == after[2]
    assert np.array_equal(w1.sum(1), np.full(4, 40.0))


def replay(name, backend):
    """Runs the chooser through every call of a golden case; returns the proposals."""
    D, N, M, P, kwargs, seed, calls = rf_cases.CASES[name]
    state = rf_cases.inputs(name)
    ch = RandomForestEIChooserB200(backend=backend, **kwargs)
    npr.seed(seed)
    props = []
    for c in range(calls):
        grid, values, complete, candidates, pending = state
        props.append(ch.next(grid, values, None, candidates, pending, complete))
        if c + 1 < calls:
            state = rf_cases.second_call(*state, proposal=props[-1])
    return props, state


@pytest.mark.parametrize("name", rf_cases.SMALL)
def test_oracle_reproduces_golden(name):
    g = np.load(os.path.join(GOLDEN, name + ".npz"))
    be = O.OracleBackend()
    props, state = replay(name, be)
    grid, values, complete, candidates, pending = state
    for t in range(5):
        _same_tree(be.forest[t], {k: g["tree%d_%s" % (t, k)] for k in
                                  ("feature", "threshold", "children_left", "children_right", "n_node_samples", "value")})
    m, v = O.predict(be.forest, grid[candidates])
    assert np.abs(m - g["mean"]).max() <= 1e-12 * np.abs(g["mean"]).max()
    assert np.abs(v - g["var"]).max() <= 1e-12 * g["var"].max()
    e = O.ei(m, v, np.min(values[complete]))
    assert np.abs(e - g["ei"]).max() <= 1e-9 * g["ei"].max()
    assert int(np.argmax(e)) == int(g["argmax"])
