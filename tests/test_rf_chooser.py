"""CPU: RandomForestEIChooserB200's host logic on the oracle backend -- the reference's proposals and global-RNG
positions on its own goldens, each reproduced quirk of RF (chooser/RandomForestEIChooser.py), each waived one, and the
option casts."""
import os

import numpy as np
import numpy.random as npr
import pytest

from spearmint_b200.chooser import RandomForestEIChooserB200 as RFmod
from spearmint_b200.chooser.RandomForestEIChooserB200 import RandomForestEIChooserB200
from spearmint_b200.forest import MAX_INT
from tests import rf_cases
from tests import rf_oracle as O

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _rng_equal(g, c):
    st = npr.get_state()
    return (np.array_equal(st[1], g["rng_key_%d" % c]) and st[2] == int(g["rng_pos_%d" % c])
            and st[3] == g["rng_gauss_%d" % c][0] and st[4] == g["rng_gauss_%d" % c][1])


@pytest.mark.parametrize("name", rf_cases.SMALL)
def test_next_reproduces_golden_proposal_and_rng(name):
    g = np.load(os.path.join(GOLDEN, name + ".npz"))
    calls = rf_cases.CASES[name][-1]
    D, N, M, P, kwargs, seed, _ = rf_cases.CASES[name]
    state = rf_cases.inputs(name)
    ch = RandomForestEIChooserB200(backend=O.OracleBackend(), **kwargs)
    npr.seed(seed)
    for c in range(calls):
        grid, values, complete, candidates, pending = state
        p = ch.next(grid, values, None, candidates, pending, complete)
        assert p == int(g["proposal_%d" % c])
        assert _rng_equal(g, c), "global RNG after call %d" % c
        state = rf_cases.second_call(*state, proposal=p)


def _problem(N=30, M=200, P=0, D=2, seed=0):
    rs = np.random.RandomState(seed)
    grid = rs.rand(N + M + P, D)
    values = np.sum((grid - 0.4) ** 2, axis=1)
    return grid, values, np.arange(N), np.arange(N, N + M), np.arange(N + M, N + M + P)


def test_fewer_than_two_complete_returns_first_candidate_without_rng():
    grid, values, _, cand, pend = _problem()
    npr.seed(1)
    before = npr.get_state()
    ch = RandomForestEIChooserB200(backend=O.OracleBackend())
    assert ch.next(grid, values, None, cand[::-1], pend, np.arange(1)) == int(cand[-1])
    assert ch.next(grid, values, None, cand, pend, np.arange(0)) == int(cand[0])
    assert np.array_equal(npr.get_state()[1], before[1]) and npr.get_state()[2] == before[2]


def test_pending_points_two_fits_and_additive_fantasy_noise():
    """Fit, fantasies m + sqrt(v) + randn(P) (the normal added, not scaled), refit on vstack / hstack (waived: RF:72
    indexes np.vstack); the draws are T seeds, randn(P), T seeds; best is the minimum of the COMPLETE values."""
    T, P = 5, 4
    grid, values, comp, cand, pend = _problem(P=P)
    values[pend] = -100.0                                 # never seen by the chooser: pending jobs have no value
    be = O.OracleBackend()
    ch = RandomForestEIChooserB200(n_trees=T, backend=be)
    npr.seed(3)
    ch.next(grid, values, None, cand, pend, comp)
    after = npr.get_state()
    assert len(be.fits) == 2
    f0, f1 = be.fits
    np.testing.assert_array_equal(f1["X"], np.vstack([grid[comp], grid[pend]]))
    npr.seed(3)
    seeds0 = [npr.randint(MAX_INT) for _ in range(T)]
    normals = npr.randn(P)
    seeds1 = [npr.randint(MAX_INT) for _ in range(T)]
    ours = npr.get_state()
    assert np.array_equal(ours[1], after[1]) and ours[2] == after[2]
    forest0 = O.fit(grid[comp], values[comp], f0["weights"], f0["rand_r_states"], 2)
    m, v = O.predict(forest0, grid[pend])
    np.testing.assert_array_equal(f1["y"], np.hstack([values[comp], m + np.sqrt(v) + normals]))
    assert be.best == np.min(values[comp])
    np.testing.assert_array_equal(f0["weights"][0], np.bincount(npr.RandomState(seeds0[0]).randint(0, 30, 30),
                                                                minlength=30))
    np.testing.assert_array_equal(f1["weights"][T - 1], np.bincount(npr.RandomState(seeds1[-1]).randint(0, 34, 34),
                                                                    minlength=34))


def test_random_state_leaves_the_global_rng_and_refits_the_same_forest():
    grid, values, comp, cand, pend = _problem()
    be = O.OracleBackend()
    ch = RandomForestEIChooserB200(n_trees=4, random_state="3", backend=be)
    npr.seed(4)
    before = npr.get_state()
    a = ch.next(grid, values, None, cand, pend, comp)
    b = ch.next(grid, values, None, cand, pend, comp)
    assert a == b
    np.testing.assert_array_equal(be.fits[0]["weights"], be.fits[1]["weights"])
    assert np.array_equal(npr.get_state()[1], before[1]) and npr.get_state()[2] == before[2]


def test_single_tree_returns_first_candidate_and_raises_with_pending():
    grid, values, comp, cand, pend = _problem()
    ch = RandomForestEIChooserB200(n_trees=1, backend=O.OracleBackend())
    assert ch.next(grid, values, None, cand, pend, comp) == int(cand[0])     # var NaN: np.argmax of all-NaN EI is 0
    grid, values, comp, cand, pend = _problem(P=2)
    with pytest.raises(ValueError):
        ch.next(grid, values, None, cand, pend, comp)


@pytest.mark.parametrize("bad", [np.nan, np.inf])
def test_non_finite_complete_values_raise(bad):
    grid, values, comp, cand, pend = _problem()
    values[3] = bad
    npr.seed(0)
    before = npr.get_state()
    with pytest.raises(ValueError):
        RandomForestEIChooserB200(backend=O.OracleBackend()).next(grid, values, None, cand, pend, comp)
    assert npr.get_state()[2] == before[2]                # raised before any seed was drawn, as sklearn's fit does


def test_option_casts_from_the_arg_string():
    ch = RFmod.init("/nonexistent", "n_trees=7,max_depth=None,min_samples_split=1,max_features=auto,"
                                    "random_state=None,n_jobs=4,max_monkeys=2")
    assert (ch.n_trees, ch.max_depth, ch.min_samples_split, ch.random_state) == (7, None, 2, None)
    assert RFmod.resolve_max_features(ch.max_features, 9) == 9
    ch = RFmod.init("x", "max_depth=6,min_samples_split=5,max_features=sqrt,random_state=3")
    assert (ch.max_depth, ch.min_samples_split, ch.random_state) == (6, 5, 3)
    assert RFmod.resolve_max_features(ch.max_features, 9) == 3
    assert RFmod.resolve_max_features(RFmod.init("x", "max_features=log2").max_features, 9) == 3
    assert RFmod.resolve_max_features(RFmod.init("x", "max_features=4").max_features, 9) == 4
    assert RFmod.resolve_max_features(RFmod.init("x", "max_features=0.5").max_features, 9) == 4
    assert RFmod.resolve_max_features(RFmod.init("x", "max_features=1.0").max_features, 9) == 9
    ch = RFmod.init("x", "")
    assert (ch.n_trees, ch.max_depth, ch.min_samples_split) == (50, None, 2)
    with pytest.raises(TypeError):
        RFmod.init("x", "n_tree=5")
