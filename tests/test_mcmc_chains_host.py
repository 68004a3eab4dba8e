"""CPU: mcmc_chains -- the step-wise slice sampler against util.slice_sample, K chains in lockstep against each chain run
alone, the chooser option (round-major samples, state pickle, resume, errors), and mcmc_chains=1 against the single
chain.  The numerics are the oracle's (tests/oracle_backend.py, batched)."""
import os
import pickle

import numpy as np
import numpy.random as npr
import pytest

from spearmint_b200 import chains, util
from tests.helpers import load
from tests.oracle_backend import OracleBackend

NEXT_CASES = ["opt_branin2d", "opt_d8_m52", "opt_d8_m52_pend", "opt_d5_ardse", "opt_d4_m32_pend", "opt_d1_m52"]


@pytest.fixture(autouse=True)
def quiet(monkeypatch):
    import spearmint_b200.locker as lk
    from spearmint_b200.chooser import GPEIOptChooserB200 as mod
    for m in (lk, mod, chains):
        monkeypatch.setattr(m, "log", lambda *a: None)


class ChainOracle(OracleBackend):
    """The batched oracle, also as the handle of several chains (DeviceBackend.loglik's ``chains``)."""

    def __init__(self, speculate=None):
        OracleBackend.__init__(self, batched=True, speculate=speculate)

    def loglik(self, kind, comp, vals, chains=1):
        return OracleBackend.loglik(self, kind, comp, vals)


class Recorder(object):
    """A batched log-likelihood of a 1-argument item that records every point it evaluates."""

    def __init__(self, f, speculate):
        self.f, self.speculate, self.seen = f, speculate, []

    def batch(self, items):
        self.seen.extend(np.asarray(h[0], dtype=float).copy() for h in items)
        return np.array([self.f(np.asarray(h[0], dtype=float)) for h in items])

    def __call__(self, x):
        v = self.batch([(x,)])[0]
        if np.isnan(v):
            raise np.linalg.LinAlgError("leading minor of the array is not positive definite")
        return v


def _identity(x):
    return (x,), ()


def _drive(gen, f, seen):
    """Runs a slice_steps generator on f, recording the points it asks for (duplicates in one request once)."""
    try:
        req = next(gen)
        while True:
            out, keys = [], {}
            for x in req:
                k = x.tobytes()
                if k not in keys:
                    keys[k] = f(x)
                    seen.append(np.asarray(x, dtype=float).copy())
                out.append(keys[k])
            req = gen.send(out)
    except StopIteration as stop:
        return stop.value


def _both(f, x0, speculate, compwise, seed):
    """(result, visited, RNG state) of slice_sample on the global RNG and of slice_steps on a copy of it."""
    npr.seed(seed)
    rs = npr.RandomState()
    rs.set_state(npr.get_state())
    rec = Recorder(f, speculate)
    out = []
    try:
        a = util.slice_sample(x0, util.CachedLogProb(rec, _identity), compwise=compwise)
    except np.linalg.LinAlgError:
        a = "not pd"
    out.append((a, rec.seen, npr.get_state()))
    seen = []
    try:
        b = _drive(util.slice_steps(x0, rs, speculate, compwise=compwise), f, seen)
    except np.linalg.LinAlgError:
        b = "not pd"
    out.append((b, seen, rs.get_state()))
    return out


def _same(a, b):
    (ra, va, sa), (rb, vb, sb) = a, b
    if isinstance(ra, str):
        assert ra == rb
    else:
        np.testing.assert_array_equal(ra, rb)
    assert len(va) == len(vb)
    for p, q in zip(va, vb):
        np.testing.assert_array_equal(p, q)
    assert sa[0] == sb[0] and np.array_equal(sa[1], sb[1]) and sa[2:] == sb[2:]


def _gauss(center, width):
    return lambda x: -0.5 * float(np.sum(((x - center) / width) ** 2))


@pytest.mark.parametrize("speculate", [(3, 0), (0, 2), (1, 3)])
@pytest.mark.parametrize("case", ["step_out", "long_shrink", "compwise", "not_pd"])
def test_steps_match_slice_sample(case, speculate):
    """Same draws, same visited points in the same order, same result as slice_sample with a CachedLogProb."""
    x0 = np.array([0.3, -0.2, 0.1])
    if case == "step_out":             # a density 20 wide: the unit interval steps out on both sides
        f, compwise = _gauss(x0, 20.0), False
    elif case == "long_shrink":        # 1e-4 wide: many shrink proposals
        f, compwise = _gauss(x0, 1e-4), False
    elif case == "compwise":
        f, compwise = _gauss(x0 + 0.5, 0.7), True
    else:                              # NaN (not positive definite) in the middle of a move
        g = _gauss(x0, 20.0)
        f, compwise = (lambda x: np.nan if x[0] > x0[0] + 1.5 else g(x)), False
    for seed in range(6):
        a, b = _both(f, x0, speculate, compwise, seed)
        _same(a, b)
        if case == "step_out":
            assert len(a[1]) > 8
        if case == "long_shrink":
            assert len(a[1]) > 12
        if case == "not_pd" and seed == 0:
            assert a[0] == "not pd"


def test_step_out_reaches_both_sides():
    """The step-out case above really steps out below and above the start."""
    x0 = np.array([0.3, -0.2, 0.1])
    npr.seed(0)
    rec = Recorder(_gauss(x0, 20.0), (3, 0))
    util.slice_sample(x0, util.CachedLogProb(rec, _identity))
    npr.seed(0)
    d = npr.randn(3)
    d = d / np.sqrt(np.sum(d ** 2))
    upper = npr.rand()
    z = [float(np.dot(p - x0, d)) for p in rec.seen]
    assert min(z) < upper - 2.0 and max(z) > upper + 1.0


def _golden_ll(name):
    from tests.helpers import sets
    g = load(name)
    comp, _, _, vals = sets(g)
    return g, comp, vals, ChainOracle((3, 0)).loglik(str(g["kind"]), comp, vals)


@pytest.mark.parametrize("noiseless", [False, True])
def test_prior_moves_match_single_chain(noiseless):
    """GPPrior.joint_steps / length_scales_steps against joint / length_scales on the golden data."""
    from spearmint_b200.chooser.GPEIOptChooserB200 import GPEIOptChooserB200 as Ch
    g, comp, vals, ll = _golden_ll("opt_d8_m52")
    prior = Ch.prior
    D = comp.shape[1]
    h = (float(np.mean(vals)), 1e-3 if noiseless else 0.05, float(np.std(vals)) + 1e-4, np.ones(D))
    for seed in range(3):
        npr.seed(seed)
        rs = npr.RandomState()
        rs.set_state(npr.get_state())
        j1 = prior.joint(ll, h[0], h[2], h[1], h[3], vals, noiseless)
        l1 = prior.length_scales(ll, j1[0], j1[2], j1[1], h[3])
        res = []

        def run():
            j = yield from prior.joint_steps(rs, h[0], h[2], h[1], h[3], vals, noiseless, ll.speculate)
            ls = yield from prior.length_scales_steps(rs, j[0], j[2], j[1], h[3], ll.speculate)
            res.append((j, ls))
        chains.lockstep([run()], ll)
        j2, l2 = res[0]
        np.testing.assert_array_equal(np.array(j1), np.array(j2))
        np.testing.assert_array_equal(l1, l2)
        s1, s2 = npr.get_state(), rs.get_state()
        assert np.array_equal(s1[1], s2[1]) and s1[2] == s2[2]


def _chain_set(K, D, vals, seed):
    npr.seed(seed)
    return chains.Chain.seeded(K, (float(np.mean(vals)), 1e-3, float(np.std(vals)) + 1e-4, np.ones(D)))


def test_lockstep_equals_chains_alone():
    """K = 4 chains in lockstep: every chain's samples and evaluation count are those of the chain run alone."""
    from spearmint_b200.chooser.GPEIOptChooserB200 import GPEIOptChooserB200 as Ch
    g, comp, vals, ll = _golden_ll("opt_d5_ardse")
    K, burn, steps = 4, 3, 2
    together = _chain_set(K, comp.shape[1], vals, 11)
    ev = [0] * K
    rounds = chains.lockstep([c.run(Ch.prior, vals, False, burn, steps, ll.speculate) for c in together], ll, ev)
    for c in range(K):
        alone = _chain_set(K, comp.shape[1], vals, 11)[c]
        ev1 = [0]
        r1 = chains.lockstep([alone.run(Ch.prior, vals, False, burn, steps, ll.speculate)], ll, ev1)
        assert r1 <= rounds and ev1[0] == ev[c]
        assert len(alone.samples) == steps
        for a, b in zip(alone.samples, together[c].samples):
            np.testing.assert_array_equal(np.hstack(a), np.hstack(b))
        assert np.array_equal(alone.rs.get_state()[1], together[c].rs.get_state()[1])
    # the chains differ from each other (own RandomStates)
    assert not np.array_equal(np.hstack(together[0].samples[-1]), np.hstack(together[1].samples[-1]))


def _make(g, d, K=None, S=None, backend=None, **extra):
    from spearmint_b200.chooser import GPEIOptChooserB200 as mod
    args = "covar=%s,mcmc_iters=%d,burnin=%d,noiseless=%d,use_multiprocessing=0,grid_subset=5" % (
        str(g["kind"]), int(S or g["S"]), int(g["burnin"]), int(g["noiseless"]))
    if K is not None:
        args += ",mcmc_chains=%d" % K
    ch = mod.init(str(d), args)
    ch._backend = backend or ChainOracle()
    return ch


def _next(ch, g, seed=None):
    if seed is not None:
        npr.seed(seed)
    return ch.next(g["grid"], g["values"], g["durations"], g["candidates"], g["pending"], g["complete"])


def test_round_major_order_and_seeding(tmp_path):
    """hyper_samples[r K + c] is step r of chain c; the chain seeds are K draws of npr.randint(2**32) right after the
    jitter cloud of the first next(), and the chains then never touch the global RNG."""
    from spearmint_b200.chooser.GPEIOptChooserB200 import GPEIOptChooserB200 as Ch
    g = load("opt_d8_m52")
    K, S = 2, 4
    ch = _make(g, tmp_path, K, S)
    _next(ch, g, 5)
    assert len(ch.hyper_samples) == S
    for r in range(S // K):
        for c in range(K):
            np.testing.assert_array_equal(np.hstack(ch.hyper_samples[r * K + c]), np.hstack(ch.chains[c].samples[r]))
    # replay by hand: the jitter cloud, the seeds, each chain alone
    from tests.helpers import sets
    comp, _, _, vals = sets(g)
    npr.seed(5)
    npr.randn(10, comp.shape[1])
    start = (np.mean(vals), 1e-3, np.std(vals) + 1e-4, np.ones(comp.shape[1]))
    mine = chains.Chain.seeded(K, start)
    ll = ChainOracle().loglik(str(g["kind"]), comp, vals)
    for c in mine:
        chains.lockstep([c.run(Ch.prior, vals, bool(int(g["noiseless"])), int(g["burnin"]), S // K, (util.SPECULATE, 0))], ll)
    for c in range(K):
        for a, b in zip(mine[c].samples, ch.chains[c].samples):
            np.testing.assert_array_equal(np.hstack(a), np.hstack(b))
    np.testing.assert_array_equal(np.hstack([ch.mean, ch.noise, ch.amp2, ch.ls]), np.hstack(mine[-1].samples[-1]))


def test_option_errors(tmp_path):
    from spearmint_b200.chooser import GPEIOptChooserB200 as mod
    for bad in ("mcmc_chains=0", "mcmc_chains=-2", "mcmc_iters=10,mcmc_chains=4", "mcmc_iters=3,mcmc_chains=2"):
        with pytest.raises(ValueError):
            mod.init(str(tmp_path), bad)
    assert mod.init(str(tmp_path), "mcmc_iters=12,mcmc_chains=4").mcmc_chains == 4
    assert mod.init(str(tmp_path), "").mcmc_chains == 1
    g = load("opt_branin2d")
    ch = mod.init(str(tmp_path), "mcmc_iters=0,mcmc_chains=2")       # mcmc_iters <= 0 keeps its own error
    ch._backend = ChainOracle()
    with pytest.raises(NotImplementedError):
        _next(ch, g, 0)
    for other in ("GPEIChooserB200", "GPEIperSecChooserB200", "GPConstrainedEIChooserB200",
                  "RandomForestEIChooserB200"):
        m = __import__("spearmint_b200.chooser." + other, fromlist=["init"])
        with pytest.raises(TypeError):
            m.init(str(tmp_path), "mcmc_chains=2")


def test_pickle_round_trip_resumes_without_burnin(tmp_path):
    """The pickle keeps the reference's keys plus ``chains``; a fresh chooser resumes exactly where the chains stopped:
    its second next() equals the first chooser's second next()."""
    g = load("opt_branin2d")
    K, S = 2, 4
    os.makedirs(tmp_path / "a")
    a = _make(g, tmp_path / "a", K, S)
    _next(a, g, 3)
    st = pickle.load(open(a.state_pkl, "rb"))
    assert sorted(st) == ["amp2", "chains", "dims", "hyper_samples", "ls", "mean", "noise"]
    assert len(st["chains"]) == K
    np.testing.assert_array_equal(np.hstack([st["mean"], st["noise"], st["amp2"], st["ls"]]),
                                  np.hstack(st["hyper_samples"][-1]))
    for c, s in zip(a.chains, st["chains"]):
        np.testing.assert_array_equal(np.hstack(s[:4]), np.hstack(c.samples[-1]))
    b = _make(g, tmp_path / "a", K, S)           # same directory: resumes from the pickle
    n0 = a._backend.loglik_calls
    _next(b, g, 4)                               # before a's second call rewrites the pickle
    _next(a, g, 4)
    assert all(not c.needs_burnin for c in b.chains)
    for x, y in zip(a.hyper_samples, b.hyper_samples):
        np.testing.assert_array_equal(np.hstack(x), np.hstack(y))
    assert b._backend.loglik_calls == a._backend.loglik_calls - n0      # no burn-in evaluations either
    # a chains list of another length
    c = _make(g, tmp_path / "a", 4, S)
    with pytest.raises(ValueError):
        _next(c, g, 4)


def test_single_chain_pickle_resumes_with_burnin(tmp_path):
    """A pickle without ``chains`` (single-chain or the reference's): every chain starts from its hypers and burns in."""
    from spearmint_b200.chooser.GPEIOptChooserB200 import GPEIOptChooserB200 as Ch
    g = load("opt_d1_m52")
    K, S = 2, 4
    one = _make(g, tmp_path, None, S)
    _next(one, g, 1)
    st = pickle.load(open(one.state_pkl, "rb"))
    assert "chains" not in st
    two = _make(g, tmp_path, K, S)
    _next(two, g, 2)
    from tests.helpers import sets
    comp, _, _, vals = sets(g)
    npr.seed(2)
    npr.randn(10, comp.shape[1])
    mine = chains.Chain.seeded(K, (st["mean"], st["noise"], st["amp2"], st["ls"]))
    ll = ChainOracle().loglik(str(g["kind"]), comp, vals)
    for c in mine:
        assert c.needs_burnin
        chains.lockstep([c.run(Ch.prior, vals, bool(int(g["noiseless"])), int(g["burnin"]), S // K, (util.SPECULATE, 0))], ll)
    for c in range(K):
        for a, b in zip(mine[c].samples, two.chains[c].samples):
            np.testing.assert_array_equal(np.hstack(a), np.hstack(b))
    # and mcmc_chains=1 resumes from a multi-chain pickle through the reference's keys (``chains`` ignored)
    one2 = _make(g, tmp_path, 1, S)
    _next(one2, g, 3)
    assert one2.chains is None and "chains" not in pickle.load(open(one2.state_pkl, "rb"))


@pytest.mark.parametrize("name", NEXT_CASES)
def test_one_chain_is_the_single_chain(name, tmp_path):
    """mcmc_chains=1: the same proposal, pickle and global RNG state as without the option."""
    g = load(name)
    outs = []
    for i, K in enumerate((None, 1)):
        d = tmp_path / str(i)
        d.mkdir()
        ch = _make(g, d, K, backend=OracleBackend())
        ret = _next(ch, g, int(g["seed"]))
        outs.append((ret, pickle.load(open(ch.state_pkl, "rb")), npr.get_state()))
    (r0, p0, s0), (r1, p1, s1) = outs
    if isinstance(r0, tuple):
        assert r0[0] == r1[0] and np.array_equal(r0[1], r1[1])
    else:
        assert r0 == r1
    assert sorted(p0) == sorted(p1)
    for k in p0:
        if k == "hyper_samples":
            for a, b in zip(p0[k], p1[k]):
                np.testing.assert_array_equal(np.hstack(a), np.hstack(b))
        else:
            np.testing.assert_array_equal(p0[k], p1[k])
    assert np.array_equal(s0[1], s1[1]) and s0[2:] == s1[2:]
