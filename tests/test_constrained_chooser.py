"""CPU: GPConstrainedEIChooserB200 on the oracle backend against whole next() runs of the reference
(tests/golden/cons_next_*.npz): proposal, both sample chains, ff_samples, pickle, stdout and the global RNG afterwards;
and the reference's quirks, each on its own."""
import contextlib
import glob
import io
import os
import pickle

import numpy as np
import numpy.random as npr
import pytest

from spearmint_b200.chooser import GPConstrainedEIChooserB200 as CB
from tests.constrained_oracle_backend import ConstrainedOracleBackend

GOLDEN_NEXT = sorted(glob.glob(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "cons_next_*.npz")))
IDS = [os.path.basename(p) for p in GOLDEN_NEXT]


def run_plugin(path, backend, tmpdir):
    """Replays a golden next() case with the plugin; returns {key: value} shaped like the golden."""
    z = np.load(path)
    opts = "covar=%s,%s" % (str(z["kind"]), str(z["options"]))
    ch = CB.init(str(tmpdir), opts)
    ch._backend = backend
    grid, values, pending, candidates = z["grid"], z["values"], z["pending"], z["candidates"]
    N = z["complete"].shape[0]
    calls = [z["complete"]] + ([np.arange(N + 1)] if bool(z["second"]) else [])
    npr.seed(int(z["seed"]))
    out = {}
    for c, cpl in enumerate(calls):
        buf = io.StringIO()
        with contextlib.redirect_stdout(buf):
            ret = ch.next(grid, values, np.zeros(grid.shape[0]), candidates, pending, cpl)
        p = "call%d_" % c
        out[p + "ret"] = ret
        out[p + "stdout"] = buf.getvalue()
        st = npr.get_state()
        out[p + "rng_after"] = np.r_[st[1][:8], st[2]].astype(np.int64)
        out[p + "hs"] = list(ch.hyper_samples)
        out[p + "chs"] = list(ch.constraint_hyper_samples)
        out[p + "ff_samples"] = np.vstack(ch.ff_samples)
        with open(ch.state_pkl, "rb") as fh:
            out[p + "pkl"] = pickle.load(fh)
    return z, out, len(calls)


def check_against_golden(z, out, ncalls, rtol, atol_point):
    for c in range(ncalls):
        p = "call%d_" % c
        ret = out[p + "ret"]
        if z[p + "ret_point"].size:
            assert isinstance(ret, tuple) and ret[0] == int(z[p + "ret_index"])
            np.testing.assert_allclose(ret[1], z[p + "ret_point"], rtol=0, atol=atol_point)
        else:
            assert ret == int(z[p + "ret_index"])
        assert out[p + "stdout"] == str(z[p + "stdout"])
        np.testing.assert_array_equal(out[p + "rng_after"], z[p + "rng_after"])
        hs, chs = out[p + "hs"], out[p + "chs"]
        np.testing.assert_allclose([h[0] for h in hs], z[p + "hs_mean"], rtol=rtol)
        np.testing.assert_allclose([h[1] for h in hs], z[p + "hs_noise"], rtol=rtol)
        np.testing.assert_allclose([h[2] for h in hs], z[p + "hs_amp2"], rtol=rtol)
        np.testing.assert_allclose(np.vstack([h[3] for h in hs]), z[p + "hs_ls"], rtol=rtol)
        np.testing.assert_allclose([h[1] for h in chs], z[p + "chs_gain"], rtol=rtol)
        np.testing.assert_allclose([h[2] for h in chs], z[p + "chs_amp2"], rtol=rtol)
        np.testing.assert_allclose(np.vstack([h[3] for h in chs]), z[p + "chs_ls"], rtol=rtol)
        np.testing.assert_allclose(out[p + "ff_samples"], z[p + "ff_samples"], rtol=rtol, atol=rtol)
        pkl = out[p + "pkl"]
        assert set(z[p + "pkl_keys"]) | {"constraint_gain"} == set(pkl)       # the reference's keys + constraint_gain
        for k in ("ls", "amp2", "noise", "mean", "constraint_ls", "constraint_amp2", "constraint_mean"):
            np.testing.assert_allclose(np.asarray(pkl[k], dtype=float), z[p + "pkl_" + k], rtol=rtol)


@pytest.mark.parametrize("path", GOLDEN_NEXT, ids=IDS)
def test_next_reproduces_the_reference(path, tmp_path):
    z, out, ncalls = run_plugin(path, ConstrainedOracleBackend(), tmp_path)
    check_against_golden(z, out, ncalls, rtol=1e-8, atol_point=1e-6)


def test_goldens_cover_the_next_cases():
    assert {"cons_next_inf_d2.npz", "cons_next_nan_pend_d3.npz", "cons_next_badval_m32.npz",
            "cons_next_twocall.npz", "cons_next_vanilla.npz"} <= set(IDS)


def test_second_call_reuses_the_first_samples_and_the_stale_latent(tmp_path):
    """Quirks 1 and 2: constraint_hyper_samples is never cleared, so the grid passes of the second call use the
    burn-in draws of the first; ff_samples is kept while ff is long enough; the pickle holds sample S-1's state."""
    path = [p for p in GOLDEN_NEXT if p.endswith("cons_next_twocall.npz")][0]
    z, out, ncalls = run_plugin(path, ConstrainedOracleBackend(), tmp_path)
    assert ncalls == 2
    S = 2
    burnin = 2
    assert len(out["call0_chs"]) == burnin + S and len(out["call1_chs"]) == burnin + 2 * S
    assert out["call1_chs"][:burnin + S] == out["call0_chs"]               # appended to, never cleared
    # one more observation makes ff shorter than comp: ff_samples restarts at the second call
    assert out["call1_ff_samples"].shape == (S, 13) and out["call0_ff_samples"].shape == (burnin + S, 12)
    pkl = out["call0_pkl"]                                                  # sample S-1 (of the FIRST draws) is pickled
    np.testing.assert_allclose(pkl["constraint_amp2"], out["call0_chs"][S - 1][2])
    np.testing.assert_allclose(pkl["constraint_gain"], out["call0_chs"][S - 1][1])


class _NoBackend(object):
    def __getattr__(self, name):
        raise AssertionError("backend used: %s" % name)


def _tiny(values):
    grid = np.random.RandomState(0).rand(len(values) + 5, 2)
    return grid, np.asarray(values, dtype=float), np.arange(len(values)), np.arange(len(values), len(values) + 5)


def test_early_returns_and_mcmc_iters_zero(tmp_path):
    """Quirk 9: candidates[0] with < 2 complete, < 2 valid results; mcmc_iters <= 0 raises Exception('mcmc_iters <= 0')
    after the jitter draw."""
    ch = CB.init(str(tmp_path), "mcmc_iters=0")
    ch._backend = _NoBackend()
    grid, vals, cpl, cand = _tiny([0.3])
    assert ch.next(grid, vals, vals, cand, np.array([], int), cpl) == int(cand[0])
    grid, vals, cpl, cand = _tiny([0.3, np.nan, np.inf])
    with contextlib.redirect_stdout(io.StringIO()) as buf:
        assert ch.next(grid, vals, vals, cand, np.array([], int), cpl) == int(cand[0])
    assert buf.getvalue() == "Found 2 constraint violating jobs\nReceived 1 valid results\n"
    grid, vals, cpl, cand = _tiny([0.3, np.nan, 0.1])
    npr.seed(3)
    with contextlib.redirect_stdout(io.StringIO()):
        with pytest.raises(Exception, match="mcmc_iters <= 0"):
            ch.next(grid, vals, vals, cand, np.array([], int), cpl)
    after = npr.get_state()[1][:4].copy()
    npr.seed(3)
    npr.randn(10, 2)                                                   # the jitter cloud is drawn before the check
    np.testing.assert_array_equal(after, npr.get_state()[1][:4])


def test_jitter_cloud_centres_on_the_first_nan(tmp_path):
    """Quirk 8: numpy's argmin over ALL values returns the first NaN; the cloud sits on that (violating) point."""
    vals = np.array([0.5, np.nan, -1.0, 0.2])
    assert int(np.argmin(vals)) == 1
    ch = CB.init(str(tmp_path), "mcmc_iters=0")
    ch._backend = _NoBackend()
    grid = np.random.RandomState(1).rand(9, 2)
    npr.seed(5)
    jitter = npr.randn(10, 2) * 0.001
    npr.seed(5)
    seen = {}
    orig_vstack = CB.np.vstack

    def spy(arrs):
        seen.setdefault("cloud", arrs[0])
        return orig_vstack(arrs)
    CB.np.vstack = spy
    try:
        with contextlib.redirect_stdout(io.StringIO()):
            with pytest.raises(Exception, match="mcmc_iters <= 0"):
                ch.next(grid, np.r_[vals, np.zeros(5)], vals, np.arange(4, 9), np.array([], int), np.arange(4))
    finally:
        CB.np.vstack = orig_vstack
    np.testing.assert_allclose(seen["cloud"], jitter + grid[1])


def test_options_parsing_and_pickle_resume(tmp_path):
    """Quirk 12 and its waivers: pending_samples is cast to int; a visualize2D from an arg string is a non-empty str,
    hence true, and raises NotImplementedError; constraint_gain is pickled, and a pickle without it (the reference's
    own) raises KeyError('constraint_gain') on resume, as the reference's _real_init does."""
    ch = CB.init(str(tmp_path), "pending_samples=7,constraint_violating_value=-1,verbosity=0")
    assert ch.pending_samples == 7 and isinstance(ch.pending_samples, int) and ch.bad_value == -1.0
    with pytest.raises(NotImplementedError):
        CB.init(str(tmp_path), "visualize2D=0")
    with pytest.raises(TypeError):
        CB.init(str(tmp_path), "use_multiprocessing=1")                  # not an option of this chooser
    state = {"dims": 2, "ls": np.ones(2), "amp2": 1.0, "noise": 1e-3, "mean": 0.0, "constraint_ls": np.ones(2),
             "constraint_amp2": 1.0, "constraint_noise": 1e-3, "constraint_mean": 0.5}
    with open(ch.state_pkl, "wb") as fh:
        pickle.dump(state, fh)
    with pytest.raises(KeyError, match="constraint_gain"):
        ch._real_init(2, np.array([0.1, 0.2]))
    state["constraint_gain"] = 2.5
    with open(ch.state_pkl, "wb") as fh:
        pickle.dump(state, fh)
    ch._real_init(2, np.array([0.1, 0.2]))
    assert ch.constraint_gain == 2.5 and ch.needs_burnin is False
