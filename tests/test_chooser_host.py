"""CPU: host logic of the drop-in chooser (plugin API, RNG order, state files, return protocol) against golden
next() outputs of the REAL reference, with the numerics supplied by the oracle stand-in backend."""
import os
import pickle

import numpy as np
import pytest

from tests.helpers import hypers, load
from tests.oracle_backend import OracleBackend

NEXT_CASES = ["opt_branin2d", "opt_d8_m52", "opt_d8_m52_pend", "opt_d5_ardse", "opt_d4_m32_pend", "opt_d1_m52"]


def _make(g, tmp_path, **extra):
    from spearmint_b200.chooser import GPEIOptChooserB200 as mod
    args = "covar=%s,mcmc_iters=%d,burnin=%d,noiseless=%d,use_multiprocessing=0,grid_subset=5" % (
        str(g["kind"]), int(g["S"]), int(g["burnin"]), int(g["noiseless"]))
    ch = mod.init(str(tmp_path), args)
    ch._backend = OracleBackend()
    return ch


@pytest.mark.parametrize("name", NEXT_CASES)
def test_next_reproduces_reference(name, tmp_path):
    g = load(name)
    ch = _make(g, tmp_path)
    np.random.seed(int(g["seed"]))
    ret = ch.next(g["grid"], g["values"], g["durations"], g["candidates"], g["pending"], g["complete"])
    # identical hyper-parameter chain (same RNG order, float64 log-likelihood)
    ref_hs = hypers(g)
    assert len(ch.hyper_samples) == len(ref_hs)
    for a, b in zip(ch.hyper_samples, ref_hs):
        np.testing.assert_allclose(a[0], b[0], rtol=1e-9)
        np.testing.assert_allclose(a[1], b[1], rtol=1e-9)
        np.testing.assert_allclose(a[2], b[2], rtol=1e-9)
        np.testing.assert_allclose(a[3], b[3], rtol=1e-9)
    assert 0 < ch._backend.loglik_calls <= int(g["n_logprob_calls"])   # golden also counts prior-rejected evaluations
    # identical proposal
    if int(g["next_is_tuple"]):
        assert isinstance(ret, tuple) and ret[0] == int(g["next_index"])
        np.testing.assert_allclose(ret[1], g["next_point"], rtol=0, atol=1e-6)
    else:
        assert isinstance(ret, int) and ret == int(g["next_index"])


def test_state_files_and_resume(tmp_path):
    g = load("opt_branin2d")
    ch = _make(g, tmp_path)
    np.random.seed(1)
    ch.next(g["grid"], g["values"], g["durations"], g["candidates"], g["pending"], g["complete"])
    assert os.path.exists(ch.state_pkl) and os.path.exists(ch.stats_file)
    assert not os.path.exists(ch.state_pkl + ".lock")
    st = pickle.load(open(ch.state_pkl, "rb"))
    assert sorted(st) == ["amp2", "dims", "hyper_samples", "ls", "mean", "noise"]       # OPT:89-94
    assert st["dims"] == 2 and len(st["hyper_samples"]) == int(g["S"])
    txt = open(ch.stats_file).read().splitlines()
    assert txt[0] == "Mean Noise Amplitude <length scales>" and "MEAN OF SAMPLES" in txt[-2]
    # a fresh chooser on the same directory resumes: no burn-in (OPT:172-183)
    ch2 = _make(g, tmp_path)
    n0 = ch2._backend.loglik_calls
    np.random.seed(2)
    ch2.next(g["grid"], g["values"], g["durations"], g["candidates"], g["pending"], g["complete"])
    assert ch2.needs_burnin is False and ch2.D == 2
    assert "Estimated mean" in ch2.generate_stats_html()


def test_plugin_protocol_edge_cases(tmp_path):
    from spearmint_b200.chooser import GPEIOptChooserB200 as mod
    ch = mod.init(str(tmp_path), "")
    assert ch.mcmc_iters == 10 and ch.burnin == 100 and ch.grid_subset == 20 and ch.pending_samples == 100
    assert ch.noiseless is False and ch.covar == "Matern52"
    # fewer than 2 completed jobs -> first candidate, no GP (OPT:221-222); no backend is touched
    grid = np.random.RandomState(0).rand(10, 2)
    vals = np.full(10, np.nan)
    assert ch.next(grid, vals, vals, np.arange(1, 10), np.array([], dtype=int), np.array([0])) == 1
    assert ch._backend is None
    with pytest.raises(TypeError):
        mod.init(str(tmp_path), "no_such_option=1")       # **args, OPT:47
    with pytest.raises(AttributeError):
        mod.init(str(tmp_path), "covar=NoKernel")
    ch = mod.init(str(tmp_path), "mcmc_iters=3,noiseless=1,burnin=7,grid_subset=4,pending_samples=9")
    assert (ch.mcmc_iters, ch.noiseless, ch.burnin, ch.grid_subset, ch.pending_samples) == (3, True, 7, 4, 9)


def test_se_kernel_raises_like_reference(tmp_path):
    """covar=SE: the reference's refinement dies with AttributeError (gp has no grad_SE); goldens record that."""
    g = load("opt_d3_se")
    assert int(g["next_raises_attribute_error"]) == 1
    from spearmint_b200.chooser import GPEIOptChooserB200 as mod
    from spearmint_b200 import engine  # noqa: F401  (RefineContext carries the same behaviour)
    ch = mod.init(str(tmp_path), "covar=SE,mcmc_iters=2,burnin=2,grid_subset=3")

    class B(OracleBackend):
        def refine_context(self, kind, *a, **k):
            if kind == "SE":
                raise AttributeError("module 'spearmint.gp' has no attribute 'grad_SE'")
            return OracleBackend.refine_context(self, kind, *a, **k)
    ch._backend = B()
    np.random.seed(6)
    with pytest.raises(AttributeError):
        ch.next(g["grid"], g["values"], g["durations"], g["candidates"], g["pending"], g["complete"])


@pytest.mark.parametrize("name", ["psec_d4", "psec_d3_pend", "psec_d3_noiseless"])
def test_per_second_next_reproduces_reference(name, tmp_path):
    from spearmint_b200.chooser import GPEIperSecChooserB200 as mod
    g = load(name)
    ch = mod.init(str(tmp_path), "covar=%s,mcmc_iters=%d,burnin=%d,grid_subset=4,noiseless=%d" % (
        str(g["kind"]), int(g["S"]), int(g["burnin"]), int(g.get("noiseless", 0))))
    ch._backend = OracleBackend()
    np.random.seed(int(g["seed"]))
    ret = ch.next(g["grid"], g["values"], g["durations"], g["candidates"], g["pending"], g["complete"])
    for a, b in zip(ch.hyper_samples, hypers(g)):
        np.testing.assert_allclose(np.hstack(a), np.hstack(b), rtol=1e-9)
    assert len(ch.time_hyper_samples) == int(g["n_time_samples"])       # burn-in samples kept (PSEC:199)
    for a, b in zip(ch.time_hyper_samples, hypers(g, "ths")):
        np.testing.assert_allclose(np.hstack(a), np.hstack(b), rtol=1e-9)
    assert isinstance(ret, tuple) == bool(int(g["next_is_tuple"]))
    if isinstance(ret, tuple):
        assert ret[0] == int(g["next_index"])
        np.testing.assert_allclose(ret[1], g["next_point"], rtol=0, atol=1e-6)
    st = pickle.load(open(ch.state_pkl, "rb"))
    assert sorted(st) == sorted(["dims", "ls", "amp2", "noise", "mean", "time_ls", "time_amp2", "time_noise",
                                 "time_mean"])                           # PSEC:87-95


def test_per_second_gradient_oracle_matches_reference():
    from oracle import gp_oracle as O
    g = load("psec_d4")
    comp = g["grid"][g["complete"]]
    vals = g["values"][g["complete"]]
    durs = np.log(g["durations"][g["complete"]])
    hs, ths = hypers(g), hypers(g, "ths")
    S = int(g["S"])
    for x, f_ref, g_ref in zip(g["grad_pts"], g["grad_f"], g["grad_g"]):
        f, gr = O.grad_optimize_ei_per_s_over_hypers(str(g["kind"]), hs[:S], ths[:S], x, comp, vals, durs)
        np.testing.assert_allclose(f, f_ref, rtol=1e-8)
        np.testing.assert_allclose(gr, g_ref, rtol=1e-7, atol=1e-12)


def test_gpei_chooser_next_reproduces_reference(tmp_path):
    """GPEIChooser (f3): interleaved sample / fantasy-normal RNG order, argmax of the mean EI on the grid."""
    from spearmint_b200.chooser import GPEIChooserB200 as mod
    g = load("gpei_d3")
    ch = mod.init(str(tmp_path), "mcmc_iters=4")
    ch._backend = OracleBackend()
    np.random.seed(int(g["seed"]))
    ret = ch.next(g["grid"], g["values"], g["durations"], g["candidates"], g["pending"], g["complete"])
    assert isinstance(ret, int) and ret == int(g["next_index"])
    ch.dump_hypers()
    st = pickle.load(open(ch.state_pkl, "rb"))
    assert sorted(st) == ["amp2", "dims", "ls", "mean", "noise"]


def _gpei_noiseless_next(tmp_path):
    from spearmint_b200.chooser import GPEIChooserB200 as mod
    g = load("gpei_d3_noiseless")
    ch = mod.init(str(tmp_path), "mcmc_iters=4,noiseless=1")
    ch._backend = OracleBackend()
    np.random.seed(int(g["seed"]))
    ret = ch.next(g["grid"], g["values"], g["durations"], g["candidates"], g["pending"], g["complete"])
    return g, ch, ret


def test_gpei_chooser_noiseless_next_reproduces_reference(tmp_path):
    """GPEIChooser with noiseless=1: the noise stays at 1e-3 and the proposal is the reference's."""
    g, ch, ret = _gpei_noiseless_next(tmp_path)
    assert isinstance(ret, int) and ret == int(g["next_index"])
    assert ch.noise == 1e-3


@pytest.mark.xfail(strict=True, reason="the noiseless joint move bounds the mean by the observed values; the "
                                       "reference's GPEIChooser._sample_noiseless does not (GPEI:322-346)")
def test_gpei_chooser_noiseless_chain_matches_reference(tmp_path):
    g, ch, ret = _gpei_noiseless_next(tmp_path)
    np.testing.assert_allclose(np.hstack([ch.mean, ch.noise, ch.amp2, ch.ls]),
                               np.hstack([g["mean"], g["noise"], g["amp2"], g["ls"]]), rtol=1e-9)


@pytest.mark.parametrize("name", ["opt_d8_m52","opt_d4_m32_pend", "opt_branin2d"])
def test_speculative_batched_sampler_keeps_the_chain(name, tmp_path):
    """The GPU log-likelihood batches the points a slice move will visit (peeked RNG).  That must not change the chain:
    same hyper-samples, same proposal, same final RNG state as the sequential path, with far fewer sequential calls."""
    g = load(name)
    outs = []
    # False: sequential; (3, 0): everything speculated up front (latency-bound sizes); (0, 2), (1, 3): the two-phase
    # schedule of flop-bound sizes (interval ends first, shrink proposals in small groups afterwards)
    for i, batched in enumerate((False, (3, 0), (0, 2), (1, 3))):
        d = tmp_path / ("b%d" % i)
        d.mkdir()
        ch = _make(g, d)
        ch._backend = OracleBackend(batched=bool(batched), speculate=batched or None)
        np.random.seed(int(g["seed"]))
        ret = ch.next(g["grid"], g["values"], g["durations"], g["candidates"], g["pending"], g["complete"])
        outs.append((ch.hyper_samples, ret, np.random.rand(), ch._backend))
    hs0, r0, u0, b0 = outs[0]
    for hs1, r1, u1, b1 in outs[1:]:
        for a, b in zip(hs0, hs1):
            np.testing.assert_array_equal(np.hstack(a), np.hstack(b))
        assert u0 == u1
        assert (r0[0], tuple(r0[1])) == (r1[0], tuple(r1[1])) if isinstance(r0, tuple) else r0 == r1
    assert outs[1][3].batches < 0.5 * b0.loglik_calls          # sequential depth at least halved
    assert outs[2][3].loglik_calls < outs[1][3].loglik_calls   # the two-phase schedule wastes fewer evaluations


@pytest.mark.parametrize("name", ["mll_d3_m52", "mll_d5_ardse", "mll_d2_m32"])
def test_gpei_ml2_branch_host_logic(name, tmp_path):
    """GPEIChooserB200 with mcmc_iters=0 (GPEI:156-176, 348-361) on the oracle backend: same optimum, same proposal as the
    reference's next()."""
    from spearmint_b200.chooser import GPEIChooserB200 as mod
    g = load(name)
    ch = mod.init(str(tmp_path), "covar=%s,mcmc_iters=0" % str(g["kind"]))
    ch._backend = OracleBackend()
    np.random.seed(5)
    ret = ch.next(g["grid"], g["values"], None, g["candidates"], np.array([], dtype=int), g["complete"])
    assert ret == int(g["next_index"])
    np.testing.assert_allclose(np.hstack([ch.mean, ch.noise, ch.amp2, ch.ls]), g["next_hypers"], rtol=1e-6)
