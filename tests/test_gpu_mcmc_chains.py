"""-m gpu: mcmc_chains on the device -- smk_loglik_small_f64 (the one-launch log-likelihood of N <= 238) against the
oracle and against the batched LogLik path, its non positive definite items, its batch independence and argument codes;
K lockstep chains against the same chains run separately, on both log-likelihood paths; next() with mcmc_chains=4
against the same chooser on the oracle."""
import numpy as np
import pytest
import torch

from oracle import gp_oracle as O
from tests.helpers import U64, cur_stream, data, lib, load, synth_hypers

pytestmark = pytest.mark.gpu

KINDS = ("SE", "ARDSE", "Matern32", "Matern52")
MAX_N = 238                       # SMK_LOGLIK_SMALL_MAX_N


@pytest.fixture(scope="module")
def eng():
    from spearmint_b200.engine import GPEIEngine
    return GPEIEngine(device="cuda:0", dtype=torch.float64)


def _small(eng, kind, X, y, hs):
    """(sum_log_diag, quad, info) of smk_loglik_small_f64 for the items ``hs``."""
    from spearmint_b200._lib import KINDS as K, check, ptr
    B = len(hs)
    hb = eng.hypers(hs, kind)
    Xd, yd = eng.to_dev(X), eng.to_dev(y)
    out = torch.full((2, B), -7.0, dtype=torch.float64, device=eng.device)
    info = torch.full((B,), -7, dtype=torch.int32, device=eng.device)
    check(lib().smk_loglik_small_f64(K[kind], X.shape[0], X.shape[1], B, ptr(Xd), ptr(hb.inv_ls), ptr(hb.amp2),
                                     ptr(hb.noise), ptr(hb.mean), ptr(yd), ptr(out[0]), ptr(out[1]), ptr(info),
                                     cur_stream()), "loglik_small")
    torch.cuda.synchronize()
    return out[0].cpu().numpy(), out[1].cpu().numpy(), info.cpu().numpy()


def _lp(sld, quad):
    return -sld - 0.5 * quad


@pytest.mark.parametrize("kind", KINDS)
def test_small_kernel_matches_oracle(eng, kind):
    """Within the 1e-10 (relative, 1e-9 absolute) the float64 log-likelihood is held to against the reference."""
    for D in (1, 8, 32):
        for N in (1, 2, 31, 32, 33, 127, 128, 200, MAX_N):
            X, y, rs = data(N, D, 100 * N + D)
            hs = synth_hypers(rs, 3, D, 1e-2) + synth_hypers(rs, 1, D, 1e-3)
            sld, quad, info = _small(eng, kind, X, y, hs)
            assert not info.any()
            for b, h in enumerate(hs):
                ref = O.gp_logprob(kind, h[0], h[1], h[2], np.asarray(h[3], float), X, y)
                np.testing.assert_allclose(_lp(sld[b], quad[b]), ref, rtol=1e-10, atol=1e-9,
                                           err_msg="%s D=%d N=%d item %d" % (kind, D, N, b))


def _first_order_bound(kind, X, y, h):
    """A-priori bound on |lp_a - lp_b| for two backward-stable Cholesky factorisations of the same augmented matrix
    (identical covariance entries: both build them with the same staged products and kernel code).  Each computed
    factor satisfies L L' = A + E with |E| <= gamma_{n+1} |L||L'| (n = N + 1), which moves
        sum log diag by   1/2 tr(A^-1 E)                 <= 1/2 gamma sum(|A^-1| o |L||L'|),
        quad         by   a' E a  (a = A^-1 r)           <= gamma |a|' |L||L'| |a|,
    to first order; the two paths are each within that of the exact value, hence the factor 2 (and 0.5 on quad)."""
    N = X.shape[0]
    ls = np.ones(X.shape[1]) if kind == "SE" else np.asarray(h[3], float)
    r2 = (((X[:, None, :] - X[None, :, :]) / ls) ** 2).sum(-1)
    from tests.helpers import kern
    A = h[2] * (kern(kind, r2) + 1e-6 * np.eye(N)) + h[1] * np.eye(N)
    L = np.linalg.cholesky(A)
    LL = np.abs(L).dot(np.abs(L).T)
    r = y - h[0]
    a = np.linalg.solve(A, r)
    g = (N + 2) * U64 / (1 - (N + 2) * U64)
    return 2 * (0.5 * g * (np.abs(np.linalg.inv(A)) * LL).sum() + 0.5 * g * np.abs(a).dot(LL).dot(np.abs(a)))


def test_small_kernel_matches_batched_path(eng):
    """Against LogLik.batch (cov_build_lower -> set_rhs -> potrf_loglik -> finish) within the first-order bound above.
    Worst measured ratio |difference| / bound: 1.9e-3 (H100 80 GB HBM3)."""
    worst = 0.0
    for kind in ("SE", "Matern52"):
        for N in (31, 128, MAX_N):
            X, y, rs = data(N, 8, N)
            hs = synth_hypers(rs, 4, 8, 1e-3)
            sld, quad, info = _small(eng, kind, X, y, hs)
            ref = eng.loglik(kind, X, y).batch(hs)
            for b, h in enumerate(hs):
                diff = abs(_lp(sld[b], quad[b]) - ref[b])
                bound = _first_order_bound(kind, X, y, h)
                worst = max(worst, diff / bound)
                assert diff <= bound, (kind, N, b, diff, bound)
    print("worst |small - batched| / bound = %.3g" % worst)


def test_non_pd_item_gives_info_and_nan_like_the_batched_path(eng):
    from spearmint_b200.engine import ChainLogLik
    X, y, rs = data(100, 4, 3)
    hs = synth_hypers(rs, 3, 4, 1e-2)
    bad = (hs[1][0], -10.0 * hs[1][2], hs[1][2], hs[1][3])           # noise far below -amp2: the first pivot fails
    items = [hs[0], bad, hs[2]]
    sld, quad, info = _small(eng, "Matern52", X, y, items)
    ll = eng.loglik("Matern52", X, y)
    ref = ll.batch(items)
    assert info[1] == int(ll.info[1].item()) == 1 and info[0] == info[2] == 0
    assert np.isnan(sld[1]) and np.isnan(quad[1])
    got = ChainLogLik(eng, "Matern52", X, y, 2).batch(items)
    assert np.isnan(got[1]) and np.isnan(ref[1])
    assert np.isfinite(got[[0, 2]]).all()
    alone = ChainLogLik(eng, "Matern52", X, y, 2).batch([hs[2]])
    assert alone[0] == got[2]
    with pytest.raises(np.linalg.LinAlgError):
        ChainLogLik(eng, "Matern52", X, y, 2)(*bad)


def test_small_kernel_is_batch_independent(eng):
    """One item alone and inside batches of 1-64 at several positions: bitwise the same."""
    X, y, rs = data(150, 6, 5)
    probe = synth_hypers(rs, 1, 6, 1e-2)[0]
    s0, q0, _ = _small(eng, "Matern32", X, y, [probe])
    for B in (1, 2, 7, 33, 64):
        for pos in sorted({0, B // 2, B - 1}):
            hs = synth_hypers(rs, B, 6, 1e-2)
            hs[pos] = probe
            s, q, info = _small(eng, "Matern32", X, y, hs)
            assert s[pos] == s0[0] and q[pos] == q0[0] and info[pos] == 0, (B, pos)


def test_small_kernel_argument_codes(eng):
    X, y, rs = data(10, 3, 1)
    hb = eng.hypers(synth_hypers(rs, 2, 3, 1e-2), "Matern52")
    Xd, yd = eng.to_dev(X), eng.to_dev(y)
    out = torch.zeros((2, 2), dtype=torch.float64, device=eng.device)
    info = torch.zeros((2,), dtype=torch.int32, device=eng.device)
    from spearmint_b200._lib import ptr
    args = [3, 10, 3, 2, ptr(Xd), ptr(hb.inv_ls), ptr(hb.amp2), ptr(hb.noise), ptr(hb.mean), ptr(yd), ptr(out[0]),
            ptr(out[1]), ptr(info), cur_stream()]
    f = lib().smk_loglik_small_f64
    assert f(*args) == 0
    torch.cuda.synchronize()
    for pos, bad in ((0, -1), (0, 4), (1, 0), (1, MAX_N + 1), (2, 0), (3, 0)):
        a = list(args)
        a[pos] = bad
        assert f(*a) == -(pos + 1), (pos, bad)
    for pos in range(4, 13):
        a = list(args)
        a[pos] = None
        assert f(*a) == -(pos + 1), pos
    Xb, yb = eng.to_dev(data(MAX_N, 3, 2)[0]), eng.to_dev(np.zeros(MAX_N))     # the largest N runs
    a = list(args)
    a[1], a[4], a[9] = MAX_N, ptr(Xb), ptr(yb)
    assert f(*a) == 0
    torch.cuda.synchronize()
    assert not info.cpu().numpy().any()


@pytest.mark.parametrize("N", [100, 600])
def test_lockstep_chains_equal_separate_chains(eng, N):
    """K = 4 chains sharing rounds vs each chain with a handle of its own: bitwise the same samples.  N = 100 runs the
    one-launch kernel, N = 600 the batched factorisation (one graph per batch size)."""
    from spearmint_b200 import chains
    from spearmint_b200.chooser.GPEIOptChooserB200 import GPEIOptChooserB200 as Ch
    from spearmint_b200.engine import ChainLogLik
    X, y, _ = data(N, 4, N)
    K = 4
    start = (0.0, 1e-3, 1.0, np.ones(4))

    def fresh():
        np.random.seed(N)
        return chains.Chain.seeded(K, start)
    together = fresh()
    ll = ChainLogLik(eng, "Matern52", X, y, K)
    assert ll.small == (N <= MAX_N)
    ev = [0] * K
    chains.lockstep([c.run(Ch.prior, y, False, 2, 2, ll.speculate) for c in together], ll, ev)
    for c in range(K):
        alone = fresh()[c]
        ll1 = ChainLogLik(eng, "Matern52", X, y, 1)
        ev1 = [0]
        chains.lockstep([alone.run(Ch.prior, y, False, 2, 2, ll1.speculate)], ll1, ev1)
        assert ev1[0] == ev[c]
        for a, b in zip(alone.samples, together[c].samples):
            np.testing.assert_array_equal(np.hstack(a), np.hstack(b))


@pytest.mark.parametrize("name", ["opt_d8_m52", "opt_d8_m52_pend", "opt_d5_ardse"])
def test_next_with_four_chains_matches_oracle_backend(name, tmp_path):
    """next() with mcmc_chains=4 on the GPU against the same chooser on the oracle: the chains within rtol 1e-6 and the
    proposal within atol 2e-4 (the tolerances of the single-chain next() tests)."""
    from spearmint_b200.backend import DeviceBackend
    from spearmint_b200.chooser import GPEIOptChooserB200 as mod
    from tests.oracle_backend import OracleBackend

    class ChainOracle(OracleBackend):
        def __init__(self):
            OracleBackend.__init__(self, batched=True)

        def loglik(self, kind, comp, vals, chains=1):
            return OracleBackend.loglik(self, kind, comp, vals)

    g = load(name)
    args = "covar=%s,mcmc_iters=4,burnin=%d,noiseless=%d,grid_subset=5,mcmc_chains=4" % (
        str(g["kind"]), int(g["burnin"]), int(g["noiseless"]))
    outs = []
    for i, be in enumerate((DeviceBackend(), ChainOracle())):
        d = tmp_path / str(i)
        d.mkdir()
        ch = mod.init(str(d), args)
        ch._backend = be
        np.random.seed(int(g["seed"]))
        ret = ch.next(g["grid"], g["values"], g["durations"], g["candidates"], g["pending"], g["complete"])
        outs.append((ret, ch.hyper_samples))
    (r0, h0), (r1, h1) = outs
    for a, b in zip(h0, h1):
        np.testing.assert_allclose(np.hstack(a), np.hstack(b), rtol=1e-6, atol=1e-9)
    p0 = r0[1] if isinstance(r0, tuple) else g["grid"][r0]
    p1 = r1[1] if isinstance(r1, tuple) else g["grid"][r1]
    np.testing.assert_allclose(p0, p1, rtol=0, atol=2e-4)
