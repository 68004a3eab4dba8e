"""The oracle against outputs of the reference on the same inputs, frozen in tests/golden/oracle_vs_reference.npz by
tests/golden/make_golden_oracle_vs_reference.py (which executes the reference through oracle/ref_shim.py).  The golden
fixtures of test_oracle_golden.py pin the chooser-level functions; this file pins the kernels, the log-probability,
compute_ei with and without pending points, the Sobol generator and the ML-II optimum."""
import os

import numpy as np
import pytest

from oracle import gp_oracle as O


@pytest.fixture(scope="module")
def G(golden_dir):
    return np.load(os.path.join(golden_dir, "oracle_vs_reference.npz"))


@pytest.mark.parametrize("kind", ["SE", "ARDSE", "Matern32", "Matern52"])
def test_kernels_and_logprob(G, kind):
    comp, cand, vals, ls = G["k_comp"], G["k_cand"], G["k_vals"], G["k_ls"]
    np.testing.assert_allclose(O.kernel(kind, ls, comp), G["K_%s" % kind], rtol=1e-12, atol=1e-14)
    np.testing.assert_allclose(O.kernel(kind, ls, comp, cand), G["Kx_%s" % kind], rtol=1e-12, atol=1e-14)
    lp = O.gp_logprob(kind, float(G["k_mean"]), float(G["k_noise"]), float(G["k_amp2"]), ls, comp, vals)
    np.testing.assert_allclose(lp, float(G["logprob_%s" % kind]), rtol=1e-11)


def test_compute_ei_with_and_without_pending(G):
    comp, cand, vals = G["ei_comp"], G["ei_cand"], G["ei_vals"]
    mean, noise, amp2 = (float(x) for x in G["ei_hyper"])
    h = (mean, noise, amp2, G["ei_ls"])
    D = comp.shape[1]
    np.testing.assert_allclose(O.compute_ei("Matern52", h, comp, np.zeros((0, D)), cand, vals), G["ei_nopend"],
                               rtol=1e-9, atol=1e-14)
    np.testing.assert_allclose(O.compute_ei("Matern52", h, comp, G["ei_pend"], cand, vals, G["ei_normals"]),
                               G["ei_withpend"], rtol=1e-9, atol=1e-14)


def test_sobol_and_optimize_hypers(G):
    from oracle import sobol_oracle as SO
    assert np.array_equal(SO.i4_sobol_generate(6, 50, 2), G["sobol_6_50_2"])
    m, noise, amp2, ls = O.gp_optimize_hypers("Matern52", G["ml_comp"], G["ml_vals"])
    np.testing.assert_allclose([m, noise, amp2], G["ml_hyper"], rtol=1e-6)
    np.testing.assert_allclose(ls, G["ml_ls"], rtol=1e-6)
