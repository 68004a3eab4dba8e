"""-m gpu: the classification-GP pieces of the constrained chooser on the device, and GPConstrainedEIChooserB200 on
DeviceBackend against whole next() runs of the reference (tests/golden/cons_next_*.npz): chains to rtol 1e-6, the
proposal to atol 2e-4 (the rule of the other choosers' next() tests)."""
import numpy as np
import pytest
import scipy.linalg as spla

from tests import constrained_oracle as CO
from tests.test_constrained_chooser import GOLDEN_NEXT, IDS, check_against_golden, run_plugin
from tests.test_constrained_oracle import GOLDEN, load_case, refine_normals

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def backend():
    from spearmint_b200.backend import DeviceBackend
    return DeviceBackend()


def _problem(N=300, D=4, seed=0):
    rs = np.random.RandomState(seed)
    comp = rs.rand(N, D)
    labels = (comp[:, 0] + comp[:, 1] < 1.2).astype(float)
    return comp, labels, rs


@pytest.mark.parametrize("kind", ["Matern52", "ARDSE", "SE"])
def test_latent_loglik_batch_each_item_its_own_ff(backend, kind):
    comp, labels, rs = _problem()
    ls = rs.uniform(0.3, 1.5, comp.shape[1])
    ll = backend.latent_loglik(kind, comp, ls, 1e-3)
    items = [(rs.uniform(0.3, 3.0), np.where(labels > 0, 1.0, -1.0) + rs.randn(comp.shape[0])) for _ in range(7)]
    got = ll.batch(items)
    ref = np.array([CO.latent_loglik(kind, a, np.ones_like(ls) if kind == "SE" else ls, f, comp) for a, f in items])
    np.testing.assert_allclose(got, ref, rtol=1e-10)
    assert abs(ll(*items[3]) - ref[3]) <= 1e-10 * abs(ref[3])


def test_latent_factor_draw(backend):
    comp, labels, rs = _problem(N=500)
    ls = rs.uniform(0.3, 1.5, comp.shape[1])
    for noise in (1e-6, 1e-3):
        fac = backend.latent_factor("Matern52", comp, 1.7, ls, noise)
        z = rs.randn(comp.shape[0], 1)
        ref = np.dot(CO.latent_factor("Matern52", 1.7, ls, comp, noise), z).ravel()
        np.testing.assert_allclose(fac.draw(z), ref, rtol=0, atol=1e-12 * np.abs(ref).max())


@pytest.mark.parametrize("path", GOLDEN, ids=[p.rsplit("/", 1)[-1] for p in GOLDEN])
def test_refine_value_grad_vs_reference(backend, path):
    """(f, g) of the refinement at the golden's 3 points: f to 1e-7, g to 1e-6 of its largest entry."""
    z, hs, chs, _ = load_case(path)
    ctx = backend.constrained_refine_context(str(z["kind"]), hs, chs, z["ff"], z["comp"], z["labels"], z["pend"],
                                             z["vals"], refine_normals(z))
    for x, f_ref, g_ref in zip(z["fg_x"], z["fg_f"], z["fg_g"]):
        f, g = ctx.value_grad(x)
        assert abs(f - f_ref) <= 1e-7 * abs(f_ref), (f, f_ref)
        assert np.abs(g - g_ref).max() <= 1e-6 * np.abs(g_ref).max(), (g, g_ref)


def test_constraint_predict_is_the_classification_gp_even_without_violations(backend):
    comp, labels, rs = _problem(N=200)
    cand = rs.rand(500, comp.shape[1])
    ch = (0.5, 1.7, 1.2, rs.uniform(0.3, 1.5, comp.shape[1]))
    ff = rs.randn(comp.shape[0])
    ref_m = CO.constraint_mean("Matern52", ch, ff, comp, cand)
    ref = CO.constraint_prob("Matern52", ch, ff, comp, cand, np.array([0.0, 1.0]))
    # the float32 grid path: |dm_c| <= 1e-4 max|m_c|, so |dp| <= gain phi(0) 1e-4 max|m_c|
    tol = ch[1] * 0.4 * 1e-4 * np.abs(ref_m).max()
    np.testing.assert_allclose(backend.constraint_predict("Matern52", ch, ff, comp, cand), ref, rtol=0, atol=tol)


@pytest.mark.parametrize("path", GOLDEN_NEXT, ids=IDS)
def test_next_reproduces_the_reference_on_the_gpu(backend, path, tmp_path):
    z, out, ncalls = run_plugin(path, backend, tmp_path)
    check_against_golden(z, out, ncalls, rtol=1e-6, atol_point=2e-4)


def test_constrained_pass_validates_its_arguments(backend):
    """Pending points without fantasy normals, mismatched sample lists or an ff of the wrong length are refused up
    front with a ValueError naming the problem."""
    eng = backend.eng32
    comp, labels, rs = _problem(N=50)
    vals = np.where(labels > 0, rs.randn(50), np.inf)
    cand, pend = rs.rand(100, comp.shape[1]), rs.rand(2, comp.shape[1])
    hs = [(0.0, 1e-3, 1.0, np.ones(comp.shape[1]))] * 2
    chs = [(0.0, 1.0, 1.0, np.ones(comp.shape[1]))] * 2
    ff = rs.randn(50)
    with pytest.raises(ValueError, match="fantasy normals"):
        eng.constrained_ei_over_hypers("Matern52", hs, chs, ff, comp, labels, pend, cand, vals, None)
    with pytest.raises(ValueError, match="fantasy normals"):
        eng.constrained_ei_over_hypers("Matern52", hs, chs, ff, comp, labels, pend, cand, vals, rs.randn(2, 4))
    with pytest.raises(ValueError, match="constraint hyper-samples"):
        eng.constrained_ei_over_hypers("Matern52", hs, chs[:1], ff, comp, labels, pend[:0], cand, vals)
    with pytest.raises(ValueError, match="ff has"):
        eng.constrained_ei_over_hypers("Matern52", hs, chs, ff[:-1], comp, labels, pend[:0], cand, vals)
