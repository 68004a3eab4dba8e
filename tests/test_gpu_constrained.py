"""-m gpu: the constrained-EI grid pass (csrc/constraint.cu, the probability-weighted sweep, engine
constrained_ei_over_hypers) against the reference's frozen outputs (tests/golden/cons_*.npz) and the float64 oracle.

Tolerances: the float64 build of the same kernels agrees to 1e-9 (latent mean) / 1e-7 (EI) relative -- a logic check;
the float32 grid path to |dEI| <= 5e-3 * max EI per sample column with the same argmax (the plain pass's rule,
tests/test_gpu_golden.py) and |dm_c| <= 1e-4 * max|m_c| for the classification GP's latent mean."""
import numpy as np
import pytest
import scipy.stats as sps

from tests import constrained_oracle as CO
from tests.test_constrained_oracle import GOLDEN, load_case

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def engines():
    import torch
    from spearmint_b200.engine import GPEIEngine
    return {"f32": GPEIEngine(dtype=torch.float32), "f64": GPEIEngine(dtype=torch.float64)}


def _check(ei, ref, prec):
    tol_rel = 5e-3 if prec == "f32" else 1e-7
    assert ei.shape == ref.shape
    assert np.all(np.isfinite(ei))
    for s in range(ref.shape[1]):
        scale = np.abs(ref[:, s]).max()
        err = np.abs(ei[:, s] - ref[:, s]).max()
        assert err <= tol_rel * scale, (s, err, scale)
    mref = ref.mean(axis=1)
    top2 = np.sort(mref)[-2:]
    if top2[1] - top2[0] > 2 * tol_rel * np.abs(mref).max():
        assert int(np.argmax(ei.mean(axis=1))) == int(np.argmax(mref))


def synth(kind, D, N, M, S, P=0, F=1, seed=0):
    """A problem with a feasible region (x0 + x1 < 1.2: about a quarter of the cube violates) and a classification
    latent that follows it."""
    rs = np.random.RandomState(seed)
    comp, cand, pend = rs.rand(N, D), rs.rand(M, D), rs.rand(P, D)
    y = np.sin(3 * comp).sum(1)
    vals = (y - y.mean()) / y.std()
    bad = comp[:, 0] + comp[:, 1] > 1.2
    vals[bad] = np.inf
    labels = CO.labels_of(vals)
    hs = [(0.05 * rs.randn(), 1e-3, float(np.exp(0.2 * rs.randn())), rs.uniform(0.4, 2.0, D)) for _ in range(S)]
    chs = [(0.0, rs.uniform(0.5, 3.0), rs.uniform(0.5, 2.0), rs.uniform(0.3, 1.5, D)) for _ in range(S)]
    ff = np.where(bad, -1.0, 1.0) + 0.3 * rs.randn(N)
    normals = rs.randn(S, P, F) if P else None
    return hs, chs, ff, comp, labels, pend, cand, vals, normals


@pytest.mark.parametrize("path", GOLDEN, ids=[p.rsplit("/", 1)[-1] for p in GOLDEN])
@pytest.mark.parametrize("prec", ["f64", "f32"])
def test_constrained_ei_vs_reference(engines, path, prec):
    z, hs, chs, normals = load_case(path)
    ei = engines[prec].constrained_ei_over_hypers(str(z["kind"]), hs, chs, z["ff"], z["comp"], z["labels"], z["pend"],
                                                  z["cand"], z["vals"], normals)
    _check(ei, z["ei"], prec)


def test_backend_constrained_matrix_vs_reference():
    """The plugin-facing entry (DeviceBackend.constrained_ei_matrix, one process) on the pending-points golden."""
    from spearmint_b200.backend import DeviceBackend
    path = [p for p in GOLDEN if p.endswith("cons_nan_pend_d3.npz")][0]
    z, hs, chs, normals = load_case(path)
    ei = DeviceBackend().constrained_ei_matrix(str(z["kind"]), hs, chs, z["ff"], z["comp"], z["labels"], z["pend"],
                                               z["cand"], z["vals"], normals)
    _check(ei, z["ei"], "f32")


@pytest.mark.parametrize("kind", ["Matern52", "ARDSE", "Matern32", "SE"])
def test_latent_mean_and_probability(engines, kind):
    import torch
    hs, chs, ff, comp, labels, pend, cand, vals, _ = synth(kind, 5, 300, 1500, 3, seed=1)
    ref_m = np.stack([CO.constraint_mean(kind, ch, ff, comp, cand) for ch in chs])
    for prec, tol in (("f64", 1e-9), ("f32", 1e-4)):
        eng = engines[prec]
        p, m = eng.constraint_prob_device(kind, chs, ff, comp, labels, eng.to_dev(cand), want_mean=True)
        torch.cuda.synchronize()
        m = m[:, :cand.shape[0]].cpu().numpy()
        p = p[:, :cand.shape[0]].cpu().numpy()
        scale = np.abs(ref_m).max(axis=1, keepdims=True)
        assert np.all(np.abs(m - ref_m) <= tol * scale), (prec, (np.abs(m - ref_m) / scale).max())
        # p is Phi(gain m) of the device's own m, evaluated in double with an erfc tail
        gain = np.array([c[1] for c in chs])[:, None]
        np.testing.assert_allclose(p, sps.norm.cdf(gain * m), rtol=1e-12, atol=1e-300)


def test_weighted_sweep_is_ei_times_weight_into_the_deep_tail(engines):
    import torch
    eng = engines["f32"]
    M, S, F = 3000, 3, 4
    ldm = (M + 127) // 128 * 128
    rs = np.random.RandomState(2)
    dev = eng.device
    mu = torch.as_tensor(rs.uniform(-1.0, 9.0, (S, F, ldm)), dtype=torch.float32, device=dev)   # u down to about -18
    var = torch.as_tensor(rs.uniform(0.2, 0.3, (S, ldm)), dtype=torch.float32, device=dev)
    best = torch.zeros((S, F), dtype=torch.float32, device=dev)
    w = torch.as_tensor(10.0 ** rs.uniform(-250, 0, (S, ldm)), dtype=torch.float64, device=dev)   # Phi deep in its tail
    ei_w, sum_w = eng.ei_sweep_weighted(M, S, F, mu, var, ldm, best, w)
    ei_p, sum_p = eng.ei_sweep(M, S, F, mu, var, ldm, best)
    torch.cuda.synchronize()
    ei_w, ei_p, w = ei_w[:, :M].cpu().numpy(), ei_p[:, :M].cpu().numpy(), w[:, :M].cpu().numpy()
    assert np.all(ei_w > 0) and ei_w.min() < 1e-250
    np.testing.assert_allclose(ei_w, ei_p * w, rtol=1e-15, atol=0)
    np.testing.assert_allclose(sum_w[:M].cpu().numpy(), ei_w.sum(axis=0), rtol=1e-14, atol=0)


@pytest.mark.parametrize("pending", [False, True])
def test_constrained_ei_at_size(engines, pending):
    """N=512, M=10k, S=10 against the float64 oracle."""
    kind = "Matern52"
    P, F = (4, 8) if pending else (0, 1)
    hs, chs, ff, comp, labels, pend, cand, vals, normals = synth(kind, 6, 512, 10000, 10, P, F, seed=3)
    ref = CO.ei_over_hypers(kind, hs, chs, ff, comp, labels, pend, cand, vals, normals)
    ei = engines["f32"].constrained_ei_over_hypers(kind, hs, chs, ff, comp, labels, pend, cand, vals, normals)
    _check(ei, ref, "f32")


def test_constrained_ei_large_factor_on_a_candidate_subset(engines):
    """The headline's N=4096, D=32 (the tensor-core chain for the objective, a 4096-point float64 classification
    factor) on 2000 candidates."""
    import torch
    kind = "Matern52"
    hs, chs, ff, comp, labels, pend, cand, vals, _ = synth(kind, 32, 4096, 2000, 2, seed=4)
    eng = engines["f32"]
    ref_m = np.stack([CO.constraint_mean(kind, ch, ff, comp, cand) for ch in chs])
    _, m = eng.constraint_prob_device(kind, chs, ff, comp, labels, eng.to_dev(cand), want_mean=True)
    torch.cuda.synchronize()
    m = m[:, :cand.shape[0]].cpu().numpy()
    assert np.all(np.abs(m - ref_m) <= 1e-4 * np.abs(ref_m).max(axis=1, keepdims=True))
    ref = CO.ei_over_hypers(kind, hs, chs, ff, comp, labels, pend, cand, vals)
    ei = eng.constrained_ei_over_hypers(kind, hs, chs, ff, comp, labels, pend, cand, vals)
    _check(ei, ref, "f32")


def test_deep_tail_constrained_pass_ranks_like_the_oracle(engines):
    """A latent that puts the whole cube deep in the infeasible region: P(feasible) ~ Phi(-9), mean EI far below the
    deep-tail threshold, so the short-list is re-scored by the float64 build of the constrained pass (tail_fix)."""
    kind = "Matern52"
    hs, chs, ff, comp, labels, pend, cand, vals, _ = synth(kind, 4, 300, 4000, 3, seed=6)
    chs = [(c[0], 3.0, c[2], c[3]) for c in chs]
    ff = -3.0 + 0.1 * np.random.RandomState(7).randn(ff.shape[0])
    eng = engines["f32"]
    ref = CO.ei_over_hypers(kind, hs, chs, ff, comp, labels, pend, cand, vals)
    assert ref.mean(axis=1).max() < eng.TAIL_MEAN_EI
    ei = eng.constrained_ei_over_hypers(kind, hs, chs, ff, comp, labels, pend, cand, vals)
    top = np.argsort(ei.mean(axis=1))[-20:]
    np.testing.assert_allclose(ei[top], ref[top], rtol=1e-5)          # the float64 short-list
    assert int(np.argmax(ei.mean(axis=1))) == int(np.argmax(ref.mean(axis=1)))


def test_vanilla_pass_weights_by_phi_of_gain(engines):
    """No violation: EI of the plain pass times Phi(gain_s * 1) (CONS:816-842), no classification GP is built."""
    kind = "Matern52"
    hs, chs, ff, comp, labels, pend, cand, vals, _ = synth(kind, 4, 200, 3000, 3, seed=5)
    ok = labels > 0
    comp, vals, ff, labels = comp[ok], vals[ok], ff[ok], labels[ok]
    eng = engines["f32"]
    ei = eng.constrained_ei_over_hypers(kind, hs, chs, ff, comp, labels, pend, cand, vals)
    plain = eng.ei_over_hypers(kind, hs, comp, pend, cand, vals)
    gain = np.array([c[1] for c in chs])
    np.testing.assert_allclose(ei, plain * sps.norm.cdf(gain)[None, :], rtol=1e-12)
