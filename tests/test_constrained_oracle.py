"""CPU: the constrained-EI oracle (tests/constrained_oracle.py) against the reference's own grid pass, frozen in
tests/golden/cons_*.npz by tests/golden/make_golden_constrained.py."""
import glob
import os

import numpy as np
import pytest
import scipy.stats as sps

from tests import constrained_oracle as CO

GOLDEN = sorted(p for p in glob.glob(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "cons_*.npz"))
                if not os.path.basename(p).startswith("cons_next_"))      # grid-pass cases; next() runs: test_constrained_chooser


def load_case(path):
    z = np.load(path)
    S = z["gain"].shape[0]
    hs = [(z["mean"][s], z["noise"][s], z["amp2"][s], z["ls"][s]) for s in range(S)]
    chs = [(z["cmean"][s], z["gain"][s], z["camp2"][s], z["cls"][s]) for s in range(S)]
    P, F = z["pend"].shape[0], int(z["F"])
    normals = None
    if P:
        rs = np.random.RandomState(int(z["seed"]))          # the global RNG, drawn anew per sample (CONS:910)
        normals = np.stack([rs.randn(P, F) for _ in range(S)])
    return z, hs, chs, normals


def test_goldens_cover_the_cases():
    names = {os.path.basename(p) for p in GOLDEN}
    assert {"cons_inf_d2.npz", "cons_nan_pend_d3.npz", "cons_vanilla.npz", "cons_m32_badval.npz"} <= names


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p) for p in GOLDEN])
def test_oracle_matches_reference_grid_pass(path):
    z, hs, chs, normals = load_case(path)
    labels = CO.labels_of(z["vals"], float(z["bad_value"]))
    np.testing.assert_array_equal(labels, z["labels"])
    ei = CO.ei_over_hypers(str(z["kind"]), hs, chs, z["ff"], z["comp"], labels, z["pend"], z["cand"], z["vals"], normals)
    np.testing.assert_allclose(ei, z["ei"], rtol=1e-9, atol=1e-12 * np.abs(z["ei"]).max())


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p) for p in GOLDEN])
def test_oracle_constraint_prob_matches_reference(path):
    z, hs, chs, _ = load_case(path)
    for s, ch in enumerate(chs):      # pred_constraint_voilation (CONS:425-447): the classification GP's mean, squashed
        p = sps.norm.cdf(ch[1] * CO.constraint_mean(str(z["kind"]), ch, z["ff"], z["comp"], z["cand"]))
        np.testing.assert_allclose(p, z["prob"][s], rtol=1e-9, atol=1e-14)


def test_vanilla_weights_every_candidate_by_phi_of_gain():
    """Quirk of CONS:816-842: with no violation the grid pass still multiplies EI by Phi(gain_s * 1)."""
    z, hs, chs, _ = load_case([p for p in GOLDEN if p.endswith("cons_vanilla.npz")][0])
    assert CO.is_vanilla(z["labels"])
    plain = np.stack([CO.G.compute_ei(str(z["kind"]), h, z["comp"], z["pend"], z["cand"], z["vals"]) for h in hs], 1)
    np.testing.assert_allclose(z["ei"], plain * sps.norm.cdf(z["gain"])[None, :], rtol=1e-9)


def test_violations_are_nan_inf_and_the_user_value():
    vals = np.array([0.5, np.nan, np.inf, -np.inf, 7.0, -1.0])
    np.testing.assert_array_equal(CO.labels_of(vals), [1, 0, 0, 0, 1, 1])
    np.testing.assert_array_equal(CO.labels_of(vals, 7.0), [1, 0, 0, 0, 0, 1])


def refine_normals(z):
    """The fantasy block of the refinement: randomstate = RandomState(seed + 100) (make_golden_constrained.py)."""
    P = z["pend"].shape[0]
    return np.random.RandomState(int(z["seed"]) + 100).randn(P, max(int(z["F"]), 1)) if P else None


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p) for p in GOLDEN])
def test_oracle_refinement_objective_matches_reference(path):
    """grad_optimize_ei_over_hypers (CONS:471-803) at 3 points: the half-scaled gradients, the variance from all points
    (no pending) and the sum over fantasies (pending) are the reference's."""
    z, hs, chs, _ = load_case(path)
    for x, f_ref, g_ref in zip(z["fg_x"], z["fg_f"], z["fg_g"]):
        f, g = CO.grad_optimize_ei_over_hypers(str(z["kind"]), hs, chs, z["ff"], x, z["comp"], z["labels"], z["pend"],
                                               z["vals"], refine_normals(z))
        np.testing.assert_allclose(f, f_ref, rtol=1e-9)
        np.testing.assert_allclose(g, g_ref, rtol=1e-8, atol=1e-12 * np.abs(g_ref).max())
