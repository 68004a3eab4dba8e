"""TEST-ONLY stand-in for the constrained-chooser part of spearmint_b200.backend.DeviceBackend, built on the CPU oracle
(tests/constrained_oracle.py), so that GPConstrainedEIChooserB200's host logic -- RNG order, state files, stdout, return
protocol, the reference's quirks -- is checked without a GPU.  Never used by the product."""
import numpy as np

from tests import constrained_oracle as CO
from tests.oracle_backend import OracleBackend


class _Factor(object):
    def __init__(self, L):
        self.L = L

    def draw(self, z):
        return np.dot(self.L, np.ravel(z))


class ConstrainedOracleBackend(OracleBackend):
    name = "oracle"

    def latent_loglik(self, kind, comp, ls, noise):
        def ll(amp2, ff):
            return CO.latent_loglik(kind, amp2, ls, ff, comp, noise)
        return ll

    def latent_factor(self, kind, comp, amp2, ls, noise):
        return _Factor(CO.latent_factor(kind, amp2, ls, comp, noise))

    def constraint_predict(self, kind, chyper, ff, comp, cand):
        return CO.constraint_prob(kind, chyper, ff, comp, cand, np.array([0.0, 1.0]))

    def constrained_ei_matrix(self, kind, hyper_samples, chyper_samples, ff, comp, labels, pend, cand, vals,
                              normals=None):
        return CO.ei_over_hypers(kind, hyper_samples, chyper_samples, ff, comp, labels, pend, cand, vals, normals)

    def constrained_refine_context(self, kind, hyper_samples, chyper_samples, ff, comp, labels, pend, vals,
                                   normals=None, noise=1e-3):
        if kind == "SE":
            raise AttributeError("module 'spearmint.gp' has no attribute 'grad_SE'")

        class Ctx(object):
            evals = 0

            def value_grad(self, x):
                self.evals += 1
                return CO.grad_optimize_ei_over_hypers(kind, hyper_samples, chyper_samples, ff, x, comp, labels, pend,
                                                       vals, normals, noise)
        return Ctx()
