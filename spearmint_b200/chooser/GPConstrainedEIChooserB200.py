"""Drop-in replacement for the reference's ``chooser/GPConstrainedEIChooser.py`` (CONS): expected improvement times the
probability of feasibility under a probit classification GP, for experiments whose jobs fail or report ``NaN``, ``inf``
or a chosen ``constraint_violating_value``.

Same plugin API, option names, state files (``<expt_dir>/<module>.pkl``, ``<module>_hyperparameters.txt``), use of
the process-global numpy RNG in the same order, stdout lines and return protocol as the reference.  Where the arithmetic
runs (``spearmint_b200.backend.DeviceBackend``):
  * objective chain     : host slice sampler, float64 log-likelihood on the GPU (as GPEIOptChooserB200)
  * classification chain: host slice / elliptical-slice control flow and the O(N) probit term; the joint [amp2, ff]
                          log-likelihood (one right-hand side per batch item) and the elliptical-slice directions
                          nu = L z from float64 factors on the GPU
  * grid passes         : constrained EI of every candidate for all sample pairs in one batched pass
  * refinement          : L-BFGS-B on the host, (f, g) from cached factors on the GPU, serially in this process

Reference behaviour kept on purpose (DESIGN section 9): the constraint samples and latents of the grid passes and the
refinement are the FIRST ``mcmc_iters`` ever drawn, the latent of sample ``mcmc_iters - 1`` is used for every sample
and is where the next call's chain continues (CONS:264, 291-299, 1017-1018); the grid pass weights by Phi(gain) when
no violation has been seen, the refinement does not; the refinement takes its variance from ALL complete points and
sums over fantasies; the second grid pass scores the refined AND the unrefined short-list; the jitter cloud centres on
``argmin`` of all values (the first NaN if there is one).  Waived: ``pending_samples`` is cast to int, a truthy
``visualize2D`` raises NotImplementedError (no plotting), ``constraint_gain`` is written to the pickle, factorisations
whose result the reference never uses are skipped.  Extra optional keys: ``device``, ``refine_dtype``, ``grid_dtype``,
``state_name``.
"""
import math

import numpy as np
import numpy.random as npr
import scipy.optimize as spo
import scipy.stats as sps

from spearmint_b200 import util
from spearmint_b200.chooser._gp import GPChooser, GPPrior, write_state, write_stats
from spearmint_b200.locker import log


def init(expt_dir, arg_string):
    args = util.unpack_args(arg_string)
    return GPConstrainedEIChooserB200(expt_dir, **args)


def probit_loglik(ff, gain, labels):
    """sum of the probit log-likelihood of the labels under the latent ff (CONS:1152-1160), probabilities clipped."""
    probs = sps.norm.cdf(ff * gain)
    probs[probs <= 0] = 1e-12
    probs[probs >= 1] = 1 - 1e-12
    return np.sum(labels * np.log(probs) + (1 - labels) * np.log(1 - probs))


def elliptical_slice(xx, factor, log_like_fn):
    """One elliptical-slice step (CONS:1234-1281, angle_range 0).  RNG order: randn(D, 1) for the direction, rand() for
    the slice height, rand() for the first angle, one rand() per shrink."""
    D = xx.shape[0]
    cur_log_like = log_like_fn(xx)
    nu = factor.draw(npr.randn(D, 1))
    hh = np.log(npr.rand()) + cur_log_like
    phi = npr.rand() * 2 * math.pi
    phi_min, phi_max = phi - 2 * math.pi, phi
    while True:
        xx_prop = xx * np.cos(phi) + nu * np.sin(phi)
        cur_log_like = log_like_fn(xx_prop)
        if cur_log_like > hh:
            return xx_prop, cur_log_like
        if phi > 0:
            phi_max = phi
        elif phi < 0:
            phi_min = phi
        else:
            raise Exception("BUG DETECTED: Shrunk to current position and still not acceptable.")
        phi = npr.rand() * (phi_max - phi_min) + phi_min


class GPConstrainedEIChooserB200(GPChooser):
    prior = GPPrior(max_ls=2, noise_times_amp2=True)      # K = amp2 (k + 1e-6 I + noise I) in the joint move only

    def __init__(self, expt_dir, covar="Matern52", mcmc_iters=20, pending_samples=100, noiseless=False, burnin=100,
                 grid_subset=20, constraint_violating_value=np.inf, verbosity=0, visualize2D=False, device=None,
                 refine_dtype="float64", state_name=None, backend=None, grid_dtype="float32"):
        GPChooser.__init__(self, expt_dir, covar, mcmc_iters, pending_samples, noiseless, state_name, device, backend,
                           refine_dtype, grid_dtype)
        if visualize2D:      # an arg string hands over a non-empty str, which the reference treats as true (CONS:308)
            raise NotImplementedError("visualize2D: the 2-D contour plots of the reference are not provided")
        self.burnin = int(burnin)
        self.needs_burnin = True
        self.grid_subset = int(grid_subset)
        self.hyper_samples = []
        self.constraint_hyper_samples = []
        self.ff = None
        self.ff_samples = []
        self.verbosity = int(verbosity)
        self.constraint_noise_scale = 0.1
        self.constraint_amp2_scale = 1
        self.constraint_gain = 1
        self.constraint_max_ls = 2
        self.bad_value = float(constraint_violating_value)
        self.visualize2D = visualize2D

    # ------------------------------------------------------------------ state files (CONS:101-191)
    def dump_hypers(self):
        write_state(self.locker, self.state_pkl,
                    {"dims": self.D, "ls": self.ls, "amp2": self.amp2, "noise": self.noise, "mean": self.mean,
                     "constraint_ls": self.constraint_ls, "constraint_amp2": self.constraint_amp2,
                     "constraint_noise": self.constraint_noise, "constraint_mean": self.constraint_mean,
                     "constraint_gain": self.constraint_gain})
        write_stats(self.stats_file, self.hyper_samples)

    def _real_init(self, dims, values):
        self.randomstate = npr.get_state()
        state = self._read_state()
        if state is not None:
            self._load_hypers(state)
            self.constraint_ls = state["constraint_ls"]
            self.constraint_amp2 = state["constraint_amp2"]
            self.constraint_noise = state["constraint_noise"]
            self.constraint_mean = state["constraint_mean"]
            self.constraint_gain = state["constraint_gain"]     # KeyError on the reference's own pickle, as CONS:161
            self.needs_burnin = False
        else:
            goodvals = np.nonzero(np.logical_and(values != self.bad_value, np.isfinite(values)))[0]
            self._init_hypers(dims, values[goodvals])
            self.constraint_ls = np.ones(self.D)
            self.constraint_amp2 = 1.0
            self.constraint_noise = 1e-3
            self.constraint_gain = 1
            self.constraint_mean = 0.5

    # ------------------------------------------------------------------ the plugin entry point (CONS:203-422)
    def next(self, grid, values, durations, candidates, pending, complete):
        if complete.shape[0] < 2:
            return int(candidates[0])
        comp = grid[complete, :]
        cand = grid[candidates, :]
        pend = grid[pending, :]
        vals = values[complete]

        idx = np.logical_and(vals != self.bad_value, np.isfinite(vals))
        goodvals = np.nonzero(idx)[0]
        badvals = np.nonzero(np.logical_not(idx))[0]
        print("Found %d constraint violating jobs" % badvals.shape[0])
        print("Received %d valid results" % goodvals.shape[0])
        if goodvals.shape[0] < 2:
            return int(candidates[0])
        labels = np.zeros(vals.shape[0])
        labels[goodvals] = 1
        if np.sum(labels) < 2:
            return int(candidates[0])

        if self.D == -1:
            self._real_init(grid.shape[1], values[complete])

        numcand = cand.shape[0]
        best_comp = np.argmin(vals)                  # over ALL values: the first NaN if there is one (CONS:244)
        cand2 = np.vstack((np.random.randn(10, comp.shape[1]) * 0.001 + comp[best_comp, :], cand))

        if self.mcmc_iters <= 0:
            print("This Chooser module permits only slice sampling with > 0 samples.")
            raise Exception("mcmc_iters <= 0")

        comp_g, vals_g = comp[goodvals, :], vals[goodvals]
        self._loglik = self.backend.loglik(self.covar, comp_g, vals_g)
        if self.needs_burnin:
            for mcmc_iter in range(self.burnin):
                self.sample_constraint_hypers(comp, labels)
                self.sample_hypers(comp_g, vals_g)
                log("BURN %d/%d] mean: %.2f  amp: %.2f noise: %.4f  min_ls: %.4f  max_ls: %.4f"
                    % (mcmc_iter + 1, self.burnin, self.mean, np.sqrt(self.amp2), self.noise,
                       np.min(self.ls), np.max(self.ls)))
            self.needs_burnin = False

        self.hyper_samples = []
        for mcmc_iter in range(self.mcmc_iters):
            self.sample_constraint_hypers(comp, labels)
            self.sample_hypers(comp_g, vals_g)
        self._loglik = None
        self.dump_hypers()

        preds = self.backend.constraint_predict(self.covar, self._constraint_state(), self.ff, comp, cand)
        comp_preds = np.zeros(labels.shape[0])
        for ii in range(self.mcmc_iters):            # leaves the state of constraint sample S-1 and ff_samples[S-1]
            self._set_constraint(self.constraint_hyper_samples[ii])
            self.ff = self.ff_samples[ii]
            if self.verbosity > 0:
                comp_preds += self.backend.constraint_predict(self.covar, self._constraint_state(), self.ff, comp, comp)
        comp_preds = comp_preds / float(self.mcmc_iters)
        print("Predicting %.2f%% constraint violations (%d/%d): "
              % (np.mean(preds < 0.5) * 100, np.sum(preds < 0.5), preds.shape[0]))
        if self.verbosity > 0:
            print("Prediction` %f%% train accuracy (%d/%d): "
                  % (np.mean((comp_preds > 0.5) == labels), np.sum((comp_preds > 0.5) == labels),
                     comp_preds.shape[0]))

        # grid pass 1: the grid_subset best by mean constrained EI (CONS:381-383)
        overall_ei = self.ei_over_hypers(comp, pend, cand2, vals, labels)
        inds = np.argsort(np.mean(overall_ei, axis=1))[-self.grid_subset:]
        cand2 = cand2[inds, :]

        # refinement: L-BFGS-B from each of them (CONS:386-396), serially; the reference runs each in a forked worker,
        # so the global RNG the refinement touches (CONS:618) never reaches this process -- saved and restored here
        b = [(0, 1)] * cand.shape[1]
        state = npr.get_state()
        ctx = self._refine_context(comp, pend, vals, labels)
        refined = []
        for c in cand2:
            ret = spo.fmin_l_bfgs_b(ctx.value_grad, c.flatten(), bounds=b)
            refined.append(ret[0])
        del ctx
        npr.set_state(state)
        for r in refined:
            cand = np.vstack((cand, r))
        cand = np.vstack((cand, cand2))              # the unrefined short-list is scored as well (CONS:408)

        overall_ei = self.ei_over_hypers(comp, pend, cand, vals, labels)
        best_cand = np.argmax(np.mean(overall_ei, axis=1))
        self.dump_hypers()
        if best_cand >= numcand:
            return (int(numcand), cand[best_cand, :])
        return int(candidates[best_cand])

    # ------------------------------------------------------------------ grid pass and refinement
    def _constraint_state(self):
        return (self.constraint_mean, self.constraint_gain, self.constraint_amp2, self.constraint_ls)

    def _set_constraint(self, h):
        self.constraint_mean, self.constraint_gain, self.constraint_amp2, self.constraint_ls = h[0], h[1], h[2], h[3]

    def ei_over_hypers(self, comp, pend, cand, vals, labels):
        """(M, mcmc_iters) constrained EI (CONS:450-468): sample pairs 0..S-1, the current ff; with pending points a
        fresh (P, F) fantasy block per sample from the global RNG (CONS:910).  Leaves the state of sample S-1 loaded."""
        S = self.mcmc_iters
        hs, chs = self.hyper_samples[:S], self.constraint_hyper_samples[:S]
        normals = None
        if pend.shape[0] > 0:
            normals = np.stack([npr.randn(pend.shape[0], self.pending_samples) for _ in range(S)])
        out = self.backend.constrained_ei_matrix(self.covar, hs, chs, self.ff, comp, labels, pend, cand, vals, normals)
        self.mean, self.noise, self.amp2, self.ls = hs[-1]
        self._set_constraint(chs[-1])
        return out

    def _refine_context(self, comp, pend, vals, labels):
        S = self.mcmc_iters
        normals = None
        if pend.shape[0] > 0:                        # CONS:618-619, the same block at every evaluation
            npr.set_state(self.randomstate)
            normals = npr.randn(pend.shape[0], self.pending_samples)
        return self.backend.constrained_refine_context(self.covar, self.hyper_samples[:S],
                                                       self.constraint_hyper_samples[:S], self.ff, comp, labels, pend,
                                                       vals, normals, self.constraint_noise)

    def grad_optimize_ei_over_hypers(self, cand, comp, pend, vals, labels, compute_grad=True):
        """(sum_s -constrained EI_s, sum_s grad) at one point (CONS:471-501); leaves the global RNG as it found it."""
        state = npr.get_state()
        f, g = self._refine_context(comp, pend, vals, labels).value_grad(cand)
        npr.set_state(state)
        return (f, g) if compute_grad else f

    # ------------------------------------------------------------------ classification-GP chain (CONS:1014-1030)
    def sample_constraint_hypers(self, comp, labels):
        if self.ff is None or self.ff.shape[0] < comp.shape[0]:
            self.ff_samples = []
            prior = self.backend.latent_factor(self.covar, comp, self.constraint_amp2, self.constraint_ls, 1e-6)
            self.ff = prior.draw(npr.randn(comp.shape[0]))
        self._sample_constraint_noisy(comp, labels)
        self._sample_constraint_ls(comp, labels)
        self.constraint_hyper_samples.append(self._constraint_state())
        self.ff_samples.append(self.ff)

    def _sample_constraint_noisy(self, comp, labels):
        """Joint slice move over [amp2, ff] (CONS:1169-1192), then 50 elliptical-slice steps on ff (CONS:1193-1201)."""
        gain, scale = self.constraint_gain, self.constraint_amp2_scale

        def hypers_of(x):
            amp2, ff = x[0], x[1:]
            if amp2 < 0:
                return None
            return (amp2, ff), (-0.5 * (np.log(amp2) / scale) ** 2, probit_loglik(ff, gain, labels))

        ll = self.backend.latent_loglik(self.covar, comp, self.constraint_ls, self.constraint_noise)
        hypers = util.slice_sample(np.hstack((np.array([self.constraint_amp2]), self.ff)),
                                   util.make_logprob(ll, hypers_of), compwise=False)
        self.constraint_amp2 = hypers[0]
        self.ff = hypers[1:]
        # here the prior covariance of the elliptical-slice steps scales the noise by amp2 as well,
        # amp2 (k + 1e-6 I + noise I) (CONS:1193-1196); the length-scale step's does not (CONS:1103)
        fac = self.backend.latent_factor(self.covar, comp, self.constraint_amp2, self.constraint_ls,
                                         self.constraint_amp2 * self.constraint_noise)
        ff = self.ff
        for _ in range(50):
            ff, _lp = elliptical_slice(ff, fac, lambda f: probit_loglik(f, gain, labels))
        self.ff = ff

    def _sample_constraint_ls(self, comp, labels):
        """Length scales (their log-probability is the probit term alone, CONS:1089-1098), 20 elliptical-slice steps,
        then the gain in [0.01, 10] (CONS:1075-1114).  The Cholesky factors the reference computes inside the two
        log-probabilities are never used and are not formed."""
        gain, max_ls = self.constraint_gain, self.constraint_max_ls

        def logprob(ls):
            if np.any(ls < 0) or np.any(ls > max_ls):
                return -np.inf
            return probit_loglik(self.ff, gain, labels)

        self.constraint_ls = util.slice_sample(self.constraint_ls, logprob, compwise=True)
        fac = self.backend.latent_factor(self.covar, comp, self.constraint_amp2, self.constraint_ls,
                                         self.constraint_noise)
        ff = self.ff
        for _ in range(20):
            ff, _lp = elliptical_slice(ff, fac, lambda f: probit_loglik(f, gain, labels))
        self.ff = ff

        def update_gain(g):
            if g < 0.01 or g > 10:
                return -np.inf
            return probit_loglik(self.ff, g, labels)

        self.constraint_gain = util.slice_sample(np.array([self.constraint_gain]), update_gain, compwise=True)[0]

    # ------------------------------------------------------------------ objective chain (CONS:1032-1056, 1116-1232)
    def sample_hypers(self, comp, vals):
        """CONS:1116-1149: the joint move scales the noise by amp2, the length-scale move does not (CONS:1047-1049)."""
        ll = self._ll(comp, vals)
        if self.noiseless:
            self.noise = 1e-3
        self.mean, self.amp2, self.noise = self.prior.joint(ll, self.mean, self.amp2, self.noise, self.ls, vals,
                                                            self.noiseless)
        self.ls = self.prior.length_scales(ll, self.mean, self.noise, self.amp2, self.ls)
        self.hyper_samples.append((self.mean, self.noise, self.amp2, self.ls))
