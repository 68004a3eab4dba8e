"""Drop-in replacement for the reference's ``chooser/GPEIperSecChooser.py`` (EI per second, two GPs).

Same plugin API, options, state pickle keys (dims, ls, amp2, noise, mean, time_ls, time_amp2, time_noise,
time_mean -- PSEC:87-95) and global-RNG order.  The reference's observable quirks are reproduced on purpose,
because they decide which point it proposes (SURVEY.md 3.4 / section 7):
  * ``ei_over_hypers`` returns from INSIDE its sample loop (PSEC:302): only column 0 is ever filled;
  * ``time_hyper_samples`` is never cleared (PSEC:199), so index [i] reads the OLDEST (burn-in) time samples (PSEC:288);
  * the refinement ignores pending points (PSEC:351-435) and is serial;
  * fantasy normals come straight from the global RNG stream, with no state reset (PSEC:521);
  * the objective and time chains are sampled with GPPrior values of their own (chooser/_gp.py).
All arithmetic runs on the GPU through spearmint_b200.backend.DeviceBackend.
"""
import numpy as np
import numpy.random as npr
import scipy.optimize as spo

from spearmint_b200 import util
from spearmint_b200.chooser._gp import GPChooser, GPPrior, write_state
from spearmint_b200.locker import log


def init(expt_dir, arg_string):
    args = util.unpack_args(arg_string)
    return GPEIperSecChooserB200(expt_dir, **args)


class GPEIperSecChooserB200(GPChooser):
    prior = GPPrior(max_ls=10)                                   # log(amp2) prior: PSEC:614
    time_prior = GPPrior(max_ls=10, amp2_prior_on_std=True)      # log(sqrt(amp2)) prior: PSEC:646

    def __init__(self, expt_dir, covar="Matern52", mcmc_iters=10, pending_samples=100, noiseless=False, burnin=100,
                 grid_subset=20, device=None, refine_dtype="float64", state_name=None, backend=None, grid_dtype="float32"):
        GPChooser.__init__(self, expt_dir, covar, mcmc_iters, pending_samples, noiseless, state_name, device, backend,
                           refine_dtype, grid_dtype)
        self.burnin = int(burnin)
        self.needs_burnin = True
        self.grid_subset = int(grid_subset)
        self.hyper_samples = []
        self.time_hyper_samples = []
        self._time_loglik = None

    # ------------------------------------------------------------------ state (PSEC:82-143)
    def dump_hypers(self):
        write_state(self.locker, self.state_pkl,
                    {"dims": self.D, "ls": self.ls, "amp2": self.amp2, "noise": self.noise, "mean": self.mean,
                     "time_ls": self.time_ls, "time_amp2": self.time_amp2, "time_noise": self.time_noise,
                     "time_mean": self.time_mean})

    def _real_init(self, dims, values, durations):
        state = self._read_state()
        if state is not None:
            self._load_hypers(state)
            self.time_ls, self.time_amp2 = state["time_ls"], state["time_amp2"]
            self.time_noise, self.time_mean = state["time_noise"], state["time_mean"]
        else:
            self._init_hypers(dims, values)
            self.time_ls = np.ones(self.D)
            self.time_amp2 = np.std(durations) + 1e-4      # std of the RAW durations (PSEC:132)
            self.time_noise = 1e-3
            self.time_mean = np.mean(np.log(durations))

    # ------------------------------------------------------------------ plugin entry point (PSEC:155-281)
    def next(self, grid, values, durations, candidates, pending, complete):
        if complete.shape[0] < 2:
            return int(candidates[0])
        if self.D == -1:
            self._real_init(grid.shape[1], values[complete], durations[complete])

        comp = grid[complete, :]
        cand = grid[candidates, :]
        pend = grid[pending, :]
        vals = values[complete]
        durs = np.log(durations[complete])          # log domain keeps durations positive (PSEC:176)

        numcand = cand.shape[0]
        best_comp = np.argmin(vals)
        cand2 = np.vstack((np.random.randn(10, comp.shape[1]) * 0.001 + comp[best_comp, :], cand))

        if self.mcmc_iters <= 0:
            raise NotImplementedError("mcmc_iters=0 is broken in the reference (GPEIperSecChooser.py:254 reads an "
                                      "undefined overall_ei) and not provided here")

        self._loglik = self.backend.loglik(self.covar, comp, vals)
        self._time_loglik = self.backend.loglik(self.covar, comp, durs.squeeze())
        if self.needs_burnin:
            for mcmc_iter in range(self.burnin):
                self.sample_hypers(comp, vals, durs)
                log("BURN %d/%d] mean: %.2f  amp: %.2f noise: %.4f  min_ls: %.4f  max_ls: %.4f"
                    % (mcmc_iter + 1, self.burnin, self.mean, np.sqrt(self.amp2), self.noise,
                       np.min(self.ls), np.max(self.ls)))
            self.needs_burnin = False

        self.hyper_samples = []                      # time_hyper_samples is NOT cleared (PSEC:199)
        for mcmc_iter in range(self.mcmc_iters):
            self.sample_hypers(comp, vals, durs)
            log("%d/%d] mean: %.2f  amp: %.2f  noise: %.4f min_ls: %.4f  max_ls: %.4f"
                % (mcmc_iter + 1, self.mcmc_iters, self.mean, np.sqrt(self.amp2), self.noise,
                   np.min(self.ls), np.max(self.ls)))
            log("%d/%d] time_mean: %.2fs time_amp: %.2f  time_noise: %.4f time_min_ls: %.4f  time_max_ls: %.4f"
                % (mcmc_iter + 1, self.mcmc_iters, np.exp(self.time_mean), np.sqrt(self.time_amp2),
                   np.exp(self.time_noise), np.min(self.time_ls), np.max(self.time_ls)))
        self.dump_hypers()
        self._loglik = self._time_loglik = None

        # grid pass 1: only sample 0 contributes (PSEC:302) -> ranking by column 0
        k = min(self.grid_subset, cand2.shape[0])
        inds = self.backend.top_mean_ei(self._grid_state(comp, pend, vals, durs), cand2, k)
        cand2 = cand2[inds, :]

        b = [(0, 1)] * cand.shape[1]
        ctx = self.backend.refine_context(self.covar, self.hyper_samples[:self.mcmc_iters], comp,
                                          np.zeros((0, comp.shape[1])), vals, None,
                                          self.time_hyper_samples[:self.mcmc_iters], durs)
        for i in range(cand2.shape[0]):
            log("Optimizing candidate %d/%d" % (i + 1, cand2.shape[0]))
            ret = spo.fmin_l_bfgs_b(ctx.value_grad, cand2[i, :].flatten(), bounds=b)
            cand2[i, :] = ret[0]
        del ctx
        cand = np.vstack((cand, cand2))

        best_cand = int(self.backend.top_mean_ei(self._grid_state(comp, pend, vals, durs), cand, 1)[-1])
        self._load_pair(0)
        self.dump_hypers()
        if best_cand >= numcand:
            return (int(numcand), cand[best_cand, :])
        return int(candidates[best_cand])

    # ------------------------------------------------------------------ EI per second over hyper-samples (PSEC:284-302)
    def _load_pair(self, i):
        (self.mean, self.noise, self.amp2, self.ls) = self.hyper_samples[i]
        (self.time_mean, self.time_noise, self.time_amp2, self.time_ls) = self.time_hyper_samples[i]

    def _grid_state(self, comp, pend, vals, durs):
        normals = npr.randn(pend.shape[0], self.pending_samples) if pend.shape[0] else None    # PSEC:521
        return self.backend.grid_state(self.covar, [self.hyper_samples[0]], comp, pend, vals, normals,
                                       [self.time_hyper_samples[0]], np.asarray(durs).squeeze())

    def ei_over_hypers(self, comp, pend, cand, vals, durs):
        """(M, mcmc_iters) with ONLY column 0 filled -- the reference returns inside its loop (PSEC:302)."""
        out = np.zeros((cand.shape[0], self.mcmc_iters))
        out[:, 0] = self.backend.ei_matrix(self._grid_state(comp, pend, vals, durs), cand)[:, 0]
        self._load_pair(0)
        return out

    def compute_ei_per_s(self, comp, pend, cand, vals, durs):
        """EI / exp(predicted log-duration) under the CURRENT hyper-parameters (PSEC:437-548)."""
        normals = npr.randn(pend.shape[0], self.pending_samples) if pend.shape[0] else None
        st = self.backend.grid_state(self.covar, [(self.mean, self.noise, self.amp2, self.ls)], comp, pend, vals,
                                     normals, [(self.time_mean, self.time_noise, self.time_amp2, self.time_ls)],
                                     np.asarray(durs).squeeze())
        return self.backend.ei_matrix(st, cand)[:, 0]

    def grad_optimize_ei_over_hypers(self, cand, comp, vals, durs, compute_grad=True):
        ctx = self.backend.refine_context(self.covar, self.hyper_samples[:self.mcmc_iters], comp,
                                          np.zeros((0, comp.shape[1])), vals, None,
                                          self.time_hyper_samples[:self.mcmc_iters], durs)
        f, g = ctx.value_grad(cand)
        return (f, g) if compute_grad else f

    # ------------------------------------------------------------------ sampling (PSEC:550-681)
    def sample_hypers(self, comp, vals, durs):
        durs = np.asarray(durs).squeeze()
        if self._loglik is None:
            self._loglik = self.backend.loglik(self.covar, comp, vals)
            self._time_loglik = self.backend.loglik(self.covar, comp, durs)
        ll, tll = self._loglik, self._time_loglik
        if self.noiseless:
            self.noise = 1e-3
        self.mean, self.amp2, self.noise = self.prior.joint(ll, self.mean, self.amp2, self.noise, self.ls, vals,
                                                            self.noiseless)
        self.ls = self.prior.length_scales(ll, self.mean, self.noise, self.amp2, self.ls)
        # the time chain is always noisy
        self.time_mean, self.time_amp2, self.time_noise = self.time_prior.joint(
            tll, self.time_mean, self.time_amp2, self.time_noise, self.time_ls, durs)
        self.time_ls = self.time_prior.length_scales(tll, self.time_mean, self.time_noise, self.time_amp2, self.time_ls)
        self.hyper_samples.append((self.mean, self.noise, self.amp2, self.ls))
        self.time_hyper_samples.append((self.time_mean, self.time_noise, self.time_amp2, self.time_ls))
