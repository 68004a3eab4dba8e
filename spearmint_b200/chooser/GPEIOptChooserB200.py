"""Drop-in replacement for the reference's default chooser, ``chooser/GPEIOptChooser.py``.

Same plugin API (SURVEY.md 8b):  ``init(expt_dir, arg_string) -> obj``;
``obj.next(grid, values, durations, candidates, pending, complete) -> int | (int, ndarray)``;
optional ``obj.generate_stats_html()``.  Same option names and string casts, same state files
(``<expt_dir>/<module>.pkl`` with keys dims/ls/amp2/noise/hyper_samples/mean, ``<module>_hyperparameters.txt``),
same use of the process-global numpy RNG in the same order, same exceptions (LinAlgError, slice-sampler errors).

What changed is where the arithmetic runs: every covariance build, Cholesky, triangular solve, prediction and EI
evaluation is a hand-written sm_90a kernel behind the C ABI (``spearmint_b200.backend.DeviceBackend``):
  * hyper-parameter chain  : host slice sampler (util.py), log-likelihood on the GPU in float64      [f2]
  * EI over the grid       : all S samples batched in one pass in float32 (``ei_over_hypers``)        [a1-a10]
  * L-BFGS-B refinement    : scipy on the host, (f, g) from the GPU with the S factors cached         [f1]
                             (the reference re-factors K for every sample at every evaluation)
``use_multiprocessing`` is accepted and ignored: a forked pool cannot share a CUDA context, and with cached
factors the 20 refinements are cheap.  Extra optional keys: ``device``, ``refine_dtype``, ``state_name``.
"""
import os
import pickle
import tempfile
import time

import numpy as np
import numpy.random as npr
import scipy.optimize as spo

from spearmint_b200 import util
from spearmint_b200.locker import Locker, log

COVARS = ("SE", "ARDSE", "Matern32", "Matern52")     # the stationary kernels of gp.py:87-127


def init(expt_dir, arg_string):
    args = util.unpack_args(arg_string)
    return GPEIOptChooserB200(expt_dir, **args)


class GPEIOptChooserB200(object):

    def __init__(self, expt_dir, covar="Matern52", mcmc_iters=10, pending_samples=100, noiseless=False, burnin=100,
                 grid_subset=20, use_multiprocessing=True, device=None, refine_dtype="float64", state_name=None,
                 backend=None):
        if covar not in COVARS:
            raise AttributeError("module 'spearmint.gp' has no attribute '%s'" % covar)   # getattr(gp, covar), OPT:57
        self.covar = covar
        self.locker = Locker()
        name = state_name if state_name else self.__module__
        self.state_pkl = os.path.join(expt_dir, name + ".pkl")
        self.stats_file = os.path.join(expt_dir, name + "_hyperparameters.txt")
        self.mcmc_iters = int(mcmc_iters)
        self.burnin = int(burnin)
        self.needs_burnin = True
        self.pending_samples = int(pending_samples)
        self.D = -1
        self.hyper_iters = 1
        self.grid_subset = int(grid_subset)
        self.noiseless = bool(int(noiseless))
        self.hyper_samples = []
        self.noise_scale = 0.1     # horseshoe prior
        self.amp2_scale = 1        # zero-mean log normal prior
        self.max_ls = 2            # top-hat prior on length scales
        self.use_multiprocessing = bool(int(use_multiprocessing))
        self._device, self._refine_dtype = device, refine_dtype
        self._backend = backend
        self.stats = {}

    # ------------------------------------------------------------------ backend (GPU; raises if unavailable)
    @property
    def backend(self):
        if self._backend is None:
            from spearmint_b200.backend import DeviceBackend
            self._backend = DeviceBackend(device=self._device, refine_dtype=self._refine_dtype)
        return self._backend

    # ------------------------------------------------------------------ state files (OPT:84-120, 150-205)
    def dump_hypers(self):
        self.locker.lock_wait(self.state_pkl)
        fh = tempfile.NamedTemporaryFile(mode="wb", delete=False)
        pickle.dump({"dims": self.D, "ls": self.ls, "amp2": self.amp2, "noise": self.noise,
                     "hyper_samples": self.hyper_samples, "mean": self.mean}, fh, protocol=2)
        fh.close()
        os.system('mv "%s" "%s"' % (fh.name, self.state_pkl))       # atomic move, as the reference
        self.locker.unlock(self.state_pkl)

        with open(self.stats_file, "w") as fh:
            fh.write("Mean Noise Amplitude <length scales>\n")
            fh.write("-----------ALL SAMPLES-------------\n")
            meanhyps = 0 * np.hstack(self.hyper_samples[0])
            for h in self.hyper_samples:
                hyps = np.hstack(h)
                meanhyps += (1 / float(len(self.hyper_samples))) * hyps
                fh.write(" ".join(str(j) for j in hyps) + " \n")
            fh.write("-----------MEAN OF SAMPLES-------------\n")
            fh.write(" ".join(str(j) for j in meanhyps) + " \n")

    def _load_state(self):
        with open(self.state_pkl, "rb") as fh:
            state = pickle.load(fh)
        self.D = state["dims"]
        self.ls = state["ls"]
        self.amp2 = state["amp2"]
        self.noise = state["noise"]
        self.mean = state["mean"]
        self.hyper_samples = state["hyper_samples"]
        self.needs_burnin = False

    def _read_only(self):
        if os.path.exists(self.state_pkl):
            self._load_state()
            return True
        return False

    def generate_stats_html(self):
        if not self._read_only():
            return "Chooser not yet ready to display output"
        mean_mean = np.mean(np.vstack([h[0] for h in self.hyper_samples]))
        mean_noise = np.mean(np.vstack([h[1] for h in self.hyper_samples]))
        mean_ls = np.mean(np.vstack([h[3][np.newaxis, :] for h in self.hyper_samples]), 0)
        try:
            output = ('<br /><span class="label label-info">Estimated mean:</span> ' + str(mean_mean) +
                      '<br /><span class="label label-info">Estimated noise:</span> ' + str(mean_noise) +
                      '<br /><br /><span class="label label-info">Inverse parameter sensitivity' +
                      ' - Gaussian Process length scales</span><br /><br />' +
                      '<div id="lschart"></div><script type="text/javascript">' +
                      'var lsdata = [' + ','.join(['%.2f' % i for i in mean_ls]) + '];')
        except Exception:
            return "Chooser not yet ready to display output."
        output += 'bar_chart("#lschart", lsdata, ' + str(self.max_ls) + ');' + '</script>'
        return output

    def _real_init(self, dims, values):
        self.locker.lock_wait(self.state_pkl)
        self.randomstate = npr.get_state()
        if os.path.exists(self.state_pkl):
            self._load_state()
        else:
            self.D = dims
            self.ls = np.ones(self.D)
            self.amp2 = np.std(values) + 1e-4       # a std, not a variance -- reference quirk kept (OPT:193)
            self.noise = 1e-3
            self.mean = np.mean(values)
            self.hyper_samples.append((self.mean, self.noise, self.amp2, self.ls))
        self.locker.unlock(self.state_pkl)

    # ------------------------------------------------------------------ the plugin entry point (OPT:217-328)
    def next(self, grid, values, durations, candidates, pending, complete):
        if complete.shape[0] < 2:
            return int(candidates[0])
        if self.D == -1:
            self._real_init(grid.shape[1], values[complete])

        comp = grid[complete, :]
        cand = grid[candidates, :]
        pend = grid[pending, :]
        vals = values[complete]
        numcand = cand.shape[0]

        # Spray a set of candidates around the min so far (OPT:236-238; global RNG)
        best_comp = np.argmin(vals)
        cand2 = np.vstack((np.random.randn(10, comp.shape[1]) * 0.001 + comp[best_comp, :], cand))

        if self.mcmc_iters <= 0:
            # The reference's mcmc_iters=0 branch calls grad_optimize_ei with mismatched arguments (OPT:316-318)
            # and raises inside numpy; there is no behaviour to reproduce.
            raise NotImplementedError("mcmc_iters=0 (ML-II hyper-parameters) is broken in the reference "
                                      "(GPEIOptChooser.py:316-318) and not provided here")

        t_phase = [time.perf_counter()]
        phase_ms = {}

        def lap(name):          # wall-clock split of next(): every phase ends in a host read, so perf_counter is exact
            t_phase.append(time.perf_counter())
            phase_ms[name] = phase_ms.get(name, 0.0) + 1e3 * (t_phase[-1] - t_phase[-2])

        self._loglik = self.backend.loglik(self.covar, comp, vals)
        if self.needs_burnin:
            for mcmc_iter in range(self.burnin):
                self.sample_hypers(comp, vals)
                log("BURN %d/%d] mean: %.2f  amp: %.2f noise: %.4f  min_ls: %.4f  max_ls: %.4f"
                    % (mcmc_iter + 1, self.burnin, self.mean, np.sqrt(self.amp2), self.noise,
                       np.min(self.ls), np.max(self.ls)))
            self.needs_burnin = False

        self.hyper_samples = []
        for mcmc_iter in range(self.mcmc_iters):
            self.sample_hypers(comp, vals)
            log("%d/%d] mean: %.2f  amp: %.2f  noise: %.4f min_ls: %.4f  max_ls: %.4f"
                % (mcmc_iter + 1, self.mcmc_iters, self.mean, np.sqrt(self.amp2), self.noise,
                   np.min(self.ls), np.max(self.ls)))
        self.dump_hypers()
        self.stats["loglik_evals"] = getattr(self._loglik, "calls", None)
        self.stats["loglik_batches"] = getattr(self._loglik, "launch_batches", None)
        self._loglik = None
        lap("mcmc")

        b = [(0, 1)] * cand.shape[1]       # optimization bounds

        # grid pass 1 (OPT:269-271): mean EI over hyper-samples, top grid_subset candidates
        state = self._grid_state(comp, pend, vals)
        inds = self.backend.top_mean_ei(state, cand2, min(self.grid_subset, cand2.shape[0]))
        cand2 = cand2[inds, :]
        lap("grid_pass_1")

        # refine each of them with L-BFGS-B on the (summed) EI (OPT:274-291), factors cached
        ctx = self._refine_context(comp, pend, vals)
        for i in range(cand2.shape[0]):
            log("Optimizing candidate %d/%d" % (i + 1, cand2.shape[0]))
            ret = spo.fmin_l_bfgs_b(ctx.value_grad, cand2[i, :].flatten(), bounds=b)
            cand2[i, :] = ret[0]
        cand = np.vstack((cand, cand2))
        self.stats["refine_evals"] = getattr(ctx, "evals", None)
        del ctx
        lap("refine")

        # grid pass 2 (OPT:293-294): argmax of the mean EI over grid + refined points
        best_cand = int(self.backend.top_mean_ei(state, cand, 1)[-1])
        self._set_current(self.hyper_samples[-1])      # ei_over_hypers leaves the last sample loaded (OPT:334-338)
        lap("grid_pass_2")
        self.stats["phase_ms"] = phase_ms

        if best_cand >= numcand:
            return (int(numcand), cand[best_cand, :])
        return int(candidates[best_cand])

    # ------------------------------------------------------------------ EI over hyper-samples (OPT:331-341)
    def _fantasy_normals(self, pend):
        """The (P,F) normals of the pending fantasies; resets the global RNG exactly like OPT:588-589."""
        if pend.shape[0] == 0:
            return None
        npr.set_state(self.randomstate)
        return npr.randn(pend.shape[0], self.pending_samples)

    def _grid_state(self, comp, pend, vals):
        return self.backend.grid_state(self.covar, self.hyper_samples, comp, pend, vals, self._fantasy_normals(pend))

    def _refine_context(self, comp, pend, vals):
        return self.backend.refine_context(self.covar, self.hyper_samples, comp, pend, vals,
                                           self._fantasy_normals(pend))

    def _set_current(self, hyper):
        self.mean, self.noise, self.amp2, self.ls = hyper[0], hyper[1], hyper[2], hyper[3]

    def ei_over_hypers(self, comp, pend, cand, vals):
        """(M, mcmc_iters) EI matrix, one column per hyper-sample -- all samples in one batched GPU pass."""
        hs = self.hyper_samples[:self.mcmc_iters]
        st = self.backend.grid_state(self.covar, hs, comp, pend, vals, self._fantasy_normals(pend))
        out = self.backend.ei_matrix(st, cand)
        self._set_current(hs[-1])
        return out

    def compute_ei(self, comp, pend, cand, vals):
        """EI under the CURRENT hyper-parameters (self.mean/noise/amp2/ls), OPT:527-619."""
        hs = [(self.mean, self.noise, self.amp2, self.ls)]
        st = self.backend.grid_state(self.covar, hs, comp, pend, vals, self._fantasy_normals(pend))
        return self.backend.ei_matrix(st, cand)[:, 0]

    def grad_optimize_ei_over_hypers(self, cand, comp, pend, vals, compute_grad=True):
        """(sum_s -EI_s, sum_s grad) at one point (OPT:360-388).  Builds a fresh cached context per call; next()
        keeps one context for the whole refinement instead."""
        f, g = self._refine_context(comp, pend, vals).value_grad(cand)
        return (f, g) if compute_grad else f

    # ------------------------------------------------------------------ hyper-parameter sampling (OPT:621-706)
    def _ll(self, comp, vals):
        if getattr(self, "_loglik", None) is None:
            self._loglik = self.backend.loglik(self.covar, comp, vals)
        return self._loglik

    def sample_hypers(self, comp, vals):
        if self.noiseless:
            self.noise = 1e-3
            self._sample_noiseless(comp, vals)
        else:
            self._sample_noisy(comp, vals)
        self._sample_ls(comp, vals)
        self.hyper_samples.append((self.mean, self.noise, self.amp2, self.ls))

    def _sample_ls(self, comp, vals):
        mean, noise, amp2, max_ls = self.mean, self.noise, self.amp2, self.max_ls

        def hypers_of(ls):
            if np.any(ls < 0) or np.any(ls > max_ls):
                return None
            return (mean, noise, amp2, ls), ()

        self.ls = util.slice_sample(self.ls, util.make_logprob(self._ll(comp, vals), hypers_of), compwise=True)

    def _sample_noisy(self, comp, vals):
        vmax, vmin, ls = np.max(vals), np.min(vals), self.ls

        def hypers_of(hypers):
            mean, amp2, noise = hypers[0], hypers[1], hypers[2]
            if mean > vmax or mean < vmin:
                return None
            if amp2 < 0 or noise < 0:
                return None
            return (mean, noise, amp2, ls), (
                np.log(np.log(1 + (self.noise_scale / noise) ** 2)),           # horseshoe prior on the noise
                -0.5 * (np.log(np.sqrt(amp2)) / self.amp2_scale) ** 2)        # log-normal prior on the amplitude

        hypers = util.slice_sample(np.array([self.mean, self.amp2, self.noise]),
                                   util.make_logprob(self._ll(comp, vals), hypers_of), compwise=False)
        self.mean, self.amp2, self.noise = hypers[0], hypers[1], hypers[2]

    def _sample_noiseless(self, comp, vals):
        vmax, vmin, ls = np.max(vals), np.min(vals), self.ls

        def hypers_of(hypers):
            mean, amp2 = hypers[0], hypers[1]
            if mean > vmax or mean < vmin:
                return None
            if amp2 < 0:
                return None
            return (mean, 1e-3, amp2, ls), (-0.5 * (np.log(np.sqrt(amp2)) / self.amp2_scale) ** 2,)

        hypers = util.slice_sample(np.array([self.mean, self.amp2, self.noise]),
                                   util.make_logprob(self._ll(comp, vals), hypers_of), compwise=False)
        self.mean, self.amp2, self.noise = hypers[0], hypers[1], 1e-3
