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
factors the 20 refinements are cheap.  Extra optional keys: ``device``, ``refine_dtype``, ``grid_dtype``,
``state_name``, ``mcmc_chains``.

``mcmc_chains=K`` (default 1) runs K independent chains of the same sampler in lockstep (chains.py): one batched
log-likelihood call per round for all of them, and under torchrun chain c on rank c mod W.  Each chain burns in on its
first call and then takes mcmc_iters / K steps; hyper_samples is round-major (step r of chain 0, of chain 1, ...).  The
chains draw from RandomStates of their own, seeded by K draws of npr.randint(2**32) from the global RNG right after the
jitter cloud of the next() that creates them; afterwards they never touch the global RNG.  The state pickle keeps the
reference's keys (mean/noise/amp2/ls: the last chain's last sample) and adds ``chains``: per chain (mean, noise, amp2,
ls, RandomState state).  A pickle with ``chains`` resumes without burn-in (its length must be K); one without starts
every chain from its hyper-parameters and burns each one in.  K = 1 is the reference's single chain, unchanged (it
reads the reference's keys of any pickle and ignores ``chains``).
"""
import time

import numpy as np
import numpy.random as npr
import scipy.optimize as spo

from spearmint_b200 import chains, util
from spearmint_b200.chooser._gp import GPChooser, GPPrior, read_state, write_state, write_stats
from spearmint_b200.locker import log


def init(expt_dir, arg_string):
    args = util.unpack_args(arg_string)
    return GPEIOptChooserB200(expt_dir, **args)


class GPEIOptChooserB200(GPChooser):
    prior = GPPrior(max_ls=2, amp2_prior_on_std=True)

    def __init__(self, expt_dir, covar="Matern52", mcmc_iters=10, pending_samples=100, noiseless=False, burnin=100,
                 grid_subset=20, use_multiprocessing=True, device=None, refine_dtype="float64", state_name=None,
                 backend=None, grid_dtype="float32", mcmc_chains=1):
        GPChooser.__init__(self, expt_dir, covar, mcmc_iters, pending_samples, noiseless, state_name, device, backend,
                           refine_dtype, grid_dtype)
        self.mcmc_chains = int(mcmc_chains)
        if self.mcmc_chains < 1:
            raise ValueError("mcmc_chains must be at least 1, got %d" % self.mcmc_chains)
        if self.mcmc_iters > 0 and self.mcmc_iters % self.mcmc_chains:
            raise ValueError("mcmc_iters (%d) must be a multiple of mcmc_chains (%d)" % (self.mcmc_iters,
                                                                                       self.mcmc_chains))
        self.chains = None          # mcmc_chains > 1: the chains.Chain list, made by the first next() or a resume
        self.burnin = int(burnin)
        self.needs_burnin = True
        self.grid_subset = int(grid_subset)
        self.hyper_samples = []
        self.use_multiprocessing = bool(int(use_multiprocessing))
        self.stats = {}

    # ------------------------------------------------------------------ state files (OPT:84-120, 150-205)
    def dump_hypers(self):
        state = {"dims": self.D, "ls": self.ls, "amp2": self.amp2, "noise": self.noise,
                 "hyper_samples": self.hyper_samples, "mean": self.mean}
        if self.chains is not None:
            state["chains"] = [c.state() for c in self.chains]
        write_state(self.locker, self.state_pkl, state)
        write_stats(self.stats_file, self.hyper_samples)

    def _load_state(self, state):
        self._load_hypers(state)
        self.hyper_samples = state["hyper_samples"]
        self.needs_burnin = False
        if self.mcmc_chains > 1 and "chains" in state:
            if len(state["chains"]) != self.mcmc_chains:
                raise ValueError("the state pickle holds %d chains, mcmc_chains is %d" % (len(state["chains"]),
                                                                                        self.mcmc_chains))
            self.chains = [chains.Chain.from_state(c, st) for c, st in enumerate(state["chains"])]

    def generate_stats_html(self):
        state = read_state(self.state_pkl)
        if state is None:
            return "Chooser not yet ready to display output"
        self._load_state(state)
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
        output += 'bar_chart("#lschart", lsdata, ' + str(self.prior.max_ls) + ');' + '</script>'
        return output

    def _real_init(self, dims, values):
        self.randomstate = npr.get_state()
        state = self._read_state()
        if state is not None:
            self._load_state(state)
        else:
            self._init_hypers(dims, values)
            self.hyper_samples.append((self.mean, self.noise, self.amp2, self.ls))

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

        if self.mcmc_chains > 1:
            self._sample_chains(comp, vals)
        else:
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

    def _sample_chains(self, comp, vals):
        """mcmc_chains > 1: every chain's burn-in (first call) and mcmc_iters / K steps, in lockstep (chains.py)."""
        K = self.mcmc_chains
        if self.chains is None:     # no chains in the state pickle: all start from the current hyper-parameters
            self.chains = chains.Chain.seeded(K, (self.mean, self.noise, self.amp2, self.ls))
        ll = self.backend.loglik(self.covar, comp, vals, chains=K)
        self.hyper_samples, rounds = chains.sample(self.chains, self.prior, ll, vals, self.noiseless, self.burnin,
                                                   self.mcmc_iters // K)
        self._set_current(self.hyper_samples[-1])
        self.needs_burnin = False
        self.dump_hypers()
        self.stats["loglik_evals"] = getattr(ll, "calls", None)
        self.stats["loglik_batches"] = getattr(ll, "launch_batches", None)
        self.stats["chain_rounds"] = rounds

    # ------------------------------------------------------------------ hyper-parameter sampling (OPT:621-706)
    def sample_hypers(self, comp, vals):
        ll = self._ll(comp, vals)
        if self.noiseless:
            self.noise = 1e-3
        self.mean, self.amp2, self.noise = self.prior.joint(ll, self.mean, self.amp2, self.noise, self.ls, vals,
                                                            self.noiseless)
        self.ls = self.prior.length_scales(ll, self.mean, self.noise, self.amp2, self.ls)
        self.hyper_samples.append((self.mean, self.noise, self.amp2, self.ls))
