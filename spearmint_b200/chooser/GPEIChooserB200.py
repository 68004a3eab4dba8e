"""Drop-in replacement for the reference's ``chooser/GPEIChooser.py`` (EI on the grid only, no refinement).

``next()`` (GPEIChooser.py:124-176): for each of ``mcmc_iters`` iterations draw one hyper-sample (no burn-in, the
chain continues from the previous call / pickle) and evaluate EI over all candidates; return the argmax of the mean.
The reference interleaves RNG use -- sample, fantasy normals (``npr.randn(P, F)``, GPEI:237, no state reset), sample,
... -- so the normals are drawn here in that same order and carried per sample; the EI passes themselves are then
done for all samples in ONE batched GPU pass (``compute_ei`` math is identical to GPEIOptChooser's, GPEI:178-266).
State pickle keys dims/ls/amp2/noise/mean, written on destruction like the reference (GPEI:66-84).
``mcmc_iters=0`` runs the ML-II branch: ``gp.GP.optimize_hypers`` (spearmint_b200/gp.py, GP:181-292) then EI under the optimum.
"""
import numpy as np
import numpy.random as npr

from spearmint_b200 import util
from spearmint_b200.chooser._gp import GPChooser, GPPrior, write_state
from spearmint_b200.locker import log


def init(expt_dir, arg_string):
    args = util.unpack_args(arg_string)
    return GPEIChooserB200(expt_dir, **args)


class GPEIChooserB200(GPChooser):
    prior = GPPrior(max_ls=2)

    def __init__(self, expt_dir, covar="Matern52", mcmc_iters=10, pending_samples=100, noiseless=False,
                 device=None, state_name=None, backend=None, grid_dtype="float32"):
        GPChooser.__init__(self, expt_dir, covar, mcmc_iters, pending_samples, noiseless, state_name, device, backend,
                           grid_dtype=grid_dtype)

    def dump_hypers(self):
        if self.D == -1:
            return
        write_state(self.locker, self.state_pkl,
                    {"dims": self.D, "ls": self.ls, "amp2": self.amp2, "noise": self.noise, "mean": self.mean})

    def __del__(self):          # the reference persists its state in the destructor (GPEI:66-84)
        try:
            self.dump_hypers()
        except Exception:
            pass

    def _real_init(self, dims, values):
        state = self._read_state()
        if state is not None:
            self._load_hypers(state)
        else:
            self._init_hypers(dims, values)

    def next(self, grid, values, durations, candidates, pending, complete):
        if complete.shape[0] < 2:
            return int(candidates[0])
        if self.D == -1:
            self._real_init(grid.shape[1], values[complete])
        comp, cand, pend = grid[complete, :], grid[candidates, :], grid[pending, :]
        vals = values[complete]
        if self.mcmc_iters <= 0:
            # ML-II branch (GPEI:156-176): optimise the hyper-parameters, EI under them, argmax
            try:
                self.optimize_hypers(comp, vals)
            except Exception:                         # the reference's bare except: fall back to the initial values
                self.ls = np.ones(self.D)
                self.amp2 = np.std(vals)
                self.noise = 1e-3
            log("mean: %f  amp: %f  noise: %f  min_ls: %f  max_ls: %f"
                % (self.mean, np.sqrt(self.amp2), self.noise, np.min(self.ls), np.max(self.ls)))
            ei = self.compute_ei(comp, pend, cand, vals)
            return int(candidates[int(np.argmax(ei))])
        P = pend.shape[0]
        self._loglik = self.backend.loglik(self.covar, comp, vals)
        hs, normals = [], []
        for mcmc_iter in range(self.mcmc_iters):
            self.sample_hypers(comp, vals)
            log("mean: %f  amp: %f  noise: %f  min_ls: %f  max_ls: %f"
                % (self.mean, np.sqrt(self.amp2), self.noise, np.min(self.ls), np.max(self.ls)))
            hs.append((self.mean, self.noise, self.amp2, self.ls))
            if P:
                normals.append(npr.randn(P, self.pending_samples))       # same stream position as GPEI:237
        self._loglik = None
        st = self.backend.grid_state(self.covar, hs, comp, pend, vals, np.array(normals) if P else None)
        best_cand = int(self.backend.top_mean_ei(st, cand, 1)[-1])
        return int(candidates[best_cand])

    def compute_ei(self, comp, pend, cand, vals):
        """EI under the current hyper-parameters (GPEI:178-266)."""
        P = pend.shape[0]
        normals = npr.randn(P, self.pending_samples) if P else None
        st = self.backend.grid_state(self.covar, [(self.mean, self.noise, self.amp2, self.ls)], comp, pend, vals,
                                     normals)
        return self.backend.ei_matrix(st, cand)[:, 0]

    def optimize_hypers(self, comp, vals):
        """GPEI:348-361: a fresh gp.GP of the same kernel, ML-II from its own start values; the result replaces ours."""
        self.mean, self.noise, self.amp2, self.ls = self.backend.optimize_hypers(self.covar, comp, vals)

    # ------------------------------------------------------------------ sampling (GPEI:268-346)
    def sample_hypers(self, comp, vals):
        ll = self._ll(comp, vals)
        if self.noiseless:
            self.noise = 1e-3
        self.mean, self.amp2, self.noise = self.prior.joint(ll, self.mean, self.amp2, self.noise, self.ls, vals,
                                                            self.noiseless)
        self.ls = self.prior.length_scales(ll, self.mean, self.noise, self.amp2, self.ls)
