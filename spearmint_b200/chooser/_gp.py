"""What the Gaussian-process choosers share: the hyper-parameter model of a GP chain and its two slice-sampler moves,
the state files, and the constructor scaffold.

The chains of GPEI-, GPEIOpt-, GPEIperSec- and GPConstrainedEIChooserB200 differ only in three reference quirks, each of
which decides the proposal (DESIGN section 9):

    chain            max_ls  amp2 prior term          noise in K, joint move  noise in K, ls move  noiseless
    GPEI             2       np.log(amp2)             noise                   noise                yes, 1e-3
    OPT              2       np.log(np.sqrt(amp2))    noise                   noise                yes, 1e-3
    PSEC objective   10      np.log(amp2)             noise                   noise                yes, 1e-3
    PSEC time        10      np.log(np.sqrt(amp2))    noise                   noise                no
    CONS objective   2       np.log(amp2)             amp2 * noise            noise (unscaled)     yes, amp2 * 1e-3

K = amp2 (k(ls) + 1e-6 I) + (noise in K) I.  The expressions are the reference's verbatim: slice acceptance is a strict
``>``, so a last-bit change in a prior term can move the chain.
"""
import os
import pickle
import tempfile

import numpy as np

from spearmint_b200 import util
from spearmint_b200.locker import Locker

COVARS = ("SE", "ARDSE", "Matern32", "Matern52")     # the stationary kernels of gp.py:87-127
GRID_DTYPES = ("float32", "float64")                 # precision of the grid pass (DeviceBackend grid_dtype)


class GPPrior(object):
    """The hyper-parameter model of one GP chain: horseshoe prior on the noise (``noise_scale``), zero-mean log-normal
    prior on the amplitude (``amp2_scale``; on log(sqrt(amp2)) when ``amp2_prior_on_std``), top-hat prior on the length
    scales in [0, ``max_ls``], the mean bounded by the chain's own targets.  ``noise_times_amp2``: the joint move puts
    amp2 * noise into K; the length-scale move always puts the noise in unscaled."""

    def __init__(self, max_ls, amp2_prior_on_std=False, noise_times_amp2=False, noise_scale=0.1, amp2_scale=1):
        self.max_ls, self.amp2_prior_on_std, self.noise_times_amp2 = max_ls, amp2_prior_on_std, noise_times_amp2
        self.noise_scale, self.amp2_scale = noise_scale, amp2_scale

    def joint(self, ll, mean, amp2, noise, ls, targets, noiseless=False):
        """Slice move over [mean, amp2, noise] (compwise=False) -> (mean, amp2, noise).  Noiseless: the noise coordinate
        is carried along (the random direction still has 3 components) but K takes 1e-3 and the noise stays 1e-3."""
        hypers_of = self._joint_map(ls, targets, noiseless)
        hypers = util.slice_sample(np.array([mean, amp2, noise]), util.make_logprob(ll, hypers_of), compwise=False)
        return hypers[0], hypers[1], (1e-3 if noiseless else hypers[2])

    def length_scales(self, ll, mean, noise, amp2, ls):
        """Component-wise slice move over the length scales -> ls."""
        return util.slice_sample(ls, util.make_logprob(ll, self._ls_map(mean, noise, amp2)), compwise=True)

    # step-wise forms (util.slice_steps): the same moves drawing from a chain's own RandomState ``rs``; they yield the
    # (mean, noise, amp2, ls) items to evaluate and expect their log-likelihoods sent back (chains.py)
    def joint_steps(self, rs, mean, amp2, noise, ls, targets, noiseless=False, speculate=(util.SPECULATE, 0)):
        hypers = yield from util.with_priors(
            util.slice_steps(np.array([mean, amp2, noise]), rs, speculate, compwise=False),
            self._joint_map(ls, targets, noiseless))
        return hypers[0], hypers[1], (1e-3 if noiseless else hypers[2])

    def length_scales_steps(self, rs, mean, noise, amp2, ls, speculate=(util.SPECULATE, 0)):
        return (yield from util.with_priors(util.slice_steps(ls, rs, speculate, compwise=True),
                                            self._ls_map(mean, noise, amp2)))

    def _joint_map(self, ls, targets, noiseless):
        """hypers_of of the joint move (util.CachedLogProb)."""
        vmax, vmin = np.max(targets), np.min(targets)
        noise_scale, amp2_scale, scaled = self.noise_scale, self.amp2_scale, self.noise_times_amp2
        log_amp = (lambda a: np.log(np.sqrt(a))) if self.amp2_prior_on_std else np.log

        if noiseless:
            def hypers_of(hypers):
                mean, amp2 = hypers[0], hypers[1]
                if mean > vmax or mean < vmin:
                    return None
                if amp2 < 0:
                    return None
                return (mean, amp2 * 1e-3 if scaled else 1e-3, amp2, ls), (-0.5 * (log_amp(amp2) / amp2_scale) ** 2,)
        else:
            def hypers_of(hypers):
                mean, amp2, noise = hypers[0], hypers[1], hypers[2]
                if mean > vmax or mean < vmin:
                    return None
                if amp2 < 0 or noise < 0:
                    return None
                return (mean, amp2 * noise if scaled else noise, amp2, ls), (
                    np.log(np.log(1 + (noise_scale / noise) ** 2)),              # horseshoe prior on the noise
                    -0.5 * (log_amp(amp2) / amp2_scale) ** 2)                     # log-normal prior on the amplitude
        return hypers_of

    def _ls_map(self, mean, noise, amp2):
        """hypers_of of the length-scale move."""
        max_ls = self.max_ls

        def hypers_of(ls):
            if np.any(ls < 0) or np.any(ls > max_ls):
                return None
            return (mean, noise, amp2, ls), ()
        return hypers_of


# ---------------------------------------------------------------------------------------------- state files
def write_state(locker, path, state):
    """Pickle ``state`` (protocol 2) to a temporary file and move it over ``path`` under the lock, as the reference."""
    locker.lock_wait(path)
    fh = tempfile.NamedTemporaryFile(mode="wb", delete=False)
    pickle.dump(state, fh, protocol=2)
    fh.close()
    os.system('mv "%s" "%s"' % (fh.name, path))
    locker.unlock(path)


def read_state(path):
    """The state dict pickled at ``path``, or None if there is none yet."""
    if not os.path.exists(path):
        return None
    with open(path, "rb") as fh:
        return pickle.load(fh)


def write_stats(path, hyper_samples):
    """The ``<module>_hyperparameters.txt`` file: every hyper-sample, then their mean."""
    with open(path, "w") as fh:
        fh.write("Mean Noise Amplitude <length scales>\n")
        fh.write("-----------ALL SAMPLES-------------\n")
        meanhyps = 0 * np.hstack(hyper_samples[0])
        for h in hyper_samples:
            hyps = np.hstack(h)
            meanhyps += (1 / float(len(hyper_samples))) * hyps
            fh.write(" ".join(str(j) for j in hyps) + " \n")
        fh.write("-----------MEAN OF SAMPLES-------------\n")
        fh.write(" ".join(str(j) for j in meanhyps) + " \n")


# ---------------------------------------------------------------------------------------------- constructor scaffold
class LazyBackend(object):
    """The ``backend`` property: a DeviceBackend made on first use (raises if there is no GPU), unless one was given."""
    _device = _backend = None
    _refine_dtype = "float64"
    _grid_dtype = "float32"

    @property
    def backend(self):
        if self._backend is None:
            from spearmint_b200.backend import DeviceBackend
            self._backend = DeviceBackend(device=self._device, refine_dtype=self._refine_dtype,
                                          grid_dtype=self._grid_dtype)
        return self._backend


class GPChooser(LazyBackend):
    """Options and file names every GP chooser takes the same way; ``_loglik`` is the objective chain's log-likelihood
    handle while a chain is being sampled."""

    def __init__(self, expt_dir, covar, mcmc_iters, pending_samples, noiseless, state_name, device, backend,
                 refine_dtype="float64", grid_dtype="float32"):
        if covar not in COVARS:
            raise AttributeError("module 'spearmint.gp' has no attribute '%s'" % covar)   # getattr(gp, covar)
        if grid_dtype not in GRID_DTYPES:
            raise ValueError("grid_dtype must be one of %s, got %r" % ("/".join(GRID_DTYPES), grid_dtype))
        self.covar = covar
        self.locker = Locker()
        name = state_name if state_name else self.__module__
        self.state_pkl = os.path.join(expt_dir, name + ".pkl")
        self.stats_file = os.path.join(expt_dir, name + "_hyperparameters.txt")
        self.mcmc_iters = int(mcmc_iters)
        self.pending_samples = int(pending_samples)
        self.D = -1
        self.hyper_iters = 1
        self.noiseless = bool(int(noiseless))
        self._device, self._refine_dtype, self._grid_dtype, self._backend = device, refine_dtype, grid_dtype, backend
        self._loglik = None

    def _ll(self, comp, vals):
        """The objective chain's log-likelihood handle; made here when sample_hypers runs outside next()."""
        if self._loglik is None:
            self._loglik = self.backend.loglik(self.covar, comp, vals)
        return self._loglik

    def _read_state(self):
        """The state pickle, read under the lock, or None if there is none yet."""
        self.locker.lock_wait(self.state_pkl)
        state = read_state(self.state_pkl)
        self.locker.unlock(self.state_pkl)
        return state

    def _load_hypers(self, state):
        """The objective chain's keys of a state pickle."""
        self.D = state["dims"]
        self.ls = state["ls"]
        self.amp2 = state["amp2"]
        self.noise = state["noise"]
        self.mean = state["mean"]

    def _init_hypers(self, dims, values):
        """The objective chain's start values when there is no state pickle yet."""
        self.D = dims
        self.ls = np.ones(self.D)
        self.amp2 = np.std(values) + 1e-4       # a std, not a variance -- reference quirk kept (OPT:193)
        self.noise = 1e-3
        self.mean = np.mean(values)
