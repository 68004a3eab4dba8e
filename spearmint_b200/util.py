"""Host helpers of the chooser plugin API: the "k=v,k=v" argument protocol and the slice sampler.

Both are part of the drop-in boundary (SURVEY.md 8b): ``init(expt_dir, arg_string)`` hands every option over as a
string, and the hyper-parameter chain must consume the process-global numpy RNG in exactly the reference's order
(util.py:34-93 of the reference) so that, with a float64 log-likelihood, the chain reproduces the reference's draws.
The log-probability callbacks are evaluated on the GPU (engine.LogLik); the sampler control flow stays on the host.
"""
import re

import numpy as np
import numpy.random as npr


def unpack_args(arg_string):
    """"a=1,b=x" -> {"a": "1", "b": "x"}; strings of length <= 1 give {} (reference util.py:26-32)."""
    if len(arg_string) > 1:
        pairs = re.split(r"\s*,\s*", arg_string)
        return dict(re.split(r"\s*=\s*", kv) for kv in pairs)
    return {}


SPECULATE = 3    # shrink proposals evaluated ahead of time when the log-probability supports batching


def _peek_shrink(lower, upper, n, rng=npr):
    """The next n shrink proposals of the interval (lower, upper) assuming each one is rejected, obtained by PEEKING
    ``rng`` (the global RNG, or a chain's RandomState; state saved and restored): the draws consumed later are exactly
    these."""
    state = rng.get_state()
    peek = rng.rand(n)
    rng.set_state(state)
    zs, lo, hi = [], lower, upper
    for r in peek:
        z = (hi - lo) * r + lo
        zs.append(z)
        if z < 0:
            lo = z
        elif z > 0:
            hi = z
    return zs


def _slice_along(direction, x0, logprob, sigma, step_out, max_steps_out):
    """One slice-sampling move along ``direction`` (reference util.py:36-75).  RNG call order:
    rand (interval placement), rand (slice height), then one rand per shrink proposal.

    If ``logprob`` has a ``prefetch(points)`` method (spearmint_b200's GPU log-likelihood), the points this move will
    most likely visit are handed to it first so that they are evaluated as ONE batched factorisation:
      phase 1: 0, lower, upper (always needed) and the first ``speculate[0]`` shrink proposals assuming no step-out;
      phase 2: once the interval is final, shrink proposals in groups of ``speculate[1]``.
    ``logprob.speculate`` = (s1, s2) tunes this to the cost model of the likelihood: a latency-bound factorisation
    (small N) evaluates 6 points for the price of one, a flop-bound one (N = 4096) pays for every wasted point.
    The proposals are obtained by PEEKING the global RNG, so the draws consumed, the points visited and therefore the
    chain are exactly the reference's."""
    def lp(z):
        return logprob(direction * z + x0)

    upper = sigma * npr.rand()
    lower = upper - sigma
    u_height = npr.rand()
    can_prefetch = hasattr(logprob, "prefetch")
    s1, s2 = getattr(logprob, "speculate", (SPECULATE, 0)) if can_prefetch else (0, 0)
    if can_prefetch:
        zs = [0.0, lower, upper] + _peek_shrink(lower, upper, s1)
        logprob.prefetch([direction * z + x0 for z in zs])
    height = np.log(u_height) + lp(0.0)
    n_lo = n_hi = 0
    if step_out:
        while lp(lower) > height and n_lo < max_steps_out:
            n_lo += 1
            lower -= sigma
        while lp(upper) > height and n_hi < max_steps_out:
            n_hi += 1
            upper += sigma
    covered = s1 if (n_lo == 0 and n_hi == 0) else 0      # proposals of phase 1 still valid (the interval did not move)
    it = 0
    while True:
        if can_prefetch and s2 > 0 and it >= covered:
            logprob.prefetch([direction * z + x0 for z in _peek_shrink(lower, upper, s2)])
            covered = it + s2
        z = (upper - lower) * npr.rand() + lower
        val = lp(z)
        it += 1
        if np.isnan(val):
            raise Exception("Slice sampler got a NaN")
        if val > height:
            return z * direction + x0
        if z < 0:
            lower = z
        elif z > 0:
            upper = z
        else:
            raise Exception("Slice sampler shrank to zero!")


def slice_sample(init_x, logprob, sigma=1.0, step_out=True, max_steps_out=1000, compwise=False, verbose=False):
    """Univariate slice sampling along a random direction, or component-wise in shuffled order
    (reference util.py:34-93).  Acceptance is a strict ``>`` on log-probabilities."""
    init_x = np.asarray(init_x, dtype=float)
    if not init_x.shape:
        init_x = np.array([init_x])
    dims = init_x.shape[0]
    if compwise:
        order = list(range(dims))
        npr.shuffle(order)
        x = init_x.copy()
        for d in order:
            e = np.zeros(dims)
            e[d] = 1.0
            x = _slice_along(e, x, logprob, sigma, step_out, max_steps_out)
        return x
    direction = npr.randn(dims)
    direction = direction / np.sqrt(np.sum(direction ** 2))
    return _slice_along(direction, init_x, logprob, sigma, step_out, max_steps_out)


# ---------------------------------------------------------------------------------------------- step-wise slice sampler
# The same sampler as a generator, so that several chains can share one batched log-likelihood call per round
# (chains.py).  It draws from an explicit RandomState, yields the list of points whose log-probabilities it needs, and
# expects the list of their values sent back (NaN: the covariance is not positive definite).  Its draws, the points it
# visits and its result are slice_sample's with a CachedLogProb of the same ``speculate`` (tests/test_mcmc_chains_host.py).
def _not_pd():
    return np.linalg.LinAlgError("leading minor of the array is not positive definite")


def _lp_step(x, cache):
    """Log-probability at ``x``: from the move's prefetched values, else one point of its own (CachedLogProb.__call__)."""
    v = cache.get(CachedLogProb._key(x))
    if v is None:
        v = (yield [x])[0]
    if np.isnan(v):
        raise _not_pd()
    return v


def _prefetch_step(points):
    """CachedLogProb.prefetch: a fresh cache holding the values of ``points``."""
    vals = yield points
    return {CachedLogProb._key(x): v for x, v in zip(points, vals)}


def _slice_along_steps(direction, x0, rs, sigma, step_out, max_steps_out, speculate):
    """_slice_along with ``rs`` for the global RNG and a prefetching log-probability of depth ``speculate``."""
    s1, s2 = speculate
    upper = sigma * rs.rand()
    lower = upper - sigma
    u_height = rs.rand()
    zs = [0.0, lower, upper] + _peek_shrink(lower, upper, s1, rs)
    cache = yield from _prefetch_step([direction * z + x0 for z in zs])
    height = np.log(u_height) + (yield from _lp_step(direction * 0.0 + x0, cache))
    n_lo = n_hi = 0
    if step_out:
        while (yield from _lp_step(direction * lower + x0, cache)) > height and n_lo < max_steps_out:
            n_lo += 1
            lower -= sigma
        while (yield from _lp_step(direction * upper + x0, cache)) > height and n_hi < max_steps_out:
            n_hi += 1
            upper += sigma
    covered = s1 if (n_lo == 0 and n_hi == 0) else 0
    it = 0
    while True:
        if s2 > 0 and it >= covered:
            cache = yield from _prefetch_step([direction * z + x0 for z in _peek_shrink(lower, upper, s2, rs)])
            covered = it + s2
        z = (upper - lower) * rs.rand() + lower
        val = yield from _lp_step(direction * z + x0, cache)
        it += 1
        if val > height:
            return z * direction + x0
        if z < 0:
            lower = z
        elif z > 0:
            upper = z
        else:
            raise Exception("Slice sampler shrank to zero!")


def slice_steps(init_x, rs, speculate=(SPECULATE, 0), sigma=1.0, step_out=True, max_steps_out=1000, compwise=False):
    """Generator form of slice_sample drawing from the RandomState ``rs``; its return value is the new point."""
    init_x = np.asarray(init_x, dtype=float)
    if not init_x.shape:
        init_x = np.array([init_x])
    dims = init_x.shape[0]
    if compwise:
        order = list(range(dims))
        rs.shuffle(order)
        x = init_x.copy()
        for d in order:
            e = np.zeros(dims)
            e[d] = 1.0
            x = yield from _slice_along_steps(e, x, rs, sigma, step_out, max_steps_out, speculate)
        return x
    direction = rs.randn(dims)
    direction = direction / np.sqrt(np.sum(direction ** 2))
    return (yield from _slice_along_steps(direction, init_x, rs, sigma, step_out, max_steps_out, speculate))


def with_priors(steps, hypers_of):
    """Runs a slice_steps generator on a log-probability made of ``hypers_of`` (CachedLogProb's map) and a GP
    log-likelihood: yields the (mean, noise, amp2, ls) items whose log-likelihoods it needs (never an empty list),
    expects their values sent back (NaN: not positive definite) and returns the sampler's result."""
    try:
        points = next(steps)
        while True:
            maps = [hypers_of(np.asarray(x, dtype=float)) for x in points]
            todo = [h[0] for h in maps if h is not None]
            lls = iter((yield todo) if todo else ())
            lps = []
            for h in maps:
                if h is None:
                    lps.append(-np.inf)
                    continue
                v = next(lls)
                for t in h[1]:                   # prior terms in the reference's order of addition
                    v = v + t
                lps.append(v)
            points = steps.send(lps)
    except StopIteration as stop:
        return stop.value


class CachedLogProb(object):
    """A slice-sampler log-probability = prior part (host) + GP log-likelihood (GPU), with a per-move cache so that
    the points handed to ``prefetch`` are evaluated in one batched GPU call.  ``hypers_of(x)`` maps a sampler point to
    ``None`` (prior is -inf, no likelihood evaluation -- exactly the reference's early returns) or to
    ``((mean, noise, amp2, ls), (prior_term, ...))`` -- the terms are added in the given order."""

    def __init__(self, loglik, hypers_of):
        self.ll, self.hypers_of = loglik, hypers_of
        self.cache = {}
        self.speculate = getattr(loglik, "speculate", (SPECULATE, 0))    # (phase 1, phase 2) depth, see _slice_along

    @staticmethod
    def _key(x):
        return np.ascontiguousarray(x, dtype=np.float64).tobytes()

    def prefetch(self, points):
        self.cache = {}
        todo, keys, priors = [], [], []
        for x in points:
            k = self._key(x)
            if k in self.cache or k in keys:
                continue
            h = self.hypers_of(np.asarray(x, dtype=float))
            if h is None:
                self.cache[k] = -np.inf
            else:
                todo.append(h[0])
                keys.append(k)
                priors.append(h[1])
        if todo:
            vals = self.ll.batch(todo)
            for k, v, p in zip(keys, vals, priors):
                for t in p:                      # prior terms in the reference's order of addition
                    v = v + t
                self.cache[k] = v                # NaN (not PD) stays NaN and is raised on use

    def __call__(self, x):
        k = self._key(x)
        if k in self.cache:
            v = self.cache[k]
            if np.isnan(v):
                raise np.linalg.LinAlgError("leading minor of the array is not positive definite")
            return v
        h = self.hypers_of(np.asarray(x, dtype=float))
        if h is None:
            return -np.inf
        v = self.ll(*h[0])
        for t in h[1]:
            v = v + t
        return v


def make_logprob(loglik, hypers_of):
    """CachedLogProb (batched, speculative) when the log-likelihood can batch, else the plain sequential callable."""
    if hasattr(loglik, "batch"):
        return CachedLogProb(loglik, hypers_of)

    def logprob(x):
        h = hypers_of(np.asarray(x, dtype=float))
        if h is None:
            return -np.inf
        v = loglik(*h[0])
        for t in h[1]:
            v = v + t
        return v
    return logprob
