"""Independent hyper-parameter chains run in lockstep (the ``mcmc_chains`` option of GPEIOptChooserB200).

Each chain is the single chain's sampler -- the same joint and length-scale slice moves, priors, strict ``>``
acceptance and speculation (util.slice_steps) -- drawing from a numpy RandomState of its own.  A chain's moves are
generators that yield the (mean, noise, amp2, ls) items they need evaluated; ``lockstep`` collects the outstanding items
of every active chain, evaluates them with ONE log-likelihood ``batch`` call per round and resumes each chain with its
values.  Chains finish at different rounds.  A non positive definite item (NaN) raises LinAlgError where the
single-chain sampler would raise it.

The log-likelihood of an item is bitwise independent of the batch it rides in (engine.ChainLogLik), so a chain's draws
are the same whether it runs alone or with others, and on whichever rank it runs: under torchrun, chain c runs on rank
c mod W and the finished chains are exchanged in one all-gather.
"""
import numpy as np
import numpy.random as npr

from spearmint_b200 import parallel, util
from spearmint_b200.locker import log


class Chain(object):
    """One chain: its current hyper-parameters, its RandomState, and whether it still has to burn in."""

    def __init__(self, index, hypers, rs, needs_burnin):
        self.index = index
        self.mean, self.noise, self.amp2, self.ls = hypers
        self.rs, self.needs_burnin = rs, needs_burnin
        self.samples, self.evals = [], 0

    @classmethod
    def seeded(cls, K, hypers):
        """K chains starting from ``hypers``, each to burn in.  The seeds are K draws of npr.randint(2**32) from the
        global RNG -- the only global draws the chains ever make."""
        seeds = npr.randint(2 ** 32, size=K)
        return [cls(c, hypers, npr.RandomState(int(s)), True) for c, s in enumerate(seeds)]

    @classmethod
    def from_state(cls, index, state):
        """A chain resumed from its ``state()``: no burn-in."""
        rs = npr.RandomState()
        rs.set_state(state[4])
        return cls(index, state[:4], rs, False)

    def state(self):
        """(mean, noise, amp2, ls, RandomState state): the chain's entry in the ``chains`` key of the state pickle."""
        return (self.mean, self.noise, self.amp2, self.ls, self.rs.get_state())

    def _step(self, prior, targets, noiseless, speculate):
        """One sample_hypers of the single chain (GPEIOptChooserB200.sample_hypers) as a generator."""
        if noiseless:
            self.noise = 1e-3
        self.mean, self.amp2, self.noise = yield from prior.joint_steps(self.rs, self.mean, self.amp2, self.noise,
                                                                        self.ls, targets, noiseless, speculate)
        self.ls = yield from prior.length_scales_steps(self.rs, self.mean, self.noise, self.amp2, self.ls, speculate)

    def _line(self):
        return "mean: %.2f  amp: %.2f  noise: %.4f min_ls: %.4f  max_ls: %.4f" % (
            self.mean, np.sqrt(self.amp2), self.noise, np.min(self.ls), np.max(self.ls))

    def run(self, prior, targets, noiseless, burnin, steps, speculate):
        """Burn-in (first call only), then ``steps`` samples kept in ``self.samples``; a generator for ``lockstep``."""
        if self.needs_burnin:
            for it in range(burnin):
                yield from self._step(prior, targets, noiseless, speculate)
                log("BURN chain %d %d/%d] %s" % (self.index, it + 1, burnin, self._line()))
            self.needs_burnin = False
        self.samples = []
        for it in range(steps):
            yield from self._step(prior, targets, noiseless, speculate)
            self.samples.append((self.mean, self.noise, self.amp2, self.ls))
            log("chain %d %d/%d] %s" % (self.index, it + 1, steps, self._line()))


def _key(item):
    return np.hstack([item[0], item[1], item[2], np.asarray(item[3], dtype=np.float64)]).astype(np.float64).tobytes()


def lockstep(runs, loglik, evals=None):
    """Drives the generators ``runs`` to completion, one ``loglik.batch`` call per round over the outstanding items of
    every active run, duplicates within a run evaluated once.  ``evals[i]`` (if given) counts run i's evaluations.
    Returns the number of rounds."""
    pending = {}
    for i, g in enumerate(runs):
        try:
            pending[i] = next(g)
        except StopIteration:
            pass
    rounds = 0
    while pending:
        items, where = [], {}
        for i, req in pending.items():
            seen, idx = {}, []
            for h in req:
                k = _key(h)
                if k not in seen:
                    seen[k] = len(items)
                    items.append(h)
                idx.append(seen[k])
            where[i] = idx
            if evals is not None:
                evals[i] += len(seen)
        vals = loglik.batch(items)
        rounds += 1
        for i in list(pending):
            try:
                pending[i] = runs[i].send([vals[j] for j in where[i]])
            except StopIteration:
                del pending[i]
    return rounds


def sample(chains, prior, loglik, targets, noiseless, burnin, steps):
    """Runs every chain (its burn-in if it needs one, then ``steps`` samples) and returns the samples round-major:
    step r of chain 0, step r of chain 1, ...  Under torchrun this rank runs chains rank, rank + W, ... in lockstep;
    every rank then holds every chain's samples and state.  Returns (hyper_samples, rounds of this rank)."""
    rank, world = parallel.world()
    mine = [chains[c] for c in parallel.shard(len(chains), rank, world)]
    speculate = getattr(loglik, "speculate", (util.SPECULATE, 0))
    device = getattr(loglik, "device", "cpu")       # a CPU stand-in log-likelihood exchanges over gloo
    evals = [0] * len(mine)
    err, rounds = None, 0
    try:
        rounds = lockstep([c.run(prior, targets, noiseless, burnin, steps, speculate) for c in mine], loglik, evals)
    except Exception as e:                          # every rank raises, or the others would wait in the all-gather
        err = e
    parallel.agree_on_error(err, device)
    for c, n in zip(mine, evals):
        c.evals = n
    done = [(c.index, c.samples, c.state(), c.evals) for c in mine]
    for part in parallel.allgather_object(done, device):
        for index, samples, state, n in part:
            c = chains[index]
            c.mean, c.noise, c.amp2, c.ls = state[:4]
            c.rs.set_state(state[4])
            c.samples, c.evals, c.needs_burnin = samples, n, False
    return [chains[c].samples[r] for r in range(steps) for c in range(len(chains))], rounds
