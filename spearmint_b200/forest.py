"""Random-forest regressor on the GPU (RandomForestEIChooser's model, RF = chooser/RandomForestEIChooser.py).

``draws`` takes the forest's randomness from numpy's RNG exactly as scikit-learn's RandomForestRegressor.fit does, so
that the host RNG ends where the reference leaves it; ``DeviceForest`` grows the trees from those draws
(smk_forest_fit_f64) and evaluates mean, variance and EI at candidates (smk_forest_predict_ei_f64).  The node arrays
stay in HBM between the fit and the predictions.
"""
import numpy as np
import numpy.random as npr
import torch

from . import _lib
from ._lib import check, ptr

MAX_INT = np.iinfo(np.int32).max       # sklearn.ensemble._forest.MAX_INT: the range of the per-tree seeds
RAND_R_MAX = 0x7FFFFFFF                # sklearn.tree._utils.RAND_R_MAX


def draws(n_trees, N, random_state=None):
    """(weights [T][N] float64, rand_r [T] uint32) of one fit: per tree, a seed s = rs.randint(MAX_INT) in tree order
    from the global RNG (random_state None) or from a fresh RandomState(random_state); the bootstrap counts
    bincount(RandomState(s).randint(0, N, N)) are the tree's sample weights and RandomState(s).randint(0, RAND_R_MAX)
    its splitter's rand_r state."""
    rs = npr if random_state is None else npr.RandomState(random_state)
    seeds = [rs.randint(MAX_INT) for _ in range(n_trees)]
    weights = np.empty((n_trees, N))
    states = np.empty(n_trees, dtype=np.uint32)
    for t, s in enumerate(seeds):
        weights[t] = np.bincount(npr.RandomState(s).randint(0, N, N), minlength=N)
        states[t] = npr.RandomState(s).randint(0, RAND_R_MAX)
    return weights, states


class DeviceForest(object):
    """T regression trees grown on ``device`` from host draws.  ``tree(t)`` returns one tree's node arrays."""

    def __init__(self, device, stream, X, y, weights, rand_r_states, max_features, max_depth=None,
                 min_samples_split=2):
        X = np.ascontiguousarray(X, dtype=np.float32)
        N, D = X.shape
        T = weights.shape[0]
        self.device, self.stream, self.N, self.D, self.T = device, stream, N, D, T
        self.ldn = 2 * N - 1
        dev = torch.device(device)
        Xd = torch.from_numpy(X).to(dev)
        yd = torch.from_numpy(np.ascontiguousarray(y, dtype=np.float64)).to(dev)
        wd = torch.from_numpy(np.ascontiguousarray(weights, dtype=np.float64)).to(dev)
        rd = torch.from_numpy(np.ascontiguousarray(rand_r_states, dtype=np.uint32).view(np.int32)).to(dev)
        shape = (T, self.ldn)
        self.feature = torch.empty(shape, dtype=torch.int32, device=dev)
        self.left = torch.empty(shape, dtype=torch.int32, device=dev)
        self.right = torch.empty(shape, dtype=torch.int32, device=dev)
        self.n_node_samples = torch.empty(shape, dtype=torch.int32, device=dev)
        self.threshold = torch.empty(shape, dtype=torch.float64, device=dev)
        self.value = torch.empty(shape, dtype=torch.float64, device=dev)
        self.node_count = torch.empty((T,), dtype=torch.int32, device=dev)
        L = _lib.lib()
        nb = L.smk_forest_workspace_bytes(N, D, T)
        ws = torch.empty((nb,), dtype=torch.uint8, device=dev)
        md = MAX_INT if max_depth is None else int(max_depth)
        check(L.smk_forest_fit_f64(N, D, T, ptr(Xd), ptr(yd), ptr(wd), ptr(rd), int(max_features), md,
                                   int(min_samples_split), self.ldn, ptr(self.feature), ptr(self.threshold),
                                   ptr(self.left), ptr(self.right), ptr(self.n_node_samples), ptr(self.value),
                                   ptr(self.node_count), ptr(ws), nb, stream), "forest_fit")
        self._keep = (Xd, yd, wd, rd, ws)          # inputs and workspace live until the stream has used them

    def predict(self, C, best=0.0, want=("mean", "var", "ei")):
        """dict of float64 device tensors [M] (RF:16-26; EI of RF:80-85 against ``best``)."""
        C = np.ascontiguousarray(C, dtype=np.float32)
        M = C.shape[0]
        dev = torch.device(self.device)
        Cd = torch.from_numpy(C).to(dev)
        out = {k: torch.empty((M,), dtype=torch.float64, device=dev) for k in want}
        check(_lib.lib().smk_forest_predict_ei_f64(M, self.D, self.T, self.ldn, ptr(Cd), ptr(self.feature),
                                                    ptr(self.threshold), ptr(self.left), ptr(self.right),
                                                    ptr(self.value), float(best), ptr(out.get("mean")),
                                                    ptr(out.get("var")), ptr(out.get("ei")), self.stream),
              "forest_predict_ei")
        return out

    def tree(self, t):
        n = int(self.node_count[t].item())
        return {k: getattr(self, k)[t, :n].cpu().numpy() for k in
                ("feature", "threshold", "left", "right", "n_node_samples", "value")}
