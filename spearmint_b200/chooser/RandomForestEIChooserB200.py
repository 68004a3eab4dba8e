"""Drop-in replacement for the reference's ``chooser/RandomForestEIChooser.py`` (RF): expected improvement under a
random-forest regressor, the forest grown and evaluated on the GPU.

``next()`` (RF:50-90): with fewer than 2 complete jobs, ``candidates[0]``; otherwise fit ``n_trees`` regression trees
to the complete jobs, and with pending jobs fantasise them as ``m + sqrt(v) + randn(P)`` (the unit normal is added, not
scaled) and refit on complete + pending; then EI with ``s = sqrt(v) + 1e-4`` against the best COMPLETE value, and the
argmax over the candidates (numpy's first-max rule).  The trees are those scikit-learn 1.9 grows
(spearmint_b200/forest.py): the forest's randomness -- one seed per tree and fit, and from it the bootstrap counts and
the splitter state -- is drawn from numpy's global RNG in sklearn's order (from a fresh RandomState per fit when
``random_state`` is set, which leaves the global RNG alone).  With ``n_trees=1`` the variance is NaN, so the proposal is
``candidates[0]``, and a pending-point refit on NaN fantasies raises ValueError, as sklearn's does; so do NaN or inf
among the complete values.

Waived (DESIGN section 9): pending points are refit on ``vstack([comp, pend])`` / ``hstack([vals, vals_pend])`` (RF:72
indexes ``np.vstack`` and raises TypeError); options are cast from their arg-string form -- ``max_features="auto"`` is
all D features, ``min_samples_split`` below 2 is 2, as in the sklearn of the reference's time; ``n_jobs`` and
``max_monkeys`` are accepted and ignored.  Extra optional keys: ``device``.  No state files: the reference keeps none.
"""
import numpy as np
import numpy.random as npr

from spearmint_b200 import util
from spearmint_b200.chooser._gp import LazyBackend
from spearmint_b200.forest import draws


def init(expt_dir, arg_string):
    args = util.unpack_args(arg_string)
    return RandomForestEIChooserB200(**args)


def _none_or_int(v):
    return None if v is None or v == "None" else int(v)


def _max_features(v):
    """"auto" / "sqrt" / "log2" / None, an int ("3") or a fraction ("0.5") -- strings from the arg string included."""
    if v is None or v in ("auto", "sqrt", "log2", "None"):
        return None if v in (None, "None") else v
    if isinstance(v, str):
        return float(v) if any(c in v for c in ".eE") else int(v)
    return v


def resolve_max_features(max_features, D):
    """sklearn's max_features_ for a regressor; None / "auto" = all D features (the regressor meaning of 2013)."""
    if max_features is None or max_features == "auto":
        return D
    if max_features == "sqrt":
        return max(1, int(np.sqrt(D)))
    if max_features == "log2":
        return max(1, int(np.log2(D)))
    if isinstance(max_features, (int, np.integer)):
        return int(max_features)
    return max(1, int(float(max_features) * D))


class RandomForestEIChooserB200(LazyBackend):

    def __init__(self, n_trees=50, max_depth=None, min_samples_split=1, max_monkeys=7, max_features="auto", n_jobs=1,
                 random_state=None, device=None, backend=None):
        self.n_trees = int(n_trees)
        self.max_depth = _none_or_int(max_depth)
        self.min_samples_split = max(2, int(min_samples_split))
        self.max_features = _max_features(max_features)
        self.random_state = _none_or_int(random_state)
        self._device, self._backend = device, backend

    def _fit(self, X, y):
        if not np.all(np.isfinite(y)):       # sklearn validates y before it draws the seeds
            raise ValueError("Input y contains NaN or infinity.")
        weights, states = draws(self.n_trees, X.shape[0], self.random_state)
        return self.backend.forest_fit(X, y, weights, states, resolve_max_features(self.max_features, X.shape[1]),
                                       self.max_depth, self.min_samples_split)

    def next(self, grid, values, durations, candidates, pending, complete):
        if complete.shape[0] < 2:
            return int(candidates[0])
        comp = grid[complete, :]
        cand = grid[candidates, :]
        pend = grid[pending, :]
        vals = values[complete]

        forest = self._fit(comp, vals)
        if pend.shape[0] != 0:
            func_m, func_v = self.backend.forest_predict(forest, pend)
            with np.errstate(invalid="ignore"):
                vals_pend = func_m + np.sqrt(func_v) + npr.randn(func_m.shape[0])
            forest = self._fit(np.vstack([comp, pend]), np.hstack([vals, vals_pend]))

        best = np.min(vals)
        return int(candidates[self.backend.forest_argmax_ei(forest, cand, best)])
