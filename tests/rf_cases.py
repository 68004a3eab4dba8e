"""TEST INFRASTRUCTURE ONLY -- the inputs of the random-forest goldens (tests/golden/rf_*.npz), rebuilt from the
Sobol oracle so that nothing on a GPU machine needs the reference or sklearn.

The grid is the reference's Sobol sequence (distinct coordinates in every dimension, also in float32); the first N
points are complete, the next M candidates, the next P pending.  The objective has its minimum away from the origin.
"""
import numpy as np

from oracle import sobol_oracle

# name: (D, N, M, P, chooser kwargs, seed of the global RNG, calls)
CASES = {
    "rf_d2_defaults": (2, 20, 1000, 0, {}, 21, 1),
    "rf_d3_pending": (3, 60, 2000, 3, {}, 22, 1),
    "rf_d8_sqrt_depth6_rs3": (8, 300, 5000, 0, dict(max_features="sqrt", max_depth=6, random_state=3), 23, 1),
    "rf_d3_twocall": (3, 40, 1500, 0, {}, 24, 2),
    "rf_d32_n4096": (32, 4096, 20000, 0, {}, 25, 1),
}
SMALL = ("rf_d2_defaults", "rf_d3_pending", "rf_d8_sqrt_depth6_rs3", "rf_d3_twocall")
LARGE_SUBSET = 2000          # candidates whose mean / var / EI the large golden stores (evenly spaced)


def objective(x):
    return np.sum((x - 0.37) ** 2, axis=1) + 0.3 * np.sin(7.0 * x[:, 0]) * np.cos(3.0 * x[:, -1])


def inputs(name):
    """(grid, values, complete, candidates, pending) of the first call; a second call (calls == 2) adds candidate 0
    to the complete set."""
    D, N, M, P, _, _, _ = CASES[name]
    grid = sobol_oracle.i4_sobol_generate(D, N + M + P, 1).T.copy()
    values = objective(grid)
    complete = np.arange(N)
    candidates = np.arange(N, N + M)
    pending = np.arange(N + M, N + M + P)
    return grid, values, complete, candidates, pending


def second_call(grid, values, complete, candidates, pending, proposal):
    """The state of a second next() after job ``proposal`` completed."""
    complete = np.append(complete, proposal)
    candidates = candidates[candidates != proposal]
    return grid, values, complete, candidates, pending


def subset(M):
    return np.linspace(0, M - 1, LARGE_SUBSET).astype(np.int64)
