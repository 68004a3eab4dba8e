"""Sobol candidate grid on the GPU: drop-in for the reference's ``sobol_lib.i4_sobol_generate``
(spearmint/spearmint/sobol_lib.py:125-156; callers ExperimentGrid.py:192-196 and spearmint-lite.py:171-173).

    i4_sobol_generate(m, n, skip) -> (m, n) float64 ndarray        same signature, same values
    sobol_grid(dims, size, seed)  -> (size, dims)                   what ExperimentGrid keeps (= the transpose)

The points are produced by one CUDA kernel (csrc/sobol.cu) from the direction-number matrix the reference builds from
its Joe-Kuo table (data/sobol_v_1111x30.npy; different from scipy.stats.qmc.Sobol for dimensions >= 3, so candidate
indices stay meaningful across the two implementations).  No CPU fallback: raises without CUDA / the shared library.
"""
import ctypes as C
import os

import numpy as np

from . import _lib

_V_host = None
_V_dev = {}


def _directions(device):
    import torch
    global _V_host
    if _V_host is None:
        _V_host = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "data", "sobol_v_1111x30.npy"))
    key = str(device)
    if key not in _V_dev:
        _V_dev[key] = torch.from_numpy(_V_host.astype(np.int32)).to(device)     # same 32 bits; torch has no uint32 copies
    return _V_dev[key]


def sobol_device(dims, size, skip, device=None, dtype=None):
    """(size, dims) torch tensor on the device (row-major, what the engine's candidate buffer wants)."""
    import torch
    if not torch.cuda.is_available():
        raise _lib.SmkError("spearmint_b200.sobol needs a CUDA device (H100, sm_90a); there is no CPU fallback")
    device = torch.device(device if device is not None else "cuda:%d" % torch.cuda.current_device())
    dtype = dtype or torch.float64
    if not 1 <= dims <= 1111:
        raise ValueError("I4_SOBOL: the spatial dimension should satisfy 1 <= DIM_NUM <= 1111")
    V = _directions(device)
    out = torch.empty((size, dims), dtype=dtype, device=device)
    st = C.c_void_p(torch.cuda.current_stream(device).cuda_stream)
    _lib.check(_lib.fn("smk_sobol_generate", dtype)(dims, size, skip, _lib.ptr(V), _lib.ptr(out), st), "sobol_generate")
    return out


def i4_sobol_generate(m, n, skip, device=None):
    """The reference's signature and return value: (m, n) float64, column j = j-th point."""
    return sobol_device(m, n, skip, device).t().contiguous().cpu().numpy()


def sobol_grid(dims, size, seed, device=None):
    """ExperimentGrid's grid (GRID:192-196): (size, dims) float64."""
    return sobol_device(dims, size, seed, device).cpu().numpy()
