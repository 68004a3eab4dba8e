"""ctypes binding of libspearmint_b200.so (the C ABI declared in include/spearmint_b200.h).

There is NO CPU fallback: if the shared library cannot be built/loaded this module raises, and
every wrapper raises on a non-zero status.  torch is used by callers only to own device memory
and streams; the signatures here are plain pointers and sizes.
"""
import ctypes as C
import os

import numpy as np

from . import build as _build

KINDS = {"SE": 0, "ARDSE": 1, "Matern32": 2, "Matern52": 3}
ERR_NOT_PD = 1
ERR_CUDA = 1000

_lib = None


class SmkError(RuntimeError):
    pass


def lib():
    global _lib
    if _lib is None:
        path = _build.build()
        if not os.path.exists(path):
            raise SmkError("libspearmint_b200.so is missing (%s); the CUDA path has no fallback" % path)
        L = C.CDLL(path)
        _declare(L)
        _lib = L
    return _lib


_p = C.c_void_p
_i = C.c_int
_ll = C.c_longlong
_sz = C.c_size_t

# name -> argtypes (the exported symbol list checked by tests/test_abi.py against the header)
SIGNATURES = {
    "smk_version": ([], _i),
    "smk_npad": ([_i], _i),
    "smk_block": ([_i], _i),
    "smk_launch_count": ([], _ll),
    "smk_last_error": ([], C.c_char_p),
    "smk_timing_enable": ([_i], None),
    "smk_timing_ms": ([C.c_char_p, _p], C.c_double),
    "smk_predict_workspace_bytes": ([_i, _i], _sz),
    "smk_topk_workspace_bytes": ([_i, _i], _sz),
    "smk_ei_over_hypers_host_f32": ([_i, _i, _i, _i, _i] + [_p] * 9, _i),
    "smk_potrf_loglik_workspace_bytes": ([_i, _i], _sz),
    "smk_potrf_loglik_f64": ([_i, _i, _p, _p, _sz, _p, _i, _p], _i),
    "smk_loglik_small_f64": ([_i] * 4 + [_p] * 10, _i),
    "smk_tc_guard_workspace_bytes": ([_i, _i], _sz),
    "smk_tc_guard_f32": ([_i] * 4 + [_p] * 8 + [_sz, _p], _i),
    "smk_ei_colsum": ([_i, _i, _p, _i, _p, _p], _i),
    "smk_tc_np": ([_i], _i),
    "smk_trtri_workspace_bytes": ([_i, _i], _sz),
    "smk_trtri_split_f32": ([_i, _i, _i, _p, _p, _p, _p, _p, _sz, _p], _i),
    "smk_predict_tc_workspace_bytes": ([_i, _i, _i, _i], _sz),
    "smk_potrf_lower_batched_tc_f32": ([_i, _i, _p, _p, _p, _p, _sz, _p], _i),
    "smk_trtri_tc_workspace_bytes": ([_i, _i, _i], _sz),
    "smk_trtri_split_tc_f32": ([_i, _i, _i, _p, _p, _p, _p, _p, _sz, _p], _i),
    "smk_potrf_trtri_tc_f32": ([_i, _i, _i, _p, _p, _p, _p, _sz, _p, _p, _p, _sz, _p], _i),
    "smk_linv_alpha_f32": ([_i, _i, _i, _p, _p, _p, _p, _p, _i, _p, _p], _i),
    "smk_kxt_pack_workspace_bytes": ([_i, _i, _i], _sz),
    "smk_debug_kxt_tc_timeline": ([_p, _i], _i),
    "smk_kxt_pack_f16": ([_i] * 7 + [_p] * 6 + [_i, _p, _p, _p, _i, _p, _sz, _p], _i),
    "smk_linv_pack_f16": ([_i, _i, _p, _p, _p, _p, _p, _p], _i),
    "smk_predict_tc_f32": ([_i] * 6 + [_p] * 9 + [_i, _p, _p, _i, _p, _sz, _p, _i, _p, _p, _p, _i, _p], _i),
    "smk_predict_tc_pregen_f32": ([_i] * 6 + [_p] * 5 + [_sz, _i, _p], _i),
    "smk_predict_mma_f64": ([_i] * 6 + [_p] * 10 + [_i, _p, _sz, _p], _i),
    "smk_lower_matvec_f64": ([_i, _i, _p, _p, _p, _p], _i),
    "smk_forest_workspace_bytes": ([_i, _i, _i], _sz),
    "smk_forest_fit_f64": ([_i] * 3 + [_p] * 4 + [_i] * 4 + [_p] * 7 + [_p, _sz, _p], _i),
    "smk_forest_predict_ei_f64": ([_i] * 4 + [_p] * 6 + [C.c_double, _p, _p, _p, _p], _i),
}
for _t in ("f32", "f64"):
    SIGNATURES.update({
        "smk_sobol_generate_" + _t: ([_i, _ll, _ll, _p, _p, _p], _i),
        "smk_mll_grad_terms_" + _t: ([_i, _i, _i, _i, _p, _p, _p, _i, _p, _i, _p, _p], _i),
        "smk_cov_build_" + _t: ([_i] * 5 + [_p] * 6 + [_i, _p], _i),
        "smk_cov_build_lower_" + _t: ([_i] * 4 + [_p] * 5 + [_i, _p], _i),
        "smk_potrf_lower_batched_" + _t: ([_i, _i, _p, _p, _p, _p], _i),
        "smk_chol_solve_" + _t: ([_i] * 4 + [_p, _p, _p, _ll, _i, _p, _p, _p, _p, _p], _i),
        "smk_chol_solve_gm_" + _t: ([_i] * 4 + [_p, _p, _p, _ll, _i, _p, _p, _p, _p, _p], _i),
        "smk_loglik_set_rhs_" + _t: ([_i, _i, _i, _p, _p, _p, _p], _i),
        "smk_loglik_finish_" + _t: ([_i, _i, _i, _p, _p, _p, _p], _i),
        "smk_predict_" + _t: ([_i] * 6 + [_p] * 10 + [_i, _p, _sz, _p], _i),
        "smk_cross_mean_" + _t: ([_i] * 7 + [_p] * 7 + [_i, _p], _i),
        "smk_ei_sweep_" + _t: ([_i, _i, _i, _p, _p, _i, _p, _p, _p, _p, _p, _p], _i),
        "smk_topk_" + _t: ([_i, _i, _p, _p, _p, _p, _sz, _p], _i),
        "smk_ei_grad_terms_" + _t: ([_i] * 7 + [_p] * 8, _i),
        "smk_loglik_set_rhs_batched_" + _t: ([_i, _i, _i, _p, _i, _p, _p], _i),
        "smk_constraint_prob_" + _t: ([_i] * 6 + [_p] * 8 + [_i, _p], _i),
        "smk_ei_sweep_weighted_" + _t: ([_i, _i, _i, _p, _p, _i, _p, _p, _p, _p, _p, _p], _i),
    })


def _declare(L):
    for name, (args, res) in SIGNATURES.items():
        try:
            fn = getattr(L, name)
        except AttributeError:
            raise SmkError("libspearmint_b200.so does not export %s" % name)
        fn.argtypes = args
        fn.restype = res


def check(rc, what):
    if rc == 0:
        return
    if rc == ERR_NOT_PD:
        raise np.linalg.LinAlgError("%s: matrix is not positive definite" % what)
    if rc >= ERR_CUDA:
        raise SmkError("%s: CUDA error: %s" % (what, lib().smk_last_error().decode()))
    raise SmkError("%s: bad argument #%d" % (what, -rc))


def suffix(dtype):
    import torch
    return "f64" if dtype == torch.float64 else "f32"


def fn(name, dtype):
    return getattr(lib(), "%s_%s" % (name, suffix(dtype)))


def ptr(t):
    """Device pointer of a torch tensor (or NULL)."""
    return None if t is None else C.c_void_p(t.data_ptr())
