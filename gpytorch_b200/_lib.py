"""ctypes binding of libgpbbmm.so (the C ABI declared in include/gp_bbmm.h).

The library is the product; there is no Python or CPU fallback.  If the shared object is missing or
cannot be loaded, importing the ops raises immediately (the driver checks that GPU tests do not pass on
a silent fallback).
"""
from __future__ import annotations

import ctypes as C
import os
import warnings

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("GPBBMM_LIB") or os.path.join(_HERE, "lib", "libgpbbmm.so")   # GPBBMM_LIB: see INTEGRATION.md

GP_OK, GP_E_SHAPE, GP_E_CUDA, GP_E_NAN_MVM, GP_W_NOT_CONVERGED, GP_W_PIVCHOL_NAN, GP_E_NCCL, GP_E_STATE, GP_W_EIG_NOT_CONVERGED = range(9)
GP_RBF, GP_MATERN12, GP_MATERN32, GP_MATERN52, GP_RQ, GP_POLY, GP_PPOLY = range(7)
GP_BACKEND_AUTO, GP_BACKEND_TCGEN05, GP_BACKEND_SIMT, GP_BACKEND_SKI, GP_BACKEND_SUM, GP_BACKEND_KRON, GP_BACKEND_DERIV, GP_BACKEND_PRODUCT, \
    GP_BACKEND_COMPACT = range(9)
KIND = {"rbf": GP_RBF, "matern12": GP_MATERN12, "matern32": GP_MATERN32, "matern52": GP_MATERN52, "rq": GP_RQ, "poly": GP_POLY,
        "ppoly": GP_PPOLY}
BACKEND = {"auto": GP_BACKEND_AUTO, "tcgen05": GP_BACKEND_TCGEN05, "simt": GP_BACKEND_SIMT}


class NumericalWarning(RuntimeWarning):
    """Mirror of gpytorch.utils.warnings.NumericalWarning (utils/warnings.py:5)."""


class NanError(RuntimeError):
    """Mirror of gpytorch.utils.errors.NanError (utils/errors.py:8-22)."""


class NotPSDError(RuntimeError):
    """Mirror of linear_operator.utils.errors.NotPSDError (re-exported by gpytorch/utils/errors.py): a Cholesky factorisation
    failed even after adding jitter to the diagonal."""


class MllOpts(C.Structure):
    _fields_ = [
        ("num_probes", C.c_int),
        ("precond_rank", C.c_int),
        ("min_precond_size", C.c_int),
        ("precond_tol", C.c_float),
        ("cg_tol", C.c_float),
        ("max_cg_iter", C.c_int),
        ("max_tridiag_iter", C.c_int),
    ]


class MllResult(C.Structure):
    _fields_ = [
        ("inv_quad", C.c_double),
        ("logdet", C.c_double),
        ("logdet_precond", C.c_double),
        ("log_prob", C.c_double),
        ("mll", C.c_double),
        ("cg_iters", C.c_int),
        ("tridiag_size", C.c_int),
        ("precond_rank", C.c_int),
        ("status_flags", C.c_int),
        ("resid", C.c_float * 16),
    ]


_P, _I, _L, _F = C.c_void_p, C.c_int, C.c_int64, C.c_float
# name -> (restype, argtypes); must list every symbol declared in include/gp_bbmm.h
PROTOTYPES = {
    "gp_version": (C.c_char_p, []),
    "gp_last_error": (C.c_char_p, []),
    "gp_status_string": (C.c_char_p, [_I]),
    "gp_plan_create": (_I, [C.POINTER(_P), _I, _P]),
    "gp_plan_destroy": (_I, [_P]),
    "gp_plan_set_backend": (_I, [_P, _I]),
    "gp_plan_set_data": (_I, [_P, _P, _L, _L, _P, _L, _L, _I, _L, _L]),
    "gp_plan_set_hypers": (_I, [_P, _I, C.POINTER(_F), _I, _F, _F]),
    "gp_plan_set_noise_diag": (_I, [_P, _P, _L]),
    "gp_plan_set_ski": (_I, [_P, C.POINTER(_I), C.POINTER(_F), C.POINTER(_F), _I]),
    "gp_plan_set_sum": (_I, [_P, C.POINTER(_P), _I]),
    "gp_plan_set_product": (_I, [_P, C.POINTER(_P), _I]),
    "gp_plan_set_additive": (_I, [_P, _I, C.POINTER(_F), _I]),
    "gp_plan_set_spectral": (_I, [_P, _I, C.POINTER(_F), C.POINTER(_F), C.POINTER(_F), _I]),
    "gp_plan_set_periodic": (_I, [_P, C.POINTER(_F), _I, _I]),
    "gp_plan_set_hypers_rq": (_I, [_P, C.POINTER(_F), _I, _F, _F, _F]),
    "gp_plan_set_hypers_poly": (_I, [_P, _I, _F, _F, _F]),
    "gp_plan_set_hypers_pp": (_I, [_P, _I, C.POINTER(_F), _I, _F, _F]),
    "gp_plan_tile_pairs": (_I, [_P, C.POINTER(_L), C.POINTER(_L)]),
    "gp_plan_set_lowrank": (_I, [_P, _P, _L, _I]),
    "gp_plan_set_tasks": (_I, [_P, _P, _P, _I]),
    "gp_plan_set_task_covar": (_I, [_P, C.POINTER(_F), _I]),
    "gp_task_covar_grad": (_I, [_P, _P, _L, _P, _L, _I, C.POINTER(C.c_double)]),
    "gp_plan_set_kron": (_I, [_P, _P, _I]),
    "gp_plan_set_kron_observed": (_I, [_P, _P, _L, _P, _L]),
    "gp_plan_set_kron_terms": (_I, [_P, C.POINTER(_P), _I, _I]),
    "gp_plan_set_kron_term_covars": (_I, [_P, C.POINTER(_F), _I, _I]),
    "gp_kron_terms_grad": (_I, [_P, _P, _L, _P, _L, _I, C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_double)]),
    "gp_plan_set_deriv": (_I, [_P, _P]),
    "gp_plan_set_deriv_kind": (_I, [_P, _P, _I]),
    "gp_ski_grid_matmul": (_I, [_P, _P, _L, _I, _P, _L]),
    "gp_ski_interp_matmul": (_I, [_P, _P, _L, _I, _P, _L]),
    "gp_ski_input_grad": (_I, [_P, _P, _L, _P, _L, _I, _P, _L]),
    "gp_kmv": (_I, [_P, _P, _L, _I, _P, _L, _I]),
    "gp_krows": (_I, [_P, _P, _L, _P, _L]),
    "gp_kdiag": (_I, [_P, _P]),
    "gp_bilinear_grad": (_I, [_P, _P, _L, _P, _L, _I, C.POINTER(C.c_double), C.POINTER(C.c_double)]),
    "gp_kmv_input_grad": (_I, [_P, _P, _L, _P, _L, _I, _P, _L, _P, _L]),
    "gp_kdense_input_grad": (_I, [_P, _P, _L, _P, _L, _P, _L]),
    "gp_pivoted_cholesky": (_I, [_P, _I, _F, _P, _P, C.POINTER(_I)]),
    "gp_precond_build": (_I, [_P, _P, _I, _P, C.POINTER(C.c_double)]),
    "gp_precond_probes": (_I, [_P, _P, _I, _P, _P, _I, _P]),
    "gp_mbcg": (_I, [_P, _P, _L, _I, _I, _F, _I, _I, _P, _I, _P, _L, _P, C.POINTER(_I), C.POINTER(_I), C.POINTER(_F)]),
    "gp_slq_logdet": (_I, [_P, _P, _I, _I, _I, _L, C.POINTER(C.c_double)]),
    "gp_lanczos": (_I, [_P, _P, _I, _F, _P, _P, C.POINTER(_I)]),
    "gp_ciq_sqrt_matmul": (_I, [_P, _P, _L, _I, C.POINTER(C.c_double), C.POINTER(C.c_double), _I, _F, _I, _P, _L,
                                C.POINTER(_I), C.POINTER(_F)]),
    "gp_ciq_precond_build": (_I, [_P, _P, _I, _P, C.POINTER(C.c_double)]),
    "gp_ciq_sqrt_matmul_precond": (_I, [_P, _P, _L, _I, _P, _I, C.POINTER(C.c_double), C.POINTER(C.c_double), _I, _F, _I, _P,
                                        _L, C.POINTER(_I), C.POINTER(_F)]),
    "gp_mll": (_I, [_P, _P, _P, _P, _P, C.POINTER(MllOpts), _P, C.POINTER(MllResult)]),
    "gp_comm_unique_id": (_I, [C.POINTER(C.c_uint8)]),
    "gp_comm_init": (_I, [C.POINTER(_P), C.POINTER(C.c_uint8), _I, _I]),
    "gp_comm_destroy": (_I, [_P]),
    "gp_plan_set_comm": (_I, [_P, _P]),
    "gp_kernel_launches": (_L, [_P]),
    "gp_plan_info": (_I, [_P, C.POINTER(_I), C.POINTER(_I), C.POINTER(_I), C.POINTER(_I)]),
    "gp_time_kmv_kernel": (_I, [_P, _P, _L, _I, _I, _I, C.POINTER(_F)]),
}

_lib = None


def load():
    """Load libgpbbmm.so and bind the prototypes.  Raises if the extension is missing."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} not found: build it with `python -m gpytorch_b200.build` "
            "(gpytorch_b200 has no CPU / PyTorch fallback)"
        )
    lib = C.CDLL(LIB_PATH, mode=C.RTLD_GLOBAL)
    for name, (res, args) in PROTOTYPES.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def last_error() -> str:
    return load().gp_last_error().decode()


def check(status: int, warn: bool = True) -> int:
    """Map a C status to the reference's exception / warning classes (SURVEY.md section 8b Errors)."""
    if status == GP_OK:
        return status
    msg = last_error()
    if status == GP_W_NOT_CONVERGED:
        if warn:
            warnings.warn(msg, NumericalWarning)
        return status
    if status in (GP_W_PIVCHOL_NAN, GP_W_EIG_NOT_CONVERGED):
        if warn:
            warnings.warn(msg, NumericalWarning)
        return status
    if status == GP_E_NAN_MVM:
        raise RuntimeError(msg)
    raise RuntimeError(f"libgpbbmm: {load().gp_status_string(status).decode()}: {msg}")
