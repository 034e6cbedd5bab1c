"""ctypes binding of libagp.so -- a 1:1 mirror of include/agp.h (and of the ``ccall`` signatures in
julia/AGPBlackwell.jl).  Host side only: no arithmetic happens here, and there is NO CPU fallback --
if the library or a CUDA device is missing every compute entry point raises."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libagp.so")

AGP_F32, AGP_F64 = 0, 1
AGP_POINT_MAJOR, AGP_FEATURE_MAJOR = 0, 1
AGP_MEM_HOST, AGP_MEM_DEVICE = 0, 1
(AGP_OK, AGP_ERR_NOT_POSDEF, AGP_ERR_DIM_MISMATCH, AGP_ERR_UNSUPPORTED, AGP_ERR_CUDA, AGP_ERR_NCCL,
 AGP_ERR_INVALID) = range(7)


AGP_RQ, AGP_PERIODIC, AGP_WHITE, AGP_CONSTANT, AGP_COMPOSITE = 5, 6, 7, 8, 9
AGP_COMPOSITE_MAX = 8  # terms, and factors in all
AGP_PANEL_SPLIT_SUBST, AGP_PANEL_SPLIT_GEMM, AGP_PANEL_FUSED = 0, 1, 2


class agp_kernel_factor(C.Structure):
    _fields_ = [("family", C.c_int32), ("transform", C.c_int32), ("scale", C.c_double), ("param", C.c_double),
                ("ard", C.c_void_p), ("r", C.c_void_p)]


class agp_kernel_composite(C.Structure):
    _fields_ = [("nterms", C.c_int32), ("nfactors", C.POINTER(C.c_int32)), ("variance", C.POINTER(C.c_double)),
                ("factors", C.POINTER(agp_kernel_factor))]


class agp_kernel(C.Structure):
    _fields_ = [("family", C.c_int32), ("transform", C.c_int32), ("variance", C.c_double),
                ("scale", C.c_double), ("linear_c", C.c_double), ("ard", C.c_void_p),
                ("composite", C.POINTER(agp_kernel_composite))]


class agp_mean(C.Structure):
    _fields_ = [("kind", C.c_int32), ("c", C.c_double), ("v", C.c_void_p)]


class agp_noise(C.Structure):
    _fields_ = [("kind", C.c_int32), ("s", C.c_double), ("v", C.c_void_p)]


class agp_config(C.Structure):
    _fields_ = [("tile_nb", C.c_int32), ("fp64_mode", C.c_int32), ("fp32_mode", C.c_int32),
                ("lookahead", C.c_int32), ("use_graph", C.c_int32), ("ozaki_slices", C.c_int32),
                ("profile_kernels", C.c_int32), ("reserved", C.c_int32 * 9)]


# every symbol include/agp.h declares: name -> (restype, argtypes)
_P = C.c_void_p
_K, _M, _N = C.POINTER(agp_kernel), C.POINTER(agp_mean), C.POINTER(agp_noise)
SIGNATURES = {
    "agp_init": (C.c_int32, [C.POINTER(_P), C.c_int32, C.POINTER(agp_config)]),
    "agp_nccl_unique_id": (C.c_int32, [_P]),
    "agp_init_dist": (C.c_int32, [C.POINTER(_P), C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, _P,
                                  C.POINTER(agp_config)]),
    "agp_destroy": (C.c_int32, [_P]),
    "agp_last_error": (C.c_char_p, [_P]),
    "agp_last_info": (C.c_int64, [_P]),
    "agp_set_memspace": (C.c_int32, [_P, C.c_int32]),
    "agp_set_config": (C.c_int32, [_P, C.POINTER(agp_config)]),
    "agp_get_config": (C.c_int32, [_P, C.POINTER(agp_config)]),
    "agp_version": (C.c_char_p, []),
    "agp_last_timings": (C.c_int32, [_P, C.POINTER(C.c_double), C.c_int32]),
    "agp_launch_count": (C.c_int64, [_P]),
    "agp_gram": (C.c_int32, [_P, C.c_int32, _K, C.c_int32, _P, C.c_int64, C.c_int32, _P, C.c_int64, _N, _P]),
    "agp_fit": (C.c_int32, [_P, C.c_int32, _K, _M, _N, C.c_int32, _P, C.c_int64, C.c_int32, _P, C.c_int32, _P, _P,
                            C.POINTER(_P)]),
    "agp_post_mean_var": (C.c_int32, [_P, C.c_int32, _P, C.c_int64, _M, _N, _P, _P]),
    "agp_post_mean_cov": (C.c_int32, [_P, C.c_int32, _P, C.c_int64, _M, _P, _P]),
    "agp_post_logpdf": (C.c_int32, [_P, C.c_int32, _P, C.c_int64, _M, _N, _P, C.c_int32, _P]),
    "agp_post_rand": (C.c_int32, [_P, C.c_int32, _P, C.c_int64, _M, _N, _P, C.c_int32, _P]),
    "agp_post_logpdf_grad": (C.c_int32, [_P, C.POINTER(C.c_double), _P]),
    "agp_post_logpdf_grad_x": (C.c_int32, [_P, C.POINTER(C.c_double), _P, C.c_int32, _P]),
    "agp_post_logpdf_grad_cols": (C.c_int32, [_P, _M, _P, C.c_int32, C.POINTER(C.c_double), C.POINTER(C.c_double), _P, _P,
                                              C.c_int32, _P, _P]),
    "agp_post_pred_logpdf_grad": (C.c_int32, [_P, C.c_int32, _P, C.c_int64, _M, _N, _P, C.c_int32, C.POINTER(C.c_double), _P,
                                              C.POINTER(C.c_double), _P, _P, _P, _P, _P, _P, _P, _P]),
    "agp_post_rand_grad": (C.c_int32, [_P, C.c_int32, _P, C.c_int64, _M, _N, _P, C.c_int32, _P, C.POINTER(C.c_double), _P,
                                       _P, _P, _P, _P, _P, _P, _P]),
    "agp_post_mean_var_grad": (C.c_int32, [_P, C.c_int32, _P, C.c_int64, _P, _P, C.POINTER(C.c_double), _P, _P, _P, _P,
                                           _P]),
    "agp_post_grad_len": (C.c_int64, [_P]),
    "agp_post_solve_lower": (C.c_int32, [_P, _P, C.c_int64, _P]),
    "agp_post_factor_export": (C.c_int32, [_P, _P]),
    "agp_post_logdet": (C.c_int32, [_P, C.POINTER(C.c_double)]),
    "agp_post_n": (C.c_int64, [_P]),
    "agp_post_extend": (C.c_int32, [_P, C.c_int32, _P, C.c_int64, _P, _M, _N, _P, C.POINTER(_P)]),
    "agp_post_free": (C.c_int32, [_P]),
    "agp_rand": (C.c_int32, [_P, C.c_int32, _K, _M, _N, C.c_int32, _P, C.c_int64, C.c_int32, _P, C.c_int32, _P]),
    "agp_rand_grad": (C.c_int32, [_P, C.c_int32, _K, _M, _N, C.c_int32, _P, C.c_int64, C.c_int32, _P, C.c_int32, _P,
                                  C.POINTER(C.c_double), _P, _P, _P, _P]),
    "agp_vfe_elbo": (C.c_int32, [_P, C.c_int32, _K, _M, _N, C.c_int32, _P, C.c_int64, C.c_int32, _P, C.c_int64, _N,
                                 _P, _P, _P]),
    "agp_vfe_elbo_grad": (C.c_int32, [_P, C.c_int32, _K, _M, _N, C.c_int32, _P, C.c_int64, C.c_int32, _P, C.c_int64, _N,
                                      _P, C.c_int32, _P, C.POINTER(C.c_double), _P, _P, _P]),
    "agp_vfe_elbo_grad_x": (C.c_int32, [_P, C.c_int32, _K, _M, _N, C.c_int32, _P, C.c_int64, C.c_int32, _P, C.c_int64,
                                        _N, _P, C.c_int32, _P, C.POINTER(C.c_double), _P, _P, _P, _P]),
    "agp_vfe_fit": (C.c_int32, [_P, C.c_int32, _K, _M, _N, C.c_int32, _P, C.c_int64, C.c_int32, _P, C.c_int64, _N,
                                _P, C.POINTER(_P)]),
    "agp_vfe_mean_var": (C.c_int32, [_P, C.c_int32, _P, C.c_int64, _P, _P]),
    "agp_vfe_mean_cov": (C.c_int32, [_P, C.c_int32, _P, C.c_int64, _P, _P]),
    "agp_vfe_post_logpdf": (C.c_int32, [_P, C.c_int32, _P, C.c_int64, _N, _P, C.c_int32, _P]),
    "agp_vfe_post_rand": (C.c_int32, [_P, C.c_int32, _P, C.c_int64, _N, _P, C.c_int32, _P]),
    "agp_vfe_post_free": (C.c_int32, [_P]),
    "agp_debug_ozaki_syrk": (C.c_int32, [_P, _P, C.c_int64, _P, C.c_int64, C.c_int64, C.c_int64, C.c_int32, C.c_int32,
                                         C.c_int32]),
    "agp_debug_ozaki_gemm": (C.c_int32, [_P, _P, C.c_int32, C.c_int64, _P, C.c_int32, C.c_int32, C.c_int64, C.c_int64, _P, C.c_int32,
                                         C.c_int32, C.c_int64, C.c_int64, C.c_int32, C.c_int32, C.c_double]),
    "agp_debug_ozaki_syrk_map": (C.c_int32, [_P, _P, C.c_int64, _P, C.c_int64, C.c_int64, C.c_int64, C.c_int64, C.c_int32,
                                             C.c_int32, C.c_int64, C.c_int64, C.c_int64, C.c_int64]),
    "agp_debug_ozaki8": (C.c_int32, [_P, _P, C.c_int64, _P, C.c_int32, C.c_int64, C.c_int64, _P, C.c_int32, C.c_int64,
                                     C.c_int64, C.c_int64, C.c_int32, C.c_double, C.c_int64, C.c_int64, C.c_int64, C.c_int64]),
    "agp_debug_gemm": (C.c_int32, [_P, C.c_int32, _P, C.c_int32, C.c_int64, _P, C.c_int32, C.c_int64, _P, C.c_int64,
                                   C.c_int64, C.c_int64, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int64,
                                   C.c_int64, C.c_int64]),
    "agp_debug_panel": (C.c_int32, [_P, C.c_int32, C.c_int32, _P, C.c_int64, C.c_int64, C.c_int32, _P, _P, _P]),
    "agp_bc_owner": (C.c_int32, [C.c_int32, C.c_int32, C.c_int32, C.c_int32]),
    "agp_bc_local_tiles": (C.c_int64, [C.c_int32, C.c_int32, C.c_int32, C.c_int32]),
}

_lib = None


class AGPError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("libagp status %d: %s" % (code, msg))
        self.code = code


class PosDefException(AGPError):
    """Mirror of LinearAlgebra.PosDefException(info) thrown by cholesky(.) in the reference
    (/root/reference/src/finite_gp_projection.jl:308)."""

    def __init__(self, info, msg):
        AGPError.__init__(self, AGP_ERR_NOT_POSDEF, msg)
        self.info = info


class DimensionMismatch(ValueError):
    """Mirror of Julia's DimensionMismatch (/root/reference/src/sparse_approximations.jl:290-294)."""


def lib():
    """Load libagp.so (needs only libcudart / libnccl on the loader path, not a GPU)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError("libagp.so is not built: run `python __graft_entry__.py` (nvcc, sm_90a). "
                              "There is no CPU fallback.")
        try:  # make the torch-bundled libnccl visible first if torch is importable (same SONAME)
            import torch  # noqa: F401
        except Exception:
            pass
        _lib = C.CDLL(LIB_PATH, mode=C.RTLD_GLOBAL)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(_lib, name)
            fn.restype = res
            fn.argtypes = args
    return _lib


def np_dtype(code):
    return np.float64 if code == AGP_F64 else np.float32


def dtype_code(dt):
    dt = np.dtype(dt)
    if dt == np.float64:
        return AGP_F64
    if dt == np.float32:
        return AGP_F32
    raise TypeError("libagp supports float32/float64, got %s" % dt)


def ptr(a):
    if a is None:
        return None
    if isinstance(a, int):
        return C.c_void_p(a)
    return a.ctypes.data_as(C.c_void_p)
