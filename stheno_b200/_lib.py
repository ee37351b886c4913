"""ctypes binding of ``libgpk.so`` -- the C-ABI declared in ``include/gpk.h``.

The library holds the hand-written sm_90a kernels; there is NO fallback: if it is missing it is built with
nvcc, and if that fails (or a function is called without a CUDA device) an error is raised."""
import ctypes
import os
from ctypes import POINTER, Structure, c_double, c_float, c_int32, c_int64, c_void_p

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "csrc", "libgpk.so")

GPK_TILE = 128
GPK_MAX_TERMS = 8
GPK_MAX_FACTORS = 16
GPK_MAX_GROUPS = 8

KM_LOWER, KM_SAME, KM_PAD_IDENTITY, KM_PAD_ZERO = 1, 2, 4, 8

KIND = {"eq": 0, "matern12": 1, "matern32": 2, "matern52": 3, "linear": 4, "delta": 5, "one": 6, "rq": 7}


class KernelDesc(Structure):
    _fields_ = [
        ("n_terms", c_int32),
        ("n_groups", c_int32),
        ("term_begin", c_int32 * (GPK_MAX_TERMS + 1)),
        ("fac_kind", c_int32 * GPK_MAX_FACTORS),
        ("fac_group", c_int32 * GPK_MAX_FACTORS),
        ("coef", c_double * GPK_MAX_TERMS),
        ("fac_param", c_double * GPK_MAX_FACTORS),
    ]


_i32, _i64, _f64, _f32, _ptr = c_int32, c_int64, c_double, c_float, c_void_p

# name -> argtypes of name_f64 / name_f32 (restype int): "T" = the scalar type of the suffix (alpha / beta); "OZ" = the
# int8-slice emulation arguments (slices, ws, ws_bytes) that only the fp64 entry points take
_SIGNATURES = {
    "gpk_kernel_matrix": [POINTER(KernelDesc), _ptr, _i64, _i64, _i64, _ptr, _i64, _i64, _i64, _i32, _f64, _ptr, _i64,
                          _f64, _i32, _ptr, _i64, _i64, _i32, _ptr],
    "gpk_kernel_diag": [POINTER(KernelDesc), _ptr, _i64, _i64, _ptr, _i64, _i64, _i64, _i32, _i32, _ptr, _i64, _i32,
                        _ptr],
    "gpk_kernel_matrix_bwd": [POINTER(KernelDesc), _ptr, _i64, _i64, _i64, _i32, _ptr, _i64, _i64, _ptr, _ptr, _ptr, _ptr,
                              _i32, _ptr],
    "gpk_kernel_cross_bwd": [POINTER(KernelDesc), _ptr, _i64, _i64, _i64, _ptr, _i64, _i64, _i64, _i32, _ptr, _i64, _i64,
                             _ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _i32, _ptr],
    "gpk_gemm_nt": [_i64, _i64, _i64, "T", _ptr, _i64, _i64, _ptr, _i64, _i64, "T", _ptr, _i64, _i64, _i32, _i32, "OZ", _ptr],
    "gpk_potrf": [_ptr, _i64, _i64, _i64, _i64, _ptr, _ptr, _i32, "OZ", _ptr],
    "gpk_trsm_right": [_ptr, _i64, _i64, _i64, _ptr, _i64, _i64, _i64, _i32, "OZ", _ptr],
    "gpk_trsm_right_t": [_ptr, _i64, _i64, _i64, _ptr, _i64, _i64, _i64, _i32, _ptr],
    "gpk_logpdf_finish": [_ptr, _i64, _i64, _i64, _i64, _i32, _ptr, _ptr, _i32, _ptr],
    "gpk_row_dot_sq": [_ptr, _i64, _i64, _i64, _i64, _ptr, _i64, _ptr, _ptr, _i64, _i32, _ptr],
    "gpk_pad_copy": [_ptr, _i64, _i64, _i64, _i64, _ptr, _i64, _i64, _i64, _i64, _f64, _i32, _i32, _ptr],
    "gpk_symmetrize": [_ptr, _i64, _i64, _i64, _i32, _ptr],
    "gpk_transpose": [_ptr, _i64, _i64, _i64, _i64, _ptr, _i64, _i64, _i32, _ptr],
    "gpk_posterior_marginals": [POINTER(KernelDesc), _ptr, _i64, _i64, _ptr, _i64, _i64, _i32, _ptr, _i64, _i64, _ptr, _ptr, _ptr,
                                _i64, _ptr, _i64, "OZ", _ptr],
    "gpk_sparse_posterior_marginals": [POINTER(KernelDesc), _ptr, _i64, _i64, _ptr, _i64, _i64, _i32, _ptr, _i64, _ptr, _i64,
                                       _i64, _ptr, _ptr, _ptr, _ptr, _i64, _ptr, _i64, "OZ", _ptr],
    "gpk_sparse_posterior_rows_bwd": [_i64, _i64, _ptr, _ptr, _i64, _ptr, _ptr, _ptr, _ptr],
    "gpk_sparse_accumulate": [POINTER(KernelDesc), _ptr, _i64, _i64, _ptr, _i64, _i64, _i32, _ptr, _i64, _i64, _ptr, _ptr, _ptr,
                              _i32, _ptr, _i64, _ptr, _ptr, _ptr, _i64, "OZ", _ptr],
    "gpk_sparse_rows_bwd": [_i64, _i64, _ptr, _i64, _ptr, _i64, _ptr, _ptr, _ptr, _ptr, _ptr, _i32, _ptr, _ptr, _ptr, _ptr],
    "gpk_feature_eval": [_ptr, _i64, _i64, _i32, _ptr, _ptr, _ptr, _i64, _ptr, _i64, _i32, _ptr, _i64, _i32, _ptr],
    "gpk_feature_eval_bwd": [_ptr, _i64, _i64, _i32, _ptr, _ptr, _ptr, _i64, _ptr, _i64, _i32, _ptr, _i64, _ptr, _i64, _i32,
                             _ptr],
    "gpk_loo_finish": [_ptr, _i64, _ptr, _i64, _i64, _ptr, _i64, _i64, _i64, _i32, _ptr, _ptr, _ptr, _ptr, _ptr, _ptr, _i32, _ptr],
    "gpk_cv_finish": [_ptr, _i32, _ptr, _i64, _i64, _ptr, _i64, _i64, _ptr, _i64, _ptr, _i64, _ptr, _i64, _i64, _i64, _i32, _ptr,
                      _ptr, _ptr, _ptr, _ptr, _ptr, _i32, _ptr],
}
_PLAIN = {
    "gpk_version": ([], c_int32),
    "gpk_round_up": ([_i64], _i64),
    "gpk_sparse_ws_elems": ([_i64, _i64], _i64),
    "gpk_sparse_posterior_ws_elems": ([_i64, _i64], _i64),
    "gpk_probe_dmma_tflops": ([], c_double),
    "gpk_debug_leaf_phase_clock": ([_ptr], c_int32),
    "gpk_debug_oz_tile": ([_i32, _i32, _i32, _i32, _i32, POINTER(c_int32), POINTER(c_int32)], c_int32),
    "gpk_launch_count": ([], _i64),
    "gpk_launch_count_reset": ([], None),
    "gpk_potrf_f64_tf32x3": ([_ptr, _i64, _i64, _i64, _i64, _ptr, _ptr, _i32, _ptr, _i64, _ptr], c_int32),
    "gpk_potrf_oz_ws_bytes": ([_i64, _i64, _i32], _i64),
    "gpk_trsm_right_oz_ws_bytes": ([_i64, _i64, _i32], _i64),
    "gpk_gemm_nt_oz_ws_bytes": ([_i64, _i64, _i64, _i32], _i64),
    "gpk_oz_ws_bytes": ([_i64, _i64, _i32], _i64),
    "gpk_gemm_nt_f64_oz": ([_i64, _i64, _i64, _f64, _ptr, _i64, _ptr, _i64, _f64, _ptr, _i64, _i32, _i32, _ptr, _i64,
                            _ptr], c_int32),
    "gpk_gemm_profile_enable": ([_i32], None),
    "gpk_gemm_profile_read": ([POINTER(c_double), POINTER(c_double), POINTER(_i64)], c_int32),
    "gpk_gemm_profile_read_kind": ([_i32, POINTER(c_double), POINTER(c_double), POINTER(_i64)], c_int32),
}

#: every symbol ``include/gpk.h`` declares (checked by tests/test_abi.py against the header text)
EXPORTED = [f"{n}_{s}" for n in _SIGNATURES for s in ("f64", "f32")] + list(_PLAIN)

_lib = None


def load(build_if_missing=True):
    """Load (building first if necessary) ``libgpk.so`` and set the argument types."""
    global _lib
    if _lib is not None:
        return _lib
    if build_if_missing:
        from .csrc.build import build_library

        build_library()
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(f"{LIB_PATH} is missing: the CUDA extension has not been built (no CPU fallback exists)")
    lib = ctypes.CDLL(LIB_PATH)
    for name, args in _SIGNATURES.items():
        for suf, scalar, oz in (("f64", c_double, [_i32, _ptr, _i64]), ("f32", c_float, [])):
            fn = getattr(lib, f"{name}_{suf}")
            fn.argtypes = [t for a in args for t in (oz if a == "OZ" else [scalar] if a == "T" else [a])]
            fn.restype = c_int32
    for name, (args, res) in _PLAIN.items():
        fn = getattr(lib, name)
        fn.argtypes = args
        fn.restype = res
    _lib = lib
    return lib


class GpkError(RuntimeError):
    pass


def check(rc, what):
    if rc != 0:
        if rc <= -1000:
            raise GpkError(f"{what}: CUDA error {-rc - 1000}")
        raise GpkError(f"{what}: bad argument / unsupported (code {rc})")
