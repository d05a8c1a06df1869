"""ctypes binding of libb200gp.so (include/b200gp.h).

There is NO CPU fallback: if the shared library is missing, or no CUDA device is
visible, every compute entry point raises.  ``load_library()`` alone (used by the
CPU-only tests to check the exported symbols) does not need a GPU.
"""

from __future__ import annotations

import ctypes
import os
import threading
from ctypes import POINTER, byref, c_char_p, c_double, c_int, c_int64, c_void_p

import numpy as np

_LIB_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "lib", "libb200gp.so")
_lib = None
_ctx = None
_lock = threading.Lock()

PROG_STRIDE = 4
QS_STRIDE = 8
c_double_p = POINTER(c_double)


class B200Error(RuntimeError):
    pass


class Profile(ctypes.Structure):
    _fields_ = [
        ("syrk_ms", c_double), ("syrk_flop", c_double), ("syrk_launches", c_int64),
        ("panel_ms", c_double), ("build_ms", c_double), ("build_bytes", c_double),
        ("solve_ms", c_double), ("qs_ms", c_double), ("qs_bytes", c_double),
        ("qs_launches", c_int64), ("i8_ops", c_double), ("trtri_ms", c_double), ("contract_ms", c_double),
    ]


# name -> (restype, argtypes); every symbol include/b200gp.h declares
_D, _I, _L, _V = c_void_p, c_int, c_int64, c_void_p
SIGNATURES = {
    "b200gp_version": (c_int, []),
    "b200gp_create": (c_int, [c_int, c_void_p, POINTER(c_void_p)]),
    "b200gp_destroy": (c_int, [c_void_p]),
    "b200gp_last_error": (c_char_p, [c_void_p]),
    "b200gp_launch_count": (c_int64, [c_void_p]),
    "b200gp_set_option": (c_int, [c_void_p, c_char_p, c_int64]),
    "b200gp_get_option": (c_int, [c_void_p, c_char_p, POINTER(c_int64)]),
    "b200gp_get_profile": (c_int, [c_void_p, POINTER(Profile), c_int]),
    "b200gp_measure_fp64_peak": (c_int, [c_void_p, c_double_p, c_double_p]),
    "b200gp_measure_dmma_shape": (c_int, [c_void_p, c_int, c_int, c_int, c_double_p]),
    "b200gp_measure_i8_peak": (c_int, [c_void_p, c_double_p]),
    "b200gp_i8_update_test": (c_int, [_V, _D, _I, _L, _L, _D, _D]),
    "b200gp_i8_update_bench": (c_int, [_V, _L, _L, _L, _I, _I, _L, _L, c_double_p, c_void_p]),
    "b200gp_kernel_matrix": (c_int, [_V, _D, _I, _D, _L, _D, _L, _I, _D]),
    "b200gp_kernel_diag": (c_int, [_V, _D, _I, _D, _L, _I, _D]),
    "b200gp_kernel_matvec": (c_int, [_V, _D, _I, _D, _L, _D, _L, _I, _D, _D]),
    "b200gp_dense_create": (c_int, [_V, _D, _I, _D, _L, _I, _D, POINTER(c_void_p), POINTER(c_int)]),
    "b200gp_dense_create_with_resid": (c_int, [_V, _D, _I, _D, _L, _I, _D, _D, POINTER(c_void_p), POINTER(c_int), c_double_p]),
    "b200gp_dense_create_dev": (c_int, [_V, _D, _I, _D, _L, _I, _D, POINTER(c_void_p), POINTER(c_int)]),
    "b200gp_dense_create_from_cov": (c_int, [_V, _D, _L, POINTER(c_void_p), POINTER(c_int)]),
    "b200gp_dense_free": (c_int, [_V]),
    "b200gp_dense_logdet_half": (c_int, [_V, c_double_p]),
    "b200gp_dense_solve_triangular": (c_int, [_V, _D, _L, _I]),
    "b200gp_dense_dot_triangular": (c_int, [_V, _D, _L]),
    "b200gp_dense_condition": (c_int, [_V, _D, _I, _D, _L, _D, _D]),
    "b200gp_gram_downdate": (c_int, [_V, _D, _L, _L, _D]),
    "b200gp_dense_covariance": (c_int, [_V, _D]),
    "b200gp_dense_get_factor": (c_int, [_V, _D]),
    "b200gp_dense_log_probability": (c_int, [_V, _D, _I, _D, _L, _I, _D, _D, c_double_p]),
    "b200gp_dense_log_probability_dev": (c_int, [_V, _D, _I, _D, _L, _I, _D, _D, c_double_p]),
    "b200gp_dense_log_probability_batched": (c_int, [_V, _D, _I, _L, _D, _L, _I, _D, _D, _D]),
    "b200gp_dense_log_probability_grad": (c_int, [_V, _D, _I, _D, _L, _I, _D, _D, c_double_p, _D, _D, _D, _D]),
    "b200gp_mg_create": (c_int, [_V, _D, _I, _D, _L, _I, _D, _D, _I, _I, POINTER(c_void_p)]),
    "b200gp_mg_free": (c_int, [_V]),
    "b200gp_mg_use_colbuf": (c_int, [_V, _D, _L]),
    "b200gp_mg_geometry": (c_int, [_V, POINTER(c_int64), POINTER(c_int64), POINTER(c_int)]),
    "b200gp_mg_update_rows": (c_int, [_V, _I, _L, _L]),
    "b200gp_mg_pack": (c_int, [_V, _I, _L, _L, _D]),
    "b200gp_mg_unpack": (c_int, [_V, _I, _L, _L, _D]),
    "b200gp_mg_panel": (c_int, [_V, _I]),
    "b200gp_mg_panel_factor": (c_int, [_V, _I, _L, _L]),
    "b200gp_mg_panel_finish": (c_int, [_V, _I]),
    "b200gp_mg_finish": (c_int, [_V, c_double_p]),
    "b200gp_qs_check_sorted": (c_int, [_V, _D, _L, POINTER(c_int)]),
    "b200gp_qs_create": (c_int, [_V, _D, _I, _D, _L, _D, _I, POINTER(c_void_p), POINTER(c_int), POINTER(c_int)]),
    "b200gp_qs_create_dev": (c_int, [_V, _D, _I, _D, _L, _D, _I, POINTER(c_void_p), POINTER(c_int), POINTER(c_int)]),
    "b200gp_qs_free": (c_int, [_V]),
    "b200gp_qs_state_dim": (c_int, [_V, POINTER(c_int)]),
    "b200gp_qs_logdet_half": (c_int, [_V, c_double_p]),
    "b200gp_qs_variance": (c_int, [_V, _D]),
    "b200gp_qs_get_factor": (c_int, [_V, _D, _D]),
    "b200gp_qs_get_generators": (c_int, [_V, _D, _D, _D, _D]),
    "b200gp_qs_solve_triangular": (c_int, [_V, _D, _L, _I]),
    "b200gp_qs_solve_sumsq": (c_int, [_V, _D, c_double_p]),
    "b200gp_qs_dot_triangular": (c_int, [_V, _D, _L]),
    "b200gp_qs_matmul": (c_int, [_V, _D, _L]),
    "b200gp_qs_log_probability": (c_int, [_V, _D, _I, _D, _L, _D, _D, _I, POINTER(c_int), c_double_p]),
    "b200gp_qs_log_probability_dev": (c_int, [_V, _D, _I, _D, _L, _D, _D, _I, POINTER(c_int), c_double_p]),
    "b200gp_qs_kernel_matmul": (c_int, [_V, _D, c_int, _D, _L, _D, _L, _D, _L, _D]),
    "b200gp_qs_inverse_diagonal": (c_int, [_V, _D]),
    "b200gp_qs_conditioned_variance": (c_int, [_V, _D, _D]),
    "b200gp_qs_condition": (c_int, [_V, _D, _I, _D, _L, _D, _D]),
    "b200gp_searchsorted_right_m1": (c_int, [_V, _D, _L, _D, _L, _D]),
    # quasiseparable-matrix algebra (qsm.cu)
    "b200gp_qsm_create": (c_int, [_V, _L, _I, _I, _I, _D, _D, _D, _D, _D, _D, _D, POINTER(c_void_p)]),
    "b200gp_qsm_free": (c_int, [_V]),
    "b200gp_qsm_info": (c_int, [_V, POINTER(c_int64), POINTER(c_int), POINTER(c_int), POINTER(c_int)]),
    "b200gp_qsm_get": (c_int, [_V, _D, _D, _D, _D, _D, _D, _D]),
    "b200gp_qsm_part": (c_int, [_V, _I, POINTER(c_void_p)]),
    "b200gp_qsm_compose": (c_int, [_V, _V, _V, _I, POINTER(c_void_p)]),
    "b200gp_qsm_transpose": (c_int, [_V, POINTER(c_void_p)]),
    "b200gp_qsm_scale": (c_int, [_V, _D, _I, POINTER(c_void_p)]),
    "b200gp_qsm_neg": (c_int, [_V, POINTER(c_void_p)]),
    "b200gp_qsm_add": (c_int, [_V, _V, POINTER(c_void_p)]),
    "b200gp_qsm_elementwise_mul": (c_int, [_V, _V, POINTER(c_void_p)]),
    "b200gp_qsm_mul": (c_int, [_V, _V, POINTER(c_void_p)]),
    "b200gp_qsm_gram": (c_int, [_V, POINTER(c_void_p)]),
    "b200gp_qsm_inv": (c_int, [_V, POINTER(c_void_p)]),
    "b200gp_qsm_cholesky": (c_int, [_V, POINTER(c_void_p), POINTER(c_int64)]),
    "b200gp_qsm_matmul": (c_int, [_V, _D, _L]),
    "b200gp_qsm_solve": (c_int, [_V, _D, _L]),
    "b200gp_qsm_sum_log_diag": (c_int, [_V, c_double_p]),
    "b200gp_qs_kernel_qsm": (c_int, [_V, _D, _I, _D, _L, POINTER(c_void_p)]),
    "b200gp_qs_factor_qsm": (c_int, [_V, POINTER(c_void_p)]),
}


def library_path() -> str:
    return _LIB_PATH


def load_library():
    """dlopen libb200gp.so and declare prototypes.  Raises if the extension is not built."""
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB_PATH):
            raise B200Error(
                f"CUDA extension not built: {_LIB_PATH} is missing "
                "(run `python -c 'import __graft_entry__ as g; g.build()'`); there is no CPU fallback"
            )
        lib = ctypes.CDLL(_LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(lib, name)  # AttributeError if the header and the library disagree
            fn.restype = res
            fn.argtypes = args
        _lib = lib
    return _lib


def _device_index() -> int:
    return int(os.environ.get("B200GP_DEVICE", os.environ.get("LOCAL_RANK", "0")))


class Context:
    """One device + one stream + buffer cache (b200gp_ctx)."""

    def __init__(self, device: int | None = None, stream: int | None = None):
        lib = load_library()
        self.lib = lib
        self.handle = c_void_p()
        dev = _device_index() if device is None else device
        rc = lib.b200gp_create(dev, c_void_p(stream) if stream else None, byref(self.handle))
        if rc != 0:
            raise B200Error(
                f"b200gp_create(device={dev}) failed (rc={rc}): no usable CUDA device; "
                "the B200 solver has no CPU fallback"
            )
        self.device = dev

    def check(self, rc: int):
        if rc != 0:
            msg = self.lib.b200gp_last_error(self.handle)
            raise B200Error((msg or b"unknown error").decode())

    def set_option(self, key: str, value: int):
        self.check(self.lib.b200gp_set_option(self.handle, key.encode(), int(value)))

    def get_option(self, key: str) -> int:
        v = c_int64()
        self.check(self.lib.b200gp_get_option(self.handle, key.encode(), byref(v)))
        return int(v.value)

    def reset_options(self):
        """every tuning option back to the library default (common.cuh member initialisers)"""
        self.set_option("reset", 0)

    def launch_count(self) -> int:
        return int(self.lib.b200gp_launch_count(self.handle))

    def profile(self, reset: bool = False) -> dict:
        p = Profile()
        self.check(self.lib.b200gp_get_profile(self.handle, byref(p), int(reset)))
        return {k: getattr(p, k) for k, _ in Profile._fields_}

    def measure_fp64_peak(self):
        a, b = c_double(), c_double()
        self.check(self.lib.b200gp_measure_fp64_peak(self.handle, byref(a), byref(b)))
        return a.value, b.value

    def measure_dmma_shape(self, m: int, n: int, k: int) -> float:
        t = c_double()
        self.check(self.lib.b200gp_measure_dmma_shape(self.handle, m, n, k, byref(t)))
        return t.value

    def measure_i8_peak(self):
        a = c_double()
        self.check(self.lib.b200gp_measure_i8_peak(self.handle, byref(a)))
        return a.value

    def close(self):
        if self.handle:
            self.lib.b200gp_destroy(self.handle)
            self.handle = c_void_p()


def get_context() -> Context:
    global _ctx
    with _lock:
        if _ctx is None:
            _ctx = Context()
        return _ctx


def set_context(ctx: Context | None):
    global _ctx
    with _lock:
        _ctx = ctx


def f64(a) -> np.ndarray:
    return np.ascontiguousarray(a, dtype=np.float64)


def ptr(a: np.ndarray) -> c_void_p:
    return c_void_p(a.ctypes.data)
