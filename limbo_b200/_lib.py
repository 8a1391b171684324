"""ctypes binding of the C ABI (include/limbo_b200.h).  There is no CPU fallback:
if the CUDA library is missing or no device is present every call fails loudly."""
from __future__ import annotations

import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "lib", "liblimbo_b200.so")

LB_OK = 0
ERR_NAMES = {-1: "LB_ERR_ARG", -2: "LB_ERR_CUDA", -3: "LB_ERR_STATE", -4: "LB_ERR_ALLOC", -5: "LB_ERR_UNSUPPORTED",
             -6: "LB_ERR_TIMEOUT"}

KERNEL_SQUARED_EXP_ARD, KERNEL_MATERN_FIVE_HALVES, KERNEL_MATERN_THREE_HALVES, KERNEL_EXP = 0, 1, 2, 3
ACQ_UCB, ACQ_EI = 0, 1
GET_K, GET_L, GET_ALPHA, GET_KINV = 0, 1, 2, 3
EHVI_MAX_K, PARETO_MAX_K = 4096, 8  # LB_EHVI_MAX_K, LB_PARETO_MAX_K
LML_BATCH_MAX_N = 200  # LB_LML_BATCH_MAX_N
CMAES_MAX_D, CMAES_MAX_LAMBDA = 64, 256


class CmaesOpts(C.Structure):
    """lb_cmaes_opts"""
    _fields_ = [("lambda_", C.c_int), ("sigma0", C.c_double), ("generations", C.c_int), ("tolx", C.c_double), ("seed", C.c_uint64),
                ("bounded", C.c_int)]

# every symbol include/limbo_b200.h declares
DECLARED_SYMBOLS = [
    "lb_create", "lb_destroy", "lb_clone", "lb_set_stream", "lb_sync", "lb_launch_count", "lb_set_data",
    "lb_set_data_dev", "lb_set_kernel", "lb_fit", "lb_load_factor", "lb_refit_alpha", "lb_append", "lb_query", "lb_query_dev",
    "lb_acq_argmax", "lb_acq_argmax_dev", "lb_acq_argmax_cols", "lb_acq_argmax_cols_dev", "lb_acq_cmaes_cols", "lb_query_grad", "lb_query_grad_dev", "lb_acq_grad", "lb_acq_grad_dev", "lb_eci_argmax", "lb_eci_argmax_dev", "lb_eci_grad", "lb_eci_grad_dev", "lb_ehvi_argmax", "lb_ehvi_argmax_dev",
    "lb_ehvi3d_argmax", "lb_ehvi3d_argmax_dev", "lb_acq_cmaes", "lb_ehvi_cmaes", "lb_eci_cmaes",
    "lb_ehvi_grad", "lb_ehvi_grad_dev", "lb_pareto_set", "lb_pareto_set_dev", "lb_log_lik", "lb_kernel_grad_log_lik", "lb_lml_grad_batch", "lb_lml_grad_batch_dev", "lb_compute_inv_kernel", "lb_log_loo_cv",
    "lb_kernel_grad_log_loo_cv", "lb_kinv_obs_mean", "lb_get", "lb_sparsify", "lb_sparsify_dev",
    "lb_nb_samples", "lb_strerror", "lb_last_cuda_error", "lb_spgp_create", "lb_spgp_destroy", "lb_spgp_set_data", "lb_spgp_lik",
    "lb_spgp_compute", "lb_spgp_query", "lb_spgp_query_dev", "lb_spgp_acq_argmax", "lb_spgp_acq_argmax_dev", "lb_spgp_acq_cmaes",
    "lb_spgp_query_grad", "lb_spgp_acq_grad", "lb_spgp_launch_count",
]

_lib = None


class LimboB200Error(RuntimeError):
    def __init__(self, code: int, where: str):
        self.code = code
        lib = load()
        msg = lib.lb_strerror(code).decode()
        cuda = lib.lb_last_cuda_error().decode() if code == -2 else ""
        super().__init__(f"{where}: {ERR_NAMES.get(code, code)}: {msg} {cuda}".strip())


class NotPositiveDefinite(LimboB200Error):
    """lb_fit / lb_append returned info > 0 (1-based index of the failing pivot)."""


def load() -> C.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(limbo_b200 has no CPU fallback)")
    lib = C.CDLL(LIB_PATH)
    p, i64, i32, dbl = C.c_void_p, C.c_int64, C.c_int, C.c_double
    dp = C.c_void_p  # raw addresses (numpy / torch data_ptr)
    sig = {
        "lb_create": ([C.POINTER(p), i32, i32], i32),
        "lb_destroy": ([p], i32),
        "lb_clone": ([p, C.POINTER(p)], i32),
        "lb_set_stream": ([p, p], i32),
        "lb_sync": ([p], i32),
        "lb_launch_count": ([p], C.c_longlong),
        "lb_debug_append_count": ([p], C.c_longlong),
        "lb_debug_pool_mallocs": ([], C.c_longlong),
        "lb_debug_pool_hits": ([], C.c_longlong),
        "lb_debug_pool_live": ([], C.c_longlong),
        "lb_pool_trim": ([], i32),
        "lb_debug_set_query_panel_min": ([C.c_longlong], i32),
        "lb_debug_potrf_plan": ([i32, i32, dp, i32], i32),
        "lb_set_data": ([p, i64, i32, i32, dp, dp], i32),
        "lb_set_data_dev": ([p, i64, i32, i32, dp, dp], i32),
        "lb_set_kernel": ([p, i32, dp, i32, dbl], i32),
        "lb_fit": ([p], i32),
        "lb_fit_async": ([p], i32),
        "lb_check_info": ([p], i32),
        "lb_stage_kbuild": ([p], i32),
        "lb_stage_potrf": ([p], i32),
        "lb_stage_alpha": ([p], i32),
        "lb_refit_alpha": ([p, dp], i32),
        "lb_load_factor": ([p, dp, dp], i32),
        "lb_append": ([p, dp, dp], i32),
        "lb_query": ([p, i64, dp, dp, dp], i32),
        "lb_query_dev": ([p, i64, dp, dp, dp], i32),
        "lb_acq_argmax": ([p, i32, dp, i64, dp, dp, dbl, dp, dp, dp], i32),
        "lb_acq_argmax_dev": ([p, i32, dp, i64, dp, dp, dbl, dp, dp, dp], i32),
        "lb_acq_argmax_cols": ([p, i32, i64, dp, i64, dp, dp, dp, dp, dp, dp], i32),
        "lb_acq_argmax_cols_dev": ([p, i32, i64, dp, i64, dp, dp, dp, dp, dp, dp], i32),
        "lb_acq_cmaes_cols": ([p, i32, i64, dp, dp, C.POINTER(CmaesOpts), i64, dp, dp, dp, dp, dp], i32),
        "lb_query_grad": ([p, i64, dp, dp, dp, dp, dp], i32),
        "lb_query_grad_dev": ([p, i64, dp, dp, dp, dp, dp], i32),
        "lb_acq_grad": ([p, i32, dp, i64, dp, dp, dbl, dp, dp, dp], i32),
        "lb_acq_grad_dev": ([p, i32, dp, i64, dp, dp, dbl, dp, dp, dp], i32),
        "lb_eci_argmax": ([p, p, dp, i64, dp, dp, dbl, dp, dbl, dp, dp, dp], i32),
        "lb_eci_argmax_dev": ([p, p, dp, i64, dp, dp, dbl, dp, dbl, dp, dp, dp], i32),
        "lb_ehvi_argmax": ([p, p, dp, i64, dp, i64, dp, dp, dbl, dp, dbl, dp, dp, dp], i32),
        "lb_ehvi_argmax_dev": ([p, p, dp, i64, dp, i64, dp, dp, dbl, dp, dbl, dp, dp, dp], i32),
        "lb_ehvi3d_argmax": ([p, p, p, dp, i64, dp, i64, dp, dp, dbl, dp, dbl, dp, dbl, dp, dp, dp], i32),
        "lb_ehvi3d_argmax_dev": ([p, p, p, dp, i64, dp, i64, dp, dp, dbl, dp, dbl, dp, dbl, dp, dp, dp], i32),
        "lb_acq_cmaes": ([p, i32, dp, dbl, C.POINTER(CmaesOpts), i64, dp, dp, dp, dp], i32),
        "lb_ehvi_cmaes": ([p, p, p, dp, i64, dp, dbl, dbl, dbl, C.POINTER(CmaesOpts), i64, dp, dp, dp, dp], i32),
        "lb_eci_cmaes": ([p, p, dp, dbl, dbl, C.POINTER(CmaesOpts), i64, dp, dp, dp, dp], i32),
        "lb_debug_cmaes_capture": ([i32], i32),
        "lb_debug_cmaes_trace": ([dp, C.c_longlong], C.c_longlong),
        "lb_eci_grad": ([p, p, dp, i64, dp, dp, dbl, dp, dp, dbl, dp, dp, dp], i32),
        "lb_eci_grad_dev": ([p, p, dp, i64, dp, dp, dbl, dp, dp, dbl, dp, dp, dp], i32),
        "lb_ehvi_grad": ([p, p, dp, i64, dp, i64, dp, dp, dbl, dp, dp, dbl, dp, dp, dp], i32),
        "lb_ehvi_grad_dev": ([p, p, dp, i64, dp, i64, dp, dp, dbl, dp, dp, dbl, dp, dp, dp], i32),
        "lb_pareto_set": ([p, i64, i32, dp, dp, dp], i32),
        "lb_pareto_set_dev": ([p, i64, i32, dp, dp, dp], i32),
        "lb_log_lik": ([p, dp], i32),
        "lb_kernel_grad_log_lik": ([p, i32, dp], i32),
        "lb_lml_grad_batch": ([p, i32, i64, i32, dp, dp, i32, dp, dp, dp], i32),
        "lb_lml_grad_batch_dev": ([p, i32, i64, i32, dp, dp, i32, dp, dp, dp], i32),
        "lb_compute_inv_kernel": ([p], i32),
        "lb_log_loo_cv": ([p, dp], i32),
        "lb_kernel_grad_log_loo_cv": ([p, i32, dp], i32),
        "lb_kinv_obs_mean": ([p, dp], i32),
        "lb_get": ([p, i32, dp], i32),
        "lb_sparsify": ([p, i64, i32, dp, i64, dp, dp, dp, dp], i32),
        "lb_sparsify_dev": ([p, i64, i32, dp, i64, dp, dp, dp, dp], i32),
        "lb_debug_sparsify_timing": ([i32], i32),
        "lb_debug_sparsify_last_ms": ([dp], i32),
        "lb_nb_samples": ([p], i64),
        "lb_spgp_create": ([C.POINTER(p), i32], i32),
        "lb_spgp_destroy": ([p], i32),
        "lb_spgp_set_data": ([p, i64, i32, dp, dp], i32),
        "lb_spgp_lik": ([p, i64, i64, dp, dbl, dp, dp], i32),
        "lb_spgp_compute": ([p, i64, i64, dp, dbl], i32),
        "lb_spgp_query": ([p, i64, dp, i32, dp, dp], i32),
        "lb_spgp_acq_argmax": ([p, i32, dp, i64, dp, i32, dp, dbl, dp, dp, dp], i32),
        "lb_spgp_query_dev": ([p, i64, dp, i32, dp, dp], i32),
        "lb_spgp_acq_argmax_dev": ([p, i32, dp, i64, dp, i32, dp, dbl, dp, dp, dp], i32),
        "lb_spgp_acq_cmaes": ([p, i32, dp, i32, dbl, C.POINTER(CmaesOpts), i64, dp, dp, dp, dp], i32),
        "lb_spgp_query_grad": ([p, i64, dp, i32, dp, dp, dp, dp], i32),
        "lb_spgp_acq_grad": ([p, i32, dp, i64, dp, i32, dp, dbl, dp, dp, dp], i32),
        "lb_spgp_launch_count": ([p], C.c_longlong),
        "lb_strerror": ([i32], C.c_char_p),
        "lb_last_cuda_error": ([], C.c_char_p),
    }
    for name, (argtypes, restype) in sig.items():
        fn = getattr(lib, name)
        fn.argtypes = argtypes
        fn.restype = restype
    _lib = lib
    return lib


def check(code: int, where: str) -> None:
    if code == LB_OK:
        return
    if code > 0:
        raise NotPositiveDefinite(code, where)
    raise LimboB200Error(code, where)
