"""ctypes binding of libmbar_b200.so (include/mbar_b200.h).  There is no CPU fallback: if the
library is missing, or no sm_90 GPU is visible when a context is created, calls raise."""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libmbar_b200.so")

UNIQUE_ID_BYTES = 128
MAX_STATES = 8192            # MBAR_B200_MAX_STATES: largest K of a context, augmented ones included
BATCH_MAX_ROWS = 192         # MBAR_B200_BATCH_MAX_ROWS: largest K_p + M_p of a batch problem with appended rows
KERNEL_AUTO, KERNEL_FUSED, KERNEL_GENERIC = 0, 1, 2

STATUS = {
    0: "OK", -1: "ERR_INVALID", -2: "ERR_CUDA", -3: "ERR_NO_DEVICE", -4: "ERR_NOT_READY",
    -5: "ERR_NAN", -6: "ERR_RANGE", -7: "ERR_COMM", -8: "ERR_SINGULAR", -9: "ERR_NOMEM",
}


class MbarB200Error(RuntimeError):
    def __init__(self, status, message):
        super().__init__(f"libmbar_b200: {STATUS.get(status, status)}: {message}")
        self.status = status


class SolveResult(C.Structure):
    _fields_ = [("success", C.c_int32), ("iterations", C.c_int32), ("nr_iterations", C.c_int32),
                ("sci_iterations", C.c_int32), ("passes", C.c_int32), ("hessian_passes", C.c_int32),
                ("max_delta", C.c_double), ("gnorm", C.c_double), ("device_ms", C.c_double)]


class AdaptiveStats(C.Structure):
    _fields_ = [(name, C.c_int32) for name in ("device_iterations", "fell_back", "ridge_retries", "newton_failed",
                                                 "newton_rejected", "newton_threads", "newton_smem", "reserved")]


class Synth(C.Structure):
    _fields_ = [("seed", C.c_uint64), ("n_offset", C.c_int64), ("N_global", C.c_int64),
                ("O_k", C.POINTER(C.c_double)), ("k_k", C.POINTER(C.c_double))]


_dp = C.POINTER(C.c_double)
_ctx = C.c_void_p

# name -> (restype, argtypes); mirrors include/mbar_b200.h one to one
SIGNATURES = {
    "mbar_b200_abi_version": (C.c_int, []),
    "mbar_b200_last_error": (C.c_char_p, []),
    "mbar_b200_device_count": (C.c_int, [C.POINTER(C.c_int)]),
    "mbar_b200_host_alloc": (C.c_int, [C.POINTER(C.c_void_p), C.c_uint64]),
    "mbar_b200_host_free": (C.c_int, [C.c_void_p]),
    "mbar_b200_gpu_numa_node": (C.c_int, [C.c_int, C.POINTER(C.c_int)]),
    "mbar_b200_host_hash": (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.POINTER(C.c_uint64)]),
    "mbar_b200_trim": (C.c_int, []),
    "mbar_b200_create": (C.c_int, [C.POINTER(_ctx), C.c_int, C.c_int32, C.c_int64, _dp]),
    "mbar_b200_destroy": (C.c_int, [_ctx]),
    "mbar_b200_get_shape": (C.c_int, [_ctx, C.POINTER(C.c_int32), C.POINTER(C.c_int64)]),
    "mbar_b200_set_pass_kernel": (C.c_int, [_ctx, C.c_int]),
    "mbar_b200_get_counters": (C.c_int, [_ctx] + [C.POINTER(C.c_int64)] * 4),
    "mbar_b200_last_pass_ms": (C.c_int, [_ctx, _dp]),
    "mbar_b200_upload_u_kn": (C.c_int, [_ctx, C.c_void_p, C.c_int64]),
    "mbar_b200_upload_u_kn_dev": (C.c_int, [_ctx, C.c_void_p, C.c_int64]),
    "mbar_b200_create_augmented": (C.c_int, [_ctx, C.c_int32, C.c_void_p, C.c_int64, C.POINTER(_ctx)]),
    "mbar_b200_synthesize": (C.c_int, [_ctx, C.POINTER(Synth)]),
    "mbar_b200_set_sample_weights": (C.c_int, [_ctx, C.c_void_p]),
    "mbar_b200_download_u_kn": (C.c_int, [_ctx, C.c_int64, C.c_int64, C.c_void_p, C.c_int64]),
    "mbar_b200_pass": (C.c_int, [_ctx, _dp, _dp, _dp, _dp]),
    "mbar_b200_pass_multi": (C.c_int, [_ctx, C.c_int32, _dp, _dp, _dp]),
    "mbar_b200_self_consistent_update": (C.c_int, [_ctx, _dp, _dp]),
    "mbar_b200_gradient": (C.c_int, [_ctx, _dp, _dp]),
    "mbar_b200_objective_and_gradient": (C.c_int, [_ctx, _dp, _dp, _dp]),
    "mbar_b200_hessian": (C.c_int, [_ctx, _dp, _dp]),
    "mbar_b200_weight_moments": (C.c_int, [_ctx, _dp, _dp, _dp]),
    "mbar_b200_log_W_nk": (C.c_int, [_ctx, _dp, C.c_void_p, C.c_int64, C.c_int]),
    "mbar_b200_log_W_nk_rows": (C.c_int, [_ctx, _dp, C.c_int64, C.c_int64, C.c_void_p, C.c_int64, C.c_int]),
    "mbar_b200_log_denominator": (C.c_int, [_ctx, _dp, _dp]),
    "mbar_b200_bin_moments": (C.c_int, [_ctx, _dp, _dp, C.POINTER(C.c_int32), C.c_int32, _dp, _dp, _dp]),
    "mbar_b200_replicate_unsampled": (C.c_int, [_ctx, C.c_int64, C.POINTER(C.c_uint16), _dp, _dp]),
    "mbar_b200_last_replicate_stats": (C.c_int, [_ctx, _dp, C.POINTER(C.c_int32), C.POINTER(C.c_int64)]),
    "mbar_b200_kde_create": (C.c_int, [C.c_int, C.c_int64, C.c_int32, _dp, _dp, C.POINTER(_ctx)]),
    "mbar_b200_kde_destroy": (C.c_int, [_ctx]),
    "mbar_b200_kde_log_sum": (C.c_int, [_ctx, C.c_int32, C.c_double, C.c_int64, _dp, _dp]),
    "mbar_b200_kde_set_replicates": (C.c_int, [_ctx, C.c_int64, _dp]),
    "mbar_b200_kde_log_sum_replicates": (C.c_int, [_ctx, C.c_int32, C.c_double, C.c_int64, _dp, _dp]),
    "mbar_b200_last_kde_stats": (C.c_int, [_ctx, _dp, C.POINTER(C.c_int32)]),
    "mbar_b200_kde_many_create": (C.c_int, [C.c_int, C.c_int32, C.POINTER(C.c_int32), C.POINTER(C.c_int64), _dp,
                                            C.POINTER(_ctx)]),
    "mbar_b200_kde_many_destroy": (C.c_int, [_ctx]),
    "mbar_b200_kde_many_log_sum": (C.c_int, [_ctx, C.c_int32, C.POINTER(C.c_int32), C.POINTER(C.c_int32), _dp, _dp,
                                             C.POINTER(C.c_int64), _dp, _dp]),
    "mbar_b200_last_kde_many_stats": (C.c_int, [_ctx, _dp, C.POINTER(C.c_int32), C.POINTER(C.c_int64)]),
    "mbar_b200_bspline_create": (C.c_int, [C.c_int, C.c_int64, _dp, _dp, C.POINTER(C.c_int32), C.c_int32,
                                           C.POINTER(_ctx)]),
    "mbar_b200_bspline_destroy": (C.c_int, [_ctx]),
    "mbar_b200_bspline_moments": (C.c_int, [_ctx, C.c_int32, C.c_int64, _dp, _dp, _dp]),
    "mbar_b200_bspline_set_replicates": (C.c_int, [_ctx, C.c_int64, _dp]),
    "mbar_b200_bspline_replicate_sums": (C.c_int, [_ctx, C.c_int32, C.c_int64, _dp, _dp]),
    "mbar_b200_last_bspline_stats": (C.c_int, [_ctx, _dp, C.POINTER(C.c_int32)]),
    "mbar_b200_acf_create": (C.c_int, [C.c_int, C.c_int64, _dp, _dp, C.c_int32, C.POINTER(C.c_int64),
                                       C.POINTER(_ctx)]),
    "mbar_b200_acf_destroy": (C.c_int, [_ctx]),
    "mbar_b200_acf_inefficiency": (C.c_int, [_ctx, C.c_int64, C.POINTER(C.c_int64), C.c_int32, C.c_int32, C.c_int32,
                                             C.c_double, C.c_int64, _dp, _dp, _dp, _dp, C.POINTER(C.c_int64),
                                             C.POINTER(C.c_int32), _dp]),
    "mbar_b200_acf_inefficiency_series": (C.c_int, [_ctx, C.c_int64, C.POINTER(C.c_int32), C.POINTER(C.c_int64),
                                                    C.c_int32, C.c_int32, _dp, _dp, _dp, _dp, C.POINTER(C.c_int64),
                                                    C.POINTER(C.c_int32)]),
    "mbar_b200_acf_correlation": (C.c_int, [_ctx, C.c_int64, C.c_int64, _dp, _dp, _dp, _dp]),
    "mbar_b200_acf_correlation_multiple": (C.c_int, [_ctx, C.c_int64, C.c_int32, _dp, C.POINTER(C.c_int64), _dp, _dp,
                                                     _dp]),
    "mbar_b200_last_acf_stats": (C.c_int, [_ctx, _dp, C.POINTER(C.c_int32), C.POINTER(C.c_int64),
                                           C.POINTER(C.c_int64)]),
    "mbar_b200_work_create": (C.c_int, [C.c_int, C.c_int64, _dp, C.c_int32, C.POINTER(C.c_int64), C.POINTER(_ctx)]),
    "mbar_b200_work_destroy": (C.c_int, [_ctx]),
    "mbar_b200_work_evaluate": (C.c_int, [_ctx, C.c_int32, C.POINTER(C.c_int32), C.POINTER(C.c_int32), _dp, _dp,
                                          _dp]),
    "mbar_b200_last_work_stats": (C.c_int, [_ctx, _dp, C.POINTER(C.c_int32), C.POINTER(C.c_int64)]),
    "mbar_b200_batch_create": (C.c_int, [C.c_int, C.c_int32, C.POINTER(C.c_int32), C.POINTER(C.c_int64), _dp, _dp,
                                         C.POINTER(_ctx)]),
    "mbar_b200_batch_destroy": (C.c_int, [_ctx]),
    "mbar_b200_batch_moments": (C.c_int, [_ctx, C.c_int32, C.POINTER(C.c_int32), _dp, C.c_int32, _dp, _dp, _dp,
                                          C.POINTER(C.c_int32), _dp]),
    "mbar_b200_batch_solve": (C.c_int, [_ctx, _dp, C.c_double, C.c_int32, C.c_int32, C.c_double, C.POINTER(C.c_int32),
                                        C.POINTER(C.c_int32)]),
    "mbar_b200_batch_set_replicates": (C.c_int, [_ctx, C.c_int32, C.POINTER(C.c_int32), C.POINTER(C.c_uint16)]),
    "mbar_b200_batch_replicate_moments": (C.c_int, [_ctx, C.c_int32, C.POINTER(C.c_int32), _dp, C.c_int32, _dp, _dp,
                                                    _dp, C.POINTER(C.c_int32), _dp]),
    "mbar_b200_batch_solve_replicates": (C.c_int, [_ctx, _dp, C.c_double, C.c_int32, C.c_int32, C.c_double,
                                                   C.POINTER(C.c_int32), C.POINTER(C.c_int32)]),
    "mbar_b200_batch_set_unsampled": (C.c_int, [_ctx, C.c_int32, C.POINTER(C.c_int32), C.POINTER(C.c_int32), _dp]),
    "mbar_b200_batch_augmented_moments": (C.c_int, [_ctx, C.c_int32, C.POINTER(C.c_int32), _dp, _dp, _dp, _dp,
                                                    C.POINTER(C.c_int32), _dp]),
    "mbar_b200_batch_replicate_augmented_moments": (C.c_int, [_ctx, C.c_int32, C.POINTER(C.c_int32), _dp, _dp, _dp,
                                                              _dp, C.POINTER(C.c_int32)]),
    "mbar_b200_batch_bin_moments": (C.c_int, [_ctx, C.c_int32, C.POINTER(C.c_int32), _dp, _dp, C.POINTER(C.c_int32),
                                              C.POINTER(C.c_int32), _dp, _dp, _dp, C.POINTER(C.c_int32)]),
    "mbar_b200_batch_replicate_bin_moments": (C.c_int, [_ctx, C.c_int32, C.POINTER(C.c_int32), _dp,
                                                        C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.c_int32,
                                                        C.POINTER(C.c_int32), C.POINTER(C.c_int32), _dp, _dp,
                                                        C.POINTER(C.c_int32)]),
    "mbar_b200_batch_log_weights": (C.c_int, [_ctx, C.c_int32, C.POINTER(C.c_int32), _dp, _dp, _dp,
                                              C.POINTER(C.c_int32)]),
    "mbar_b200_last_batch_stats": (C.c_int, [_ctx, _dp, C.POINTER(C.c_int32), C.POINTER(C.c_int32),
                                             C.POINTER(C.c_int64)]),
    "mbar_b200_solve_sci":(C.c_int, [_ctx, _dp, C.c_double, C.c_int32, C.POINTER(SolveResult)]),
    "mbar_b200_solve_adaptive": (C.c_int, [_ctx, _dp, C.c_double, C.c_int32, C.c_int32, C.c_double,
                                           C.POINTER(SolveResult)]),
    "mbar_b200_set_loop_mode": (C.c_int, [_ctx, C.c_int32, C.c_int32]),
    "mbar_b200_get_loop_stats": (C.c_int, [_ctx, C.POINTER(C.c_int64), C.POINTER(C.c_int32), C.POINTER(C.c_int32)]),
    "mbar_b200_get_graph_stats": (C.c_int, [_ctx, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    "mbar_b200_get_adaptive_stats": (C.c_int, [_ctx, C.POINTER(AdaptiveStats)]),
    "mbar_b200_last_kernels": (C.c_int, [_ctx, C.c_char_p, C.c_char_p, C.c_int32]),
    "mbar_b200_last_hessian_ms": (C.c_int, [_ctx, _dp, _dp]),
    "mbar_b200_last_bin_stats": (C.c_int, [_ctx, _dp, C.POINTER(C.c_int32)]),
    "mbar_b200_measure_fp64_peak": (C.c_int, [C.c_int, _dp, _dp]),
    "mbar_b200_probe_exp": (C.c_int, [C.c_int, C.c_int, C.c_int64, _dp, _dp]),
    "mbar_b200_sci_iterate": (C.c_int, [_ctx, _dp, C.c_int32]),
    "mbar_b200_last_loop_ms": (C.c_int, [_ctx, _dp, _dp, C.POINTER(C.c_int32)]),
    "mbar_b200_self_consistent_update_host": (C.c_int, [C.c_int, C.c_int32, C.c_int64, C.c_void_p, C.c_int64,
                                                        _dp, _dp, _dp]),
    "mbar_b200_comm_unique_id": (C.c_int, [C.c_void_p]),
    "mbar_b200_comm_init": (C.c_int, [_ctx, C.c_int32, C.c_int32, C.c_void_p]),
    "mbar_b200_comm_destroy": (C.c_int, [_ctx]),
    "mbar_b200_peer_export": (C.c_int, [_ctx, C.c_void_p]),
    "mbar_b200_peer_attach": (C.c_int, [_ctx, C.c_int32, C.c_int32, C.c_void_p]),
}

_lib = None


def load():
    """Load the shared library (building is the job of __graft_entry__.build / pymbar_b200.build)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} is missing: build it with `python -m pymbar_b200.build` "
            "(pymbar_b200 has no CPU fallback)")
    lib = C.CDLL(LIB_PATH, mode=C.RTLD_GLOBAL)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)           # AttributeError if the .so lacks a declared symbol
        fn.restype = res
        fn.argtypes = args
    if lib.mbar_b200_abi_version() != 1:
        raise ImportError("libmbar_b200.so ABI version mismatch")
    _lib = lib
    return lib


def check(status):
    if status != 0:
        msg = load().mbar_b200_last_error()
        raise MbarB200Error(status, msg.decode() if msg else "")


def device_count():
    n = C.c_int(0)
    check(load().mbar_b200_device_count(C.byref(n)))
    return n.value
