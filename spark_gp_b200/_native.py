"""ctypes binding of the C-ABI in include/sgp.h (the same .so a JNI shim would load).

There is NO CPU fallback: if libsgp.so is missing or no H100 is visible, calls raise."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libsgp.so")

SGP_OK, SGP_E_BADARG, SGP_E_CUDA, SGP_E_NOT_PD, SGP_E_NCCL, SGP_E_STATE, SGP_E_SINGULAR, SGP_E_NOMEM, SGP_E_RANGE = range(9)
SGP_TERM_ARD, SGP_TERM_RBF, SGP_TERM_EYE = 0, 1, 2
SGP_PREC_F64, SGP_PREC_F64_STRICT, SGP_PREC_I8, SGP_PREC_AUTO, SGP_PREC_I8_DIRECT = 0, 1, 2, 3, 4
SGP_UNIQUE_ID_BYTES = 128

# every symbol include/sgp.h declares (tests/test_abi.py checks the .so exports each of them)
EXPORTS = ["sgp_ctx_create", "sgp_ctx_destroy", "sgp_last_error", "sgp_set_precision", "sgp_version",
           "sgp_comm_unique_id", "sgp_comm_init", "sgp_stats_begin", "sgp_stats_accumulate",
           "sgp_stats_accumulate_device", "sgp_stats_finish", "sgp_sync", "sgp_magic", "sgp_predict", "sgp_predict_device",
           "sgp_launch_count", "sgp_gram_kernel_time", "sgp_cross_kernel", "sgp_event_record",
           "sgp_event_elapsed_ms", "sgp_debug_i8_tile", "sgp_last_path", "sgp_experts_upload",
           "sgp_bcm_nll", "sgp_laplace_nll", "sgp_experts_get_f", "sgp_set_magic", "sgp_last_tail_path", "sgp_last_bcm_path", "sgp_experts_upload_grouped", "sgp_kmn_sweep", "sgp_kmn_sweep_device", "sgp_greedy_active_set", "sgp_kmeans",
           "sgp_laplace_nll_classes", "sgp_experts_get_f_class", "sgp_experts_upload_folds", "sgp_bcm_nll_folds",
           "sgp_laplace_nll_any_size", "sgp_laplace_nll_classes_any_size", "sgp_last_laplace_path",
           "sgp_laplace_nll_slots_any_size", "sgp_experts_get_f_slot", "sgp_experts_upload_grouped_device",
           "sgp_experts_upload_folds_device", "sgp_experts_get_f_rows_device", "sgp_kmeans_device",
           "sgp_greedy_active_set_device", "sgp_laplace_nll_fold_slots_any_size", "sgp_experts_get_f_fold_slot",
           "sgp_experts_get_f_fold_rows_device", "sgp_gauss_hermite_rule", "sgp_predict_probability",
           "sgp_predict_probability_device", "sgp_bcm_nll_slots", "sgp_kernel_eval", "sgp_kernel_eval_device",
           "sgp_experts_upload_strided_device", "sgp_kmeans_sharded", "sgp_kmeans_sharded_device",
           "sgp_experts_upload_fold_sets_device", "sgp_column_sums_device", "sgp_scale_apply_device"]


class KernelTerm(C.Structure):
    _fields_ = [("type", C.c_int32), ("reserved", C.c_int32), ("scale", C.c_double), ("sigma", C.c_double),
                ("beta", C.POINTER(C.c_double))]


class Hyper(C.Structure):
    _fields_ = [("kind", C.c_int32), ("term", C.c_int32), ("dim", C.c_int32), ("reserved", C.c_int32),
                ("value", C.c_double), ("coef", C.POINTER(C.c_double))]


SGP_HYPER_SCALE, SGP_HYPER_ARD_BETA, SGP_HYPER_RBF_SIGMA = 0, 1, 2
SGP_MODES_BINARY, SGP_MODES_CLASS, SGP_MODES_SLOT = 0, 1, 2
SGP_KEVAL_CROSS, SGP_KEVAL_TRAINING = 0, 1


class KernelDesc(C.Structure):
    _fields_ = [("n_terms", C.c_int32), ("reserved", C.c_int32), ("terms", C.POINTER(KernelTerm))]


_lib = None


def load() -> C.CDLL:
    """Loads libsgp.so (building is `python -m spark_gp_b200.build` / __graft_entry__.build())."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError("spark_gp_b200: %s is missing -- run `python __graft_entry__.py build`. "
                           "There is no CPU fallback." % LIB_PATH)
    lib = C.CDLL(LIB_PATH)
    vp, i32, i64, dp = C.c_void_p, C.c_int32, C.c_int64, C.POINTER(C.c_double)
    lib.sgp_ctx_create.argtypes = [C.POINTER(vp), C.c_int]
    lib.sgp_ctx_destroy.argtypes = [vp]
    lib.sgp_last_error.argtypes = [vp]
    lib.sgp_last_error.restype = C.c_char_p
    lib.sgp_set_precision.argtypes = [vp, C.c_int]
    lib.sgp_comm_unique_id.argtypes = [vp]
    lib.sgp_comm_init.argtypes = [vp, vp, C.c_int, C.c_int]
    lib.sgp_stats_begin.argtypes = [vp, C.POINTER(KernelDesc), vp, i32, i32]
    lib.sgp_stats_accumulate.argtypes = [vp, vp, i32, vp, i64]
    lib.sgp_stats_accumulate_device.argtypes = [vp, vp, i32, vp, i64]
    lib.sgp_stats_finish.argtypes = [vp, vp, vp]
    lib.sgp_sync.argtypes = [vp]
    lib.sgp_magic.argtypes = [vp, vp, vp, vp, vp]
    lib.sgp_predict.argtypes = [vp, vp, i64, vp, vp]
    lib.sgp_predict_device.argtypes = [vp, vp, i32, i64, vp, vp]
    lib.sgp_gauss_hermite_rule.argtypes = [i32, vp, vp]
    lib.sgp_predict_probability.argtypes = [vp, vp, i64, i32, vp, vp, vp]
    lib.sgp_predict_probability_device.argtypes = [vp, vp, i32, i64, i32, vp, vp, vp]
    lib.sgp_set_magic.argtypes = [vp, vp, vp]
    lib.sgp_launch_count.argtypes = [vp]
    lib.sgp_launch_count.restype = i64
    lib.sgp_gram_kernel_time.argtypes = [vp, dp, C.POINTER(i64)]
    lib.sgp_cross_kernel.argtypes = [vp, vp, i64, vp]
    lib.sgp_greedy_active_set.argtypes = [vp, vp, vp, vp, i64, C.c_int32, i64, i64, C.c_int32, vp]
    lib.sgp_kmeans.argtypes = [vp, vp, i32, i64, i32, i32, i32, C.c_double, i64, vp, vp, vp, vp, vp, vp]
    lib.sgp_event_record.argtypes = [vp, C.c_int]
    lib.sgp_debug_i8_tile.argtypes = [vp, vp, vp]
    lib.sgp_last_path.argtypes = [vp]
    lib.sgp_last_tail_path.argtypes = [vp]
    lib.sgp_last_bcm_path.argtypes = [vp]
    lib.sgp_experts_upload.argtypes = [vp, vp, vp, vp, i64, i32]
    lib.sgp_experts_upload_grouped.argtypes = [vp, vp, i32, vp, i64, i32, i32]
    lib.sgp_kmn_sweep.argtypes = [vp, vp, i32, i64, vp]
    lib.sgp_kmn_sweep_device.argtypes = [vp, vp, i32, i64, vp]
    lib.sgp_bcm_nll.argtypes = [vp, C.POINTER(KernelDesc), vp, i32, dp, vp]
    lib.sgp_laplace_nll.argtypes = [vp, C.POINTER(KernelDesc), vp, i32, C.c_double, dp, vp]
    lib.sgp_experts_get_f.argtypes = [vp, vp]
    lib.sgp_laplace_nll_classes.argtypes = [vp, i32, vp, i32, vp, vp, i32, C.c_double, vp, vp]
    lib.sgp_laplace_nll_any_size.argtypes = [vp, C.POINTER(KernelDesc), vp, i32, C.c_double, dp, vp]
    lib.sgp_laplace_nll_classes_any_size.argtypes = [vp, i32, vp, i32, vp, vp, i32, C.c_double, vp, vp]
    lib.sgp_last_laplace_path.argtypes = [vp]
    lib.sgp_experts_get_f_class.argtypes = [vp, i32, vp]
    lib.sgp_laplace_nll_slots_any_size.argtypes = [vp, i32, vp, vp, i32, vp, vp, i32, C.c_double, vp, vp]
    lib.sgp_experts_get_f_slot.argtypes = [vp, i32, vp]
    lib.sgp_experts_upload_folds.argtypes = [vp, vp, i32, vp, i64, i32, vp, i32, i32]
    lib.sgp_bcm_nll_folds.argtypes = [vp, vp, i32, vp, vp, i32, vp, vp]
    lib.sgp_bcm_nll_slots.argtypes = [vp, i32, vp, vp, i32, vp, vp]
    lib.sgp_experts_upload_grouped_device.argtypes = lib.sgp_experts_upload_grouped.argtypes
    lib.sgp_experts_upload_folds_device.argtypes = lib.sgp_experts_upload_folds.argtypes
    lib.sgp_experts_get_f_rows_device.argtypes = [vp, i32, i32, vp]
    lib.sgp_laplace_nll_fold_slots_any_size.argtypes = [vp, i32, vp, vp, vp, i32, vp, vp, i32, C.c_double, vp, vp]
    lib.sgp_experts_get_f_fold_slot.argtypes = [vp, i32, i32, vp]
    lib.sgp_experts_get_f_fold_rows_device.argtypes = [vp, i32, i32, vp]
    lib.sgp_kmeans_device.argtypes = lib.sgp_kmeans.argtypes
    lib.sgp_greedy_active_set_device.argtypes = lib.sgp_greedy_active_set.argtypes
    lib.sgp_kernel_eval.argtypes = [vp, C.POINTER(KernelDesc), vp, i32, vp, i32, i64, vp, i32, i32, i32, vp, vp]
    lib.sgp_kernel_eval_device.argtypes = lib.sgp_kernel_eval.argtypes
    lib.sgp_experts_upload_strided_device.argtypes = [vp, vp, i32, vp, i64, i32, i64]
    lib.sgp_experts_upload_fold_sets_device.argtypes = [vp, vp, i32, vp, vp, vp, i32, i32]
    lib.sgp_kmeans_sharded.argtypes = [vp, vp, i32, i64, i64, i64, i32, i32, i32, C.c_double, i64, vp, vp, vp, vp, vp, vp]
    lib.sgp_kmeans_sharded_device.argtypes = lib.sgp_kmeans_sharded.argtypes
    lib.sgp_event_elapsed_ms.argtypes = [vp, C.c_int, C.c_int, dp]
    lib.sgp_column_sums_device.argtypes = [vp, vp, i32, i64, i32, vp, vp]
    lib.sgp_scale_apply_device.argtypes = [vp, vp, i32, i64, i32, vp, vp, vp]
    for name in EXPORTS:
        if name not in ("sgp_last_error", "sgp_launch_count"):
            getattr(lib, name).restype = C.c_int
    _lib = lib
    return lib


def ptr(a: np.ndarray):
    return a.ctypes.data_as(C.c_void_p)
