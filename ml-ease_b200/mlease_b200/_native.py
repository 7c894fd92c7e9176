"""ctypes binding of include/mlease_b200.h (libmlease_b200.so, built in-tree under ml-ease_b200/lib).

There is no Python/CPU fallback: if the shared library is missing this module raises, and every
compute entry point of the library itself fails without a CUDA device.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
SO_PATH = os.path.join(os.path.dirname(_HERE), "lib", "libmlease_b200.so")


class MleaseError(RuntimeError):
    """Non-zero status from the C ABI (code, message). Codes: include/mlease_b200.h MLEASE_ERR_*."""

    def __init__(self, code, msg):
        super().__init__("mlease_b200 error %d: %s" % (code, msg))
        self.code = code
        self.message = msg


class AdmmConfigC(C.Structure):
    _fields_ = [("device", C.c_int32), ("num_blocks", C.c_int32), ("num_features", C.c_int32), ("num_lambdas", C.c_int32),
                ("lambdas", C.POINTER(C.c_float)), ("rhos", C.POINTER(C.c_float)), ("lambda_map", C.POINTER(C.c_float)),
                ("regularizer", C.c_int32), ("penalize_intercept", C.c_int32), ("aggressive_decay", C.c_int32),
                ("binary_feature", C.c_int32), ("epsilon", C.c_double), ("rho_adapt_coefficient", C.c_float),
                ("newton_xtol", C.c_double), ("max_newton", C.c_int32), ("hessian_policy", C.c_int32), ("stream", C.c_void_p)]


class StatsC(C.Structure):
    _fields_ = [("k1_passes", C.c_int64), ("gram_builds", C.c_int64), ("newton_steps", C.c_int64), ("rejected_steps", C.c_int64),
                ("kernel_launches", C.c_int64), ("not_converged", C.c_int32), ("last_iter_slots", C.c_int32),
                ("last_maxdiff", C.c_double), ("liblinear_epsilon", C.c_float), ("k1_fused", C.c_int32), ("k1_shared_bytes", C.c_double)]


ALLREDUCE_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p)

_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(SO_PATH):
            raise RuntimeError("libmlease_b200.so is not built (%s). Run `python __graft_entry__.py build` or "
                               "`python -m mlease_b200.build`; there is no fallback path." % SO_PATH)
        _lib = C.CDLL(SO_PATH)
        _lib.mlease_last_error.restype = C.c_char_p
        vp, i32, i64, f32, f64 = C.c_void_p, C.c_int32, C.c_int64, C.c_float, C.c_double
        sig = {
            "mlease_session_create": [C.POINTER(AdmmConfigC), C.POINTER(vp)],
            "mlease_session_destroy": [vp],
            "mlease_add_partition_dense": [vp, i32, i64, vp, i64, vp, vp, vp],
            "mlease_add_partition_csr": [vp, i32, i64, vp, vp, vp, vp, vp, vp],
            "mlease_admm_begin": [vp],
            "mlease_admm_begin_initialized": [vp, vp, C.c_float],
            "mlease_admm_local_step": [vp, vp],
            "mlease_admm_consensus": [vp, vp, C.POINTER(f64), C.POINTER(i32)],
            "mlease_admm_run": [vp, i32, vp, vp, C.POINTER(i32)],
            "mlease_admm_iterate": [vp, C.POINTER(f64), C.POINTER(i32)],
            "mlease_get_z": [vp, i32, vp],
            "mlease_get_final_model": [vp, i32, vp],
            "mlease_get_x": [vp, i32, i32, vp],
            "mlease_get_u": [vp, i32, i32, vp],
            "mlease_get_uplusx": [vp, i32, i32, vp],
            "mlease_get_stats": [vp, C.POINTER(StatsC)],
            "mlease_objective": [vp, i32, vp, vp, vp, C.POINTER(f64), vp, vp, i32],
            "mlease_fit_partition": [vp, i32, vp, vp, vp, C.POINTER(i32)],
            "mlease_hessian_vector": [vp, i32, vp, vp, vp, vp],
            "mlease_naive_train_dense": [i32, vp, i32, i32, vp, vp, i64, vp, vp, vp, f32, vp, f32, i32, i32, i32, vp, vp],
            "mlease_score": [i32, vp, i32, i64, vp, vp, vp, i64, vp, vp, i32, i32, vp],
            "mlease_test_loglik": [i32, vp, i64, vp, vp, vp, i64, C.POINTER(f32), C.POINTER(f64)],
            "mlease_score_keyed": [i32, vp, i32, i32, vp, vp, vp, vp, vp, i32, vp, vp, vp, i32, vp],
            "mlease_score_keyed_var": [i32, vp, i32, i32, vp, vp, vp, vp, vp, i32, vp, vp, vp, vp, vp, vp, vp, i32, vp, vp],
            "mlease_score_keyed_cov": [i32, vp, i32, i32, vp, vp, vp, vp, vp, i32, vp, vp, vp, vp, vp, vp, vp, i32, vp, vp],
            "mlease_test_loglik_keyed": [i32, vp, i64, vp, vp, vp, vp, vp, i32, vp, vp],
            "mlease_test_auc": [i32, vp, i64, i32, vp, vp, vp, i32, vp, vp, vp, vp, vp],
            "mlease_time_kernel": [vp, i32, i32, i32, i32, C.POINTER(f32)],
            "mlease_profile": [vp, i32, vp, vp, C.POINTER(f64), C.POINTER(f64), C.POINTER(f64)],
            "mlease_posterior_variance": [vp, i32, vp, vp, i32, vp, vp],
            "mlease_admm_posterior": [vp, i32, vp, i32, vp, vp],
            "mlease_world_admm_posterior": [vp, i32, vp, i32, vp, vp],
            "mlease_score_var": [i32, vp, i32, i64, vp, vp, vp, vp, vp, i32, i32, vp, vp, vp, vp],
            "mlease_naive_train": [i32, vp, i32, i32, vp, vp, vp, vp, i64, vp, vp, vp, i32, vp, vp, f32, i32, i32, i32, i32, vp, vp],
            "mlease_item_model_train": [i32, vp, i32, i32, vp, vp, vp, vp, vp, vp, vp, vp, i32, vp, i32, vp, vp, i32, i32, vp, vp],
            "mlease_naive_train_sparse": [i32, vp, i32, i32, vp, vp, vp, vp, vp, vp, vp, i32, vp, vp, f32, i32, i32, i32, i32, i64, vp, vp, vp,
                                          vp],
            "mlease_item_model_train_sparse": [i32, vp, i32, i32, vp, vp, vp, vp, vp, vp, vp, vp, i32, vp, i32, vp, vp, i32, i32, i64, vp, vp,
                                               vp, vp],
            "mlease_item_model_train_cov": [i32, vp, i32, i32, vp, vp, vp, vp, vp, vp, vp, vp, i32, vp, i32, vp, vp, i32, i64, vp, vp, vp, vp,
                                            i64, vp, vp],
            "mlease_item_model_train_prior": [i32, vp, i32, i32, vp, vp, vp, vp, vp, vp, vp, vp, i32, vp, i32, vp, vp, i32, i32, i64, vp, vp,
                                              vp, vp, vp, vp, vp, vp],
            "mlease_comm_unique_id": [vp],
            "mlease_comm_create": [vp, i32, i32, i32, C.POINTER(vp)],
            "mlease_comm_destroy": [vp],
            "mlease_comm_info": [vp, C.POINTER(i32), C.POINTER(i32), C.POINTER(i32)],
            "mlease_session_set_comm": [vp, vp],
            "mlease_world_create": [C.POINTER(AdmmConfigC), vp, i32, C.POINTER(vp)],
            "mlease_world_destroy": [vp],
            "mlease_world_num_devices": [vp],
            "mlease_world_add_partition_dense": [vp, i32, i64, vp, i64, vp, vp, vp],
            "mlease_world_add_partition_csr": [vp, i32, i64, vp, vp, vp, vp, vp, vp],
            "mlease_world_begin": [vp],
            "mlease_world_begin_initialized": [vp, vp, C.c_float],
            "mlease_world_iterate": [vp, C.POINTER(f64), C.POINTER(i32)],
            "mlease_world_run": [vp, i32, C.POINTER(i32)],
            "mlease_world_get_z": [vp, i32, vp],
            "mlease_world_get_final_model": [vp, i32, vp],
            "mlease_world_get_x": [vp, i32, i32, vp],
            "mlease_world_get_u": [vp, i32, i32, vp],
            "mlease_world_get_uplusx": [vp, i32, i32, vp],
            "mlease_world_fit_partition": [vp, i32, vp, vp, vp, C.POINTER(i32)],
            "mlease_world_get_stats": [vp, C.POINTER(StatsC)],
        }
        for name, args in sig.items():
            fn = getattr(_lib, name)
            fn.argtypes = args
            fn.restype = C.c_int
        _lib.mlease_abi_version.restype = C.c_int
    return _lib


EXPORTED = ["mlease_last_error", "mlease_abi_version", "mlease_session_create", "mlease_session_destroy",
            "mlease_add_partition_dense", "mlease_add_partition_csr", "mlease_admm_begin", "mlease_admm_begin_initialized", "mlease_admm_local_step",
            "mlease_admm_consensus", "mlease_admm_run", "mlease_admm_iterate", "mlease_get_z", "mlease_get_final_model", "mlease_get_x", "mlease_get_u",
            "mlease_get_uplusx", "mlease_get_stats", "mlease_objective", "mlease_fit_partition", "mlease_hessian_vector", "mlease_naive_train_dense",
            "mlease_score", "mlease_test_loglik", "mlease_score_keyed", "mlease_score_keyed_var", "mlease_score_keyed_cov", "mlease_test_loglik_keyed", "mlease_test_auc", "mlease_time_kernel", "mlease_profile",
            "mlease_posterior_variance", "mlease_admm_posterior", "mlease_world_admm_posterior", "mlease_score_var", "mlease_naive_train", "mlease_item_model_train", "mlease_naive_train_sparse", "mlease_item_model_train_sparse", "mlease_item_model_train_cov", "mlease_item_model_train_prior", "mlease_comm_unique_id", "mlease_comm_create", "mlease_comm_destroy", "mlease_comm_info", "mlease_session_set_comm",
            "mlease_world_create", "mlease_world_destroy", "mlease_world_num_devices", "mlease_world_add_partition_dense",
            "mlease_world_add_partition_csr", "mlease_world_begin", "mlease_world_begin_initialized", "mlease_world_iterate",
            "mlease_world_run", "mlease_world_get_z", "mlease_world_get_final_model", "mlease_world_get_x", "mlease_world_get_u",
            "mlease_world_get_uplusx", "mlease_world_fit_partition", "mlease_world_get_stats"]


def check(rc):
    if rc != 0:
        raise MleaseError(rc, lib().mlease_last_error().decode(errors="replace"))


def ptr(a):
    """Raw address of a numpy array / torch tensor (host or CUDA) / int / None."""
    if a is None:
        return None
    if isinstance(a, int):
        return a
    if hasattr(a, "data_ptr"):
        return a.data_ptr()
    return a.ctypes.data
