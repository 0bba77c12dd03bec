"""ctypes binding of include/skelly_b200.h.

Array convention = the reference's: an Eigen column-major ``3 x n`` matrix is a C-contiguous ``(n, 3)``
float64 numpy array here (same bytes); stresslet strengths are ``(n, 9)``.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

KERNEL_STOKESLET = 0
KERNEL_STRESSLET = 1

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = os.environ.get("SKB_LIBRARY") or os.path.join(_HERE, "lib", "libskelly_b200.so")  # override: tuning A/B only
_dp = C.POINTER(C.c_double)
_lib = None
BOUND_FUNCTIONS = ()  # names of the C-ABI functions this binding declares signatures for (filled by library())


class SkbError(RuntimeError):
    """Raised for every non-zero status of the C ABI (mirrors the std::runtime_error of the C++ wrapper)."""


class EvalStats(C.Structure):
    _fields_ = [("kernel_ms", C.c_double), ("total_ms", C.c_double), ("n_pairs", C.c_int64),
                ("launches", C.c_int32), ("targets_per_thread", C.c_int32), ("source_splits", C.c_int32),
                ("grid_ctas", C.c_int32)]


class FlowStats(C.Structure):
    _fields_ = [("device_ms", C.c_double), ("total_ms", C.c_double), ("n_pairs", C.c_int64), ("launches", C.c_int32)]


class SolveInfo(C.Structure):
    """skb_solve_info (include/skelly_b200_flow.h): the outcome of skb_flow_solve_system."""
    _fields_ = [("converged", C.c_int32), ("iterations", C.c_int32), ("restarts", C.c_int32), ("reserved", C.c_int32),
                ("implicit_residual", C.c_double), ("explicit_residual", C.c_double), ("residual", C.c_double)]

    def as_dict(self):
        return {name: getattr(self, name) for name, _ in self._fields_ if name != "reserved"}


GMRES_MAX_BLOCKS = 1024  # SKB_GMRES_MAX_BLOCKS
ERR_STATE = 4  # SKB_ERR_STATE


class StepInfo(C.Structure):
    """skb_step_info (include/skelly_b200_flow.h): the outcome of skb_flow_step."""
    _fields_ = [("solve", SolveInfo), ("fiber_error", C.c_double), ("worst_fiber", C.c_int32), ("collided", C.c_int32)]

    def as_dict(self):
        return dict(self.solve.as_dict(), fiber_error=self.fiber_error, worst_fiber=self.worst_fiber,
                    collided=self.collided)


PERIPHERY_NONE, PERIPHERY_SPHERE, PERIPHERY_ELLIPSOID = 0, 1, 2  # SKB_PERIPHERY_*


class PeripheryShape(C.Structure):
    """skb_periphery_shape (include/skelly_b200_flow.h)"""
    _fields_ = [("kind", C.c_int32), ("binding_active", C.c_int32), ("a", C.c_double), ("b", C.c_double),
                ("c", C.c_double), ("f_0", C.c_double), ("l_0", C.c_double), ("polar_angle_start", C.c_double),
                ("polar_angle_end", C.c_double), ("binding_threshold", C.c_double)]


class LineRequest(C.Structure):
    _fields_ = [("dt_init", C.c_double), ("t_final", C.c_double), ("abs_err", C.c_double), ("rel_err", C.c_double),
                ("back_integrate", C.c_int32), ("max_points", C.c_int32)]


class DenseStats(C.Structure):
    _fields_ = [("kernel_ms", C.c_double), ("total_ms", C.c_double), ("bytes", C.c_int64)]


class DynamicInstability(C.Structure):
    """skb_dynamic_instability (include/skelly_b200_flow.h): the [dynamic_instability] table (params.hpp:30-42)"""
    _fields_ = [("n_nodes", C.c_int32), ("reserved", C.c_int32), ("v_growth", C.c_double),
                ("f_catastrophe", C.c_double), ("v_grow_collision_scale", C.c_double),
                ("f_catastrophe_collision_scale", C.c_double), ("nucleation_rate", C.c_double), ("radius", C.c_double),
                ("min_length", C.c_double), ("bending_rigidity", C.c_double)]


class DynamicInfo(C.Structure):
    _fields_ = [("removed", C.c_int32), ("nucleated", C.c_int32), ("grown", C.c_int32), ("reserved", C.c_int32),
                ("mu", C.c_double)]


class FiberParams(C.Structure):
    """skb_fiber_params (include/skelly_b200_flow.h): the per-fiber scalars of skb_flow_build_fiber_operators."""
    _fields_ = [("length_prev", C.c_double), ("bending_rigidity", C.c_double), ("radius", C.c_double),
                ("penalty_param", C.c_double), ("beta_tstep", C.c_double), ("minus_clamped", C.c_int32),
                ("plus_hinged", C.c_int32)]


# the same record as a numpy dtype: a whole container's parameters are filled column by column
FIBER_PARAMS_DTYPE = np.dtype([(name, np.float64 if ct is C.c_double else np.int32) for name, ct in FiberParams._fields_])


def library_path() -> str:
    return _LIB


def build_library(force: bool = False) -> str:
    """Compile libskelly_b200.so for sm_90a with nvcc (cross-compiles without a GPU)."""
    src = os.path.join(_HERE, "csrc")
    if force:
        subprocess.run(["make", "-C", src, "clean"], check=True, stdout=subprocess.DEVNULL)
    r = subprocess.run(["make", "-C", src], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError("building libskelly_b200.so failed:\n" + r.stdout[-4000:])
    return _LIB


def library() -> C.CDLL:
    """Load the CUDA library.  Missing library == hard error: there is no other implementation to fall back to."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(_LIB):
        raise SkbError(f"{_LIB} is missing: build it with skellysim_b200.build_library() "
                       "(nvcc, sm_90a). There is no CPU or PyTorch fallback.")
    L = C.CDLL(_LIB)
    ctxp = C.c_void_p
    sig = {
        "skb_version": ([], C.c_char_p),
        "skb_last_error_string": ([], C.c_char_p),
        "skb_device_count": ([C.POINTER(C.c_int)], C.c_int),
        "skb_stokeslet_direct": ([_dp, _dp, C.c_int, _dp, _dp, C.c_int], C.c_int),
        "skb_stresslet_direct": ([_dp, _dp, C.c_int, _dp, _dp, C.c_int], C.c_int),
        "skb_ctx_create": ([C.c_int, C.POINTER(ctxp)], C.c_int),
        "skb_ctx_create_on": ([C.POINTER(C.c_int), C.c_int, C.POINTER(ctxp)], C.c_int),
        "skb_ctx_destroy": ([ctxp], C.c_int),
        "skb_ctx_n_gpus": ([ctxp, C.POINTER(C.c_int)], C.c_int),
        "skb_set_targets": ([ctxp, _dp, C.c_int64], C.c_int),
        "skb_set_sources": ([ctxp, C.c_int, _dp, C.c_int64], C.c_int),
        "skb_eval": ([ctxp, C.c_int, _dp, _dp, C.c_int], C.c_int),
        "skb_eval_fused": ([ctxp, _dp, _dp, _dp], C.c_int),
        "skb_set_source_normals": ([ctxp, _dp, C.c_int64], C.c_int),
        "skb_eval_double_layer": ([ctxp, _dp, C.c_double, _dp, C.c_int], C.c_int),
        "skb_set_source_exclusion_ids": ([ctxp, C.POINTER(C.c_int32), C.c_int64], C.c_int),
        "skb_set_targets_device": ([ctxp, C.c_void_p, C.c_int64, C.c_void_p], C.c_int),
        "skb_set_sources_device": ([ctxp, C.c_int, C.c_void_p, C.c_int64, C.c_void_p], C.c_int),
        "skb_eval_device": ([ctxp, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p], C.c_int),
        "skb_sync": ([ctxp], C.c_int),
        "skb_last_eval_stats": ([ctxp, C.POINTER(EvalStats)], C.c_int),
        "skb_launch_count": ([], C.c_int64),
        "skb_buffer_alloc_count": ([], C.c_int64),
        "skb_ctx_set_tuning": ([ctxp, C.c_int, C.c_int], C.c_int),
        "skb_measure_fp64_peak": ([ctxp, C.POINTER(C.c_double)], C.c_int),
        "skb_ctx_set_symmetric": ([ctxp, C.c_int], C.c_int),
        "skb_plan_query": ([C.c_int, C.c_int64, C.c_int64, C.c_int, C.POINTER(C.c_int), C.c_int, C.c_int]
                           + [C.POINTER(C.c_int)] * 4, C.c_int),
        "skb_sym_plan_query": ([C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int),
                                C.POINTER(C.c_int)], C.c_int),
        "skb_sym_groups_per_block": ([], C.c_int),
        "skb_ctx_set_sym_partition": ([ctxp, C.c_int, C.c_int], C.c_int),
        "skb_ctx_last_sym_kernel": ([ctxp, C.POINTER(C.c_double), C.POINTER(C.c_int64)], C.c_int),
        "skb_flow_last_sym_kernel": ([ctxp, C.POINTER(C.c_double), C.POINTER(C.c_int64)], C.c_int),
        "skb_ctx_last_eval_was_symmetric": ([ctxp, C.POINTER(C.c_int)], C.c_int),
        # include/skelly_b200_flow.h
        "skb_flow_create": ([C.c_int, C.POINTER(ctxp)], C.c_int),
        "skb_flow_destroy": ([ctxp], C.c_int),
        "skb_flow_set_fibers": ([ctxp, _dp, C.POINTER(C.c_int), _dp, C.c_int], C.c_int),
        "skb_flow_set_periphery": ([ctxp, _dp, _dp, C.c_int64], C.c_int),
        "skb_flow_set_bodies": ([ctxp, _dp, _dp, C.c_int64, _dp, C.c_int], C.c_int),
        "skb_flow_fibers": ([ctxp, _dp, C.c_int64, _dp, C.c_double, C.c_int, _dp], C.c_int),
        "skb_flow_periphery": ([ctxp, _dp, C.c_int64, _dp, C.c_double, _dp], C.c_int),
        "skb_flow_bodies": ([ctxp, _dp, C.c_int64, _dp, _dp, C.c_double, _dp], C.c_int),
        "skb_flow_matvec": ([ctxp, _dp, _dp, _dp, _dp, C.c_double, _dp], C.c_int),
        "skb_flow_last_stats": ([ctxp, C.POINTER(FlowStats)], C.c_int),
        "skb_flow_set_point_sources": ([ctxp, _dp, _dp, _dp, C.c_int], C.c_int),
        "skb_flow_set_background": ([ctxp, C.POINTER(C.c_int), _dp, _dp], C.c_int),
        "skb_flow_velocity_at_targets": ([ctxp, _dp, C.c_int64, _dp, _dp, _dp, _dp, C.c_double, _dp], C.c_int),
        "skb_flow_set_listener_frame": ([ctxp, _dp, _dp, _dp, _dp, _dp, C.POINTER(C.c_int32), _dp, C.c_double],
                                        C.c_int),
        "skb_flow_set_listener_state": ([ctxp, C.POINTER(FiberParams), C.c_double, C.c_double, _dp, _dp,
                                         C.POINTER(C.c_int32), _dp, C.c_int32], C.c_int),
        "skb_flow_set_listener_state_device": ([ctxp, C.POINTER(FiberParams), C.c_double, C.c_double, C.c_void_p,
                                                C.c_void_p, C.POINTER(C.c_int32), _dp, C.c_int32, C.c_void_p], C.c_int),
        "skb_flow_listener_velocity": ([ctxp, _dp, C.c_int64, _dp], C.c_int),
        "skb_flow_listener_gradient": ([ctxp, _dp, C.c_int64, _dp, _dp], C.c_int),
        "skb_flow_listener_lines": ([ctxp, C.c_int, _dp, C.c_int32, C.POINTER(LineRequest), _dp, _dp, _dp,
                                     C.POINTER(C.c_int32), C.POINTER(C.c_int32)], C.c_int),
        "skb_flow_set_target_window": ([ctxp, C.c_int64, C.c_int64], C.c_int),
        "skb_flow_set_self_exclusion": ([ctxp, C.c_int], C.c_int),
        "skb_flow_set_overlap": ([ctxp, C.c_int], C.c_int),
        "skb_dense_apply_background_device": ([ctxp, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p], C.c_int),
        "skb_flow_set_cross": ([ctxp, C.c_int], C.c_int),
        "skb_flow_group_init": ([ctxp, C.c_int, C.c_int], C.c_int),
        "skb_flow_group_export": ([ctxp, C.c_void_p], C.c_int),
        "skb_flow_group_import": ([ctxp, C.c_int, C.c_void_p], C.c_int),
        "skb_flow_group_connect": ([ctxp, C.c_int, ctxp], C.c_int),
        "skb_flow_group_error": ([ctxp, C.POINTER(C.c_int)], C.c_int),
        "skb_flow_group_warmup": ([ctxp], C.c_int),
        "skb_flow_group_set_solo": ([ctxp, C.c_int], C.c_int),
        "skb_flow_apply_matvec_device": ([ctxp, ctxp] + [C.c_void_p] * 6 + [C.c_double] + [C.c_void_p] * 4, C.c_int),
        "skb_partition_query": ([C.POINTER(C.c_int), C.c_int, C.c_int64, C.c_int64, C.c_int, C.c_int,
                                 C.POINTER(C.c_int64)], C.c_int),
        "skb_mflow_create": ([C.POINTER(C.c_int), C.c_int, C.POINTER(ctxp)], C.c_int),
        "skb_mflow_n_devices": ([ctxp, C.POINTER(C.c_int)], C.c_int),
        "skb_mflow_partition": ([ctxp, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int)] + [C.POINTER(C.c_int64)] * 4,
                                C.c_int),
        "skb_mflow_set_dense": ([ctxp, C.c_int, _dp, C.c_int64, C.c_int64], C.c_int),
        "skb_mflow_apply_system_matvec": ([ctxp, _dp, C.c_double, _dp], C.c_int),
        "skb_mflow_apply_system_preconditioner": ([ctxp, _dp, _dp], C.c_int),
        "skb_flow_set_target_ranges": ([ctxp, C.c_int, C.c_int] + [C.c_int64] * 4, C.c_int),
        "skb_flow_apply_fiber_force_device": ([ctxp, C.c_void_p, C.c_void_p, C.c_void_p], C.c_int),
        "skb_flow_fiber_matvec_device": ([ctxp] + [C.c_void_p] * 5, C.c_int),
        "skb_flow_set_fiber_class": ([ctxp, C.c_int, _dp, _dp], C.c_int),
        "skb_flow_set_fiber_operators": ([ctxp, _dp, _dp, _dp, _dp, C.POINTER(C.c_int)], C.c_int),
        "skb_flow_apply_fiber_force": ([ctxp, _dp, _dp], C.c_int),
        "skb_flow_set_fiber_preconditioner": ([ctxp, _dp], C.c_int),
        "skb_flow_apply_fiber_preconditioner": ([ctxp, _dp, _dp], C.c_int),
        "skb_flow_apply_fiber_preconditioner_device": ([ctxp, C.c_void_p, C.c_void_p, C.c_void_p], C.c_int),
        "skb_flow_fiber_matvec": ([ctxp, _dp, _dp, _dp, _dp], C.c_int),
        "skb_flow_set_fiber_class_derivatives": ([ctxp, C.c_int, _dp, _dp, _dp], C.c_int),
        "skb_flow_build_fiber_operators": ([ctxp, C.POINTER(FiberParams), C.c_double, C.c_double], C.c_int),
        "skb_flow_get_fiber_operators": ([ctxp, _dp, _dp, _dp, _dp], C.c_int),
        "skb_flow_build_fiber_rhs": ([ctxp, C.POINTER(FiberParams), _dp, _dp, _dp, _dp, C.c_double, C.c_double, _dp],
                                     C.c_int),
        "skb_flow_build_fiber_rhs_device": ([ctxp, C.POINTER(FiberParams), _dp, _dp, C.c_void_p, C.c_void_p,
                                             C.c_double, C.c_double, C.c_void_p, C.c_void_p], C.c_int),
        "skb_flow_apply_matvec": ([ctxp, _dp, _dp, _dp, _dp, _dp, C.c_double, _dp, _dp, _dp], C.c_int),
        "skb_flow_apply_matvec_dense": ([ctxp, ctxp, _dp, _dp, _dp, _dp, _dp, C.c_double, _dp, _dp, _dp], C.c_int),
        "skb_dense_apply_device": ([ctxp, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p], C.c_int),
        "skb_dense_shape": ([ctxp, C.c_int, C.POINTER(C.c_int64), C.POINTER(C.c_int64)], C.c_int),
        # include/skelly_b200_dense.h
        "skb_dense_create": ([C.c_int, C.POINTER(ctxp)], C.c_int),
        "skb_dense_create_on": ([C.POINTER(C.c_int), C.c_int, C.POINTER(ctxp)], C.c_int),
        "skb_dense_device": ([ctxp, C.c_int, C.POINTER(C.c_int)], C.c_int),
        "skb_dense_destroy": ([ctxp], C.c_int),
        "skb_dense_set_matrix": ([ctxp, C.c_int, _dp, C.c_int64, C.c_int64], C.c_int),
        "skb_dense_apply": ([ctxp, C.c_int, _dp, _dp, _dp], C.c_int),
        "skb_dense_last_stats": ([ctxp, C.POINTER(DenseStats)], C.c_int),
        "skb_flow_matvec_device": ([ctxp] + [C.c_void_p] * 5 + [C.c_double, C.c_void_p, C.c_void_p], C.c_int),
        "skb_flow_set_body_operators": ([ctxp, C.POINTER(C.c_int), C.c_int, _dp, _dp, _dp, _dp, _dp], C.c_int),
        "skb_flow_set_fiber_links": ([ctxp, C.POINTER(C.c_int), _dp, _dp], C.c_int),
        "skb_flow_apply_system_matvec": ([ctxp, ctxp, _dp, C.c_double, _dp], C.c_int),
        "skb_flow_apply_system_matvec_device": ([ctxp, ctxp, C.c_void_p, C.c_double, C.c_void_p, C.c_void_p], C.c_int),
        "skb_flow_apply_system_preconditioner": ([ctxp, ctxp, _dp, _dp], C.c_int),
        "skb_flow_apply_system_preconditioner_device": ([ctxp, ctxp, C.c_void_p, C.c_void_p, C.c_void_p], C.c_int),
        "skb_flow_build_system_rhs": ([ctxp, C.POINTER(FiberParams), _dp, _dp, _dp, _dp, C.c_double, C.c_double, _dp],
                                      C.c_int),
        "skb_flow_build_system_rhs_device": ([ctxp, C.POINTER(FiberParams), _dp, _dp] + [C.c_void_p] * 3
                                             + [C.c_double, C.c_double, C.c_void_p, C.c_void_p], C.c_int),
        "skb_group_body_pieces": ([C.POINTER(C.c_int), C.c_int, C.c_int64, C.c_int64, C.POINTER(C.c_int64), C.c_int,
                                   C.POINTER(C.c_int)], C.c_int),
        "skb_flow_set_body_frames": ([ctxp, C.POINTER(C.c_int), C.c_int] + [_dp] * 7, C.c_int),
        "skb_flow_place_bodies": ([ctxp, _dp, _dp], C.c_int),
        "skb_flow_get_body_operators": ([ctxp, _dp, _dp, _dp, _dp], C.c_int),
        "skb_flow_set_gmres": ([ctxp, C.c_int], C.c_int),
        "skb_flow_solve_system": ([ctxp, ctxp, _dp, C.c_double, C.c_double, C.c_int, C.c_int, _dp,
                                   C.POINTER(SolveInfo), _dp], C.c_int),
        "skb_flow_solve_system_device": ([ctxp, ctxp, C.c_void_p, C.c_double, C.c_double, C.c_int, C.c_int,
                                          C.c_void_p, C.POINTER(SolveInfo), _dp, C.c_void_p], C.c_int),
        "skb_flow_group_solve_system_device": ([ctxp, ctxp, ctxp, C.c_void_p, C.c_double, C.c_double, C.c_int, C.c_int,
                                                C.c_void_p, C.POINTER(SolveInfo), _dp, C.c_void_p], C.c_int),
        "skb_flow_step": ([ctxp, ctxp, C.POINTER(FiberParams), _dp, _dp, _dp, _dp, C.POINTER(C.c_int), _dp, C.c_double,
                           C.c_double, C.c_double, C.c_int, C.c_int, _dp, _dp, C.POINTER(StepInfo)], C.c_int),
        "skb_flow_fiber_error": ([ctxp, _dp, _dp], C.c_int),
        "skb_flow_get_placement": ([ctxp, _dp, _dp], C.c_int),
        "skb_flow_get_fibers": ([ctxp, _dp], C.c_int),
        "skb_mflow_step": ([ctxp, C.POINTER(FiberParams), _dp, _dp, _dp, _dp, C.POINTER(C.c_int), _dp, C.c_double,
                            C.c_double, C.c_double, C.c_int, C.c_int, _dp, _dp, C.POINTER(StepInfo)], C.c_int),
        "skb_flow_group_step_device": ([ctxp, ctxp, ctxp, C.POINTER(FiberParams), _dp, _dp] + [C.c_void_p] * 3
                                       + [C.POINTER(C.c_int), _dp, C.c_double, C.c_double, C.c_double, C.c_int,
                                          C.c_int, C.c_void_p, C.c_void_p, C.POINTER(StepInfo), C.c_void_p], C.c_int),
        "skb_flow_set_periphery_shape": ([ctxp, C.POINTER(PeripheryShape), C.POINTER(C.c_int32), _dp], C.c_int),
        "skb_flow_periphery_interaction": ([ctxp, _dp, C.POINTER(C.c_int32), C.POINTER(C.c_int32)], C.c_int),
        "skb_flow_set_nucleation_sites": ([ctxp, C.POINTER(C.c_int), _dp], C.c_int),
        "skb_flow_dynamic_instability": ([ctxp, C.POINTER(DynamicInstability), C.c_double, C.c_uint64, C.c_uint64,
                                          C.c_int, C.POINTER(FiberParams), C.POINTER(C.c_int32),
                                          C.POINTER(C.c_int32), C.c_int, C.POINTER(C.c_int), C.POINTER(FiberParams),
                                          C.POINTER(C.c_int32), _dp, C.POINTER(C.c_int32), C.POINTER(DynamicInfo)],
                                         C.c_int),
        "skb_flow_step_flags": ([ctxp, C.POINTER(C.c_int32)], C.c_int),
        "skb_mflow_solve_system": ([ctxp, _dp, C.c_double, C.c_double, C.c_int, C.c_int, _dp, C.POINTER(SolveInfo),
                                    _dp], C.c_int),
    }
    # the skb_mflow_ and skb_flow_group_ calls whose arguments are those of their skb_flow_ twin
    for name in ("destroy", "set_fibers", "set_periphery", "set_bodies", "set_self_exclusion", "set_cross",
                 "set_overlap", "set_fiber_class", "set_fiber_class_derivatives", "set_fiber_operators",
                 "set_fiber_preconditioner", "build_fiber_operators", "build_fiber_rhs", "matvec", "apply_matvec",
                 "velocity_at_targets", "set_point_sources", "set_background", "set_body_operators", "set_body_frames",
                 "place_bodies", "set_fiber_links", "set_periphery_shape", "periphery_interaction", "build_system_rhs",
                 "set_gmres", "get_fibers", "get_placement", "last_stats"):
        sig["skb_mflow_" + name] = sig["skb_flow_" + name]
    for name in ("set_body_operators", "set_body_frames", "place_bodies", "set_fiber_links",
                 "apply_system_matvec_device", "apply_system_preconditioner_device", "build_system_rhs_device"):
        sig["skb_flow_group_" + name] = sig["skb_flow_" + name]
    global BOUND_FUNCTIONS
    BOUND_FUNCTIONS = tuple(sorted(sig))
    for name, (args, res) in sig.items():
        fn = getattr(L, name)
        fn.argtypes = args
        fn.restype = res
    _lib = L
    return L


def _check(rc: int):
    if rc != 0:
        raise SkbError(f"skelly_b200 error {rc}: {library().skb_last_error_string().decode()}")


def _arr(x, cols):
    x = np.ascontiguousarray(x, dtype=np.float64)
    if x.size == 0:
        return x.reshape(0, cols)
    if x.ndim != 2 or x.shape[1] != cols:
        raise ValueError(f"expected an (n, {cols}) array, got {x.shape}")
    return x


def _p(x):
    return x.ctypes.data_as(_dp)


def _class_derivatives(n_nodes, D_2_0, D_3_0, D_4_0):
    n = int(n_nodes)
    Ds = [np.asfortranarray(D, dtype=np.float64) for D in (D_2_0, D_3_0, D_4_0)]
    if any(D.shape != (n, n) for D in Ds):
        raise ValueError(f"derivative matrices for n={n}: got {[D.shape for D in Ds]}")
    return n, Ds


def fiber_params(n_fibers, length_prev, bending_rigidity, radius, penalty_param, beta_tstep, minus_clamped,
                 plus_hinged):
    """skb_fiber_params of n_fibers fibers; every argument is a per-fiber array or a scalar for all of them."""
    p = np.zeros(int(n_fibers), dtype=FIBER_PARAMS_DTYPE)
    for name, v in zip(FIBER_PARAMS_DTYPE.names, (length_prev, bending_rigidity, radius, penalty_param, beta_tstep,
                                                   minus_clamped, plus_hinged)):
        v = np.asarray(v)
        if v.ndim and v.shape != (int(n_fibers),):
            raise ValueError(f"{name}: expected a scalar or {int(n_fibers)} values, got shape {v.shape}")
        p[name] = v
    return p


def _params_ptr(p):
    return p.ctypes.data_as(C.POINTER(FiberParams)) if p.size else None


def _per_fiber(v, n_fibers):
    """None (the C ABI's NULL) or a per-fiber array / scalar as n_fibers contiguous doubles"""
    if v is None:
        return None
    v = np.asarray(v, dtype=np.float64)
    if v.ndim and v.shape != (int(n_fibers),):
        raise ValueError(f"expected a scalar or {int(n_fibers)} values, got shape {v.shape}")
    return np.ascontiguousarray(np.broadcast_to(v, (int(n_fibers),)))


def _opt_p(x):
    return None if x is None else _p(x)


def _vp(a):
    """a device address (an int, e.g. torch.Tensor.data_ptr()) as a void pointer; 0 is NULL"""
    return C.c_void_p(a) if a else None


def _dense_h(dense):
    """the handle of a Dense, or NULL for None"""
    return dense._h if dense is not None else None


# The body and fiber-link set-up of a flow through its C call `name`: the plain call, or on a Flow its group_ twin,
# which takes the same arguments.
def _body_operators_call(fl, name, n_nodes, node_weights, ex, ey, ez, A_inv_list):
    n = np.ascontiguousarray(n_nodes, dtype=np.int32)
    w = np.ascontiguousarray(node_weights, dtype=np.float64).reshape(-1)
    ex, ey, ez = _arr(ex, 3), _arr(ey, 3), _arr(ez, 3)
    Ai = None if A_inv_list is None else fl._colmajor_concat(A_inv_list)
    fl._call(name, n.ctypes.data_as(C.POINTER(C.c_int)), int(n.shape[0]), _p(w), _p(ex), _p(ey), _p(ez), _opt_p(Ai))
    fl._body_sol, fl._body_n = int(np.sum(3 * n + 6)), n


def _frame_call(fl, name, n_nodes, node_pos_ref, node_normal_ref, node_weights, ex0, ey0, ez0, A_inv0_list):
    n = np.ascontiguousarray(n_nodes, dtype=np.int32)
    w = np.ascontiguousarray(node_weights, dtype=np.float64).reshape(-1)
    Ai = None if A_inv0_list is None else fl._colmajor_concat(A_inv0_list)
    rest = (_arr(node_pos_ref, 3), _arr(node_normal_ref, 3), w, _arr(ex0, 3), _arr(ey0, 3), _arr(ez0, 3))
    fl._call(name, n.ctypes.data_as(C.POINTER(C.c_int)), int(n.shape[0]), *(_p(a) for a in rest), _opt_p(Ai))
    fl._body_sol, fl._body_n = int(np.sum(3 * n + 6)), n


def _place_call(fl, name, centers, orientations):
    c, q = _arr(centers, 3), _arr(orientations, 4)
    assert c.shape[0] == q.shape[0]
    fl._call(name, _p(c), _p(q))


def _links_call(fl, name, body, site, bending_rigidity):
    if body is None:
        fl._call(name, None, None, None)
        return
    b = np.ascontiguousarray(body, dtype=np.int32)
    st = _arr(site, 3)
    E = np.ascontiguousarray(np.broadcast_to(np.asarray(bending_rigidity, dtype=np.float64), b.shape))
    assert st.shape[0] == b.shape[0]
    fl._call(name, b.ctypes.data_as(C.POINTER(C.c_int)), _p(st), _p(E))


def _fiber_rhs_args(n_fibers, n_nodes, params, v_growth, force_scale, v_on_fibers, f_external):
    """skb_fiber_params, v_growth, force_scale and the (n_nodes, 3) inputs of a fiber RHS call, each None where absent"""
    p = fiber_params(n_fibers, *params)
    v, f = (None if a is None else _arr(a, 3) for a in (v_on_fibers, f_external))
    for a in (v, f):
        if a is not None and a.shape[0] != n_nodes:
            raise ValueError(f"expected ({n_nodes}, 3) node values, got {a.shape}")
    return p, _per_fiber(v_growth, n_fibers), _per_fiber(force_scale, n_fibers), v, f


def _system_rhs_args(n_fibers, n_nodes, n_bodies, params, v_growth, force_scale, f_external, body_forces_torques):
    """_fiber_rhs_args of a system RHS call (f_external in place of the flow) and its (n_bodies, 6) external F_T, each
    None where absent"""
    p, vg, fs, _, f = _fiber_rhs_args(n_fibers, n_nodes, params, v_growth, force_scale, None, f_external)
    ft = None if body_forces_torques is None else _arr(body_forces_torques, 6)
    if ft is not None and ft.shape[0] != n_bodies:
        raise ValueError(f"expected ({n_bodies}, 6) body forces and torques, got {ft.shape}")
    return p, vg, fs, f, ft


def _interaction_call(fl, n_nodes, n_fibers):
    f = np.empty((n_nodes, 3))
    hinged = np.empty(n_fibers, dtype=np.int32)
    collided = C.c_int32(0)
    fl._call("periphery_interaction", _p(f), hinged.ctypes.data_as(C.POINTER(C.c_int32)), C.byref(collided))
    return f, hinged, bool(collided.value)


def device_count() -> int:
    n = C.c_int(0)
    library().skb_device_count(C.byref(n))
    return n.value


def launch_count() -> int:
    return int(library().skb_launch_count())


def buffer_alloc_count() -> int:
    """device allocations of the library's grow-only buffers in this process (skb_buffer_alloc_count)"""
    return int(library().skb_buffer_alloc_count())


def stokeslet_direct(r_src, f_src, r_trg):
    """kernels::stokeslet_direct_gpu_impl semantics (kernels.hpp:17): 1/(8 pi) included, 1/eta not."""
    r_src, f_src, r_trg = _arr(r_src, 3), _arr(f_src, 3), _arr(r_trg, 3)
    if r_src.shape[0] != f_src.shape[0]:
        raise ValueError("r_src / f_src size mismatch")
    u = np.empty((r_trg.shape[0], 3))
    _check(library().skb_stokeslet_direct(_p(r_src), _p(f_src), r_src.shape[0], _p(r_trg), _p(u), r_trg.shape[0]))
    return u


def stresslet_direct(r_src, f_src, r_trg):
    """kernels::stresslet_direct_gpu_impl semantics (kernels.hpp:19)."""
    r_src, f_src, r_trg = _arr(r_src, 3), _arr(f_src, 9), _arr(r_trg, 3)
    if r_src.shape[0] != f_src.shape[0]:
        raise ValueError("r_src / f_src size mismatch")
    u = np.empty((r_trg.shape[0], 3))
    _check(library().skb_stresslet_direct(_p(r_src), _p(f_src), r_src.shape[0], _p(r_trg), _p(u), r_trg.shape[0]))
    return u


class _Handle:
    """The lifetime of a library handle self._h: close() (or the end of a with block, or garbage collection) releases
    it once through the C function named _destroy; closing again does nothing."""
    _destroy = None

    def close(self):
        if getattr(self, "_h", None) and self._h.value:
            getattr(library(), self._destroy)(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()


class Context(_Handle):
    """Evaluator context: positions cached on the device(s), strengths shipped per evaluation."""
    _destroy = "skb_ctx_destroy"

    def __init__(self, n_gpus: int = 1, device_ids=None):
        self._h = C.c_void_p()
        L = library()
        if device_ids is None:
            _check(L.skb_ctx_create(int(n_gpus), C.byref(self._h)))
        else:
            ids = (C.c_int * len(device_ids))(*device_ids)
            _check(L.skb_ctx_create_on(ids, len(device_ids), C.byref(self._h)))
        self.n_trg = 0
        self.n_src = {KERNEL_STOKESLET: 0, KERNEL_STRESSLET: 0}

    @property
    def n_gpus(self) -> int:
        n = C.c_int(0)
        _check(library().skb_ctx_n_gpus(self._h, C.byref(n)))
        return n.value

    # ---- host-pointer API ----
    def set_targets(self, r_trg):
        r_trg = _arr(r_trg, 3)
        _check(library().skb_set_targets(self._h, _p(r_trg), r_trg.shape[0]))
        self.n_trg = r_trg.shape[0]

    def set_sources(self, kind, r_src):
        r_src = _arr(r_src, 3)
        _check(library().skb_set_sources(self._h, int(kind), _p(r_src), r_src.shape[0]))
        self.n_src[int(kind)] = r_src.shape[0]

    def set_source_exclusion_ids(self, ids):
        """Opt-in fused self-exclusion: Stokeslet sources that are the leading targets; pairs with equal ids (fiber
        indices) contribute exactly 0.  None switches it off."""
        if ids is None:
            _check(library().skb_set_source_exclusion_ids(self._h, None, 0))
            return
        ids = np.ascontiguousarray(ids, dtype=np.int32).reshape(-1)
        _check(library().skb_set_source_exclusion_ids(self._h, ids.ctypes.data_as(C.POINTER(C.c_int32)), ids.shape[0]))

    def set_source_normals(self, normals):
        normals = _arr(normals, 3)
        _check(library().skb_set_source_normals(self._h, _p(normals), normals.shape[0]))

    def eval(self, kind, f_src, out=None, accumulate=False):
        f_src = _arr(f_src, 3 if kind == KERNEL_STOKESLET else 9)
        if f_src.shape[0] != self.n_src[int(kind)]:
            raise ValueError("strength count does not match the sources set")
        if out is None:
            if accumulate:
                raise ValueError("accumulate needs an output array")
            out = np.empty((self.n_trg, 3))
        assert out.flags.c_contiguous and out.dtype == np.float64 and out.shape == (self.n_trg, 3)
        _check(library().skb_eval(self._h, int(kind), _p(f_src), _p(out), int(bool(accumulate))))
        return out

    def eval_fused(self, f_sl=None, f_dl=None):
        out = np.empty((self.n_trg, 3))
        a = _arr(f_sl, 3) if f_sl is not None else None
        b = _arr(f_dl, 9) if f_dl is not None else None
        _check(library().skb_eval_fused(self._h, _p(a) if a is not None else None,
                                        _p(b) if b is not None else None, _p(out)))
        return out

    def eval_double_layer(self, density, eta, out=None, accumulate=False):
        density = _arr(density, 3)
        if out is None:
            out = np.empty((self.n_trg, 3))
        _check(library().skb_eval_double_layer(self._h, _p(density), float(eta), _p(out), int(bool(accumulate))))
        return out

    # ---- device-pointer API (addresses as ints, e.g. torch.Tensor.data_ptr()) ----
    def set_targets_device(self, ptr: int, n_trg: int, stream: int = 0):
        _check(library().skb_set_targets_device(self._h, C.c_void_p(ptr), int(n_trg), C.c_void_p(stream)))
        self.n_trg = int(n_trg)

    def set_sources_device(self, kind, ptr: int, n_src: int, stream: int = 0):
        _check(library().skb_set_sources_device(self._h, int(kind), C.c_void_p(ptr), int(n_src), C.c_void_p(stream)))
        self.n_src[int(kind)] = int(n_src)

    def eval_device(self, kind, f_ptr: int, u_ptr: int, accumulate=False, stream: int = 0):
        _check(library().skb_eval_device(self._h, int(kind), C.c_void_p(f_ptr), C.c_void_p(u_ptr),
                                         int(bool(accumulate)), C.c_void_p(stream)))

    def sync(self):
        _check(library().skb_sync(self._h))

    # ---- instrumentation ----
    def stats(self) -> dict:
        s = EvalStats()
        _check(library().skb_last_eval_stats(self._h, C.byref(s)))
        return {k: getattr(s, k) for k, _ in EvalStats._fields_}

    def set_tuning(self, targets_per_thread=0, source_splits=0):
        _check(library().skb_ctx_set_tuning(self._h, int(targets_per_thread), int(source_splits)))

    def set_symmetric(self, mode: int):
        """-1 auto, 0 off, 1 on: Newton's-third-law kernel for sources that are the leading targets."""
        _check(library().skb_ctx_set_symmetric(self._h, int(mode)))

    def set_sym_partition(self, part: int, n_parts: int):
        """One rank per GPU: evaluate only the block rows of the self-interaction owned by `part`; the leading
        n_src rows of the result are partial sums to be all-reduced over the parts."""
        _check(library().skb_ctx_set_sym_partition(self._h, int(part), int(n_parts)))

    def last_sym_kernel(self):
        ms, pairs = C.c_double(0), C.c_int64(0)
        _check(library().skb_ctx_last_sym_kernel(self._h, C.byref(ms), C.byref(pairs)))
        return ms.value, pairs.value

    def last_eval_was_symmetric(self) -> bool:
        y = C.c_int(0)
        _check(library().skb_ctx_last_eval_was_symmetric(self._h, C.byref(y)))
        return bool(y.value)

    def measure_fp64_peak(self) -> float:
        v = C.c_double(0)
        _check(library().skb_measure_fp64_peak(self._h, C.byref(v)))
        return v.value


class _FlowBase(_Handle):
    """What Flow and MultiFlow share: every call whose C twins (skb_flow_* and skb_mflow_*) take the same arguments
    after the handle.  A subclass names its C prefix, and its _own_fibers() / _pieces() give the fibers and rows the
    calls cover: a Flow's own window or ranges, all of them on a MultiFlow."""
    _prefix = None
    _step_takes_dense = False  # skb_flow_step takes the Dense handle after the flow's; skb_mflow_step does not

    def _fn(self, name):
        return getattr(library(), self._prefix + name)

    def _call(self, name, *args):
        _check(self._fn(name)(self._h, *args))

    def _n_fibers(self):
        return len(getattr(self, "_fiber_off", [0])) - 1

    def set_fibers(self, r_fib, n_nodes, lengths):
        r_fib = _arr(r_fib, 3)
        n_nodes = np.ascontiguousarray(n_nodes, dtype=np.int32)
        lengths = np.ascontiguousarray(lengths, dtype=np.float64)
        assert n_nodes.shape == lengths.shape and int(n_nodes.sum()) == r_fib.shape[0]
        self._call("set_fibers", _p(r_fib), n_nodes.ctypes.data_as(C.POINTER(C.c_int)), _p(lengths),
                   int(n_nodes.shape[0]))
        self.n_fib = r_fib.shape[0]
        self._fiber_off = np.concatenate([[0], np.cumsum(n_nodes, dtype=np.int64)])
        self._lengths = lengths.copy()

    def set_periphery(self, node_pos, node_normal):
        node_pos, node_normal = _arr(node_pos, 3), _arr(node_normal, 3)
        self._call("set_periphery", _p(node_pos), _p(node_normal), node_pos.shape[0])
        self.n_shell = node_pos.shape[0]

    def set_bodies(self, node_pos, node_normal, centers):
        node_pos, node_normal, centers = _arr(node_pos, 3), _arr(node_normal, 3), _arr(centers, 3)
        self._call("set_bodies", _p(node_pos), _p(node_normal), node_pos.shape[0], _p(centers), centers.shape[0])
        self.n_body, self.n_bodies = node_pos.shape[0], centers.shape[0]

    def set_point_sources(self, positions, forces, torques):
        """The point sources (velocity_at_targets and build_system_rhs include them)."""
        positions, forces, torques = _arr(positions, 3), _arr(forces, 3), _arr(torques, 3)
        self._call("set_point_sources", _p(positions), _p(forces), _p(torques), positions.shape[0])

    def set_background(self, components, scale_factor, uniform):
        comp = (C.c_int * 3)(*[int(c) for c in components])
        sc = np.ascontiguousarray(scale_factor, dtype=np.float64)
        un = np.ascontiguousarray(uniform, dtype=np.float64)
        self._call("set_background", comp, _p(sc), _p(un))

    def velocity_at_targets(self, r_trg, fib_forces, shell_density, body_densities, body_forces_torques, eta):
        """System::velocity_at_targets (system.cpp:355-359): fiber (no self subtraction) + body + periphery flows."""
        r_trg = _arr(r_trg, 3)
        a, b, c = _arr(fib_forces, 3), _arr(shell_density, 3), _arr(body_densities, 3)
        ft = _arr(body_forces_torques, 6)
        vel = np.empty((r_trg.shape[0], 3))
        self._call("velocity_at_targets", _p(r_trg), r_trg.shape[0], _p(a), _p(b), _p(c), _p(ft), float(eta), _p(vel))
        return vel

    def set_cross(self, mode: int):
        """Fiber <-> periphery pairs of the matvec in one geometry pass: -1 auto (default), 0 never, 1 whenever applicable."""
        self._call("set_cross", int(mode))

    def set_self_exclusion(self, fused: bool):
        """Matvec self term: False = the reference's compute-then-subtract (default); True = the pair kernels skip
        intra-fiber pairs (SURVEY.md 8f N3)."""
        self._call("set_self_exclusion", int(bool(fused)))

    def set_overlap(self, on: bool):
        """Periphery dense operator beside the pair kernels on a side stream (default) or as one kernel at the end."""
        self._call("set_overlap", int(bool(on)))

    def matvec(self, fib_forces, shell_density, body_densities, body_forces_torques, eta):
        a, b, c = _arr(fib_forces, 3), _arr(shell_density, 3), _arr(body_densities, 3)
        ft = _arr(body_forces_torques, 6)
        v = np.empty((sum(self._pieces()), 3))
        self._call("matvec", _p(a), _p(b), _p(c), _p(ft), float(eta), _p(v))
        return v

    # ---- per-fiber dense operators (SURVEY.md §8f N2); matrices go in column-major like Eigen's .data() ----
    def set_fiber_class(self, n_nodes: int, D_1_0, P_downsample_bc):
        """FiberFiniteDifference::matrices_.at(n): D_1_0 (n,n), P_downsample_bc (4n-14,4n)."""
        n = int(n_nodes)
        D = np.asfortranarray(D_1_0, dtype=np.float64)
        P = np.asfortranarray(P_downsample_bc, dtype=np.float64)
        if D.shape != (n, n) or P.shape != (4 * n - 14, 4 * n):
            raise ValueError(f"class matrices for n={n}: got {D.shape}, {P.shape}")
        self._call("set_fiber_class", n, _p(D), _p(P))

    @staticmethod
    def _colmajor_concat(mats):
        """Per-fiber matrices -> one buffer, every matrix column-major (Eigen's .data()).  A 3-D C-ordered stack of
        equal shapes is transposed in one pass; a list may be ragged."""
        if isinstance(mats, np.ndarray) and mats.ndim == 3:
            return np.ascontiguousarray(np.asarray(mats, dtype=np.float64).transpose(0, 2, 1)).reshape(-1)
        if len(mats) == 0:
            return np.zeros(0)
        return np.concatenate([np.asarray(m, dtype=np.float64).ravel(order="F") for m in mats])

    def set_fiber_preconditioner(self, A_inv_list):
        """Explicit inverses of A_ (fib.A_LU_.inverse()), same fibers and order as set_fiber_operators."""
        Ai = self._colmajor_concat(A_inv_list)
        self._call("set_fiber_preconditioner", _p(Ai))

    def set_fiber_class_derivatives(self, n_nodes: int, D_2_0, D_3_0, D_4_0):
        """The higher derivative matrices of FiberFiniteDifference::matrices_.at(n) (pre-transposed like D_1_0), needed
        by build_fiber_operators for every node count in use."""
        n, (D2, D3, D4) = _class_derivatives(n_nodes, D_2_0, D_3_0, D_4_0)
        self._call("set_fiber_class_derivatives", n, _p(D2), _p(D3), _p(D4))

    def build_fiber_operators(self, length_prev, bending_rigidity, radius, penalty_param, beta_tstep, minus_clamped,
                              plus_hinged, dt, eta):
        """A_, force_operator_, xs_ and A_^-1 of the (own) fibers built on the device from the positions and lengths of
        set_fibers (update_derivatives, update_linear_operator, update_force_operator, the operator half of
        apply_bc_rectangular, update_preconditioner).  Per-fiber arrays or scalars; the flags are 0 / 1.  A MultiFlow
        takes them for all fibers, and every device builds its own slice."""
        f0, f1 = self._own_fibers()
        p = fiber_params(f1 - f0, length_prev, bending_rigidity, radius, penalty_param, beta_tstep, minus_clamped,
                         plus_hinged)
        self._call("build_fiber_operators", _params_ptr(p), float(dt), float(eta))

    def build_fiber_rhs(self, length_prev, bending_rigidity, radius, penalty_param, beta_tstep, minus_clamped,
                        plus_hinged, dt, eta, v_on_fibers=None, f_external=None, v_growth=None, force_scale=None):
        """The fiber block of the RHS (4 N_own,) as System::prep_state_for_solver leaves it: update_RHS with f_external
        + force_scale xs_, then the RHS half of apply_bc_rectangular with f_external.  Parameters as for
        build_fiber_operators; v_on_fibers / f_external (N_own, 3) and v_growth / force_scale (per-fiber arrays or
        scalars) may be None: no flow / force, zero growth, no motors."""
        f0, f1 = self._own_fibers()
        n_own = self._pieces()[0]
        p, vg, fs, v, f = _fiber_rhs_args(f1 - f0, n_own, (length_prev, bending_rigidity, radius, penalty_param,
                                                           beta_tstep, minus_clamped, plus_hinged),
                                          v_growth, force_scale, v_on_fibers, f_external)
        rhs = np.empty(4 * n_own)
        self._call("build_fiber_rhs", _params_ptr(p), _opt_p(vg), _opt_p(fs), _opt_p(v), _opt_p(f), float(dt),
                   float(eta), _p(rhs))
        return rhs

    # ---- the whole solution vector [fibers | shell | bodies] with the bodies on the device ----
    def set_body_operators(self, n_nodes, node_weights, ex, ey, ez, A_inv_list=None):
        """Per body (order of set_bodies = order in the solution vector): node count, node_weights_ (N_b,), ex_ / ey_ /
        ez_ (N_b, 3) each, and A_^-1 ((3n+6, 3n+6) per body, a list) or None (no system preconditioner for bodies).
        On a MultiFlow every device keeps the bodies it owns rows of."""
        _body_operators_call(self, "set_body_operators", n_nodes, node_weights, ex, ey, ez, A_inv_list)

    def set_body_frames(self, n_nodes, node_pos_ref, node_normal_ref, node_weights, ex0, ey0, ez0, A_inv0_list=None):
        """The bodies' operators in their body frame, once per run after set_bodies: per body its node count, per node
        node_positions_ref_ / node_normals_ref_ (N_b, 3) and node_weights_ (N_b,), ex_ / ey_ / ez_ (N_b, 3) and
        A_^-1 ((3n+6, 3n+6) per body, a list, or None) of the body at identity orientation.  place_bodies then forms
        the placed operators on the device.  On a MultiFlow every device keeps the body-frame inverses it owns rows
        of."""
        _frame_call(self, "set_body_frames", n_nodes, node_pos_ref, node_normal_ref, node_weights, ex0, ey0, ez0,
                    A_inv0_list)

    def place_bodies(self, centers, orientations):
        """Once per timestep: the bodies at centres (n_bodies, 3) and unit quaternions (w, x, y, z) (n_bodies, 4) --
        their nodes, normals and operators, as set_bodies + set_body_operators with the placed ones would leave them.
        The fiber links are dropped."""
        _place_call(self, "place_bodies", centers, orientations)

    def set_fiber_links(self, body=None, site=None, bending_rigidity=None):
        """Per fiber: body index (-1 free), lab-frame nucleation site (n_fibers, 3), bending_rigidity_; body=None: no
        fiber is bound."""
        _links_call(self, "set_fiber_links", body, site, bending_rigidity)

    def solution_size(self) -> int:
        """4 N_f + 3 N_s + sum(3 n_b + 6) (the bodies' part as set_body_operators was last given)"""
        return 4 * self.n_fib + 3 * self.n_shell + (getattr(self, "_body_sol", 0) if self.n_bodies else 0)

    def build_system_rhs(self, length_prev, bending_rigidity, radius, penalty_param, beta_tstep, minus_clamped,
                         plus_hinged, dt, eta, f_external=None, body_forces_torques=None, v_growth=None,
                         force_scale=None):
        """System::prep_state_for_solver's RHS (system.cpp:398-458) as a whole solution vector (solution_size(),):
        the flow of f_external (N_f, 3) and of the bodies' external forces / torques (n_bodies, 6), plus the point
        sources and the background flow, into the fiber block (build_fiber_rhs's parameters), -v_shell and
        [-v_body ; 0] per body.  f_external / body_forces_torques None: zero."""
        f0, f1 = self._own_fibers()
        p, vg, fs, f, ft = _system_rhs_args(f1 - f0, self.n_fib, self.n_bodies,
                                            (length_prev, bending_rigidity, radius, penalty_param, beta_tstep,
                                             minus_clamped, plus_hinged), v_growth, force_scale, f_external,
                                            body_forces_torques)
        rhs = np.empty(self.solution_size())
        self._call("build_system_rhs", _params_ptr(p), _opt_p(vg), _opt_p(fs), _opt_p(f), _opt_p(ft), float(dt),
                   float(eta), _p(rhs))
        return rhs

    def set_gmres(self, num_blocks: int = 300):
        """Size the workspace of solve_system for the current solution size and up to num_blocks basis vectors (after
        set_body_operators; a MultiFlow also lays out every member's local rows)."""
        self._call("set_gmres", int(num_blocks))
        self._gmres_blocks = int(num_blocks)

    def set_periphery_shape(self, kind, a, b=0.0, c=0.0, f_0=20.0, l_0=0.05, binding_active=False,
                            polar_angle_start=0.0, polar_angle_end=np.pi, binding_threshold=0.75,
                            fiber_minus_clamped=None, body_radius=None):
        """The periphery's shape for the step (skb_flow_set_periphery_shape): kind PERIPHERY_SPHERE (radius a),
        PERIPHERY_ELLIPSOID (semi-axes a, b, c) or PERIPHERY_NONE (clears it); fiber_periphery_interaction f_0, l_0;
        periphery_binding active, polar angles and threshold; per fiber the TOML flag minus_clamped_ (None: all 0);
        per body the radius of a spherical body (0: not spherical; None: no body takes part).  The step then adds the
        repulsion to f_external, takes plus_hinged from the binding and reports the collision test in info["collided"]."""
        n_fibers = self._n_fibers()
        s = PeripheryShape(int(kind), int(binding_active), float(a), float(b), float(c), float(f_0), float(l_0),
                           float(polar_angle_start), float(polar_angle_end), float(binding_threshold))
        mc = None if fiber_minus_clamped is None else np.ascontiguousarray(fiber_minus_clamped, dtype=np.int32)
        if mc is not None and mc.shape != (n_fibers,):
            raise ValueError(f"expected {n_fibers} fiber_minus_clamped flags, got {mc.shape}")
        br = None if body_radius is None else np.ascontiguousarray(body_radius, dtype=np.float64)
        if br is not None and br.shape != (self.n_bodies,):
            raise ValueError(f"expected {self.n_bodies} body radii, got {br.shape}")
        self._call("set_periphery_shape", C.byref(s), None if mc is None else mc.ctypes.data_as(C.POINTER(C.c_int32)),
                   _opt_p(br))
        # kept so that the shape can be set again for another fiber set (timestep.Stepper.restore)
        self._shape = dict(kind=kind, a=a, b=b, c=c, f_0=f_0, l_0=l_0, binding_active=binding_active,
                           polar_angle_start=polar_angle_start, polar_angle_end=polar_angle_end,
                           binding_threshold=binding_threshold, body_radius=body_radius,
                           fiber_minus_clamped=np.zeros(n_fibers, dtype=np.int32)
                           if fiber_minus_clamped is None else np.array(fiber_minus_clamped, dtype=np.int32))

    def step(self, length_prev, bending_rigidity, radius, penalty_param, beta_tstep, minus_clamped, plus_hinged, dt,
             eta, dense=None, f_external=None, body_forces_torques=None, fiber_body=None, site_ref=None,
             v_growth=None, force_scale=None, tol=1e-10, num_blocks=300, max_iters=1000):
        """System::step (system.cpp:482-492) on the device: links, fiber operators, RHS and solve at the current
        geometry, then the fibers' and bodies' step and the new geometry installed.  fiber_body (N_fibers,) ints, -1
        free, or None; site_ref (N_fibers, 3) body-frame nucleation sites, or None.  Returns (x, tension, info): info
        a dict of skb_step_info (the solve's fields, fiber_error, worst_fiber, collided).  A solution with non-finite
        new positions installs nothing and returns fiber_error NaN.  With set_periphery_shape, plus_hinged is ignored
        (the binding sets it) and the repulsion is added to f_external.  A MultiFlow does not use dense: the
        periphery's operators come from set_dense."""
        n_fibers = self._n_fibers()
        p, vg, fs, f, ft = _system_rhs_args(n_fibers, self.n_fib, self.n_bodies,
                                            (length_prev, bending_rigidity, radius, penalty_param, beta_tstep,
                                             minus_clamped, plus_hinged), v_growth, force_scale, f_external,
                                            body_forces_torques)
        fb = None if fiber_body is None else np.ascontiguousarray(fiber_body, dtype=np.int32).reshape(-1)
        if fb is not None and fb.shape[0] != n_fibers:
            raise ValueError(f"expected {n_fibers} fiber_body entries, got {fb.shape[0]}")
        sr = None if site_ref is None else _arr(site_ref, 3)
        x = np.empty(self.solution_size())
        tension = np.empty(self.n_fib)
        info = StepInfo()
        handles = (self._h, _dense_h(dense)) if self._step_takes_dense else (self._h,)
        rc = self._fn("step")(*handles, _params_ptr(p), _opt_p(vg), _opt_p(fs), _opt_p(f), _opt_p(ft),
                              None if fb is None else fb.ctypes.data_as(C.POINTER(C.c_int)), _opt_p(sr), float(dt),
                              float(eta), float(tol), int(num_blocks), int(max_iters), _p(x), _p(tension),
                              C.byref(info))
        # SKB_ERR_STATE with a NaN fiber_error is the step that was not installed: reported, not raised
        if not (rc == ERR_STATE and np.isnan(info.fiber_error)):
            _check(rc)
        return x, tension, info.as_dict()

    def fibers(self):
        """the fiber positions (N_f, 3) of the last set_fibers or step"""
        r = np.empty((self.n_fib, 3))
        self._call("get_fibers", _p(r))
        return r

    def placement(self):
        """(centres (n_bodies, 3), quaternions (n_bodies, 4)) of the last place_bodies or step"""
        c, q = np.empty((self.n_bodies, 3)), np.empty((self.n_bodies, 4))
        self._call("get_placement", _p(c), _p(q))
        return c, q

    def stats(self) -> dict:
        s = FlowStats()
        self._call("last_stats", C.byref(s))
        return {k: getattr(s, k) for k, _ in FlowStats._fields_}


class Flow(_FlowBase):
    """Device-resident flow() layer (include/skelly_b200_flow.h): FiberContainer / Periphery / BodyContainer flows
    and the fused hydrodynamic part of System::apply_matvec."""
    _destroy = "skb_flow_destroy"
    _prefix = "skb_flow_"
    _step_takes_dense = True

    def __init__(self, device: int = 0):
        self._h = C.c_void_p()
        _check(library().skb_flow_create(int(device), C.byref(self._h)))
        self.n_fib = self.n_shell = self.n_body = self.n_bodies = 0

    def fiber_flow(self, r_trg, fib_forces, eta, subtract_self=True):
        r_trg, fib_forces = _arr(r_trg, 3), _arr(fib_forces, 3)
        vel = np.empty((r_trg.shape[0], 3))
        _check(library().skb_flow_fibers(self._h, _p(r_trg), r_trg.shape[0], _p(fib_forces), float(eta),
                                         int(bool(subtract_self)), _p(vel)))
        return vel

    def periphery_flow(self, r_trg, density, eta):
        r_trg, density = _arr(r_trg, 3), _arr(density, 3)
        vel = np.empty((r_trg.shape[0], 3))
        _check(library().skb_flow_periphery(self._h, _p(r_trg), r_trg.shape[0], _p(density), float(eta), _p(vel)))
        return vel

    def body_flow(self, r_trg, densities, forces_torques, eta):
        r_trg, densities = _arr(r_trg, 3), _arr(densities, 3)
        ft = _arr(forces_torques, 6)
        vel = np.empty((r_trg.shape[0], 3))
        _check(library().skb_flow_bodies(self._h, _p(r_trg), r_trg.shape[0], _p(densities), _p(ft), float(eta),
                                         _p(vel)))
        return vel

    def set_listener_frame(self, fib_forces, shell_density, body_densities, body_forces_torques, body_velocities,
                           body_kind, body_radii, eta):
        """The listener's frame (listener.cpp): the strengths of velocity_at_targets, and per body [U, omega]
        (body_velocities, (n_bodies, 6)), the interior test (body_kind: 0 none, 1 sphere, 2 ellipsoid) and its radii
        ((n_bodies, 3); a sphere reads the first).  Stale once the geometry, point sources or background change."""
        a, b, c = _arr(fib_forces, 3), _arr(shell_density, 3), _arr(body_densities, 3)
        ft, uv, radii = _arr(body_forces_torques, 6), _arr(body_velocities, 6), _arr(body_radii, 3)
        kind = np.ascontiguousarray(body_kind, dtype=np.int32).reshape(-1)
        _check(library().skb_flow_set_listener_frame(self._h, _p(a), _p(b), _p(c), _p(ft), _p(uv),
                                                     kind.ctypes.data_as(C.POINTER(C.c_int32)), _p(radii),
                                                     float(eta)))

    def velocity_field(self, r):
        """The listener's velocity_field: System::velocity_at_targets on the frame, (n, 3), with the rigid motion
        U + omega x dx at points inside a body."""
        r = _arr(r, 3)
        vel = np.empty((r.shape[0], 3))
        _check(library().skb_flow_listener_velocity(self._h, _p(r), r.shape[0], _p(vel)))
        return vel

    def _lines(self, kind, x0, dt_init, t_final, abs_err, rel_err, back_integrate, max_points):
        x0 = _arr(x0, 3)
        n, mp = x0.shape[0], int(max_points)
        req = LineRequest(float(dt_init), float(t_final), float(abs_err), float(rel_err), int(bool(back_integrate)), mp)
        row = max(2 * mp - 1, 1)
        x, val, t = np.empty((n, row, 3)), np.empty((n, row, 3)), np.empty((n, row))
        n_points, status = np.empty(n, dtype=np.int32), np.empty((n, 2), dtype=np.int32)
        i32 = C.POINTER(C.c_int32)
        _check(library().skb_flow_listener_lines(self._h, int(kind), _p(x0), n, C.byref(req), _p(x), _p(t), _p(val),
                                                 n_points.ctypes.data_as(i32), status.ctypes.data_as(i32)))
        return [{"x": x[i, :k].copy(), "time": t[i, :k].copy(), "val": val[i, :k].copy(),
                 "status": (int(status[i, 0]), int(status[i, 1]))} for i, k in enumerate(n_points)]

    def streamlines(self, x0, dt_init=0.1, t_final=1.0, abs_err=1e-10, rel_err=1e-6, back_integrate=True,
                    max_points=1000):
        """The listener's streamlines (StreamLine::compute) from the seeds x0 (n, 3), all at once on the device.
        One dict per seed, the reader's keys: "x" (m, 3), "time" (m,), "val" (m, 3) the velocity there, and
        "status" (back, forward): 0 reached +-t_final, 1 |v| > 1e3, 2 500 failed tries, 3 max_points in that
        direction."""
        return self._lines(0, x0, dt_init, t_final, abs_err, rel_err, back_integrate, max_points)

    def vortexlines(self, x0, dt_init=0.1, t_final=1.0, abs_err=1e-10, rel_err=1e-6, back_integrate=True,
                    max_points=1000):
        """The listener's vortex lines (VortexLine::compute): streamlines() of the vorticity (central differences at
        +-1e-7); "val" is the vorticity, the exits still test the velocity."""
        return self._lines(1, x0, dt_init, t_final, abs_err, rel_err, back_integrate, max_points)

    def set_target_window(self, begin: int, end: int = -1):
        """Evaluate only rows [begin, end) of [fibers | periphery | bodies] in matvec() (one rank's block)."""
        _check(library().skb_flow_set_target_window(self._h, int(begin), int(end)))
        self._window, self._ranges = (int(begin), int(end)), None

    def set_target_ranges(self, fiber_begin, fiber_end, shell_begin, shell_end, body_begin, body_end):
        """The reference's MPI decomposition: whole fibers [fiber_begin, fiber_end), periphery rows, body-node rows;
        matvec() then returns [own fiber nodes | own shell rows | own body rows]."""
        r = tuple(int(v) for v in (fiber_begin, fiber_end, shell_begin, shell_end, body_begin, body_end))
        _check(library().skb_flow_set_target_ranges(self._h, *r))
        self._ranges, self._window = r, None

    def _pieces(self):
        """(own fiber nodes, own shell rows, own body rows) of the current window / ranges."""
        nf, ns, nb = self.n_fib, self.n_shell, self.n_body
        cl = lambda x, lo, hi: min(max(x, lo), hi)
        if getattr(self, "_ranges", None):
            f0, f1, s0, s1, b0, b1 = self._ranges
            off = getattr(self, "_fiber_off", np.zeros(1, dtype=np.int64))
            nfib = len(off) - 1
            f0 = cl(f0, 0, nfib)
            f1 = cl(f1, f0, nfib)
            s0 = cl(s0, 0, ns)
            b0 = cl(b0, 0, nb)
            return int(off[f1] - off[f0]), cl(s1, s0, ns) - s0, cl(b1, b0, nb) - b0
        w0, w1 = getattr(self, "_window", None) or (0, -1)
        n_all = nf + ns + nb
        w0 = cl(w0, 0, n_all)
        w1 = n_all if w1 < 0 else cl(w1, w0, n_all)
        return (cl(w1, 0, nf) - cl(w0, 0, nf), cl(w1 - nf, 0, ns) - cl(w0 - nf, 0, ns),
                cl(w1 - nf - ns, 0, nb) - cl(w0 - nf - ns, 0, nb))

    def matvec_device(self, d_fib_forces: int, d_shell_density: int, d_body_densities: int, d_body_forces: int,
                      d_body_torques: int, eta: float, d_v_window: int, stream: int = 0):
        """Device-pointer matvec (addresses as ints); asynchronous on `stream`."""
        _check(library().skb_flow_matvec_device(self._h, C.c_void_p(d_fib_forces), C.c_void_p(d_shell_density),
                                                C.c_void_p(d_body_densities), C.c_void_p(d_body_forces),
                                                C.c_void_p(d_body_torques), float(eta), C.c_void_p(d_v_window),
                                                C.c_void_p(stream)))

    # ---- per-fiber dense operators (SURVEY.md §8f N2); matrices go in column-major like Eigen's .data() ----
    def set_fiber_operators(self, A_list, force_list, xs, length_prev, plus_bc_velocity, colmajor=False):
        """A_ (4n,4n) and force_operator_ (3n,4n) per fiber (lists, or (n_fibers, rows, cols) stacks), tangents xs
        (N_f,3), length_prev_, plus-end velocity BC -- of the OWN fibers when target ranges are set.  colmajor=True:
        A_list / force_list are already the concatenated column-major buffers (Eigen's .data()), passed through."""
        if colmajor:
            A = np.ascontiguousarray(A_list, dtype=np.float64).reshape(-1)
            F = np.ascontiguousarray(force_list, dtype=np.float64).reshape(-1)
        else:
            A, F = self._colmajor_concat(A_list), self._colmajor_concat(force_list)
        xs = _arr(xs, 3)
        lp = np.ascontiguousarray(length_prev, dtype=np.float64)
        pl = np.ascontiguousarray(plus_bc_velocity, dtype=np.int32)
        assert xs.shape[0] == self._pieces()[0] and lp.shape == pl.shape and (colmajor or lp.shape == (len(A_list),))
        _check(library().skb_flow_set_fiber_operators(self._h, _p(A), _p(F), _p(xs), _p(lp),
                                                      pl.ctypes.data_as(C.POINTER(C.c_int))))

    def _own_fibers(self):
        """(first, end) fiber of the current window / ranges (all fibers without either)."""
        off = getattr(self, "_fiber_off", np.zeros(1, dtype=np.int64))
        nfib = len(off) - 1
        if getattr(self, "_ranges", None):
            f0 = min(max(self._ranges[0], 0), nfib)
            return f0, min(max(self._ranges[1], f0), nfib)
        w0, w1 = getattr(self, "_window", None) or (0, -1)
        nf = int(off[-1])
        w0 = min(max(w0, 0), nf)
        w1 = nf if w1 < 0 else min(max(w1, w0), nf)
        return int(np.searchsorted(off, w0)), int(np.searchsorted(off, w1))

    def build_fiber_rhs_device(self, length_prev, bending_rigidity, radius, penalty_param, beta_tstep, minus_clamped,
                               plus_hinged, dt, eta, d_v_on_fibers: int, d_f_external: int, d_rhs: int, v_growth=None,
                               force_scale=None, stream: int = 0):
        """build_fiber_rhs on device pointers (0: none for the inputs), asynchronous on `stream`; returns once the
        per-fiber tables are staged."""
        f0, f1 = self._own_fibers()
        p, vg, fs, _, _ = _fiber_rhs_args(f1 - f0, 0, (length_prev, bending_rigidity, radius, penalty_param,
                                                       beta_tstep, minus_clamped, plus_hinged),
                                          v_growth, force_scale, None, None)
        _check(library().skb_flow_build_fiber_rhs_device(self._h, _params_ptr(p), _opt_p(vg), _opt_p(fs),
                                                         _vp(d_v_on_fibers), _vp(d_f_external), float(dt), float(eta),
                                                         C.c_void_p(d_rhs), C.c_void_p(stream)))

    def get_fiber_operators(self, inverse=True):
        """The resident operators of the (own) fibers: dict(A=[(4n,4n)], force=[(3n,4n)], xs=(N_own,3),
        A_inv=[(4n,4n)] or None)."""
        f0, f1 = self._own_fibers()
        n_nodes = np.diff(getattr(self, "_fiber_off", np.zeros(1, dtype=np.int64)))[f0:f1].astype(int)
        A = np.empty(int(np.sum(16 * n_nodes ** 2)))
        F = np.empty(int(np.sum(12 * n_nodes ** 2)))
        Ai = np.empty_like(A) if inverse else None
        xs = np.empty((int(np.sum(n_nodes)), 3))
        _check(library().skb_flow_get_fiber_operators(self._h, _p(A), _p(F), _p(xs), _p(Ai) if inverse else None))

        def split(buf, rows):
            out, o = [], 0
            for n in n_nodes:
                out.append(buf[o:o + rows * n * 4 * n].reshape(4 * n, rows * n).T)
                o += rows * n * 4 * n
            return out
        return dict(A=split(A, 4), force=split(F, 3), xs=xs, A_inv=split(Ai, 4) if inverse else None)

    def apply_fiber_preconditioner(self, x_fibers):
        """fc.apply_preconditioner (fcfd.cpp:331-339): y = A_^-1 x per (own) fiber."""
        x = np.ascontiguousarray(x_fibers, dtype=np.float64).reshape(-1)
        assert x.shape[0] == 4 * self._pieces()[0]
        y = np.empty_like(x)
        _check(library().skb_flow_apply_fiber_preconditioner(self._h, _p(x), _p(y)))
        return y

    def apply_fiber_preconditioner_device(self, d_x_fibers: int, d_y: int, stream: int = 0):
        _check(library().skb_flow_apply_fiber_preconditioner_device(self._h, C.c_void_p(d_x_fibers), C.c_void_p(d_y),
                                                                    C.c_void_p(stream)))

    def apply_fiber_force(self, x_fibers):
        """fc.apply_fiber_force (fcfd.cpp:272-287): (4 N_f,) -> fw (N_f, 3)."""
        x = np.ascontiguousarray(x_fibers, dtype=np.float64).reshape(-1)
        n_own = self._pieces()[0]
        assert x.shape[0] == 4 * n_own
        fw = np.empty((n_own, 3))
        _check(library().skb_flow_apply_fiber_force(self._h, _p(x), _p(fw)))
        return fw

    def fiber_matvec(self, x_fibers, v_fibers, v_fib_boundary=None):
        """fc.matvec (fcfd.cpp:216-232): x (4 N_f,), v (N_f,3), v_fib_boundary (n_fibers,7) or None -> res (4 N_f,)."""
        x = np.ascontiguousarray(x_fibers, dtype=np.float64).reshape(-1)
        v = _arr(v_fibers, 3)
        n_own = self._pieces()[0]
        assert x.shape[0] == 4 * n_own and v.shape[0] == n_own
        vb = None if v_fib_boundary is None else _arr(v_fib_boundary, 7)
        res = np.empty(4 * n_own)
        _check(library().skb_flow_fiber_matvec(self._h, _p(x), _p(v), None if vb is None else _p(vb), _p(res)))
        return res

    def apply_fiber_force_device(self, d_x_fibers: int, d_fw: int, stream: int = 0):
        _check(library().skb_flow_apply_fiber_force_device(self._h, C.c_void_p(d_x_fibers), C.c_void_p(d_fw),
                                                           C.c_void_p(stream)))

    def fiber_matvec_device(self, d_x_fibers: int, d_v_fibers: int, d_v_fib_boundary: int, d_res: int,
                            stream: int = 0):
        _check(library().skb_flow_fiber_matvec_device(self._h, C.c_void_p(d_x_fibers), C.c_void_p(d_v_fibers),
                                                      _vp(d_v_fib_boundary), C.c_void_p(d_res), C.c_void_p(stream)))

    def apply_matvec(self, x_fibers, shell_density, body_densities, body_forces_torques, eta,
                     fiber_link_conditions=None, dense=None, out=None):
        """System::apply_matvec (system.cpp:298-318) with the fiber operators on the device.
        Returns (res_fibers (4 N_f,), v_shell (N_s,3), v_bodies (N_b,3)); with dense= a single-device Dense holding
        stresslet_plus_complementary the second item is res_shell = shell.matvec(x_shell, v_shell) instead."""
        x = np.ascontiguousarray(x_fibers, dtype=np.float64).reshape(-1)
        assert x.shape[0] == 4 * self.n_fib
        b, c = _arr(shell_density, 3), _arr(body_densities, 3)
        ft = _arr(body_forces_torques, 6)
        vb = None if fiber_link_conditions is None else _arr(fiber_link_conditions, 7)
        if out is not None:  # caller's (e.g. pinned) buffers: (res (4 N_f,), v_shell (N_s,3), v_bodies (N_b,3))
            res, v_s, v_b = out
            assert res.shape == (4 * self.n_fib,) and v_s.shape == (self.n_shell, 3) and v_b.shape == (self.n_body, 3)
            assert all(a.flags.c_contiguous and a.dtype == np.float64 for a in out)
        else:
            res = np.empty(4 * self.n_fib)
            v_s, v_b = np.empty((self.n_shell, 3)), np.empty((self.n_body, 3))
        if dense is not None:
            _check(library().skb_flow_apply_matvec_dense(self._h, dense._h, _p(x), _p(b), _p(c), _p(ft),
                                                         None if vb is None else _p(vb), float(eta), _p(res), _p(v_s),
                                                         _p(v_b)))
        else:
            _check(library().skb_flow_apply_matvec(self._h, _p(x), _p(b), _p(c), _p(ft),
                                                   None if vb is None else _p(vb), float(eta), _p(res), _p(v_s),
                                                   _p(v_b)))
        return res, v_s, v_b

    def apply_matvec_device(self, dense, d_x_fibers: int, d_x_shell: int, d_body_densities: int, d_body_forces: int,
                            d_body_torques: int, d_fiber_link_conditions: int, eta: float, d_res_fibers: int,
                            d_out_shell: int, d_v_bodies: int, stream: int = 0):
        """System::apply_matvec with every operand already on the device (addresses as ints, 0 = NULL); OWN slices
        for a group member.  Asynchronous on `stream`."""
        _check(library().skb_flow_apply_matvec_device(self._h, _dense_h(dense), _vp(d_x_fibers), _vp(d_x_shell),
                                                      _vp(d_body_densities), _vp(d_body_forces), _vp(d_body_torques),
                                                      _vp(d_fiber_link_conditions), float(eta), _vp(d_res_fibers),
                                                      _vp(d_out_shell), _vp(d_v_bodies), _vp(stream)))

    # ---- the whole solution vector [fibers | shell | bodies] with the bodies on the device ----
    def get_body_operators(self, inverse=True):
        """The resident body operators: dict(ex, ey, ez (N_b, 3) each, A_inv = per body its (3n+6, 3n+6) inverse, None
        for a body whose inverse a group member does not keep; A_inv None with inverse=False)."""
        n = np.asarray(getattr(self, "_body_n", np.zeros(0, dtype=np.int32)), dtype=np.int64)
        nb = int(n.sum())
        ex, ey, ez = (np.empty((nb, 3)) for _ in range(3))
        node0 = np.concatenate([[0], np.cumsum(n)])
        kept = np.ones(len(n), dtype=bool)
        if getattr(self, "_member", False):  # the bodies with a node in the member's body rows
            b0, b1 = self._ranges[4], self._ranges[5]
            kept = (node0[:-1] < b1) & (node0[1:] > b0)
        m = 3 * n + 6
        Ai = np.empty(int(np.sum(m[kept] ** 2))) if inverse else None
        _check(library().skb_flow_get_body_operators(self._h, _p(ex), _p(ey), _p(ez), _opt_p(Ai)))
        out, o = [], 0
        for k, mk in zip(kept, m):
            if inverse and k:
                out.append(Ai[o:o + mk * mk].reshape(mk, mk).T)
                o += mk * mk
            else:
                out.append(None)
        return dict(ex=ex, ey=ey, ez=ez, A_inv=out if inverse else None)

    def apply_system_matvec(self, x, eta, dense=None):
        """System::apply_matvec (system.cpp:269-324) on the whole solution vector x: returns res = A x."""
        x = np.ascontiguousarray(x, dtype=np.float64).reshape(-1)
        assert x.shape[0] == self.solution_size()
        res = np.empty_like(x)
        _check(library().skb_flow_apply_system_matvec(self._h, _dense_h(dense), _p(x), float(eta), _p(res)))
        return res

    def apply_system_matvec_device(self, dense, d_x: int, eta: float, d_res: int, stream: int = 0):
        _check(library().skb_flow_apply_system_matvec_device(self._h, _dense_h(dense), C.c_void_p(d_x), float(eta),
                                                             C.c_void_p(d_res), C.c_void_p(stream)))

    def apply_system_preconditioner(self, x, dense=None):
        """System::apply_preconditioner (system.cpp:248-262) on the whole solution vector x: returns y = P^-1 x."""
        x = np.ascontiguousarray(x, dtype=np.float64).reshape(-1)
        assert x.shape[0] == self.solution_size()
        y = np.empty_like(x)
        _check(library().skb_flow_apply_system_preconditioner(self._h, _dense_h(dense), _p(x), _p(y)))
        return y

    def apply_system_preconditioner_device(self, dense, d_x: int, d_y: int, stream: int = 0):
        _check(library().skb_flow_apply_system_preconditioner_device(self._h, _dense_h(dense), C.c_void_p(d_x),
                                                                     C.c_void_p(d_y), C.c_void_p(stream)))

    def build_system_rhs_device(self, length_prev, bending_rigidity, radius, penalty_param, beta_tstep,
                                minus_clamped, plus_hinged, dt, eta, d_f_external: int, d_body_forces: int,
                                d_body_torques: int, d_rhs: int, v_growth=None, force_scale=None, stream: int = 0):
        """build_system_rhs on device pointers (0: none for the inputs; forces and torques (n_bodies, 3) each),
        asynchronous on `stream`; returns once the per-fiber tables are staged."""
        f0, f1 = self._own_fibers()
        p, vg, fs, _, _ = _system_rhs_args(f1 - f0, 0, self.n_bodies,
                                           (length_prev, bending_rigidity, radius, penalty_param, beta_tstep,
                                            minus_clamped, plus_hinged), v_growth, force_scale, None, None)
        _check(library().skb_flow_build_system_rhs_device(self._h, _params_ptr(p), _opt_p(vg), _opt_p(fs),
                                                          _vp(d_f_external), _vp(d_body_forces), _vp(d_body_torques),
                                                          float(dt), float(eta), _vp(d_rhs), _vp(stream)))

    def solve_system(self, rhs, eta, dense=None, tol=1e-10, num_blocks=300, max_iters=1000):
        """Solver::solve (solver_hydro.cpp:64-95): x = A^-1 rhs by restarted right-preconditioned GMRES on the device.
        Returns (x, info, history): info a dict of skb_solve_info, history the implicit relative residual after each
        Arnoldi step (history[0] = 1)."""
        b = np.ascontiguousarray(rhs, dtype=np.float64).reshape(-1)
        assert b.shape[0] == self.solution_size()
        x = np.empty_like(b)
        info = SolveInfo()
        hist = np.full(max(int(max_iters), 0) + 1, np.nan)
        _check(library().skb_flow_solve_system(self._h, _dense_h(dense), _p(b), float(eta), float(tol), int(num_blocks),
                                               int(max_iters), _p(x), C.byref(info), _p(hist)))
        return x, info.as_dict(), hist[:info.iterations + 1]

    def solve_system_device(self, dense, d_rhs: int, eta: float, d_x: int, tol=1e-10, num_blocks=300,
                            max_iters=1000, stream: int = 0):
        """solve_system on device pointers, asynchronous on `stream` except for one host wait per Arnoldi step.
        Returns (info, history) as solve_system."""
        info = SolveInfo()
        hist = np.full(max(int(max_iters), 0) + 1, np.nan)
        _check(library().skb_flow_solve_system_device(self._h, _dense_h(dense), C.c_void_p(d_rhs), float(eta),
                                                      float(tol), int(num_blocks), int(max_iters), C.c_void_p(d_x),
                                                      C.byref(info), _p(hist), C.c_void_p(stream)))
        return info.as_dict(), hist[:info.iterations + 1]

    def periphery_interaction(self, n_own_nodes=None, n_own_fibers=None):
        """(repulsion (N, 3) of the own nodes, plus_hinged (own fibers,) int32, collided bool over all fibers and
        bodies) at the current geometry (skb_flow_periphery_interaction); by default all nodes and fibers"""
        return _interaction_call(self, self.n_fib if n_own_nodes is None else int(n_own_nodes),
                                 self._n_fibers() if n_own_fibers is None else int(n_own_fibers))

    def set_nucleation_sites(self, n_sites_per_body, site_ref):
        """the bodies' nucleation_sites_ref_ (body frame), concatenated: n_sites_per_body per body, site_ref (total, 3)
        (skb_flow_set_nucleation_sites)"""
        n = np.ascontiguousarray(n_sites_per_body, dtype=np.int32).reshape(-1)
        s = _arr(site_ref, 3)
        if n.shape[0] != self.n_bodies or int(n.sum()) != s.shape[0]:
            raise ValueError(f"expected {self.n_bodies} site counts summing to {s.shape[0]}, got {n}")
        _check(library().skb_flow_set_nucleation_sites(self._h, n.ctypes.data_as(C.POINTER(C.c_int)), _p(s)))
        self._sites = (n.copy(), s.copy())

    def dynamic_instability(self, di, dt, seed, counter, params, binding, plus_pinned):
        """System::dynamic_instability on the device (skb_flow_dynamic_instability).  di: a dict (or
        DynamicInstability) of the [dynamic_instability] table; params: the seven per-fiber parameters of
        build_fiber_operators (scalars or per fiber) or a FIBER_PARAMS_DTYPE array; binding (N_fibers, 2) ints (body,
        site), -1 free; plus_pinned (N_fibers,) ints.  The flow then holds the new fiber set.  Returns a dict: params
        (FIBER_PARAMS_DTYPE), binding, v_growth, origin (the input fiber of each output fiber, -1 nucleated), n_nodes,
        lengths, and the info fields removed, nucleated, grown, mu."""
        if not isinstance(di, DynamicInstability):
            di = DynamicInstability(**{k: di.get(k, 0) for k, _ in DynamicInstability._fields_ if k != "reserved"})
        nf = self._n_fibers()
        p = params if isinstance(params, np.ndarray) and params.dtype == FIBER_PARAMS_DTYPE else fiber_params(nf, *params)
        p = np.ascontiguousarray(p)
        b = np.ascontiguousarray(binding, dtype=np.int32).reshape(nf, 2)
        pp = np.ascontiguousarray(np.broadcast_to(np.asarray(plus_pinned, dtype=np.int32), (nf,)))
        n_sites = int(self._sites[0].sum()) if getattr(self, "_sites", None) is not None and self.n_bodies else 0
        cap = nf + n_sites
        p_out = np.zeros(cap, dtype=FIBER_PARAMS_DTYPE)
        b_out = np.zeros((cap, 2), dtype=np.int32)
        v_out, origin = np.zeros(cap), np.zeros(cap, dtype=np.int32)
        n_out, info = C.c_int(0), DynamicInfo()
        i32 = lambda a: a.ctypes.data_as(C.POINTER(C.c_int32))
        _check(library().skb_flow_dynamic_instability(self._h, C.byref(di), float(dt), int(seed), int(counter), nf,
                                                       _params_ptr(p), i32(b), i32(pp), cap, C.byref(n_out),
                                                       _params_ptr(p_out), i32(b_out), _p(v_out), i32(origin),
                                                       C.byref(info)))
        m = n_out.value
        origin = origin[:m].copy()
        out = dict(params=p_out[:m].copy(), binding=b_out[:m].copy(), origin=origin, removed=info.removed,
                   nucleated=info.nucleated, grown=info.grown, mu=info.mu)
        old_n = np.diff(self._fiber_off).astype(np.int32) if nf else np.zeros(0, dtype=np.int32)
        if di.n_nodes == 0:
            out.update(v_growth=None, n_nodes=old_n, lengths=self._lengths.copy())
            return out
        out["v_growth"] = v_out[:m].copy()
        out["n_nodes"] = np.where(origin >= 0, old_n[np.maximum(origin, 0)] if nf else 0, di.n_nodes).astype(np.int32)
        # the lengths the device installed: length_prev + dt v (one rounded product and one rounded sum; min_length
        # for a new fiber, whose v is 0)
        out["lengths"] = out["params"]["length_prev"] + float(dt) * out["v_growth"]
        self.n_fib = int(out["n_nodes"].sum())
        self._fiber_off = np.concatenate([[0], np.cumsum(out["n_nodes"], dtype=np.int64)])
        self._lengths = out["lengths"].copy()
        if getattr(self, "_shape", None) is not None:
            mc = self._shape["fiber_minus_clamped"]
            self._shape["fiber_minus_clamped"] = np.where(origin >= 0, mc[np.maximum(origin, 0)] if nf else 0,
                                                          0).astype(np.int32)
        return out

    def step_flags(self):
        """plus_hinged (N_fibers,) int32 of each fiber as the last installed step built it (skb_flow_step_flags)"""
        h = np.empty(self._n_fibers(), dtype=np.int32)
        _check(library().skb_flow_step_flags(self._h, h.ctypes.data_as(C.POINTER(C.c_int32))))
        return h

    def fiber_error(self):
        """fiber_error_local (fcfd.cpp:79-89) of the current geometry on the device: (max, per-fiber maxima)"""
        m = C.c_double(0)
        per = np.empty(self._n_fibers())
        _check(library().skb_flow_fiber_error(self._h, C.byref(m), _p(per)))
        return m.value, per

    # ---- multi-GPU groups (peer memory) ----
    def last_sym_kernel(self):
        """(ms, ordered pairs) of the last launch of the symmetric fiber-fiber kernel inside matvec()."""
        ms, pairs = C.c_double(0), C.c_int64(0)
        _check(library().skb_flow_last_sym_kernel(self._h, C.byref(ms), C.byref(pairs)))
        return ms.value, pairs.value

    def group_init(self, rank: int, size: int):
        _check(library().skb_flow_group_init(self._h, int(rank), int(size)))
        self._member = int(size) > 1

    def group_export(self) -> bytes:
        buf = C.create_string_buffer(64)
        _check(library().skb_flow_group_export(self._h, C.cast(buf, C.c_void_p)))
        return buf.raw

    def group_import(self, peer_rank: int, handle: bytes):
        assert len(handle) == 64
        buf = C.create_string_buffer(handle, 64)
        _check(library().skb_flow_group_import(self._h, int(peer_rank), C.cast(buf, C.c_void_p)))

    def group_connect(self, peer_rank: int, peer: "Flow"):
        _check(library().skb_flow_group_connect(self._h, int(peer_rank), peer._h))

    def group_warmup(self):
        _check(library().skb_flow_group_warmup(self._h))

    def group_set_solo(self, solo: bool):
        _check(library().skb_flow_group_set_solo(self._h, int(bool(solo))))

    def group_error(self) -> int:
        m = C.c_int(-1)
        _check(library().skb_flow_group_error(self._h, C.byref(m)))
        return m.value

    # ---- the whole-vector calls of one rank per GPU, on the member's local vector ----
    def group_set_body_operators(self, n_nodes, node_weights, ex, ey, ez, A_inv_list=None):
        """set_body_operators on a group member (arrays of ALL bodies): it keeps what its body rows need, lays out its
        local vector's body rows and sizes the buffers of the group_* system calls.  Not a member: set_body_operators."""
        _body_operators_call(self, "group_set_body_operators", n_nodes, node_weights, ex, ey, ez, A_inv_list)

    def group_set_body_frames(self, n_nodes, node_pos_ref, node_normal_ref, node_weights, ex0, ey0, ez0,
                              A_inv0_list=None):
        """set_body_frames on a group member (arrays of ALL bodies): it keeps the body-frame inverses of the bodies it
        owns rows of, lays out its body rows and sizes every buffer, as group_set_body_operators does."""
        _frame_call(self, "group_set_body_frames", n_nodes, node_pos_ref, node_normal_ref, node_weights, ex0, ey0, ez0,
                    A_inv0_list)

    def group_place_bodies(self, centers, orientations):
        """place_bodies on a group member; allocates no device memory"""
        _place_call(self, "group_place_bodies", centers, orientations)

    def group_set_fiber_links(self, body=None, site=None, bending_rigidity=None):
        """set_fiber_links on a group member: body index, nucleation site (n, 3) and bending_rigidity_ of the OWN
        fibers; body=None: none of them is bound."""
        _links_call(self, "group_set_fiber_links", body, site, bending_rigidity)

    def group_apply_system_matvec_device(self, dense, d_x_local: int, eta: float, d_res_local: int, stream: int = 0):
        """the member's rows of A x from its rows of x (distributed.system_rows), asynchronous on `stream`"""
        _check(library().skb_flow_group_apply_system_matvec_device(self._h, _dense_h(dense), _vp(d_x_local), float(eta),
                                                                   _vp(d_res_local), _vp(stream)))

    def group_apply_system_preconditioner_device(self, dense, d_x_local: int, d_y_local: int, stream: int = 0):
        """the member's rows of P^-1 x from its rows of x, asynchronous on `stream`"""
        _check(library().skb_flow_group_apply_system_preconditioner_device(
            self._h, _dense_h(dense), _vp(d_x_local), _vp(d_y_local), _vp(stream)))

    def group_solve_system_device(self, dense_matvec, dense_minv, d_rhs_local: int, eta: float, d_x_local: int,
                                  tol=1e-10, num_blocks=300, max_iters=1000, stream: int = 0):
        """solve_system_device on the member's local rows (set_gmres after group_set_body_operators); every member
        calls it alike.  Returns (info, history), bitwise the same on every member."""
        info = SolveInfo()
        hist = np.full(max(int(max_iters), 0) + 1, np.nan)
        _check(library().skb_flow_group_solve_system_device(self._h, _dense_h(dense_matvec), _dense_h(dense_minv),
                                                            _vp(d_rhs_local), float(eta), float(tol), int(num_blocks),
                                                            int(max_iters), _vp(d_x_local), C.byref(info), _p(hist),
                                                            _vp(stream)))
        return info.as_dict(), hist[:info.iterations + 1]

    def group_build_system_rhs_device(self, length_prev, bending_rigidity, radius, penalty_param, beta_tstep,
                                      minus_clamped, plus_hinged, dt, eta, d_f_external: int, d_body_forces: int,
                                      d_body_torques: int, d_rhs_local: int, v_growth=None, force_scale=None,
                                      stream: int = 0):
        """build_system_rhs_device on a group member: per-fiber arrays of the OWN fibers, f_external of their nodes,
        forces and torques of ALL bodies ((n_bodies, 3) each; 0: none); the member's rows of the RHS."""
        f0, f1 = self._own_fibers()
        p, vg, fs, _, _ = _system_rhs_args(f1 - f0, 0, self.n_bodies,
                                           (length_prev, bending_rigidity, radius, penalty_param, beta_tstep,
                                            minus_clamped, plus_hinged), v_growth, force_scale, None, None)
        _check(library().skb_flow_group_build_system_rhs_device(self._h, _params_ptr(p), _opt_p(vg), _opt_p(fs),
                                                                _vp(d_f_external), _vp(d_body_forces),
                                                                _vp(d_body_torques), float(dt), float(eta),
                                                                _vp(d_rhs_local), _vp(stream)))

    def group_step_device(self, length_prev, bending_rigidity, radius, penalty_param, beta_tstep, minus_clamped,
                          plus_hinged, dt, eta, dense_matvec=None, dense_minv=None, d_f_external: int = 0,
                          d_body_forces: int = 0, d_body_torques: int = 0, fiber_body=None, site_ref=None,
                          v_growth=None, force_scale=None, tol=1e-10, num_blocks=300, max_iters=1000,
                          d_x_local: int = 0, d_tension: int = 0, stream: int = 0):
        """step on a group member (skb_flow_group_step_device): the fibers' parameters, fiber_body and site_ref of the
        OWN fibers, f_external of their nodes and the forces / torques ((n_bodies, 3) each) of ALL bodies as device
        pointers (0: none); d_x_local / d_tension (0: not wanted) receive the member's local rows of the solution and
        its own fibers' tensions.  Every member calls it alike and gets the same info dict; a solution with non-finite
        new positions installs nothing on any member and returns fiber_error NaN.  Not a member: step()."""
        f0, f1 = self._own_fibers()
        p, vg, fs, _, _ = _system_rhs_args(f1 - f0, 0, self.n_bodies,
                                           (length_prev, bending_rigidity, radius, penalty_param, beta_tstep,
                                            minus_clamped, plus_hinged), v_growth, force_scale, None, None)
        fb = None if fiber_body is None else np.ascontiguousarray(fiber_body, dtype=np.int32).reshape(-1)
        if fb is not None and fb.shape[0] != f1 - f0:
            raise ValueError(f"expected {f1 - f0} fiber_body entries (the own fibers), got {fb.shape[0]}")
        sr = None if site_ref is None else _arr(site_ref, 3)
        info = StepInfo()
        rc = library().skb_flow_group_step_device(
            self._h, _dense_h(dense_matvec), _dense_h(dense_minv), _params_ptr(p), _opt_p(vg), _opt_p(fs),
            _vp(d_f_external), _vp(d_body_forces), _vp(d_body_torques),
            None if fb is None else fb.ctypes.data_as(C.POINTER(C.c_int)), _opt_p(sr), float(dt), float(eta),
            float(tol), int(num_blocks), int(max_iters), _vp(d_x_local), _vp(d_tension), C.byref(info), _vp(stream))
        if not (rc == ERR_STATE and np.isnan(info.fiber_error)):
            _check(rc)
        return info.as_dict()


class MultiFlow(_FlowBase):
    """skb_mflow: ONE process driving n GPUs (include/skelly_b200_flow.h) -- same conventions as Flow, complete host
    arrays in and out; fibers / periphery rows / body rows are partitioned over the devices, which exchange strengths
    and partial velocities through peer memory."""
    _destroy = "skb_mflow_destroy"
    _prefix = "skb_mflow_"

    def __init__(self, devices):
        devs = list(range(devices)) if isinstance(devices, int) else [int(d) for d in devices]
        arr = (C.c_int * len(devs))(*devs)
        self._h = C.c_void_p()
        _check(library().skb_mflow_create(arr, len(devs), C.byref(self._h)))
        self.devices = devs
        self.n_fib = self.n_shell = self.n_body = self.n_bodies = 0

    @property
    def n_fibers(self) -> int:
        """the number of fibers of the last set_fibers"""
        return self._n_fibers()

    def _own_fibers(self):
        """every call covers all fibers"""
        return 0, self._n_fibers()

    def _pieces(self):
        """(fiber nodes, shell rows, body rows): every call covers all of them"""
        return self.n_fib, self.n_shell, self.n_body

    def partition(self, member: int):
        f0, f1 = C.c_int(), C.c_int()
        r = [C.c_int64() for _ in range(4)]
        _check(library().skb_mflow_partition(self._h, int(member), C.byref(f0), C.byref(f1), *[C.byref(x) for x in r]))
        return (f0.value, f1.value) + tuple(x.value for x in r)

    def set_fiber_operators(self, A_list, force_list, xs, length_prev, plus_bc_velocity, colmajor=False):
        if colmajor:
            A = np.ascontiguousarray(A_list, dtype=np.float64).reshape(-1)
            F = np.ascontiguousarray(force_list, dtype=np.float64).reshape(-1)
        else:
            A, F = self._colmajor_concat(A_list), self._colmajor_concat(force_list)
        xs = _arr(xs, 3)
        lp = np.ascontiguousarray(length_prev, dtype=np.float64)
        pl = np.ascontiguousarray(plus_bc_velocity, dtype=np.int32)
        assert xs.shape[0] == self.n_fib and lp.shape == pl.shape == (self.n_fibers,)
        _check(library().skb_mflow_set_fiber_operators(self._h, _p(A), _p(F), _p(xs), _p(lp),
                                                       pl.ctypes.data_as(C.POINTER(C.c_int))))

    def set_dense(self, op: int, A):
        A = np.ascontiguousarray(A, dtype=np.float64)
        _check(library().skb_mflow_set_dense(self._h, int(op), _p(A), A.shape[0], A.shape[1]))
        self._has_dense = True

    def apply_matvec(self, x_fibers, x_shell, body_densities, body_forces_torques, eta, fiber_link_conditions=None):
        """Returns (res_fibers (4 N_f,), out_shell (N_s,3), v_bodies (N_b,3)); out_shell is res_shell once
        set_dense(DENSE_STRESSLET_PLUS_COMPLEMENTARY, ...) was called, else v_shell."""
        x = np.ascontiguousarray(x_fibers, dtype=np.float64).reshape(-1)
        assert x.shape[0] == 4 * self.n_fib
        b, c = _arr(x_shell, 3), _arr(body_densities, 3)
        ft = _arr(body_forces_torques, 6)
        vb = None if fiber_link_conditions is None else _arr(fiber_link_conditions, 7)
        res = np.empty(4 * self.n_fib)
        o_s, v_b = np.empty((self.n_shell, 3)), np.empty((self.n_body, 3))
        _check(library().skb_mflow_apply_matvec(self._h, _p(x), _p(b), _p(c), _p(ft), None if vb is None else _p(vb),
                                                float(eta), _p(res), _p(o_s), _p(v_b)))
        return res, o_s, v_b

    def periphery_interaction(self):
        """Flow.periphery_interaction over the devices: the complete arrays of all fibers"""
        return _interaction_call(self, self.n_fib, self.n_fibers)

    def apply_system_matvec(self, x, eta):
        """System::apply_matvec on the whole solution vector x over the devices: returns res = A x.  The periphery's
        operator is set_dense(DENSE_STRESSLET_PLUS_COMPLEMENTARY, ...)."""
        x = np.ascontiguousarray(x, dtype=np.float64).reshape(-1)
        assert x.shape[0] == self.solution_size()
        res = np.empty_like(x)
        _check(library().skb_mflow_apply_system_matvec(self._h, _p(x), float(eta), _p(res)))
        return res

    def apply_system_preconditioner(self, x):
        """System::apply_preconditioner on the whole solution vector x over the devices: returns y = P^-1 x.  The
        periphery's operator is set_dense(DENSE_M_INV, ...)."""
        x = np.ascontiguousarray(x, dtype=np.float64).reshape(-1)
        assert x.shape[0] == self.solution_size()
        y = np.empty_like(x)
        _check(library().skb_mflow_apply_system_preconditioner(self._h, _p(x), _p(y)))
        return y

    def solve_system(self, rhs, eta, tol=1e-10, num_blocks=300, max_iters=1000):
        """Flow.solve_system over the devices, every member solving its own rows: returns (x, info, history)."""
        b = np.ascontiguousarray(rhs, dtype=np.float64).reshape(-1)
        assert b.shape[0] == self.solution_size()
        x = np.empty_like(b)
        info = SolveInfo()
        hist = np.full(max(int(max_iters), 0) + 1, np.nan)
        _check(library().skb_mflow_solve_system(self._h, _p(b), float(eta), float(tol), int(num_blocks),
                                                int(max_iters), _p(x), C.byref(info), _p(hist)))
        return x, info.as_dict(), hist[:info.iterations + 1]


DENSE_STRESSLET_PLUS_COMPLEMENTARY = 0
DENSE_M_INV = 1


class Dense(_Handle):
    """The periphery's dense operators on the GPU (include/skelly_b200_dense.h): Periphery::matvec and
    Periphery::apply_preconditioner (periphery.cpp:21-47) as row-partitioned GEMVs."""
    _destroy = "skb_dense_destroy"

    def __init__(self, n_gpus: int = 1, device_ids=None):
        self._h = C.c_void_p()
        if device_ids is not None:
            arr = (C.c_int * len(device_ids))(*[int(d) for d in device_ids])
            _check(library().skb_dense_create_on(arr, len(device_ids), C.byref(self._h)))
        else:
            _check(library().skb_dense_create(int(n_gpus), C.byref(self._h)))
        self.shape = {}

    def set_matrix(self, op: int, A):
        A = np.ascontiguousarray(A, dtype=np.float64)
        assert A.ndim == 2
        _check(library().skb_dense_set_matrix(self._h, int(op), _p(A), A.shape[0], A.shape[1]))
        self.shape[int(op)] = A.shape

    def apply(self, op: int, x, v_add=None):
        rows, cols = self.shape[int(op)]
        x = np.ascontiguousarray(x, dtype=np.float64).reshape(-1)
        assert x.shape[0] == cols
        y = np.empty(rows)
        v = None
        if v_add is not None:
            v = np.ascontiguousarray(v_add, dtype=np.float64).reshape(-1)
            assert v.shape[0] == rows
        _check(library().skb_dense_apply(self._h, int(op), _p(x), _p(v) if v is not None else None, _p(y)))
        return y

    def apply_device(self, op: int, d_x: int, d_v_add: int, d_y: int, stream: int = 0):
        """Single-device handle, operands already on its device (addresses as ints, 0 = NULL v_add); asynchronous."""
        _check(library().skb_dense_apply_device(self._h, int(op), C.c_void_p(d_x), _vp(d_v_add), C.c_void_p(d_y),
                                                _vp(stream)))

    def apply_background_device(self, op: int, d_x: int, d_y: int, stream: int = 0):
        """y = A x with the background row streamer (one small CTA per SM, TMA-fed): the form that can share the SMs
        with the pair kernels.  Single-device handle, device addresses as ints; asynchronous."""
        _check(library().skb_dense_apply_background_device(self._h, int(op), C.c_void_p(d_x), C.c_void_p(d_y),
                                                           _vp(stream)))

    def stats(self) -> dict:
        s = DenseStats()
        _check(library().skb_dense_last_stats(self._h, C.byref(s)))
        return {k: getattr(s, k) for k, _ in DenseStats._fields_}


def plan_query(kind, n_trg, n_src, num_sms=132, occupancy=(8, 6, 4, 2), force_T=0, force_S=0) -> dict:
    """Host-side launch planner of the plain pair kernel (no GPU needed)."""
    occ = (C.c_int * 4)(*occupancy)
    T, S, per, gx = C.c_int(), C.c_int(), C.c_int(), C.c_int()
    _check(library().skb_plan_query(int(kind), int(n_trg), int(n_src), int(num_sms), occ, int(force_T), int(force_S),
                                    C.byref(T), C.byref(S), C.byref(per), C.byref(gx)))
    return {"T": T.value, "n_splits": S.value, "tiles_per_split": per.value, "grid_x": gx.value}


def partition_query(fiber_n_nodes, n_shell, n_body, n_members, member):
    """Rows of [fibers | periphery | bodies] member `member` of `n_members` owns (the partition of skb_mflow; no GPU
    needed): (fiber_begin, fiber_end, shell_begin, shell_end, body_begin, body_end)."""
    nn = np.ascontiguousarray(fiber_n_nodes, dtype=np.int32)
    out = (C.c_int64 * 6)()
    _check(library().skb_partition_query(nn.ctypes.data_as(C.POINTER(C.c_int)), int(nn.shape[0]), int(n_shell),
                                         int(n_body), int(n_members), int(member), out))
    return tuple(int(v) for v in out)


def group_body_pieces(body_n_nodes, body_begin, body_end):
    """The places of a group member's own body rows [body_begin, body_end) (no GPU needed): an (n, 3) int64 array of
    runs (offset in the local vector's body part, offset in the whole vector's body part, length), ascending."""
    nn = np.ascontiguousarray(body_n_nodes, dtype=np.int32)
    out = np.zeros((8, 3), dtype=np.int64)
    k = C.c_int(0)
    _check(library().skb_group_body_pieces(nn.ctypes.data_as(C.POINTER(C.c_int)), int(nn.shape[0]), int(body_begin),
                                           int(body_end), out.ctypes.data_as(C.POINTER(C.c_int64)), out.shape[0],
                                           C.byref(k)))
    return out[:k.value].copy()


def sym_groups_per_block() -> int:
    return int(library().skb_sym_groups_per_block())


def sym_plan_query(n_blocks, part=0, n_parts=1, num_sms=132):
    """Host-side work list of the symmetric kernel (no GPU needed): list of (I, g0, g1, slot), row_begin; block I
    meets the 32-node groups [g0, g1) (sym_groups_per_block() groups per block)."""
    n = C.c_int()
    _check(library().skb_sym_plan_query(int(n_blocks), int(part), int(n_parts), int(num_sms), 0, None, C.byref(n),
                                        None))
    items = (C.c_int * (4 * max(n.value, 1)))()
    rb = (C.c_int * (n_blocks + 1))()
    _check(library().skb_sym_plan_query(int(n_blocks), int(part), int(n_parts), int(num_sms), n.value, items,
                                        C.byref(n), rb))
    return [tuple(items[4 * i:4 * i + 4]) for i in range(n.value)], list(rb)


def _state_args(flow, params, body_kind, body_radii):
    p = fiber_params(flow._n_fibers(), *params)
    kind = np.ascontiguousarray(np.zeros(0) if body_kind is None else body_kind, dtype=np.int32).reshape(-1)
    radii = _arr(np.zeros((0, 3)) if body_radii is None else body_radii, 3)
    if kind.shape != (flow.n_bodies,) or radii.shape[0] != flow.n_bodies:
        raise ValueError(f"expected {flow.n_bodies} body kinds and radii, got {kind.shape} and {radii.shape}")
    return p, kind, radii


# The listener's frame of a step (skb_flow_set_listener_state), on a Flow only: the listener is single-device, and an
# skb_mflow handle must never reach an skb_flow_ call.  Module functions taking the Flow rather than Flow methods:
# Flow's public methods are pinned one by one by tests/test_capi_binding_cpu.py; these are marshalled and checked
# the same way in tests/test_listener_state_binding_cpu.py and tests/test_listener_gradient_cpu.py.
def _listener_flow(flow):
    if not isinstance(flow, Flow):
        raise TypeError(f"the listener's frame needs a capi.Flow (one device), got {type(flow).__name__}")


def set_listener_state(flow, length_prev, bending_rigidity, radius, penalty_param, beta_tstep, minus_clamped,
                       plus_hinged, dt, eta, tension, x, body_kind=None, body_radii=None, periphery_interaction=False):
    """The listener's frame of `flow` (a Flow) from its installed geometry and a step's solution, as the reference's
    listener unpacks a trajectory frame: the fiber forces of [positions; tension] with the operators built at the
    installed positions (the fiber parameters of Flow.build_fiber_operators; the call leaves them resident without their
    inverse, so the fiber preconditioner refuses until the next build), plus the
    periphery repulsion when periphery_interaction; the bodies' link forces and torques (no external ones); the shell
    and body densities and each body's [U, omega] from x (the step's whole solution vector).  tension (N_f,);
    body_kind / body_radii as Flow.set_listener_frame.  Afterwards flow.velocity_field, .streamlines and .vortexlines
    answer on that frame."""
    _listener_flow(flow)
    p, kind, radii = _state_args(flow, (length_prev, bending_rigidity, radius, penalty_param, beta_tstep,
                                        minus_clamped, plus_hinged), body_kind, body_radii)
    t = np.ascontiguousarray(tension, dtype=np.float64).reshape(-1)
    xs = np.ascontiguousarray(x, dtype=np.float64).reshape(-1)
    if t.shape != (flow.n_fib,) or xs.shape != (flow.solution_size(),):
        raise ValueError(f"expected {flow.n_fib} tensions and a solution of {flow.solution_size()}, got {t.shape} "
                         f"and {xs.shape}")
    _check(library().skb_flow_set_listener_state(flow._h, _params_ptr(p), float(dt), float(eta), _p(t), _p(xs),
                                                 kind.ctypes.data_as(C.POINTER(C.c_int32)), _p(radii),
                                                 int(bool(periphery_interaction))))


def set_listener_state_device(flow, length_prev, bending_rigidity, radius, penalty_param, beta_tstep, minus_clamped,
                              plus_hinged, dt, eta, d_tension: int, d_x: int, body_kind=None, body_radii=None,
                              periphery_interaction=False, stream: int = 0):
    """set_listener_state from device addresses (ints, e.g. torch.Tensor.data_ptr()) on the flow's device, after the
    caller's work on `stream`; the solution never passes through the host."""
    _listener_flow(flow)
    p, kind, radii = _state_args(flow, (length_prev, bending_rigidity, radius, penalty_param, beta_tstep,
                                        minus_clamped, plus_hinged), body_kind, body_radii)
    _check(library().skb_flow_set_listener_state_device(flow._h, _params_ptr(p), float(dt), float(eta), _vp(d_tension),
                                                        _vp(d_x), kind.ctypes.data_as(C.POINTER(C.c_int32)),
                                                        _p(radii), int(bool(periphery_interaction)),
                                                        C.c_void_p(stream)))


def listener_gradient(flow, r):
    """The velocity gradient and the pressure of `flow`'s listener frame (a Flow) at the points r (n, 3), on the
    device: grad (n, 3, 3) with grad[t, i, j] = d u_i / d x_j, and pressure (n,).  The frame, staleness and refusals
    are those of Flow.velocity_field; inside a body the gradient is the rigid motion's and the pressure NaN.  The
    vorticity is omega_i = eps_ijk d_j u_k (omega = (G[2,1] - G[1,2], G[0,2] - G[2,0], G[1,0] - G[0,1])), the strain
    rate E = (G + G^T) / 2."""
    _listener_flow(flow)
    r = _arr(r, 3)
    grad, pressure = np.empty((r.shape[0], 3, 3)), np.empty(r.shape[0])
    _check(library().skb_flow_listener_gradient(flow._h, _p(r), r.shape[0], _p(grad), _p(pressure)))
    return grad, pressure
