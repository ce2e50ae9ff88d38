"""Host-side mirror of the reference's solver interface for the batched H100 path.

Class and option names follow momentum (``SolverOptions`` / ``GaussNewtonSolverOptions`` —
solver/solver.h:19-34, solver/gauss_newton_solver.h:17-59; ``SkeletonSolverFunction`` —
character_solver/skeleton_solver_function.h:21-95; ``GaussNewtonSolver`` —
solver/gauss_newton_solver.h:67-137) with a leading batch dimension on parameters and results.
Everything here is a thin ctypes veneer over the C-ABI in include/momentum_b200.h; the compute is
in momentum_b200/lib/libmomentum_b200.so (hand-written sm_90a kernels). There is no CPU fallback:
if the library or an H100 (sm_90) is missing, construction raises.
"""
from __future__ import annotations

import ctypes as C
import os
from dataclasses import dataclass
from typing import List, Optional, Sequence

import numpy as np

from . import character as mc

_HERE = os.path.dirname(os.path.abspath(__file__))
DEFAULT_LIB = os.path.join(_HERE, "lib", "libmomentum_b200.so")

SIZE_MAX = 2 ** 64 - 1

JTJ_AUTO, JTJ_FP32_SIMT, JTJ_TF32X3, JTJ_TF32, JTJ_SPARSE_TILES = 0, 1, 2, 3, 4
INSTANCE_OK, INSTANCE_CHOLESKY_BREAKDOWN, INSTANCE_NON_FINITE = 0, 1, 2
CHOLESKY_AUTO, CHOLESKY_DENSE_EIGEN, CHOLESKY_TILES_DENSE, CHOLESKY_TILES_SPARSE = 0, 1, 2, 3
FUSED_AUTO, FUSED_OFF, FUSED_PERSISTENT, FUSED_GRAM_CHOLESKY = 0, 1, 2, 3
FUSED_ON = FUSED_PERSISTENT
LINEAR_SOLVER_CHOLESKY, LINEAR_SOLVER_QR, LINEAR_SOLVER_TRUST_REGION_QR = 0, 1, 2


class MomentumB200Error(RuntimeError):
    """std::runtime_error of the reference's MT_CHECK/MT_THROW (common/exception.h:31)."""


class _Limit(C.Structure):
    _fields_ = [("type", C.c_int32), ("weight", C.c_float), ("i", C.c_int32 * 4), ("f", C.c_float * 27)]


class _Options(C.Structure):
    _fields_ = [("min_iterations", C.c_uint64), ("max_iterations", C.c_uint64), ("threshold", C.c_float), ("verbose", C.c_int32),
                ("regularization", C.c_float), ("do_line_search", C.c_int32), ("use_block_jtj", C.c_int32),
                ("target_rows_per_chunk", C.c_uint64), ("subset_line_search", C.c_int32), ("jtj_mode", C.c_int32),
                ("store_error_history", C.c_int32), ("cholesky_mode", C.c_int32), ("fused_mode", C.c_int32), ("linear_solver", C.c_int32),
                ("trust_region_radius", C.c_float)]


_fp = C.POINTER(C.c_float)
_ip = C.POINTER(C.c_int32)
_dp = C.POINTER(C.c_double)
_up = C.POINTER(C.c_uint64)

# every symbol include/momentum_b200.h declares (checked by tests/test_cabi_symbols.py)
CABI_SYMBOLS = [
    "mb2_last_error", "mb2_device_count", "mb2_default_gauss_newton_options", "mb2_character_create", "mb2_character_set_parameter_limits",
    "mb2_character_destroy", "mb2_solver_function_create", "mb2_solver_function_destroy", "mb2_solver_function_num_parameters",
    "mb2_solver_function_actual_parameters", "mb2_solver_function_batch", "mb2_solver_function_jacobian_rows",
    "mb2_solver_function_jacobian_stride", "mb2_add_position_error_function", "mb2_add_position_error_function_instanced", "mb2_add_orientation_error_function",
    "mb2_add_plane_error_function", "mb2_add_model_parameters_error_function",
    "mb2_add_state_error_function", "mb2_add_limit_error_function", "mb2_set_error_function_weight", "mb2_set_targets",
    "mb2_set_targets_device", "mb2_set_constraint_weights", "mb2_solver_function_set_enabled_parameters", "mb2_solver_function_get_error",
    "mb2_solver_function_get_jacobian", "mb2_solver_function_get_jtjr", "mb2_solver_function_get_skeleton_state", "mb2_solver_create",
    "mb2_solver_destroy", "mb2_solver_set_options", "mb2_solver_set_enabled_parameters", "mb2_solver_solve", "mb2_solver_solve_device",
    "mb2_solver_get_results", "mb2_solver_get_error_history", "mb2_solver_get_counters", "mb2_solver_set_profiling",
    "mb2_solver_get_phase_times", "mb2_solver_get_plan_stats", "mb2_solver_get_fused_profile", "mb2_solver_solve_async", "mb2_solver_wait",
    "mb2_set_constraint_weights_device", "mb2_solver_function_get_jacobian_device",
    "mb2_mixed_batch_last_error", "mb2_mixed_batch_create", "mb2_mixed_batch_destroy", "mb2_mixed_batch_add_rig", "mb2_mixed_batch_use_limits",
    "mb2_mixed_batch_add_instance", "mb2_mixed_batch_set_parameters", "mb2_mixed_batch_solve", "mb2_mixed_batch_get_result", "mb2_mixed_batch_get_results",
    "mb2_mixed_batch_stats", "mb2_mixed_batch_bucket_info",
    "mb2_character_clone", "mb2_solver_function_clone", "mb2_character_device", "mb2_solver_function_character", "mb2_solver_function_num_error_functions",
    "mb2_solver_function_target_size", "mb2_sharded_last_error", "mb2_sharded_solver_create", "mb2_sharded_solver_destroy", "mb2_sharded_solver_num_shards",
    "mb2_sharded_solver_shard_info", "mb2_sharded_solver_set_options", "mb2_sharded_solver_set_targets", "mb2_sharded_solver_solve", "mb2_sharded_solver_get_aggregate",
    "mb2_character_skeleton_state_device", "mb2_character_skeleton_state_backward_device",
    "mb2_add_orientation_error_function_instanced", "mb2_solver_function_input_gradients_device",
    "mb2_solver_function_implicit_direction_device", "mb2_solver_function_get_sweep_launch", "mb2_solver_get_solve_path",
    "mb2_character_set_skinning", "mb2_character_num_vertices", "mb2_character_skin_points_device", "mb2_character_skin_points_backward_device",
]

_libs = {}


def load_library(path: Optional[str] = None):
    path = path or DEFAULT_LIB
    if path in _libs:
        return _libs[path]
    if not os.path.exists(path):
        raise MomentumB200Error(f"{path} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                                "(momentum_b200 has no CPU fallback)")
    L = C.CDLL(path)
    L.mb2_last_error.restype = C.c_char_p
    vp = C.c_void_p
    L.mb2_character_create.argtypes = [C.c_int, C.c_int32, _ip, _fp, _fp, C.c_int32, _ip, _ip, _fp, _fp, C.POINTER(vp)]
    L.mb2_character_set_parameter_limits.argtypes = [vp, C.c_int32, C.POINTER(_Limit)]
    L.mb2_character_destroy.argtypes = [vp]
    L.mb2_solver_function_create.argtypes = [vp, C.c_int32, C.POINTER(vp)]
    L.mb2_solver_function_destroy.argtypes = [vp]
    for name in ("num_parameters", "actual_parameters", "batch", "jacobian_rows", "jacobian_stride"):
        getattr(L, f"mb2_solver_function_{name}").argtypes = [vp]
    L.mb2_add_position_error_function.argtypes = [vp, C.c_float, C.c_float, C.c_float, C.c_int32, _ip, _fp, _fp, _ip]
    if hasattr(L, "mb2_add_position_error_function_instanced"):
        L.mb2_add_position_error_function_instanced.argtypes = [vp, C.c_float, C.c_float, C.c_float, C.c_int32, _ip, _fp, _ip]
    L.mb2_add_orientation_error_function.argtypes = [vp, C.c_float, C.c_float, C.c_float, C.c_int32, C.c_int32, _ip, _fp, _fp, _ip]
    L.mb2_add_state_error_function.argtypes = [vp, C.c_float, C.c_int32, C.c_float, C.c_float, _fp, _fp, _ip]
    L.mb2_add_limit_error_function.argtypes = [vp, C.c_float, C.c_float, C.c_float, _ip]
    if hasattr(L, "mb2_add_plane_error_function"):
        L.mb2_add_plane_error_function.argtypes = [vp, C.c_float, C.c_float, C.c_float, C.c_int32, C.c_int32, _ip, _fp, _fp, _ip]
        L.mb2_add_model_parameters_error_function.argtypes = [vp, C.c_float, _fp, _ip]
    L.mb2_set_error_function_weight.argtypes = [vp, C.c_int32, C.c_float]
    L.mb2_set_targets.argtypes = [vp, C.c_int32, _fp]
    if hasattr(L, "mb2_set_targets_device"):
        L.mb2_set_targets_device.argtypes = [vp, C.c_int32, vp, vp]
    L.mb2_set_constraint_weights.argtypes = [vp, C.c_int32, _fp, C.c_int32]
    L.mb2_solver_function_set_enabled_parameters.argtypes = [vp, _up]
    L.mb2_solver_function_get_error.argtypes = [vp, _fp, _dp]
    L.mb2_solver_function_get_jacobian.argtypes = [vp, _fp, _fp, _fp, _dp, _ip]
    L.mb2_solver_function_get_jtjr.argtypes = [vp, _fp, C.c_int32, _fp, _fp, _dp]
    L.mb2_solver_function_get_skeleton_state.argtypes = [vp, _fp, _fp]
    L.mb2_solver_create.argtypes = [vp, C.POINTER(_Options), C.POINTER(vp)]
    L.mb2_solver_destroy.argtypes = [vp]
    L.mb2_solver_set_options.argtypes = [vp, C.POINTER(_Options)]
    L.mb2_solver_set_enabled_parameters.argtypes = [vp, _up]
    L.mb2_solver_solve.argtypes = [vp, vp, _dp, _ip, _ip]
    if hasattr(L, "mb2_solver_solve_device"):
        L.mb2_solver_solve_device.argtypes = [vp, vp, vp]
        L.mb2_solver_get_results.argtypes = [vp, _dp, _ip, _ip]
        L.mb2_solver_set_profiling.argtypes = [vp, C.c_int32]
        L.mb2_solver_get_phase_times.argtypes = [vp, _dp, _up]
    L.mb2_solver_get_error_history.argtypes = [vp, _dp]
    L.mb2_solver_get_counters.argtypes = [vp, _up, _up]
    if hasattr(L, "mb2_solver_get_plan_stats"):
        L.mb2_solver_get_plan_stats.argtypes = [vp, C.POINTER(C.c_int64)]
    if hasattr(L, "mb2_solver_get_fused_profile"):
        L.mb2_solver_get_fused_profile.argtypes = [vp, _ip, _ip, _dp, _up]
    L.mb2_default_gauss_newton_options.argtypes = [C.POINTER(_Options)]
    if hasattr(L, "mb2_set_constraint_weights_device"):
        L.mb2_set_constraint_weights_device.argtypes = [vp, C.c_int32, vp, vp]
        L.mb2_solver_function_get_jacobian_device.argtypes = [vp, vp, C.POINTER(vp), _ip, vp]
    if hasattr(L, "mb2_mixed_batch_create"):
        L.mb2_solver_solve_async.argtypes = [vp, vp]
        L.mb2_solver_wait.argtypes = [vp, _dp, _ip, _ip]
        L.mb2_mixed_batch_last_error.restype = C.c_char_p
        L.mb2_mixed_batch_create.argtypes = [C.c_int, C.c_int32, C.POINTER(vp)]
        L.mb2_mixed_batch_destroy.argtypes = [vp]
        L.mb2_mixed_batch_add_rig.argtypes = [vp, vp, C.c_int32, _ip]
        L.mb2_mixed_batch_use_limits.argtypes = [vp, C.c_int32, C.c_float]
        L.mb2_mixed_batch_add_instance.argtypes = [vp, C.c_int32, C.c_int32, _ip, _fp, _fp, _fp, _fp, _ip]
        L.mb2_mixed_batch_set_parameters.argtypes = [vp, C.c_int32, _fp]
        L.mb2_mixed_batch_solve.argtypes = [vp, C.POINTER(_Options)]
        L.mb2_mixed_batch_get_result.argtypes = [vp, C.c_int32, _fp, _dp, _ip, _ip]
        L.mb2_mixed_batch_get_results.argtypes = [vp, _fp, C.POINTER(C.c_int64), _dp, _ip, _ip]
        L.mb2_mixed_batch_stats.argtypes = [vp, C.POINTER(C.c_int64)]
        L.mb2_mixed_batch_bucket_info.argtypes = [vp, C.c_int32, C.POINTER(C.c_int64)]
    if hasattr(L, "mb2_sharded_solver_create"):
        L.mb2_sharded_last_error.restype = C.c_char_p
        L.mb2_character_clone.argtypes = [vp, C.c_int, C.POINTER(vp)]
        L.mb2_solver_function_clone.argtypes = [vp, vp, C.c_int32, C.POINTER(vp)]
        L.mb2_character_device.argtypes = [vp]
        L.mb2_solver_function_character.argtypes = [vp]
        L.mb2_solver_function_character.restype = vp
        L.mb2_solver_function_num_error_functions.argtypes = [vp]
        L.mb2_solver_function_target_size.argtypes = [vp, C.c_int32]
        L.mb2_sharded_solver_create.argtypes = [vp, C.c_int32, C.c_int32, _ip, C.POINTER(_Options), C.POINTER(vp)]
        L.mb2_sharded_solver_destroy.argtypes = [vp]
        L.mb2_sharded_solver_num_shards.argtypes = [vp]
        L.mb2_sharded_solver_shard_info.argtypes = [vp, C.c_int32, _ip]
        L.mb2_sharded_solver_set_options.argtypes = [vp, C.POINTER(_Options)]
        L.mb2_sharded_solver_set_targets.argtypes = [vp, C.c_int32, _fp]
        L.mb2_sharded_solver_solve.argtypes = [vp, vp, _dp, _ip, _ip]
        L.mb2_sharded_solver_get_aggregate.argtypes = [vp, _dp]
    if hasattr(L, "mb2_character_skeleton_state_device"):
        L.mb2_character_skeleton_state_device.argtypes = [vp, C.c_int32, vp, vp, vp]
        L.mb2_character_skeleton_state_backward_device.argtypes = [vp, C.c_int32, vp, vp, vp, vp]
    if hasattr(L, "mb2_add_orientation_error_function_instanced"):
        L.mb2_add_orientation_error_function_instanced.argtypes = [vp, C.c_float, C.c_float, C.c_float, C.c_int32, C.c_int32, _ip, _fp, _ip]
    if hasattr(L, "mb2_solver_function_input_gradients_device"):
        L.mb2_solver_function_input_gradients_device.argtypes = [vp, C.c_int32, vp, vp, vp, vp, vp, vp]
    if hasattr(L, "mb2_solver_function_implicit_direction_device"):
        L.mb2_solver_function_implicit_direction_device.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp]
    if hasattr(L, "mb2_solver_function_get_sweep_launch"):
        L.mb2_solver_function_get_sweep_launch.argtypes = [vp, C.c_int32, C.POINTER(C.c_int64)]
    if hasattr(L, "mb2_solver_get_solve_path"):
        L.mb2_solver_get_solve_path.argtypes = [vp, C.POINTER(C.c_int64)]
    if hasattr(L, "mb2_character_set_skinning"):
        L.mb2_character_set_skinning.argtypes = [vp, C.c_int32, _fp, _ip, _fp, _fp]
        L.mb2_character_num_vertices.argtypes = [vp]
        L.mb2_character_skin_points_device.argtypes = [vp, C.c_int32, vp, vp, C.c_int32, vp, vp]
        L.mb2_character_skin_points_backward_device.argtypes = [vp, C.c_int32, vp, vp, C.c_int32, vp, vp, vp, vp]
    _libs[path] = L
    return L


def _f32(a):
    a = np.ascontiguousarray(a, np.float32)
    return a, a.ctypes.data_as(_fp)


def _i32(a):
    a = np.ascontiguousarray(a, np.int32)
    return a, a.ctypes.data_as(_ip)


def parameter_set_bits(enabled: Sequence[bool]) -> np.ndarray:
    """ParameterSet (std::bitset<2048>, math/types.h:426-429) as 32 uint64 words."""
    bits = np.zeros(32, np.uint64)
    for i, e in enumerate(enabled):
        if e:
            bits[i >> 6] |= np.uint64(1) << np.uint64(i & 63)
    return bits


@dataclass
class SolverOptions:
    """solver/solver.h:19-34"""
    min_iterations: int = 1
    max_iterations: int = 2
    threshold: float = 1.0
    verbose: bool = False


@dataclass
class GaussNewtonSolverOptions(SolverOptions):
    """solver/gauss_newton_solver.h:17-59 (+ device extensions ``jtj_mode``, ``subset_line_search``)."""
    regularization: float = 0.05
    do_line_search: bool = False
    use_block_jtj: bool = False
    target_rows_per_chunk: int = SIZE_MAX
    subset_line_search: bool = False
    jtj_mode: int = JTJ_AUTO
    store_error_history: bool = False
    cholesky_mode: int = 0  # CHOLESKY_AUTO
    fused_mode: int = 0     # FUSED_AUTO: Gram + Cholesky in one launch per iteration when the plan fits (momentum_b200.h mb2_fused_mode)
    linear_solver: int = 0  # LINEAR_SOLVER_CHOLESKY; LINEAR_SOLVER_QR = GaussNewtonSolverQRT's Householder step; LINEAR_SOLVER_TRUST_REGION_QR = TrustRegionQRT
    trust_region_radius: float = 1.0  # TrustRegionQROptions::trustRegionRadius_

    def _c(self) -> _Options:
        return _Options(self.min_iterations, self.max_iterations, self.threshold, int(self.verbose), self.regularization,
                        int(self.do_line_search), int(self.use_block_jtj), self.target_rows_per_chunk, int(self.subset_line_search),
                        int(self.jtj_mode), int(self.store_error_history), int(self.cholesky_mode), int(self.fused_mode), int(self.linear_solver),
                        float(self.trust_region_radius))


class _Base:
    def _check(self, rc):
        if rc != 0:
            raise MomentumB200Error(self._L.mb2_last_error().decode())


class DeviceCharacter(_Base):
    """Character (Skeleton + ParameterTransform + ParameterLimits) resident on one GPU."""

    def __init__(self, character: mc.Character, device: int = 0, lib_path: Optional[str] = None):
        self._L = load_library(lib_path)
        self.character = character
        self.device = device
        self._h = C.c_void_p()
        pa, pp = _i32(character.parents)
        of, op = _f32(character.offsets)
        pr, prp = _f32(character.prerot)
        ou, oup = _i32(character.pt_outer)
        inn, inp = _i32(character.pt_inner)
        va, vap = _f32(character.pt_vals)
        po, pop = _f32(character.pt_offsets)
        self._check(self._L.mb2_character_create(device, character.num_joints, pp, op, prp, character.num_params, oup, inp, vap, pop,
                                                 C.byref(self._h)))
        if character.limits:
            arr = (_Limit * len(character.limits))()
            for k, lim in enumerate(character.limits):
                ii, ff = lim.packed()
                arr[k].type = int(lim.type)
                arr[k].weight = float(lim.weight)
                for j in range(4):
                    arr[k].i[j] = int(ii[j])
                for j in range(27):
                    arr[k].f[j] = float(ff[j])
            self._check(self._L.mb2_character_set_parameter_limits(self._h, len(character.limits), arr))
        self.skinning = None
        if character.skinning is not None:
            self.set_skinning(character.skinning)

    def set_skinning(self, skinning: mc.Skinning):
        """Uploads ``skinning`` (replacing any earlier one); ``self.skinning`` is the object uploaded."""
        V = skinning.num_vertices
        rv, rvp = _f32(np.asarray(skinning.rest_vertices).reshape(V, 3))
        si, sip = _i32(np.asarray(skinning.skin_index).reshape(V, mc.MAX_SKIN_JOINTS))
        sw, swp = _f32(np.asarray(skinning.skin_weight).reshape(V, mc.MAX_SKIN_JOINTS))
        ib, ibp = _f32(np.asarray(skinning.inverse_bind_pose).reshape(self.character.num_joints, 12))
        self._check(self._L.mb2_character_set_skinning(self._h, V, rvp, sip, swp, ibp))
        self.skinning = skinning

    @property
    def num_vertices(self) -> int:
        return int(self._L.mb2_character_num_vertices(self._h))

    def skin_points_device(self, batch: int, state_device_ptr: int, rest_device_ptr: int, rest_batched: bool, points_device_ptr: int, stream: int = 0):
        """Skinned points [B][V][3] of skeleton states [B][J][8]; rest points: 0 = the rest mesh, else [V][3] (shared) or [B][V][3]
        (``rest_batched``). float32 device memory on this character's device, enqueued on ``stream``."""
        self._check(self._L.mb2_character_skin_points_device(self._h, int(batch), C.c_void_p(state_device_ptr), C.c_void_p(rest_device_ptr or None),
                                                             int(bool(rest_batched)), C.c_void_p(points_device_ptr), C.c_void_p(stream)))

    def skin_points_backward_device(self, batch: int, state_device_ptr: int, rest_device_ptr: int, rest_batched: bool, grad_points_device_ptr: int,
                                    grad_state_device_ptr: int, grad_rest_device_ptr: int, stream: int = 0):
        """dLoss/d skeleton state [B][J][8] and dLoss/d rest points (the rest-point layout; the batch sum when shared) from dLoss/d points
        [B][V][3]. A 0 output pointer is skipped."""
        self._check(self._L.mb2_character_skin_points_backward_device(
            self._h, int(batch), C.c_void_p(state_device_ptr), C.c_void_p(rest_device_ptr or None), int(bool(rest_batched)),
            C.c_void_p(grad_points_device_ptr), C.c_void_p(grad_state_device_ptr or None), C.c_void_p(grad_rest_device_ptr or None), C.c_void_p(stream)))

    def skeleton_state_device(self, batch: int, params_device_ptr: int, state_device_ptr: int, stream: int = 0):
        """Skeleton state [B][J][8] (t, q xyzw, s) of model parameters [B][n], float32 device memory on this character's device, enqueued
        on ``stream`` (0: the legacy default stream)."""
        self._check(self._L.mb2_character_skeleton_state_device(self._h, int(batch), C.c_void_p(params_device_ptr), C.c_void_p(state_device_ptr),
                                                                C.c_void_p(stream)))

    def skeleton_state_backward_device(self, batch: int, params_device_ptr: int, grad_state_device_ptr: int, grad_params_device_ptr: int, stream: int = 0):
        """dLoss/d model parameters [B][n] (overwritten) from dLoss/d skeleton state [B][J][8], float32 device memory, on ``stream``."""
        self._check(self._L.mb2_character_skeleton_state_backward_device(self._h, int(batch), C.c_void_p(params_device_ptr), C.c_void_p(grad_state_device_ptr),
                                                                         C.c_void_p(grad_params_device_ptr), C.c_void_p(stream)))

    def __del__(self):
        if getattr(self, "_h", None):
            self._L.mb2_character_destroy(self._h)
            self._h = None


class SkeletonSolverFunction(_Base):
    """Batch of B ``SkeletonSolverFunctionT<float>`` sharing one character and constraint topology."""

    def __init__(self, character, batch: int, error_functions: Sequence = (), device: int = 0, lib_path: Optional[str] = None):
        self._L = load_library(lib_path)
        self.dev_character = character if isinstance(character, DeviceCharacter) else DeviceCharacter(character, device, lib_path)
        self.character = self.dev_character.character
        self.batch = batch
        self._h = C.c_void_p()
        self._check(self._L.mb2_solver_function_create(self.dev_character._h, batch, C.byref(self._h)))
        self.error_functions: List = []
        for ef in error_functions:
            self.add_error_function(ef)

    def __del__(self):
        if getattr(self, "_h", None):
            self._L.mb2_solver_function_destroy(self._h)
            self._h = None

    # addErrorFunction (skeleton_solver_function.cpp:161-169)
    def add_error_function(self, ef) -> int:
        idx = C.c_int32(-1)
        alpha = float(getattr(ef, "loss_alpha", 2.0))
        if ef.kind == mc.KIND_POSITION and getattr(ef, "instance_offsets", None) is not None:
            pa, pp = _i32(ef.parents); w, wp = _f32(ef.weights)
            self._check(self._L.mb2_add_position_error_function_instanced(self._h, ef.weight, alpha, ef.loss_c, len(pa), pp, wp, C.byref(idx)))
        elif ef.kind == mc.KIND_POSITION:
            pa, pp = _i32(ef.parents); of, op = _f32(ef.offsets); w, wp = _f32(ef.weights)
            self._check(self._L.mb2_add_position_error_function(self._h, ef.weight, alpha, ef.loss_c, len(pa), pp, op, wp, C.byref(idx)))
        elif ef.kind in (mc.KIND_ORIENTATION, mc.KIND_ORIENTATION_ROTDIFF) and getattr(ef, "instance_offsets", None) is not None:
            pa, pp = _i32(ef.parents); w, wp = _f32(ef.weights)
            self._check(self._L.mb2_add_orientation_error_function_instanced(self._h, ef.weight, alpha, ef.loss_c, int(ef.rot_diff), len(pa), pp, wp,
                                                                             C.byref(idx)))
        elif ef.kind in (mc.KIND_ORIENTATION, mc.KIND_ORIENTATION_ROTDIFF):
            pa, pp = _i32(ef.parents); of, op = _f32(ef.offsets); w, wp = _f32(ef.weights)
            self._check(self._L.mb2_add_orientation_error_function(self._h, ef.weight, alpha, ef.loss_c, int(ef.rot_diff), len(pa), pp, op, wp,
                                                                   C.byref(idx)))
        elif ef.kind == mc.KIND_STATE:
            pw, pwp = _f32(ef.pos_weights); rw, rwp = _f32(ef.rot_weights)
            self._check(self._L.mb2_add_state_error_function(self._h, ef.weight, int(ef.rotation_error_type), ef.pos_wgt, ef.rot_wgt, pwp, rwp,
                                                             C.byref(idx)))
        elif ef.kind == mc.KIND_LIMIT:
            self._check(self._L.mb2_add_limit_error_function(self._h, ef.weight, alpha, ef.loss_c, C.byref(idx)))
        elif ef.kind == mc.KIND_PLANE:
            pa, pp = _i32(ef.parents); of, op = _f32(ef.offsets); w, wp = _f32(ef.weights)
            self._check(self._L.mb2_add_plane_error_function(self._h, ef.weight, alpha, ef.loss_c, int(bool(ef.above)), len(pa), pp, op, wp, C.byref(idx)))
        elif ef.kind == mc.KIND_MODEL_PARAMETERS:
            tw, twp = _f32(ef.target_weights)
            assert tw.size == self.character.num_params if hasattr(self, "character") else True
            self._check(self._L.mb2_add_model_parameters_error_function(self._h, ef.weight, twp, C.byref(idx)))
        else:
            raise ValueError(ef.kind)
        self.error_functions.append(ef)
        return idx.value

    def upload_targets(self):
        """(Re)send every block's per-instance targets from the spec objects."""
        for idx, ef in enumerate(self.error_functions):
            if getattr(ef, "targets", None) is not None and ef.kind != mc.KIND_LIMIT:
                if getattr(ef, "instance_offsets", None) is not None:  # record = target, then offset (xyz or xyzw)
                    self.set_targets(idx, np.concatenate([np.asarray(ef.targets, np.float32), np.asarray(ef.instance_offsets, np.float32)], -1))
                else:
                    self.set_targets(idx, ef.targets)

    def set_targets(self, index: int, targets):
        t, tp = _f32(targets)
        assert t.shape[0] == self.batch, (t.shape, self.batch)
        self._check(self._L.mb2_set_targets(self._h, index, tp))

    def set_targets_device(self, index: int, device_ptr: int, stream: int = 0):
        self._check(self._L.mb2_set_targets_device(self._h, index, C.c_void_p(device_ptr), C.c_void_p(stream)))

    def set_constraint_weights(self, index: int, weights, per_instance: bool = False):
        w, wp = _f32(weights)
        self._check(self._L.mb2_set_constraint_weights(self._h, index, wp, int(per_instance)))

    def set_constraint_weights_device(self, index: int, device_ptr: int, stream: int = 0):
        self._check(self._L.mb2_set_constraint_weights_device(self._h, index, C.c_void_p(device_ptr), C.c_void_p(stream)))

    def get_jacobian_device(self, params_device_ptr: int, stream: int = 0):
        """(device pointer to [B][n + 1][ld] floats, ld): Jacobian columns then the residual column, in the handle's own buffer."""
        ptr = C.c_void_p(); ld = C.c_int32(0)
        self._check(self._L.mb2_solver_function_get_jacobian_device(self._h, C.c_void_p(params_device_ptr), C.byref(ptr), C.byref(ld), C.c_void_p(stream)))
        return ptr.value, ld.value

    def input_gradients_device(self, index: int, params_device_ptr: int, direction_device_ptr: int, grad_weights_ptr: int = 0,
                               grad_offsets_ptr: int = 0, grad_targets_ptr: int = 0, stream: int = 0):
        """d/d input [grad_theta E_index . v] per instance for a Position or Orientation (matrix difference, L2) block: constraint weights
        [B][nc], offsets and targets [B][nc][3|4] (0 = skip that output), from parameters and directions [B][n]; float32 device memory,
        enqueued on ``stream``."""
        self._check(self._L.mb2_solver_function_input_gradients_device(self._h, int(index), C.c_void_p(params_device_ptr), C.c_void_p(direction_device_ptr),
                                                                       C.c_void_p(grad_weights_ptr or None), C.c_void_p(grad_offsets_ptr or None),
                                                                       C.c_void_p(grad_targets_ptr or None), C.c_void_p(stream)))

    def implicit_direction_device(self, params_device_ptr: int, grad_params_device_ptr: int, direction_ptr: int, jacobian_direction_ptr: int = 0,
                                  residual_ptr: int = 0, gradient_rms_ptr: int = 0, stream: int = 0):
        """The direction of solve_ik's implicit-function backward per instance: v = (2 J_E^T J_E)^+ g [B][n] (0 on disabled
        parameters), J v and the residual [B][jacobian_rows] and the gradient RMS [B], from parameters and dLoss/dtheta [B][n]; float32
        device memory (0 = skip that output; the direction is required), enqueued on ``stream``."""
        self._check(self._L.mb2_solver_function_implicit_direction_device(self._h, C.c_void_p(params_device_ptr), C.c_void_p(grad_params_device_ptr),
                                                                          C.c_void_p(direction_ptr or None), C.c_void_p(jacobian_direction_ptr or None),
                                                                          C.c_void_p(residual_ptr or None), C.c_void_p(gradient_rms_ptr or None),
                                                                          C.c_void_p(stream)))

    def set_error_function_weight(self, index: int, weight: float):
        self._check(self._L.mb2_set_error_function_weight(self._h, index, weight))

    def set_enabled_parameters(self, enabled):
        bits = parameter_set_bits(enabled)
        self._check(self._L.mb2_solver_function_set_enabled_parameters(self._h, bits.ctypes.data_as(_up)))

    @property
    def num_parameters(self):
        return self._L.mb2_solver_function_num_parameters(self._h)

    @property
    def actual_parameters(self):
        return self._L.mb2_solver_function_actual_parameters(self._h)

    @property
    def jacobian_rows(self):
        return self._L.mb2_solver_function_jacobian_rows(self._h)

    def get_error(self, params) -> np.ndarray:
        p, pp = _f32(params)
        out = np.zeros(self.batch, np.float64)
        self._check(self._L.mb2_solver_function_get_error(self._h, pp, out.ctypes.data_as(_dp)))
        return out

    def get_jacobian(self, params):
        """(errors [B], J [B, rows, n], residual [B, rows], rows)"""
        p, pp = _f32(params)
        rows, n = self.jacobian_rows, self.num_parameters
        jac = np.zeros((self.batch, n, rows), np.float32)
        res = np.zeros((self.batch, rows), np.float32)
        err = np.zeros(self.batch, np.float64)
        ar = C.c_int32(0)
        self._check(self._L.mb2_solver_function_get_jacobian(self._h, pp, jac.ctypes.data_as(_fp), res.ctypes.data_as(_fp),
                                                             err.ctypes.data_as(_dp), C.byref(ar)))
        return err, jac.transpose(0, 2, 1), res, ar.value

    def get_jtjr(self, params, jtj_mode: int = JTJ_FP32_SIMT):
        """(errors [B], JtJ [B, ap, ap] lower triangle, Jtr [B, ap])"""
        p, pp = _f32(params)
        ap = self.actual_parameters
        H = np.zeros((self.batch, ap, ap), np.float32)
        g = np.zeros((self.batch, ap), np.float32)
        err = np.zeros(self.batch, np.float64)
        self._check(self._L.mb2_solver_function_get_jtjr(self._h, pp, jtj_mode, H.ctypes.data_as(_fp), g.ctypes.data_as(_fp), err.ctypes.data_as(_dp)))
        return err, H, g

    def get_skeleton_state(self, params) -> np.ndarray:
        p, pp = _f32(params)
        out = np.zeros((self.batch, self.character.num_joints, 8), np.float32)
        self._check(self._L.mb2_solver_function_get_skeleton_state(self._h, pp, out.ctypes.data_as(_fp)))
        return out

    def get_sweep_launch(self, jacobian: bool = True) -> dict:
        """The variant of the FK + residual sweep this handle last launched, for the Jacobian sweep or the error-only one: table
        staging (1 all tables in shared memory, 2 all but cells / contributions, 0 none), warps per instance, instances per CTA, CTAs
        and dynamic shared memory bytes. All zero before the first such sweep and after one whose instance did not fit."""
        out = (C.c_int64 * 5)()
        self._check(self._L.mb2_solver_function_get_sweep_launch(self._h, int(bool(jacobian)), out))
        return dict(zip(("stage", "warps", "groups", "grid", "smem"), (int(v) for v in out)))


class GaussNewtonSolver(_Base):
    """Batch of B ``GaussNewtonSolverT<float>`` (one per IK instance, all stepping together on the GPU)."""

    def __init__(self, options: GaussNewtonSolverOptions, solver_function: SkeletonSolverFunction):
        self._L = solver_function._L
        self.fn = solver_function
        self.options = options
        self._h = C.c_void_p()
        o = options._c()
        self._check(self._L.mb2_solver_create(solver_function._h, C.byref(o), C.byref(self._h)))

    def __del__(self):
        if getattr(self, "_h", None):
            self._L.mb2_solver_destroy(self._h)
            self._h = None

    def get_name(self):
        return "GaussNewton"

    def set_options(self, options: GaussNewtonSolverOptions):
        self.options = options
        o = options._c()
        self._check(self._L.mb2_solver_set_options(self._h, C.byref(o)))

    def set_enabled_parameters(self, enabled):
        bits = parameter_set_bits(enabled)
        self._check(self._L.mb2_solver_set_enabled_parameters(self._h, bits.ctypes.data_as(_up)))

    def solve(self, params):
        """SolverT::solve for every instance. ``params`` [B, n] float32 (host). Returns dict with
        params, errors (objective before the last update, what ``solve`` returns), iterations, status."""
        p = np.ascontiguousarray(params, np.float32).copy()
        B = self.fn.batch
        err = np.zeros(B, np.float64); it = np.zeros(B, np.int32); st = np.zeros(B, np.int32)
        self._check(self._L.mb2_solver_solve(self._h, p.ctypes.data_as(C.c_void_p), err.ctypes.data_as(_dp), it.ctypes.data_as(_ip),
                                             st.ctypes.data_as(_ip)))
        return {"params": p, "errors": err, "iterations": it, "status": st}

    def solve_host_pointer(self, host_ptr: int, results: bool = False):
        """Same through a raw (e.g. pinned) host pointer; per-instance results returned when ``results`` (one mb2_solver_solve call),
        else via get_results()."""
        if not results:
            self._check(self._L.mb2_solver_solve(self._h, C.c_void_p(host_ptr), None, None, None))
            return None
        B = self.fn.batch
        err = np.zeros(B, np.float64); it = np.zeros(B, np.int32); st = np.zeros(B, np.int32)
        self._check(self._L.mb2_solver_solve(self._h, C.c_void_p(host_ptr), err.ctypes.data_as(_dp), it.ctypes.data_as(_ip), st.ctypes.data_as(_ip)))
        return {"errors": err, "iterations": it, "status": st}

    def solve_host_pointer_async(self, host_ptr: int):
        """mb2_solver_solve_async: H2D of the parameters, the solve and the D2H of the result are enqueued on the handle's stream; the
        (pinned) buffer belongs to the library until wait()."""
        self._check(self._L.mb2_solver_solve_async(self._h, C.c_void_p(host_ptr)))

    def wait(self):
        """mb2_solver_wait: blocks until the asynchronous solve is done; per-instance results."""
        B = self.fn.batch
        err = np.zeros(B, np.float64); it = np.zeros(B, np.int32); st = np.zeros(B, np.int32)
        self._check(self._L.mb2_solver_wait(self._h, err.ctypes.data_as(_dp), it.ctypes.data_as(_ip), st.ctypes.data_as(_ip)))
        return {"errors": err, "iterations": it, "status": st}

    def solve_device(self, device_ptr: int, stream: int = 0):
        self._check(self._L.mb2_solver_solve_device(self._h, C.c_void_p(device_ptr), C.c_void_p(stream)))

    def get_results(self):
        B = self.fn.batch
        err = np.zeros(B, np.float64); it = np.zeros(B, np.int32); st = np.zeros(B, np.int32)
        self._check(self._L.mb2_solver_get_results(self._h, err.ctypes.data_as(_dp), it.ctypes.data_as(_ip), st.ctypes.data_as(_ip)))
        return {"errors": err, "iterations": it, "status": st}

    def get_error_history(self):
        B = self.fn.batch
        h = np.zeros((B, max(1, self.options.max_iterations)), np.float64)
        self._check(self._L.mb2_solver_get_error_history(self._h, h.ctypes.data_as(_dp)))
        return h

    def get_counters(self):
        a = C.c_uint64(0); b = C.c_uint64(0)
        self._check(self._L.mb2_solver_get_counters(self._h, C.byref(a), C.byref(b)))
        return a.value, b.value

    def get_plan_stats(self):
        """Per-instance algorithmic sizes of the plan the last solve ran on (see momentum_b200.h)."""
        st = (C.c_int64 * 12)()
        self._check(self._L.mb2_solver_get_plan_stats(self._h, st))
        keys = ["jacobian_nonzeros", "jacobian_columns", "ldj", "normal_parameters", "cholesky_tiles", "cholesky_tile_ops", "cholesky_levels", "rows",
                "strip_floats", "gram_macs", "gram_pairs", "fused_groups"]
        return dict(zip(keys, (int(v) for v in st)))

    FUSED_PHASES = ["fetch", "joint_parameters", "fk", "units", "cells", "gram", "parked_tiles", "chol_diag", "chol_panel", "chol_update",
                    "chol_backward", "update_bookkeeping"]

    def get_fused_profile(self):
        """{fused, groups, kernel_ms, phase_cycles{name: cycles}} of the last solve (kernel_ms / cycles need set_profiling(True))."""
        fused = C.c_int32(0); groups = C.c_int32(0); ms_ = C.c_double(0.0); cyc = (C.c_uint64 * 12)()
        self._check(self._L.mb2_solver_get_fused_profile(self._h, C.byref(fused), C.byref(groups), C.byref(ms_), cyc))
        return {"fused": int(fused.value), "groups": groups.value, "kernel_ms": ms_.value, "phase_cycles": dict(zip(self.FUSED_PHASES, (int(v) for v in cyc)))}

    SOLVE_PATH_KINDS = {0: None, 1: "dense", 2: "tiles_kmajor", 3: "tiles", 4: "gram_cholesky", 5: "persistent", 6: "qr", 7: "trust_region_qr"}
    SOLVE_PATH_KEYS = ["kind", "plan_mode", "sched_dense", "strips", "jtj_mode", "dense_nb", "dense_in_smem", "gram_threads", "chol_threads",
                       "qr_max_chunk_rows", "qr_chunks", "qr_widest_chunk", "tr_r_floats", "fused_groups", "fused_smem"]

    def get_solve_path(self) -> dict:
        """The linear-solve path of the last solve (mb2_solver_get_solve_path): kind as a name (None before the first solve), the
        plan request, the resolved JtJ mode and the launch variants of the kernels it runs."""
        out = (C.c_int64 * 15)()
        self._check(self._L.mb2_solver_get_solve_path(self._h, out))
        d = dict(zip(self.SOLVE_PATH_KEYS, (int(v) for v in out)))
        d["kind"] = self.SOLVE_PATH_KINDS[d["kind"]]
        return d

    def set_profiling(self, level):
        """0 off, 1 CUDA events around every launch (production kernels), 2 + in-kernel phase cycles (instrumented, slower kernels)."""
        self._check(self._L.mb2_solver_set_profiling(self._h, int(level)))

    def get_phase_times(self):
        ms = (C.c_double * 4)(); ln = (C.c_uint64 * 4)()
        self._check(self._L.mb2_solver_get_phase_times(self._h, ms, ln))
        return list(ms), list(ln)


class MixedBatch(_Base):
    """Heterogeneous IK instances (different rigs, different constraint sets) -> buckets that share a plan -> one batched solve per
    bucket -> results in input order (BASELINE.json configs[4]; the reference loops over batch elements, tensor_ik.cpp:127-177)."""

    def __init__(self, device: int = 0, granule: int = 8, lib_path: Optional[str] = None):
        self._L = load_library(lib_path)
        self._h = C.c_void_p()
        self._check(self._L.mb2_mixed_batch_create(device, granule, C.byref(self._h)))
        self.device = device
        self._rigs: List[DeviceCharacter] = []
        self._sizes: List[int] = []   # parameters per instance, input order
        self.lib_path = lib_path

    def _check(self, rc):
        if rc != 0:
            raise MomentumB200Error(self._L.mb2_mixed_batch_last_error().decode())

    def __del__(self):
        if getattr(self, "_h", None):
            self._L.mb2_mixed_batch_destroy(self._h)
            self._h = None

    def add_rig(self, character) -> int:
        dc = character if isinstance(character, DeviceCharacter) else DeviceCharacter(character, self.device, self.lib_path)
        rid = C.c_int32(-1)
        self._check(self._L.mb2_mixed_batch_add_rig(self._h, dc._h, dc.character.num_params, C.byref(rid)))
        self._rigs.append(dc)  # keeps the device character alive
        return rid.value

    def use_limits(self, enabled: bool = True, weight: float = 1.0):
        self._check(self._L.mb2_mixed_batch_use_limits(self._h, int(enabled), weight))

    def add_instance(self, rig: int, parents, offsets, weights, targets, theta0) -> int:
        pa, pp = _i32(parents); of, op = _f32(offsets); w, wp = _f32(weights); tg, tp = _f32(targets); th, thp = _f32(theta0)
        assert of.size == 3 * pa.size and tg.size == 3 * pa.size and w.size == pa.size and th.size == self._rigs[rig].character.num_params
        iid = C.c_int32(-1)
        self._check(self._L.mb2_mixed_batch_add_instance(self._h, rig, pa.size, pp, op, wp, tp, thp, C.byref(iid)))
        self._sizes.append(th.size)
        return iid.value

    def set_parameters(self, instance: int, theta0):
        th, thp = _f32(theta0)
        self._check(self._L.mb2_mixed_batch_set_parameters(self._h, instance, thp))

    def solve(self, options: "GaussNewtonSolverOptions"):
        o = options._c()
        self._check(self._L.mb2_mixed_batch_solve(self._h, C.byref(o)))
        N = len(self._sizes)
        offs = np.zeros(N + 1, np.int64)
        np.cumsum(self._sizes, out=offs[1:])
        theta = np.zeros(int(offs[-1]), np.float32)
        err = np.zeros(N, np.float64); it = np.zeros(N, np.int32); st = np.zeros(N, np.int32)
        self._check(self._L.mb2_mixed_batch_get_results(self._h, theta.ctypes.data_as(_fp), offs.ctypes.data_as(C.POINTER(C.c_int64)), err.ctypes.data_as(_dp),
                                                        it.ctypes.data_as(_ip), st.ctypes.data_as(_ip)))
        return {"params": [theta[offs[i]:offs[i + 1]] for i in range(N)], "errors": err, "iterations": it, "status": st}

    def stats(self):
        st = (C.c_int64 * 6)()
        self._check(self._L.mb2_mixed_batch_stats(self._h, st))
        d = dict(zip(["instances", "buckets", "rows", "padded_rows", "largest_bucket", "singleton_buckets"], (int(v) for v in st)))
        d["padding_waste"] = 1.0 - d["rows"] / d["padded_rows"] if d["padded_rows"] else 0.0
        return d

    def bucket_info(self, bucket: int):
        info = (C.c_int64 * 4)()
        self._check(self._L.mb2_mixed_batch_bucket_info(self._h, bucket, info))
        return dict(zip(["rig", "instances", "constraints", "iterations"], (int(v) for v in info)))


class ShardedGaussNewtonSolver(_Base):
    """One batch over several GPUs from ONE process (mb2_sharded_solver_*): contiguous blocks of instances, one per device, each an
    ordinary batched solver driven by its own host thread; no data-path collective (the reference's batch loop is an independent
    parallel_for over instances, tensor_ik.cpp:127-177). ``function`` is the prototype: its definition (error functions, weights,
    enabled set) is replicated on every device; ``error_functions`` supplies the per-instance targets of the whole batch."""

    def __init__(self, options: "GaussNewtonSolverOptions", function: "SkeletonSolverFunction", total_batch: int, devices, error_functions=None):
        self._L = function._L
        self._h = C.c_void_p()
        self.options = options
        self.total_batch = int(total_batch)
        self.num_params = function.character.num_params
        dv, dp = _i32(devices)
        o = options._c()
        self._check(self._L.mb2_sharded_solver_create(function._h, self.total_batch, dv.size, dp, C.byref(o), C.byref(self._h)))
        if error_functions is not None:
            for idx, ef in enumerate(error_functions):
                if getattr(ef, "targets", None) is not None and np.asarray(ef.targets).size:
                    self.set_targets(idx, ef.targets)

    def _check(self, rc):
        if rc != 0:
            raise MomentumB200Error(self._L.mb2_sharded_last_error().decode())

    def __del__(self):
        if getattr(self, "_h", None):
            self._L.mb2_sharded_solver_destroy(self._h)
            self._h = None

    def shards(self):
        out = []
        for k in range(self._L.mb2_sharded_solver_num_shards(self._h)):
            info = (C.c_int32 * 3)()
            self._check(self._L.mb2_sharded_solver_shard_info(self._h, k, info))
            out.append({"device": info[0], "first": info[1], "count": info[2]})
        return out

    def set_targets(self, index: int, targets):
        t, tp = _f32(targets)
        assert t.shape[0] == self.total_batch
        self._check(self._L.mb2_sharded_solver_set_targets(self._h, index, tp))

    def solve(self, theta0):
        p = np.ascontiguousarray(theta0, np.float32).copy()
        assert p.shape == (self.total_batch, self.num_params)
        B = self.total_batch
        err = np.zeros(B, np.float64); it = np.zeros(B, np.int32); st = np.zeros(B, np.int32)
        self._check(self._L.mb2_sharded_solver_solve(self._h, p.ctypes.data_as(C.c_void_p), err.ctypes.data_as(_dp), it.ctypes.data_as(_ip), st.ctypes.data_as(_ip)))
        agg = (C.c_double * 3)()
        self._check(self._L.mb2_sharded_solver_get_aggregate(self._h, agg))
        return {"params": p, "errors": err, "iterations": it, "status": st, "aggregate": {"error_sum": agg[0], "iterations": int(agg[1]), "instances_ok": int(agg[2])}}

    def solve_host_pointer(self, host_ptr: int):
        """In place on a raw (pinned) host buffer [total_batch][n]; the aggregate via get_aggregate()."""
        self._check(self._L.mb2_sharded_solver_solve(self._h, C.c_void_p(host_ptr), None, None, None))

    def get_aggregate(self):
        agg = (C.c_double * 3)()
        self._check(self._L.mb2_sharded_solver_get_aggregate(self._h, agg))
        return {"error_sum": agg[0], "iterations": int(agg[1]), "instances_ok": int(agg[2])}
