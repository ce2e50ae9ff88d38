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
_lp = C.POINTER(C.c_int64)

# The signature, (restype, argtypes), of every function include/momentum_b200.h declares, in its order (tests/test_cabi_symbols.py
# checks the names and argument counts against the header). Handles, device memory and streams are c_void_p: a plain int is a
# pointer and 0 is NULL. Host arrays keep their element type.
_vp, _int, _int32, _float = C.c_void_p, C.c_int, C.c_int32, C.c_float
_out, _opt = C.POINTER(_vp), C.POINTER(_Options)
CABI_SIGNATURES = {
    "mb2_last_error": (C.c_char_p, []),
    "mb2_device_count": (_int, []),
    "mb2_default_gauss_newton_options": (None, [_opt]),
    "mb2_character_create": (_int, [_int, _int32, _ip, _fp, _fp, _int32, _ip, _ip, _fp, _fp, _out]),
    "mb2_character_set_parameter_limits": (_int, [_vp, _int32, C.POINTER(_Limit)]),
    "mb2_character_destroy": (None, [_vp]),
    "mb2_solver_function_create": (_int, [_vp, _int32, _out]),
    "mb2_solver_function_destroy": (None, [_vp]),
    "mb2_solver_function_num_parameters": (_int32, [_vp]),
    "mb2_solver_function_actual_parameters": (_int32, [_vp]),
    "mb2_solver_function_batch": (_int32, [_vp]),
    "mb2_solver_function_jacobian_rows": (_int32, [_vp]),
    "mb2_solver_function_jacobian_stride": (_int32, [_vp]),
    "mb2_add_position_error_function": (_int, [_vp, _float, _float, _float, _int32, _ip, _fp, _fp, _ip]),
    "mb2_add_position_error_function_instanced": (_int, [_vp, _float, _float, _float, _int32, _ip, _fp, _ip]),
    "mb2_add_orientation_error_function_instanced": (_int, [_vp, _float, _float, _float, _int32, _int32, _ip, _fp, _ip]),
    "mb2_add_plane_error_function": (_int, [_vp, _float, _float, _float, _int32, _int32, _ip, _fp, _fp, _ip]),
    "mb2_add_model_parameters_error_function": (_int, [_vp, _float, _fp, _ip]),
    "mb2_add_orientation_error_function": (_int, [_vp, _float, _float, _float, _int32, _int32, _ip, _fp, _fp, _ip]),
    "mb2_add_state_error_function": (_int, [_vp, _float, _int32, _float, _float, _fp, _fp, _ip]),
    "mb2_add_limit_error_function": (_int, [_vp, _float, _float, _float, _ip]),
    "mb2_set_error_function_weight": (_int, [_vp, _int32, _float]),
    "mb2_set_targets": (_int, [_vp, _int32, _fp]),
    "mb2_set_targets_device": (_int, [_vp, _int32, _vp, _vp]),
    "mb2_set_constraint_weights": (_int, [_vp, _int32, _fp, _int32]),
    "mb2_set_constraint_weights_device": (_int, [_vp, _int32, _vp, _vp]),
    "mb2_solver_function_set_enabled_parameters": (_int, [_vp, _up]),
    "mb2_solver_function_get_error": (_int, [_vp, _fp, _dp]),
    "mb2_solver_function_get_jacobian": (_int, [_vp, _fp, _fp, _fp, _dp, _ip]),
    "mb2_solver_function_get_jacobian_device": (_int, [_vp, _vp, _out, _ip, _vp]),
    "mb2_solver_function_get_jtjr": (_int, [_vp, _fp, _int32, _fp, _fp, _dp]),
    "mb2_solver_function_get_skeleton_state": (_int, [_vp, _fp, _fp]),
    "mb2_character_skeleton_state_device": (_int, [_vp, _int32, _vp, _vp, _vp]),
    "mb2_character_skeleton_state_backward_device": (_int, [_vp, _int32, _vp, _vp, _vp, _vp]),
    "mb2_character_apply_parameter_transform_device": (_int, [_vp, _int32, _vp, _vp, _vp]),
    "mb2_character_apply_parameter_transform_backward_device": (_int, [_vp, _int32, _vp, _vp, _vp]),
    "mb2_character_apply_inverse_parameter_transform_device": (_int, [_vp, _int32, _vp, _vp, _vp]),
    "mb2_character_apply_inverse_parameter_transform_backward_device": (_int, [_vp, _int32, _vp, _vp, _vp]),
    "mb2_character_joint_parameters_to_skeleton_state_device": (_int, [_vp, _int32, _vp, _vp, _vp]),
    "mb2_character_joint_parameters_to_skeleton_state_backward_device": (_int, [_vp, _int32, _vp, _vp, _vp, _vp]),
    "mb2_character_joint_parameters_to_local_skeleton_state_device": (_int, [_vp, _int32, _vp, _vp, _vp]),
    "mb2_character_joint_parameters_to_local_skeleton_state_backward_device": (_int, [_vp, _int32, _vp, _vp, _vp, _vp]),
    "mb2_character_local_skeleton_state_to_joint_parameters_device": (_int, [_vp, _int32, _vp, _vp, _vp]),
    "mb2_character_local_skeleton_state_to_joint_parameters_backward_device": (_int, [_vp, _int32, _vp, _vp, _vp, _vp]),
    "mb2_character_skeleton_state_to_joint_parameters_device": (_int, [_vp, _int32, _vp, _vp, _vp]),
    "mb2_character_skeleton_state_to_joint_parameters_backward_device": (_int, [_vp, _int32, _vp, _vp, _vp, _vp]),
    "mb2_character_model_parameters_to_positions_device": (_int, [_vp, _int32, _vp, _int32, _ip, _vp, _int32, _vp, _vp]),
    "mb2_character_joint_parameters_to_positions_device": (_int, [_vp, _int32, _vp, _int32, _ip, _vp, _int32, _vp, _vp]),
    "mb2_character_model_parameters_to_positions_backward_device": (_int, [_vp, _int32, _vp, _int32, _ip, _vp, _int32, _vp, _vp, _vp, _vp]),
    "mb2_character_joint_parameters_to_positions_backward_device": (_int, [_vp, _int32, _vp, _int32, _ip, _vp, _int32, _vp, _vp, _vp, _vp]),
    "mb2_character_set_skinning": (_int, [_vp, _int32, _fp, _ip, _fp, _fp]),
    "mb2_character_num_vertices": (_int32, [_vp]),
    "mb2_character_skin_points_device": (_int, [_vp, _int32, _vp, _vp, _int32, _vp, _vp]),
    "mb2_character_skin_points_backward_device": (_int, [_vp, _int32, _vp, _vp, _int32, _vp, _vp, _vp, _vp]),
    "mb2_character_set_blend_shape": (_int, [_vp, _int32, _int32, _fp, _fp]),
    "mb2_character_num_blend_shapes": (_int32, [_vp]),
    "mb2_character_skin_with_blend_shapes_device": (_int, [_vp, _int32, _vp, _vp, _int32, _vp, _vp]),
    "mb2_character_skin_with_blend_shapes_backward_device": (_int, [_vp, _int32, _vp, _vp, _int32, _vp, _vp, _vp, _vp]),
    "mb2_character_set_mesh_faces": (_int, [_vp, _int32, _int32, _ip]),
    "mb2_character_num_faces": (_int32, [_vp]),
    "mb2_character_vertex_normals_device": (_int, [_vp, _int32, _vp, _vp, _vp]),
    "mb2_character_vertex_normals_backward_device": (_int, [_vp, _int32, _vp, _vp, _vp, _vp]),
    "mb2_character_set_mesh_tree": (_int, [_vp, _int32, _fp]),
    "mb2_character_closest_points_on_mesh_device": (_int, [_vp, _int32, _int32, _vp, _vp, _float, _vp, _vp, _vp, _vp]),
    "mb2_closest_points_device": (_int, [_int, _int32, _int32, _int32, _int32, _vp, _vp, _vp, _vp, _float, _float, _vp, _vp, _vp, _vp]),
    "mb2_solver_function_input_gradients_device": (_int, [_vp, _int32, _vp, _vp, _vp, _vp, _vp, _vp]),
    "mb2_solver_function_implicit_direction_device": (_int, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "mb2_solver_create": (_int, [_vp, _opt, _out]),
    "mb2_solver_destroy": (None, [_vp]),
    "mb2_solver_set_options": (_int, [_vp, _opt]),
    "mb2_solver_set_enabled_parameters": (_int, [_vp, _up]),
    "mb2_solver_solve": (_int, [_vp, _vp, _dp, _ip, _ip]),
    "mb2_solver_solve_async": (_int, [_vp, _vp]),
    "mb2_solver_wait": (_int, [_vp, _dp, _ip, _ip]),
    "mb2_solver_solve_device": (_int, [_vp, _vp, _vp]),
    "mb2_solver_get_results": (_int, [_vp, _dp, _ip, _ip]),
    "mb2_solver_get_error_history": (_int, [_vp, _dp]),
    "mb2_solver_get_counters": (_int, [_vp, _up, _up]),
    "mb2_solver_set_profiling": (_int, [_vp, _int32]),
    "mb2_solver_get_phase_times": (_int, [_vp, _dp, _up]),
    "mb2_solver_get_plan_stats": (_int, [_vp, _lp]),
    "mb2_solver_get_fused_profile": (_int, [_vp, _ip, _ip, _dp, _up]),
    "mb2_solver_function_get_sweep_launch": (_int, [_vp, _int32, _lp]),
    "mb2_character_get_instance_launch": (_int, [_vp, _int32, _int32, _int32, _int32, _lp]),
    "mb2_character_set_collision_geometry": (_int, [_vp, _int32, _vp]),
    "mb2_character_num_collision_pairs": (_int, [_vp, _ip]),
    "mb2_character_get_collision_pairs": (_int, [_vp, _vp]),
    "mb2_character_collision_residual_device": (_int, [_vp, _int32, _vp, _vp, _vp]),
    "mb2_character_collision_residual_backward_device": (_int, [_vp, _int32, _vp, _vp, _vp, _vp]),
    "mb2_character_num_limit_residuals": (_int, [_vp, _ip]),
    "mb2_character_parameter_limits_residual_device": (_int, [_vp, _int32, _vp, _vp, _vp]),
    "mb2_character_parameter_limits_residual_backward_device": (_int, [_vp, _int32, _vp, _vp, _vp, _vp]),
    "mb2_character_apply_model_parameter_limits_device": (_int, [_vp, _int32, _vp, _vp, _vp]),
    "mb2_character_apply_model_parameter_limits_backward_device": (_int, [_vp, _int32, _vp, _vp, _vp, _vp]),
    "mb2_solver_function_get_input_gradient_launch": (_int, [_vp, _lp]),
    "mb2_solver_get_solve_path": (_int, [_vp, _lp]),
    "mb2_mixed_batch_last_error": (C.c_char_p, []),
    "mb2_mixed_batch_create": (_int, [_int, _int32, _out]),
    "mb2_mixed_batch_destroy": (None, [_vp]),
    "mb2_mixed_batch_add_rig": (_int, [_vp, _vp, _int32, _ip]),
    "mb2_mixed_batch_use_limits": (_int, [_vp, _int32, _float]),
    "mb2_mixed_batch_add_instance": (_int, [_vp, _int32, _int32, _ip, _fp, _fp, _fp, _fp, _ip]),
    "mb2_mixed_batch_set_parameters": (_int, [_vp, _int32, _fp]),
    "mb2_mixed_batch_solve": (_int, [_vp, _opt]),
    "mb2_mixed_batch_get_result": (_int, [_vp, _int32, _fp, _dp, _ip, _ip]),
    "mb2_mixed_batch_get_results": (_int, [_vp, _fp, _lp, _dp, _ip, _ip]),
    "mb2_mixed_batch_stats": (_int, [_vp, _lp]),
    "mb2_mixed_batch_bucket_info": (_int, [_vp, _int32, _lp]),
    "mb2_character_clone": (_int, [_vp, _int, _out]),
    "mb2_solver_function_clone": (_int, [_vp, _vp, _int32, _out]),
    "mb2_character_device": (_int, [_vp]),
    "mb2_solver_function_character": (_vp, [_vp]),
    "mb2_solver_function_num_error_functions": (_int32, [_vp]),
    "mb2_solver_function_target_size": (_int32, [_vp, _int32]),
    "mb2_sharded_last_error": (C.c_char_p, []),
    "mb2_sharded_solver_create": (_int, [_vp, _int32, _int32, _ip, _opt, _out]),
    "mb2_sharded_solver_destroy": (None, [_vp]),
    "mb2_sharded_solver_num_shards": (_int32, [_vp]),
    "mb2_sharded_solver_shard_info": (_int, [_vp, _int32, _ip]),
    "mb2_sharded_solver_set_options": (_int, [_vp, _opt]),
    "mb2_sharded_solver_set_targets": (_int, [_vp, _int32, _fp]),
    "mb2_sharded_solver_solve": (_int, [_vp, _vp, _dp, _ip, _ip]),
    "mb2_sharded_solver_get_aggregate": (_int, [_vp, _dp]),
}
CABI_SYMBOLS = sorted(CABI_SIGNATURES)

# the skeleton-state family of DeviceCharacter.joint_op_device: name -> (forward entry, backward entry)
JOINT_OPS = {
    "model_parameters_to_skeleton_state": ("mb2_character_skeleton_state_device", "mb2_character_skeleton_state_backward_device"),
    **{name: (f"mb2_character_{name}_device", f"mb2_character_{name}_backward_device")
       for name in ("apply_parameter_transform", "apply_inverse_parameter_transform", "joint_parameters_to_skeleton_state",
                    "joint_parameters_to_local_skeleton_state", "local_skeleton_state_to_joint_parameters", "skeleton_state_to_joint_parameters",
                    "apply_model_parameter_limits")},
}
# the operations whose backward does not read their input (P^T and W^T), so their backward takes no input pointer
LINEAR_JOINT_OPS = frozenset({"apply_parameter_transform", "apply_inverse_parameter_transform"})

_libs = {}


def load_library(path: Optional[str] = None):
    path = path or DEFAULT_LIB
    if path in _libs:
        return _libs[path]
    if not os.path.exists(path):
        raise MomentumB200Error(f"{path} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                                "(momentum_b200 has no CPU fallback)")
    L = C.CDLL(path)
    for name, (restype, argtypes) in CABI_SIGNATURES.items():
        if hasattr(L, name):  # the CPU emulator library of the tests exports a subset of the C-ABI
            fn = getattr(L, name)
            fn.restype, fn.argtypes = restype, argtypes
    _libs[path] = L
    return L


def closest_points_device(device: int, batch: int, num_source: int, num_target: int, target_batched: bool, source_ptr: int,
                          source_normals_ptr: int, target_ptr: int, target_normals_ptr: int, max_dist: float, max_normal_dot: float,
                          out_points_ptr: int, out_normals_ptr: int, out_index_ptr: int, stream: int = 0, lib: Optional[str] = None):
    """mb2_closest_points_device: the closest target point of each query point, source [B][N][3] against target [B or 1][M][3] (one
    shared target unless ``target_batched``), device float32 memory on ``device``; the normal pointers are all 0 (the plain variant) or
    all set. Writes out points [B][N][3], out normals [B][N][3] and out index [B][N] int32 (-1 without a candidate), enqueued on
    ``stream``. Raises MomentumB200Error with the library's message when it rejects the call."""
    L = load_library(lib)
    rc = L.mb2_closest_points_device(int(device), int(batch), int(num_source), int(num_target), int(bool(target_batched)), source_ptr,
                                     source_normals_ptr, target_ptr, target_normals_ptr, float(max_dist), float(max_normal_dot), out_points_ptr,
                                     out_normals_ptr, out_index_ptr, stream)
    if rc != 0:
        raise MomentumB200Error(L.mb2_last_error().decode())


def _f32(a):
    a = np.ascontiguousarray(a, np.float32)
    return a, a.ctypes.data_as(_fp)


def _i32(a):
    a = np.ascontiguousarray(a, np.int32)
    return a, a.ctypes.data_as(_ip)


def _results(n: int):
    """Per-instance results of n instances, {errors float64, iterations int32, status int32} zeroed, and their pointers in the
    C-ABI's (errors, iterations, status) order."""
    r = {"errors": np.zeros(n, np.float64), "iterations": np.zeros(n, np.int32), "status": np.zeros(n, np.int32)}
    return r, (r["errors"].ctypes.data_as(_dp), r["iterations"].ctypes.data_as(_ip), r["status"].ctypes.data_as(_ip))


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


# the skeleton-state and positions operations mb2_character_get_instance_launch reports on, by its op code
INSTANCE_OPS = {"model_parameters_to_skeleton_state": 0, "joint_parameters_to_skeleton_state": 1, "model_parameters_to_positions": 2,
                "joint_parameters_to_positions": 3}
# its op code of parameter_limits_residual, whose launch depends on the character's limits rather than on a rig alone
PARAMETER_LIMITS_INSTANCE_OP = 5
# and of collision_residual, whose launch depends on the character's capsules
COLLISION_INSTANCE_OP = 6


def _instance_launch(out) -> dict:
    return dict(zip(("warps", "groups", "threads", "grid", "smem", "staged"), (int(v) for v in out)))


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
        # Capsules the library rejects are reported by the collision calls, as a rejected blend shape is: nothing else depends on them.
        self.collision, self.collision_error = None, None
        if character.collision is not None:
            try:
                self.set_collision_geometry(character.collision)
            except (MomentumB200Error, ValueError) as e:
                self.collision_error = str(e)
        self.skinning, self.faces, self.faces_error, self.mesh_tree_error = None, None, None, None
        if character.skinning is not None:
            self.set_skinning(character.skinning)
        # A blend shape the library rejects is reported by the blend-shape calls, not here: the rig, its skinning and every other use of
        # the handle do not depend on it.
        self.blend_shape, self.blend_shape_error = None, None
        if character.blend_shape is not None:
            try:
                self.set_blend_shape(character.blend_shape)
            except (MomentumB200Error, ValueError) as e:
                self.blend_shape_error = str(e)

    def set_skinning(self, skinning: mc.Skinning):
        """Uploads ``skinning`` (replacing any earlier one) and its ``faces``, or removes the faces when it has none; ``self.skinning`` and
        ``self.faces`` are the objects uploaded. Faces the library rejects do not fail the skinning upload: ``self.faces`` is then None
        and ``self.faces_error`` the reason, which ``torch_skeleton.compute_vertex_normals`` raises."""
        V = skinning.num_vertices
        rv, rvp = _f32(np.asarray(skinning.rest_vertices).reshape(V, 3))
        si, sip = _i32(np.asarray(skinning.skin_index).reshape(V, mc.MAX_SKIN_JOINTS))
        sw, swp = _f32(np.asarray(skinning.skin_weight).reshape(V, mc.MAX_SKIN_JOINTS))
        ib, ibp = _f32(np.asarray(skinning.inverse_bind_pose).reshape(self.character.num_joints, 12))
        self._check(self._L.mb2_character_set_skinning(self._h, V, rvp, sip, swp, ibp))
        self.skinning = skinning
        self.faces, self.faces_error = None, None
        self.mesh_tree_error = None
        try:
            self._set_mesh_faces(V, skinning.faces)
            self.faces = skinning.faces
        except (MomentumB200Error, ValueError) as e:
            self._check(self._L.mb2_character_set_mesh_faces(self._h, 0, 0, None))  # no faces left from an earlier skinning
            self.faces_error = str(e)
        if self.faces is not None and self.faces.shape[0] > 0:
            # the closest-point tree over the rest mesh; replacing the faces above dropped any earlier one
            try:
                self.set_mesh_tree(skinning.rest_vertices)
            except MomentumB200Error as e:
                self.mesh_tree_error = str(e)

    def set_mesh_tree(self, reference_positions):
        """Builds the closest-point tree over the uploaded faces from ``reference_positions`` [V, 3] (``set_skinning`` uses the rest mesh),
        or removes it when None. The pose changes how fast ``closest_points_on_mesh_device`` is, never what it returns."""
        if reference_positions is None:
            self._check(self._L.mb2_character_set_mesh_tree(self._h, 0, None))
            return
        x = np.asarray(reference_positions)
        if x.ndim != 2 or x.shape[1] != 3:
            raise ValueError(f"mesh tree: reference_positions must be [V, 3], got {x.shape}")
        xa, xp = _f32(x)
        self._check(self._L.mb2_character_set_mesh_tree(self._h, int(x.shape[0]), xp))
        self.mesh_tree_error = None

    def closest_points_on_mesh_device(self, batch: int, num_points: int, vertices_device_ptr: int, points_device_ptr: int, max_dist: float,
                                      out_points_device_ptr: int, out_face_device_ptr: int, out_bary_device_ptr: int, stream: int = 0):
        """The closest point on each instance's mesh (vertices [B][V][3]) of its query points [B][N][3]: out points [B][N][3], faces
        [B][N] int32 (-1 without a face within ``max_dist``) and barycentrics [B][N][3]. Device memory on this character's device,
        enqueued on ``stream``."""
        self._check(self._L.mb2_character_closest_points_on_mesh_device(self._h, int(batch), int(num_points), vertices_device_ptr, points_device_ptr,
                                                                        float(max_dist), out_points_device_ptr, out_face_device_ptr,
                                                                        out_bary_device_ptr, stream))

    def _set_mesh_faces(self, num_vertices: int, faces):
        if faces is None:
            self._check(self._L.mb2_character_set_mesh_faces(self._h, 0, 0, None))
            return
        f = np.asarray(faces)
        if f.ndim != 2 or f.shape[1] != 3 or f.dtype.kind not in "iu":
            raise ValueError(f"mesh faces: faces must be an integer array [F, 3], got {f.dtype} {f.shape}")
        if f.size and (f.min() < np.iinfo(np.int32).min or f.max() > np.iinfo(np.int32).max):
            raise ValueError("mesh faces: a face index is outside [0, num_vertices)")
        fa, fp = _i32(f)
        self._check(self._L.mb2_character_set_mesh_faces(self._h, int(num_vertices), int(f.shape[0]), fp))

    @property
    def num_faces(self) -> int:
        return int(self._L.mb2_character_num_faces(self._h))

    def vertex_normals_device(self, batch: int, positions_device_ptr: int, normals_device_ptr: int, stream: int = 0):
        """Area-weighted vertex normals [B][V][3] of vertex positions [B][V][3] over the uploaded faces. float32 device memory on this
        character's device, enqueued on ``stream``."""
        self._check(self._L.mb2_character_vertex_normals_device(self._h, int(batch), positions_device_ptr, normals_device_ptr, stream))

    def vertex_normals_backward_device(self, batch: int, positions_device_ptr: int, grad_normals_device_ptr: int, grad_positions_device_ptr: int,
                                       stream: int = 0):
        """dLoss/d positions [B][V][3] (overwritten) from dLoss/d normals [B][V][3]."""
        self._check(self._L.mb2_character_vertex_normals_backward_device(self._h, int(batch), positions_device_ptr, grad_normals_device_ptr,
                                                                         grad_positions_device_ptr, stream))

    @property
    def num_vertices(self) -> int:
        return int(self._L.mb2_character_num_vertices(self._h))

    def skin_points_device(self, batch: int, state_device_ptr: int, rest_device_ptr: int, rest_batched: bool, points_device_ptr: int, stream: int = 0):
        """Skinned points [B][V][3] of skeleton states [B][J][8]; rest points: 0 = the rest mesh, else [V][3] (shared) or [B][V][3]
        (``rest_batched``). float32 device memory on this character's device, enqueued on ``stream``."""
        self._check(self._L.mb2_character_skin_points_device(self._h, int(batch), state_device_ptr, rest_device_ptr, int(bool(rest_batched)),
                                                             points_device_ptr, stream))

    def skin_points_backward_device(self, batch: int, state_device_ptr: int, rest_device_ptr: int, rest_batched: bool, grad_points_device_ptr: int,
                                    grad_state_device_ptr: int, grad_rest_device_ptr: int, stream: int = 0):
        """dLoss/d skeleton state [B][J][8] and dLoss/d rest points (the rest-point layout; the batch sum when shared) from dLoss/d points
        [B][V][3]. A 0 output pointer is skipped."""
        self._check(self._L.mb2_character_skin_points_backward_device(self._h, int(batch), state_device_ptr, rest_device_ptr, int(bool(rest_batched)),
                                                                      grad_points_device_ptr, grad_state_device_ptr, grad_rest_device_ptr, stream))

    def set_blend_shape(self, blend_shape: mc.BlendShape):
        """Uploads ``blend_shape`` (replacing any earlier one); ``self.blend_shape`` is the object uploaded."""
        base, vectors = np.asarray(blend_shape.base_shape), np.asarray(blend_shape.shape_vectors)
        if base.ndim != 2 or base.shape[1] != 3 or vectors.ndim != 3 or vectors.shape[1:] != base.shape:
            raise ValueError(f"blend shape: base_shape must be [V, 3] and shape_vectors [K, V, 3] with the same V, got {base.shape} and {vectors.shape}")
        K, V = vectors.shape[0], base.shape[0]
        bs, bsp = _f32(base)
        sv, svp = _f32(vectors)
        self._check(self._L.mb2_character_set_blend_shape(self._h, K, V, bsp, svp))
        self.blend_shape, self.blend_shape_error = blend_shape, None

    @property
    def num_blend_shapes(self) -> int:
        return int(self._L.mb2_character_num_blend_shapes(self._h))

    def skin_with_blend_shapes_device(self, batch: int, state_device_ptr: int, weights_device_ptr: int, num_weights: int, points_device_ptr: int,
                                      stream: int = 0):
        """Points [B][V][3] of skeleton states [B][J][8], the rest mesh shaped by blend weights [B][num_weights]. float32 device memory on
        this character's device, enqueued on ``stream``."""
        self._check(self._L.mb2_character_skin_with_blend_shapes_device(self._h, int(batch), state_device_ptr, weights_device_ptr, int(num_weights),
                                                                        points_device_ptr, stream))

    def skin_with_blend_shapes_backward_device(self, batch: int, state_device_ptr: int, weights_device_ptr: int, num_weights: int,
                                               grad_points_device_ptr: int, grad_state_device_ptr: int, grad_weights_device_ptr: int, stream: int = 0):
        """dLoss/d skeleton state [B][J][8] and dLoss/d blend weights [B][num_weights] from dLoss/d points [B][V][3]. A 0 output pointer
        is skipped."""
        self._check(self._L.mb2_character_skin_with_blend_shapes_backward_device(self._h, int(batch), state_device_ptr, weights_device_ptr,
                                                                                 int(num_weights), grad_points_device_ptr, grad_state_device_ptr,
                                                                                 grad_weights_device_ptr, stream))

    def joint_op_device(self, name: str, backward: bool, batch: int, *ptrs: int, stream: int = 0):
        """One direction of an operation of the skeleton-state family (``JOINT_OPS``: model_parameters_to_skeleton_state,
        apply_parameter_transform, apply_inverse_parameter_transform, joint_parameters_to_skeleton_state,
        joint_parameters_to_local_skeleton_state, local_skeleton_state_to_joint_parameters, skeleton_state_to_joint_parameters), float32
        device memory on this character's device, enqueued on ``stream`` (0: the legacy default stream). ``ptrs``: forward (input,
        output); backward (input, dLoss/d output, dLoss/d input), except the backward of the two linear ops in ``LINEAR_JOINT_OPS``,
        which takes (dLoss/d output, dLoss/d input). A 0 pointer is passed as null."""
        fn = getattr(self._L, JOINT_OPS[name][1 if backward else 0])
        self._check(fn(self._h, int(batch), *ptrs, stream))

    def get_instance_launch(self, op: str, backward: bool, batch: int, num_points: int = 0) -> dict:
        """What the per-instance kernel of ``op`` (a key of ``INSTANCE_OPS``, "parameter_limits_residual" or "collision_residual") would launch for ``batch``
        instances (and ``num_points`` points): warps per instance, instances per CTA, threads per CTA, CTAs, dynamic shared memory bytes
        and whether the point tables are staged. All zero when nothing runs; raises when one instance does not fit in shared memory."""
        code = {"parameter_limits_residual": PARAMETER_LIMITS_INSTANCE_OP, "collision_residual": COLLISION_INSTANCE_OP}.get(op)
        code = INSTANCE_OPS[op] if code is None else code
        out = (C.c_int64 * 6)()
        self._check(self._L.mb2_character_get_instance_launch(self._h, code, int(bool(backward)), int(batch), int(num_points), out))
        return _instance_launch(out)

    def set_collision_geometry(self, capsules):
        """Uploads the tapered capsules (a list of ``character.TaperedCapsule``, replacing any earlier geometry; empty is valid) and plans
        their valid pairs; ``self.collision`` is the list uploaded and ``self.num_collision_pairs`` P. Raises naming the capsule when one is rejected, and keeps the earlier
        geometry then."""
        arr = mc.capsule_array(capsules)
        self._check(self._L.mb2_character_set_collision_geometry(self._h, len(arr), arr.ctypes.data if len(arr) else None))
        self.collision, self.collision_error = list(capsules), None
        n = C.c_int32(0)
        self._check(self._L.mb2_character_num_collision_pairs(self._h, C.byref(n)))
        self.num_collision_pairs = int(n.value)

    def collision_pairs(self) -> np.ndarray:
        """The planned pairs of the uploaded geometry: int32 [P, 2], i < j ascending."""
        n = C.c_int32(0)
        self._check(self._L.mb2_character_num_collision_pairs(self._h, C.byref(n)))
        out = np.zeros((int(n.value), 2), np.int32)
        self._check(self._L.mb2_character_get_collision_pairs(self._h, out.ctypes.data if out.size else None))
        return out

    def collision_residual_device(self, batch: int, state_device_ptr: int, residual_device_ptr: int, stream: int = 0):
        """The collision rows [B][P] of skeleton states [B][J][8]; float32 device memory on this character's device, enqueued on
        ``stream``."""
        self._check(self._L.mb2_character_collision_residual_device(self._h, int(batch), state_device_ptr, residual_device_ptr, stream))

    def collision_residual_backward_device(self, batch: int, state_device_ptr: int, grad_residual_device_ptr: int, grad_state_device_ptr: int,
                                           stream: int = 0):
        """dLoss/d skeleton states [B][J][8] from dLoss/d rows [B][P], overwritten."""
        self._check(self._L.mb2_character_collision_residual_backward_device(self._h, int(batch), state_device_ptr, grad_residual_device_ptr,
                                                                           grad_state_device_ptr, stream))

    def num_limit_residuals(self) -> int:
        """R, the rows of parameter_limits_residual for the limits this handle was made with (one per limit, none for
        MinMaxJointPassive, three for an Ellipsoid). Raises with the reason when a limit's index is out of range."""
        out = C.c_int32(0)
        self._check(self._L.mb2_character_num_limit_residuals(self._h, C.byref(out)))
        return int(out.value)

    def parameter_limits_residual_device(self, batch: int, theta_device_ptr: int, residual_device_ptr: int, stream: int = 0):
        """The LimitErrorFunction rows [B][R] (weight 1, L2 loss) of model parameters [B][n]; float32 device memory on this character's
        device, enqueued on ``stream``."""
        self._check(self._L.mb2_character_parameter_limits_residual_device(self._h, int(batch), theta_device_ptr, residual_device_ptr, stream))

    def parameter_limits_residual_backward_device(self, batch: int, theta_device_ptr: int, grad_residual_device_ptr: int,
                                                  grad_theta_device_ptr: int, stream: int = 0):
        """dLoss/d model parameters [B][n] from dLoss/d residual [B][R], overwritten."""
        self._check(self._L.mb2_character_parameter_limits_residual_backward_device(self._h, int(batch), theta_device_ptr, grad_residual_device_ptr,
                                                                                  grad_theta_device_ptr, stream))

    def positions_device(self, joint: bool, batch: int, params_device_ptr: int, parents: np.ndarray, offsets_device_ptr: int, offsets_batched: bool,
                         positions_device_ptr: int, stream: int = 0):
        """World positions [B][N][3] of N points fixed in joints' frames from model parameters [B][n] (``joint``: joint parameters
        [B][7 J]). ``parents``: an int32 host array [N] of joint indices; offsets [N][3], or [B][N][3] when ``offsets_batched``. float32
        device memory on this character's device, enqueued on ``stream``."""
        p = np.ascontiguousarray(parents, np.int32)
        fn = self._L.mb2_character_joint_parameters_to_positions_device if joint else self._L.mb2_character_model_parameters_to_positions_device
        self._check(fn(self._h, int(batch), params_device_ptr, int(p.size), p.ctypes.data_as(_ip), offsets_device_ptr, int(bool(offsets_batched)),
                       positions_device_ptr, stream))

    def positions_backward_device(self, joint: bool, batch: int, params_device_ptr: int, parents: np.ndarray, offsets_device_ptr: int,
                                  offsets_batched: bool, grad_positions_device_ptr: int, grad_params_device_ptr: int, grad_offsets_device_ptr: int,
                                  stream: int = 0):
        """dLoss/d parameters and dLoss/d offsets (the offset layout; the batch sum when shared) from dLoss/d positions [B][N][3]. A 0
        output pointer is skipped; not both."""
        p = np.ascontiguousarray(parents, np.int32)
        fn = (self._L.mb2_character_joint_parameters_to_positions_backward_device if joint
              else self._L.mb2_character_model_parameters_to_positions_backward_device)
        self._check(fn(self._h, int(batch), params_device_ptr, int(p.size), p.ctypes.data_as(_ip), offsets_device_ptr, int(bool(offsets_batched)),
                       grad_positions_device_ptr, grad_params_device_ptr, grad_offsets_device_ptr, stream))

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
        self._check(self._L.mb2_set_targets_device(self._h, index, device_ptr, stream))

    def set_constraint_weights(self, index: int, weights, per_instance: bool = False):
        w, wp = _f32(weights)
        self._check(self._L.mb2_set_constraint_weights(self._h, index, wp, int(per_instance)))

    def set_constraint_weights_device(self, index: int, device_ptr: int, stream: int = 0):
        self._check(self._L.mb2_set_constraint_weights_device(self._h, index, device_ptr, stream))

    def get_jacobian_device(self, params_device_ptr: int, stream: int = 0):
        """(device pointer to [B][n + 1][ld] floats, ld): Jacobian columns then the residual column, in the handle's own buffer."""
        ptr = C.c_void_p(); ld = C.c_int32(0)
        self._check(self._L.mb2_solver_function_get_jacobian_device(self._h, params_device_ptr, C.byref(ptr), C.byref(ld), stream))
        return ptr.value, ld.value

    def input_gradients_device(self, index: int, params_device_ptr: int, direction_device_ptr: int, grad_weights_ptr: int = 0,
                               grad_offsets_ptr: int = 0, grad_targets_ptr: int = 0, stream: int = 0):
        """d/d input [grad_theta E_index . v] per instance for a Position or Orientation (matrix difference, L2) block: constraint weights
        [B][nc], offsets and targets [B][nc][3|4] (0 = skip that output), from parameters and directions [B][n]; float32 device memory,
        enqueued on ``stream``."""
        self._check(self._L.mb2_solver_function_input_gradients_device(self._h, int(index), params_device_ptr, direction_device_ptr, grad_weights_ptr,
                                                                       grad_offsets_ptr, grad_targets_ptr, stream))

    def implicit_direction_device(self, params_device_ptr: int, grad_params_device_ptr: int, direction_ptr: int, jacobian_direction_ptr: int = 0,
                                  residual_ptr: int = 0, gradient_rms_ptr: int = 0, stream: int = 0):
        """The direction of solve_ik's implicit-function backward per instance: v = (2 J_E^T J_E)^+ g [B][n] (0 on disabled
        parameters), J v and the residual [B][jacobian_rows] and the gradient RMS [B], from parameters and dLoss/dtheta [B][n]; float32
        device memory (0 = skip that output; the direction is required), enqueued on ``stream``."""
        self._check(self._L.mb2_solver_function_implicit_direction_device(self._h, params_device_ptr, grad_params_device_ptr, direction_ptr,
                                                                          jacobian_direction_ptr, residual_ptr, gradient_rms_ptr, stream))

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

    def get_input_gradient_launch(self) -> dict:
        """What ``input_gradients_device`` launches over this handle's batch, as ``DeviceCharacter.get_instance_launch`` reports it."""
        out = (C.c_int64 * 6)()
        self._check(self._L.mb2_solver_function_get_input_gradient_launch(self._h, out))
        return _instance_launch(out)


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
        r, ptrs = _results(self.fn.batch)
        self._check(self._L.mb2_solver_solve(self._h, p.ctypes.data, *ptrs))
        return {"params": p, **r}

    def solve_host_pointer(self, host_ptr: int, results: bool = False):
        """Same through a raw (e.g. pinned) host pointer; per-instance results returned when ``results`` (one mb2_solver_solve call),
        else via get_results()."""
        if not results:
            self._check(self._L.mb2_solver_solve(self._h, host_ptr, None, None, None))
            return None
        r, ptrs = _results(self.fn.batch)
        self._check(self._L.mb2_solver_solve(self._h, host_ptr, *ptrs))
        return r

    def solve_host_pointer_async(self, host_ptr: int):
        """mb2_solver_solve_async: H2D of the parameters, the solve and the D2H of the result are enqueued on the handle's stream; the
        (pinned) buffer belongs to the library until wait()."""
        self._check(self._L.mb2_solver_solve_async(self._h, host_ptr))

    def wait(self):
        """mb2_solver_wait: blocks until the asynchronous solve is done; per-instance results."""
        r, ptrs = _results(self.fn.batch)
        self._check(self._L.mb2_solver_wait(self._h, *ptrs))
        return r

    def solve_device(self, device_ptr: int, stream: int = 0):
        self._check(self._L.mb2_solver_solve_device(self._h, device_ptr, stream))

    def get_results(self):
        r, ptrs = _results(self.fn.batch)
        self._check(self._L.mb2_solver_get_results(self._h, *ptrs))
        return r

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
                       "qr_max_chunk_rows", "qr_chunks", "qr_widest_chunk", "tr_r_floats", "fused_groups", "fused_smem", "slices"]

    def get_solve_path(self) -> dict:
        """The linear-solve path of the last solve (mb2_solver_get_solve_path): kind as a name (None before the first solve), the
        plan request, the resolved JtJ mode, the launch variants of the kernels it runs and the instance slices it ran as."""
        out = (C.c_int64 * 16)()
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
        r, ptrs = _results(N)
        self._check(self._L.mb2_mixed_batch_get_results(self._h, theta.ctypes.data_as(_fp), offs.ctypes.data_as(_lp), *ptrs))
        return {"params": [theta[offs[i]:offs[i + 1]] for i in range(N)], **r}

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
        r, ptrs = _results(self.total_batch)
        self._check(self._L.mb2_sharded_solver_solve(self._h, p.ctypes.data, *ptrs))
        return {"params": p, **r, "aggregate": self.get_aggregate()}

    def solve_host_pointer(self, host_ptr: int):
        """In place on a raw (pinned) host buffer [total_batch][n]; the aggregate via get_aggregate()."""
        self._check(self._L.mb2_sharded_solver_solve(self._h, host_ptr, None, None, None))

    def get_aggregate(self):
        agg = (C.c_double * 3)()
        self._check(self._L.mb2_sharded_solver_get_aggregate(self._h, agg))
        return {"error_sum": agg[0], "iterations": int(agg[1]), "instances_ok": int(agg[2])}
