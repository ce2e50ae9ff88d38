"""The CPU emulator library, tests/emu/libmb2_emu.so: built by tests/emu/Makefile, opened once per process, with the signature of every
emu_* entry of the operation emulators declared here. Test modules and scripts take it from load(); the modules that drive the emulated
mb2_* C-ABI open EMU_LIB through momentum_b200.solver.load_library after build()."""
import ctypes
import functools
import os
import subprocess

import numpy as np

EMU_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu")
EMU_LIB = os.path.join(EMU_DIR, "libmb2_emu.so")

_i32, _i64, _f32, _p = ctypes.c_int32, ctypes.c_int64, ctypes.c_float, ctypes.c_void_p
_CHARACTER = [_i32, _p, _p, _p, _i32, _p, _p, _p, _p]  # mb2_character_create's arguments
_SKINNING = _CHARACTER + [_i32, _p, _p, _p, _p]  # V, rest vertices, skin index, skin weight, inverse bind poses
_BLEND = _SKINNING + [_i32, _i32, _p, _p]  # K, V, base shape, shape vectors
_SIGNATURES = {
    "emu_skinning_tables": _SKINNING + [_p] * 2,
    "emu_skin_points": _SKINNING + [_i32, _p, _p, _i32, _p],
    "emu_skin_points_backward": _SKINNING + [_i32, _p, _p, _i32] + [_p] * 3,
    "emu_skin_with_blend_shapes": _BLEND + [_i32, _p, _p, _i32, _p],
    "emu_skin_with_blend_shapes_backward": _BLEND + [_i32, _p, _p, _i32] + [_p] * 3,
    "emu_blend_shape_replace": [_i32, _i32, _p, _p] * 2 + [_p],
    "emu_skeleton_state_backward": _CHARACTER + [_i32] + [_p] * 3,
    "emu_input_gradients": _CHARACTER + [_i32, _i32, _i32, _p, _p, _f32, _f32, _p, _i32] + [_p] * 7,
    "emu_implicit_direction": [_i32, _i32] + [_p] * 7,
    "emu_mesh_faces_tables": [_i32, _i32] + [_p] * 3,
    "emu_vertex_normals": [_i32, _i32, _p, _i32, _p, _p],
    "emu_vertex_normals_backward": [_i32, _i32, _p, _i32] + [_p] * 3,
    "emu_mesh_tree": [_i32, _i32, _p, _i32, _p, _p, _p, _p, _p, _p],
    "emu_mesh_tree_boxes": [_i32, _i32, _p, _p, _p, _p],
    "emu_closest_points": [_i32, _i32, _p, _p, _i32, _i32, _p, _p, _f32, _i32, _p, _p, _p, _p],
    "emu_plan_instance_groups": [_i64] * 4 + [_i32, _p],
    "emu_instance_launch": _CHARACTER + [_i32, _i32, _i64, _i32, _i64, _i32, _p],
}


@functools.cache
def build():
    """Bring the library up to date (make compiles only what changed); returns its path."""
    subprocess.check_call(["make", "-C", EMU_DIR, "-s", f"-j{os.cpu_count()}"])
    return EMU_LIB


@functools.cache
def load():
    """The library, built and opened once, emu_last_error() returning the message of the last emu_* entry that failed."""
    L = ctypes.CDLL(build())
    L.emu_last_error.restype = ctypes.c_char_p
    for name, argtypes in _SIGNATURES.items():
        getattr(L, name).argtypes = argtypes
    return L


def character_args(ch, keep):
    """The nine character values in mb2_character_create order; the arrays behind the pointers go to keep, which must outlive the call."""
    arrays = [np.ascontiguousarray(ch.parents, np.int32), np.ascontiguousarray(ch.offsets, np.float32), np.ascontiguousarray(ch.prerot, np.float32),
              np.ascontiguousarray(ch.pt_outer, np.int32), np.ascontiguousarray(ch.pt_inner, np.int32), np.ascontiguousarray(ch.pt_vals, np.float32),
              np.ascontiguousarray(ch.pt_offsets, np.float32)]
    keep.extend(arrays)
    p = [a.ctypes.data for a in arrays]
    return [ch.num_joints] + p[:3] + [ch.num_params] + p[3:]
