"""The skeleton-state family on the device: apply_parameter_transform, joint_parameters_to_skeleton_state,
joint_parameters_to_local_skeleton_state, model_parameters_to_local_skeleton_state, local_skeleton_state_to_joint_parameters and
skeleton_state_to_joint_parameters, forward and backward, against float64 torch restatements of pymomentum's compositions.

The reference gradient is float64 autograd through those restatements. Per instance, a forward passes when its error is at most
K_FWD[op]: translations relative to max(1, the instance's largest |t|), angles compared on the circle, quaternions, scales and log2
scales absolutely. A backward passes when ||g - g64||_inf <= K_BWD[op] * max(||g64||_inf, 1). The inputs keep |ry| <= 1.2 rad, away
from gimbal lock, where the Euler extraction is ill-conditioned. Each K is pinned at about four times the worst value measured over
the fixtures and seeds (emulator / H100 80GB HBM3 at a 700 W power limit, in the comments); the self-checks show that the bounds reject a
global-inverse backward that drops the children's terms, swapped rx and rz, and a missing ln 2.
"""
import ctypes
import math

import numpy as np
import pytest
import torch

from momentum_b200 import character as mc
from momentum_b200 import solver as ms
from tests import emu_lib
from tests.test_skeleton_state import FIXTURES, _fk64, _pt_dense, _qmul, _inputs

OPS = ["apply_parameter_transform", "joint_parameters_to_local_skeleton_state", "local_skeleton_state_to_joint_parameters",
       "skeleton_state_to_joint_parameters", "joint_parameters_to_skeleton_state"]
EMU_OP = {name: i for i, name in enumerate(OPS)}

# worst measured error over the fixtures and seeds, emulator / H100 -> the pinned bound, about four times the larger
K_FWD = {
    "apply_parameter_transform": 1.2e-7,                # 2.98e-8 / 2.98e-8
    "joint_parameters_to_local_skeleton_state": 8e-7,   # 1.62e-7 / 2.01e-7
    "local_skeleton_state_to_joint_parameters": 3.6e-6, # 8.88e-7 / 7.56e-7
    "skeleton_state_to_joint_parameters": 4.7e-6,       # 1.12e-6 / 1.17e-6
    "joint_parameters_to_skeleton_state": 1.2e-5,       # 2.51e-6 / 2.86e-6
}
K_BWD = {
    "apply_parameter_transform": 1.8e-7,                # 4.10e-8 / 4.40e-8
    "joint_parameters_to_local_skeleton_state": 1.1e-6, # 2.05e-7 / 2.75e-7
    "local_skeleton_state_to_joint_parameters": 3.5e-6, # 8.62e-7 / 7.52e-7
    "skeleton_state_to_joint_parameters": 1e-5,         # 2.32e-6 / 2.55e-6
    "joint_parameters_to_skeleton_state": 8e-6,         # 1.92e-6 / 1.95e-6
}


# ---- inputs --------------------------------------------------------------------------------------------------------------------------
def _joint_params(ch, B, seed, ry_max=1.2, angle_max=3.0):
    """[B, J, 7] float64: translations in +-0.5, rx and rz in +-angle_max, ry in +-ry_max, log2 scales in +-0.3"""
    rng = np.random.default_rng(seed)
    J = ch.num_joints
    p = np.empty((B, J, 7))
    p[..., :3] = rng.uniform(-0.5, 0.5, (B, J, 3))
    p[..., 3] = rng.uniform(-angle_max, angle_max, (B, J))
    p[..., 4] = rng.uniform(-ry_max, ry_max, (B, J))
    p[..., 5] = rng.uniform(-angle_max, angle_max, (B, J))
    p[..., 6] = rng.uniform(-0.3, 0.3, (B, J))
    return p


def _denormalise(st, seed):
    """quaternions scaled by 1 +- 1e-3: the inverses take slightly non-unit states as they come"""
    rng = np.random.default_rng(seed)
    st = st.copy()
    st[..., 3:7] *= 1.0 + rng.uniform(-1e-3, 1e-3, st.shape[:-1] + (1,))
    return st


def _input(ch, name, B, seed):
    """[B, in_numel] float32 input of the operation"""
    J = ch.num_joints
    if name == "apply_parameter_transform":
        return _inputs(ch, B, seed)[0]
    jp = _joint_params(ch, B, seed)
    if name in ("joint_parameters_to_local_skeleton_state", "joint_parameters_to_skeleton_state"):
        return jp.reshape(B, 7 * J).astype(np.float32)
    if name == "local_skeleton_state_to_joint_parameters":
        st = _local64(ch, torch.from_numpy(jp)).numpy()
    else:
        st = _fk64(ch, torch.from_numpy(jp)).numpy()
    return _denormalise(st, seed + 1).reshape(B, 8 * J).astype(np.float32)


def _out_numel(ch, name):
    J = ch.num_joints
    return 8 * J if name in ("joint_parameters_to_local_skeleton_state", "joint_parameters_to_skeleton_state") else 7 * J


# ---- float64 restatements of pymomentum's compositions -------------------------------------------------------------------------------
def _prerot(ch):
    return torch.from_numpy(ch.prerot.astype(np.float64))


def _offsets(ch):
    return torch.from_numpy(ch.offsets.astype(np.float64))


def _local64(ch, jp):
    """jp [B, J, 7] -> local states [B, J, 8]: the local part of _fk64 (joint_state.cpp:44-62)"""
    B, J = jp.shape[:2]
    ql = _prerot(ch).expand(B, J, 4)
    zero = torch.zeros_like(jp[..., 0])
    for k in (2, 1, 0):
        h = 0.5 * jp[..., 3 + k]
        c = [zero, zero, zero, torch.cos(h)]
        c[k] = torch.sin(h)
        ql = _qmul(ql, torch.stack(c, -1))
    return torch.cat([_offsets(ch) + jp[..., :3], ql, torch.exp2(jp[..., 6:7])], -1)


def _qinverse(q):  # quaternionInverse (tensor_quaternion.cpp:209)
    return torch.cat([-q[..., :3], q[..., 3:]], -1) / (q * q).sum(-1, keepdim=True)


def _rotate(q, v):  # quaternionRotateVector (tensor_quaternion.cpp:226)
    av = torch.linalg.cross(q[..., :3], v)
    return v + 2 * (av * q[..., 3:4] + torch.linalg.cross(q[..., :3], av))


def _euler(q, swap=False):  # quaternionToXYZEuler (tensor_quaternion.cpp:213), the asin argument clamped
    x, y, z, w = q.unbind(-1)
    rx = torch.atan2(2 * (w * x + y * z), 1 - 2 * (x * x + y * y))
    ry = torch.asin((2 * (w * y - z * x)).clamp(-1.0, 1.0))
    rz = torch.atan2(2 * (w * z + x * y), 1 - 2 * (y * y + z * z))
    return torch.stack([rz, ry, rx] if swap else [rx, ry, rz], -1)


def _from_local64(ch, ls, swap=False):
    """local states [B, J, 8] -> [B, J, 7] (localSkeletonStateToJointParameters, tensor_skeleton_state.cpp:611-648)"""
    pre = _prerot(ch).expand(ls.shape[:-1] + (4,))
    return torch.cat([ls[..., :3] - _offsets(ch), _euler(_qmul(_qinverse(pre), ls[..., 3:7]), swap), torch.log2(ls[..., 7:8])], -1)


def _world_to_local64(ch, X, detach_parent=False):
    """inv(X_parent) o X_j with the identity above a root (skeletonStateToJointParameters, :650-668)"""
    ident = torch.zeros_like(X[:, :1])
    ident[..., 6] = 1.0
    ident[..., 7] = 1.0
    parents = torch.from_numpy(ch.parents.astype(np.int64) + 1)
    P = torch.cat([ident, X], 1)[:, parents]
    if detach_parent:
        P = P.detach()
    qi, si = _qinverse(P[..., 3:7]), 1.0 / P[..., 7:8]
    ti = -si * _rotate(qi, P[..., :3])
    return torch.cat([ti + _rotate(qi, si * X[..., :3]), _qmul(qi, X[..., 3:7]), si * X[..., 7:8]], -1)


def _ref64(ch, name, x, variant=None):
    """the operation on x [B, in_numel] float64 -> [B, out_numel]"""
    B, J = x.shape[0], ch.num_joints
    if name == "apply_parameter_transform":
        return x @ _pt_dense(ch).T + torch.from_numpy(ch.pt_offsets.astype(np.float64))
    if name == "joint_parameters_to_skeleton_state":
        return _fk64(ch, x.reshape(B, J, 7)).reshape(B, -1)
    if name == "joint_parameters_to_local_skeleton_state":
        return _local64(ch, x.reshape(B, J, 7)).reshape(B, -1)
    st = x.reshape(B, J, 8)
    if name == "skeleton_state_to_joint_parameters":
        st = _world_to_local64(ch, st, detach_parent=variant == "no_children")
    return _from_local64(ch, st, swap=variant == "swap").reshape(B, -1)


def _grad64(ch, name, x, G, variant=None):
    x = torch.from_numpy(np.asarray(x, np.float64)).requires_grad_(True)
    (_ref64(ch, name, x, variant) * torch.from_numpy(np.asarray(G, np.float64))).sum().backward()
    return x.grad.numpy()


# ---- error measures ------------------------------------------------------------------------------------------------------------------
def _wrap(d):
    return np.abs(np.arctan2(np.sin(d), np.cos(d)))


def _forward_error(ch, name, x, out, ref):
    """per instance: the error of out against ref [B, out_numel] under the measures of the module docstring"""
    B, J = x.shape[0], ch.num_joints
    out, ref = np.asarray(out, np.float64), np.asarray(ref, np.float64)
    if name == "apply_parameter_transform":
        return np.abs(out - ref).max(1) / np.maximum(np.abs(ref).max(1), 1.0)
    if out.shape[1] == 8 * J:  # states
        o, r = out.reshape(B, J, 8), ref.reshape(B, J, 8)
        scale = np.maximum(np.abs(r[..., :3]).max((1, 2)), 1.0)
        return np.maximum(np.abs(o[..., :3] - r[..., :3]).max((1, 2)) / scale, np.abs(o[..., 3:] - r[..., 3:]).max((1, 2)))
    o, r = out.reshape(B, J, 7), ref.reshape(B, J, 7)
    scale = np.maximum(np.abs(np.asarray(x, np.float64).reshape(B, J, 8)[..., :3]).max((1, 2)), 1.0)
    et = np.abs(o[..., :3] - r[..., :3]).max((1, 2)) / scale
    return np.maximum(et, np.maximum(_wrap(o[..., 3:6] - r[..., 3:6]).max((1, 2)), np.abs(o[..., 6] - r[..., 6]).max(1)))


def _bound_ratio(g, g64):
    g, g64 = np.asarray(g, np.float64), np.asarray(g64, np.float64)
    return np.abs(g - g64).max(axis=1) / np.maximum(np.abs(g64).max(axis=1), 1.0)


# ---- the two implementations: the CPU emulator and the device through the torch wrappers ----------------------------------------------
# the entry of tests/emu/emu_joint_parameters.cu (the nine character values, op, backward, batch, in, grad, out), declared here next to
# the only tests that call it
_EMU_SIGNATURE = [ctypes.c_int32, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int32] + [ctypes.c_void_p] * 4 + \
    [ctypes.c_int32] * 3 + [ctypes.c_void_p] * 3


@pytest.fixture(scope="module")
def emu():
    L = emu_lib.load()
    L.emu_joint_parameters.argtypes = _EMU_SIGNATURE
    return L


def _emu_run(L, ch, name, x, G=None):
    """forward: op(x) [B, out_numel]; backward (G given): dLoss / dx [B, in_numel]"""
    keep = []
    x = np.ascontiguousarray(x, np.float32)
    B = x.shape[0]
    out = np.full((B, x.shape[1] if G is not None else _out_numel(ch, name)), np.nan, np.float32)
    g = np.ascontiguousarray(G, np.float32) if G is not None else None
    rc = L.emu_joint_parameters(*emu_lib.character_args(ch, keep), EMU_OP[name], int(G is not None), B, x.ctypes.data,
                                g.ctypes.data if g is not None else None, out.ctypes.data)
    assert rc == 0, L.emu_last_error().decode()
    return out


def _wrapper(name):
    from momentum_b200 import torch_skeleton as tsk

    return getattr(tsk, name)


def _dev_in(ch, name, x):
    J = ch.num_joints
    x = torch.from_numpy(np.ascontiguousarray(x, np.float32)).cuda()
    return x.reshape(-1, J, 8) if name.endswith("to_joint_parameters") else x


def _dev_run(ch, name, x, G=None):
    xd = _dev_in(ch, name, x).requires_grad_(G is not None)
    out = _wrapper(name)(ch, xd)
    if G is None:
        return out.reshape(x.shape[0], -1).cpu().numpy()
    out.backward(torch.from_numpy(np.ascontiguousarray(G, np.float32)).cuda().reshape(out.shape))
    return xd.grad.reshape(x.shape[0], -1).cpu().numpy()


def _measure(run, ch, name, B, seed):
    x = _input(ch, name, B, seed)
    G = np.random.default_rng(seed + 7).normal(size=(B, _out_numel(ch, name))).astype(np.float32)
    ref = _ref64(ch, name, torch.from_numpy(x.astype(np.float64))).detach().numpy()
    fwd = _forward_error(ch, name, x, run(ch, name, x), ref)
    bwd = _bound_ratio(run(ch, name, x, G), _grad64(ch, name, x, G))
    return fwd.max(), bwd.max()


# ---- CPU ---------------------------------------------------------------------------------------------------------------------------
def test_restatements_agree_with_the_forward_kinematics():
    """_local64 composed level by level is _fk64, and skeleton_state_to_joint_parameters of _fk64 gives back the joint parameters (with
    the pre-rotations normalised in float64: the inverse rotation as written undoes a rotation only for unit quaternions)"""
    for name, make in FIXTURES.items():
        ch = make()
        ch.prerot = ch.prerot.astype(np.float64) / np.linalg.norm(ch.prerot.astype(np.float64), axis=1, keepdims=True)
        jp = torch.from_numpy(_joint_params(ch, 3, 1, ry_max=1.4, angle_max=3.0))
        X = _fk64(ch, jp)
        back = _ref64(ch, "skeleton_state_to_joint_parameters", X.reshape(3, -1)).reshape(jp.shape)
        assert (back - jp).abs().max().item() <= 1e-9, name
        loc = _local64(ch, jp)
        assert (_from_local64(ch, loc) - jp).abs().max().item() <= 1e-12, name
        assert (_world_to_local64(ch, X) - loc).abs().max().item() <= 1e-9 * max(1.0, X[..., :3].abs().max().item()), name


@pytest.mark.parametrize("name", OPS)
@pytest.mark.parametrize("fixture", list(FIXTURES))
def test_emulated_operation_meets_the_float64_bounds(emu, name, fixture):
    ch = FIXTURES[fixture]()
    fwd, bwd = _measure(lambda *a: _emu_run(emu, *a), ch, name, 4, 31)
    assert fwd <= K_FWD[name], (fixture, name, fwd)
    assert bwd <= K_BWD[name], (fixture, name, bwd)


def test_bounds_reject_a_wrong_backward():
    """dropping the children's terms of the global inverse, swapping rx and rz, and dropping ln 2 each fail by far more than the bound"""
    for fixture in ("chain6", "humanoid72", "humanoid72_far", "two_roots"):
        ch = FIXTURES[fixture]()
        B = 4
        for name in ("skeleton_state_to_joint_parameters", "local_skeleton_state_to_joint_parameters"):
            x = _input(ch, name, B, 41)
            G = np.random.default_rng(42).normal(size=(B, 7 * ch.num_joints))
            g64 = _grad64(ch, name, x, G)
            if name == "skeleton_state_to_joint_parameters":
                assert _bound_ratio(_grad64(ch, name, x, G, "no_children"), g64).min() > 100 * K_BWD[name], fixture
            assert _bound_ratio(_grad64(ch, name, x, G, "swap"), g64).min() > 100 * K_BWD[name], (fixture, name)
            no_ln2 = g64.reshape(B, -1, 8).copy()
            no_ln2[..., 7] *= math.log(2.0)  # d log2 s / ds taken as 1 / s
            assert _bound_ratio(no_ln2.reshape(B, -1), g64).min() > 100 * K_BWD[name], (fixture, name)
        name = "joint_parameters_to_local_skeleton_state"
        x = _input(ch, name, B, 43)
        G = np.random.default_rng(44).normal(size=(B, 8 * ch.num_joints))
        g64 = _grad64(ch, name, x, G)
        no_ln2 = g64.reshape(B, -1, 7).copy()
        no_ln2[..., 6] /= math.log(2.0)  # d 2^p / dp taken as 2^p
        assert _bound_ratio(no_ln2.reshape(B, -1), g64).min() > 100 * K_BWD[name], fixture


def _same_rotation_error(q, r):
    """per instance max over joints of min(|q - r|, |q + r|) for [B, J, 4]"""
    return np.minimum(np.abs(q - r).max(-1), np.abs(q + r).max(-1)).max(-1)


@pytest.mark.parametrize("fixture", list(FIXTURES))
def test_emulated_round_trips(emu, fixture):
    """state -> joint parameters -> state reproduces the state for any angles; joint parameters -> state -> joint parameters
    reproduces the parameters inside the principal range"""
    ch = FIXTURES[fixture]()
    B, J = 4, ch.num_joints
    jp = _joint_params(ch, B, 51, ry_max=math.pi, angle_max=math.pi)  # any angles
    X = _fk64(ch, torch.from_numpy(jp)).numpy().astype(np.float32)
    back = _emu_run(emu, ch, "skeleton_state_to_joint_parameters", X.reshape(B, -1))
    X2 = _emu_run(emu, ch, "joint_parameters_to_skeleton_state", back).reshape(B, J, 8)
    scale = np.maximum(np.abs(X[..., :3]).max((1, 2)), 1.0)
    # any angles include ry within a few 1e-3 of +-pi/2, where the Euler angles amplify rounding by 1 / cos(ry)
    assert (np.abs(X2[..., :3] - X[..., :3]).max((1, 2)) / scale).max() <= 2e-4
    assert _same_rotation_error(X2[..., 3:7], X[..., 3:7]).max() <= 2e-4
    assert np.abs(X2[..., 7] - X[..., 7]).max() <= 1e-5
    L = _emu_run(emu, ch, "joint_parameters_to_local_skeleton_state", back).reshape(B, J, 8)
    back_l = _emu_run(emu, ch, "local_skeleton_state_to_joint_parameters", L.reshape(B, -1))
    L2 = _emu_run(emu, ch, "joint_parameters_to_local_skeleton_state", back_l).reshape(B, J, 8)
    assert np.abs(L2[..., :3] - L[..., :3]).max() <= 1e-5 and np.abs(L2[..., 7] - L[..., 7]).max() <= 1e-5
    assert _same_rotation_error(L2[..., 3:7], L[..., 3:7]).max() <= 2e-4
    jp = _joint_params(ch, B, 52, ry_max=math.pi / 2 - 0.05, angle_max=math.pi - 0.05).reshape(B, -1).astype(np.float32)
    for fwd, inv in (("joint_parameters_to_skeleton_state", "skeleton_state_to_joint_parameters"),
                     ("joint_parameters_to_local_skeleton_state", "local_skeleton_state_to_joint_parameters")):
        again = _emu_run(emu, ch, inv, _emu_run(emu, ch, fwd, jp)).reshape(B, J, 7)
        ref = jp.reshape(B, J, 7)
        assert np.abs(again[..., :3] - ref[..., :3]).max() <= 2e-4 * max(1.0, np.abs(X[..., :3]).max()), (fixture, fwd)
        assert _wrap(again[..., 3:6] - ref[..., 3:6]).max() <= 2e-3, (fixture, fwd)
        assert np.abs(again[..., 6] - ref[..., 6]).max() <= 1e-5, (fixture, fwd)


def _gimbal_character():
    ch = mc.create_test_character(3)
    ch.prerot = np.tile(np.array([0, 0, 0, 1], np.float32), (ch.num_joints, 1))
    return ch


def _gimbal_quaternions():
    """float32 (a, b) near 1/sqrt(2) with 2 fl(a b) == 1 exactly and == 1 + 2^-23: q = (0, a, 0, b) is at gimbal lock (ry = pi/2), and
    just past it, in the arithmetic of the Euler extraction (with an identity pre-rotation r is q bit for bit)"""
    c = np.float32(1 / math.sqrt(2))
    near = [np.nextafter(c, np.float32(k), dtype=np.float32) for k in (0, 2)] + [c]
    near += [np.nextafter(v, np.float32(2), dtype=np.float32) for v in near]
    found = {}
    for a in near:
        for b in near:
            A = np.float32(2) * np.float32(a * b)
            for key, want in (("exact", np.float32(1)), ("past", np.nextafter(np.float32(1), np.float32(2), dtype=np.float32))):
                if A == want:
                    found.setdefault(key, (a, b))
    assert set(found) == {"exact", "past"}, found
    return found


def _gimbal_checks(run, ch):
    J = ch.num_joints
    for key, (a, b) in _gimbal_quaternions().items():
        for name in ("local_skeleton_state_to_joint_parameters", "skeleton_state_to_joint_parameters"):
            st = np.zeros((1, J, 8), np.float32)
            st[..., 6] = 1.0
            st[..., 7] = 1.0
            st[0, 0, 3:7] = (0.0, a, 0.0, b)  # the root: its local state is its world state
            jp = run(ch, name, st.reshape(1, -1))
            assert np.all(np.isfinite(jp)), (key, name)
            assert abs(jp[0, 4] - math.pi / 2) <= 1e-6, (key, name, jp[0, :7])
            G = np.zeros((1, 7 * J), np.float32)
            G[0, 4] = 1.0  # ry of the root only
            g = run(ch, name, st.reshape(1, -1), G)
            assert np.all(g == 0.0), (key, name, g[0, :8])
            again = run(ch, "joint_parameters_to_local_skeleton_state", jp).reshape(1, J, 8)
            q = st[0, 0, 3:7] / np.linalg.norm(st[0, 0, 3:7])
            assert _same_rotation_error(again[:, :1, 3:7], q[None, None]).max() <= 1e-6, (key, name)


def test_emulated_gimbal_lock_is_finite_with_a_zero_ry_derivative(emu):
    _gimbal_checks(lambda *a: _emu_run(emu, *a), _gimbal_character())


def test_cpu_tensors_and_bad_shapes_are_rejected_before_any_library_call(monkeypatch):
    from momentum_b200 import torch_skeleton as tsk

    def no_call(*a, **k):
        raise AssertionError("library reached")

    monkeypatch.setattr(ms, "load_library", no_call)
    monkeypatch.setattr(ms, "DeviceCharacter", type("NoDevice", (), {"__init__": no_call}))
    ch = mc.create_test_character(4)
    n, J = ch.num_params, ch.num_joints
    good = {"apply_parameter_transform": (n,), "joint_parameters_to_skeleton_state": (7 * J,),
            "joint_parameters_to_local_skeleton_state": (7 * J,), "model_parameters_to_local_skeleton_state": (n,),
            "local_skeleton_state_to_joint_parameters": (J, 8), "skeleton_state_to_joint_parameters": (J, 8)}
    for name, shape in good.items():
        fn = getattr(tsk, name)
        with pytest.raises(ValueError, match="CUDA"):
            fn(ch, torch.zeros(shape))
        with pytest.raises(ValueError, match="CUDA"):
            fn(ch, torch.zeros((2,) + shape, dtype=torch.float64))
        bad = (shape[0] + 1,) + shape[1:]
        with pytest.raises(ValueError, match=r"must be \[.*\] or \[B, .*\], got"):
            fn(ch, torch.zeros(bad))
        with pytest.raises(ValueError, match=r"must be \[.*\] or \[B, .*\], got"):
            fn(ch, torch.zeros((2, 3) + shape))
    with pytest.raises(ValueError, match=r"\[7 J = 28\]|7 J = 28"):
        tsk.joint_parameters_to_skeleton_state(ch, torch.zeros(J, 7))  # the [J, 7] layout is not taken: flatten(-2) first


# ---- GPU --------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", OPS)
@pytest.mark.parametrize("fixture", list(FIXTURES))
def test_device_operation_meets_the_float64_bounds(name, fixture):
    ch = FIXTURES[fixture]()
    fwd, bwd = _measure(_dev_run, ch, name, 8, 61)
    assert fwd <= K_FWD[name], (fixture, name, fwd)
    assert bwd <= K_BWD[name], (fixture, name, bwd)


@pytest.mark.gpu
def test_device_gimbal_lock_is_finite_with_a_zero_ry_derivative():
    _gimbal_checks(_dev_run, _gimbal_character())


@pytest.mark.gpu
@pytest.mark.parametrize("fixture", list(FIXTURES))
def test_joint_parameter_fk_agrees_with_the_model_parameter_fk(fixture):
    """joint_parameters_to_skeleton_state(apply_parameter_transform(theta)) against model_parameters_to_skeleton_state(theta): within
    the FK bound of tests/test_skeleton_state.py, and reported bitwise (both paths sum the rows of P theta + o with jointParameterRow;
    forward and backward were bitwise equal on every fixture on an H100, but the test does not require it)"""
    from momentum_b200 import torch_skeleton as tsk

    ch = FIXTURES[fixture]()
    theta, G = _inputs(ch, 16, 71)
    th = torch.from_numpy(theta).cuda().requires_grad_(True)
    a = tsk.joint_parameters_to_skeleton_state(ch, tsk.apply_parameter_transform(ch, th))
    a.backward(torch.from_numpy(G).cuda())
    ga = th.grad.clone()
    th.grad = None
    b = tsk.model_parameters_to_skeleton_state(ch, th)
    b.backward(torch.from_numpy(G).cuda())
    ref = b.detach().cpu().numpy()
    assert np.abs(a.detach().cpu().numpy() - ref).max() <= 2e-5 * max(1.0, np.abs(ref).max())
    assert _bound_ratio(ga.cpu().numpy(), th.grad.cpu().numpy()).max() <= 7e-6
    print(f"{fixture}: forward bitwise {torch.equal(a, b)}, backward bitwise {torch.equal(ga, th.grad)}")


@pytest.mark.gpu
@pytest.mark.parametrize("fixture", list(FIXTURES))
def test_end_to_end_round_trip_and_gradient(fixture):
    """skeleton_state_to_joint_parameters(model_parameters_to_skeleton_state(theta)).flatten(-2) ~ apply_parameter_transform(theta)
    with theta in the principal range, and the gradient of sum(G * that composition) ~ P^T G: every backward chain at once"""
    from momentum_b200 import torch_skeleton as tsk

    ch = FIXTURES[fixture]()
    B, J = 8, ch.num_joints
    theta = np.random.default_rng(81).uniform(-0.4, 0.4, (B, ch.num_params)).astype(np.float32)
    th = torch.from_numpy(theta).cuda().requires_grad_(True)
    jp = tsk.skeleton_state_to_joint_parameters(ch, tsk.model_parameters_to_skeleton_state(ch, th)).flatten(-2)
    ref64 = _ref64(ch, "apply_parameter_transform", torch.from_numpy(theta.astype(np.float64))).numpy()
    assert np.abs(ref64.reshape(B, J, 7)[..., 3:6]).max() < math.pi / 2  # inside the principal range
    scale = np.maximum(np.abs(_fk64(ch, torch.from_numpy(ref64.reshape(B, J, 7))).numpy()[..., :3]).max((1, 2)), 1.0)
    err = np.abs(jp.detach().cpu().numpy() - ref64).reshape(B, J, 7)
    assert (err[..., :3].max((1, 2)) / scale).max() <= 1e-5 and err[..., 3:].max() <= 1e-4, err.max()
    G = np.random.default_rng(82).normal(size=(B, 7 * J)).astype(np.float32)
    (jp * torch.from_numpy(G).cuda()).sum().backward()
    want = G.astype(np.float64) @ _pt_dense(ch).numpy()
    assert _bound_ratio(th.grad.cpu().numpy(), want).max() <= 1e-4, _bound_ratio(th.grad.cpu().numpy(), want).max()


def _raw(dc, name, backward, x, g=None, out_numel=None):
    stream = torch.cuda.current_stream().cuda_stream
    B = x.shape[0]
    if not backward:
        out = torch.empty(B, out_numel, device="cuda")
        dc.joint_op_device(name, False, B, x.data_ptr(), out.data_ptr(), stream=stream)
    else:
        out = torch.empty(B, x.shape[1], device="cuda")
        ptrs = (g.data_ptr(), out.data_ptr()) if name == "apply_parameter_transform" else (x.data_ptr(), g.data_ptr(), out.data_ptr())
        dc.joint_op_device(name, True, B, *ptrs, stream=stream)
    return out


@pytest.mark.gpu
def test_batch_independence_and_determinism():
    """one instance alone and inside a batch of several waves give identical bits, and two runs give identical bits"""
    from momentum_b200 import torch_skeleton as tsk

    ch = mc.humanoid72()[0]
    B = 8192 + 37
    dc = tsk._device_character(ch, torch.device("cuda", 0))
    for name in OPS:
        x = torch.from_numpy(_input(ch, name, B, 91)).cuda()
        g = torch.from_numpy(np.random.default_rng(92).normal(size=(B, _out_numel(ch, name))).astype(np.float32)).cuda()
        f1, f2 = _raw(dc, name, False, x, out_numel=g.shape[1]), _raw(dc, name, False, x, out_numel=g.shape[1])
        b1, b2 = _raw(dc, name, True, x, g), _raw(dc, name, True, x, g)
        assert torch.equal(f1, f2) and torch.equal(b1, b2), name
        for b in (0, 1, B // 2, B - 38, B - 1):
            assert torch.equal(_raw(dc, name, False, x[b:b + 1].contiguous(), out_numel=g.shape[1]), f1[b:b + 1]), (name, b)
            assert torch.equal(_raw(dc, name, True, x[b:b + 1].contiguous(), g[b:b + 1].contiguous()), b1[b:b + 1]), (name, b)


@pytest.mark.gpu
def test_torch_wrappers_shapes_dtypes_streams_and_errors():
    from momentum_b200 import torch_skeleton as tsk

    ch = mc.humanoid72()[0]
    n, J = ch.num_params, ch.num_joints
    dev = torch.device("cuda", 0)
    theta = torch.from_numpy(_inputs(ch, 3, 101)[0]).to(dev)
    # shapes and dtypes, batched and not
    jp = tsk.apply_parameter_transform(ch, theta.double())
    assert jp.shape == (3, 7 * J) and jp.dtype == torch.float64
    assert tsk.apply_parameter_transform(ch, theta[1]).shape == (7 * J,)
    for fn in (tsk.joint_parameters_to_skeleton_state, tsk.joint_parameters_to_local_skeleton_state):
        st = fn(ch, jp)
        assert st.shape == (3, J, 8) and st.dtype == torch.float64
        assert torch.equal(fn(ch, jp[1].float()), st[1].float())
    loc = tsk.model_parameters_to_local_skeleton_state(ch, theta)
    assert loc.shape == (3, J, 8) and torch.equal(loc, tsk.joint_parameters_to_local_skeleton_state(ch, tsk.apply_parameter_transform(ch, theta)))
    st = tsk.model_parameters_to_skeleton_state(ch, theta)
    for fn, x in ((tsk.skeleton_state_to_joint_parameters, st), (tsk.local_skeleton_state_to_joint_parameters, loc)):
        out = fn(ch, x.double())
        assert out.shape == (3, J, 7) and out.dtype == torch.float64
        assert torch.equal(fn(ch, x[2]), fn(ch, x)[2])
    # gradients come back in the input's shape and dtype; batch 0
    x = st.double().requires_grad_(True)
    tsk.skeleton_state_to_joint_parameters(ch, x).sum().backward()
    assert x.grad.shape == (3, J, 8) and x.grad.dtype == torch.float64
    t0 = torch.zeros(0, n, device=dev, requires_grad=True)
    out0 = tsk.skeleton_state_to_joint_parameters(ch, tsk.model_parameters_to_local_skeleton_state(ch, t0))
    assert out0.shape == (0, J, 7)
    out0.sum().backward()
    assert t0.grad.shape == (0, n)
    # a non-default current stream gives the same bits
    def chain(t):
        t = t.clone().requires_grad_(True)
        out = tsk.local_skeleton_state_to_joint_parameters(ch, tsk.model_parameters_to_local_skeleton_state(ch, t))
        out = out + tsk.skeleton_state_to_joint_parameters(ch, tsk.joint_parameters_to_skeleton_state(ch, tsk.apply_parameter_transform(ch, t)))
        out.backward(torch.ones_like(out))
        return out.detach(), t.grad
    ref = chain(theta)
    side = torch.cuda.Stream(dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side):
        got = chain(theta)
    torch.cuda.current_stream(dev).wait_stream(side)
    torch.cuda.synchronize(dev)
    assert torch.equal(got[0], ref[0]) and torch.equal(got[1], ref[1])
    # errors
    with pytest.raises(ValueError, match="must be"):
        tsk.skeleton_state_to_joint_parameters(ch, torch.zeros(3, J + 1, 8, device=dev))
    with pytest.raises(ValueError, match="must be"):
        tsk.joint_parameters_to_skeleton_state(ch, torch.zeros(3, J, 7, device=dev))
    dc = ms.DeviceCharacter(ch, 0)
    dc.device = 1  # a handle that belongs to another device than the tensor
    with pytest.raises(ValueError, match="device character"):
        tsk.apply_parameter_transform(dc, theta)
    dc.device = 0
    assert torch.equal(tsk.apply_parameter_transform(dc, theta), tsk.apply_parameter_transform(ch, theta))


@pytest.mark.gpu
def test_c_abi_rejects_bad_arguments():
    ch = mc.create_test_character(4)
    dc = ms.DeviceCharacter(ch, 0)
    n, J = ch.num_params, ch.num_joints
    th = torch.zeros(2, n, device="cuda")
    jp = torch.zeros(2, 7 * J, device="cuda")
    st = torch.zeros(2, J, 8, device="cuda")
    host = np.zeros((2, 8 * J), np.float32)
    for name in OPS:
        x = th if name == "apply_parameter_transform" else (st if name.endswith("to_joint_parameters") else jp)
        y = jp if name in ("apply_parameter_transform",) or name.endswith("to_joint_parameters") else st
        with pytest.raises(ms.MomentumB200Error, match="device memory"):
            dc.joint_op_device(name, False, 2, x.data_ptr(), host.ctypes.data)
        with pytest.raises(ms.MomentumB200Error, match="null"):
            dc.joint_op_device(name, False, 2, 0, y.data_ptr())
        with pytest.raises(ms.MomentumB200Error, match="negative"):
            dc.joint_op_device(name, False, -1, x.data_ptr(), y.data_ptr())
        bwd = (y.data_ptr(), 0) if name == "apply_parameter_transform" else (x.data_ptr(), y.data_ptr(), 0)
        with pytest.raises(ms.MomentumB200Error, match="null"):
            dc.joint_op_device(name, True, 2, *bwd)
        bwd = (host.ctypes.data, x.data_ptr()) if name == "apply_parameter_transform" else (x.data_ptr(), host.ctypes.data, x.data_ptr())
        with pytest.raises(ms.MomentumB200Error, match="device memory"):
            dc.joint_op_device(name, True, 2, *bwd)
        dc.joint_op_device(name, False, 0, 0, 0)  # batch 0: nothing to do
        dc.joint_op_device(name, True, 0, *([0] * len(bwd)))
