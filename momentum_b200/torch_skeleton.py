"""Differentiable forward kinematics on CUDA tensors: ``model_parameters_to_skeleton_state`` and the rest of pymomentum's skeleton-state
family (``apply_parameter_transform`` and its inverse, joint parameters to world and local states, and back, and the positions of
points fixed in joints' frames), then skinning, normals and closest points.

Mirror of ``pymomentum.geometry.model_parameters_to_skeleton_state`` (pymomentum/tensor_momentum/tensor_skeleton_state.cpp:500-502:
``jointParametersToSkeletonState(applyParamTransform(theta))``) for the batched device path. The forward pass is the solver's own FK
device code (``mb2_character_skeleton_state_device``); the backward pass replaces the reference's per-joint ``ceres::Jet`` ancestor
walks (``computeSkelStateBackward``, :62-134) with one reverse sweep over the joint tree and the transposed ParameterTransform
(``mb2_character_skeleton_state_backward_device``). Both run on torch's current stream and never leave the device, so a loss on joint
positions or rotations after ``torch_ik.solve_ik`` back-propagates to the solver's inputs without a host round trip.
"""
from __future__ import annotations

from collections import namedtuple

import numpy as np
import torch
from torch.autograd.function import once_differentiable

from . import character as mc
from . import solver as ms

# The registry entry of one (character, device): the character, kept alive so that its id stays unique; the (skinning, faces, blend
# shape, collision) its DeviceCharacter ``dc`` was made with; and the solver functions ``torch_ik._build`` made on ``dc``.
_Handle = namedtuple("_Handle", "character mesh dc solver_functions")
_handles = {}


def _device_index(device: torch.device) -> int:
    return device.index if device.index is not None else torch.cuda.current_device()


def _handle(character: mc.Character, device: torch.device) -> _Handle:
    """The torch layer's one entry per (character, device). When ``skinning``, its ``faces``, ``blend_shape`` or ``collision`` is replaced, a new entry
    with a new DeviceCharacter is made instead of uploading into the old one: a graph recorded before keeps its handle (``ctx.dc``) and
    tables, and no kernel in flight on another stream reads tables being replaced. The old entry's solver functions go with it."""
    index = _device_index(device)
    entry = _handles.get((id(character), index))
    mesh = (character.skinning, None if character.skinning is None else character.skinning.faces, character.blend_shape, character.collision)
    if entry is None or any(a is not b for a, b in zip(entry.mesh, mesh)):
        entry = _handles[id(character), index] = _Handle(character, mesh, ms.DeviceCharacter(character, index), {})
    return entry


def _device_character(character, device: torch.device) -> ms.DeviceCharacter:
    """The handle every operation here runs on: a DeviceCharacter as given, or for a Character its registry entry's (``_handle``)."""
    if not isinstance(character, ms.DeviceCharacter):
        return _handle(character, device).dc
    if character.device != _device_index(device):
        raise ValueError(f"model parameters are on cuda:{_device_index(device)} but the device character lives on cuda:{character.device}")
    return character


def _stream(device: torch.device) -> int:
    return torch.cuda.current_stream(device).cuda_stream


def _float32(t: torch.Tensor, *shape, device=None) -> torch.Tensor:
    """``t`` detached, as contiguous float32 on ``device`` (default: its own), reshaped to ``shape`` when one is given."""
    return t.detach().to(device=device, dtype=torch.float32).reshape(shape or t.shape).contiguous()


def _restore(t, shape, dtype):
    return None if t is None else t.reshape(shape).to(dtype)


def _ptr(t) -> int:
    return 0 if t is None else t.data_ptr()


def _batch_sum(g, shape):
    """A per-element gradient [B, ...] of an input of ``shape``: the sum over the batch when the input is shared by it ([...])."""
    return g.sum(dim=0) if g is not None and g.dim() == len(shape) + 1 else g


def _resolve(character, need=None):
    """(Character, skinning) of a ``Character`` (its attributes) or of a ``DeviceCharacter`` (what was uploaded to it). ``need`` "skinning"
    raises without a skinning, "faces" without a skinning with mesh faces."""
    is_handle = isinstance(character, ms.DeviceCharacter)
    ch = character.character if is_handle else character
    if not isinstance(ch, mc.Character):
        raise ValueError("character must be a momentum_b200.character.Character or a DeviceCharacter")
    sk = character.skinning
    if need is not None and sk is None:
        raise ValueError("the character has no skinning" + (", so no mesh faces" if need == "faces" else ""))
    if need == "faces" and is_handle and character.faces is None:
        rejected = character.faces_error
        raise ValueError("the character has no mesh faces" + (f" (their upload was rejected: {rejected})" if rejected else ""))
    if need == "faces" and not is_handle and sk.faces is None:
        raise ValueError("the character has no mesh faces (character.skinning.faces)")
    return ch, sk


class _JointOp(torch.autograd.Function):
    """One operation of the skeleton-state family (``solver.JOINT_OPS``) on [B, in_numel] float32 rows, forward and backward on the
    device."""

    @staticmethod
    def forward(ctx, dc, name, x, out_trailing):
        lead = x.shape[:-2] if name.endswith("to_joint_parameters") else x.shape[:-1]
        rows = _float32(x, -1, int(np.prod(x.shape[len(lead):])))
        B = rows.shape[0]
        out = torch.empty(B, int(np.prod(out_trailing)), device=x.device, dtype=torch.float32)
        dc.joint_op_device(name, False, B, rows.data_ptr(), out.data_ptr(), stream=_stream(x.device))
        ctx.dc, ctx.name, ctx.out_numel = dc, name, out.shape[1]
        ctx.in_shape, ctx.in_dtype = x.shape, x.dtype
        ctx.save_for_backward(rows)
        return _restore(out, (*lead, *out_trailing), x.dtype)

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_out):
        (rows,) = ctx.saved_tensors
        B = rows.shape[0]
        g = _float32(grad_out, B, ctx.out_numel)
        gx = torch.empty_like(rows)
        ptrs = (g.data_ptr(), gx.data_ptr())
        if ctx.name not in ms.LINEAR_JOINT_OPS:  # P^T and W^T do not read their input
            ptrs = (rows.data_ptr(),) + ptrs
        ctx.dc.joint_op_device(ctx.name, True, B, *ptrs, stream=_stream(rows.device))
        return None, None, _restore(gx, ctx.in_shape, ctx.in_dtype), None


def _joint_op(name, character, x, what, trailing, out_trailing):
    """Checks x ([*trailing] or [B, *trailing], a CUDA tensor) before any library call, then runs the operation."""
    if not torch.is_tensor(x):
        raise ValueError(f"{name}: {what} must be a tensor")
    k = len(trailing)
    if x.dim() not in (k, k + 1) or tuple(x.shape[-k:]) != tuple(trailing):
        shape = ", ".join(str(t) for t in trailing)
        raise ValueError(f"{name}: {what} must be [{shape}] or [B, {shape}], got {tuple(x.shape)}")
    if not x.is_cuda:
        raise ValueError(f"{name} runs on CUDA tensors (there is no CPU fallback)")
    return _JointOp.apply(_device_character(character, x.device), name, x, tuple(out_trailing))


def model_parameters_to_skeleton_state(character, model_parameters: torch.Tensor) -> torch.Tensor:
    """Skeleton state of ``model_parameters`` ([n] or [B, n], on a CUDA device): [J, 8] or [B, J, 8] rows (t, q xyzw, s) in the input
    dtype, computed in float32. ``character`` is a ``momentum_b200.character.Character`` or a ``solver.DeviceCharacter`` on the
    tensor's device. Differentiable once with respect to ``model_parameters``."""
    ch, _ = _resolve(character)
    return _joint_op("model_parameters_to_skeleton_state", character, model_parameters, f"model_parameters (n = {ch.num_params})",
                     (ch.num_params,), (ch.num_joints, 8))


def apply_parameter_transform(character, model_parameters: torch.Tensor) -> torch.Tensor:
    """Joint parameters P theta + o of ``model_parameters`` (pymomentum ``apply_parameter_transform``): [n] or [B, n] on a CUDA device
    -> [7 J] or [B, 7 J] in the input dtype, computed in float32, each row's products summed in the ParameterTransform's order.
    ``character`` is a ``momentum_b200.character.Character`` or a ``solver.DeviceCharacter`` on the tensor's device. Differentiable
    once; the gradient is P^T applied on the device."""
    ch, _ = _resolve(character)
    return _joint_op("apply_parameter_transform", character, model_parameters, f"model_parameters (n = {ch.num_params})", (ch.num_params,),
                     (7 * ch.num_joints,))


def apply_inverse_parameter_transform(character, joint_parameters: torch.Tensor) -> torch.Tensor:
    """Model parameters of flat ``joint_parameters`` (pymomentum ``apply_inverse_parameter_transform``): [7 J] or [B, 7 J] on a CUDA
    device -> [n] or [B, n] in the input dtype, computed in float32: theta = P^+ (jp - o), the offsets o subtracted first. P^+ is the
    Moore-Penrose pseudo-inverse of the ParameterTransform with pymomentum's truncation (a singular value above 1e-6, absolute, is
    inverted, any other is 0), so theta is the minimum-norm least-squares solution of P theta + o = jp. It is built once per device
    character, in float64 for each connected component of P's sparsity pattern, and rounded to float32 entry by entry: more accurate than
    pymomentum's float SVD, so the two can differ by that SVD's error. ``character`` is a ``momentum_b200.character.Character`` or a
    ``solver.DeviceCharacter`` on the tensor's device. Differentiable once; the gradient is (P^+)^T applied on the device."""
    ch, _ = _resolve(character)
    return _joint_op("apply_inverse_parameter_transform", character, joint_parameters, f"joint_parameters (7 J = {7 * ch.num_joints})",
                     (7 * ch.num_joints,), (ch.num_params,))


def joint_parameters_to_skeleton_state(character, joint_parameters: torch.Tensor) -> torch.Tensor:
    """Skeleton state of flat ``joint_parameters`` (pymomentum ``joint_parameters_to_skeleton_state``): [7 J] or [B, 7 J] on a CUDA
    device -> [J, 8] or [B, J, 8] rows (t, q xyzw, s) in the input dtype, computed in float32 by the forward kinematics of
    ``model_parameters_to_skeleton_state``. Differentiable once; the backward is that of ``model_parameters_to_skeleton_state``
    without the ParameterTransform."""
    ch, _ = _resolve(character)
    J = ch.num_joints
    return _joint_op("joint_parameters_to_skeleton_state", character, joint_parameters, f"joint_parameters (7 J = {7 * J})", (7 * J,), (J, 8))


def joint_parameters_to_local_skeleton_state(character, joint_parameters: torch.Tensor) -> torch.Tensor:
    """Local skeleton state, each joint's transform to its parent, of flat ``joint_parameters`` (pymomentum
    ``joint_parameters_to_local_skeleton_state``): [7 J] or [B, 7 J] on a CUDA device -> [J, 8] or [B, J, 8] rows (t, q xyzw, s) in
    the input dtype, computed in float32. Joint j's seven parameters p give t = offset_j + p[0:3], q = preRot_j Rz(p5) Ry(p4) Rx(p3),
    s = 2^p6, bit for bit the local part of the forward kinematics. Differentiable once."""
    ch, _ = _resolve(character)
    J = ch.num_joints
    return _joint_op("joint_parameters_to_local_skeleton_state", character, joint_parameters, f"joint_parameters (7 J = {7 * J})", (7 * J,),
                     (J, 8))


def model_parameters_to_local_skeleton_state(character, model_parameters: torch.Tensor) -> torch.Tensor:
    """``joint_parameters_to_local_skeleton_state(apply_parameter_transform(model_parameters))``, as pymomentum composes
    ``model_parameters_to_local_skeleton_state``: [n] or [B, n] -> [J, 8] or [B, J, 8]. Differentiable once."""
    return joint_parameters_to_local_skeleton_state(character, apply_parameter_transform(character, model_parameters))


_EULER_NOTE = """
    The rotation parameters are the XYZ Euler angles of r = inv(preRot_j) q, with inv(q) = conj(q) / |q|^2, read off r as it is (a
    slightly non-unit q is not normalised): rx = atan2(2 (w x + y z), 1 - 2 (x^2 + y^2)), ry = asin(2 (w y - z x)),
    rz = atan2(2 (w z + x y), 1 - 2 (y^2 + z^2)). One deliberate difference from pymomentum: the asin argument is clamped to [-1, 1],
    so that a float32 state at gimbal lock, whose argument can round to 1 + eps, gives ry = +-pi/2 where pymomentum gives NaN; where
    the clamp holds (|argument| >= 1) the derivative of ry is 0. Other non-finite inputs, and s <= 0, propagate as in torch.
    Differentiable once."""


def local_skeleton_state_to_joint_parameters(character, local_skel_state: torch.Tensor) -> torch.Tensor:
    """Joint parameters of local skeleton states (pymomentum ``local_skeleton_state_to_joint_parameters``): [J, 8] or [B, J, 8] on a
    CUDA device -> [J, 7] or [B, J, 7] in the input dtype, computed in float32 (``.flatten(-2)`` gives the [.., 7 J] layout the other
    functions take): t - offset_j, the Euler angles below, log2 s.
    """
    ch, _ = _resolve(character)
    J = ch.num_joints
    return _joint_op("local_skeleton_state_to_joint_parameters", character, local_skel_state, f"local_skel_state (J = {J})", (J, 8), (J, 7))


def skeleton_state_to_joint_parameters(character, skel_state: torch.Tensor) -> torch.Tensor:
    """Joint parameters of world skeleton states (pymomentum ``skeleton_state_to_joint_parameters``): [J, 8] or [B, J, 8] on a CUDA
    device -> [J, 7] or [B, J, 7] in the input dtype, computed in float32 (``.flatten(-2)`` gives the [.., 7 J] layout). Each joint's
    local state is inv(X_parent) X_j (the identity above a root), with inv(t, q, s) = (-s^-1 rot(q^-1, t), q^-1, s^-1) and
    (t1, q1, s1)(t2, q2, s2) = (t1 + rot(q1, s1 t2), q1 q2, s1 s2), rot(q, v) = v + 2 (w (u x v) + u x (u x v)) unnormalised, as
    pymomentum writes them; then ``local_skeleton_state_to_joint_parameters``. The gradient of X_j gathers its own local's term and its
    children's, in a fixed order.
    """
    ch, _ = _resolve(character)
    J = ch.num_joints
    return _joint_op("skeleton_state_to_joint_parameters", character, skel_state, f"skel_state (J = {J})", (J, 8), (J, 7))


local_skeleton_state_to_joint_parameters.__doc__ += _EULER_NOTE
skeleton_state_to_joint_parameters.__doc__ += _EULER_NOTE


class _Positions(torch.autograd.Function):
    """model_parameters_to_positions (joint False) and joint_parameters_to_positions (joint True) on float32 rows, forward and backward on
    the device; ``parents`` is the checked int32 host array."""

    @staticmethod
    def forward(ctx, dc, joint, params, parents, offsets):
        N = parents.shape[0]
        rows = _float32(params, -1, params.shape[-1])
        B = rows.shape[0]
        off = _float32(offsets)
        batched = off.dim() == 3
        out = torch.empty(B, N, 3, device=params.device, dtype=torch.float32)
        if B * N > 0:
            dc.positions_device(joint, B, rows.data_ptr(), parents, off.data_ptr(), batched, out.data_ptr(), _stream(params.device))
        ctx.dc, ctx.joint, ctx.parents, ctx.batched = dc, joint, parents, batched
        ctx.params_shape, ctx.params_dtype, ctx.offsets_dtype = params.shape, params.dtype, offsets.dtype
        ctx.save_for_backward(rows, off)
        return _restore(out, (*params.shape[:-1], N, 3), params.dtype)

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_positions):
        rows, off = ctx.saved_tensors
        B, N = rows.shape[0], ctx.parents.shape[0]
        need_params, need_offsets = ctx.needs_input_grad[2], ctx.needs_input_grad[4]
        gp = torch.zeros_like(rows) if need_params else None
        go = torch.zeros_like(off) if need_offsets else None
        if B * N > 0 and (need_params or need_offsets):  # else the gradients are zero
            g = _float32(grad_positions, B, N, 3)
            ctx.dc.positions_backward_device(ctx.joint, B, rows.data_ptr(), ctx.parents, off.data_ptr(), ctx.batched, g.data_ptr(), _ptr(gp),
                                             _ptr(go), _stream(rows.device))
        return None, None, _restore(gp, ctx.params_shape, ctx.params_dtype), None, _restore(go, off.shape, ctx.offsets_dtype)


def _point_parents(name, parents, J):
    """parents as a checked int32 host array [N]: a sequence, a numpy array or an integer tensor (a CUDA tensor is copied to the host)."""
    if torch.is_tensor(parents):
        if parents.dtype.is_floating_point or parents.dtype.is_complex or parents.dtype == torch.bool:
            raise ValueError(f"{name}: parents must hold integer joint indices, got {parents.dtype}")
        p = parents.detach().cpu().numpy()
    else:
        p = np.asarray(parents)
        if p.size == 0:
            p = p.astype(np.int32)
        if not np.issubdtype(p.dtype, np.integer):
            raise ValueError(f"{name}: parents must hold integer joint indices, got {p.dtype}")
    if p.ndim != 1:
        raise ValueError(f"{name}: parents must be [N], got {tuple(p.shape)}")
    if p.size and (p.min() < 0 or p.max() >= J):
        raise ValueError(f"{name}: every parent must be a joint index in [0, {J})")
    return np.ascontiguousarray(p, np.int32)


def _positions(name, joint, character, params, parents, offsets, what, width):
    """Checks the arguments before any library call, then runs the operation."""
    if not torch.is_tensor(params):
        raise ValueError(f"{name}: {what} must be a tensor")
    if params.dim() not in (1, 2) or params.shape[-1] != width:
        raise ValueError(f"{name}: {what} must be [{width}] or [B, {width}], got {tuple(params.shape)}")
    ch, _ = _resolve(character)
    p = _point_parents(name, parents, ch.num_joints)
    N = p.shape[0]
    if not torch.is_tensor(offsets) or not offsets.dtype.is_floating_point:
        raise ValueError(f"{name}: offsets must be a floating-point tensor")
    B = params.shape[0] if params.dim() == 2 else None
    if not (offsets.shape == (N, 3) or (B is not None and offsets.shape == (B, N, 3))):
        raise ValueError(f"{name}: offsets must be [N, 3] or [B, N, 3] with N = {N} and the parameters' B, got {tuple(offsets.shape)}")
    if not params.is_cuda or not offsets.is_cuda:
        raise ValueError(f"{name} runs on CUDA tensors (there is no CPU fallback)")
    if offsets.device != params.device:
        raise ValueError(f"{name}: offsets must be on the parameters' device")
    return _Positions.apply(_device_character(character, params.device), joint, params, p, offsets)


_POSITIONS_NOTE = """
    ``parents`` [N] holds joint indices in [0, J): a sequence, a numpy array or an integer tensor. A CUDA tensor is copied to the host
    once per call, which synchronises with its device. ``offsets`` is [N, 3], shared by the batch (its gradient is the batch sum), or
    [B, N, 3] with the parameters' B. Point i is at t_a + rot(q_a, s_a offsets_i) for the world state (t_a, q_a, s_a) of joint
    a = parents[i]. Returns [N, 3] or [B, N, 3] in the parameters' dtype, computed in float32. N = 0 gives an empty result and zero
    gradients. Differentiable once with respect to the parameters and the offsets, not ``parents``. The backward seeds the skeleton-state
    backward's subtree sums from the points, so it costs O(J + N) per instance whatever the depth of the joints."""


def model_parameters_to_positions(character, model_parameters: torch.Tensor, parents, offsets: torch.Tensor) -> torch.Tensor:
    """World positions of points fixed in joints' frames (pymomentum ``model_parameters_to_positions``): markers, keypoints or locators
    of ``model_parameters`` ([n] or [B, n], on a CUDA device), without the [B, J, 8] skeleton state in memory. ``character`` is a
    ``momentum_b200.character.Character`` or a ``solver.DeviceCharacter`` on the tensor's device.
    """
    ch, _ = _resolve(character)
    return _positions("model_parameters_to_positions", False, character, model_parameters, parents, offsets, f"model_parameters (n = {ch.num_params})",
                      ch.num_params)


def joint_parameters_to_positions(character, joint_parameters: torch.Tensor, parents, offsets: torch.Tensor) -> torch.Tensor:
    """``model_parameters_to_positions`` from flat joint parameters (pymomentum ``joint_parameters_to_positions``): [7 J] or [B, 7 J] on a
    CUDA device, the layout of ``joint_parameters_to_skeleton_state``.
    """
    ch, _ = _resolve(character)
    J = ch.num_joints
    return _positions("joint_parameters_to_positions", True, character, joint_parameters, parents, offsets, f"joint_parameters (7 J = {7 * J})", 7 * J)


model_parameters_to_positions.__doc__ += _POSITIONS_NOTE
joint_parameters_to_positions.__doc__ += _POSITIONS_NOTE


class _ParameterLimits(torch.autograd.Function):
    """parameter_limits_residual on [B, n] float32 rows, forward and backward on the device."""

    @staticmethod
    def forward(ctx, dc, R, theta):
        rows = _float32(theta, -1, theta.shape[-1])
        B = rows.shape[0]
        out = torch.empty(B, R, device=theta.device, dtype=torch.float32)
        if B * R > 0:
            dc.parameter_limits_residual_device(B, rows.data_ptr(), out.data_ptr(), _stream(theta.device))
        ctx.dc, ctx.R, ctx.shape, ctx.dtype = dc, R, theta.shape, theta.dtype
        ctx.save_for_backward(rows)
        return _restore(out, (*theta.shape[:-1], R), theta.dtype)

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_residual):
        (rows,) = ctx.saved_tensors
        B = rows.shape[0]
        gt = torch.zeros_like(rows)
        if B * ctx.R > 0:  # else the gradient is zero
            g = _float32(grad_residual, B, ctx.R)
            ctx.dc.parameter_limits_residual_backward_device(B, rows.data_ptr(), g.data_ptr(), gt.data_ptr(), _stream(rows.device))
        return None, None, _restore(gt, ctx.shape, ctx.dtype)


_LIMITS_NOTE = """
    The limits are those of the device handle: for a ``Character``, ``character.limits`` as they were when the torch layer first made
    its handle for it on that device (``solve_ik`` reads them at the same moment). A changed limit list needs a new ``Character`` or
    ``DeviceCharacter``. A limit whose index is out of range raises ``MomentumB200Error`` naming it; ``solve_ik`` only rejects it when its
    objective has a limit block."""


def parameter_limits_residual(character, model_parameters: torch.Tensor) -> torch.Tensor:
    """The residual of momentum's ``LimitErrorFunction`` over the character's ParameterLimits, at weight 1 with the L2 loss, for
    ``model_parameters`` ([n] or [B, n], on a CUDA device): [R] or [B, R] in the input dtype, computed in float32, so that
    ``residual.square().sum(-1)`` is ``LimitErrorFunction::getError``. The rows are those its ``getJacobian`` returns: one per limit in
    ``character.limits`` order, none for MinMaxJointPassive, three for an Ellipsoid; sqrt(10 w) times the limit's residual
    (Ellipsoid: sqrt(10 * 1e-4 w)); 0 for an inactive limit. MinMax gives theta - min below the minimum and theta - max above the
    maximum; Linear and LinearJoint apply only where the target is in [rangeMin, rangeMax), (0, 0) meaning everywhere; HalfPlane only
    where its value is negative. Joint-space limits read P theta + o, Ellipsoids the skeleton state of theta. A character without live
    limits gives [B, 0].

    Against pymomentum's torch module ``pymomentum.torch.parameter_limits.ParameterLimits``: the module groups its rows by limit type,
    its MinMax rows below the minimum have the opposite sign (min - theta), and it lacks the (0, 0) rule of Linear and LinearJoint
    ranges. Where that rule does not apply, the sum of squares is the same.

    Differentiable once with respect to ``model_parameters``. The gradient is the exact derivative of these rows: for an Ellipsoid it
    includes the projection onto the ellipsoid and the motion of the ellipsoid's parent joint, where momentum's
    ``computeEllipsoidJacobian`` walks only the joints from the parent up to the ellipsoid parent and holds the projected point fixed.
    It costs O(J + limits) per instance."""
    name = "parameter_limits_residual"
    ch, _ = _resolve(character)
    n = ch.num_params
    if not torch.is_tensor(model_parameters):
        raise ValueError(f"{name}: model_parameters must be a tensor")
    if model_parameters.dim() not in (1, 2) or model_parameters.shape[-1] != n:
        raise ValueError(f"{name}: model_parameters must be [{n}] or [B, {n}], got {tuple(model_parameters.shape)}")
    if not model_parameters.is_cuda:
        raise ValueError(f"{name} runs on CUDA tensors (there is no CPU fallback)")
    dc = _device_character(character, model_parameters.device)
    return _ParameterLimits.apply(dc, dc.num_limit_residuals(), model_parameters)


def apply_model_param_limits(character, model_parameters: torch.Tensor) -> torch.Tensor:
    """pymomentum ``apply_model_param_limits``: ``model_parameters`` ([n] or [B, n], on a CUDA device) with every parameter that a MinMax
    limit names clamped to [min, max] as ``torch.clamp`` does it (NaN stays NaN), every other parameter passed through, in the input
    dtype, computed in float32. Other limit types are ignored. When several MinMax limits name one parameter, the last in list order
    decides both the value and the gradient, as a sequential ``index_copy`` would. Differentiable once: the gradient is ``torch.clamp``'s,
    the upstream gradient where min <= theta <= max and 0 elsewhere."""
    ch, _ = _resolve(character)
    return _joint_op("apply_model_parameter_limits", character, model_parameters, f"model_parameters (n = {ch.num_params})", (ch.num_params,),
                     (ch.num_params,))


parameter_limits_residual.__doc__ += _LIMITS_NOTE
apply_model_param_limits.__doc__ += _LIMITS_NOTE


class _Collision(torch.autograd.Function):
    """collision_residual on [B, J, 8] float32 states, forward and backward on the device."""

    @staticmethod
    def forward(ctx, dc, P, skel_state):
        J = dc.character.num_joints
        st = _float32(skel_state, -1, J, 8)
        B = st.shape[0]
        out = torch.empty(B, P, device=st.device, dtype=torch.float32)
        if B * P > 0:
            dc.collision_residual_device(B, st.data_ptr(), out.data_ptr(), _stream(st.device))
        ctx.dc, ctx.P, ctx.shape, ctx.dtype = dc, P, skel_state.shape, skel_state.dtype
        ctx.save_for_backward(st)
        return _restore(out, (*skel_state.shape[:-2], P), skel_state.dtype)

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_residual):
        (st,) = ctx.saved_tensors
        B = st.shape[0]
        gs = torch.zeros_like(st)
        if B * ctx.P > 0:  # else the gradient is zero
            g = _float32(grad_residual, B, ctx.P)
            ctx.dc.collision_residual_backward_device(B, st.data_ptr(), g.data_ptr(), gs.data_ptr(), _stream(st.device))
        return None, None, _restore(gs, ctx.shape, ctx.dtype)


def _collision_handle(character, device):
    """The handle of ``character`` with its collision geometry uploaded, or ValueError."""
    ch, _ = _resolve(character)
    if isinstance(character, ms.DeviceCharacter):
        dc = _device_character(character, device)
    else:
        if ch.collision is None:
            raise ValueError("the character has no collision geometry (character.collision is None)")
        dc = _device_character(character, device)
    if dc.collision is None:
        rejected = dc.collision_error
        raise ValueError("the character has no collision geometry" + (f" (its upload was rejected: {rejected})" if rejected else ""))
    return dc


def collision_residual(character, skel_state: torch.Tensor) -> torch.Tensor:
    """Self-collision of the character's tapered capsules, the residual of momentum's ``CollisionErrorFunction`` at weight 1:
    ``skel_state`` [J, 8] or [B, J, 8] (t, q xyzw, s; q is normalised) on a CUDA device -> [P] or [B, P] in the input dtype, computed
    in float32. Row k belongs to valid pair k (``collision_pairs``): sqrt(5e-3) times the pair's overlap where the reference's
    ``overlaps`` reports a contact, 0 otherwise, so that ``residual.square().sum(-1)`` is ``CollisionErrorFunction::getError`` and the
    nonzero rows, in order, are the compacted residual of its ``getJacobian``. The narrow phase is ``closestPointsOnSegments`` branch for
    branch in float, its quirks included: two nearly parallel capsules (D < 1e-7) whose origins are farther apart than the sum of their
    largest radii have no contact even when their sides touch. A world capsule is T_parent o T_local: origin T.t, direction R(T.q) e_x
    T.s length, radii radius times the parent's scale only. A capsule's local rotation is normalised when the geometry is uploaded; the
    reference composes a non-unit rotation as it is, so the two differ for one (a zero rotation is rejected).

    The valid pairs are planned when the geometry is uploaded: a pair of world-fixed capsules is dropped, a pair with exactly one is
    kept, capsules on the same or parent-child joints are dropped, and the rest are kept unless they overlap at the rest pose (model
    parameters zero), which is evaluated in double where the reference's float build evaluates it in float. An empty geometry gives
    [B, 0]; ``character.collision`` None raises ValueError.

    Differentiable once with respect to ``skel_state``. The gradient is the exact derivative of these rows, including the motion of
    the closest-point parameters (s, t) through the closed form of the branch taken; a clamped or snapped parameter is constant. Momentum's
    ``getJacobian`` holds (s, t) fixed and so drops delta ds/dtheta: it agrees with this gradient for untapered capsules (r0 = r1) and
    differs for tapered ones. Compose with ``model_parameters_to_skeleton_state`` for a loss in model parameters.

    ``character`` is a ``momentum_b200.character.Character``, whose ``collision`` list is read when the torch layer makes its handle:
    replacing the attribute makes a new handle, as replacing ``skinning`` does (changing the list in place does not). Or it is a
    ``solver.DeviceCharacter``, with what was uploaded to it."""
    if not torch.is_tensor(skel_state) or not skel_state.is_cuda:
        raise ValueError("collision_residual runs on CUDA tensors (there is no CPU fallback)")
    ch, _ = _resolve(character)
    J = ch.num_joints
    if skel_state.dim() not in (2, 3) or skel_state.shape[-2:] != (J, 8):
        raise ValueError(f"skel_state must be [J, 8] or [B, J, 8] with J = {J}, got {tuple(skel_state.shape)}")
    dc = _collision_handle(character, skel_state.device)
    return _Collision.apply(dc, dc.num_collision_pairs, skel_state)


def collision_pairs(character, device=None) -> torch.Tensor:
    """The valid pairs of ``collision_residual``'s rows: a CPU int64 tensor [P, 2], capsule indices i < j, row k for pair k. ``device``
    (a CUDA device, default the current one) is where a ``Character``'s handle lives. The pairs are planned on the host, but reading them
    makes (or reuses) that device handle, so this needs a CUDA device; ``character.collision_pairs`` restates the same rules in float64
    without one."""
    if isinstance(character, ms.DeviceCharacter):
        dc = _collision_handle(character, torch.device("cuda", character.device))
    else:
        dc = _collision_handle(character, torch.device("cuda") if device is None else torch.device(device))
    return torch.from_numpy(dc.collision_pairs().astype(np.int64))


class _SkinPoints(torch.autograd.Function):
    @staticmethod
    def forward(ctx, dc, skel_state, rest_points):
        J, V = dc.character.num_joints, dc.skinning.num_vertices
        st = _float32(skel_state, -1, J, 8)
        B = st.shape[0]
        rest = None if rest_points is None else _float32(rest_points)
        batched = rest is not None and rest.dim() == 3
        out = st.new_empty(B, V, 3)
        dc.skin_points_device(B, st.data_ptr(), _ptr(rest), batched, out.data_ptr(), _stream(st.device))
        ctx.dc, ctx.skinning, ctx.V, ctx.batched = dc, dc.skinning, V, batched
        ctx.state_shape, ctx.state_dtype = skel_state.shape, skel_state.dtype
        ctx.rest_dtype = None if rest_points is None else rest_points.dtype
        ctx.save_for_backward(st, rest)
        return _restore(out, (*skel_state.shape[:-2], V, 3), skel_state.dtype)

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_points):
        st, rest = ctx.saved_tensors
        dc = ctx.dc
        if dc.skinning is not ctx.skinning:
            raise RuntimeError("skin_points backward: the DeviceCharacter's skinning was replaced (set_skinning) after the forward; "
                               "keep one DeviceCharacter per skinning, or pass the Character and replace character.skinning instead")
        B, J, _ = st.shape
        g = _float32(grad_points, B, ctx.V, 3)
        need_state, need_rest = ctx.needs_input_grad[1:]  # no gradient is asked of rest_points None
        gs = st.new_empty(B, J, 8) if need_state else None
        gr = torch.empty_like(rest) if need_rest else None
        dc.skin_points_backward_device(B, st.data_ptr(), _ptr(rest), ctx.batched, g.data_ptr(), _ptr(gs), _ptr(gr), _stream(st.device))
        return None, _restore(gs, ctx.state_shape, ctx.state_dtype), None if gr is None else gr.to(ctx.rest_dtype)


def skin_points(character, skel_state: torch.Tensor, rest_points=None) -> torch.Tensor:
    """Linear-blend skinning (pymomentum ``Character.skin_points``): ``skel_state`` [J, 8] or [B, J, 8] (t, q xyzw, s; q is normalised)
    on a CUDA device -> points [V, 3] or [B, V, 3] in the input dtype, computed in float32. ``rest_points``: None = the rest mesh,
    [V, 3] shared by the batch (its gradient is the batch sum) or [B, V, 3]. Differentiable once with respect to ``skel_state`` and
    ``rest_points``.

    ``character`` is a ``momentum_b200.character.Character``, skinned with ``character.skinning``: replacing that attribute is safe at
    any time, and graphs recorded before keep the skinning they were recorded with. Or it is a ``solver.DeviceCharacter``, skinned with
    what was uploaded to it (``DeviceCharacter.skinning``); the backward of a graph recorded before a later ``set_skinning`` on the same
    handle raises."""
    if not torch.is_tensor(skel_state) or not skel_state.is_cuda:
        raise ValueError("skin_points runs on CUDA tensors (there is no CPU fallback)")
    ch, sk = _resolve(character, "skinning")
    J, V = ch.num_joints, sk.num_vertices
    if skel_state.shape[-2:] == (4, 4):
        raise ValueError("skin_points takes skeleton states [.., J, 8] (t, q xyzw, s), not 4x4 matrices")
    if skel_state.dim() not in (2, 3) or skel_state.shape[-2:] != (J, 8):
        raise ValueError(f"skel_state must be [J, 8] or [B, J, 8] with J = {J}, got {tuple(skel_state.shape)}")
    if rest_points is not None:
        if not torch.is_tensor(rest_points) or rest_points.device != skel_state.device:
            raise ValueError("rest_points must be a tensor on the skel_state's device")
        B = skel_state.shape[0] if skel_state.dim() == 3 else None
        if not (rest_points.shape == (V, 3) or (B is not None and rest_points.shape == (B, V, 3))):
            raise ValueError(f"rest_points must be [V, 3] or [B, V, 3] with V = {V} and the skel_state's B, got {tuple(rest_points.shape)}")
    return _SkinPoints.apply(_device_character(character, skel_state.device), skel_state, rest_points)


class _SkinWithBlendShapes(torch.autograd.Function):
    @staticmethod
    def forward(ctx, dc, skel_state, blend_weights):
        J, V = dc.character.num_joints, dc.skinning.num_vertices
        st = _float32(skel_state, -1, J, 8)
        B, K = st.shape[0], blend_weights.shape[-1]
        w = _float32(blend_weights.expand(B, K))
        out = st.new_empty(B, V, 3)
        dc.skin_with_blend_shapes_device(B, st.data_ptr(), w.data_ptr(), K, out.data_ptr(), _stream(st.device))
        ctx.dc, ctx.skinning, ctx.blend_shape, ctx.V = dc, dc.skinning, dc.blend_shape, V
        ctx.state_shape, ctx.state_dtype = skel_state.shape, skel_state.dtype
        ctx.weights_shape, ctx.weights_dtype = blend_weights.shape, blend_weights.dtype
        ctx.save_for_backward(st, w)
        return _restore(out, (*skel_state.shape[:-2], V, 3), skel_state.dtype)

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_points):
        st, w = ctx.saved_tensors
        dc = ctx.dc
        if dc.skinning is not ctx.skinning or dc.blend_shape is not ctx.blend_shape:
            raise RuntimeError("skin_with_blend_shapes backward: the DeviceCharacter's skinning or blend shape was replaced (set_skinning / "
                               "set_blend_shape) after the forward; keep one DeviceCharacter per mesh, or pass the Character and replace "
                               "its attributes instead")
        B, J, _ = st.shape
        g = _float32(grad_points, B, ctx.V, 3)
        need_state, need_weights = ctx.needs_input_grad[1:]
        gs = st.new_empty(B, J, 8) if need_state else None
        gw = torch.empty_like(w) if need_weights else None
        dc.skin_with_blend_shapes_backward_device(B, st.data_ptr(), w.data_ptr(), w.shape[1], g.data_ptr(), _ptr(gs), _ptr(gw), _stream(st.device))
        return None, _restore(gs, ctx.state_shape, ctx.state_dtype), _restore(_batch_sum(gw, ctx.weights_shape), ctx.weights_shape, ctx.weights_dtype)


def skin_with_blend_shapes(character, skel_state: torch.Tensor, blend_weights: torch.Tensor) -> torch.Tensor:
    """Skinning with the character's identity blend shape (momentum ``skinWithBlendShapes``): the rest mesh of each instance is
    ``base_shape + sum_k w_k shape_vectors[k]`` over the first K' = ``blend_weights.shape[-1]`` shape vectors, skinned as ``skin_points``
    skins, without a shaped rest mesh in memory. ``skel_state`` [J, 8] or [B, J, 8] on a CUDA device; ``blend_weights`` [K'] shared by
    the batch (its gradient is the batch sum) or [B, K'], 1 <= K' <= K. Returns points [V, 3] or [B, V, 3] in the skel_state's dtype,
    computed in float32. Differentiable once with respect to ``skel_state`` and ``blend_weights``.

    ``character`` is a ``momentum_b200.character.Character`` with ``skinning`` and ``blend_shape`` set: replacing either attribute is safe
    at any time, and graphs recorded before keep what they were recorded with. Or it is a ``solver.DeviceCharacter``, which uses what was
    uploaded to it; the backward of a graph recorded before a later ``set_skinning`` or ``set_blend_shape`` on that handle raises."""
    if not torch.is_tensor(skel_state) or not skel_state.is_cuda:
        raise ValueError("skin_with_blend_shapes runs on CUDA tensors (there is no CPU fallback)")
    ch, sk = _resolve(character, "skinning")
    bs = character.blend_shape
    if bs is None:
        rejected = character.blend_shape_error if isinstance(character, ms.DeviceCharacter) else None
        raise ValueError("the character has no blend shape" + (f" (its upload was rejected: {rejected})" if rejected else ""))
    if bs.num_vertices != sk.num_vertices:
        raise ValueError(f"the blend shape has {bs.num_vertices} vertices but the skinning has {sk.num_vertices}")
    J = ch.num_joints
    if skel_state.dim() not in (2, 3) or skel_state.shape[-2:] != (J, 8):
        raise ValueError(f"skel_state must be [J, 8] or [B, J, 8] with J = {J}, got {tuple(skel_state.shape)}")
    if not torch.is_tensor(blend_weights) or blend_weights.device != skel_state.device:
        raise ValueError("blend_weights must be a tensor on the skel_state's device")
    B = skel_state.shape[0] if skel_state.dim() == 3 else None
    K = blend_weights.shape[-1] if blend_weights.dim() in (1, 2) else 0
    if not (1 <= K <= bs.num_shapes and (blend_weights.dim() == 1 or (B is not None and blend_weights.shape[0] == B))):
        raise ValueError(f"blend_weights must be [K'] or [B, K'] with 1 <= K' <= {bs.num_shapes} and the skel_state's B, got {tuple(blend_weights.shape)}")
    dc = _device_character(character, skel_state.device)
    if dc.blend_shape is None:
        raise ValueError(f"the character's blend shape was rejected: {dc.blend_shape_error}")
    return _SkinWithBlendShapes.apply(dc, skel_state, blend_weights)


class _VertexNormals(torch.autograd.Function):
    @staticmethod
    def forward(ctx, dc, vertex_positions):
        x = _float32(vertex_positions, -1, dc.skinning.num_vertices, 3)
        out = torch.empty_like(x)
        dc.vertex_normals_device(x.shape[0], x.data_ptr(), out.data_ptr(), _stream(x.device))
        ctx.dc, ctx.skinning, ctx.faces = dc, dc.skinning, dc.faces
        ctx.in_shape, ctx.in_dtype = vertex_positions.shape, vertex_positions.dtype
        ctx.save_for_backward(x)
        return _restore(out, ctx.in_shape, ctx.in_dtype)

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_normals):
        (x,) = ctx.saved_tensors
        dc = ctx.dc
        if dc.skinning is not ctx.skinning or dc.faces is not ctx.faces:
            raise RuntimeError("compute_vertex_normals backward: the DeviceCharacter's skinning was replaced (set_skinning) after the forward; "
                               "keep one DeviceCharacter per mesh, or pass the Character and replace character.skinning instead")
        g = _float32(grad_normals, *x.shape)
        gx = torch.empty_like(x)
        dc.vertex_normals_backward_device(x.shape[0], x.data_ptr(), g.data_ptr(), gx.data_ptr(), _stream(x.device))
        return None, _restore(gx, ctx.in_shape, ctx.in_dtype)


def compute_vertex_normals(character, vertex_positions: torch.Tensor) -> torch.Tensor:
    """Area-weighted vertex normals (pymomentum ``diff_geometry.compute_vertex_normals``): ``vertex_positions`` [V, 3] or [B, V, 3] on a
    CUDA device -> normals of the same shape in the input dtype, computed in float32. Per vertex, the sum of (x1 - x0) x (x2 - x0) over
    every corner of every face that is that vertex, faces ascending and corners in order, divided by max(|n|, 1e-12): an isolated vertex
    gives exactly 0. Non-finite positions propagate (momentum's ``Mesh::updateNormals`` skips NaN faces; this does not). Differentiable
    once with respect to ``vertex_positions``, with the exact derivative of the clamp.

    The faces are ``character.skinning.faces`` (int32 [F, 3] over the rest vertices), not an argument as in pymomentum's
    ``(vertex_positions, triangles)``: the library validates them and builds its vertex -> face table once, when they are uploaded, so
    a call copies nothing from the device to the host. ``character`` is a ``momentum_b200.character.Character``: replacing
    ``character.skinning`` or its ``faces`` is safe at any time, and graphs recorded before keep the faces they were recorded with. Or it
    is a ``solver.DeviceCharacter``, which uses what was uploaded with its skinning; the backward of a graph recorded before a later
    ``set_skinning`` on that handle raises."""
    if not torch.is_tensor(vertex_positions) or not vertex_positions.is_cuda:
        raise ValueError("compute_vertex_normals runs on CUDA tensors (there is no CPU fallback)")
    _, sk = _resolve(character, "faces")
    V = sk.num_vertices
    if vertex_positions.dim() not in (2, 3) or vertex_positions.shape[-2:] != (V, 3):
        raise ValueError(f"vertex_positions must be [V, 3] or [B, V, 3] with V = {V}, got {tuple(vertex_positions.shape)}")
    dc = _device_character(character, vertex_positions.device)
    if dc.faces is None:
        raise ValueError(f"the character's mesh faces were rejected: {dc.faces_error}")
    return _VertexNormals.apply(dc, vertex_positions)


def find_closest_points_on_mesh(character, points_source: torch.Tensor, vertices_target: torch.Tensor, max_dist: float = float("inf")):
    """The closest point on the character's posed mesh of each query point (pymomentum ``geometry.find_closest_points_on_mesh``):
    ``points_source`` [N, 3] or [B, N, 3] and ``vertices_target`` [V, 3] or [B, V, 3] on one CUDA device; B broadcasts when one side is
    unbatched. Returns ``(valid, points, face_index, bary)`` in pymomentum's order: bool [.., N], the closest points [.., N, 3] and the
    barycentrics [.., N, 3] in the inputs' dtype (computed in float32), and int32 face indices [.., N]. Per query the result is the face
    with the smallest (squared distance, face index) among the faces with finite vertices within ``max_dist`` (default: no bound); a
    query without one (a non-finite query included) gives valid False, face -1 and zeros. It does not depend on the search tree.

    The faces are ``character.skinning.faces``, as in ``compute_vertex_normals``; the search tree is built once over the rest mesh when
    they are uploaded, and each call refits its boxes to ``vertices_target``. ``character`` is a ``momentum_b200.character.Character``
    or a ``solver.DeviceCharacter``.

    Not differentiable: the outputs carry no gradient. For fitting, recompose the point from the vertices with the returned face and
    barycentrics, ``q = sum_k bary[..., k] * x[face[..., k]]``::

        with torch.no_grad():
            valid, _, face, bary = find_closest_points_on_mesh(ch, p, x)
        tri = faces_t[face.clamp(min=0).long()]                                 # [B, N, 3] vertex indices
        corners = torch.gather(x, 1, tri.reshape(B, -1, 1).expand(-1, -1, 3)).reshape(B, N, 3, 3)
        q = (bary.unsqueeze(-1) * corners).sum(-2)
        loss = (((p - q) ** 2).sum(-1) * valid).sum()

    Wherever the closest face is unique, the gradient of ``|p - q|^2`` through this composition, with respect to p and to x, is the exact
    gradient of the squared point-to-mesh distance (the envelope theorem: the closest point moves along the surface, orthogonally to
    p - q)."""
    for name, t in (("points_source", points_source), ("vertices_target", vertices_target)):
        if not torch.is_tensor(t) or not t.is_cuda:
            raise ValueError(f"find_closest_points_on_mesh runs on CUDA tensors (there is no CPU fallback); {name} is not one")
    if points_source.device != vertices_target.device:
        raise ValueError("points_source and vertices_target must be on the same device")
    _, sk = _resolve(character, "faces")
    V = sk.num_vertices
    if vertices_target.dim() not in (2, 3) or vertices_target.shape[-2:] != (V, 3):
        raise ValueError(f"vertices_target must be [V, 3] or [B, V, 3] with V = {V}, got {tuple(vertices_target.shape)}")
    if points_source.dim() not in (2, 3) or points_source.shape[-1] != 3:
        raise ValueError(f"points_source must be [N, 3] or [B, N, 3], got {tuple(points_source.shape)}")
    if points_source.dim() == 3 and vertices_target.dim() == 3 and points_source.shape[0] != vertices_target.shape[0]:
        raise ValueError(f"points_source and vertices_target have batches {points_source.shape[0]} and {vertices_target.shape[0]}")
    max_dist = float(max_dist)
    if not max_dist >= 0.0:
        raise ValueError(f"max_dist must be >= 0 (float('inf') for no bound), got {max_dist}")
    dev = points_source.device
    dc = _device_character(character, dev)
    if dc.faces is None:
        raise ValueError(f"the character's mesh faces were rejected: {dc.faces_error}")
    if dc.faces.shape[0] == 0 or dc.mesh_tree_error is not None:
        raise ValueError("the character's mesh has no closest-point tree" + (f": {dc.mesh_tree_error}" if dc.mesh_tree_error else " (no faces)"))
    batched = points_source.dim() == 3 or vertices_target.dim() == 3
    B = points_source.shape[0] if points_source.dim() == 3 else (vertices_target.shape[0] if vertices_target.dim() == 3 else 1)
    N = points_source.shape[-2]
    dtype = torch.promote_types(points_source.dtype, vertices_target.dtype)
    with torch.no_grad():
        p = _float32(points_source.expand(B, N, 3))
        x = _float32(vertices_target.expand(B, V, 3))
        q = torch.empty(B, N, 3, device=dev, dtype=torch.float32)
        face = torch.empty(B, N, device=dev, dtype=torch.int32)
        bary = torch.empty(B, N, 3, device=dev, dtype=torch.float32)
        dc.closest_points_on_mesh_device(B, N, x.data_ptr(), p.data_ptr(), max_dist, q.data_ptr(), face.data_ptr(), bary.data_ptr(), _stream(dev))
        valid = face >= 0
        q, bary = q.to(dtype), bary.to(dtype)
    if not batched:
        valid, q, face, bary = valid[0], q[0], face[0], bary[0]
    return valid, q, face, bary


def find_closest_points(*args, **kwargs):
    """The closest target point of each query point (pymomentum ``geometry.find_closest_points``), in its two overloads, told apart by
    the number of leading tensor arguments (neither takes a character)::

        points, index, valid = find_closest_points(points_source, points_target, max_dist=inf)
        points, normals, index, valid = find_closest_points(points_source, normals_source, points_target, normals_target,
                                                            max_dist=inf, max_normal_dot=0.0)

    Sources are [N, D] or [B, N, D] and targets [M, D] or [B, M, D], D = 2 or 3 (3 for the normal variant), on one CUDA device; B
    broadcasts when one side is unbatched, and an unbatched target is searched as one cloud for the whole batch. Per query p the result
    is the target j with the smallest (squared distance, j) among the candidates: finite targets within ``max_dist`` (d² ≤ max_dist², as
    ``find_closest_points_on_mesh``; pymomentum's kd-tree uses <) and, in the normal variant, with dot(n_p, n_j) ≥ ``max_normal_dot``.
    Despite its pymomentum name, ``max_normal_dot`` is that lower bound: 0 keeps targets facing the same half-space. Equal distances go
    to the lowest index (pymomentum leaves the choice open). A query without a candidate (a non-finite query included) gives valid
    False, index -1 and zeros. Returned: the target points [.., N, D] (and normals [.., N, 3]) copied from the targets, int32 indices
    [.., N] and bool validity [.., N]; computed in float32 and returned in the promoted input dtype. D = 2 is searched with z = 0, which
    gives the same squared distances. A tree is built over each target cloud on the device per call; the result does not depend on it.

    Not differentiable: the outputs carry no gradient. For fitting, gather the targets with the returned indices outside the query::

        with torch.no_grad():
            _, _, index, valid = find_closest_points(x, n, scan, scan_normals, max_dist=d, max_normal_dot=0.5)
        t = torch.gather(scan, -2, index.clamp(min=0).long().unsqueeze(-1).expand(*index.shape, 3))
        nt = torch.gather(scan_normals, -2, index.clamp(min=0).long().unsqueeze(-1).expand(*index.shape, 3))
        loss = ((((x - t) * nt).sum(-1) ** 2) * valid).sum()             # point-to-plane, differentiable in x (and the scan)
    """
    names = ("points_source", "points_target", "max_dist")
    names_n = ("points_source", "normals_source", "points_target", "normals_target", "max_dist", "max_normal_dot")
    lead = 0
    while lead < len(args) and torch.is_tensor(args[lead]):
        lead += 1
    normals = lead >= 4 or "normals_source" in kwargs or "normals_target" in kwargs
    order = names_n if normals else names
    if len(args) > len(order):
        raise TypeError(f"find_closest_points takes at most {len(order)} positional arguments, got {len(args)}")
    given = dict(zip(order, args))
    for k, v in kwargs.items():
        if k not in order:
            raise TypeError(f"find_closest_points got an unexpected keyword argument {k!r}")
        if k in given:
            raise TypeError(f"find_closest_points got multiple values for {k!r}")
        given[k] = v
    tensors = [n for n in order if n.startswith(("points", "normals"))]
    missing = [n for n in tensors if n not in given]
    if missing:
        raise TypeError(f"find_closest_points is missing {', '.join(missing)}")
    for n in tensors:
        t = given[n]
        if not torch.is_tensor(t) or not t.is_cuda:
            raise ValueError(f"find_closest_points runs on CUDA tensors (there is no CPU fallback); {n} is not one")
    src, tgt = given["points_source"], given["points_target"]
    dev = src.device
    if any(given[n].device != dev for n in tensors):
        raise ValueError("find_closest_points: every tensor must be on the same device")
    max_dist = float(given.get("max_dist", float("inf")))
    max_normal_dot = float(given.get("max_normal_dot", 0.0))
    if not max_dist >= 0.0:
        raise ValueError(f"max_dist must be >= 0 (float('inf') for no bound), got {max_dist}")
    if max_normal_dot != max_normal_dot:
        raise ValueError("max_normal_dot must not be NaN")
    if src.dim() not in (2, 3) or src.shape[-1] not in (2, 3):
        raise ValueError(f"points_source must be [N, D] or [B, N, D] with D = 2 or 3, got {tuple(src.shape)}")
    D = src.shape[-1]
    if tgt.dim() not in (2, 3) or tgt.shape[-1] != D:
        raise ValueError(f"points_target must be [M, {D}] or [B, M, {D}] like points_source, got {tuple(tgt.shape)}")
    if src.dim() == 3 and tgt.dim() == 3 and src.shape[0] != tgt.shape[0]:
        raise ValueError(f"points_source and points_target have batches {src.shape[0]} and {tgt.shape[0]}")
    if normals:
        if D != 3:
            raise ValueError("the normal variant takes 3-D points and normals")
        for pn, nn in (("points_source", "normals_source"), ("points_target", "normals_target")):
            if given[nn].shape != given[pn].shape:
                raise ValueError(f"{nn} must have the shape of {pn}, {tuple(given[pn].shape)}, got {tuple(given[nn].shape)}")
    batched = src.dim() == 3 or tgt.dim() == 3
    B = src.shape[0] if src.dim() == 3 else (tgt.shape[0] if tgt.dim() == 3 else 1)
    N, M = src.shape[-2], tgt.shape[-2]
    dtype = src.dtype
    for n in tensors[1:]:
        dtype = torch.promote_types(dtype, given[n].dtype)
    if not dtype.is_floating_point:
        dtype = torch.float32
    target_batched = tgt.dim() == 3

    def prep(t, rows, shared):
        t = t.detach().to(torch.float32)
        if D == 2:
            t = torch.nn.functional.pad(t, (0, 1))
        t = t if t.dim() == 3 else t.unsqueeze(0)
        return (t if shared else t.expand(B, rows, 3)).contiguous()

    index = _device_index(dev)
    with torch.no_grad(), torch.cuda.device(index):
        p = prep(src, N, False)
        x = prep(tgt, M, not target_batched)
        pn = prep(given["normals_source"], N, False) if normals else None
        xn = prep(given["normals_target"], M, not target_batched) if normals else None
        q = torch.empty(B, N, 3, device=dev, dtype=torch.float32)
        qn = torch.empty(B, N, 3, device=dev, dtype=torch.float32) if normals else None
        idx = torch.empty(B, N, device=dev, dtype=torch.int32)
        ptr = lambda t: 0 if t is None or t.numel() == 0 else t.data_ptr()  # noqa: E731
        if B * N > 0:
            ms.closest_points_device(index, B, N, M, target_batched, ptr(p), ptr(pn), ptr(x), ptr(xn), max_dist, max_normal_dot, ptr(q),
                                     ptr(qn), ptr(idx), _stream(dev))
        valid = idx >= 0
        q = q[..., :D].to(dtype)
        qn = qn.to(dtype) if normals else None
    if not batched:
        q, qn, idx, valid = q[0], (qn[0] if normals else None), idx[0], valid[0]
    return (q, qn, idx, valid) if normals else (q, idx, valid)
