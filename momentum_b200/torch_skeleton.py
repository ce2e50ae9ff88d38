"""Differentiable forward kinematics on CUDA tensors: ``model_parameters_to_skeleton_state``.

Mirror of ``pymomentum.geometry.model_parameters_to_skeleton_state`` (pymomentum/tensor_momentum/tensor_skeleton_state.cpp:500-502:
``jointParametersToSkeletonState(applyParamTransform(theta))``) for the batched device path. The forward pass is the solver's own FK
device code (``mb2_character_skeleton_state_device``); the backward pass replaces the reference's per-joint ``ceres::Jet`` ancestor
walks (``computeSkelStateBackward``, :62-134) with one reverse sweep over the joint tree and the transposed ParameterTransform
(``mb2_character_skeleton_state_backward_device``). Both run on torch's current stream and never leave the device, so a loss on joint
positions or rotations after ``torch_ik.solve_ik`` back-propagates to the solver's inputs without a host round trip.
"""
from __future__ import annotations

import torch
from torch.autograd.function import once_differentiable

from . import character as mc
from . import solver as ms

_handles = {}


def _device_character(character, device: torch.device) -> ms.DeviceCharacter:
    """One DeviceCharacter per (character, device), kept for the life of the process like torch_ik's solver functions."""
    index = device.index if device.index is not None else torch.cuda.current_device()
    if isinstance(character, ms.DeviceCharacter):
        if character.device != index:
            raise ValueError(f"model parameters are on cuda:{index} but the device character lives on cuda:{character.device}")
        return character
    key = (id(character), index)
    if key not in _handles:
        _handles[key] = (character, ms.DeviceCharacter(character, index))  # the character is kept alive so that its id stays unique
    return _handles[key][1]


class _SkeletonState(torch.autograd.Function):
    @staticmethod
    def forward(ctx, dc, model_parameters):
        n, J = dc.character.num_params, dc.character.num_joints
        dev = model_parameters.device
        theta = model_parameters.detach().to(torch.float32).reshape(-1, n).contiguous()
        B = theta.shape[0]
        state = torch.empty(B, J, 8, device=dev, dtype=torch.float32)
        dc.skeleton_state_device(B, theta.data_ptr(), state.data_ptr(), torch.cuda.current_stream(dev).cuda_stream)
        ctx.dc = dc
        ctx.in_shape, ctx.in_dtype = model_parameters.shape, model_parameters.dtype
        ctx.save_for_backward(theta)
        return state.reshape(*model_parameters.shape[:-1], J, 8).to(model_parameters.dtype)

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_state):
        (theta,) = ctx.saved_tensors
        dc = ctx.dc
        B, n = theta.shape
        dev = theta.device
        g = grad_state.to(device=dev, dtype=torch.float32).reshape(B, dc.character.num_joints, 8).contiguous()
        grad_theta = torch.empty(B, n, device=dev, dtype=torch.float32)
        dc.skeleton_state_backward_device(B, theta.data_ptr(), g.data_ptr(), grad_theta.data_ptr(), torch.cuda.current_stream(dev).cuda_stream)
        return None, grad_theta.reshape(ctx.in_shape).to(ctx.in_dtype)


def model_parameters_to_skeleton_state(character, model_parameters: torch.Tensor) -> torch.Tensor:
    """Skeleton state of ``model_parameters`` ([n] or [B, n], on a CUDA device): [J, 8] or [B, J, 8] rows (t, q xyzw, s) in the input
    dtype, computed in float32. ``character`` is a ``momentum_b200.character.Character`` or a ``solver.DeviceCharacter`` on the
    tensor's device. Differentiable once with respect to ``model_parameters``."""
    if not torch.is_tensor(model_parameters) or not model_parameters.is_cuda:
        raise ValueError("model_parameters_to_skeleton_state runs on CUDA tensors (there is no CPU fallback)")
    ch = character.character if isinstance(character, ms.DeviceCharacter) else character
    if not isinstance(ch, mc.Character):
        raise ValueError("character must be a momentum_b200.character.Character or a DeviceCharacter")
    if model_parameters.dim() not in (1, 2) or model_parameters.shape[-1] != ch.num_params:
        raise ValueError(f"model_parameters must be [n] or [B, n] with n = {ch.num_params}, got {tuple(model_parameters.shape)}")
    return _SkeletonState.apply(_device_character(character, model_parameters.device), model_parameters)
