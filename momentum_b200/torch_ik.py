"""Torch front end of the batched device solver: ``solve_ik`` on CUDA tensors, with the implicit-function backward.

Mirror of ``pymomentum.solver.solve_ik`` (pymomentum/tensor_ik/tensor_ik.cpp:95-188: per batch element build the error functions, a
solver function, a solver, solve, NaN guard) for the error functions of the device path — Limit, Position, Orientation, Motion
(= ModelParametersErrorFunction) — with the same keyword names. The forward pass never leaves the GPU: targets and weights are read
from the caller's tensors (``mb2_set_targets_device`` / ``mb2_set_constraint_weights_device``), the solve runs on torch's current
stream (``mb2_solver_solve_device``) and the result is a CUDA tensor.

The backward pass is ``d_solveTensorIKProblem`` (tensor_ik.cpp:191-340) with ``d_modelParams_d_inputs``
(momentum/diff_ik/fully_differentiable_body_ik.cpp:112-238): at the solution, v = (2 J^T J)^+ dLoss/dtheta through the SVD of the
Jacobian restricted to the active parameters (singular values with s^2 < 1e-5 dropped), then
    dLoss/d weight_k       = -(grad_theta E_k / weight_k) . v
    dLoss/d input          = d/d input [ grad_theta E_k . (-v) ]
and no gradient for an element whose gradient RMS exceeds 0.01 (the solve did not converge, tensor_ik.cpp:254). v, J v, the residual
and the gradient RMS come from one device call (``mb2_solver_function_implicit_direction_device``: the Jacobian sweep, then a float64
Jacobi eigen-solve of the Gram matrix of the enabled columns in a CUDA kernel), on the current stream and without a host
synchronisation. The input contractions of the Position offsets and of every Orientation input need the motion of each constraint's
parent frame under v, one sweep over the joint tree per element: a CUDA kernel computes them
(``mb2_solver_function_input_gradients_device``). The per-block formulas on r and J v are elementwise torch. Position targets
and weights come from the Jacobian rows, Motion targets and weights are elementwise. Before it reads the handle, the backward sends it
this forward's targets, weights and offsets again, so another solve on the same cached handle in between does not change the result.
torch is plumbing here (tensors, streams, autograd bookkeeping): every kernel on the forward path is this repo's.
"""
from __future__ import annotations

from dataclasses import dataclass
from enum import IntEnum
from typing import Optional, Sequence

import numpy as np
import torch

from . import character as mc
from . import solver as ms
from . import torch_skeleton as tsk

GRADIENT_RMSE_THRESHOLD = 0.01  # tensor_ik.cpp:46


class ErrorFunctionType(IntEnum):
    """The subset of pymomentum's ErrorFunctionType served by the device path."""

    Position = 0
    Orientation = 1
    Limit = 2
    Motion = 3


class LinearSolverType(IntEnum):
    """pymomentum/tensor_ik/solver_options.h:12-26."""

    Cholesky = 0       # SubsetGaussNewtonSolverT (tensor_ik.cpp:143-148): the tile-scheduled device path (the fast one)
    QR = 1             # GaussNewtonSolverQRT (tensor_ik.cpp:153-158): Householder QR of [sqrt(lambda) I; J], the reference's default
    TrustRegionQR = 2  # TrustRegionQRT (tensor_ik.cpp:149-152): the device trust-region iteration (ik_tr_qr.cuh); levmar_lambda / line_search do not apply


@dataclass
class SolverOptions:
    """pymomentum/tensor_ik/solver_options.h:27-47. The reference defaults to QR; here the default is Cholesky, the path this
    repository accelerates (same normal equations, same minimiser); QR and TrustRegionQR run the device Householder kernels."""

    linear_solver_type: LinearSolverType = LinearSolverType.Cholesky
    levmar_lambda: float = 0.01
    min_iter: int = 4
    max_iter: int = 50
    threshold: float = 10.0
    line_search: bool = True
    verbose: bool = False


def _build(character: mc.Character, B, device, pos_parents, pos_offsets, ori_parents, ori_offsets, motion_weights, use_limit, active):
    """One cached solver function per (character, device, batch, constraint topology), on the character's DeviceCharacter and in its
    registry entry (``torch_skeleton._handle``): the plan is built once. ``pos_offsets`` / ``ori_offsets`` None with parents given select
    the instanced block (offsets per element, in the target records): the key then holds the parents only, so new values reuse it."""
    def key_of(a):
        return None if a is None else a.tobytes()

    handle = tsk._handle(character, device)
    key = (B, key_of(pos_parents), "instanced" if pos_parents is not None and pos_offsets is None else key_of(pos_offsets),
           key_of(ori_parents), "instanced" if ori_parents is not None and ori_offsets is None else key_of(ori_offsets),
           key_of(motion_weights), use_limit, active.tobytes())
    if key in handle.solver_functions:
        return handle.solver_functions[key]
    fn = ms.SkeletonSolverFunction(handle.dc, B)
    blocks = {}
    n = character.num_params
    if pos_parents is not None:
        nc = len(pos_parents)
        inst = None if pos_offsets is not None else np.zeros((B, nc, 3), np.float32)
        offs = pos_offsets if pos_offsets is not None else np.zeros((nc, 3), np.float32)
        blocks["position"] = fn.add_error_function(mc.PositionErrorFunction(pos_parents, offs, np.ones(nc, np.float32), np.zeros((B, nc, 3), np.float32), weight=1.0,
                                                                            instance_offsets=inst))
    if ori_parents is not None:
        nc = len(ori_parents)
        identity = np.tile(np.array([0, 0, 0, 1], np.float32), (nc, 1))
        inst = None if ori_offsets is not None else np.broadcast_to(identity, (B, nc, 4)).copy()
        offs = ori_offsets if ori_offsets is not None else identity
        blocks["orientation"] = fn.add_error_function(mc.OrientationErrorFunction(ori_parents, offs, np.ones(nc, np.float32), np.zeros((B, nc, 4), np.float32), weight=1.0,
                                                                                  instance_offsets=inst))
    if use_limit:
        blocks["limit"] = fn.add_error_function(mc.LimitErrorFunction(weight=1.0))
    if motion_weights is not None:
        blocks["motion"] = fn.add_error_function(mc.ModelParametersErrorFunction(motion_weights, np.zeros((B, n), np.float32), weight=1.0))
    fn.set_enabled_parameters(active)
    handle.solver_functions[key] = (fn, blocks)
    return fn, blocks


def _normalization_backward(g, q):
    """Gradient w.r.t. a raw quaternion q from the gradient g w.r.t. its normalisation q / |q|: (I - q^ q^T) g / |q|."""
    nrm = torch.linalg.vector_norm(q, dim=-1, keepdim=True)
    qh = q / nrm
    return (g - qh * (qh * g).sum(dim=-1, keepdim=True)) / nrm


class _SolveIK(torch.autograd.Function):
    @staticmethod
    def forward(ctx, cfg, theta0, efw, pos_targets, pos_weights, pos_offsets, ori_targets, ori_weights, ori_offsets, motion_targets, motion_weights):
        fn, blocks, opts, kinds = cfg["fn"], cfg["blocks"], cfg["options"], cfg["kinds"]
        dev = theta0.device
        efw32 = tsk._float32(efw, device=dev)
        saved = {}  # device copies of everything the handle was given: the backward sends them again before it reads the handle
        # per-element error-function weights (buildMomentumErrorFunctions, tensor_ik_utility.cpp:149-181): folded into the per-instance
        # constraint weights for Position / Orientation; Limit and Motion carry one weight for the whole batch on the device
        for name, tgt, w, off in (("position", pos_targets, pos_weights, pos_offsets), ("orientation", ori_targets, ori_weights, ori_offsets)):
            if name not in blocks:
                continue
            k = kinds.index(ErrorFunctionType.Position if name == "position" else ErrorFunctionType.Orientation)
            rec = tsk._float32(tgt, device=dev)
            if off is not None:  # instanced block: the record is target, then offset, per constraint
                rec = torch.cat([rec, tsk._float32(off, device=dev).expand(rec.shape)], dim=-1).contiguous()
            saved[name + "_record"] = rec
            saved[name + "_weights"] = (tsk._float32(w, device=dev) * efw32[:, k:k + 1]).contiguous()
        if "motion" in blocks:
            saved["motion_targets"] = tsk._float32(motion_targets, device=dev)
        for name, kind in (("limit", ErrorFunctionType.Limit), ("motion", ErrorFunctionType.Motion)):
            if name not in blocks:
                continue
            col = efw32[:, kinds.index(kind)]
            if not bool(torch.all(col == col[0])):
                raise ValueError(f"{name} error-function weights must be the same for every batch element on the device path")
        _SolveIK._send(cfg, efw32, saved, tsk._stream(dev))
        solver = ms.GaussNewtonSolver(opts, fn)
        theta = tsk._float32(theta0, device=dev).clone()
        solver.solve_device(theta.data_ptr(), tsk._stream(dev))
        res = solver.get_results()  # synchronises; the NaN / Inf guard (tensor_ik.cpp:168-173) already ran on the device
        ctx.cfg = cfg
        ctx.names = list(saved)
        raw = [t.detach() if t is not None else None for t in (ori_targets, ori_offsets, pos_offsets, motion_weights)]
        ctx.raw_present = [t is not None for t in raw]
        ctx.save_for_backward(theta, efw32, *saved.values(), *[t for t in raw if t is not None])
        ctx.in_dtypes = {k: (None if t is None else t.dtype) for k, t in (("efw", efw), ("pos_targets", pos_targets), ("pos_weights", pos_weights),
                                                                           ("pos_offsets", pos_offsets), ("ori_targets", ori_targets), ("ori_weights", ori_weights),
                                                                           ("ori_offsets", ori_offsets), ("motion_targets", motion_targets),
                                                                           ("motion_weights", motion_weights))}
        cfg["last_results"] = res
        return theta.to(theta0.dtype)

    @staticmethod
    def _send(cfg, efw32, saved, stream):
        """Targets, constraint weights, offsets and block weights into the cached handle (device to device, on ``stream``)."""
        fn, blocks, kinds = cfg["fn"], cfg["blocks"], cfg["kinds"]
        for name in ("position", "orientation"):
            if name in blocks:
                fn.set_targets_device(blocks[name], saved[name + "_record"].data_ptr(), stream)
                fn.set_constraint_weights_device(blocks[name], saved[name + "_weights"].data_ptr(), stream)
        for name, kind in (("limit", ErrorFunctionType.Limit), ("motion", ErrorFunctionType.Motion)):
            if name in blocks:
                fn.set_error_function_weight(blocks[name], float(efw32[0, kinds.index(kind)]))
        if "motion" in blocks:
            fn.set_targets_device(blocks["motion"], saved["motion_targets"].data_ptr(), stream)

    @staticmethod
    def backward(ctx, grad_theta):
        cfg = ctx.cfg
        fn, blocks, kinds, active = cfg["fn"], cfg["blocks"], cfg["kinds"], cfg["active"]
        tensors = ctx.saved_tensors
        theta, efw32 = tensors[0], tensors[1]
        saved = dict(zip(ctx.names, tensors[2:2 + len(ctx.names)]))
        rest = iter(tensors[2 + len(ctx.names):])
        ori_targets_raw, ori_offsets_raw, pos_offsets_raw, motion_weights_raw = [next(rest) if p else None for p in ctx.raw_present]
        dev = theta.device
        B, n = theta.shape
        stream = tsk._stream(dev)
        # another solve on the same cached handle may have run since this forward: give it this forward's inputs again
        _SolveIK._send(cfg, efw32, saved, stream)
        # v = (2 J^T J)^+ g (fully_differentiable_body_ik.cpp:78-109), J v, the residual and the gradient RMS, all on the device: the
        # Jacobian sweep and a float64 Jacobi eigen-solve of the Gram matrix of the enabled columns, on this stream
        rows = sum(cfg["block_rows"].values())
        stride = fn.jacobian_rows
        g32 = tsk._float32(grad_theta, device=dev)
        v32 = torch.empty(B, n, device=dev)
        jv32, r32 = torch.empty(B, stride, device=dev), torch.empty(B, stride, device=dev)
        rms32 = torch.empty(B, device=dev)
        fn.implicit_direction_device(theta.data_ptr(), g32.data_ptr(), v32.data_ptr(), jv32.data_ptr(), r32.data_ptr(), rms32.data_ptr(), stream)
        r = r32[:, :rows].double()                                   # [B, rows]
        ok = (rms32.double() <= GRADIENT_RMSE_THRESHOLD).double()[:, None]
        v = v32.double()
        Jv = jv32[:, :rows].double() * ok                            # [B, rows], zero for unconverged elements
        v_ok32 = (v * ok).float().contiguous()                       # the direction the input contractions use (zero for unconverged elements)
        # rows of each block in the API-parity layout: blocks in the order they were added
        grad_efw = torch.zeros(B, len(kinds), dtype=torch.float64, device=dev)
        grads = {}
        need = dict(zip(("pos_targets", "pos_weights", "pos_offsets", "ori_targets", "ori_weights", "ori_offsets", "motion_targets", "motion_weights"),
                        ctx.needs_input_grad[3:]))
        row = 0
        sizes = cfg["block_rows"]
        for name in cfg["block_order"]:
            nr = sizes[name]
            rk, Jvk = r[:, row:row + nr], Jv[:, row:row + nr]
            kind = {"position": ErrorFunctionType.Position, "orientation": ErrorFunctionType.Orientation, "limit": ErrorFunctionType.Limit, "motion": ErrorFunctionType.Motion}[name]
            k = kinds.index(kind)
            wk = efw32[:, k].double()
            # E_k = sum r^2, grad E_k = 2 J_k^T r_k (rows already carry sqrt(weight)): dLoss/dw_k = -(grad E_k / w_k) . v
            grad_efw[:, k] = torch.where(wk != 0, -2.0 * (rk * Jvk).sum(dim=1) / wk.clamp_min(1e-30) * (wk != 0), torch.zeros_like(wk))
            if name == "position":
                nc = nr // 3
                w_eff = saved["position_weights"].double()   # [B, nc] = constraint weight x error-function weight
                sq = torch.sqrt(w_eff)[:, :, None]
                Jv3, r3 = Jvk.reshape(B, nc, 3), rk.reshape(B, nc, 3)
                # rows = sqrt(w) (p - t): d/dt [grad E . (-v)] = 2 sqrt(w) (J_dev v)
                grads["pos_targets"] = 2.0 * sq * Jv3
                # d/d(constraint weight): grad E_c = 2 w J_c^T f_c -> -(2 J_c^T f_c) . v * efw = -(2 r_c . Jv_c) / w_eff * efw
                cwg = -2.0 * (r3 * Jv3).sum(dim=2) / w_eff.clamp_min(1e-30) * (w_eff != 0)
                grads["pos_weights"] = cwg * wk[:, None]
                if need["pos_offsets"] and pos_offsets_raw is not None:
                    go = torch.empty(B, nc, 3, device=dev)
                    fn.input_gradients_device(blocks["position"], theta.data_ptr(), v_ok32.data_ptr(), grad_offsets_ptr=go.data_ptr(), stream=stream)
                    grads["pos_offsets"] = tsk._batch_sum(-go.double(), pos_offsets_raw.shape)
            elif name == "orientation":
                nc = nr // 9
                if not (need["ori_targets"] or need["ori_weights"] or need["ori_offsets"]):
                    row += nr
                    continue
                gw = torch.empty(B, nc, device=dev)
                gt = torch.empty(B, nc, 4, device=dev)
                go = torch.empty(B, nc, 4, device=dev) if ori_offsets_raw is not None else None
                fn.input_gradients_device(blocks["orientation"], theta.data_ptr(), v_ok32.data_ptr(), gw.data_ptr(), tsk._ptr(go), gt.data_ptr(), stream)
                grads["ori_weights"] = -gw.double() * wk[:, None]   # the device weight is constraint weight x error-function weight
                grads["ori_targets"] = _normalization_backward(-gt.double(), ori_targets_raw.to(dev).double())
                if go is not None:
                    off = ori_offsets_raw.to(dev).double().expand(B, nc, 4)
                    grads["ori_offsets"] = tsk._batch_sum(_normalization_backward(-go.double(), off), ori_offsets_raw.shape)
            elif name == "motion":
                # E = efw 0.1 sum_i w_i^2 (theta_i - t_i)^2 over the enabled parameters with w_i > 0 (model_parameters_error_function.cpp,
                # kMotionWeight = 0.1): d/dt_i [grad E . v] = -2 s w_i^2 v_i,  d/dw_i = 4 s w_i (theta_i - t_i) v_i
                mw = torch.as_tensor(cfg["motion_weights"], device=dev, dtype=torch.float64)
                on = torch.as_tensor(active[:n] & (cfg["motion_weights"] > 0), device=dev)
                sc = 0.1 * wk[:, None]
                vv = (v * ok) * on
                grads["motion_targets"] = 2.0 * sc * mw * mw * vv
                gmw = -4.0 * sc * mw * (theta.double() - saved["motion_targets"].double()) * vv
                if motion_weights_raw is not None:  # the device block holds the first row of [B, n] weights for the whole batch
                    grads["motion_weights"] = gmw.sum(dim=0) if motion_weights_raw.dim() == 1 else torch.cat([gmw.sum(dim=0, keepdim=True), torch.zeros_like(gmw[1:])])
            row += nr
        dt = ctx.in_dtypes

        def out(name):
            t = grads.get(name)
            return None if t is None or dt[name] is None or not need[name] else t.to(dt[name])

        return (None, None, grad_efw.to(dt["efw"]), out("pos_targets"), out("pos_weights"), out("pos_offsets"), out("ori_targets"), out("ori_weights"),
                out("ori_offsets"), out("motion_targets"), out("motion_weights"))


def _device_view(ptr: int, shape, device):
    """float32 CUDA tensor over foreign device memory (the handle's Jacobian buffer) through __cuda_array_interface__."""

    class _Arr:
        pass

    a = _Arr()
    a.__cuda_array_interface__ = {"shape": tuple(shape), "typestr": "<f4", "data": (int(ptr), False), "version": 2}
    return torch.as_tensor(a, device=device)


def solve_ik(character: mc.Character, active_parameters, model_parameters_init: torch.Tensor, active_error_functions: Sequence[ErrorFunctionType],
             error_function_weights: torch.Tensor, options: Optional[SolverOptions] = None,
             position_cons_parents=None, position_cons_offsets=None, position_cons_weights=None, position_cons_targets=None,
             orientation_cons_parents=None, orientation_cons_offsets=None, orientation_cons_weights=None, orientation_cons_targets=None,
             motion_targets=None, motion_weights=None) -> torch.Tensor:
    """Batched IK on the GPU; arguments as pymomentum.solver.solve_ik. ``model_parameters_init`` [B, n] must live on a CUDA device;
    constraint parents are shared by the batch ([nc]); offsets are shared ([nc, 3] / [nc, 4]) or per element ([B, nc, 3] / [B, nc, 4]),
    as tensors or arrays; targets and weights are per element.

    Differentiable w.r.t. ``error_function_weights``, the position targets, weights and offsets, the orientation targets, weights and
    offsets, and the motion targets and weights. Offsets that are batched or require grad use the instanced device block (offsets in
    the per-element records), whose cached handle does not depend on the offset values; other offsets keep the shared block."""
    if not model_parameters_init.is_cuda:
        raise ValueError("momentum_b200.torch_ik.solve_ik runs on CUDA tensors (there is no CPU fallback)")
    options = options or SolverOptions()
    dev = model_parameters_init.device
    B, n = model_parameters_init.shape
    kinds = [ErrorFunctionType(k) for k in active_error_functions]
    efw = error_function_weights
    if efw.dim() == 1:
        efw = efw[None].expand(B, -1)
    active = np.asarray(active_parameters.cpu() if torch.is_tensor(active_parameters) else active_parameters, bool)

    def np_or_none(x, dt):
        return None if x is None else np.ascontiguousarray(x.detach().cpu().numpy() if torch.is_tensor(x) else x, dt)

    def offsets(x, use, count, default):
        """(shared offsets for the cache key, or None for the instanced block; the offsets as a tensor for the instanced block)"""
        if not use:
            return None, None
        if x is None:
            return np.tile(np.asarray(default, np.float32), (count, 1)), None
        if (torch.is_tensor(x) and x.requires_grad) or np.ndim(x) == 3:
            return None, x if torch.is_tensor(x) else torch.as_tensor(np.asarray(x, np.float32))
        return np_or_none(x, np.float32), None

    use_pos = ErrorFunctionType.Position in kinds and position_cons_parents is not None
    use_ori = ErrorFunctionType.Orientation in kinds and orientation_cons_parents is not None
    use_motion = ErrorFunctionType.Motion in kinds and motion_targets is not None
    pp = np_or_none(position_cons_parents, np.int32) if use_pos else None
    op = np_or_none(orientation_cons_parents, np.int32) if use_ori else None
    po, po_t = offsets(position_cons_offsets, use_pos, 0 if pp is None else len(pp), [0, 0, 0])
    oo, oo_t = offsets(orientation_cons_offsets, use_ori, 0 if op is None else len(op), [0, 0, 0, 1])
    mw = None
    if use_motion:
        mwt = motion_weights if motion_weights is not None else torch.ones(n)
        mw = np_or_none(mwt[0] if (torch.is_tensor(mwt) and mwt.dim() == 2) else mwt, np.float32)
    fn, blocks = _build(character, B, dev, pp, po, op, oo, mw, ErrorFunctionType.Limit in kinds, active)
    order = [name for name in ("position", "orientation", "limit", "motion") if name in blocks]
    block_rows = {}
    for name in order:
        block_rows[name] = {"position": lambda: 3 * len(pp), "orientation": lambda: 9 * len(op),
                            "limit": lambda: mc.jacobian_size(character, mc.LimitErrorFunction()), "motion": lambda: int(((mw > 0) & active[: len(mw)]).sum())}[name]()
    lst = LinearSolverType(options.linear_solver_type)
    linear = {LinearSolverType.Cholesky: ms.LINEAR_SOLVER_CHOLESKY, LinearSolverType.QR: ms.LINEAR_SOLVER_QR, LinearSolverType.TrustRegionQR: ms.LINEAR_SOLVER_TRUST_REGION_QR}[lst]
    # Cholesky: SubsetGaussNewtonSolverT's line search (c1 = 1e-4 with the directional derivative); QR: GaussNewtonSolverQRT's (same rule,
    # gauss_newton_solver_qr.cpp:118-143): both are the subset variant on the device. TrustRegionQR takes the plain SolverOptions
    # (tensor_ik.cpp:149-152): iterations / threshold only, radius 1.
    opts = ms.GaussNewtonSolverOptions(min_iterations=options.min_iter, max_iterations=options.max_iter, threshold=options.threshold, regularization=options.levmar_lambda,
                                       do_line_search=options.line_search, subset_line_search=True, linear_solver=linear)
    cfg = {"fn": fn, "blocks": blocks, "options": opts, "kinds": kinds, "active": active, "block_order": order, "block_rows": block_rows, "motion_weights": mw}
    ones = lambda nc: torch.ones(B, nc, device=dev)
    pw = position_cons_weights if position_cons_weights is not None else (ones(len(pp)) if use_pos else None)
    ow = orientation_cons_weights if orientation_cons_weights is not None else (ones(len(op)) if use_ori else None)
    mwt = motion_weights if (use_motion and torch.is_tensor(motion_weights)) else None
    out = _SolveIK.apply(cfg, model_parameters_init, efw, position_cons_targets if use_pos else None, pw if use_pos else None, po_t,
                         orientation_cons_targets if use_ori else None, ow if use_ori else None, oo_t, motion_targets if use_motion else None, mwt)
    solve_ik.last_results = cfg.get("last_results")
    return out
