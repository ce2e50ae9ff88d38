"""One DeviceCharacter per (character, device) for the whole torch layer: ``solve_ik``'s solver functions are built on the handle the
skeleton, skinning and mesh operations use (``torch_skeleton._handle``), and cached in its registry entry.

The CPU tests replace ``DeviceCharacter`` and ``SkeletonSolverFunction`` with fakes that count constructions and drive the registry and
``torch_ik._build`` directly. The GPU test runs ``solve_ik`` -> skinning -> normals with a backward on a skinned humanoid72 and compares
it bit for bit with the same calls on solver functions that each upload their own character and on a DeviceCharacter made directly.
"""
import copy
import dataclasses

import numpy as np
import pytest
import torch

from momentum_b200 import character as mc
from momentum_b200 import solver as ms
from momentum_b200 import torch_ik as ti
from momentum_b200 import torch_skeleton as tsk

DEV = torch.device("cuda", 0)


# ---- CPU: the registry with fake handles ---------------------------------------------------------------------------------------------
@pytest.fixture
def fakes(monkeypatch):
    """An empty registry, and DeviceCharacter / SkeletonSolverFunction fakes that record each construction."""
    made = {"characters": [], "functions": []}

    class FakeDeviceCharacter:
        def __init__(self, character, device=0, lib_path=None):
            self.character, self.device = character, device
            made["characters"].append(self)

    class FakeSolverFunction:
        def __init__(self, dev_character, batch):
            self.dev_character, self.batch, self.blocks = dev_character, batch, []
            made["functions"].append(self)

        def add_error_function(self, ef):
            self.blocks.append(ef)
            return len(self.blocks) - 1

        def set_enabled_parameters(self, active):
            self.active = active

    monkeypatch.setattr(tsk, "_handles", {})
    monkeypatch.setattr(ms, "DeviceCharacter", FakeDeviceCharacter)
    monkeypatch.setattr(ms, "SkeletonSolverFunction", FakeSolverFunction)
    return made


def _skinned_chain():
    ch = mc.create_test_character(5)
    ch.skinning = mc.synthetic_tube_mesh(ch, 4, 6, 5)
    ch.blend_shape = mc.synthetic_blend_shape(ch, ch.skinning, 3, 1)
    return ch


def _topologies(ch):
    """(pos_parents, pos_offsets, ori_parents, ori_offsets, motion_weights, use_limit, active) of four constraint topologies; every call
    makes new arrays, so equal keys are equal values, not the same objects."""
    n = ch.num_params
    pp, po = np.array([1, 2, 4], np.int32), np.full((3, 3), 0.25, np.float32)
    op, oo = np.array([2, 3], np.int32), np.tile(np.array([0, 0, 0, 1], np.float32), (2, 1))
    active = np.ones(n, bool)
    return [(pp, po, None, None, None, False, active),
            (pp, None, op, None, None, True, active),
            (pp, po, op, oo, np.ones(n, np.float32), False, active),
            (pp, po, None, None, None, False, np.arange(n) != 6)]


def _build_all(ch, batches, device=DEV):
    return [ti._build(ch, B, device, *t) for B in batches for t in _topologies(ch)]


def test_one_device_character_per_character_and_device(fakes):
    ch = _skinned_chain()
    built = _build_all(ch, (1, 4, 7))
    dc = tsk._device_character(ch, DEV)
    assert fakes["characters"] == [dc]
    assert len(fakes["functions"]) == 12 and len(tsk._handle(ch, DEV).solver_functions) == 12
    for fn, _ in built:
        assert fn.dev_character is dc  # built on the registry's handle
    # another device and another character each get their own handle
    other = tsk._device_character(ch, torch.device("cuda", 1))
    assert other is not dc and other.device == 1
    twin = copy.copy(ch)
    assert tsk._device_character(twin, DEV) not in (dc, other)
    assert len(fakes["characters"]) == 3 and len(fakes["functions"]) == 12


def test_solver_functions_are_reused_for_equal_keys(fakes):
    ch = _skinned_chain()
    first = _build_all(ch, (2, 5))
    again = _build_all(ch, (2, 5))
    assert all(a[0] is b[0] and a[1] == b[1] for a, b in zip(first, again))
    assert len(fakes["functions"]) == 8 and len(fakes["characters"]) == 1
    # the operations of torch_skeleton reuse it too
    assert tsk._device_character(ch, DEV) is first[0][0].dev_character
    # reassigning the same objects is not a replacement
    ch.skinning, ch.blend_shape = ch.skinning, ch.blend_shape
    assert _build_all(ch, (2,))[0][0] is first[0][0] and len(fakes["characters"]) == 1


@pytest.mark.parametrize("replace", ["skinning", "faces", "blend_shape"])
def test_a_replaced_mesh_makes_a_new_handle_and_rebuilds_its_solver_functions_once(fakes, replace):
    ch = _skinned_chain()
    old = _build_all(ch, (3,))
    old_dc = tsk._device_character(ch, DEV)
    if replace == "skinning":
        ch.skinning = dataclasses.replace(ch.skinning)
    elif replace == "faces":
        ch.skinning.faces = ch.skinning.faces[::-1].copy()
    else:
        ch.blend_shape = mc.synthetic_blend_shape(ch, ch.skinning, 3, 2)
    new = _build_all(ch, (3,))
    dc = tsk._device_character(ch, DEV)
    assert dc is not old_dc and len(fakes["characters"]) == 2
    assert len(fakes["functions"]) == 8
    for (fn, _), (fn_old, _) in zip(new, old):
        assert fn is not fn_old and fn.dev_character is dc and fn_old.dev_character is old_dc
    assert len(tsk._handle(ch, DEV).solver_functions) == 4  # the old entry's solver functions went with it
    assert [fn for fn, _ in _build_all(ch, (3,))] == [fn for fn, _ in new]
    assert len(fakes["functions"]) == 8 and len(fakes["characters"]) == 2


# ---- GPU: solve_ik -> skin_points -> normals on a skinned humanoid72 ----------------------------------------------------------------
def _fit_then_skin(ch, efs, skin_with):
    """solve_ik on two topologies (Position; Position + Orientation) at two batch sizes, each result skinned and its normals taken on
    ``skin_with``, one loss over all of it and its backward: (outputs, gradients of the targets and weights) as host arrays."""
    pos, ori = efs
    weights = {ti.ErrorFunctionType.Position: pos.weight, ti.ErrorFunctionType.Orientation: ori.weight}  # the legacy weights converge
    rng = np.random.default_rng(3)
    n = ch.num_params
    active = np.ones(n, bool)
    opts = ti.SolverOptions(levmar_lambda=0.01, min_iter=20, max_iter=20, threshold=1.0, line_search=True)
    outputs, leaves, loss = [], [], 0.0
    for B in (2, 5):
        theta_star = np.zeros((B, n))
        theta_star[:, 7:] = rng.uniform(-0.3, 0.3, (B, n - 7))
        pt = torch.from_numpy(mc.world_points(ch, theta_star, pos.parents, pos.offsets)).to(DEV).requires_grad_(True)
        ot = torch.from_numpy(mc.world_rotations(ch, theta_star, ori.parents, ori.offsets)).to(DEV).requires_grad_(True)
        pw = torch.ones(B, len(pos.parents), device=DEV, dtype=torch.float64, requires_grad=True)
        leaves += [pt, ot, pw]
        for kinds, orientation in (([ti.ErrorFunctionType.Position], {}),
                                   ([ti.ErrorFunctionType.Position, ti.ErrorFunctionType.Orientation],
                                    dict(orientation_cons_parents=ori.parents, orientation_cons_offsets=ori.offsets, orientation_cons_targets=ot))):
            efw = torch.tensor([[weights[k] for k in kinds]] * B, device=DEV, dtype=torch.float64)
            theta = ti.solve_ik(ch, active, torch.zeros(B, n, device=DEV), kinds, efw, opts, position_cons_parents=pos.parents,
                                position_cons_offsets=pos.offsets, position_cons_weights=pw, position_cons_targets=pt, **orientation)
            points = tsk.skin_points(skin_with, tsk.model_parameters_to_skeleton_state(skin_with, theta.double()))
            normals = tsk.compute_vertex_normals(skin_with, points)
            wv = torch.from_numpy(rng.normal(size=points.shape)).to(DEV)
            loss = loss + (points * wv).sum() + (normals * wv.flip(-1)).sum()
            outputs += [theta, points, normals]
    loss.backward()
    grads = [t.grad for t in leaves]
    assert all(g is not None for g in grads) and min(float(g.abs().max()) for g in grads) > 0.0
    return [t.detach().cpu().numpy() for t in outputs + grads]


@pytest.mark.gpu
def test_solve_ik_then_skinning_uploads_the_character_once_and_matches_separate_handles(monkeypatch):
    from momentum_b200.problems import humanoid_problem

    ch, efs, _, _ = humanoid_problem(1)
    ch.skinning = mc.synthetic_tube_mesh(ch, 4, 6, 5)
    real_device_character, real_solver_function = ms.DeviceCharacter, ms.SkeletonSolverFunction
    made = []

    class CountingDeviceCharacter(real_device_character):
        def __init__(self, *args, **kwargs):
            made.append(self)
            super().__init__(*args, **kwargs)

    with monkeypatch.context() as m:
        m.setattr(ms, "DeviceCharacter", CountingDeviceCharacter)
        shared = _fit_then_skin(ch, efs, ch)
    assert len(made) == 1 and made[0] is tsk._device_character(ch, DEV)
    functions = tsk._handle(ch, DEV).solver_functions
    assert len(functions) == 4 and all(fn.dev_character is made[0] for fn, _ in functions.values())

    # the parent's paths: a DeviceCharacter per solver function, and one made directly for the skinning and normals
    twin = copy.copy(ch)
    with monkeypatch.context() as m:
        m.setattr(ms, "SkeletonSolverFunction", lambda dc, B: real_solver_function(dc.character, B, device=dc.device))
        separate = _fit_then_skin(twin, efs, ms.DeviceCharacter(twin, 0))
    assert not any(fn.dev_character is tsk._device_character(twin, DEV) for fn, _ in tsk._handle(twin, DEV).solver_functions.values())
    assert len(shared) == len(separate)
    for a, b in zip(shared, separate):
        assert a.shape == b.shape and np.array_equal(a, b)
