"""model_parameters_to_positions and joint_parameters_to_positions on the device and their backward, against float64 restatements.

The reference is ``_fk64`` of test_skeleton_state (the forward kinematics written in torch, float64), the point t_a + rot(q_a, s_a off)
of each point's joint a, and float64 autograd through both for the gradients with respect to the parameters and the offsets. A float32
result x passes when ||x - x64||_inf <= K * max(||x64||_inf, 1) per instance, K pinned at about four times the worst value measured
over the fixtures, point sets and layouts below (emulator and H100, in the comments). The self-checks show that the bounds reject a
backward without ln 2, one that attaches each point to its parent's parent, and an offset gradient that rotates by q instead of conj(q).
"""
import ctypes
import math

import numpy as np
import pytest
import torch

from momentum_b200 import character as mc
from momentum_b200 import solver as ms
from tests import emu_lib
from tests.test_skeleton_state import FIXTURES, _ancestry_parameters, _bound_ratio, _fk64, _joint_parameters, _pt_dense, _qrot

# worst measured ratio (see the module docstring) on the emulator / on an H100 80GB HBM3 at a 700 W power limit: positions 7.9e-7 /
# 7.6e-7, parameter gradients 1.6e-6 / 9.4e-7, offset gradients 1.1e-6 / 1.1e-6; the wrong backwards below are off by 100 K or more
K_POS = 3e-6
K_GRAD = 6e-6
K_OFF = 4.5e-6


# ---- inputs -----------------------------------------------------------------------------------------------------------------------------
def _children(ch):
    return {int(p) for p in ch.parents if p >= 0}


def _point_sets(ch):
    """name -> parents: several points per joint with joints that have none (roots included), points on the roots only, one point on
    the last leaf, and none."""
    J = ch.num_joints
    rng = np.random.default_rng(J)
    roots = [j for j in range(J) if ch.parents[j] < 0]
    used = rng.choice(J, size=max(2, J // 3), replace=False)
    several = np.concatenate([rng.choice(used, size=min(3 * J, 90)), roots])
    leaf = max(j for j in range(J) if j not in _children(ch))
    return {"several": several.astype(np.int32), "roots": np.array(roots * 2, np.int32), "leaf": np.array([leaf], np.int32),
            "none": np.zeros(0, np.int32)}


def _inputs(ch, joint, B, N, batched, seed):
    rng = np.random.default_rng(seed)
    theta = rng.uniform(-0.5, 0.5, (B, ch.num_params)).astype(np.float32)
    params = _joint_parameters(ch, theta).reshape(B, -1).numpy().astype(np.float32) if joint else theta
    off = rng.normal(scale=0.3, size=(B, N, 3) if batched else (N, 3)).astype(np.float32)
    G = rng.normal(size=(B, N, 3)).astype(np.float32)
    return params, off, G


# ---- float64 reference ----------------------------------------------------------------------------------------------------------------
def _jp64(ch, joint, params):
    """float64 joint parameters [B, J, 7] of params, differentiable with respect to params"""
    if joint:
        return params.reshape(params.shape[0], ch.num_joints, 7)
    return (params @ _pt_dense(ch).T + torch.from_numpy(ch.pt_offsets.astype(np.float64))).reshape(-1, ch.num_joints, 7)


def _positions64(ch, jp, parents, off):
    st = _fk64(ch, jp)[:, torch.as_tensor(parents, dtype=torch.long)]
    return st[..., :3] + _qrot(st[..., 3:7], st[..., 7:8] * off)


def _reference(ch, joint, params, parents, off, G, attach=None):
    """float64 (positions, dLoss/d params, dLoss/d offsets) of Loss = sum(positions * G). attach(st, p): positions moved as if attached
    elsewhere (self-checks)."""
    x = torch.as_tensor(np.asarray(params, np.float64)).requires_grad_(True)
    o = torch.as_tensor(np.asarray(off, np.float64)).requires_grad_(True)
    jp = _jp64(ch, joint, x)
    p = _positions64(ch, jp, parents, o)
    if attach is not None:
        p = attach(_fk64(ch, jp), p)
    (p * torch.as_tensor(np.asarray(G, np.float64))).sum().backward()
    return p.detach().numpy(), x.grad.numpy(), (o.grad if o.grad is not None else torch.zeros_like(o)).numpy()


def _ratio(x, x64):
    B = x64.shape[0]
    return _bound_ratio(np.asarray(x).reshape(B, -1), np.asarray(x64).reshape(B, -1)) if x64.size else np.zeros(B)


# ---- CPU: the emulator runs the kernel's pass functions lane by lane --------------------------------------------------------------------
# the emulator entries' signatures (tests/emu/emu_positions.cu): mb2_character_create's nine arguments, then variant, batch, parameters,
# N, parents, offsets, offsets batched, and the outputs (forward: positions; backward: upstream gradient, parameter and offset gradients)
_CHARACTER = [ctypes.c_int32, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int32] + [ctypes.c_void_p] * 4
_POINTS = [ctypes.c_int32, ctypes.c_int32, ctypes.c_void_p, ctypes.c_int32, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int32]


@pytest.fixture(scope="module")
def emu():
    L = emu_lib.load()
    L.emu_positions.argtypes = _CHARACTER + _POINTS + [ctypes.c_void_p]
    L.emu_positions_backward.argtypes = _CHARACTER + _POINTS + [ctypes.c_void_p] * 3
    return L


def _emu_forward(L, ch, joint, params, parents, off):
    keep = []
    params, off, parents = (np.ascontiguousarray(a) for a in (params, off, parents))
    B, N = params.shape[0], parents.shape[0]
    out = np.full((B, N, 3), np.nan, np.float32)
    rc = L.emu_positions(*emu_lib.character_args(ch, keep), int(joint), B, params.ctypes.data, N, parents.ctypes.data, off.ctypes.data,
                         int(off.ndim == 3), out.ctypes.data)
    assert rc == 0, L.emu_last_error().decode()
    return out


def _emu_backward(L, ch, joint, params, parents, off, G):
    keep = []
    params, off, parents, G = (np.ascontiguousarray(a) for a in (params, off, parents, G))
    gp = np.full(params.shape, np.nan, np.float32)
    go = np.full(off.shape, np.nan, np.float32)
    rc = L.emu_positions_backward(*emu_lib.character_args(ch, keep), int(joint), params.shape[0], params.ctypes.data, parents.shape[0],
                                  parents.ctypes.data, off.ctypes.data, int(off.ndim == 3), G.ctypes.data, gp.ctypes.data, go.ctypes.data)
    assert rc == 0, L.emu_last_error().decode()
    return gp, go


def _offset_ratio(go, go64, batched):
    """the offset gradient's ratio: per instance when batched, else over the batch sum"""
    return _ratio(go, go64) if batched else _ratio(go[None], go64[None])


@pytest.mark.parametrize("J", [3, 22, 129])
def test_emulated_forward_known_answer(emu, J):
    """KA-1 (forward_kinematics_test.cpp:78-87): the point (1, 1, 1) on joint 2 of the test character."""
    ch = mc.create_test_character(J)
    theta = np.zeros((1, ch.num_params), np.float32)
    theta[0, :10] = [1.0, 1.0, 1.0, np.pi, 0.0, -np.pi, 0.1, np.pi, np.pi, -np.pi]
    p = _emu_forward(emu, ch, False, theta, np.array([2], np.int32), np.ones((1, 3), np.float32))
    assert np.linalg.norm(p[0, 0] - np.array([-1.14354682, 3.14354706, -0.0717732906])) <= 1e-6


@pytest.mark.parametrize("batched", [False, True], ids=["shared", "batched"])
@pytest.mark.parametrize("joint", [False, True], ids=["model", "joint"])
@pytest.mark.parametrize("name", list(FIXTURES))
def test_emulated_forward_and_backward_meet_the_float64_bounds(emu, name, joint, batched):
    ch = FIXTURES[name]()
    for k, (set_name, parents) in enumerate(_point_sets(ch).items()):
        params, off, G = _inputs(ch, joint, 3, len(parents), batched, 100 + k)
        p64, gp64, go64 = _reference(ch, joint, params, parents, off, G)
        p = _emu_forward(emu, ch, joint, params, parents, off)
        gp, go = _emu_backward(emu, ch, joint, params, parents, off, G)
        assert _ratio(p, p64).max() <= K_POS, (set_name, _ratio(p, p64).max())
        assert _ratio(gp, gp64).max() <= K_GRAD, (set_name, _ratio(gp, gp64).max())
        assert _offset_ratio(go, go64, batched).max() <= K_OFF, (set_name, _offset_ratio(go, go64, batched).max())
        if len(parents) == 0:
            assert p.shape == (3, 0, 3) and np.all(gp == 0.0) and go.size == 0


def test_bounds_reject_a_wrong_backward():
    """a missing ln 2 on the scale rows, each point attached to its parent's parent, and the offset gradient rotated by q instead of
    conj(q), each against the float64 gradient"""
    for name in ("chain6", "humanoid72", "humanoid72_far", "two_roots"):
        ch = FIXTURES[name]()
        parents = np.array([j for j in _point_sets(ch)["several"] if ch.parents[j] >= 0], np.int32)
        params, off, G = _inputs(ch, True, 4, len(parents), True, 7)
        _, g64, go64 = _reference(ch, True, params, parents, off, G)
        no_ln2 = g64.reshape(4, -1, 7).copy()
        no_ln2[..., 6] /= math.log(2.0)
        assert _ratio(no_ln2, g64).min() > 100 * K_GRAD, name
        gpar = torch.as_tensor(ch.parents[parents].astype(np.int64))

        def grandparent(st, p):  # the same point, moving rigidly with the parent of its joint
            a = st[:, gpar]
            rel = (_qrot(a[..., 3:7] * torch.tensor([-1.0, -1.0, -1.0, 1.0], dtype=torch.float64), p - a[..., :3]) / a[..., 7:8]).detach()
            return a[..., :3] + _qrot(a[..., 3:7], a[..., 7:8] * rel)

        _, g_wrong, _ = _reference(ch, True, params, parents, off, G, attach=grandparent)
        assert _ratio(g_wrong, g64).min() > 100 * K_GRAD, name
        st = _fk64(ch, _jp64(ch, True, torch.as_tensor(params, dtype=torch.float64)))[:, torch.as_tensor(parents, dtype=torch.long)]
        go_wrong = (st[..., 7:8] * _qrot(st[..., 3:7], torch.as_tensor(G, dtype=torch.float64))).numpy()
        assert _ratio(go_wrong, go64).min() > 100 * K_OFF, name


@pytest.mark.parametrize("name", ["humanoid72", "bodyhands300", "two_roots"])
def test_emulated_sparse_upstream_gradient_reaches_only_the_ancestry(emu, name):
    ch = FIXTURES[name]()
    parents = _point_sets(ch)["several"]
    N = len(parents)
    params, off, G = _inputs(ch, False, 3, N, True, 31)
    picks = [N - 1, N // 2, 0]
    for b, i in enumerate(picks):
        keep = G[b, i].copy(); G[b] = 0.0; G[b, i] = keep
    gp, go = _emu_backward(emu, ch, False, params, parents, off, G)
    _, gp64, _ = _reference(ch, False, params, parents, off, G)
    assert _ratio(gp, gp64).max() <= K_GRAD
    for b, i in enumerate(picks):
        allowed = _ancestry_parameters(ch, int(parents[i]))
        outside = [p for p in range(ch.num_params) if p not in allowed]
        assert np.all(gp[b, outside] == 0.0), (name, i)
        assert np.any(gp[b, sorted(allowed)] != 0.0)
        rows = [k for k in range(N) if k != i]
        assert np.all(go[b, rows] == 0.0) and np.any(go[b, i] != 0.0)


def test_bad_arguments_are_rejected_before_any_library_call(monkeypatch):
    from momentum_b200 import torch_skeleton as tsk

    def no_call(*a, **k):
        raise AssertionError("library reached")

    monkeypatch.setattr(ms, "load_library", no_call)
    monkeypatch.setattr(ms, "DeviceCharacter", type("NoDevice", (), {"__init__": no_call}))
    ch = mc.create_test_character(4)
    n, J = ch.num_params, ch.num_joints
    th, jp, off = torch.zeros(2, n), torch.zeros(2, 7 * J), torch.zeros(3, 3)
    for f, x in ((tsk.model_parameters_to_positions, th), (tsk.joint_parameters_to_positions, jp)):
        with pytest.raises(ValueError, match="CUDA"):
            f(ch, x, [0, 1, 3], off)
        with pytest.raises(ValueError, match="CUDA"):
            f(ch, x, np.array([0, 1, 3]), torch.zeros(2, 3, 3, dtype=torch.float64))
        with pytest.raises(ValueError, match="must be"):
            f(ch, x[:, 1:], [0, 1, 3], off)
        with pytest.raises(ValueError, match="must be"):
            f(ch, x[None], [0, 1, 3], off)
        with pytest.raises(ValueError, match=r"\[0, 4\)"):
            f(ch, x, [0, 1, 4], off)
        with pytest.raises(ValueError, match=r"\[0, 4\)"):
            f(ch, x, torch.tensor([0, -1, 2]), off)
        with pytest.raises(ValueError, match="integer"):
            f(ch, x, torch.tensor([0.0, 1.0, 2.0]), off)
        with pytest.raises(ValueError, match="integer"):
            f(ch, x, [0.5, 1, 2], off)
        with pytest.raises(ValueError, match=r"\[N\]"):
            f(ch, x, [[0, 1, 2]], off)
        with pytest.raises(ValueError, match="offsets must be"):
            f(ch, x, [0, 1], off)
        with pytest.raises(ValueError, match="offsets must be"):
            f(ch, x[0], [0, 1, 3], torch.zeros(2, 3, 3))
        with pytest.raises(ValueError, match="offsets must be"):
            f(ch, x, [0, 1, 3], torch.zeros(3, 3, 3))
        with pytest.raises(ValueError, match="floating-point"):
            f(ch, x, [0, 1, 3], torch.zeros(3, 3, dtype=torch.int32))


# ---- GPU --------------------------------------------------------------------------------------------------------------------------------
def _op(joint):
    from momentum_b200 import torch_skeleton as tsk

    return tsk.joint_parameters_to_positions if joint else tsk.model_parameters_to_positions


def _dev(ch, joint, params, parents, off, G, character=None):
    """device positions and both gradients through the torch wrapper"""
    x = torch.from_numpy(np.ascontiguousarray(params)).cuda().requires_grad_(True)
    o = torch.from_numpy(np.ascontiguousarray(off)).cuda().requires_grad_(True)
    p = _op(joint)(character if character is not None else ch, x, parents, o)
    p.backward(torch.from_numpy(np.ascontiguousarray(G)).cuda())
    return p.detach(), x.grad, o.grad


@pytest.mark.gpu
@pytest.mark.parametrize("batched", [False, True], ids=["shared", "batched"])
@pytest.mark.parametrize("joint", [False, True], ids=["model", "joint"])
@pytest.mark.parametrize("name", list(FIXTURES))
def test_device_meets_the_float64_bounds(name, joint, batched):
    from momentum_b200 import torch_skeleton as tsk

    ch = FIXTURES[name]()
    for k, (set_name, parents) in enumerate(_point_sets(ch).items()):
        params, off, G = _inputs(ch, joint, 8, len(parents), batched, 200 + k)
        p64, gp64, go64 = _reference(ch, joint, params, parents, off, G)
        p, gp, go = (t.cpu().numpy() for t in _dev(ch, joint, params, parents, off, G))
        assert _ratio(p, p64).max() <= K_POS, (set_name, _ratio(p, p64).max())
        assert _ratio(gp, gp64).max() <= K_GRAD, (set_name, _ratio(gp, gp64).max())
        assert _offset_ratio(go, go64, batched).max() <= K_OFF, (set_name, _offset_ratio(go, go64, batched).max())
        if not joint and len(parents):
            # against the skeleton state's float32 rows transformed in float64
            st = tsk.model_parameters_to_skeleton_state(ch, torch.from_numpy(params).cuda()).double().cpu()[:, torch.as_tensor(parents, dtype=torch.long)]
            ref = (st[..., :3] + _qrot(st[..., 3:7], st[..., 7:8] * torch.as_tensor(off, dtype=torch.float64))).numpy()
            assert _ratio(p, ref).max() <= K_POS, set_name


def _calls(dc, joint, params, parents, off, G, need=(True, True)):
    """one forward and one backward through DeviceCharacter on the current stream: positions, parameter and offset gradients"""
    B = params.shape[0]
    s = torch.cuda.current_stream().cuda_stream
    p = torch.empty(B, len(parents), 3, device="cuda")
    dc.positions_device(joint, B, params.data_ptr(), parents, off.data_ptr(), off.dim() == 3, p.data_ptr(), stream=s)
    gp = torch.empty_like(params) if need[0] else None
    go = torch.empty_like(off) if need[1] else None
    dc.positions_backward_device(joint, B, params.data_ptr(), parents, off.data_ptr(), off.dim() == 3, G.data_ptr(),
                                 0 if gp is None else gp.data_ptr(), 0 if go is None else go.data_ptr(), stream=s)
    return p, gp, go


@pytest.mark.gpu
@pytest.mark.parametrize("joint", [False, True], ids=["model", "joint"])
def test_bitwise_invariance(joint):
    from momentum_b200 import torch_skeleton as tsk

    ch = mc.humanoid72()[0]
    B = 4096
    parents = _point_sets(ch)["several"]
    N = len(parents)
    params, off, G = (torch.from_numpy(a).cuda() for a in _inputs(ch, joint, B, N, False, 41))
    dc = tsk._device_character(ch, params.device)
    p1, gp1, go1 = _calls(dc, joint, params, parents, off, G)
    p2, gp2, go2 = _calls(dc, joint, params, parents, off, G)
    assert torch.equal(p1, p2) and torch.equal(gp1, gp2) and torch.equal(go1, go2)
    rep = off.expand(B, N, 3).contiguous()
    pr, gpr, gor = _calls(dc, joint, params, parents, rep, G)
    assert torch.equal(pr, p1) and torch.equal(gpr, gp1)
    # the shared-offset gradient is the batch sum of the per-instance ones
    go64 = gor.double().sum(0).cpu().numpy()
    assert _ratio(go1.cpu().numpy()[None], go64[None]).max() <= K_OFF
    for b in [0, 1, B // 3, B - 1]:
        pb, gpb, gob = _calls(dc, joint, params[b:b + 1].contiguous(), parents, rep[b:b + 1].contiguous(), G[b:b + 1].contiguous())
        assert torch.equal(pb, p1[b:b + 1]) and torch.equal(gpb, gp1[b:b + 1]) and torch.equal(gob, gor[b:b + 1]), b
    clone = ms.C.c_void_p()
    dc._check(dc._L.mb2_character_clone(dc._h, 0, ms.C.byref(clone)))
    try:
        other = ms.DeviceCharacter.__new__(ms.DeviceCharacter)
        other._L, other._h = dc._L, clone.value
        pc, gpc, goc = _calls(other, joint, params, parents, off, G)
        torch.cuda.synchronize()
        assert torch.equal(pc, p1) and torch.equal(gpc, gp1) and torch.equal(goc, go1)
    finally:
        other._h = None
        dc._L.mb2_character_destroy(clone)


@pytest.mark.gpu
def test_sliced_scratch_and_unstaged_point_tables():
    """A shared-offset gradient whose per-instance rows need two scratch slices (4096 x 6000 x 12 bytes > 256 MiB), and 40000 points, whose
    tables (320 KB) cannot sit in the 227 KB of shared memory of a CTA: each instance alone gives the same bits, and the offset gradient
    meets the bound against the float64 sum of the batched rows."""
    from momentum_b200 import torch_skeleton as tsk

    ch = mc.humanoid72()[0]
    dc = tsk._device_character(ch, torch.device("cuda", 0))
    rng = np.random.default_rng(43)
    for B, N in ((4096, 6000), (64, 40000)):
        parents = rng.integers(0, ch.num_joints, N).astype(np.int32)
        params, off, G = (torch.from_numpy(a).cuda() for a in _inputs(ch, False, B, N, False, 44))
        p, gp, go = _calls(dc, False, params, parents, off, G)
        _, _, gor = _calls(dc, False, params, parents, off.expand(B, N, 3).contiguous(), G, need=(False, True))
        go64 = gor.double().sum(0).cpu().numpy()
        assert _ratio(go.cpu().numpy()[None], go64[None]).max() <= K_OFF, (B, N)
        del gor
        for b in [0, B // 2, B - 1]:
            pb, gpb, _ = _calls(dc, False, params[b:b + 1].contiguous(), parents, off, G[b:b + 1].contiguous())
            assert torch.equal(pb, p[b:b + 1]) and torch.equal(gpb, gp[b:b + 1]), (B, N, b)
        sample = [0, B - 1]
        p64, gp64, _ = _reference(ch, False, params[sample].cpu().numpy(), parents, off.cpu().numpy(), G[sample].cpu().numpy())
        assert _ratio(p[sample].cpu().numpy(), p64).max() <= K_POS and _ratio(gp[sample].cpu().numpy(), gp64).max() <= K_GRAD


@pytest.mark.gpu
def test_torch_wrapper_shapes_dtypes_streams_and_gradients():
    from momentum_b200 import torch_skeleton as tsk

    ch = mc.humanoid72()[0]
    n, J = ch.num_params, ch.num_joints
    dev = torch.device("cuda", 0)
    parents = _point_sets(ch)["several"]
    N = len(parents)
    params, off, G = _inputs(ch, False, 3, N, False, 51)
    p64, gp64, go64 = _reference(ch, False, params, parents, off, G)
    # float64 in: float64 out and gradients; parents as a list, a numpy array, a CPU and a CUDA tensor
    for par in (parents.tolist(), parents, torch.from_numpy(parents.astype(np.int64)), torch.from_numpy(parents).to(dev)):
        x = torch.from_numpy(params.astype(np.float64)).to(dev).requires_grad_(True)
        o = torch.from_numpy(off.astype(np.float64)).to(dev).requires_grad_(True)
        p = tsk.model_parameters_to_positions(ch, x, par, o)
        assert p.shape == (3, N, 3) and p.dtype == torch.float64
        p.backward(torch.from_numpy(G.astype(np.float64)).to(dev))
        assert x.grad.dtype == torch.float64 and o.grad.dtype == torch.float64 and o.grad.shape == (N, 3)
        assert _ratio(p.detach().cpu().numpy(), p64).max() <= K_POS
        assert _ratio(x.grad.cpu().numpy(), gp64).max() <= K_GRAD
        assert _ratio(o.grad.cpu().numpy()[None], go64[None]).max() <= K_OFF
    # [n] with [N, 3]
    x1 = torch.from_numpy(params[1]).to(dev).requires_grad_(True)
    p1 = tsk.model_parameters_to_positions(ch, x1, parents, torch.from_numpy(off).to(dev))
    assert p1.shape == (N, 3)
    p1.backward(torch.from_numpy(G[1]).to(dev))
    assert x1.grad.shape == (n,)
    # joint parameters, [B, N, 3] offsets
    jp, offb, Gb = _inputs(ch, True, 3, N, True, 52)
    xj = torch.from_numpy(jp).to(dev).requires_grad_(True)
    ob = torch.from_numpy(offb).to(dev).requires_grad_(True)
    pj = tsk.joint_parameters_to_positions(ch, xj, parents, ob)
    pj.backward(torch.from_numpy(Gb).to(dev))
    assert pj.shape == (3, N, 3) and xj.grad.shape == (3, 7 * J) and ob.grad.shape == (3, N, 3)
    # every needs_input_grad combination gives the same bits as the full backward
    for need_x, need_o in ((True, False), (False, True), (True, True)):
        x = torch.from_numpy(jp).to(dev).requires_grad_(need_x)
        o = torch.from_numpy(offb).to(dev).requires_grad_(need_o)
        tsk.joint_parameters_to_positions(ch, x, parents, o).backward(torch.from_numpy(Gb).to(dev))
        assert (x.grad is not None) == need_x and (o.grad is not None) == need_o
        if need_x:
            assert torch.equal(x.grad, xj.grad)
        if need_o:
            assert torch.equal(o.grad, ob.grad)
    with torch.no_grad():
        assert torch.equal(tsk.joint_parameters_to_positions(ch, xj, parents, ob), pj.detach())
    # N = 0 and B = 0
    x0 = torch.from_numpy(params).to(dev).requires_grad_(True)
    o0 = torch.zeros(0, 3, device=dev, requires_grad=True)
    e = tsk.model_parameters_to_positions(ch, x0, [], o0)
    assert e.shape == (3, 0, 3)
    e.sum().backward()
    assert torch.equal(x0.grad, torch.zeros_like(x0)) and o0.grad.shape == (0, 3)
    xb = torch.zeros(0, n, device=dev, requires_grad=True)
    ob0 = torch.from_numpy(off).to(dev).requires_grad_(True)
    eb = tsk.model_parameters_to_positions(ch, xb, parents, ob0)
    eb.sum().backward()
    assert eb.shape == (0, N, 3) and torch.equal(ob0.grad, torch.zeros_like(ob0))
    # a non-default current stream gives the same bits
    ref = _dev(ch, False, params, parents, off, G)
    side = torch.cuda.Stream(dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side):
        out = _dev(ch, False, params, parents, off, G)
    torch.cuda.current_stream(dev).wait_stream(side)
    torch.cuda.synchronize(dev)
    assert all(torch.equal(a, b) for a, b in zip(out, ref))
    # ValueErrors
    th = torch.from_numpy(params).to(dev)
    od = torch.from_numpy(off).to(dev)
    with pytest.raises(ValueError, match="CUDA"):
        tsk.model_parameters_to_positions(ch, th.cpu(), parents, od)
    with pytest.raises(ValueError, match="CUDA"):
        tsk.model_parameters_to_positions(ch, th, parents, od.cpu())
    with pytest.raises(ValueError, match=r"\[0, 72\)"):
        tsk.model_parameters_to_positions(ch, th, torch.tensor([0, 72], device=dev), od[:2])
    with pytest.raises(ValueError, match="must be"):
        tsk.joint_parameters_to_positions(ch, th, parents, od)
    with pytest.raises(ValueError, match="offsets must be"):
        tsk.model_parameters_to_positions(ch, th, parents, od[:-1])
    dc = ms.DeviceCharacter(ch, 0)
    dc.device = 1  # a handle that belongs to another device than the tensor
    with pytest.raises(ValueError, match="device character"):
        tsk.model_parameters_to_positions(dc, th, parents, od)


@pytest.mark.gpu
def test_c_abi_rejects_bad_arguments():
    ch = mc.create_test_character(4)
    dc = ms.DeviceCharacter(ch, 0)
    n = ch.num_params
    th = torch.zeros(2, n, device="cuda")
    off = torch.zeros(3, 3, device="cuda")
    out = torch.zeros(2, 3, 3, device="cuda")
    par = np.array([0, 1, 3], np.int32)
    host = np.zeros((2, 3, 3), np.float32)
    L = dc._L
    for entry, args in (
            ("mb2_character_model_parameters_to_positions_device", (3, np.array([0, 1, 4], np.int32), off.data_ptr(), 0, out.data_ptr())),
            ("mb2_character_model_parameters_to_positions_device", (3, np.array([0, -1, 2], np.int32), off.data_ptr(), 0, out.data_ptr())),
            ("mb2_character_joint_parameters_to_positions_device", (-1, par, off.data_ptr(), 0, out.data_ptr())),
            ("mb2_character_model_parameters_to_positions_device", (3, par, off.data_ptr(), 0, host.ctypes.data)),
            ("mb2_character_model_parameters_to_positions_device", (3, par, 0, 0, out.data_ptr())),
            ("mb2_character_model_parameters_to_positions_backward_device", (3, par, off.data_ptr(), 0, out.data_ptr(), 0, 0)),
            ("mb2_character_joint_parameters_to_positions_backward_device", (3, par, off.data_ptr(), 0, 0, th.data_ptr(), 0))):
        p = np.ascontiguousarray(args[1], np.int32)
        rc = getattr(L, entry)(dc._h, 2, th.data_ptr(), args[0], p.ctypes.data_as(ms._ip), *args[2:], None)
        assert rc == 1, (entry, args[0])  # MB2_ERR_INVALID_ARGUMENT
        assert L.mb2_last_error()
    # batch 0 and N = 0 are valid
    assert L.mb2_character_model_parameters_to_positions_device(dc._h, 0, 0, 3, par.ctypes.data_as(ms._ip), 0, 0, 0, None) == 0
    assert L.mb2_character_model_parameters_to_positions_device(dc._h, 2, th.data_ptr(), 0, None, 0, 0, 0, None) == 0
    torch.cuda.synchronize()


@pytest.mark.gpu
def test_solve_ik_then_positions_backward_matches_finite_differences():
    """solve_ik -> model_parameters_to_positions -> a loss on some markers: the position-target gradient of the whole pipeline against
    central differences, on the zero-residual problem where the solver's implicit-function derivative is exact (tests/test_torch_ik.py)."""
    from momentum_b200 import torch_ik as ti
    from momentum_b200 import torch_skeleton as tsk
    from tests.test_torch_ik import _problem

    ch, parents, offsets, targets, active, _ = _problem(B=2, seed=9)
    rng = np.random.default_rng(5)
    B, n = targets.shape[0], ch.num_params
    theta_star = rng.uniform(-0.3, 0.3, (B, n)); theta_star[:, 6] = 0
    targets = mc.world_points(ch, theta_star, parents, offsets).astype(np.float32)
    dev = torch.device("cuda", 0)
    opts = ti.SolverOptions(levmar_lambda=0.01, min_iter=80, max_iter=80, threshold=1.0, line_search=True)
    efw = torch.ones(B, 1, device=dev, dtype=torch.float64)
    pw = torch.ones(B, len(parents), device=dev, dtype=torch.float64)
    markers = np.array([1, 3, 4, 4], np.int32)
    moff = torch.from_numpy(rng.normal(scale=0.2, size=(len(markers), 3))).to(dev)
    w = torch.from_numpy(rng.normal(size=(len(markers), 3))).to(dev)

    def pipeline(tg):
        theta = ti.solve_ik(ch, active, torch.zeros(B, n, device=dev), [ti.ErrorFunctionType.Position], efw, opts, position_cons_parents=parents,
                            position_cons_offsets=offsets, position_cons_weights=pw, position_cons_targets=tg)
        p = tsk.model_parameters_to_positions(ch, theta.double(), markers, moff)
        return (p * w).sum() + 0.5 * (p ** 2).sum()

    tg = torch.from_numpy(targets).to(dev).double().requires_grad_(True)
    pipeline(tg).backward()
    g_tg = tg.grad.clone()
    assert g_tg.abs().max().item() > 0.0
    eps = 5e-3
    with torch.no_grad():
        for (b, c, k) in [(0, 0, 0), (0, 3, 1), (1, 5, 2), (1, 7, 0)]:
            d = torch.zeros_like(tg); d[b, c, k] = eps
            fd = (pipeline(tg + d).item() - pipeline(tg - d).item()) / (2 * eps)
            assert abs(fd - g_tg[b, c, k].item()) <= 0.1 * max(abs(fd), abs(g_tg[b, c, k].item()), 0.05), ("target", b, c, k, fd, g_tg[b, c, k].item())
