"""model_parameters_to_skeleton_state on the device and its backward, against a float64 restatement of the forward kinematics.

The reference gradient g64 is torch autograd through ``_fk64`` (the FK of ``character.forward_kinematics`` written in torch, float64),
taken with respect to the joint parameters and mapped to the model parameters by the transposed ParameterTransform. A float32 result
g passes when ||g - g64||_inf <= K * max(||g64||_inf, 1) per instance. K is pinned at about four times the worst value measured over
the fixtures below (emulator and H100); the self-checks show that the bound rejects a backward that drops the quaternion term or swaps
two rotation DOFs.
"""
import numpy as np
import pytest
import torch

from momentum_b200 import character as mc
from momentum_b200 import solver as ms
from tests import emu_lib


# worst measured ||g - g64||_inf / max(||g64||_inf, 1) over these fixtures and seeds: 1.64e-6 on the emulator, 1.77e-6 on an
# H100 80GB HBM3 at a 700 W power limit (humanoid72 both times); the quaternion-term and swapped-DOF errors below are >= 5e-3
K_BOUND = 7e-6

OP = "model_parameters_to_skeleton_state"  # its entry in solver.JOINT_OPS


# ---- fixtures ----------------------------------------------------------------------------------------------------------------------
def _far_humanoid():
    """humanoid72 with non-zero ParameterTransform offsets on every row (scale rows included) and the root 100 units from the origin."""
    ch, _ = mc.humanoid72()
    rng = np.random.default_rng(77)
    ch.pt_offsets = rng.uniform(-0.2, 0.2, ch.pt_offsets.shape).astype(np.float32)
    ch.offsets = ch.offsets.copy()
    ch.offsets[0] += np.float32(100.0)
    ch.name = "humanoid72_far"
    return ch


def _two_roots():
    """Two trees (roots 0 and 2, children interleaved in index order) driven by a shared 0.5-coefficient parameter and a shared scale."""
    parents = np.array([-1, 0, -1, 2, 1, 3, 3, 0], np.int32)
    J = len(parents)
    rng = np.random.default_rng(5)
    offsets = rng.uniform(-1, 1, (J, 3)).astype(np.float32)
    prerot = np.stack([mc._random_prerot(rng) for _ in range(J)]).astype(np.float32)
    trip, p = [], 0
    for j in range(J):
        for d in range(6):
            if parents[j] < 0 or d >= 3:
                trip.append((7 * j + d, p, 1.0)); p += 1
    shared = p
    trip += [(7 * 1 + 5, shared, 0.5), (7 * 5 + 5, shared, 0.5), (7 * 0 + 6, shared + 1, 1.0), (7 * 2 + 6, shared + 1, 1.0)]
    n = shared + 2
    outer, inner, vals = mc._csr_from_triplets(7 * J, n, trip)
    return mc.Character(parents, offsets, prerot, n, outer, inner, vals, np.zeros(7 * J, np.float32), [], "two_roots")


FIXTURES = {
    "chain3": lambda: mc.create_test_character(3),
    "chain6": lambda: mc.create_test_character(6),
    "humanoid72": lambda: mc.humanoid72()[0],
    "bodyhands300": lambda: mc.bodyhands300()[0],
    "humanoid72_far": _far_humanoid,
    "two_roots": _two_roots,
}


def _inputs(ch, B, seed):
    rng = np.random.default_rng(seed)
    theta = rng.uniform(-0.5, 0.5, (B, ch.num_params)).astype(np.float32)
    G = rng.normal(size=(B, ch.num_joints, 8)).astype(np.float32)
    return theta, G


# ---- float64 reference -------------------------------------------------------------------------------------------------------------
def _pt_dense(ch):
    P = np.zeros((7 * ch.num_joints, ch.num_params))
    rows = np.repeat(np.arange(7 * ch.num_joints), np.diff(ch.pt_outer))
    np.add.at(P, (rows, ch.pt_inner), ch.pt_vals.astype(np.float64))
    return torch.from_numpy(P)


def _qmul(a, b):
    ax, ay, az, aw = a.unbind(-1)
    bx, by, bz, bw = b.unbind(-1)
    return torch.stack([aw * bx + ax * bw + ay * bz - az * by, aw * by + ay * bw + az * bx - ax * bz,
                        aw * bz + az * bw + ax * by - ay * bx, aw * bw - ax * bx - ay * by - az * bz], -1)


def _qrot(q, v):
    u = q[..., :3]
    uv = 2.0 * torch.linalg.cross(u, v)
    return v + q[..., 3:4] * uv + torch.linalg.cross(u, uv)


def _fk64(ch, jp):
    """jp [B, J, 7] float64 -> [B, J, 8] (t, q xyzw, s): character.forward_kinematics in torch (joint_state.cpp:22-65)."""
    B = jp.shape[0]
    prerot = torch.from_numpy(ch.prerot.astype(np.float64))
    offsets = torch.from_numpy(ch.offsets.astype(np.float64))
    ts, qs, ss = [], [], []
    zero = torch.zeros(B, dtype=torch.float64)
    for j in range(ch.num_joints):
        p = jp[:, j]
        ql = prerot[j].expand(B, 4)
        for k in (2, 1, 0):
            h = 0.5 * p[:, 3 + k]
            c = [zero, zero, zero, torch.cos(h)]
            c[k] = torch.sin(h)
            ql = _qmul(ql, torch.stack(c, -1))
        tl = offsets[j] + p[:, :3]
        sl = torch.exp2(p[:, 6])
        par = int(ch.parents[j])
        if par < 0:
            t, q, s = tl, ql, sl
        else:
            t = ts[par] + _qrot(qs[par], ss[par][:, None] * tl)
            q = _qmul(qs[par], ql)
            s = ss[par] * sl
        ts.append(t); qs.append(q); ss.append(s)
    return torch.cat([torch.stack(ts, 1), torch.stack(qs, 1), torch.stack(ss, 1)[..., None]], -1)


def _joint_parameters(ch, theta):
    P = _pt_dense(ch)
    return (torch.as_tensor(np.asarray(theta, np.float64)) @ P.T + torch.from_numpy(ch.pt_offsets.astype(np.float64))).reshape(-1, ch.num_joints, 7)


def _g64_joint(ch, theta, G):
    """float64 dLoss/d joint parameters [B, J, 7] of Loss = sum(state * G)."""
    jp = _joint_parameters(ch, theta).requires_grad_(True)
    (_fk64(ch, jp) * torch.as_tensor(np.asarray(G, np.float64))).sum().backward()
    return jp.grad


def _to_model(ch, g_jp):
    return (g_jp.reshape(g_jp.shape[0], -1) @ _pt_dense(ch)).numpy()


def _g64(ch, theta, G):
    return _to_model(ch, _g64_joint(ch, theta, G))


def _bound_ratio(g, g64):
    """per instance ||g - g64||_inf / max(||g64||_inf, 1)"""
    g, g64 = np.asarray(g, np.float64), np.asarray(g64, np.float64)
    return np.abs(g - g64).max(axis=1) / np.maximum(np.abs(g64).max(axis=1), 1.0)


# ---- CPU: the emulator runs the device functions lane by lane ------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu():
    return emu_lib.load()


def _emu_backward(L, ch, theta, G):
    keep = []
    theta = np.ascontiguousarray(theta, np.float32)
    G = np.ascontiguousarray(G, np.float32)
    out = np.full(theta.shape, np.nan, np.float32)
    rc = L.emu_skeleton_state_backward(*emu_lib.character_args(ch, keep), theta.shape[0], theta.ctypes.data, G.ctypes.data, out.ctypes.data)
    assert rc == 0, L.emu_last_error().decode()
    return out


def test_fk64_restates_forward_kinematics():
    for name, make in FIXTURES.items():
        ch = make()
        theta, _ = _inputs(ch, 3, 1)
        t, q, s = mc.forward_kinematics(ch, theta)
        ref = np.concatenate([t, q, s[..., None]], -1)
        st = _fk64(ch, _joint_parameters(ch, theta)).numpy()
        assert np.abs(st - ref).max() <= 1e-12 * max(1.0, np.abs(ref).max()), name


@pytest.mark.parametrize("name", list(FIXTURES))
def test_emulated_backward_meets_the_float64_bound(emu, name):
    ch = FIXTURES[name]()
    theta, G = _inputs(ch, 4, 11)
    ratio = _bound_ratio(_emu_backward(emu, ch, theta, G), _g64(ch, theta, G))
    assert ratio.max() <= K_BOUND, (name, ratio.max())


def test_bound_rejects_a_wrong_backward():
    """The two errors a reverse sweep most easily makes, each measured against the pinned bound: dropping S_c (the quaternion part of
    the upstream gradient, the only place g_q enters) and swapping two rotation DOFs."""
    for name in ("chain6", "humanoid72", "humanoid72_far", "two_roots"):
        ch = FIXTURES[name]()
        theta, G = _inputs(ch, 4, 12)
        g_jp = _g64_joint(ch, theta, G)
        g64 = _to_model(ch, g_jp)
        Gq0 = G.copy(); Gq0[..., 3:7] = 0.0
        assert _bound_ratio(_g64(ch, theta, Gq0), g64).min() > 100 * K_BOUND, name
        swapped = g_jp.clone(); swapped[:, :, [3, 4]] = g_jp[:, :, [4, 3]]
        assert _bound_ratio(_to_model(ch, swapped), g64).min() > 100 * K_BOUND, name


def _ancestry_parameters(ch, joint):
    chain = set()
    j = joint
    while j >= 0:
        chain.add(j); j = int(ch.parents[j])
    rows = np.repeat(np.arange(7 * ch.num_joints), np.diff(ch.pt_outer))
    return set(int(p) for p, r in zip(ch.pt_inner, rows) if r // 7 in chain)


@pytest.mark.parametrize("name", ["humanoid72", "bodyhands300", "two_roots"])
def test_emulated_sparse_upstream_gradient_reaches_only_the_ancestry(emu, name):
    ch = FIXTURES[name]()
    theta, G = _inputs(ch, 3, 13)
    joints = [ch.num_joints - 1, ch.num_joints // 2, 1]
    for b, joint in enumerate(joints):
        keep = G[b, joint].copy(); G[b] = 0.0; G[b, joint] = keep
    g = _emu_backward(emu, ch, theta, G)
    assert _bound_ratio(g, _g64(ch, theta, G)).max() <= K_BOUND
    for b, joint in enumerate(joints):
        allowed = _ancestry_parameters(ch, joint)
        outside = [p for p in range(ch.num_params) if p not in allowed]
        assert np.all(g[b, outside] == 0.0), (name, joint)
        assert np.any(g[b, sorted(allowed)] != 0.0)


def test_cpu_tensor_is_rejected_before_any_library_call(monkeypatch):
    from momentum_b200 import torch_skeleton as tsk

    def no_call(*a, **k):
        raise AssertionError("library reached")

    monkeypatch.setattr(ms, "load_library", no_call)
    monkeypatch.setattr(ms, "DeviceCharacter", type("NoDevice", (), {"__init__": no_call}))
    ch = mc.create_test_character(4)
    with pytest.raises(ValueError, match="CUDA"):
        tsk.model_parameters_to_skeleton_state(ch, torch.zeros(ch.num_params))
    with pytest.raises(ValueError, match="CUDA"):
        tsk.model_parameters_to_skeleton_state(ch, torch.zeros(2, ch.num_params, dtype=torch.float64))


# ---- GPU --------------------------------------------------------------------------------------------------------------------------
def _dev_forward(ch, theta):
    from momentum_b200 import torch_skeleton as tsk

    return tsk.model_parameters_to_skeleton_state(ch, torch.from_numpy(theta).cuda()).cpu().numpy()


def _dev_backward(ch, theta, G):
    from momentum_b200 import torch_skeleton as tsk

    th = torch.from_numpy(np.ascontiguousarray(theta)).cuda().requires_grad_(True)
    tsk.model_parameters_to_skeleton_state(ch, th).backward(torch.from_numpy(np.ascontiguousarray(G)).cuda())
    return th.grad.cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(FIXTURES))
def test_forward_equals_the_solver_function_state_and_fk(name):
    ch = FIXTURES[name]()
    B = 5
    theta, _ = _inputs(ch, B, 21)
    st = _dev_forward(ch, theta)
    assert st.shape == (B, ch.num_joints, 8)
    # the solver function's state comes from the sweep kernel, which runs the same device functions
    ef = mc.PositionErrorFunction(np.array([0], np.int32), np.zeros((1, 3), np.float32), np.ones(1, np.float32), np.zeros((B, 1, 3), np.float32), weight=1.0)
    fn = ms.SkeletonSolverFunction(ch, B, [ef], device=0)
    assert np.array_equal(st, fn.get_skeleton_state(theta))
    t, q, s = mc.forward_kinematics(ch, theta)
    ref = np.concatenate([t, q, s[..., None]], -1)
    assert np.abs(st - ref).max() <= 2e-5 * max(1.0, np.abs(ref).max()), name


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(FIXTURES))
def test_backward_meets_the_float64_bound(name):
    ch = FIXTURES[name]()
    theta, G = _inputs(ch, 8, 22)
    ratio = _bound_ratio(_dev_backward(ch, theta, G), _g64(ch, theta, G))
    assert ratio.max() <= K_BOUND, (name, ratio.max())


def _many_waves(ch):
    """A batch of at least three full waves plus a remainder for any launch shape: no SM holds more backward instances than its
    228 KB of shared memory fits at theta [n] + states [J][17] + sums [J][11] + joint-parameter gradient [7 J] floats each."""
    J, n = ch.num_joints, ch.num_params
    up4 = lambda v: (v + 3) // 4 * 4
    per = 4 * (up4(n) + up4(17 * J) + up4(11 * J) + up4(7 * J))
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return 3 * sms * (228 * 1024 // per) + 37


@pytest.mark.gpu
def test_large_batch_bound_and_determinism_through_joint_op_device():
    from momentum_b200 import torch_skeleton as tsk

    ch = mc.humanoid72()[0]
    B = max(8192, _many_waves(ch))
    theta, G = _inputs(ch, B, 23)
    th = torch.from_numpy(theta).cuda()
    Gd = torch.from_numpy(G).cuda()
    dc = tsk._device_character(ch, th.device)

    def backward(t, g):
        out = torch.empty_like(t)
        dc.joint_op_device(OP, True, t.shape[0], t.data_ptr(), g.contiguous().data_ptr(), out.data_ptr(), stream=torch.cuda.current_stream().cuda_stream)
        return out

    def forward(t):
        out = torch.empty(t.shape[0], ch.num_joints, 8, device=t.device)
        dc.joint_op_device(OP, False, t.shape[0], t.data_ptr(), out.data_ptr(), stream=torch.cuda.current_stream().cuda_stream)
        return out

    g1, g2 = backward(th, Gd), backward(th, Gd)
    s1, s2 = forward(th), forward(th)
    assert torch.equal(g1, g2) and torch.equal(s1, s2)
    sample = np.random.default_rng(3).choice(B, 64, replace=False)
    ratio = _bound_ratio(g1[sample].cpu().numpy(), _g64(ch, theta[sample], G[sample]))
    assert ratio.max() <= K_BOUND, ratio.max()
    for b in [0, 1, B // 3, B // 2, B - 38, B - 1]:  # B - 37 .. B - 1 is the remainder
        assert torch.equal(backward(th[b:b + 1].contiguous(), Gd[b:b + 1]), g1[b:b + 1]), b
        assert torch.equal(forward(th[b:b + 1].contiguous()), s1[b:b + 1]), b


@pytest.mark.gpu
def test_torch_wrapper_shapes_dtypes_streams_and_errors():
    from momentum_b200 import torch_skeleton as tsk

    ch = mc.humanoid72()[0]
    n, J = ch.num_params, ch.num_joints
    theta, G = _inputs(ch, 3, 24)
    dev = torch.device("cuda", 0)
    # [n] and [B, n], float64 in -> float64 out and float64 gradient, on the device
    t64 = torch.from_numpy(theta.astype(np.float64)).to(dev).requires_grad_(True)
    st = tsk.model_parameters_to_skeleton_state(ch, t64)
    assert st.shape == (3, J, 8) and st.dtype == torch.float64 and st.is_cuda
    st.backward(torch.from_numpy(G.astype(np.float64)).to(dev))
    assert t64.grad.dtype == torch.float64 and t64.grad.is_cuda
    assert _bound_ratio(t64.grad.cpu().numpy(), _g64(ch, theta, G)).max() <= K_BOUND
    t1 = torch.from_numpy(theta[1]).to(dev).requires_grad_(True)
    s1 = tsk.model_parameters_to_skeleton_state(ch, t1)
    assert s1.shape == (J, 8)
    assert torch.equal(s1, st[1].float())
    s1.backward(torch.from_numpy(G[1]).to(dev))
    assert t1.grad.shape == (n,)
    # batch 0
    t0 = torch.zeros(0, n, device=dev, requires_grad=True)
    s0 = tsk.model_parameters_to_skeleton_state(ch, t0)
    assert s0.shape == (0, J, 8)
    s0.sum().backward()
    assert t0.grad.shape == (0, n)
    # a non-default current stream gives the same bits
    tf = torch.from_numpy(theta).to(dev).requires_grad_(True)
    ref = tsk.model_parameters_to_skeleton_state(ch, tf)
    ref.backward(torch.from_numpy(G).to(dev))
    side = torch.cuda.Stream(dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side):
        ts = torch.from_numpy(theta).to(dev).requires_grad_(True)
        out = tsk.model_parameters_to_skeleton_state(ch, ts)
        out.backward(torch.from_numpy(G).to(dev))
    torch.cuda.current_stream(dev).wait_stream(side)
    torch.cuda.synchronize(dev)
    assert torch.equal(out, ref) and torch.equal(ts.grad, tf.grad)
    # the ValueError cases
    with pytest.raises(ValueError, match="CUDA"):
        tsk.model_parameters_to_skeleton_state(ch, torch.from_numpy(theta))
    with pytest.raises(ValueError, match="must be"):
        tsk.model_parameters_to_skeleton_state(ch, torch.zeros(3, n + 1, device=dev))
    with pytest.raises(ValueError, match="must be"):
        tsk.model_parameters_to_skeleton_state(ch, torch.zeros(2, 3, n, device=dev))
    dc = ms.DeviceCharacter(ch, 0)
    dc.device = 1  # a handle that belongs to another device than the tensor
    with pytest.raises(ValueError, match="device character"):
        tsk.model_parameters_to_skeleton_state(dc, torch.zeros(n, device=dev))
    dc.device = 0
    assert torch.equal(tsk.model_parameters_to_skeleton_state(dc, tf.detach()), ref.detach())


@pytest.mark.gpu
def test_c_abi_rejects_bad_arguments_through_joint_op_device():
    ch = mc.create_test_character(4)
    dc = ms.DeviceCharacter(ch, 0)
    n, J = ch.num_params, ch.num_joints
    th = torch.zeros(2, n, device="cuda")
    st = torch.zeros(2, J, 8, device="cuda")
    host = np.zeros((2, J, 8), np.float32)
    with pytest.raises(ms.MomentumB200Error, match="device memory"):
        dc.joint_op_device(OP, False, 2, th.data_ptr(), host.ctypes.data)
    with pytest.raises(ms.MomentumB200Error, match="null"):
        dc.joint_op_device(OP, False, 2, 0, st.data_ptr())
    with pytest.raises(ms.MomentumB200Error, match="negative"):
        dc.joint_op_device(OP, False, -1, th.data_ptr(), st.data_ptr())
    with pytest.raises(ms.MomentumB200Error, match="null"):
        dc.joint_op_device(OP, True, 2, th.data_ptr(), 0, th.data_ptr())
    dc.joint_op_device(OP, False, 0, 0, 0)  # batch 0: nothing to do
    dc.joint_op_device(OP, True, 0, 0, 0, 0)


@pytest.mark.gpu
def test_cloned_character_computes_the_same_state():
    """mb2_character_clone re-creates the character, backward tables included."""
    ch = mc.humanoid72()[0]
    dc = ms.DeviceCharacter(ch, 0)
    clone = ms.C.c_void_p()
    dc._check(dc._L.mb2_character_clone(dc._h, 0, ms.C.byref(clone)))
    try:
        theta, G = _inputs(ch, 4, 26)
        th, g = torch.from_numpy(theta).cuda(), torch.from_numpy(G).cuda()
        outs = []
        for h in (dc._h, clone):
            o = torch.empty_like(th)
            dc._check(dc._L.mb2_character_skeleton_state_backward_device(h, 4, ms.C.c_void_p(th.data_ptr()), ms.C.c_void_p(g.data_ptr()),
                                                                        ms.C.c_void_p(o.data_ptr()), None))
            outs.append(o)
        torch.cuda.synchronize()
        assert torch.equal(outs[0], outs[1])
    finally:
        dc._L.mb2_character_destroy(clone)


@pytest.mark.gpu
def test_solve_ik_then_skeleton_state_backward_matches_finite_differences():
    """solve_ik -> model_parameters_to_skeleton_state -> a loss on some joints' translations and rotations: the position-target
    gradient of the whole pipeline against central differences, on the zero-residual problem where the solver's implicit-function
    derivative is exact (tests/test_torch_ik.py)."""
    from momentum_b200 import torch_ik as ti
    from momentum_b200 import torch_skeleton as tsk
    from tests.test_torch_ik import _problem

    ch, parents, offsets, targets, active, _ = _problem(B=2, seed=9)
    rng = np.random.default_rng(4)
    B, n = targets.shape[0], ch.num_params
    theta_star = rng.uniform(-0.3, 0.3, (B, n)); theta_star[:, 6] = 0
    targets = mc.world_points(ch, theta_star, parents, offsets).astype(np.float32)
    dev = torch.device("cuda", 0)
    opts = ti.SolverOptions(levmar_lambda=0.01, min_iter=80, max_iter=80, threshold=1.0, line_search=True)
    efw = torch.ones(B, 1, device=dev, dtype=torch.float64)
    pw = torch.ones(B, len(parents), device=dev, dtype=torch.float64)
    joints = [1, 3, 4]
    wt = torch.from_numpy(rng.normal(size=(len(joints), 3))).to(dev)
    wq = torch.from_numpy(rng.normal(size=(len(joints), 4))).to(dev)

    def pipeline(tg):
        theta = ti.solve_ik(ch, active, torch.zeros(B, n, device=dev), [ti.ErrorFunctionType.Position], efw, opts, position_cons_parents=parents,
                            position_cons_offsets=offsets, position_cons_weights=pw, position_cons_targets=tg)
        st = tsk.model_parameters_to_skeleton_state(ch, theta.double())[:, joints]
        return (st[..., :3] * wt).sum() + (st[..., 3:7] * wq).sum() + 0.5 * (st[..., :3] ** 2).sum()

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
