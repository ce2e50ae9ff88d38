"""Input gradients of solve_ik's implicit-function backward: d/d input [grad_theta E . v] for Position and Orientation constraints.

The reference g64 is float64 torch autograd of grad_theta E . v, with E restated from the residuals of ``evalUnit`` on a torch FK
(``_fk64`` of tests/test_skeleton_state.py), taken with respect to the constraint weights, offsets and targets (quaternions: at the
normalised values the device stores). The reference is checked first: its J v against the float64 oracle Jacobian, and its input
gradients against central differences. A float32 result g passes when ||g - g64||_inf <= K * max(||g64||_inf, 1) per instance, the
outputs of one instance taken together. The self-checks show that the bound rejects the four errors a closed form most easily makes.
"""
import numpy as np
import pytest
import torch

from momentum_b200 import character as mc
from momentum_b200 import solver as ms
from tests import emu_lib
from tests.test_skeleton_state import FIXTURES, _fk64, _pt_dense, _qmul, _qrot


# worst measured ||g - g64||_inf / max(||g64||_inf, 1) over the fixtures below: 1.36e-5 on the emulator (humanoid72) and 1.84e-5 on an
# H100 80GB HBM3 at a 400 W power limit (bodyhands300), both Position blocks; pinned about four times above. The errors of the self-check
# below are 2.5e-2 or more.
K_BOUND = 7e-5


# ---- problems ---------------------------------------------------------------------------------------------------------------------
def _problem(ch, kind, B, seed, instanced):
    """Random constraints on random joints, targets near the constraint points, per-instance weights, a strict enabled subset."""
    rng = np.random.default_rng(seed)
    J, n = ch.num_joints, ch.num_params
    nc = min(8, J)
    parents = rng.choice(J, nc, replace=J < nc).astype(np.int32)
    theta = rng.uniform(-0.5, 0.5, (B, n)).astype(np.float32)
    v = rng.normal(size=(B, n)).astype(np.float32)
    enabled = np.ones(n, bool)
    enabled[rng.choice(n, max(1, n // 4), replace=False)] = False
    cw = rng.uniform(0.5, 2.0, (B, nc)).astype(np.float32)
    if kind == 0:
        off = rng.uniform(-0.5, 0.5, (B if instanced else 1, nc, 3)).astype(np.float32)
        off = np.broadcast_to(off, (B, nc, 3)).copy()
        st = _fk64(ch, _jp64(ch, torch.from_numpy(theta.astype(np.float64)))).numpy()
        p = st[:, parents, :3] + _qrot(torch.from_numpy(st[:, parents, 3:7]), torch.from_numpy(st[:, parents, 7:8] * off.astype(np.float64))).numpy()
        tgt = (p + 0.3 * rng.normal(size=p.shape)).astype(np.float32)
    else:
        off = _unit(rng.normal(size=(B if instanced else 1, nc, 4)))
        off = np.broadcast_to(off, (B, nc, 4)).copy()
        tgt = _unit(rng.normal(size=(B, nc, 4)))
    return dict(kind=kind, parents=parents, theta=theta, v=v, enabled=enabled, cw=cw, off=off, tgt=tgt, ew=0.7, c=1.5, instanced=instanced)


def _unit(q):
    return (q / np.linalg.norm(q, axis=-1, keepdims=True)).astype(np.float32)


def _jp64(ch, theta):
    """joint parameters [B, J, 7] of a float64 tensor theta (ParameterTransform with its offsets)"""
    return (theta @ _pt_dense(ch).T + torch.from_numpy(ch.pt_offsets.astype(np.float64))).reshape(theta.shape[0], ch.num_joints, 7)


def _qmat64(q):
    """qmat's quadratic form, [..., 3, 3] (row, col)"""
    x, y, z, w = q.unbind(-1)
    return torch.stack([torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)], -1),
                        torch.stack([2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)], -1),
                        torch.stack([2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)], -1)], -2)


def _residuals64(ch, P, theta, cw, off, tgt):
    """[B, nc, 3] (Position) or [B, nc, 3, 3] (Orientation, F = R_j R(q_o) - R(q_t)) with the rows of evalUnit, before sqrt(weight)."""
    st = _fk64(ch, _jp64(ch, theta))[:, P["parents"]]
    if P["kind"] == 0:
        return st[..., :3] + _qrot(st[..., 3:7], st[..., 7:8] * off) - tgt
    return _qmat64(st[..., 3:7]) @ _qmat64(off) - _qmat64(tgt)


def _grad_dot_v64(ch, P, mask_v=True, inputs=None):
    """(g = grad_theta E . v [B], inputs (cw, off, tgt) as float64 leaves): E = ew / c^2 sum_c cw_c |f_c|^2"""
    f64 = lambda a: torch.from_numpy(np.asarray(a, np.float64))
    cw, off, tgt = inputs if inputs is not None else [f64(P[k]).requires_grad_(True) for k in ("cw", "off", "tgt")]
    theta = f64(P["theta"]).requires_grad_(True)
    v = f64(P["v"]) * (f64(P["enabled"]) if mask_v else 1.0)
    f = _residuals64(ch, P, theta, cw, off, tgt)
    sq = (f * f).flatten(2).sum(-1)
    E = (P["ew"] / P["c"] ** 2 * cw * sq).sum()
    (gth,) = torch.autograd.grad(E, theta, create_graph=True)
    return (gth * v).sum(-1), (cw, off, tgt)


def _g64(ch, P, mask_v=True):
    """float64 (d/d cw [B, nc], d/d offset [B, nc, k], d/d target [B, nc, k])"""
    g, leaves = _grad_dot_v64(ch, P, mask_v)
    return [t.numpy() for t in torch.autograd.grad(g.sum(), leaves)]


def _closed_form64(ch, P, drop_sigma=False, drop_w_cross_d=False, rc_for_rt=False, mask_v=True):
    """The formulas of the device code in float64, with the motion of each parent frame from a forward-mode derivative of the FK:
    the four switches are the errors the self-check must catch."""
    f64 = lambda a: torch.from_numpy(np.asarray(a, np.float64))
    theta, v = f64(P["theta"]), f64(P["v"]) * (f64(P["enabled"]) if mask_v else 1.0)
    st, dst = torch.func.jvp(lambda th: _fk64(ch, _jp64(ch, th)), (theta,), (v,))
    st, dst = st[:, P["parents"]], dst[:, P["parents"]]
    q, s = st[..., 3:7], st[..., 7:8]
    qc = q * torch.tensor([-1.0, -1.0, -1.0, 1.0], dtype=torch.float64)
    w = 2.0 * _qmul(dst[..., 3:7], qc)[..., :3]          # dq = 1/2 (w, 0) q
    sig = torch.zeros_like(s) if drop_sigma else dst[..., 7:8] / s
    cw, off, tgt = f64(P["cw"]), f64(P["off"]), f64(P["tgt"])
    ew = P["ew"] / P["c"] ** 2
    W = (ew * cw)[..., None]
    if P["kind"] == 0:
        rel = _qrot(q, s * off)
        d = st[..., :3] + rel - tgt
        pdot = dst[..., :3] + torch.linalg.cross(w, rel) + sig * rel
        inner = pdot + sig * d - (0.0 if drop_w_cross_d else torch.linalg.cross(w, d))
        return [(2 * ew * (d * pdot).sum(-1)).numpy(), (2 * W * s * _qrot(qc, inner)).numpy(), (-2 * W * pdot).numpy()]
    Rj, Ro, Rt = _qmat64(q), _qmat64(off), _qmat64(tgt)
    Rc = Rj @ Ro
    wx = torch.zeros(w.shape[:-1] + (3, 3), dtype=torch.float64)
    wx[..., 0, 1], wx[..., 0, 2], wx[..., 1, 0], wx[..., 1, 2], wx[..., 2, 0], wx[..., 2, 1] = -w[..., 2], w[..., 1], w[..., 2], -w[..., 0], -w[..., 1], w[..., 0]
    Xt = wx @ Rc
    Xo = Rj.transpose(-1, -2) @ wx @ (Rc if rc_for_rt else Rt)

    def ddot(qq, X):  # <dR/dq (qq), X>
        qq = qq.clone().requires_grad_(True)
        (g,) = torch.autograd.grad((_qmat64(qq) * X).sum(), qq)
        return g

    return [(2 * ew * ((Rc - Rt) * Xt).sum((-1, -2))).numpy(), (2 * W * ddot(off, Xo)).numpy(), (-2 * W * ddot(tgt, Xt)).numpy()]


def _bound_ratio(g, g64):
    """per instance ||g - g64||_inf / max(||g64||_inf, 1) over all outputs of the instance"""
    B = g64[0].shape[0]
    a = np.concatenate([np.asarray(x, np.float64).reshape(B, -1) for x in g], 1)
    b = np.concatenate([np.asarray(x, np.float64).reshape(B, -1) for x in g64], 1)
    return np.abs(a - b).max(axis=1) / np.maximum(np.abs(b).max(axis=1), 1.0)


def _records(P):
    """the per-instance records the handle holds: [B][nc * k] shared, [B][nc * 2k] instanced (target, then offset)"""
    B = P["theta"].shape[0]
    rec = np.concatenate([P["tgt"], P["off"]], -1) if P["instanced"] else P["tgt"]
    return np.ascontiguousarray(rec.reshape(B, -1), np.float32)


CASES = [(name, kind, inst) for name in FIXTURES for kind in (0, 1) for inst in (False, True)]


# ---- CPU: the float64 reference -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", [0, 1])
def test_reference_jv_matches_the_float64_oracle_jacobian(kind):
    from oracle.binding import OracleFunction

    # measured: 1e-7 relative or less; chains agree to 1e-10. The oracle's rig and the float64 FK differ in the last float bits of
    # the character tables, which the bound K (float32 arithmetic) is far above
    for name in ("chain6", "humanoid72", "two_roots"):
        ch = FIXTURES[name]()
        P = _problem(ch, kind, 2, 31, True)
        f64 = lambda a: torch.from_numpy(np.asarray(a, np.float64))
        v = f64(P["v"]) * f64(P["enabled"])
        for b in range(2):
            sel = lambda a: f64(a)[b:b + 1]
            f, Jf = torch.func.jvp(lambda th: _residuals64(ch, P, th, None, sel(P["off"]), sel(P["tgt"])), (sel(P["theta"]),), (v[b:b + 1],))
            scale = np.sqrt(P["ew"] / P["c"] ** 2 * P["cw"][b].astype(np.float64))
            # evalUnit's rows: xyz per Position constraint, the 3 x 3 difference column by column per Orientation constraint
            rows = (Jf[0] if kind == 0 else Jf[0].transpose(-1, -2)).reshape(len(P["parents"]), -1).numpy() * scale[:, None]
            cls = mc.PositionErrorFunction if kind == 0 else mc.OrientationErrorFunction
            ef = cls(P["parents"], P["off"][b], P["cw"][b], P["tgt"][b:b + 1], weight=P["ew"], loss_c=P["c"])
            orc = OracleFunction(ch, [ef], "float64")
            orc.set_enabled_parameters(P["enabled"])
            _, J, r, _ = orc.get_jacobian(P["theta"][b].astype(np.float64))
            ref = (J[:rows.size] @ v[b].numpy()).reshape(rows.shape)
            assert np.abs(rows - ref).max() <= 1e-6 * max(1.0, np.abs(ref).max()), (name, kind, b)


@pytest.mark.parametrize("kind", [0, 1])
def test_reference_input_gradients_match_central_differences(kind):
    ch = FIXTURES["humanoid72_far"]()
    P = _problem(ch, kind, 2, 32, True)
    g64 = _g64(ch, P)
    rng = np.random.default_rng(3)
    for which, key in enumerate(("cw", "off", "tgt")):
        for _ in range(4):
            idx = tuple(int(rng.integers(0, s)) for s in P[key].shape)
            eps = 1e-6
            vals = []
            for sgn in (1, -1):
                Q = dict(P)
                Q[key] = P[key].astype(np.float64).copy()
                Q[key][idx] += sgn * eps
                with torch.enable_grad():
                    vals.append(_grad_dot_v64(ch, Q)[0].sum().item())
            fd = (vals[0] - vals[1]) / (2 * eps)
            assert abs(fd - g64[which][idx]) <= 1e-6 * max(1.0, abs(fd)), (key, idx, fd, g64[which][idx])


def test_closed_form_is_the_reference_and_the_bound_rejects_its_likely_errors():
    """The formulas of the device code equal the autograd reference; each of the errors a closed form most easily makes - no log-scale
    rate sigma, no -w x d in the offset gradient, R_c where R(q_t) belongs, v not gated by the enabled set - misses the bound by 100x.
    On the large rigs the only scale DOF is the global one and the constraint points sit close to their joints, so dropping sigma or
    -w x d costs less there (4e-4 to 9e-3): those two are checked on the rigs with per-joint scales."""
    for name in FIXTURES:
        ch = FIXTURES[name]()
        small = name in ("chain3", "chain6", "two_roots")
        for kind in (0, 1):
            P = _problem(ch, kind, 3, 33, True)
            g64 = _g64(ch, P)
            # 1e-6: the closed form takes the joint rotations as exact rotations, while the pre-rotations (float32 input) and so the
            # FK quaternions are unit only to float precision
            assert _bound_ratio(_closed_form64(ch, P), g64).max() <= 1e-6, (name, kind)
            wrong = [dict(mask_v=False)] + ([dict(drop_sigma=True), dict(drop_w_cross_d=True)] if kind == 0 and small else []) + \
                    ([dict(rc_for_rt=True)] if kind == 1 else [])
            for w in wrong:
                assert _bound_ratio(_closed_form64(ch, P, **w), g64).min() > 100 * K_BOUND, (name, kind, w)


# ---- CPU: the emulator runs the device functions lane by lane ------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu():
    return emu_lib.load()


def _emu(L, ch, P):
    keep = []
    B, nc, k = P["off"].shape
    arrs = dict(cp=np.ascontiguousarray(P["parents"], np.int32), co=np.ascontiguousarray(P["off"][0], np.float32),
                en=np.ascontiguousarray(P["enabled"], np.uint8), rec=_records(P), cw=np.ascontiguousarray(P["cw"], np.float32),
                th=np.ascontiguousarray(P["theta"], np.float32), v=np.ascontiguousarray(P["v"], np.float32))
    out = [np.full((B, nc), np.nan, np.float32), np.full((B, nc, k), np.nan, np.float32), np.full((B, nc, k), np.nan, np.float32)]
    rc = L.emu_input_gradients(*emu_lib.character_args(ch, keep), P["kind"], int(P["instanced"]), nc,
                               arrs["cp"].ctypes.data, arrs["co"].ctypes.data, P["ew"], P["c"], arrs["en"].ctypes.data, B, arrs["rec"].ctypes.data,
                               arrs["cw"].ctypes.data, arrs["th"].ctypes.data, arrs["v"].ctypes.data, *(o.ctypes.data for o in out))
    assert rc == 0, L.emu_last_error().decode()
    return out


@pytest.mark.parametrize("name,kind,instanced", CASES)
def test_emulated_input_gradients_meet_the_float64_bound(emu, name, kind, instanced):
    ch = FIXTURES[name]()
    P = _problem(ch, kind, 3, 41, instanced)
    ratio = _bound_ratio(_emu(emu, ch, P), _g64(ch, P))
    print(f"emu {name} kind={kind} instanced={instanced}: worst ratio {ratio.max():.3e}")
    assert ratio.max() <= K_BOUND, (name, kind, instanced, ratio.max())


# ---- GPU: the kernel ----------------------------------------------------------------------------------------------------------------
def _dev_function(ch, P, B=None, sl=slice(None)):
    """A solver function holding the block of P (instances ``sl``) with its records and per-instance weights."""
    B = P["theta"][sl].shape[0] if B is None else B
    nc = len(P["parents"])
    inst = P["off"][sl] if P["instanced"] else None
    cls = mc.PositionErrorFunction if P["kind"] == 0 else mc.OrientationErrorFunction
    ef = cls(P["parents"], P["off"][0], np.ones(nc, np.float32), P["tgt"][sl], weight=P["ew"], loss_c=P["c"], instance_offsets=inst)
    fn = ms.SkeletonSolverFunction(ch, B, [ef], device=0)
    fn.set_enabled_parameters(P["enabled"])
    Q = dict(P, tgt=P["tgt"][sl], off=P["off"][sl], theta=P["theta"][sl])
    fn.set_targets(0, _records(Q))
    fn.set_constraint_weights(0, np.ascontiguousarray(P["cw"][sl]), per_instance=True)
    return fn


def _dev_grads(fn, theta, v, k, outputs=(True, True, True)):
    B, nc = theta.shape[0], fn.error_functions[0].parents.shape[0]
    th, vv = torch.from_numpy(np.ascontiguousarray(theta)).cuda(), torch.from_numpy(np.ascontiguousarray(v)).cuda()
    outs = [torch.full((B, nc), float("nan"), device="cuda"), torch.full((B, nc, k), float("nan"), device="cuda"),
            torch.full((B, nc, k), float("nan"), device="cuda")]
    ptrs = [o.data_ptr() if want else 0 for o, want in zip(outs, outputs)]
    fn.input_gradients_device(0, th.data_ptr(), vv.data_ptr(), *ptrs, stream=torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return outs


@pytest.mark.gpu
@pytest.mark.parametrize("name,kind,instanced", CASES)
def test_kernel_input_gradients_meet_the_float64_bound(name, kind, instanced):
    ch = FIXTURES[name]()
    P = _problem(ch, kind, 6, 51, instanced)
    g = _dev_grads(_dev_function(ch, P), P["theta"], P["v"], 3 if kind == 0 else 4)
    ratio = _bound_ratio([o.cpu().numpy() for o in g], _g64(ch, P))
    print(f"kernel {name} kind={kind} instanced={instanced}: worst ratio {ratio.max():.3e}")
    assert ratio.max() <= K_BOUND, (name, kind, instanced, ratio.max())


def _many_waves(ch):
    """at least three full waves plus a remainder for any launch shape: no SM holds more instances than its 228 KB of shared memory fits
    at theta [n] + v [n] + states [J][17] + motions [J][7] floats each"""
    up4 = lambda x: (x + 3) // 4 * 4
    per = 4 * (2 * up4(ch.num_params) + up4(17 * ch.num_joints) + up4(7 * ch.num_joints))
    return 3 * torch.cuda.get_device_properties(0).multi_processor_count * (228 * 1024 // per) + 37


@pytest.mark.gpu
@pytest.mark.parametrize("kind", [0, 1])
def test_kernel_is_deterministic_and_independent_of_the_batch(kind):
    ch = FIXTURES["humanoid72"]()
    B = max(8192, _many_waves(ch))
    P = _problem(ch, kind, B, 52, True)
    k = 3 if kind == 0 else 4
    fn = _dev_function(ch, P)
    g1, g2 = _dev_grads(fn, P["theta"], P["v"], k), _dev_grads(fn, P["theta"], P["v"], k)
    assert all(torch.equal(a, b) for a, b in zip(g1, g2))
    sample = np.random.default_rng(3).choice(B, 16, replace=False)
    Q = dict(P, **{key: P[key][sample] for key in ("theta", "v", "cw", "off", "tgt")})
    assert _bound_ratio([o[sample].cpu().numpy() for o in g1], _g64(ch, Q)).max() <= K_BOUND
    for b in [0, 1, B // 3, B - 38, B - 1]:  # B - 37 .. B - 1 is the remainder
        one = _dev_grads(_dev_function(ch, P, sl=slice(b, b + 1)), P["theta"][b:b + 1], P["v"][b:b + 1], k)
        assert all(torch.equal(a, o[b:b + 1]) for a, o in zip(one, g1)), b


@pytest.mark.gpu
def test_c_abi_rejects_what_it_does_not_differentiate_and_skips_null_outputs():
    ch = FIXTURES["chain6"]()
    P = _problem(ch, 0, 2, 53, False)
    fn = _dev_function(ch, P)
    th, v = torch.from_numpy(P["theta"]).cuda(), torch.from_numpy(P["v"]).cuda()
    nc = len(P["parents"])
    out = torch.zeros(2, nc, 3, device="cuda")
    with pytest.raises(ms.MomentumB200Error, match="out of range"):
        fn.input_gradients_device(1, th.data_ptr(), v.data_ptr(), 0, 0, out.data_ptr())
    with pytest.raises(ms.MomentumB200Error, match="null"):
        fn.input_gradients_device(0, 0, v.data_ptr(), 0, 0, out.data_ptr())
    with pytest.raises(ms.MomentumB200Error, match="null"):
        fn.input_gradients_device(0, th.data_ptr(), 0, 0, 0, out.data_ptr())
    host = np.zeros((2, nc, 3), np.float32)
    with pytest.raises(ms.MomentumB200Error, match="device memory"):
        fn.input_gradients_device(0, th.data_ptr(), v.data_ptr(), 0, 0, host.ctypes.data)
    with pytest.raises(ms.MomentumB200Error, match="device memory"):
        fn.input_gradients_device(0, P["theta"].ctypes.data, v.data_ptr(), 0, 0, out.data_ptr())
    q = np.tile(np.array([0, 0, 0, 1], np.float32), (nc, 1))
    other = ms.SkeletonSolverFunction(ch, 2, [mc.OrientationErrorFunction(P["parents"], q, np.ones(nc), np.zeros((2, nc, 4)) + q, rot_diff=True),
                                             mc.PositionErrorFunction(P["parents"], P["off"][0], np.ones(nc), P["tgt"], loss_alpha=1.0),
                                             mc.LimitErrorFunction()], device=0)
    for idx, msg in ((0, "Position and Orientation"), (1, "L2"), (2, "Position and Orientation")):
        with pytest.raises(ms.MomentumB200Error, match=msg):
            other.input_gradients_device(idx, th.data_ptr(), v.data_ptr(), 0, 0, out.data_ptr())
    # a null output is skipped: the others are the same bits as with every output requested
    full = _dev_grads(fn, P["theta"], P["v"], 3)
    for mask in ((True, False, False), (False, True, False), (False, False, True)):
        part = _dev_grads(fn, P["theta"], P["v"], 3, mask)
        for want, a, b in zip(mask, part, full):
            assert torch.equal(a, b) if want else bool(torch.isnan(a).all())


# ---- GPU: the instanced Orientation block -------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_instanced_orientation_with_one_offset_solves_like_the_shared_block():
    from momentum_b200.problems import humanoid_problem

    B = 64
    ch, efs, theta0, _ = humanoid_problem(B, orientation=True)
    pos, ori = efs
    inst = mc.OrientationErrorFunction(ori.parents, ori.offsets, ori.weights, ori.targets, weight=ori.weight,
                                       instance_offsets=np.broadcast_to(np.asarray(ori.offsets, np.float32), (B,) + np.shape(ori.offsets)).copy())
    runs = [dict(fused_mode=ms.FUSED_AUTO), dict(fused_mode=ms.FUSED_GRAM_CHOLESKY), dict(fused_mode=ms.FUSED_OFF),
            dict(fused_mode=ms.FUSED_OFF, cholesky_mode=ms.CHOLESKY_DENSE_EIGEN), dict(linear_solver=ms.LINEAR_SOLVER_QR),
            dict(linear_solver=ms.LINEAR_SOLVER_TRUST_REGION_QR)]
    for kw in runs:
        opts = ms.GaussNewtonSolverOptions(min_iterations=1, max_iterations=6, threshold=1.0, regularization=0.05, **kw)
        outs = []
        for o in (ori, inst):
            fn = ms.SkeletonSolverFunction(ch, B, [pos, o], device=0)
            fn.upload_targets()
            outs.append(ms.GaussNewtonSolver(opts, fn).solve(theta0))
        assert np.array_equal(outs[0]["params"], outs[1]["params"]), kw
        assert np.array_equal(outs[0]["errors"], outs[1]["errors"]), kw


@pytest.mark.gpu
def test_instanced_orientation_offsets_match_per_element_oracle_solves():
    from momentum_b200.problems import humanoid_problem
    from tests import parity

    B = 6
    ch, efs, theta0, theta_star = humanoid_problem(B, orientation=True)
    pos, ori = efs
    rng = np.random.default_rng(7)
    off = _unit(np.asarray(ori.offsets)[None] + 0.5 * rng.normal(size=(B, len(ori.parents), 4)))
    tg = np.stack([mc.world_rotations(ch, theta_star[b:b + 1], ori.parents, off[b])[0] for b in range(B)])
    inst = mc.OrientationErrorFunction(ori.parents, ori.offsets, ori.weights, tg, weight=ori.weight, instance_offsets=off)
    opts = ms.GaussNewtonSolverOptions(min_iterations=6, max_iterations=6, regularization=0.05)
    parity.check_solve(ch, [pos, inst], theta0, opts, param_tol=2e-4)


# ---- GPU: solve_ik's backward --------------------------------------------------------------------------------------------------------
def _ik_problem(B, seed, reachable):
    """The chain of tests/test_torch_ik.py with Position, Orientation (shared offsets), Motion and its MinMax limit; ``reachable``: every
    target from one pose theta*, so that the residual vanishes at the optimum."""
    ch = mc.create_test_character(5)
    rng = np.random.default_rng(seed)
    n = ch.num_params
    pp = np.array([1, 2, 3, 4, 4, 2, 3, 1], np.int32)
    po = rng.uniform(-1, 1, (B, len(pp), 3)).astype(np.float32)
    op = np.array([2, 4, 3], np.int32)
    oo = _unit(rng.normal(size=(len(op), 4)))
    theta_star = rng.uniform(-0.3, 0.3, (B, n)); theta_star[:, 6] = 0
    noise = 0.0 if reachable else 1.0
    pt = np.stack([mc.world_points(ch, theta_star[b:b + 1], pp, po[b])[0] for b in range(B)]) + 0.05 * noise * rng.normal(size=(B, len(pp), 3))
    ot = mc.world_rotations(ch, theta_star, op, oo) + 0.05 * noise * rng.normal(size=(B, len(op), 4))
    ot = ot * rng.uniform(0.8, 1.2, (B, len(op), 1))  # raw quaternions: solve_ik normalises them
    mt = theta_star + 0.1 * noise * rng.normal(size=(B, n))
    mw = rng.uniform(0.3, 1.0, n)
    active = np.ones(n, bool); active[6] = False
    return dict(ch=ch, pp=pp, po=po, op=op, oo=oo, pt=pt, ot=ot, mt=mt, mw=mw, active=active, pw=1.0 + 0.3 * rng.uniform(size=(B, len(pp))),
                ow=1.0 + 0.3 * rng.uniform(size=(B, len(op))), theta_star=theta_star)


def _solve(Pr, kinds, opts, **inputs):
    from momentum_b200 import torch_ik as ti

    dev = torch.device("cuda", 0)
    t = lambda a: a if torch.is_tensor(a) else torch.from_numpy(np.asarray(a, np.float64)).to(dev)
    x = {k: inputs.get(k, Pr[k]) for k in ("pp", "po", "pw", "pt", "op", "oo", "ow", "ot", "mt", "mw")}
    B, n = x["pt"].shape[0], Pr["ch"].num_params
    return ti.solve_ik(Pr["ch"], Pr["active"], torch.zeros(B, n, device=dev), kinds, torch.ones(B, len(kinds), device=dev, dtype=torch.float64), opts,
                       position_cons_parents=x["pp"], position_cons_offsets=t(x["po"]), position_cons_weights=t(x["pw"]), position_cons_targets=t(x["pt"]),
                       orientation_cons_parents=x["op"], orientation_cons_offsets=t(x["oo"]), orientation_cons_weights=t(x["ow"]),
                       orientation_cons_targets=t(x["ot"]), motion_targets=t(x["mt"]), motion_weights=t(x["mw"]))


def _leaves(Pr):
    dev = torch.device("cuda", 0)
    return {k: torch.from_numpy(np.asarray(Pr[k], np.float64)).to(dev).requires_grad_(True) for k in ("po", "pw", "pt", "oo", "ow", "ot", "mt", "mw")}


def _ift64(Pr, b, theta_b, gout_b):
    """The reference IFT of one element in float64: v = (2 J^T J)^+ g from the double oracle's Jacobian of every block, then
    dLoss/d input = -d/d input [grad E_k . v] from the float64 reference of this module (Position, Orientation) and the elementwise
    Motion formulas."""
    from oracle.binding import OracleFunction

    ch, n = Pr["ch"], Pr["ch"].num_params
    otn = Pr["ot"][b] / np.linalg.norm(Pr["ot"][b], axis=-1, keepdims=True)
    efs = [mc.PositionErrorFunction(Pr["pp"], Pr["po"][b], Pr["pw"][b], Pr["pt"][b:b + 1], weight=1.0),
           mc.OrientationErrorFunction(Pr["op"], Pr["oo"], Pr["ow"][b], otn[None], weight=1.0), mc.LimitErrorFunction(weight=1.0),
           mc.ModelParametersErrorFunction(Pr["mw"], Pr["mt"][b:b + 1], weight=1.0)]
    orc = OracleFunction(ch, efs, "float64")
    orc.set_enabled_parameters(Pr["active"])
    _, J, r, _ = orc.get_jacobian(theta_b.astype(np.float64))
    act = np.nonzero(Pr["active"])[0]
    assert np.sqrt(np.mean((2 * J[:, act].T @ r) ** 2)) <= 0.01  # converged: the backward gives this element a gradient
    U, S, Vt = np.linalg.svd(J[:, act], full_matrices=False)
    tmp = Vt @ gout_b[act]
    tmp = np.where(S * S < 1e-5, 0.0, tmp / np.maximum(S * S, 1e-300))
    v = np.zeros(n); v[act] = 0.5 * Vt.T @ tmp
    common = dict(theta=theta_b[None].astype(np.float64), v=v[None], enabled=Pr["active"], ew=1.0, c=1.0, instanced=True)
    gp = _g64(ch, dict(common, kind=0, parents=Pr["pp"], cw=Pr["pw"][b:b + 1], off=Pr["po"][b:b + 1], tgt=Pr["pt"][b:b + 1]))
    go = _g64(ch, dict(common, kind=1, parents=Pr["op"], cw=Pr["ow"][b:b + 1], off=Pr["oo"][None], tgt=otn[None]))
    norm_bw = lambda g, q: _normalization_backward64(torch.from_numpy(g), torch.from_numpy(np.asarray(q, np.float64))).numpy()
    on = Pr["active"] & (Pr["mw"] > 0)
    s = 0.1
    return dict(po=-gp[1][0], ow=-go[0][0], ot=norm_bw(-go[2][0], Pr["ot"][b]), oo=norm_bw(-go[1][0], Pr["oo"]),
                mt=2 * s * Pr["mw"] ** 2 * v * on, mw=-4 * s * Pr["mw"] * (theta_b - Pr["mt"][b]) * v * on)


def _normalization_backward64(g, q):
    nrm = torch.linalg.vector_norm(q, dim=-1, keepdim=True)
    qh = q / nrm
    return (g - qh * (qh * g).sum(-1, keepdim=True)) / nrm


def _kinds():
    from momentum_b200 import torch_ik as ti

    return [ti.ErrorFunctionType.Position, ti.ErrorFunctionType.Orientation, ti.ErrorFunctionType.Limit, ti.ErrorFunctionType.Motion]


@pytest.mark.gpu
def test_solve_ik_backward_is_the_reference_implicit_function_derivative_for_every_new_input():
    from momentum_b200 import torch_ik as ti

    B = 2
    Pr = _ik_problem(B, 9, reachable=False)
    opts = ti.SolverOptions(levmar_lambda=0.01, min_iter=80, max_iter=80, threshold=1.0, line_search=True)
    L = _leaves(Pr)
    theta = _solve(Pr, _kinds(), opts, **L)
    gout = np.random.default_rng(1).normal(size=theta.shape)
    (theta.double() * torch.from_numpy(gout).to(theta.device)).sum().backward()
    th = theta.detach().cpu().numpy()
    refs = [_ift64(Pr, b, th[b], gout[b]) for b in range(B)]
    for key in ("po", "ow", "ot", "mt"):  # per element
        for b in range(B):
            got, ref = L[key].grad[b].cpu().numpy(), refs[b][key]
            assert np.abs(got - ref).max() <= 2e-3 * max(1.0, np.abs(ref).max()), (key, b, np.abs(got - ref).max(), np.abs(ref).max())
    for key in ("oo", "mw"):  # shared by the batch: the sum of the per-element gradients
        got, ref = L[key].grad.cpu().numpy(), sum(r[key] for r in refs)
        assert np.abs(got - ref).max() <= 2e-3 * max(1.0, np.abs(ref).max()), (key, np.abs(got - ref).max(), np.abs(ref).max())
    assert all(np.abs(L[k].grad.cpu().numpy()).max() > 1e-3 for k in ("po", "ow", "ot", "oo", "mt", "mw"))


@pytest.mark.gpu
def test_kernel_position_target_and_weight_contractions_agree_with_the_jacobian_formulas():
    """The kernel's Position target / weight outputs against the existing torch formulas of the backward, 2 sqrt(w) J v and
    -2 (r . J v) / w, on the device Jacobian of the same handle."""
    from momentum_b200 import torch_ik as ti

    ch = FIXTURES["humanoid72"]()
    P = _problem(ch, 0, 4, 54, True)
    P["ew"], P["c"] = 1.0, 1.0
    fn = _dev_function(ch, P)
    gw, _, gt = [o.double() for o in _dev_grads(fn, P["theta"], P["v"], 3)]
    th = torch.from_numpy(P["theta"]).cuda()
    ptr, ld = fn.get_jacobian_device(th.data_ptr(), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    n, nc = ch.num_params, len(P["parents"])
    Jall = ti._device_view(ptr, (4, n + 1, ld), th.device).clone().double()
    J, r = Jall[:, :n, :3 * nc].transpose(1, 2), Jall[:, n, :3 * nc]
    v = torch.from_numpy(P["v"] * P["enabled"]).cuda().double()
    Jv = torch.einsum("brn,bn->br", J, v).reshape(4, nc, 3)
    w = torch.from_numpy(P["cw"]).cuda().double()
    # dLoss/dt = -d/dt [grad E . v] = 2 sqrt(w) J v; dLoss/dw = -(2 r . J v) / w
    assert torch.allclose(-gt, 2 * w.sqrt()[..., None] * Jv, rtol=1e-4, atol=1e-4 * Jv.abs().max().item())
    ref_w = -2 * (r.reshape(4, nc, 3) * Jv).sum(-1) / w
    assert torch.allclose(-gw, ref_w, rtol=1e-3, atol=1e-4 * ref_w.abs().max().item())


@pytest.mark.gpu
def test_solve_ik_backward_matches_finite_differences_for_offsets_orientations_and_motion_targets():
    from momentum_b200 import torch_ik as ti

    B = 2
    Pr = _ik_problem(B, 11, reachable=True)
    kinds = [ti.ErrorFunctionType.Position, ti.ErrorFunctionType.Orientation, ti.ErrorFunctionType.Motion]
    opts = ti.SolverOptions(levmar_lambda=0.01, min_iter=80, max_iter=80, threshold=1.0, line_search=True)
    gout = torch.from_numpy(np.random.default_rng(4).normal(size=(B, Pr["ch"].num_params))).cuda().float()
    L = _leaves(Pr)
    (_solve(Pr, kinds, opts, **L).float() * gout).sum().backward()
    rng = np.random.default_rng(5)
    eps = 5e-3
    for key in ("po", "ot", "oo", "mt"):
        for _ in range(3):
            idx = tuple(int(rng.integers(0, s)) for s in L[key].shape)
            with torch.no_grad():
                vals = []
                for sgn in (1, -1):
                    x = {k: t.detach() for k, t in L.items()}
                    x[key] = x[key].clone(); x[key][idx] += sgn * eps
                    vals.append((_solve(Pr, kinds, opts, **x).float() * gout).sum().item())
            fd, g = (vals[0] - vals[1]) / (2 * eps), L[key].grad[idx].item()
            assert abs(fd - g) <= 0.1 * max(abs(fd), abs(g), 0.05), (key, idx, fd, g)


@pytest.mark.gpu
def test_shared_offsets_cache_and_an_interleaved_forward():
    from momentum_b200 import torch_ik as ti

    B = 3
    Pr = _ik_problem(B, 13, reachable=False)
    kinds = [ti.ErrorFunctionType.Position, ti.ErrorFunctionType.Orientation]
    opts = ti.SolverOptions(levmar_lambda=0.01, min_iter=40, max_iter=40, threshold=1.0, line_search=True)
    gout = torch.from_numpy(np.random.default_rng(6).normal(size=(B, Pr["ch"].num_params))).cuda()
    dev = torch.device("cuda", 0)
    # shared [nc, 3] position offsets that require grad: the batch sum of the per-element gradients of the same offsets given per element
    shared = torch.from_numpy(Pr["po"][0].astype(np.float64)).to(dev).requires_grad_(True)
    batched = shared.detach()[None].expand(B, -1, -1).clone().requires_grad_(True)
    for off in (shared, batched):
        (_solve(Pr, kinds, opts, po=off).double() * gout).sum().backward()
    assert torch.allclose(shared.grad, batched.grad.sum(0), rtol=1e-12, atol=0.0)
    # new offset values reuse the cached handle
    count = len(ti._handles)
    for k in range(3):
        off = (shared.detach() + 0.01 * k).requires_grad_(True)
        (_solve(Pr, kinds, opts, po=off).double() * gout).sum().backward()
    assert len(ti._handles) == count
    # a forward on the same handle between a forward and its backward does not change that backward

    def grads(interleave):
        L = _leaves(Pr)
        out = _solve(Pr, kinds, opts, **{k: L[k] for k in ("po", "pw", "pt", "oo", "ow", "ot")})
        if interleave:
            other = {k: (L[k].detach() * 1.1) for k in ("po", "pt", "ot")}
            _solve(Pr, kinds, opts, pw=L["pw"].detach() * 0.5, ow=L["ow"].detach() * 2.0, oo=L["oo"].detach().flip(-1)[None].expand(B, -1, -1), **other)
        (out.double() * gout).sum().backward()
        return {k: L[k].grad for k in ("po", "pw", "pt", "oo", "ow", "ot")}

    a, b = grads(False), grads(True)
    for k in a:
        assert torch.equal(a[k], b[k]), k
