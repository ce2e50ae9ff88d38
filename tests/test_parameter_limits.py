"""parameter_limits_residual and apply_model_param_limits on the device, against the float64 oracle's LimitErrorFunction.

The forward is compared row by row with the rows the oracle's float64 ``get_jacobian`` returns for ``[LimitErrorFunction()]`` (weight 1,
L2 loss), and its sum of squares with ``get_error``. A row passes when |r - r64| <= K_FWD * s, with s the row's scale times the size of
what it reads: w (1 + |theta|_inf + |P theta + o|_inf) for a parameter- or joint-space limit, w (1 + max_j |t_j|) for an Ellipsoid.
The backward is compared with central differences of the oracle's float64 residual contracted with random upstream gradients G, per
instance: ||g - g64||_inf <= K_BWD * max_p sum_r |J64_rp| |G_r|; the rows of the non-Ellipsoid limits are also compared with the
oracle's own Jacobian. The self-checks show that this bound rejects three wrong backwards: the reference's truncated Ellipsoid Jacobian
(computeEllipsoidJacobian, what the oracle's get_jacobian returns for those rows), joint-space terms added without P^T, and one flipped
row sign. The Ellipsoid rows have bounds of their own (K_FWD_ELLIPSOID, K_BWD_ELLIPSOID). Each bound is pinned at 2.5 to 4 times the
worst ratio measured (emulator and H100, in the comments).
"""
import ctypes

import numpy as np
import pytest
import torch

from momentum_b200 import character as mc
from momentum_b200 import solver as ms
from momentum_b200.problems import add_test_limits
from oracle.binding import OracleFunction
from tests import emu_lib

# worst measured ratio on the emulator / on an H100 80GB HBM3 at a 700 W power limit: forward 9.9e-8 / 8.0e-8, Ellipsoid rows 4.9e-6 /
# 5.0e-6; backward 6.1e-8 / 6.1e-8, Ellipsoid rows 1.5e-5 / 2.3e-5. The Ellipsoid rows are conditioned by 1 / |u|, the distance of the
# point from the ellipsoid's centre in ellipsoid space, which the scale does not carry.
K_FWD = 4e-7
K_FWD_ELLIPSOID = 2e-5
K_BWD = 2.5e-7
K_BWD_ELLIPSOID = 6e-5

H100_SXM = (132, 232448)  # SMs, opt-in shared memory per block: the launch the tests size rigs for


# ---- fixtures -------------------------------------------------------------------------------------------------------------------------
def _chain(ellipsoid):
    ch = mc.create_test_character(6)
    return add_test_limits(ch, np.random.default_rng(3), ellipsoid)


def _rig(name):
    if name == "chain_ellipsoid":
        return _chain(True)
    if name == "chain_plain":
        return _chain(False)
    ch = mc.humanoid72()[0] if name == "humanoid72" else mc.bodyhands300()[0]
    ch.limits = mc.synthetic_limits(ch, seed=7)
    return ch


RIGS = ["chain_ellipsoid", "chain_plain", "humanoid72", "bodyhands300"]
_RIG_CACHE = {}


def rig(name):
    if name not in _RIG_CACHE:
        _RIG_CACHE[name] = _rig(name)
    return _RIG_CACHE[name]


def _half_ranges(ch):
    """per model parameter the half width of its first MinMax limit (1 without one)"""
    h = np.ones(ch.num_params)
    seen = set()
    for lim in ch.limits:
        if lim.type == mc.LIMIT_MINMAX and lim.i[0] not in seen:
            seen.add(lim.i[0])
            h[lim.i[0]] = max(abs(lim.f[0]), abs(lim.f[1]), 1e-3)
    return h


def _thetas(ch, B, seed):
    """B instances from well inside every range (scale 0.05) to well outside (scale 3), so that each limit is active in some and inactive
    in others"""
    rng = np.random.default_rng(seed)
    scale = np.geomspace(0.05, 3.0, B)[:, None]
    u = rng.choice([-1.0, 1.0], (B, ch.num_params)) * rng.uniform(0.8, 1.0, (B, ch.num_params))
    return (u * scale * _half_ranges(ch)).astype(np.float32)


# ---- float64 reference ----------------------------------------------------------------------------------------------------------------
def _oracle(ch):
    orc = OracleFunction(ch, [mc.LimitErrorFunction()], "float64")
    orc.R = len(_row_info(ch))
    return orc


def _rows64(orc, theta):
    """(error, J [R, n], residual [R]): the block's rows, without getJacobian's padding to 8"""
    err, J, res, _ = orc.get_jacobian(np.asarray(theta, np.float64))
    return err, J[:orc.R], res[:orc.R]


def _fd_gradient(orc, theta, G, h=1e-6):
    """central differences of the float64 residual: (J64 [R, n], G^T J64 [n])"""
    x = np.asarray(theta, np.float64)
    cols = []
    for p in range(x.size):
        d = np.zeros_like(x)
        d[p] = h * max(1.0, abs(x[p]))
        cols.append((_rows64(orc, x + d)[2] - _rows64(orc, x - d)[2]) / (2 * d[p]))
    J = np.stack(cols, 1) if cols else np.zeros((G.size, 0))
    return J, G @ J


def _row_info(ch):
    """per residual row: (limit index, type, row scale w)"""
    out = []
    for k, lim in enumerate(ch.limits):
        if lim.type == mc.LIMIT_MINMAX_JOINT_PASSIVE:
            continue
        if lim.type == mc.LIMIT_ELLIPSOID:
            out += [(k, lim.type, np.sqrt(10.0 * 1e-4 * lim.weight))] * 3
        else:
            out.append((k, lim.type, np.sqrt(10.0 * lim.weight)))
    return out


def _forward_scale(ch, theta):
    """per instance and row, the scale of the forward bound (module docstring)"""
    info = _row_info(ch)
    th = np.asarray(theta, np.float64)
    jp = (_pt_dense(ch) @ th.T).T + ch.pt_offsets
    t, _, _ = mc.forward_kinematics(ch, th)
    S = np.zeros((th.shape[0], len(info)))
    for r, (_, ty, w) in enumerate(info):
        S[:, r] = w * (1 + (np.abs(t).max(axis=(1, 2)) if ty == mc.LIMIT_ELLIPSOID else np.maximum(np.abs(th).max(1), np.abs(jp).max(1))))
    return S


def _pt_dense(ch):
    """the ParameterTransform P [7 J, n] (sparse, float64)"""
    import scipy.sparse

    return scipy.sparse.csr_matrix((ch.pt_vals.astype(np.float64), ch.pt_inner, ch.pt_outer), shape=(7 * ch.num_joints, ch.num_params))


def _joint_terms(ch, theta, G):
    """the joint-space limits' gradient with respect to the joint parameters [7 J] (float64): what P^T maps to theta"""
    th = np.asarray(theta, np.float64)
    jp = _pt_dense(ch) @ th + ch.pt_offsets
    t = np.zeros(7 * ch.num_joints)
    row = 0
    for lim in ch.limits:
        if lim.type == mc.LIMIT_MINMAX_JOINT_PASSIVE:
            continue
        w = np.sqrt(10.0 * lim.weight)
        f = np.asarray(lim.f, np.float32).astype(np.float64)
        if lim.type == mc.LIMIT_MINMAX_JOINT:
            r = 7 * lim.i[0] + lim.i[1]
            if jp[r] < f[0] or jp[r] > f[1]:
                t[r] += w * G[row]
        elif lim.type == mc.LIMIT_LINEAR_JOINT:
            ri, ti = 7 * lim.i[0] + lim.i[1], 7 * lim.i[2] + lim.i[3]
            if (f[2] == 0 and f[3] == 0) or (f[2] <= jp[ti] < f[3]):
                t[ti] += w * f[0] * G[row]
                t[ri] -= w * G[row]
        row += 3 if lim.type == mc.LIMIT_ELLIPSOID else 1
    return t


def _backward_ratio(g, g64, J64, G):
    return np.abs(np.asarray(g, np.float64) - g64).max() / max((np.abs(J64) * np.abs(G)[:, None]).sum(0).max(), 1e-30)


# ---- the emulator ---------------------------------------------------------------------------------------------------------------------
_CHARACTER = [ctypes.c_int32, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int32] + [ctypes.c_void_p] * 4
_LIMITS = [ctypes.c_int32] + [ctypes.c_void_p] * 4


@pytest.fixture(scope="module")
def emu():
    L = emu_lib.load()
    L.emu_parameter_limits_tables.argtypes = _CHARACTER + _LIMITS + [ctypes.c_void_p] * 2
    L.emu_parameter_limits.argtypes = _CHARACTER + _LIMITS + [ctypes.c_int32, ctypes.c_int32] + [ctypes.c_void_p] * 3
    L.emu_apply_model_parameter_limits.argtypes = _CHARACTER + _LIMITS + [ctypes.c_int32, ctypes.c_int32] + [ctypes.c_void_p] * 3
    L.emu_parameter_limits_launch.argtypes = _CHARACTER + _LIMITS + [ctypes.c_int32, ctypes.c_int64, ctypes.c_int64, ctypes.c_int32, ctypes.c_void_p]
    return L


def _args(ch, keep):
    K = len(ch.limits)
    types = np.array([lim.type for lim in ch.limits], np.int32)
    weights = np.array([lim.weight for lim in ch.limits], np.float32)
    ints = np.zeros((K, 4), np.int32)
    floats = np.zeros((K, 27), np.float32)
    for k, lim in enumerate(ch.limits):
        ints[k], floats[k] = lim.packed()
    keep += [types, weights, ints, floats]
    return emu_lib.character_args(ch, keep) + [K, types.ctypes.data, weights.ctypes.data, ints.ctypes.data, floats.ctypes.data]


def _emu_tables(L, ch):
    keep, rows, ell = [], ctypes.c_int32(-1), ctypes.c_int32(-1)
    rc = L.emu_parameter_limits_tables(*_args(ch, keep), ctypes.byref(rows), ctypes.byref(ell))
    return rc, (L.emu_last_error().decode() if rc else (rows.value, bool(ell.value)))


def _emu_run(entry, ch, backward, theta, G=None):
    keep = []
    theta = np.ascontiguousarray(theta, np.float32)
    B = theta.shape[0]
    width = ch.num_params if backward or entry.__name__ == "emu_apply_model_parameter_limits" else len(_row_info(ch))
    out = np.full((B, width), np.nan, np.float32)
    g = None if G is None else np.ascontiguousarray(G, np.float32)
    rc = entry(*_args(ch, keep), int(backward), B, theta.ctypes.data, 0 if g is None else g.ctypes.data, out.ctypes.data)
    assert rc == 0
    return out


def _emu_forward(L, ch, theta):
    return _emu_run(L.emu_parameter_limits, ch, False, theta)


def _emu_backward(L, ch, theta, G):
    return _emu_run(L.emu_parameter_limits, ch, True, theta, G)


def _emu_launch(L, ch, backward, batch=4096):
    keep = []
    out = np.zeros(5, np.int64)
    assert L.emu_parameter_limits_launch(*_args(ch, keep), int(backward), batch, H100_SXM[1], H100_SXM[0], out.ctypes.data) == 0
    return out


# ---- shared checks (emulator and device) ----------------------------------------------------------------------------------------------
def _check_forward(ch, theta, r):
    """per-row ratios |r - r64| / s against K_FWD (parameter- and joint-space rows) and K_FWD_ELLIPSOID; returns both worsts"""
    orc = _oracle(ch)
    S = _forward_scale(ch, theta)
    ell = np.array([ty == mc.LIMIT_ELLIPSOID for _, ty, _ in _row_info(ch)], bool)
    worst = np.zeros(2)
    for b in range(theta.shape[0]):
        err, _, r64 = _rows64(orc, theta[b])
        assert r64.shape == r[b].shape
        ratio = np.abs(r[b] - r64) / S[b]
        worst = np.maximum(worst, [ratio[~ell].max(initial=0.0), ratio[ell].max(initial=0.0)])
        assert abs(np.sum(r64 ** 2) - err) <= 1e-7 * max(err, 1e-30)  # getError returns float
        assert abs(np.sum(r[b].astype(np.float64) ** 2) - err) <= 1e-4 * max(err, 1e-30)
    assert worst[0] <= K_FWD and worst[1] <= K_FWD_ELLIPSOID, worst
    return worst


def _check_backward(ch, theta, G, run, self_checks=False):
    """the backward bound per instance, run(G) giving the gradient [B, n] of upstream G [B, R], in two parts whose sum is the whole: G on
    the parameter- and joint-space rows (K_BWD) and G on the Ellipsoid rows (K_BWD_ELLIPSOID). With self_checks, that the three wrong
    backwards miss their part's bound by 100x. Returns the two worst ratios and the smallest ratio of each wrong backward."""
    orc = _oracle(ch)
    ell = np.array([ty == mc.LIMIT_ELLIPSOID for _, ty, _ in _row_info(ch)], bool)
    P = _pt_dense(ch)
    Gp, Ge = G * ~ell, G * ell
    gp, ge = run(Gp.astype(np.float32)), run(Ge.astype(np.float32))
    worst, wrong_worst = np.zeros(2), {}
    for b in range(theta.shape[0]):
        J64, _ = _fd_gradient(orc, theta[b], G[b])
        gp64, ge64 = Gp[b] @ J64, Ge[b] @ J64
        worst = np.maximum(worst, [_backward_ratio(gp[b], gp64, J64, Gp[b]), _backward_ratio(ge[b], ge64, J64, Ge[b])])
        # the parameter- and joint-space rows against the oracle's own Jacobian
        _, Jo, _ = _rows64(orc, theta[b])
        assert np.abs(Jo[~ell] - J64[~ell]).max(initial=0.0) <= 1e-6 * max(np.abs(Jo).max(initial=0.0), 1.0)
        if not self_checks:
            continue
        wrong = {}
        if ell.any():  # computeEllipsoidJacobian: what the reference's getJacobian gives for those rows
            wrong["truncated ellipsoid Jacobian"] = (_backward_ratio(Ge[b] @ Jo, ge64, J64, Ge[b]), K_BWD_ELLIPSOID)
        t = _joint_terms(ch, theta[b], Gp[b])
        if np.abs(t).max(initial=0) > 0:
            tn = np.zeros(ch.num_params)
            tn[: min(t.size, ch.num_params)] = t[: ch.num_params]
            wrong["joint terms without P^T"] = (_backward_ratio(gp64 - P.T @ t + tn, gp64, J64, Gp[b]), K_BWD)
        k = int(np.argmax(np.abs(J64).sum(1) * np.abs(Gp[b])))
        Gf = Gp[b].copy()
        Gf[k] = -Gf[k]
        wrong["flipped row sign"] = (_backward_ratio(Gf @ J64, gp64, J64, Gp[b]), K_BWD)
        for name, (ratio, bound) in wrong.items():
            wrong_worst[name] = min(wrong_worst.get(name, np.inf), ratio / bound)
    assert worst[0] <= K_BWD and worst[1] <= K_BWD_ELLIPSOID, worst
    for name, over in wrong_worst.items():
        assert over > 100, (name, over)
    return worst, wrong_worst


def _activity_covered(ch, theta):
    """every MinMax, MinMaxJoint and HalfPlane limit is active in some instance and inactive in another"""
    orc = _oracle(ch)
    R = np.stack([_rows64(orc, t)[2] for t in theta])
    row = 0
    for lim in ch.limits:
        if lim.type == mc.LIMIT_MINMAX_JOINT_PASSIVE:
            continue
        if lim.type in (mc.LIMIT_MINMAX, mc.LIMIT_MINMAX_JOINT, mc.LIMIT_HALFPLANE):
            on = R[:, row] != 0
            assert on.any() and not on.all(), (lim, on)
        row += 3 if lim.type == mc.LIMIT_ELLIPSOID else 1


# ---- CPU ------------------------------------------------------------------------------------------------------------------------------
def _ka_character():
    ch = mc.create_test_character(4)  # n = 11: root t (0-2), r (3-5), scale 6, joint1 rx 7, shared rz 8, joint2 rx 9, joint3 rx 10
    ch.limits = [mc.ParameterLimit(mc.LIMIT_MINMAX, 1.0, (0,), (-0.1, 0.2)),
                 mc.ParameterLimit(mc.LIMIT_MINMAX_JOINT_PASSIVE, 1.0, (1, 3), (-0.1, 0.1)),
                 mc.ParameterLimit(mc.LIMIT_MINMAX_JOINT, 0.4, (1, 3), (-0.5, 0.25)),
                 mc.ParameterLimit(mc.LIMIT_LINEAR, 0.9, (1, 2), (2.0, 0.5, 0.0, 0.0)),
                 mc.ParameterLimit(mc.LIMIT_LINEAR, 0.9, (1, 2), (2.0, 0.5, -0.25, 0.5)),
                 mc.ParameterLimit(mc.LIMIT_LINEAR_JOINT, 1.6, (0, 1, 1, 3), (0.5, 0.0, -1.0, 1.0)),
                 mc.ParameterLimit(mc.LIMIT_HALFPLANE, 2.5, (3, 4), (1.0, -1.0, 0.5)),
                 mc.ParameterLimit(mc.LIMIT_MINMAX, 0.1, (9,), (-0.3, 0.3)),
                 mc.ParameterLimit(mc.LIMIT_MINMAX, 0.1, (9,), (-0.2, 0.1))]
    return ch


def test_emulated_known_answers(emu):
    """Each type inside, outside and exactly on its bounds, by hand: a MinMax at its min is 0, rangeMin is in and rangeMax out, (0, 0) is
    everywhere, a HalfPlane at 0 is 0; the passive limit has no row; duplicate MinMax limits clamp by the last one."""
    ch = _ka_character()
    assert _emu_tables(emu, ch) == (0, (8, False))
    n = ch.num_params
    th = np.zeros((4, n), np.float32)
    # 0: everything on a bound. p0 = min; jp 1.3 = p7 = 0.25 = max; Linear p2 = rangeMin = -0.25 (in), target 2 p2 - 0.5 - p1
    th[0, [0, 7, 1, 2, 3, 4]] = [-0.1, 0.25, 0.0, -0.25, 0.5, 0.0]  # HalfPlane p3 - p4 - 0.5 = 0
    # 1: outside: p0 below min, jp 1.3 above max, Linear target p2 = rangeMax = 0.5 (out for the ranged one), HalfPlane < 0
    th[1, [0, 7, 1, 2, 3, 4]] = [-0.4, 0.75, 0.1, 0.5, 0.0, 0.5]
    # 2: p0 above max, p9 inside the first of its limits and above the second, HalfPlane positive; 3: zero
    th[2, [0, 7, 1, 2, 3, 4, 9]] = [0.5, 0.0, 0.0, 0.0, 1.0, 0.0, 0.15]
    th[3, 3] = 0.0
    r = _emu_forward(emu, ch, th).astype(np.float64)
    s = lambda w: np.sqrt(10 * np.float64(np.float32(w)))  # noqa: E731
    expect = np.array([
        [0, 0, s(0.9) * -1.0, s(0.9) * -1.0, s(1.6) * 0.125, 0, 0, 0],
        [s(1) * -0.3, s(0.4) * 0.5, s(0.9) * 0.4, 0, s(1.6) * 0.275, s(2.5) * -1.0, 0, 0],
        [s(1) * 0.3, 0, s(0.9) * -0.5, s(0.9) * -0.5, 0, 0, 0, s(0.1) * 0.05],
        [0, 0, s(0.9) * -0.5, s(0.9) * -0.5, 0, s(2.5) * -0.5, 0, 0]])
    assert np.array_equal(r == 0, expect == 0)
    np.testing.assert_allclose(r, expect, rtol=3e-6, atol=0)
    # the clamp: parameter 0 to [-0.1, 0.2], parameter 9 to [-0.2, 0.1] (the last of its two limits), the rest passed through
    x = np.array([[-0.1, 0.3, 7, -3, 0, 0, 0, 0, 0, -0.25, 5], [0.2, -9, 0, 0, 0, 0, 0, 0, 0, 0.1, 0], [0.3, 0, 0, 0, 0, 0, 0, 0, 0, -0.3, 0]],
                 np.float32)
    y = _emu_run(emu.emu_apply_model_parameter_limits, ch, False, x)
    want = x.copy()
    want[:, 0] = np.clip(x[:, 0], np.float32(-0.1), np.float32(0.2))
    want[:, 9] = np.clip(x[:, 9], np.float32(-0.2), np.float32(0.1))
    assert np.array_equal(y, want)
    gy = _emu_run(emu.emu_apply_model_parameter_limits, ch, True, x, np.ones_like(x))
    mask = np.ones_like(x)
    mask[:, 0] = (x[:, 0] >= np.float32(-0.1)) & (x[:, 0] <= np.float32(0.2))
    mask[:, 9] = (x[:, 9] >= np.float32(-0.2)) & (x[:, 9] <= np.float32(0.1))
    assert np.array_equal(gy, mask)


@pytest.mark.parametrize("name", RIGS)
def test_emulated_forward_matches_float64_oracle(emu, name):
    ch = rig(name)
    theta = _thetas(ch, 24, 3)
    _activity_covered(ch, theta)
    r = _emu_forward(emu, ch, theta)
    assert r.shape == (24, len(_row_info(ch)))
    _check_forward(ch, theta, r)


@pytest.mark.parametrize("name", RIGS)
def test_emulated_backward_matches_float64(emu, name):
    ch = rig(name)
    B = 3 if name == "bodyhands300" else 6
    theta = _thetas(ch, B, 2)
    G = np.random.default_rng(3).normal(size=(B, len(_row_info(ch)))).astype(np.float32)
    _check_backward(ch, theta, G, lambda g: _emu_backward(emu, ch, theta, g), self_checks=True)


def _variant_rig(emu, W, ellipsoid, backward):
    """the shortest chain with add_test_limits on a geometric grid of lengths whose launch puts parameterLimitsKernel on W warps per
    instance at H100 SXM limits"""
    for J in np.unique(np.geomspace(6, 8000, 160).astype(int)):
        ch = add_test_limits(mc.create_test_character(int(J)), np.random.default_rng(3), ellipsoid)
        w = int(_emu_launch(emu, ch, backward)[0])
        if w == W:
            return ch
        if w == 0:
            break
    pytest.fail(f"no chain reaches W = {W}")


VARIANTS = [(W, e, b) for W in (1, 2, 4, 8) for e in (False, True) for b in (False, True)]


@pytest.mark.parametrize("W,ellipsoid,backward", VARIANTS)
def test_emulated_launch_variants(emu, W, ellipsoid, backward):
    """every warps-per-instance launch on both kEllipsoid sides: the planner reaches it on a chain, and the emulated kernel meets the bounds
    there"""
    ch = _variant_rig(emu, W, ellipsoid, backward)
    assert _emu_tables(emu, ch)[1][1] == ellipsoid
    theta = _thetas(ch, 2, 4)
    if backward and ch.num_params <= 400:
        G = np.random.default_rng(5).normal(size=(2, len(_row_info(ch)))).astype(np.float32)
        _check_backward(ch, theta, G, lambda g: _emu_backward(emu, ch, theta, g))
    else:
        _check_forward(ch, theta, _emu_forward(emu, ch, theta))


def _clamp_reference(ch, x, grad=None):
    """pymomentum's composition: for each MinMax limit in list order, index_copy of torch.clamp of the original parameter"""
    x = x.detach().requires_grad_(grad is not None)
    y = x
    for lim in ch.limits:
        if lim.type == mc.LIMIT_MINMAX:
            idx = torch.tensor([lim.i[0]], device=x.device)
            lo = torch.tensor([np.float32(lim.f[0])], device=x.device)
            hi = torch.tensor([np.float32(lim.f[1])], device=x.device)
            y = y.index_copy(-1, idx, torch.clamp(x.index_select(-1, idx), lo, hi))
    if grad is None:
        return y.detach(), None
    y.backward(grad)
    return y.detach(), x.grad


def _clamp_inputs(ch, B, seed):
    x = _thetas(ch, B, seed)
    for lim in ch.limits[:6]:  # values exactly on bounds, and a NaN
        if lim.type == mc.LIMIT_MINMAX:
            x[0, lim.i[0]], x[1, lim.i[0]] = lim.f[0], lim.f[1]
    x[2, 0] = np.nan
    return x


@pytest.mark.parametrize("name", ["humanoid72", "bodyhands300"])
def test_emulated_clamp_is_torch_clamp_bit_for_bit(emu, name):
    ch = rig(name)
    x = _clamp_inputs(ch, 8, 6)
    G = np.random.default_rng(7).normal(size=x.shape).astype(np.float32)
    y_ref, g_ref = _clamp_reference(ch, torch.from_numpy(x), torch.from_numpy(G))
    y = _emu_run(emu.emu_apply_model_parameter_limits, ch, False, x)
    g = _emu_run(emu.emu_apply_model_parameter_limits, ch, True, x, G)
    assert np.array_equal(y, y_ref.numpy(), equal_nan=True)
    assert np.array_equal(g, g_ref.numpy())


def test_emulated_rejections_and_no_limits(emu):
    from momentum_b200 import torch_skeleton as tsk

    # an out-of-range index: set_parameter_limits accepts it, the tables record the reason naming the limit
    for lim, what in ((mc.ParameterLimit(mc.LIMIT_MINMAX, 1.0, (99,), (0, 1)), "limit 1 (MinMax)"),
                      (mc.ParameterLimit(mc.LIMIT_ELLIPSOID, 1.0, (0, 9), tuple(np.eye(3, 4).ravel()) * 2 + (0, 0, 0)), "limit 1 (Ellipsoid)"),
                      (mc.ParameterLimit(mc.LIMIT_LINEAR_JOINT, 1.0, (0, 7, 1, 3), (1, 0, 0, 0)), "limit 1 (LinearJoint)")):
        ch = mc.create_test_character(4)
        ch.limits = ch.limits + [lim]
        rc, msg = _emu_tables(emu, ch)
        assert rc == 1 and what in msg, msg
    # no limits, and passive limits only: R = 0 and a zero gradient
    for limits in ([], [mc.ParameterLimit(mc.LIMIT_MINMAX_JOINT_PASSIVE, 1.0, (1, 3), (-0.1, 0.1))]):
        ch = mc.create_test_character(4)
        ch.limits = limits
        assert _emu_tables(emu, ch) == (0, (0, False))
        th = _thetas(ch, 3, 1)
        assert _emu_forward(emu, ch, th).shape == (3, 0)
        assert np.array_equal(_emu_backward(emu, ch, th, np.zeros((3, 0), np.float32)), np.zeros_like(th))
    # the torch functions check before any library call
    ch = rig("chain_plain")
    n = ch.num_params
    for fn in (tsk.parameter_limits_residual, tsk.apply_model_param_limits):
        with pytest.raises(ValueError, match="must be"):
            fn(ch, torch.zeros(2, n + 1))
        with pytest.raises(ValueError, match="must be"):
            fn(ch, torch.zeros(2, 3, n))
        with pytest.raises(ValueError, match="CUDA"):
            fn(ch, torch.zeros(2, n))


def test_synthetic_limits_cover_every_live_type():
    for name in ("humanoid72", "bodyhands300"):
        ch = rig(name)
        types = [lim.type for lim in ch.limits]
        assert set(types) == set(range(7))
        leaves = [j for j in range(ch.num_joints) if j not in set(ch.parents.tolist()) and ch.depth()[j] >= 2]
        assert types.count(mc.LIMIT_ELLIPSOID) == len(leaves)
        per_param = np.bincount([lim.i[0] for lim in ch.limits if lim.type == mc.LIMIT_MINMAX], minlength=ch.num_params)
        assert per_param.min() >= 1 and per_param.max() == 2
    a, b = mc.synthetic_limits(mc.humanoid72()[0], 3), mc.synthetic_limits(mc.humanoid72()[0], 3)
    assert a == b


# ---- GPU ------------------------------------------------------------------------------------------------------------------------------
def _dev_forward(dc, theta):
    return _run_dev(dc, theta, None)[0]


def _run_dev(dc, theta, G):
    from momentum_b200 import torch_skeleton as tsk

    x = torch.from_numpy(np.ascontiguousarray(theta)).cuda().requires_grad_(G is not None)
    r = tsk.parameter_limits_residual(dc, x)
    g = None
    if G is not None:
        r.backward(torch.from_numpy(np.ascontiguousarray(G)).cuda())
        g = x.grad.cpu().numpy()
    torch.cuda.synchronize()
    return r.detach().cpu().numpy(), g


@pytest.mark.gpu
@pytest.mark.parametrize("name", RIGS)
def test_device_matches_float64(name):
    ch = rig(name)
    dc = ms.DeviceCharacter(ch, 0)
    B = 3 if name == "bodyhands300" else 6
    theta = _thetas(ch, 24, 3)
    _check_forward(ch, theta, _dev_forward(dc, theta))
    theta = _thetas(ch, B, 2)
    G = np.random.default_rng(3).normal(size=(B, len(_row_info(ch)))).astype(np.float32)
    _check_backward(ch, theta, G, lambda g: _run_dev(dc, theta, g)[1], self_checks=True)


@pytest.mark.gpu
@pytest.mark.parametrize("W,ellipsoid,backward", VARIANTS)
def test_device_launch_variants(emu, W, ellipsoid, backward):
    ch = _variant_rig(emu, W, ellipsoid, backward)
    dc = ms.DeviceCharacter(ch, 0)
    B = 2 * torch.cuda.get_device_properties(0).multi_processor_count + 3
    launch = dc.get_instance_launch("parameter_limits_residual", backward, B)
    assert launch["warps"] == W, launch
    theta = np.concatenate([_thetas(ch, 2, 4)] * (B // 2 + 1))[:B]
    if backward:
        G = np.random.default_rng(5).normal(size=(B, len(_row_info(ch)))).astype(np.float32)
        g = _run_dev(dc, theta, G)[1]
        if ch.num_params <= 400:
            _check_backward(ch, theta[:2], G[:2], lambda gg: _run_dev(dc, theta[:2], gg)[1])
        g1 = _run_dev(dc, theta[B - 1:], G[B - 1:])[1]
        assert np.array_equal(g1[0], g[B - 1])
    else:
        r = _dev_forward(dc, theta)
        _check_forward(ch, theta[:2], r[:2])
        assert np.array_equal(_dev_forward(dc, theta[B - 1:])[0], r[B - 1])


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["humanoid72", "bodyhands300"])
def test_device_clamp_is_torch_clamp_bit_for_bit(name):
    from momentum_b200 import torch_skeleton as tsk

    ch = rig(name)
    x = torch.from_numpy(_clamp_inputs(ch, 64, 6)).cuda()
    G = torch.from_numpy(np.random.default_rng(7).normal(size=tuple(x.shape)).astype(np.float32)).cuda()
    y_ref, g_ref = _clamp_reference(ch, x, G)
    xr = x.clone().requires_grad_(True)
    y = tsk.apply_model_param_limits(ch, xr)
    y.backward(G)
    assert torch.equal(torch.nan_to_num(y.detach(), 7.0), torch.nan_to_num(y_ref, 7.0)) and torch.isnan(y).sum() == 1
    assert torch.equal(xr.grad, g_ref)
    # float64 in, float64 out; [n] in, [n] out
    y64 = tsk.apply_model_param_limits(ch, x[3].double())
    assert y64.dtype == torch.float64 and torch.equal(y64.float(), y[3].detach())


@pytest.mark.gpu
def test_device_bitwise_invariance_dtype_and_rejections():
    from momentum_b200 import torch_skeleton as tsk

    ch = rig("humanoid72")
    dc = ms.DeviceCharacter(ch, 0)
    R = dc.num_limit_residuals()
    assert R == len(_row_info(ch))
    theta = _thetas(ch, 300, 8)
    G = np.random.default_rng(9).normal(size=(300, R)).astype(np.float32)
    r, g = _run_dev(dc, theta, G)
    for sl in (slice(0, 1), slice(17, 18), slice(5, 133), slice(299, 300)):  # batch size and instance position
        rs, gs = _run_dev(dc, theta[sl], G[sl])
        assert np.array_equal(rs, r[sl]) and np.array_equal(gs, g[sl])
    r2, g2 = _run_dev(dc, theta, G)  # repeated call
    assert np.array_equal(r2, r) and np.array_equal(g2, g)
    clone = C_clone(dc)  # a cloned character carries the tables
    rc_, gc_ = _run_dev(clone, theta, G)
    assert np.array_equal(rc_, r) and np.array_equal(gc_, g)
    # the Character path uses the registry handle and gives the same bits; float64 round trips; [n] gives [R]
    x64 = torch.from_numpy(theta[:4]).cuda().double()
    r64 = tsk.parameter_limits_residual(ch, x64)
    assert r64.dtype == torch.float64 and np.array_equal(r64.float().cpu().numpy(), r[:4])
    assert tsk.parameter_limits_residual(ch, x64[1]).shape == (R,)
    # out-of-range limits: the DeviceCharacter and solve_ik accept the character, the limit operations raise the reason
    bad = mc.create_test_character(4)
    bad.limits = bad.limits + [mc.ParameterLimit(mc.LIMIT_MINMAX, 1.0, (99,), (0, 1))]
    dcb = ms.DeviceCharacter(bad, 0)
    xb = torch.zeros(2, bad.num_params, device="cuda")
    with pytest.raises(ms.MomentumB200Error, match=r"limit 1 \(MinMax\)"):
        tsk.parameter_limits_residual(dcb, xb)
    with pytest.raises(ms.MomentumB200Error, match=r"limit 1 \(MinMax\)"):
        tsk.apply_model_param_limits(dcb, xb)
    assert tsk.model_parameters_to_skeleton_state(dcb, xb).shape == (2, 4, 8)
    # no limits: [B, 0] and a zero gradient
    none = mc.create_test_character(4)
    none.limits = []
    x0 = torch.ones(3, none.num_params, device="cuda", requires_grad=True)
    e = tsk.parameter_limits_residual(none, x0)
    assert e.shape == (3, 0)
    e.sum().backward()
    assert torch.equal(x0.grad, torch.zeros_like(x0))
    # C-ABI pointer checks
    L = dc._L
    th = torch.zeros(2, ch.num_params, device="cuda")
    host = np.zeros((2, R), np.float32)
    assert L.mb2_character_parameter_limits_residual_device(dc._h, 2, th.data_ptr(), host.ctypes.data, None) == 1
    assert L.mb2_character_parameter_limits_residual_device(dc._h, -1, th.data_ptr(), 0, None) == 1
    assert L.mb2_character_parameter_limits_residual_backward_device(dc._h, 2, th.data_ptr(), 0, 0, None) == 1


def C_clone(dc):
    """a DeviceCharacter whose handle is mb2_character_clone of dc's, on the same device"""
    import ctypes as C

    out = C.c_void_p()
    dc._check(dc._L.mb2_character_clone(dc._h, dc.device, C.byref(out)))
    clone = object.__new__(ms.DeviceCharacter)
    clone.__dict__.update({k: v for k, v in dc.__dict__.items() if k != "_h"})
    clone._h = out
    return clone


@pytest.mark.gpu
def test_solve_ik_then_limit_loss_backward_matches_finite_differences():
    """solve_ik -> parameter_limits_residual -> its sum of squares: the position-target gradient of the whole pipeline against central
    differences, on the zero-residual problem where the solver's implicit-function derivative is exact (tests/test_torch_ik.py)."""
    from momentum_b200 import torch_ik as ti
    from momentum_b200 import torch_skeleton as tsk
    from tests.test_torch_ik import _problem

    ch, parents, offsets, targets, active, _ = _problem(B=2, seed=9)
    ch.limits = mc.synthetic_limits(ch, seed=4)
    rng = np.random.default_rng(5)
    B, n = targets.shape[0], ch.num_params
    theta_star = rng.uniform(-0.3, 0.3, (B, n)); theta_star[:, 6] = 0
    targets = mc.world_points(ch, theta_star, parents, offsets).astype(np.float32)
    dev = torch.device("cuda", 0)
    opts = ti.SolverOptions(levmar_lambda=0.01, min_iter=80, max_iter=80, threshold=1.0, line_search=True)
    efw = torch.ones(B, 1, device=dev, dtype=torch.float64)
    pw = torch.ones(B, len(parents), device=dev, dtype=torch.float64)

    def pipeline(tg):
        theta = ti.solve_ik(ch, active, torch.zeros(B, n, device=dev), [ti.ErrorFunctionType.Position], efw, opts, position_cons_parents=parents,
                            position_cons_offsets=offsets, position_cons_weights=pw, position_cons_targets=tg)
        return tsk.parameter_limits_residual(ch, theta.double()).square().sum()

    tg = torch.from_numpy(targets).to(dev).double().requires_grad_(True)
    pipeline(tg).backward()
    g_tg = tg.grad.clone()
    assert g_tg.abs().max().item() > 0.0
    eps = 5e-3
    fd = torch.zeros_like(tg)
    with torch.no_grad():
        for b in range(B):
            for c in range(tg.shape[1]):
                for k in range(3):
                    d = torch.zeros_like(tg); d[b, c, k] = eps
                    fd[b, c, k] = (pipeline(tg + d).item() - pipeline(tg - d).item()) / (2 * eps)
    cos = float((fd * g_tg).sum() / (fd.norm() * g_tg.norm()))
    assert cos >= 0.99, cos
