"""collision_residual on the device, against the float64 restatement of CollisionErrorFunction in ``momentum_b200.character``.

``character.capsule_contact`` restates overlaps() over closestPointsOnSegments branch for branch; run on float64 geometry it is the
reference the rows are measured against. A row passes when |r - r64| <= K_FWD * sqrt(5e-3) * m, with m the pair's coordinate magnitude
(the largest |origin|, |origin + direction| and radius of its two capsules). Pairs that are nearly parallel (D64 < 1e-3 a c) or whose
float64 evaluation takes a decision within a relative 1e-4 of its threshold are left out and counted; the count must stay small.
The backward is compared with central differences of the float64 rows with respect to the state, pair by pair over the 16 state values
of its two parents, with the upstream gradient of a pair set to 0 where its branch changes within +-h:
||g - g64||_inf <= K_BWD * sqrt(5e-3) * sum_k |G_k| * (1 + max_j |t_j|) per instance. The self-checks show that this bound rejects three wrong backwards:
the taper term dropped (momentum's getJacobian, which holds (s, t) fixed), radii not scaled by the parent's s, and a flipped normal.
Each bound is pinned at about four times the worst ratio measured (in the comments).
"""
import ctypes

import numpy as np
import pytest
import torch

from momentum_b200 import character as mc
from momentum_b200 import solver as ms
from tests import emu_lib

# worst measured ratio on the emulator / on an H100 80GB HBM3 at a 700 W power limit: forward 1.9e-7 / 1.6e-7; backward
# 1.4e-7 / 3.2e-7
K_FWD = 8e-7
K_BWD = 1.3e-6
# the emulated backward composed with the skeleton-state emulator's backward against getJacobian^T g, restated from model parameters on
# untapered capsules: worst measured 1.2e-8 (the chain), 1.7e-9 (humanoid72); on tapered capsules the two differ by 5e-5 to 3e-3
K_JAC = 5e-8
WGT = np.sqrt(5e-3)
H100_SXM = (132, 232448)  # SMs, opt-in shared memory per block: the launch the tests size rigs for

_p, _i32, _i64 = ctypes.c_void_p, ctypes.c_int32, ctypes.c_int64
_CHARACTER = [_i32, _p, _p, _p, _i32, _p, _p, _p, _p]
_CAPSULES = [_i32, _p]


@pytest.fixture(scope="module")
def emu():
    L = emu_lib.load()
    L.emu_collision_pairs.argtypes = _CHARACTER + _CAPSULES + [_p, _p]
    L.emu_collision.argtypes = _CHARACTER + _CAPSULES + [_i32, _i32, _p, _p, _p]
    L.emu_capsule_contact.argtypes = [_p] * 5
    L.emu_capsule_contact.restype = None
    L.emu_collision_launch.argtypes = _CHARACTER + _CAPSULES + [_i32, _i64, _i64, _i32, _p]
    return L


def _args(ch, caps, keep):
    arr = mc.capsule_array(caps)
    keep.append(arr)
    return emu_lib.character_args(ch, keep) + [len(arr), arr.ctypes.data if len(arr) else None]


def _check(L, rc):
    assert rc == 0, L.emu_last_error().decode()


def emu_pairs(L, ch, caps):
    keep, n = [], ctypes.c_int32(0)
    _check(L, L.emu_collision_pairs(*_args(ch, caps, keep), ctypes.byref(n), None))
    out = np.zeros((n.value, 2), np.int32)
    _check(L, L.emu_collision_pairs(*_args(ch, caps, keep), ctypes.byref(n), out.ctypes.data))
    return out


def emu_rows(L, ch, caps, st, P):
    keep = []
    st = np.ascontiguousarray(st, np.float32)
    out = np.zeros((st.shape[0], P), np.float32)
    _check(L, L.emu_collision(*_args(ch, caps, keep), 0, st.shape[0], st.ctypes.data, None, out.ctypes.data))
    return out


def emu_grad(L, ch, caps, st, G):
    keep = []
    st = np.ascontiguousarray(st, np.float32)
    G = np.ascontiguousarray(G, np.float32)
    out = np.zeros(st.shape, np.float32)
    _check(L, L.emu_collision(*_args(ch, caps, keep), 1, st.shape[0], st.ctypes.data, G.ctypes.data, out.ctypes.data))
    return out


def emu_contact(L, A, B):
    A, B = np.asarray(A, np.float32), np.asarray(B, np.float32)
    out, gA, gB = np.zeros(7, np.float32), np.zeros(8, np.float32), np.zeros(8, np.float32)
    L.emu_capsule_contact(A.ctypes.data, B.ctypes.data, out.ctypes.data, gA.ctypes.data, gB.ctypes.data)
    return out, gA, gB


# ---- fixtures -------------------------------------------------------------------------------------------------------------------------
def _chain_rig():
    """a 6-joint chain folded back on itself, its capsules tapered, untapered, on scaled joints, and two world-fixed ones"""
    ch = mc.create_test_character(6)
    caps = mc.synthetic_collision(ch, seed=2)
    return ch, caps


def _rig(name):
    if name == "chain":
        return _chain_rig()
    ch = mc.humanoid72()[0] if name == "humanoid72" else mc.bodyhands300()[0]
    return ch, mc.synthetic_collision(ch, seed=0)


RIGS = ["chain", "humanoid72", "bodyhands300"]
_CACHE = {}


def rig(name):
    if name not in _CACHE:
        _CACHE[name] = _rig(name)
    return _CACHE[name]


def states(ch, B, seed, spread=0.6):
    """B skeleton states [B, J, 8] (float32) of random poses, their quaternions scaled off the unit sphere (0.8 to 1.25) and their
    scales multiplied by 0.8 to 1.2"""
    rng = np.random.default_rng(seed)
    theta = rng.normal(scale=spread, size=(B, ch.num_params))
    t, q, s = mc.forward_kinematics(ch, theta)
    q = q * rng.uniform(0.8, 1.25, (B, ch.num_joints, 1))
    s = s * rng.uniform(0.8, 1.2, (B, ch.num_joints))
    return np.concatenate([t, q, s[..., None]], -1).astype(np.float32)


def _magnitude(geo, i, j):
    g = geo[[i, j]]
    return max(np.abs(g[:, :3]).max(), np.abs(g[:, :3] + g[:, 3:6]).max(), np.abs(g[:, 6:]).max(), 1e-30)


def _usable(A, B):
    """whether a float64 pair evaluation is clear of every branch boundary and not nearly parallel"""
    d1, d2 = A[3:6], B[3:6]
    a, b, c = d1 @ d1, d1 @ d2, d2 @ d2
    if a * c - b * b < 1e-3 * a * c:
        return False
    margins = []
    mc.capsule_contact(A, B, margins=margins)
    return min(v for _, v in margins) >= 1e-4


def check_rows(caps, pairs, st, rows):
    """rows [B, P] against the float64 rows of the float32 states st; returns (worst ratio, excluded, contacts)"""
    geo = mc.capsule_world(caps, st.astype(np.float64))
    worst, excluded, contacts = 0.0, 0, 0
    for b in range(st.shape[0]):
        for k, (i, j) in enumerate(pairs):
            if not _usable(geo[b, i], geo[b, j]):
                excluded += 1
                continue
            c = mc.capsule_contact(geo[b, i], geo[b, j])
            r64 = WGT * c[4] if c[0] else 0.0
            contacts += bool(c[0])
            worst = max(worst, abs(float(rows[b, k]) - r64) / (WGT * _magnitude(geo[b], i, j)))
    return worst, excluded, contacts


def _signature(A, B):
    c = mc.capsule_contact(A, B)
    return c[0], c[5], c[6]


def fd_grad(caps, pairs, st, G, h=1e-6):
    """central differences of sum_k G_k row_k in float64, pair by pair over its parents' states; G_k is zeroed (in the returned copy)
    where pair k's branch changes within +-h"""
    st = st.astype(np.float64)
    par = np.array([c.parent for c in caps])
    G = np.array(G, np.float64)
    out = np.zeros_like(st)
    geo = mc.capsule_world(caps, st)
    for b in range(st.shape[0]):
        for k, (i, j) in enumerate(pairs):
            if G[b, k] == 0.0:
                continue
            base = _signature(geo[b, i], geo[b, j])
            joints = sorted({int(p) for p in (par[i], par[j]) if p >= 0})
            terms, stable = [], True
            for jt in joints:
                for e in range(8):
                    vals = []
                    for sgn in (1.0, -1.0):
                        x = st[b:b + 1].copy()
                        x[0, jt, e] += sgn * h
                        g = mc.capsule_world([caps[i], caps[j]], x)[0]
                        c = mc.capsule_contact(g[0], g[1])
                        if (c[0], c[5], c[6]) != base:
                            stable = False
                        vals.append(WGT * c[4] if c[0] else 0.0)
                    terms.append((jt, e, (vals[0] - vals[1]) / (2 * h)))
            if not stable:
                G[b, k] = 0.0
                continue
            for jt, e, d in terms:
                out[b, jt, e] += G[b, k] * d
    return out, G


def bwd_ratio(g, g64, G, st):
    """per instance ||g - g64||_inf over sqrt(5e-3) sum_k |G_k| (1 + max_j |t_j|): a state's gradient carries the rig's size"""
    size = 1.0 + np.abs(np.asarray(st, np.float64)[..., :3]).max(axis=(1, 2))
    scale = (WGT * np.abs(G).sum(-1) * size)[:, None, None] + 1e-30
    return float((np.abs(g - g64) / scale).max())


# ---- known answers --------------------------------------------------------------------------------------------------------------------
def _cap(o, d, r0, r1):
    return np.array([*o, *d, r0, r1], np.float32)


KNOWN = {
    # name: (A, B, hit, s, t, dist, sForm, tForm)
    "crossing interior": (_cap((-1, 0, 0), (2, 0, 0), 0.3, 0.3), _cap((0, -1, 0.2), (0, 2, 0), 0.3, 0.3), True, 0.5, 0.5, 0.2,
                          mc.SEG_INTERIOR, mc.SEG_INTERIOR),
    "endpoint t = 0": (_cap((-1, 0, 0), (2, 0, 0), 0.3, 0.3), _cap((0.5, 0.2, 0), (0, 1, 0), 0.3, 0.3), True, 0.75, 0.0, 0.2,
                       mc.SEG_EDGE0, mc.SEG_CONST),
    "endpoint t = 1": (_cap((-1, 0, 0), (2, 0, 0), 0.3, 0.3), _cap((0.5, -1.2, 0), (0, 1, 0), 0.3, 0.3), True, 0.75, 1.0, 0.2,
                       mc.SEG_EDGE1, mc.SEG_CONST),
    "endpoint s = 0": (_cap((0, 0, 0), (1, 0, 0), 0.3, 0.3), _cap((-0.2, -1, 0.1), (0, 2, 0), 0.3, 0.3), True, 0.0, 0.5, np.hypot(0.2, 0.1),
                       mc.SEG_CONST, mc.SEG_EDGE0),
    "endpoint s = 1": (_cap((0, 0, 0), (1, 0, 0), 0.3, 0.3), _cap((1.2, -1, 0.1), (0, 2, 0), 0.3, 0.3), True, 1.0, 0.5, np.hypot(0.2, 0.1),
                       mc.SEG_CONST, mc.SEG_EDGE1),
    "both clamped": (_cap((0, 0, 0), (1, 0, 0), 0.3, 0.3), _cap((1.2, 0.3, 0), (1, 1, 0), 0.3, 0.3), True, 1.0, 0.0, np.hypot(0.2, 0.3),
                     mc.SEG_CONST, mc.SEG_CONST),
    "tapered": (_cap((-1, 0, 0), (2, 0, 0), 0.5, 0.1), _cap((0, -1, 0.2), (0, 2, 0), 0.05, 0.25), True, 0.5, 0.5, 0.2,
                mc.SEG_INTERIOR, mc.SEG_INTERIOR),
    "parallel, close origins": (_cap((0, 0, 0), (1, 0, 0), 0.3, 0.3), _cap((0.1, 0.2, 0), (1, 0, 0), 0.3, 0.3), True, 0.1, 0.0, 0.2,
                                mc.SEG_EDGE0, mc.SEG_CONST),
    "parallel, distant origins": (_cap((0, 0, 0), (3, 0, 0), 0.3, 0.3), _cap((2, 0.2, 0), (1, 0, 0), 0.3, 0.3), False, 0, 0, 0, 0, 0),
    "snap of s": (_cap((0, 0, 0), (1, 0, 0), 0.3, 0.3), _cap((1e-8, -1, 0.1), (0, 2, 0), 0.3, 0.3), True, 0.0, 0.5, 0.1,
                  mc.SEG_CONST, mc.SEG_INTERIOR),
    "dist < 1e-8": (_cap((-1, 0, 0), (2, 0, 0), 0.3, 0.3), _cap((0, -1, 0), (0, 2, 0), 0.3, 0.3), False, 0, 0, 0, 0, 0),
    "apart": (_cap((-1, 0, 0), (2, 0, 0), 0.3, 0.3), _cap((0, -1, 0.7), (0, 2, 0), 0.3, 0.3), False, 0, 0, 0, 0, 0),
}


@pytest.mark.parametrize("name", list(KNOWN))
def test_emulated_contact_known_answers(emu, name):
    """each branch of closestPointsOnSegments: the contact, its parameters and branch, and the float64 restatement agreeing on them"""
    A, B, hit, s, t, dist, sf, tf = KNOWN[name]
    out, gA, gB = emu_contact(emu, A, B)
    c64 = mc.capsule_contact(A.astype(np.float64), B.astype(np.float64))
    assert bool(out[0]) == hit == c64[0]
    if not hit:
        assert not gA.any() and not gB.any()
        return
    assert out[1] == pytest.approx(s, abs=1e-6) and out[2] == pytest.approx(t, abs=1e-6)
    assert out[3] == pytest.approx(dist, rel=1e-5)
    assert (int(out[5]), int(out[6])) == (sf, tf) == (c64[5], c64[6])
    ra, rb = A[6] + s * (A[7] - A[6]), B[6] + t * (B[7] - B[6])
    assert out[4] == pytest.approx(ra + rb - dist, rel=1e-5)
    # the exact derivative: central differences of the float64 overlap, the branch held
    A64, B64 = A.astype(np.float64), B.astype(np.float64)
    fd = np.zeros(16)
    for k in range(16):
        v = []
        for sgn in (1, -1):
            x = np.concatenate([A64, B64])
            x[k] += sgn * 1e-9
            c = mc.capsule_contact(x[:8], x[8:])
            assert (c[0], c[5], c[6]) == (True, sf, tf)
            v.append(c[4])
        fd[k] = (v[0] - v[1]) / 2e-9
    np.testing.assert_allclose(np.concatenate([gA, gB]), fd, atol=2e-5 * (1 + np.abs(fd).max()))


def test_snap_changes_the_parameter():
    """the 1e-7 snap sets s to 0 where the division would give 1e-8, and makes it a constant of the backward"""
    A, B = KNOWN["snap of s"][:2]
    c = mc.capsule_contact(A.astype(np.float64), B.astype(np.float64))
    assert c[1] == 0.0 and c[5] == mc.SEG_CONST


# ---- the planner ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", RIGS)
def test_emulated_planner_matches_float64(emu, name):
    ch, caps = rig(name)
    pairs = emu_pairs(emu, ch, caps)
    ref = mc.collision_pairs(ch, caps)
    assert np.array_equal(pairs, ref)
    par = np.array([c.parent for c in caps])
    parents = np.asarray(ch.parents)
    kept = {tuple(p) for p in pairs.tolist()}
    # world-fixed pairs: both dropped, one kept; adjacent and same-joint pairs dropped; some rest-pose overlaps dropped
    world = np.nonzero(par < 0)[0]
    assert len(world) == 2 and tuple(world) not in kept
    assert all((int(w), int(k)) in kept or (int(k), int(w)) in kept for w in world for k in np.nonzero(par >= 0)[0])
    adjacent = [(i, j) for i in range(len(caps)) for j in range(i + 1, len(caps))
                if par[i] >= 0 and par[j] >= 0 and (par[i] == par[j] or parents[par[i]] == par[j] or parents[par[j]] == par[i])]
    assert adjacent and not kept & set(adjacent)
    candidates = len(caps) * (len(caps) - 1) // 2 - len(adjacent) - 1
    assert len(pairs) < candidates or name == "chain"  # the rest-pose filter dropped some


def test_synthetic_collision_rest_pose_is_clear():
    """every rest-pose pair the planner tests is overlapping or apart by a relative 1e-3, most capsules are tapered, some are not"""
    for name in ("humanoid72", "bodyhands300"):
        ch, caps = rig(name)
        r = np.array([c.radius for c in caps])
        assert (r[:, 0] != r[:, 1]).mean() > 0.5 and (r[:, 0] == r[:, 1]).any()
        assert sum(c.parent < 0 for c in caps) == 2
        t, q, s = mc.forward_kinematics(ch, np.zeros((1, ch.num_params)))
        geo = mc.capsule_world(caps, np.concatenate([t, q, s[..., None]], -1))[0]
        parents = np.asarray(ch.parents)
        worst, tested = np.inf, 0
        for i in range(len(caps)):
            for j in range(i + 1, len(caps)):
                p0, p1 = caps[i].parent, caps[j].parent
                if (p0 < 0 and p1 < 0) or (p0 >= 0 and p1 >= 0 and (p0 == p1 or parents[p0] == p1 or parents[p1] == p0)):
                    continue
                margins = []
                mc.capsule_contact(geo[i], geo[j], 1e-17, margins)
                worst = min(worst, min(v for what, v in margins if what != "branch"))
                tested += 1
        assert tested > 100 and worst >= 1e-3


# ---- rows and backward on the emulator ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", RIGS)
def test_emulated_rows_match_float64(emu, name):
    ch, caps = rig(name)
    pairs = emu_pairs(emu, ch, caps)
    B = 4 if name == "bodyhands300" else 12
    st = states(ch, B, 11)
    rows = emu_rows(emu, ch, caps, st, len(pairs))
    worst, excluded, contacts = check_rows(caps, pairs, st, rows)
    print(f"{name}: P = {len(pairs)}, worst {worst:.2e}, excluded {excluded} of {B * len(pairs)}, contacts {contacts}")
    assert worst <= K_FWD
    assert excluded <= 0.01 * B * len(pairs)
    assert contacts >= min(10 * B, B * len(pairs) // 10)
    # the sum of squares is getError's, and the nonzero rows are getJacobian's compacted residual
    r64 = mc.collision_rows(caps, pairs, st.astype(np.float64))
    np.testing.assert_allclose(np.square(rows.astype(np.float64)).sum(-1), np.square(r64).sum(-1), rtol=1e-4)


def _grad_case(emu, name, B=3, seed=21):
    ch, caps = rig(name)
    pairs = emu_pairs(emu, ch, caps)
    st = states(ch, B, seed)
    G = np.random.default_rng(seed).normal(size=(B, len(pairs))).astype(np.float32)
    rows = emu_rows(emu, ch, caps, st, len(pairs))
    G[rows == 0] = 0.0  # pairs without contact have no gradient; keeps the differences cheap
    g64, G = fd_grad(caps, pairs, st, G)
    return ch, caps, pairs, st, G.astype(np.float32), g64


@pytest.mark.parametrize("name", ["chain", "humanoid72"])
def test_emulated_backward_matches_central_differences(emu, name):
    ch, caps, pairs, st, G, g64 = _grad_case(emu, name)
    g = emu_grad(emu, ch, caps, st, G)
    ratio = bwd_ratio(g, g64, G, st)
    print(f"{name}: backward worst {ratio:.2e}, contacts used {(G != 0).sum()}")
    assert (G != 0).sum() >= 5
    assert ratio <= K_BWD
    # joints without a capsule get 0
    has = {c.parent for c in caps}
    none = [j for j in range(ch.num_joints) if j not in has]
    assert not g[:, none].any()


def _wrong(caps, pairs, st, G, variant):
    """float64 backwards that are wrong on purpose: the taper term dropped (getJacobian's fixed (s, t)), radii not scaled by the
    parent's s, or the normal flipped"""
    st64 = st.astype(np.float64)
    out = np.zeros_like(st64)
    for b in range(st.shape[0]):
        for k, (i, j) in enumerate(pairs):
            if G[b, k] == 0:
                continue
            for cap in (caps[i], caps[j]):
                if cap.parent < 0:
                    continue
                jt = cap.parent
                for e in range(8):
                    vals = []
                    for sgn in (1.0, -1.0):
                        x = st64[b:b + 1].copy()
                        x[0, jt, e] += sgn * 1e-6
                        geo = mc.capsule_world([caps[i], caps[j]], x)[0]
                        base = mc.capsule_world([caps[i], caps[j]], st64[b:b + 1])[0]
                        c0 = mc.capsule_contact(base[0], base[1])
                        if variant == "radii unscaled" and e == 7:
                            geo[:, 6:] = base[:, 6:]
                        if variant == "taper dropped":  # hold (s, t) at the base point
                            dP = geo[0, :3] + geo[0, 3:6] * c0[1] - geo[1, :3] - geo[1, 3:6] * c0[2]
                            ov = geo[0, 6] + c0[1] * (geo[0, 7] - geo[0, 6]) + geo[1, 6] + c0[2] * (geo[1, 7] - geo[1, 6]) - np.linalg.norm(dP)
                        elif variant == "normal flipped":
                            dP = geo[0, :3] + geo[0, 3:6] * c0[1] - geo[1, :3] - geo[1, 3:6] * c0[2]
                            ov = geo[0, 6] + c0[1] * (geo[0, 7] - geo[0, 6]) + geo[1, 6] + c0[2] * (geo[1, 7] - geo[1, 6]) + np.linalg.norm(dP)
                        else:
                            ov = mc.capsule_contact(geo[0], geo[1])[4]
                        vals.append(WGT * ov)
                    out[b, jt, e] += G[b, k] * (vals[0] - vals[1]) / 2e-6
    return out


@pytest.mark.parametrize("variant", ["taper dropped", "radii unscaled", "normal flipped"])
def test_bound_rejects_wrong_backwards(emu, variant):
    ch, caps, pairs, st, G, g64 = _grad_case(emu, "chain")
    wrong = _wrong(caps, pairs, st, G, variant)
    ratio = bwd_ratio(wrong.astype(np.float32), g64, G, st)
    print(f"{variant}: {ratio / K_BWD:.0f} x the bound")
    assert ratio > 10 * K_BWD


# ---- independent restatements: an exhaustive closest-point search, and momentum's getError / getJacobian from model parameters -------
# These do not follow closestPointsOnSegments' branches. The closest points of two segments are the best of the interior stationary
# point and the eight edge and corner candidates; CollisionErrorFunction::getJacobian is restated from collision_error_function.cpp and
# accumulateChainDerivatives (error_function_utils.h) over JointStateT's derivative axes (joint_state.cpp:22-82), in float64.
def closest_exhaustive(A, B):
    """(s, t, dist) minimising |o_A + s d_A - o_B - t d_B| over [0, 1]^2 by candidates"""
    d1, d2, w = A[3:6], B[3:6], A[:3] - B[:3]
    a, b, c, d, e = d1 @ d1, d1 @ d2, d2 @ d2, d1 @ w, d2 @ w
    cands = []
    D = a * c - b * b
    if D > 0:
        s_, t_ = (b * e - c * d) / D, (a * e - b * d) / D
        if 0 <= s_ <= 1 and 0 <= t_ <= 1:
            cands.append((s_, t_))
    for s_ in (0.0, 1.0):
        cands.append((s_, float(np.clip((e + s_ * b) / c, 0, 1)) if c > 0 else 0.0))
    for t_ in (0.0, 1.0):
        cands.append((float(np.clip((t_ * b - d) / a, 0, 1)) if a > 0 else 0.0, t_))
    best = min(cands, key=lambda st_: np.linalg.norm(w + st_[0] * d1 - st_[1] * d2))
    return best[0], best[1], float(np.linalg.norm(w + best[0] * d1 - best[1] * d2))


def overlap_exhaustive(A, B):
    """overlaps() at the exhaustive closest points: (hit, s, t, dist, overlap)"""
    s_, t_, dist = closest_exhaustive(A, B)
    ov = A[6] + s_ * (A[7] - A[6]) + B[6] + t_ * (B[7] - B[6]) - dist
    return ov > 0 and dist >= 1e-8, s_, t_, dist, ov


def planner_exhaustive(ch, caps):
    """isValidCollisionPair with the rest-pose test on overlap_exhaustive"""
    t, q, s = mc.forward_kinematics(ch, np.zeros((1, ch.num_params)))
    geo = mc.capsule_world(caps, np.concatenate([t, q, s[..., None]], -1))[0]
    parents = np.asarray(ch.parents)
    out = []
    for i in range(len(caps)):
        for j in range(i + 1, len(caps)):
            p0, p1 = caps[i].parent, caps[j].parent
            if p0 < 0 or p1 < 0:
                ok = p0 != p1
            elif p0 == p1 or parents[p0] == p1 or parents[p1] == p0:
                ok = False
            else:
                ok = not overlap_exhaustive(geo[i], geo[j])[0]
            if ok:
                out.append((i, j))
    return np.array(out, np.int64).reshape(-1, 2)


def _qmat(q):
    x, y, z, w = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def _joint_states(ch, theta):
    """JointStateT::set with derivatives, float64: per joint t, R, s, translationAxis (3x3), rotationAxis (3x3)"""
    J = ch.num_joints
    P = np.zeros((7 * J, ch.num_params))
    rows = np.repeat(np.arange(7 * J), np.diff(ch.pt_outer))
    np.add.at(P, (rows, ch.pt_inner), ch.pt_vals.astype(np.float64))
    jp = (P @ theta + ch.pt_offsets.astype(np.float64)).reshape(J, 7)
    out = []
    for j in range(J):
        p = jp[j]
        par = ch.parents[j]
        tp, Rp, sp = (np.zeros(3), np.eye(3), 1.0) if par < 0 else out[par][:3]
        pre = np.asarray(ch.prerot[j], np.float64)
        Rl = _qmat(pre / np.linalg.norm(pre))
        rot_axis = np.zeros((3, 3))
        for k in (2, 1, 0):
            rot_axis[:, k] = Rp @ Rl[:, k]
            ang = p[3 + k]
            c_, s_ = np.cos(ang), np.sin(ang)
            Rk = np.eye(3)
            i1, i2 = [(1, 2), (2, 0), (0, 1)][k]
            Rk[i1, i1], Rk[i1, i2], Rk[i2, i1], Rk[i2, i2] = c_, -s_, s_, c_
            Rl = Rl @ Rk
        tl = ch.offsets[j].astype(np.float64) + p[:3]
        out.append((tp + sp * Rp @ tl, Rp @ Rl, sp * np.exp2(p[6]), sp * Rp, rot_axis))
    return out, P


def reference_error_and_jacobian(ch, caps, pairs, theta, usable):
    """CollisionErrorFunction::getError, and getJacobian's residual and Jacobian [rows, n], at weight 1 for model parameters theta [n];
    pairs where usable[k] is False are skipped"""
    js, P = _joint_states(ch, theta)
    st = np.array([np.concatenate([t, _quat(R), [s]]) for t, R, s, _, _ in js])
    geo = mc.capsule_world(caps, st[None])[0]
    parents = np.asarray(ch.parents)
    wgt, ln2 = WGT, np.log(2.0)
    J = ch.num_joints

    def ancestor(a, b):
        while a != b:
            if a < 0 or b < 0:
                return -1
            if a < b:
                b = parents[b]
            else:
                a = parents[a]
        return a

    def chain(row, pos, direction, weight, start, stop, scale_corr):
        jt = start
        while jt >= 0 and jt != stop:
            t, _, _, tax, rax = js[jt]
            posd = pos - t
            for d in range(3):
                row[7 * jt + d] += direction @ tax[:, d] * weight
                row[7 * jt + 3 + d] += direction @ np.cross(rax[:, d], posd) * weight
            row[7 * jt + 6] += (direction @ (posd * ln2) + scale_corr) * weight
            jt = parents[jt]

    error, residual, jac, which = 0.0, [], [], []
    for k, (i, j) in enumerate(pairs):
        if not usable[k]:
            continue
        hit, s_, t_, dist, ov = overlap_exhaustive(geo[i], geo[j])
        if not hit:
            continue
        error += ov * ov * 5e-3
        pa, pb = geo[i, :3] + geo[i, 3:6] * s_, geo[j, :3] + geo[j, 3:6] * t_
        ra, rb = geo[i, 6] + s_ * (geo[i, 7] - geo[i, 6]), geo[j, 6] + t_ * (geo[j, 7] - geo[j, 6])
        direction, fac = pa - pb, wgt / dist
        lca = ancestor(caps[i].parent, caps[j].parent)
        row = np.zeros(7 * J)
        chain(row, pa, direction, -fac, caps[i].parent, lca, -dist * ra * ln2)
        chain(row, pb, direction, fac, caps[j].parent, lca, dist * rb * ln2)
        net = -fac * ln2 * (direction @ direction) + wgt * (ra + rb) * ln2
        a = lca
        while a >= 0:
            row[7 * a + 6] += net
            a = parents[a]
        residual.append(ov * wgt)
        jac.append(row @ P)
        which.append(k)
    return error, np.array(residual), np.array(jac).reshape(-1, ch.num_params), which


def _quat(R):
    w = np.sqrt(max(1.0 + R[0, 0] + R[1, 1] + R[2, 2], 1e-30)) / 2
    if w > 1e-3:
        return np.array([(R[2, 1] - R[1, 2]) / (4 * w), (R[0, 2] - R[2, 0]) / (4 * w), (R[1, 0] - R[0, 1]) / (4 * w), w])
    x = np.sqrt(max(1.0 + R[0, 0] - R[1, 1] - R[2, 2], 1e-30)) / 2
    return np.array([x, (R[0, 1] + R[1, 0]) / (4 * x), (R[0, 2] + R[2, 0]) / (4 * x), (R[2, 1] - R[1, 2]) / (4 * x)])


def _emu_model_gradient(L, ch, theta, gstate):
    keep = []
    th = np.ascontiguousarray(theta, np.float32)
    gs = np.ascontiguousarray(gstate, np.float32)
    out = np.zeros(th.shape, np.float32)
    L.emu_skeleton_state_backward.argtypes = _CHARACTER + [_i32, _p, _p, _p]
    _check(L, L.emu_skeleton_state_backward(*emu_lib.character_args(ch, keep), th.shape[0], th.ctypes.data, gs.ctypes.data, out.ctypes.data))
    return out


def _reference_case(L, ch, caps, B=4, seed=31):
    """model parameters, their float32 states, the emulated rows, and getError / getJacobian restated at every instance"""
    pairs = emu_pairs(L, ch, caps)
    theta = np.random.default_rng(seed).normal(scale=0.6, size=(B, ch.num_params))
    t, q, s = mc.forward_kinematics(ch, theta)
    st = np.concatenate([t, q, s[..., None]], -1).astype(np.float32)
    rows = emu_rows(L, ch, caps, st, len(pairs))
    geo = mc.capsule_world(caps, st.astype(np.float64))
    refs = []
    for b in range(B):
        usable = [_usable(geo[b, i], geo[b, j]) for i, j in pairs]
        refs.append(reference_error_and_jacobian(ch, caps, pairs, theta[b], usable) + (usable,))
    return pairs, theta, st, rows, refs


def check_rows_exhaustive(caps, pairs, st, rows):
    """rows [B, P] against overlap_exhaustive on the float64 geometry of the float32 states st, the pairs _usable leaves in:
    (worst ratio, contacts)"""
    geo = mc.capsule_world(caps, st.astype(np.float64))
    worst, contacts = 0.0, 0
    for b in range(st.shape[0]):
        for k, (i, j) in enumerate(pairs):
            if not _usable(geo[b, i], geo[b, j]):
                continue
            hit, _, _, _, ov = overlap_exhaustive(geo[b, i], geo[b, j])
            contacts += hit
            worst = max(worst, abs(float(rows[b, k]) - (WGT * ov if hit else 0.0)) / (WGT * _magnitude(geo[b], i, j)))
    return worst, contacts


@pytest.mark.parametrize("name", ["chain", "humanoid72", "bodyhands300"])
def test_emulated_planner_and_rows_match_exhaustive_search(emu, name):
    """the planned pairs and the rows against the exhaustive closest-point search, which shares no branch with closestPointsOnSegments"""
    ch, caps = rig(name)
    pairs = emu_pairs(emu, ch, caps)
    assert np.array_equal(pairs, planner_exhaustive(ch, caps))
    B = {"chain": 16, "humanoid72": 8, "bodyhands300": 2}[name]
    st = states(ch, B, 13)
    worst, contacts = check_rows_exhaustive(caps, pairs, st, emu_rows(emu, ch, caps, st, len(pairs)))
    print(f"{name}: rows against the exhaustive search, worst {worst:.2e}, contacts {contacts}")
    assert contacts >= B and worst <= K_FWD


@pytest.mark.parametrize("name", ["chain", "humanoid72"])
def test_emulated_rows_are_geterror_and_getjacobian_residual(emu, name):
    """the sum of squares of the usable rows is getError, and their nonzero rows in order are getJacobian's compacted residual"""
    ch, caps = rig(name)
    pairs, theta, st, rows, refs = _reference_case(emu, ch, caps, B=16 if name == "chain" else 4)
    for b, (error, residual, _, which, usable) in enumerate(refs):
        r = rows[b, np.asarray(usable, bool)].astype(np.float64)
        assert np.square(r).sum() == pytest.approx(error, rel=1e-5, abs=1e-12)
        assert np.array_equal(np.nonzero(rows[b])[0][np.isin(np.nonzero(rows[b])[0], which)], np.array(which, int))
        np.testing.assert_allclose(rows[b, which], residual, rtol=1e-5, atol=1e-6 * WGT * np.abs(st[b, :, :3]).max())


@pytest.mark.parametrize("name", ["chain", "humanoid72"])
def test_getjacobian_composed_through_the_skeleton_state_backward(emu, name):
    """momentum's getJacobian^T g, restated from model parameters (chains to the common ancestor, the ln2 scale corrections, P^T), equals
    the emulated backward composed with the skeleton-state emulator's backward on untapered capsules; on tapered ones it misses the
    taper term, so the two differ by far more than the bound"""
    ch, caps = rig(name)
    flat = [mc.dataclasses.replace(c, radius=(c.radius[0], c.radius[0])) for c in caps]
    for capsules, tapered in ((flat, False), (caps, True)):
        pairs, theta, st, rows, refs = _reference_case(emu, ch, capsules, B=16 if name == "chain" else 4)
        G = np.random.default_rng(2).normal(size=rows.shape).astype(np.float32)
        jtg = np.zeros(theta.shape)
        for b, (_, _, jac, which, usable) in enumerate(refs):
            G[b, ~np.asarray(usable, bool)] = 0.0
            jtg[b] = jac.T @ G[b, which].astype(np.float64) if which else 0.0
        g = _emu_model_gradient(emu, ch, theta, emu_grad(emu, ch, capsules, st, G))
        size = 1.0 + np.abs(st[..., :3]).max(axis=(1, 2))
        ratio = float((np.abs(g - jtg) / (WGT * np.abs(G).sum(-1) * size + 1e-30)[:, None]).max())
        print(f"{name} {'tapered' if tapered else 'untapered'}: |g - J^T g| ratio {ratio:.2e}, contacts {sum(len(r[3]) for r in refs)}")
        assert sum(len(r[3]) for r in refs) >= 5
        if tapered:
            assert ratio > 10 * K_JAC
        else:
            assert ratio <= K_JAC


def test_emulated_coverage_of_branches(emu):
    """the random poses reach every branch: interior, both edges of each parameter, clamps, and tapered, untapered and world-fixed
    capsules in contact"""
    seen_s, seen_t, kinds = set(), set(), set()
    for name in ("chain", "humanoid72"):
        ch, caps = rig(name)
        pairs = emu_pairs(emu, ch, caps)
        geo = mc.capsule_world(caps, states(ch, 8, 5).astype(np.float64))
        for b in range(geo.shape[0]):
            for i, j in pairs:
                c = mc.capsule_contact(geo[b, i], geo[b, j])
                if c[0]:
                    seen_s.add(c[5]); seen_t.add(c[6])
                    for k in (i, j):
                        cap = caps[k]
                        kinds.add("world" if cap.parent < 0 else "tapered" if cap.radius[0] != cap.radius[1] else "untapered")
    assert seen_s == seen_t == {mc.SEG_CONST, mc.SEG_INTERIOR, mc.SEG_EDGE0, mc.SEG_EDGE1}
    assert kinds == {"world", "tapered", "untapered"}


# ---- launches -------------------------------------------------------------------------------------------------------------------------
def ballast(ch, caps, count):
    """caps plus `count` small capsules on joint 0 far from the body: their pairs are valid and never in contact"""
    far = [mc.TaperedCapsule(0, (1e4 + 10.0 * k, 0.0, 0.0), (0.0, 0.0, 0.0, 1.0), 1.0, (0.01, 0.01), 0.1) for k in range(count)]
    return caps + far


def emu_launch(L, ch, caps, backward, batch=4096):
    keep, out = [], np.zeros(5, np.int64)
    _check(L, L.emu_collision_launch(*_args(ch, caps, keep), int(backward), batch, H100_SXM[1], H100_SXM[0], out.ctypes.data))
    return out


def variant_rig(L, W, backward):
    """the chain rig with enough ballast capsules that the planner picks W warps per instance"""
    ch, caps = rig("chain")
    per = {1: 0, 2: 5, 4: 3, 8: 1}[W]  # instances per CTA that give W
    count = 0 if W == 1 else int(np.ceil((H100_SXM[1] - 16) / (per + 1) / 32 / (2 if backward else 1))) + 1 - len(caps)
    big = ballast(ch, caps, count)
    assert emu_launch(L, ch, big, backward)[0] == W
    return ch, big


VARIANTS = [(W, b) for W in (1, 2, 4, 8) for b in (False, True)]


@pytest.mark.parametrize("W,backward", VARIANTS)
def test_emulated_launch_variants(emu, W, backward):
    ch, big = variant_rig(emu, W, backward)
    _, caps = rig("chain")
    pairs, small = emu_pairs(emu, ch, big), emu_pairs(emu, ch, caps)
    idx = [k for k, p in enumerate(map(tuple, pairs.tolist())) if p in set(map(tuple, small.tolist()))]
    st = states(ch, 2, 9)
    if backward:
        G = np.zeros((2, len(pairs)), np.float32)
        G[:, idx] = np.random.default_rng(1).normal(size=(2, len(idx)))
        assert np.array_equal(emu_grad(emu, ch, big, st, G), emu_grad(emu, ch, caps, st, G[:, idx]))
    else:
        rows = emu_rows(emu, ch, big, st, len(pairs))
        assert np.array_equal(rows[:, idx], emu_rows(emu, ch, caps, st, len(small)))
        assert not np.delete(rows, idx, axis=1).any()


# ---- rejections -----------------------------------------------------------------------------------------------------------------------
BAD = {
    "parent": (dict(parent=6), "parent 6 is outside"),
    "parent below -1": (dict(parent=-2), "parent -2 is outside"),
    "radius": (dict(radius=(0.1, -0.1)), "radius is negative"),
    "length": (dict(length=-1.0), "length is negative"),
    "nan": (dict(translation=(0.0, float("nan"), 0.0)), "must be finite"),
    "inf": (dict(scale=float("inf")), "must be finite"),
    "overflow": (dict(scale=1e30, length=1e30), "overflows float"),
}


@pytest.mark.parametrize("what", list(BAD))
def test_emulated_rejections(emu, what):
    ch, caps = rig("chain")
    change, message = BAD[what]
    bad = list(caps)
    bad[3] = mc.dataclasses.replace(bad[3], **change)
    keep, n = [], ctypes.c_int32(0)
    assert emu.emu_collision_pairs(*_args(ch, bad, keep), ctypes.byref(n), None) != 0
    err = emu.emu_last_error().decode()
    assert "capsule 3" in err and message in err


def test_emulated_empty_geometry(emu):
    ch, _ = rig("chain")
    assert len(emu_pairs(emu, ch, [])) == 0
    st = states(ch, 2, 1)
    assert not emu_grad(emu, ch, [], st, np.zeros((2, 0), np.float32)).any()


def test_wrappers_reject_without_a_device():
    from momentum_b200 import torch_skeleton as tsk
    ch, _ = rig("chain")
    with pytest.raises(ValueError, match="CUDA"):
        tsk.collision_residual(ch, torch.zeros(ch.num_joints, 8))


# ---- on the GPU -----------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", RIGS)
def test_device_matches_float64(name):
    from momentum_b200 import torch_skeleton as tsk
    ch, caps = rig(name)
    c = mc.dataclasses.replace(ch, collision=caps)
    pairs = tsk.collision_pairs(c).numpy()
    assert np.array_equal(pairs, mc.collision_pairs(ch, caps))
    B = 4 if name == "bodyhands300" else 12
    st = states(ch, B, 11)
    x = torch.from_numpy(st).cuda().requires_grad_(True)
    rows = tsk.collision_residual(c, x)
    worst, excluded, contacts = check_rows(caps, pairs, st, rows.detach().cpu().numpy())
    print(f"{name}: forward worst {worst:.2e}, excluded {excluded}, contacts {contacts}")
    assert worst <= K_FWD and excluded <= 0.01 * B * len(pairs)
    assert np.array_equal(pairs, planner_exhaustive(ch, caps))
    worst_x, _ = check_rows_exhaustive(caps, pairs, st, rows.detach().cpu().numpy())
    print(f"{name}: forward against the exhaustive search, worst {worst_x:.2e}")
    assert worst_x <= K_FWD
    if name != "bodyhands300":
        G = np.random.default_rng(21).normal(size=(B, len(pairs))).astype(np.float32)
        G[rows.detach().cpu().numpy() == 0] = 0.0
        g64, G = fd_grad(caps, pairs, st, G)
        (g,) = torch.autograd.grad(rows, x, torch.from_numpy(G).cuda())
        ratio = bwd_ratio(g.cpu().numpy(), g64, G, st)
        print(f"{name}: backward worst {ratio:.2e}")
        assert ratio <= K_BWD


@pytest.mark.gpu
@pytest.mark.parametrize("W,backward", VARIANTS)
def test_device_launch_variants(emu, W, backward):
    """every W launch bitwise equal to the default launch of the unballasted rig"""
    ch, big = variant_rig(emu, W, backward)
    _, caps = rig("chain")
    dc, dc0 = ms.DeviceCharacter(mc.dataclasses.replace(ch, collision=big)), ms.DeviceCharacter(mc.dataclasses.replace(ch, collision=caps))
    B = 300
    launch = dc.get_instance_launch("collision_residual", backward, B)
    assert launch["warps"] == W
    pairs, small = dc.collision_pairs(), dc0.collision_pairs()
    idx = [k for k, p in enumerate(map(tuple, pairs.tolist())) if p in set(map(tuple, small.tolist()))]
    from momentum_b200 import torch_skeleton as tsk
    st = torch.from_numpy(states(ch, B, 9)).cuda().requires_grad_(True)
    rows, rows0 = tsk.collision_residual(dc, st), tsk.collision_residual(dc0, st)
    assert torch.equal(rows[:, idx], rows0)
    if backward:
        G0 = torch.randn(rows0.shape, device="cuda", generator=torch.Generator("cuda").manual_seed(3))
        G = torch.zeros_like(rows)
        G[:, idx] = G0
        (g,) = torch.autograd.grad(rows, st, G)
        (g0,) = torch.autograd.grad(rows0, st, G0)
        assert torch.equal(g, g0)


@pytest.mark.gpu
def test_device_batch_independence_and_dtype():
    from momentum_b200 import torch_skeleton as tsk
    ch, caps = rig("humanoid72")
    c = mc.dataclasses.replace(ch, collision=caps)
    st = torch.from_numpy(states(ch, 257, 2)).cuda().requires_grad_(True)
    rows = tsk.collision_residual(c, st)
    G = torch.randn(rows.shape, device="cuda", generator=torch.Generator("cuda").manual_seed(1))
    (g,) = torch.autograd.grad(rows, st, G)
    for b in (0, 100, 256):
        one = st[b].detach().clone().requires_grad_(True)
        r1 = tsk.collision_residual(c, one)
        assert r1.shape == rows.shape[1:] and torch.equal(r1, rows[b])
        (g1,) = torch.autograd.grad(r1, one, G[b])
        assert torch.equal(g1, g[b])
    s64 = st.detach().double().requires_grad_(True)
    r64 = tsk.collision_residual(c, s64)
    assert r64.dtype == torch.float64 and torch.equal(r64.float(), rows)
    (g64,) = torch.autograd.grad(r64, s64, G.double())
    assert g64.dtype == torch.float64 and torch.equal(g64.float(), g)


@pytest.mark.gpu
def test_model_parameter_loss_gradient_matches_central_differences():
    """model_parameters_to_skeleton_state -> collision_residual -> .square().sum(): its gradient against float64 central differences in
    the model parameters, over the parameters whose perturbation leaves every pair's branch unchanged"""
    from momentum_b200 import torch_skeleton as tsk
    ch, caps = rig("chain")
    c = mc.dataclasses.replace(ch, collision=caps)
    pairs = mc.collision_pairs(ch, caps)
    rng = np.random.default_rng(8)
    theta = rng.normal(scale=0.6, size=(4, ch.num_params))
    x = torch.from_numpy(theta.astype(np.float32)).cuda().requires_grad_(True)
    loss = tsk.collision_residual(c, tsk.model_parameters_to_skeleton_state(c, x)).square().sum()
    (g,) = torch.autograd.grad(loss, x)
    g = g.cpu().numpy()

    def state(th):
        t, q, s = mc.forward_kinematics(ch, th)
        return np.concatenate([t, q, s[..., None]], -1)

    def signature(st):
        geo = mc.capsule_world(caps, st)
        return [_signature(geo[0, i], geo[0, j]) for i, j in pairs]

    h, used, worst = 1e-6, 0, 0.0
    for b in range(theta.shape[0]):
        base = signature(state(theta[b:b + 1]))
        if not any(s[0] for s in base):
            continue
        scale = float(np.abs(mc.collision_rows(caps, pairs, state(theta[b:b + 1]))).sum()) * WGT * 10 + 1e-12
        for p in range(ch.num_params):
            vals = []
            stable = True
            for sgn in (1.0, -1.0):
                th = theta[b:b + 1].copy()
                th[0, p] += sgn * h
                st = state(th)
                stable &= signature(st) == base
                vals.append(np.square(mc.collision_rows(caps, pairs, st)).sum())
            if not stable:
                continue
            used += 1
            worst = max(worst, abs(g[b, p] - (vals[0] - vals[1]) / (2 * h)) / scale)
    print(f"model-parameter gradient: {used} components, worst {worst:.2e}")
    assert used >= 10 and worst <= 1e-4


@pytest.mark.gpu
def test_device_rejections_and_empty_geometry():
    from momentum_b200 import torch_skeleton as tsk
    ch, caps = rig("chain")
    st = torch.from_numpy(states(ch, 3, 1)).cuda()
    with pytest.raises(ValueError, match="no collision geometry"):
        tsk.collision_residual(ch, st)
    empty = mc.dataclasses.replace(ch, collision=[])
    r = tsk.collision_residual(empty, st.requires_grad_(True))
    assert r.shape == (3, 0) and tsk.collision_pairs(empty).shape == (0, 2)
    (g,) = torch.autograd.grad(r.sum() + 0 * st.sum(), st)
    assert not g.any()
    with pytest.raises(ValueError, match="skel_state"):
        tsk.collision_residual(mc.dataclasses.replace(ch, collision=caps), st[:, :-1])
    bad = list(caps)
    bad[2] = mc.dataclasses.replace(bad[2], radius=(-1.0, 1.0))
    dc = ms.DeviceCharacter(ch)
    with pytest.raises(ms.MomentumB200Error, match="capsule 2"):
        dc.set_collision_geometry(bad)
    with pytest.raises(ValueError, match="capsule 2"):
        tsk.collision_residual(mc.dataclasses.replace(ch, collision=bad), st)
    with pytest.raises(ms.MomentumB200Error, match="no collision geometry"):
        dc.collision_pairs()
    dc.set_collision_geometry(caps)
    assert np.array_equal(dc.collision_pairs(), mc.collision_pairs(ch, caps))
    # replacing the attribute makes a new handle; the old graph keeps its own
    c = mc.dataclasses.replace(ch, collision=caps)
    h0 = tsk._handle(c, st.device).dc
    c.collision = caps[:-1]
    assert tsk._handle(c, st.device).dc is not h0
