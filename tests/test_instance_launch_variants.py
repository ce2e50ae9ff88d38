"""The per-instance kernels of the character operations (skeletonStateKernel, positionsKernel, inputGradientKernel) at every launch
variant, against the float64 references of their own test modules.

One host rule (ik_instance_launch.cpp, planInstanceOp) picks the warps per instance W and the instance groups per CTA from how many
instances fit in shared memory next to the tables; the library launches what it plans and reports it (get_instance_launch,
get_input_gradient_launch), and the CPU emulator library runs the same rule. The rigs that reach each variant are the fixtures of
test_skeleton_state with a "ballast" appended: a second root tree (a 4-ary tree, 7 levels at most, shallower than bodyhands300) with
random offsets and pre-rotations, a root with six DOFs of its own and a 3-DOF rotation on every eighth joint. Its size is searched on the
CPU through the emulated rule and asserted on the device through the query.

Two properties make this a strong check. The original joints' states and the original parameters' gradients do not depend on the
ballast: every output element is one lane's fixed-order sum, and the ballast is a separate tree with its own parameters; so they must
equal the unballasted W = 1 run bit for bit. And the ballast joints are served by lanes 32 .. 32 W - 1 and by the deeper levels, where a
stride or barrier error would show; they are held to the pinned float64 bounds (K_BOUND, K_POS / K_GRAD / K_OFF, the joint-parameter FK
bounds, the input gradients' K_BOUND). A variant's point tables are unstaged when the rig is sized to the top of its fit range, where no
point table fits in the slack; staged when sized to the bottom.
"""
import collections
import ctypes

import numpy as np
import pytest
import torch

from momentum_b200 import character as mc
from momentum_b200 import solver as ms
from tests import emu_lib
from tests import test_joint_parameters as tjp
from tests import test_positions as tpos
from tests import test_skeleton_state as tss
from tests import test_solve_ik_input_gradients as tig

FIXTURES = tss.FIXTURES
H100_SMEM, H100_SMS = 227 * 1024, 132  # opt-in shared memory per CTA and SMs of an H100 SXM: the CPU tables below
OP_CODES = {**ms.INSTANCE_OPS, "input_gradients": 4}  # emu_instance_launch's op codes
# variant -> instances that fit next to the tables (before a small batch is spread), and the W the rule gives them
VARIANTS = {"W1x16": (16, 1), "W2": (6, 2), "W4": (3, 4), "W8fit2": (2, 8), "W8fit1": (1, 8)}
REPORT = {"worst": collections.defaultdict(dict), "census": set(), "cases": []}


# ---- the rule ---------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu():
    L = emu_lib.load()
    L.emu_positions.argtypes = tpos._CHARACTER + tpos._POINTS + [ctypes.c_void_p]
    L.emu_positions_backward.argtypes = tpos._CHARACTER + tpos._POINTS + [ctypes.c_void_p] * 3
    L.emu_joint_parameters.argtypes = tjp._EMU_SIGNATURE
    return L


def _rule(L, per, tables, batch, smem=H100_SMEM, sms=H100_SMS):
    out = (ctypes.c_int64 * 5)()
    assert L.emu_plan_instance_groups(per, tables, batch, smem, sms, out) == 0
    return dict(zip(("warps", "groups", "threads", "smem"), (int(v) for v in out[:4])))


def _plan(L, ch, op, backward, batch, N=0, smem=H100_SMEM, sms=H100_SMS):
    keep, out = [], (ctypes.c_int64 * 5)()
    rc = L.emu_instance_launch(*emu_lib.character_args(ch, keep), OP_CODES[op], int(backward), batch, N, smem, sms, out)
    assert rc == 0, L.emu_last_error().decode()
    return dict(zip(("warps", "groups", "threads", "smem", "staged"), (int(v) for v in out)))


# fit -> (W, groups per CTA before spreading): fit >= 8 one warp each, up to 16; 5-7 two warps; 3-4 four; 1-2 eight
EXPECTED_RULE = {1: (8, 1), 2: (8, 2), 3: (4, 3), 4: (4, 4), 5: (2, 5), 6: (2, 6), 7: (2, 7), **{f: (1, min(f, 16)) for f in range(8, 21)}}


@pytest.mark.parametrize("fit", list(range(1, 21)))
def test_rule_table(emu, fit):
    """Per-instance bytes that fit exactly `fit` instances next to 10 000 bytes of tables: W and the groups per CTA as listed, and a
    batch just below SMs x groups spread at ceil(B / SMs) groups per CTA."""
    tables = 10000
    per = (H100_SMEM - tables - 16) // fit  # exactly `fit` instances
    W, groups = EXPECTED_RULE[fit]
    full = _rule(emu, per, tables, H100_SMS * groups)
    assert full == {"warps": W, "groups": groups, "threads": 32 * W * groups, "smem": per * groups + tables + 16}, full
    assert _rule(emu, per, tables, H100_SMS * groups + 1) == full
    below = _rule(emu, per, tables, H100_SMS * groups - 1)
    assert below["warps"] == W and below["groups"] == -(-(H100_SMS * groups - 1) // H100_SMS)
    assert _rule(emu, per, tables, 1)["groups"] == 1 and _rule(emu, per, tables, H100_SMS)["groups"] == 1
    assert _rule(emu, per + 1, tables, 10 ** 6)["groups"] == min(fit - 1, 16)


def test_rule_refuses_an_instance_that_does_not_fit(emu):
    tables = 50000
    per = H100_SMEM - tables - 16
    assert _rule(emu, per, tables, 5)["groups"] == 1
    assert _rule(emu, per + 1, tables, 5) == {"warps": 0, "groups": 0, "threads": 0, "smem": 0}
    assert _rule(emu, 100, H100_SMEM, 5)["groups"] == 0
    assert _rule(emu, 100, 1000, 0)["groups"] == 0  # an empty batch launches nothing


# ---- rigs -------------------------------------------------------------------------------------------------------------------------------
_BALLAST = {}


def ballast(ch, K):
    """ch with a second root tree of K joints appended (see the module docstring); the original joints and parameters keep their
    indices"""
    if K == 0:
        return ch
    if (ch.name, K) in _BALLAST:
        return _BALLAST[ch.name, K]
    rng = np.random.default_rng(1000 + K)
    J, n = ch.num_joints, ch.num_params
    parents = np.concatenate([ch.parents, [-1], J + (np.arange(1, K) - 1) // 4]).astype(np.int32)
    offsets = np.concatenate([ch.offsets, rng.uniform(-0.5, 0.5, (K, 3))]).astype(np.float32)
    axis = rng.normal(size=(K, 3))
    half = np.deg2rad(rng.uniform(0, 30, (K, 1))) / 2  # mc._random_prerot, vectorised
    q = np.concatenate([axis / np.linalg.norm(axis, axis=1, keepdims=True) * np.sin(half), np.cos(half)], 1)
    prerot = np.concatenate([ch.prerot, q]).astype(np.float32)
    rows = np.repeat(np.arange(7 * J), np.diff(ch.pt_outer))
    trip = list(zip(rows.tolist(), ch.pt_inner.tolist(), ch.pt_vals.tolist()))
    p = n
    for k in range(0, K, 8):
        for d in (range(6) if k == 0 else range(3, 6)):
            trip.append((7 * (J + k) + d, p, 1.0)); p += 1
    outer, inner, vals = mc._csr_from_triplets(7 * (J + K), p, trip)
    pt_off = np.concatenate([ch.pt_offsets, np.zeros(7 * K)]).astype(np.float32)
    rig = _BALLAST[ch.name, K] = mc.Character(parents, offsets, prerot, p, outer, inner, vals, pt_off, [], f"{ch.name}+{K}")
    return rig


def _points(ch, J0, K, N):
    """N point parents: the fixture's point set (N = 0) or N - 16 random original joints, then 16 on ballast joints"""
    rng = np.random.default_rng(J0 + N)
    base = tpos._point_sets(ch)["several"] if N == 0 else rng.integers(0, J0, N - 16).astype(np.int32)
    extra = rng.integers(J0, J0 + K, 16) if K else np.zeros(0)
    return np.concatenate([base, extra]).astype(np.int32), len(base)


def _fit_range(L, ch, op, backward, N, fit):
    """the least and the largest ballast with `fit` instance groups per CTA (None when the fixture alone fits fewer)"""
    groups = lambda K: _plan(L, ballast(ch, K), op, backward, 1 << 40, _points(ch, ch.num_joints, K, N)[0].size if "positions" in op else 0)["groups"]
    if groups(0) < fit:
        return None
    def least(pred):  # the least K in [0, 1 << 13] where pred holds (pred is monotone)
        lo, hi = 0, 1 << 13
        while lo < hi:
            mid = (lo + hi) // 2
            lo, hi = (lo, mid) if pred(mid) else (mid + 1, hi)
        return lo
    lo = max(16, least(lambda K: groups(K) <= fit)) if fit < 16 else 16
    hi = least(lambda K: groups(K) < fit) - 1
    return (lo, hi) if lo <= hi and groups(lo) == fit else None


_RIGS = {}


def rig_for(L, op, backward, variant, staged=True, start=0):
    """(fixture name, ballasted rig, K, point parents, original point count) reaching `variant` with the point tables staged or not,
    the fixture alone launching W = 1: fixtures tried in turn from `start`"""
    key = (op, backward, variant, staged, start)
    if key not in _RIGS:
        _RIGS[key] = _rig_for(L, *key)
    return _RIGS[key]


def _rig_for(L, op, backward, variant, staged, start):
    fit, W = VARIANTS[variant]
    names = list(FIXTURES)
    for i in range(len(names)):
        name = names[(start + i) % len(names)]
        ch = FIXTURES[name]()
        N = (0 if staged else 1024) if "positions" in op else 0
        if _plan(L, ch, op, backward, 1 << 40, _points(ch, ch.num_joints, 0, N)[0].size if N or "positions" in op else 0)["warps"] != 1:
            continue
        r = _fit_range(L, ch, op, backward, N, fit)
        if r is None:
            continue
        K = r[0] if staged else r[1]
        rig = ballast(ch, K)
        parents, n0 = _points(ch, ch.num_joints, K, N) if "positions" in op else (np.zeros(0, np.int32), 0)
        p = _plan(L, rig, op, backward, 1 << 40, parents.size)
        if (p["warps"], p["groups"]) == (W, fit) and ("positions" not in op or p["staged"] == int(staged)):
            return name, ch, rig, K, parents, n0
    raise AssertionError(f"no fixture reaches {op} backward={backward} {variant} staged={staged}")


# ---- the cases --------------------------------------------------------------------------------------------------------------------------
OPS = [(op, bwd, st) for op in ("model_parameters_to_skeleton_state", "joint_parameters_to_skeleton_state") for bwd in (False, True) for st in (True,)] + \
      [(op, bwd, st) for op in ("model_parameters_to_positions", "joint_parameters_to_positions") for bwd in (False, True) for st in (True, False)] + \
      [("input_gradients", False, True)]
CASES = [(op, bwd, st, v) for (op, bwd, st) in OPS for v in VARIANTS]
IG_BLOCKS = [(0, False), (1, True), (0, True), (1, False), (0, False)]  # (kind, instanced) per variant: Position and Orientation, both layouts


def _case_id(c):
    op, bwd, st, v = c
    return f"{op}-{'bwd' if bwd else 'fwd'}{'' if 'positions' not in op else '-staged' if st else '-unstaged'}-{v}"


def _joint(op):
    return op.startswith("joint")


def _inputs(ch, op, B, seed, rig=None):
    """inputs of the rig whose first columns are those of the fixture ch: (params [B, in], G) for the skeleton state"""
    rig = rig or ch
    rng = np.random.default_rng(seed)
    if _joint(op):
        x = tjp._joint_params(rig, B, seed).reshape(B, -1).astype(np.float32)
    else:
        x = rng.uniform(-0.5, 0.5, (B, rig.num_params)).astype(np.float32)
    G = rng.normal(size=(B, rig.num_joints, 8)).astype(np.float32)
    return x, G


def _skeleton_emu(L, ch, op, backward, x, G):
    if _joint(op):
        return tjp._emu_run(L, ch, "joint_parameters_to_skeleton_state", x, G if backward else None)
    assert backward  # the model-parameter forward has no emulator entry of its own: its FK is the joint-parameter one after the transform
    return tss._emu_backward(L, ch, x, G)


def _skeleton_bounds(ch, op, backward, x, G, out):
    """per instance error / pinned bound"""
    if not backward:
        jp = tss._joint_parameters(ch, x) if not _joint(op) else torch.from_numpy(x.astype(np.float64)).reshape(x.shape[0], -1, 7)
        ref = tss._fk64(ch, jp).reshape(x.shape[0], -1).numpy()
        xin = jp.reshape(x.shape[0], -1).numpy()
        return tjp._forward_error(ch, "joint_parameters_to_skeleton_state", xin, out.reshape(x.shape[0], -1), ref) / tjp.K_FWD["joint_parameters_to_skeleton_state"]
    if _joint(op):
        g64 = tjp._grad64(ch, "joint_parameters_to_skeleton_state", x, G.reshape(x.shape[0], -1))
        return tjp._bound_ratio(out, g64) / tjp.K_BWD["joint_parameters_to_skeleton_state"]
    return tss._bound_ratio(out, tss._g64(ch, x, G)) / tss.K_BOUND


# ---- CPU: the emulator on the ballasted rigs ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("variant", ["W4", "W8fit1"])
@pytest.mark.parametrize("op", ["model_parameters_to_skeleton_state", "joint_parameters_to_skeleton_state", "model_parameters_to_positions",
                                "joint_parameters_to_positions", "input_gradients"])
def test_emulated_ballast_keeps_the_original_bits_and_meets_the_bounds(emu, op, variant):
    """The emulator (one lane at a time, no W) on a ballasted rig: the fixture's outputs bit for bit as without the ballast, and every
    output, ballast included, within the pinned float64 bound."""
    backward = op != "input_gradients"
    name, ch, rig, K, parents, n0 = rig_for(emu, op, backward, variant, start=len(op))
    B = 2
    if "skeleton_state" in op:
        x, G = _inputs(ch, op, B, 3, rig)
        x0 = x[:, :7 * ch.num_joints] if _joint(op) else x[:, :ch.num_params]
        g = _skeleton_emu(emu, rig, op, True, x, G)
        g0 = _skeleton_emu(emu, ch, op, True, x0, G[:, :ch.num_joints])
        assert np.array_equal(g[:, :x0.shape[1]], g0)
        assert _skeleton_bounds(rig, op, True, x, G, g).max() <= 1.0
        if _joint(op):
            s = _skeleton_emu(emu, rig, op, False, x, None).reshape(B, -1, 8)
            assert np.array_equal(s[:, :ch.num_joints], _skeleton_emu(emu, ch, op, False, x0, None).reshape(B, -1, 8))
            assert _skeleton_bounds(rig, op, False, x, None, s).max() <= 1.0
    elif "positions" in op:
        joint = _joint(op)
        params, off, G = _positions_inputs(ch, rig, joint, B, parents, False, 5)
        p0x = params[:, :7 * ch.num_joints] if joint else params[:, :ch.num_params]
        p = tpos._emu_forward(emu, rig, joint, params, parents, off)
        gp, go = tpos._emu_backward(emu, rig, joint, params, parents, off, G)
        q = tpos._emu_forward(emu, ch, joint, p0x, parents[:n0], off[:n0])
        gq, goq = tpos._emu_backward(emu, ch, joint, p0x, parents[:n0], off[:n0], G[:, :n0])
        assert np.array_equal(p[:, :n0], q) and np.array_equal(gp[:, :p0x.shape[1]], gq) and np.array_equal(go[:n0], goq)
        p64, gp64, go64 = tpos._reference(rig, joint, params, parents, off, G)
        assert tpos._ratio(p, p64).max() <= tpos.K_POS and tpos._ratio(gp, gp64).max() <= tpos.K_GRAD
        assert tpos._offset_ratio(go, go64, False).max() <= tpos.K_OFF
    else:
        for kind, instanced in IG_BLOCKS[:2]:
            P0, P = _ig_problems(ch, rig, kind, B, instanced, 7)
            g, g0 = tig._emu(emu, rig, P), tig._emu(emu, ch, P0)
            nc0 = len(P0["parents"])
            assert all(np.array_equal(a[:, :nc0], b) for a, b in zip(g, g0))
            assert tig._bound_ratio(g, tig._closed_form64(rig, P)).max() <= tig.K_BOUND


def _positions_inputs(ch, rig, joint, B, parents, batched, seed):
    rng = np.random.default_rng(seed)
    N = parents.size
    params = tjp._joint_params(rig, B, seed).reshape(B, -1).astype(np.float32) if joint else rng.uniform(-0.5, 0.5, (B, rig.num_params)).astype(np.float32)
    off = rng.normal(scale=0.3, size=(B, N, 3) if batched else (N, 3)).astype(np.float32)
    return params, off, rng.normal(size=(B, N, 3)).astype(np.float32)


def _ig_problems(ch, rig, kind, B, instanced, seed):
    """the fixture's block P0 (tig._problem) and the rig's P: P0's constraints, then four on ballast joints; P0's parameters first"""
    P0 = tig._problem(ch, kind, B, seed, instanced)
    J0, n0 = ch.num_joints, ch.num_params
    if rig is ch:
        return P0, P0
    rng = np.random.default_rng(seed + 1)
    extra = rng.integers(J0, rig.num_joints, 4).astype(np.int32)
    k = 3 if kind == 0 else 4
    more = lambda a, shape: np.concatenate([a, shape], 1)
    P = dict(P0, parents=np.concatenate([P0["parents"], extra]),
             theta=more(P0["theta"], rng.uniform(-0.5, 0.5, (B, rig.num_params - n0)).astype(np.float32)),
             v=more(P0["v"], rng.normal(size=(B, rig.num_params - n0)).astype(np.float32)),
             enabled=np.concatenate([P0["enabled"], rng.random(rig.num_params - n0) < 0.8]),
             cw=more(P0["cw"], rng.uniform(0.5, 2.0, (B, 4)).astype(np.float32)))
    if kind == 0:
        off = rng.uniform(-0.5, 0.5, (B if instanced else 1, 4, 3)).astype(np.float32)
        P["off"] = more(P0["off"], np.broadcast_to(off, (B, 4, 3)))
        P["tgt"] = more(P0["tgt"], rng.normal(size=(B, 4, 3)).astype(np.float32))
    else:
        P["off"] = more(P0["off"], np.broadcast_to(tig._unit(rng.normal(size=(B if instanced else 1, 4, 4))), (B, 4, 4)))
        P["tgt"] = more(P0["tgt"], tig._unit(rng.normal(size=(B, 4, 4))))
    P["off"] = np.ascontiguousarray(P["off"])
    assert P["off"].shape[-1] == k
    return P0, P


# ---- GPU --------------------------------------------------------------------------------------------------------------------------------
def _device_figures():
    props = torch.cuda.get_device_properties(0)
    return int(props.shared_memory_per_block_optin), int(props.multi_processor_count)


def _census(op, backward, W, staged):
    if op == "input_gradients":
        return f"inputGradientKernel<{W}>"
    kernel = "positionsKernel" if "positions" in op else "skeletonStateKernel"
    return f"{kernel}<{str(backward).lower()}, {W}, {str(_joint(op)).lower()}" + (f", {str(bool(staged)).lower()}>" if "positions" in op else ">")


def _check_launch(L, rig, op, backward, B, N, q, variant, shape):
    """the query against the emulated rule on this device's figures, and the variant and launch shape the case is for"""
    smem, sms = _device_figures()
    p = _plan(L, rig, op, backward, B, N, smem, sms)
    assert {k: q[k] for k in ("warps", "groups", "threads", "smem", "staged")} == p, (q, p)
    fit, W = VARIANTS[variant]
    assert q["warps"] == W, (variant, q)
    if shape == "spread":
        assert q["groups"] == 1 and q["grid"] == B
    else:
        assert q["groups"] == fit and B > 3 * q["grid"] * q["groups"], (variant, B, q)
    REPORT["census"].add(_census(op, backward, W, q["staged"]))


def _batches(query):
    """the two launch shapes: a batch of one instance group per CTA, and three full waves plus a remainder (the grid of a batch
    large enough that the persistent CTAs loop)"""
    B = 4 * _device_figures()[1]
    while True:
        full = query(B)
        if full["grid"] * full["groups"] < B:
            return {"spread": 7, "waves": 3 * full["grid"] * full["groups"] + 37}
        B *= 4


def _note(variant, op, worst):
    d = REPORT["worst"][variant]
    d[op] = max(d.get(op, 0.0), float(worst))
    assert worst <= 1.0, (variant, op, worst)


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=_case_id)
def test_device_variant(emu, case):
    from momentum_b200 import torch_skeleton as tsk

    op, backward, staged, variant = case
    name, ch, rig, K, parents, n0 = rig_for(emu, op, backward, variant, staged, start=CASES.index(case))
    REPORT["cases"].append((_case_id(case), name, K))
    if op == "input_gradients":
        return _input_gradient_case(emu, ch, rig, variant, CASES.index(case))
    dc, dc0 = ms.DeviceCharacter(rig, 0), ms.DeviceCharacter(ch, 0)
    N = parents.size
    for shape, B in _batches(lambda b: dc.get_instance_launch(op, backward, b, N)).items():
        q = dc.get_instance_launch(op, backward, B, N)
        _check_launch(emu, rig, op, backward, B, N, q, variant, shape)
        sample = [0, B // 2, B - 1]
        if "skeleton_state" in op:
            x, G = _inputs(ch, op, B, 11 + B, rig)
            x0 = x[:, :7 * ch.num_joints] if _joint(op) else x[:, :ch.num_params]
            f = getattr(tsk, op)

            def run(c, xx, GG):
                xt = torch.from_numpy(xx).cuda().requires_grad_(backward)
                out = f(c, xt)
                if not backward:
                    return out.detach()
                out.backward(torch.from_numpy(GG).cuda())
                return xt.grad

            out, out0 = run(dc, x, G), run(dc0, x0, np.ascontiguousarray(G[:, :ch.num_joints]))
            orig = out[:, :ch.num_joints] if not backward else out[:, :x0.shape[1]]
            assert torch.equal(orig, out0), (variant, shape)
            for b in (0, B - 1):
                assert torch.equal(run(dc, x[b:b + 1], G[b:b + 1]), out[b:b + 1]), (variant, shape, b)
            o = out[sample].cpu().numpy()
            _note(variant, op + (" bwd" if backward else ""), _skeleton_bounds(rig, op, backward, x[sample], G[sample], o).max())
        else:
            joint = _joint(op)
            params, off, G = _positions_inputs(ch, rig, joint, B, parents, False, 13 + B)
            p0x = np.ascontiguousarray(params[:, :7 * ch.num_joints] if joint else params[:, :ch.num_params])
            fwd = getattr(tsk, op)

            def run(c, xx, par, oo, GG):
                xt = torch.from_numpy(np.ascontiguousarray(xx)).cuda().requires_grad_(backward)
                ot = torch.from_numpy(np.ascontiguousarray(oo)).cuda().requires_grad_(backward)
                p = fwd(c, xt, par, ot)
                if not backward:
                    return (p.detach(),)
                p.backward(torch.from_numpy(np.ascontiguousarray(GG)).cuda())
                return xt.grad, ot.grad

            out = run(dc, params, parents, off, G)
            out0 = run(dc0, p0x, parents[:n0], off[:n0], G[:, :n0])
            if backward:
                assert torch.equal(out[0][:, :p0x.shape[1]], out0[0]) and torch.equal(out[1][:n0], out0[1]), (variant, shape)
                for b in (0, B - 1):
                    assert torch.equal(run(dc, params[b:b + 1], parents, off, G[b:b + 1])[0], out[0][b:b + 1]), (variant, shape, b)
            else:
                assert torch.equal(out[0][:, :n0], out0[0]), (variant, shape)
                for b in (0, B - 1):
                    assert torch.equal(run(dc, params[b:b + 1], parents, off, None)[0], out[0][b:b + 1]), (variant, shape, b)
            p64, gp64, _ = tpos._reference(rig, joint, params[sample], parents, off, G[sample])
            if backward:
                _note(variant, op + " bwd", tpos._ratio(out[0][sample].cpu().numpy(), gp64).max() / tpos.K_GRAD)
            else:
                _note(variant, op, tpos._ratio(out[0][sample].cpu().numpy(), p64).max() / tpos.K_POS)


def _input_gradient_case(L, ch, rig, variant, seed):
    kind, instanced = IG_BLOCKS[list(VARIANTS).index(variant)]
    k = 3 if kind == 0 else 4
    sizes = _batches(lambda b: _ig_launch(rig, b))
    for shape, B in sizes.items():
        P0, P = _ig_problems(ch, rig, kind, B, instanced, seed)
        fn = tig._dev_function(rig, P)
        q = fn.get_input_gradient_launch()
        _check_launch(L, rig, "input_gradients", False, B, 0, q, variant, shape)
        g = tig._dev_grads(fn, P["theta"], P["v"], k)
        g0 = tig._dev_grads(tig._dev_function(ch, P0), P0["theta"], P0["v"], k)
        nc0 = len(P0["parents"])
        assert all(torch.equal(a[:, :nc0], b) for a, b in zip(g, g0)), (variant, shape)
        for b in (0, B - 1):
            one = tig._dev_grads(tig._dev_function(rig, P, sl=slice(b, b + 1)), P["theta"][b:b + 1], P["v"][b:b + 1], k)
            assert all(torch.equal(a, o[b:b + 1]) for a, o in zip(one, g)), (variant, shape, b)
        sample = [0, B // 2, B - 1]
        Q = dict(P, **{key: P[key][sample] for key in ("theta", "v", "cw", "off", "tgt")})
        worst = tig._bound_ratio([o[sample].cpu().numpy() for o in g], tig._closed_form64(rig, Q)).max() / tig.K_BOUND
        _note(variant, f"input_gradients kind={kind} instanced={instanced}", worst)


def _ig_launch(rig, B):
    """the input-gradient launch of a B-instance function on rig (a Position block on joint 0)"""
    ef = mc.PositionErrorFunction(np.array([0], np.int32), np.zeros((1, 3), np.float32), np.ones(1, np.float32), np.zeros((B, 1, 3), np.float32))
    return ms.SkeletonSolverFunction(rig, B, [ef], device=0).get_input_gradient_launch()


def _too_large():
    """chain3 with a ballast whose single instance does not fit (4000 joints: 17 floats of joint state alone per joint)"""
    return ballast(FIXTURES["chain3"](), 4000)


@pytest.mark.gpu
def test_device_refuses_an_instance_that_does_not_fit():
    """Every per-instance entry refuses the rig with an error before any launch; the torch wrappers raise; the output stays as it was,
    and the handle and the stream still work."""
    from momentum_b200 import torch_skeleton as tsk

    rig = _too_large()
    dc = ms.DeviceCharacter(rig, 0)
    B, J, n = 2, rig.num_joints, rig.num_params
    th = torch.zeros(B, n, device="cuda")
    jp = torch.zeros(B, 7 * J, device="cuda")
    par = np.array([0, J - 1], np.int32)
    off = torch.zeros(2, 3, device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    for op in ms.INSTANCE_OPS:
        for backward in (False, True):
            with pytest.raises(ms.MomentumB200Error, match="invalid configuration"):
                dc.get_instance_launch(op, backward, B, 2)
            x = jp if _joint(op) else th
            if "skeleton_state" in op:
                out = torch.full((B, J * 8) if not backward else x.shape, 7.0, device="cuda")
                g = torch.zeros(B, J, 8, device="cuda")
                args = (x.data_ptr(), out.data_ptr()) if not backward else (x.data_ptr(), g.data_ptr(), out.data_ptr())
                with pytest.raises(ms.MomentumB200Error, match="invalid configuration"):
                    dc.joint_op_device(op, backward, B, *args, stream=s)
            else:
                out = torch.full((B, 2, 3) if not backward else x.shape, 7.0, device="cuda")
                with pytest.raises(ms.MomentumB200Error, match="invalid configuration"):
                    if backward:
                        dc.positions_backward_device(_joint(op), B, x.data_ptr(), par, off.data_ptr(), False, torch.ones(B, 2, 3, device="cuda").data_ptr(),
                                                     out.data_ptr(), 0, stream=s)
                    else:
                        dc.positions_device(_joint(op), B, x.data_ptr(), par, off.data_ptr(), False, out.data_ptr(), stream=s)
            torch.cuda.synchronize()
            assert bool((out == 7.0).all()), (op, backward)
    with pytest.raises(ms.MomentumB200Error):
        tsk.model_parameters_to_skeleton_state(dc, th)
    with pytest.raises(ms.MomentumB200Error):
        tsk.joint_parameters_to_positions(dc, jp, par, off)
    xg = th.clone().requires_grad_(True)
    with pytest.raises(ms.MomentumB200Error):
        tsk.model_parameters_to_positions(dc, xg, par, off)
    # the input gradients of a solver function on the rig
    P = dict(kind=0, parents=np.array([J - 1], np.int32), theta=np.zeros((B, n), np.float32), v=np.ones((B, n), np.float32),
             enabled=np.ones(n, bool), cw=np.ones((B, 1), np.float32), off=np.zeros((B, 1, 3), np.float32), tgt=np.zeros((B, 1, 3), np.float32),
             ew=1.0, c=1.0, instanced=False)
    fn = tig._dev_function(rig, P)
    with pytest.raises(ms.MomentumB200Error, match="invalid configuration"):
        fn.get_input_gradient_launch()
    with pytest.raises(ms.MomentumB200Error, match="invalid configuration"):
        tig._dev_grads(fn, P["theta"], P["v"], 3)
    # the handle and the stream still work: a flat operation on the same handle, then a small rig on the same stream
    import scipy.sparse

    x = np.random.default_rng(3).uniform(-0.5, 0.5, (B, n)).astype(np.float32)
    out = torch.empty(B, 7 * J, device="cuda")
    dc.joint_op_device("apply_parameter_transform", False, B, torch.from_numpy(x).cuda().data_ptr(), out.data_ptr(), stream=s)
    P = scipy.sparse.csr_matrix((rig.pt_vals.astype(np.float64), rig.pt_inner, rig.pt_outer), shape=(7 * J, n))
    ref = (P @ x.astype(np.float64).T).T + rig.pt_offsets
    assert np.abs(out.cpu().numpy() - ref).max() <= 1e-5
    small = FIXTURES["chain6"]()
    x, _ = _inputs(small, "model_parameters_to_skeleton_state", 3, 4)
    st = tsk.model_parameters_to_skeleton_state(small, torch.from_numpy(x).cuda())
    assert _skeleton_bounds(small, "model_parameters_to_skeleton_state", False, x, None, st.cpu().numpy()).max() <= 1.0


@pytest.mark.gpu
def test_zz_report_instance_launch_variants():
    """The worst k (error over the pinned bound) per variant and operation, and the census of the 52 kernel instantiations reached."""
    print("\n[instance launch] worst k per variant:")
    for variant in VARIANTS:
        for op, k in sorted(REPORT["worst"][variant].items()):
            print(f"    {variant:7s} {op:52s} {k:.3f}")
    print("[instance launch] cases:", ", ".join(f"{c} ({name}+{K})" for c, name, K in REPORT["cases"]))
    expected = {_census(op, bwd, W, st) for op in ms.INSTANCE_OPS for bwd in (False, True) for W in (1, 2, 4, 8)
                for st in ((False, True) if "positions" in op else (False,))} | {_census("input_gradients", False, W, 0) for W in (1, 2, 4, 8)}
    assert len(expected) == 52
    print(f"[instance launch] {len(REPORT['census'] & expected)} of {len(expected)} instantiations reached:")
    for name in sorted(expected):
        print(f"    {'reached' if name in REPORT['census'] else 'MISSING'}  {name}")
    assert REPORT["census"] == expected
