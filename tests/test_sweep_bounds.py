"""The FK + residual + Jacobian sweep (sweepKernel, K1 / K4) against the DOUBLE oracle on float32-rounded inputs, row by row
(tests/f64ref.py: rounded_inputs, sweep_reference, sweep_ratios).

CPU part: the float oracle (an independent faithful float implementation) and the lane emulator (tests/emu, the one-warp lane order)
pass the bound on every fixture, so the bound is fair and not tuned to the kernel; and each mutation of the double reference that
stands for a class of kernel bug fails it by at least 10x wherever it applies, so the bound is tight enough to matter.

GPU part (-m gpu): every fixture and every launch variant of the sweep (warps per instance, table staging, groups per CTA, small-batch
spread, several waves) through get_jacobian, get_jacobian_device, get_error, get_skeleton_state and one solver step; each case asserts
the variant it reached from get_sweep_launch, and test_zz_report_sweep_bounds prints the worst k per variant and per family."""
import dataclasses

import numpy as np
import pytest

from momentum_b200 import character as mc
from momentum_b200 import solver as ms
from momentum_b200.problems import chain_problem, humanoid_problem, random_unit_quats, small_rotation_quats
from tests import emu_lib
from tests import f64ref as R


@dataclasses.dataclass
class Fixture:
    name: str
    family: str
    ch: object
    efs: list
    theta: np.ndarray                       # [B, n] float32
    enabled: object = None
    instance_weights: dict = dataclasses.field(default_factory=dict)  # block index -> [B, nc] per-instance constraint weights

    def efs_of(self, b):
        """The blocks as instance b sees them (per-instance constraint weights folded into the shared weights)."""
        out = list(self.efs)
        for i, w in self.instance_weights.items():
            out[i] = dataclasses.replace(out[i], weights=np.asarray(w)[b].astype(np.float64))
        return out


def _rounded(name, family, ch, efs, theta, **kw):
    ch, efs = R.rounded_inputs(ch, efs)
    iw = {i: np.asarray(w, np.float32).astype(np.float64) for i, w in kw.pop("instance_weights", {}).items()}
    return Fixture(name, family, ch, efs, np.asarray(theta, np.float32), instance_weights=iw, **kw)


def _two_roots():
    """Two test-character chains side by side, each with its own root (6 DOF + scale): parameters 0-6 and 7-13 drive the two roots."""
    J = 10
    parents = np.array([-1, 0, 1, 2, 3, -1, 5, 6, 7, 8], np.int32)
    offsets = np.zeros((J, 3), np.float32)
    offsets[[1, 2, 3, 4, 6, 7, 8, 9], 1] = 1.0
    offsets[5] = (3.0, 0.0, 0.5)
    prerot = np.zeros((J, 4), np.float32); prerot[:, 3] = 1.0
    trip = [(k, k, 1.0) for k in range(7)] + [(35 + k, 7 + k, 1.0) for k in range(7)]
    p = 14
    for j in (1, 2, 3, 4, 6, 7, 8, 9):
        trip += [(7 * j + 3, p, 1.0), (7 * j + 5, p + 1, 1.0)]
        p += 2
    outer, inner, vals = mc._csr_from_triplets(7 * J, p, trip)
    return mc.Character(parents, offsets, prerot, p, outer, inner, vals, np.zeros(7 * J, np.float32), [], "two_roots")


def _position_block(ch, rng, theta_star, parents, weight=1.0, noise=0.05, **kw):
    off = rng.uniform(-1, 1, (len(parents), 3))
    w = rng.uniform(0.5, 1.5, len(parents))
    tg = mc.world_points(ch, theta_star, parents, off) + noise * rng.normal(size=(theta_star.shape[0], len(parents), 3))
    return mc.PositionErrorFunction(np.asarray(parents, np.int32), off, w, tg, weight=weight, **kw)


def random_rig(J, seed, three_dof_every=4):
    """A J-joint chain with side branches (every 7th joint hangs off its grandparent), random offsets (length 0.3 - 1.2) and
    pre-rotations (up to 30 degrees), a 6-DOF + scale root, three rotation DOFs on joints 1 - 5 and on every ``three_dof_every``-th
    joint, one (rx) elsewhere; and the limit set of momentum_b200.problems.add_test_limits (MinMax, MinMaxJoint + passive, Linear,
    LinearJoint, HalfPlane, Ellipsoid). Unlike createTestCharacter, no two joints share an offset or a pre-rotation, so a table read off
    by one joint moves the result."""
    from momentum_b200.problems import add_test_limits

    rng = np.random.default_rng(seed)
    parents = np.array([-1] + [j - 2 if j % 7 == 0 and j >= 2 else j - 1 for j in range(1, J)], np.int32)
    d = rng.normal(size=(J, 3))
    offsets = (d / np.linalg.norm(d, axis=1, keepdims=True) * rng.uniform(0.3, 1.2, (J, 1))).astype(np.float32)
    offsets[0] = 0.0
    prerot = np.stack([[0, 0, 0, 1.0]] + [mc._random_prerot(rng) for _ in range(1, J)]).astype(np.float32)
    trip = [(k, k, 1.0) for k in range(7)]
    p = 7
    for j in range(1, J):
        for dof in ((3, 4, 5) if j <= 5 or j % three_dof_every == 0 else (3,)):
            trip.append((7 * j + dof, p, 1.0))
            p += 1
    outer, inner, vals = mc._csr_from_triplets(7 * J, p, trip)
    ch = mc.Character(parents, offsets, prerot, p, outer, inner, vals, np.zeros(7 * J, np.float32), [], f"rig{J}")
    return add_test_limits(ch, rng)


def _variant_fixture(J, P, B=2, seed=0):
    """random_rig(J) with P Position constraints spread over the joints (weights 1 and 1e-4 alternating: rows of two magnitudes in
    one matrix), an Orientation block on three joints, a State block on four joints and the limits."""
    ch = random_rig(J, seed)
    rng = np.random.default_rng(seed + 1)
    n = ch.num_params
    ts = rng.uniform(-0.25, 0.25, (B, n))
    par = np.round(np.linspace(J - 1, 1, P)).astype(np.int32)
    pos = _position_block(ch, rng, ts, par, noise=0.1)
    pos.weights = np.where(np.arange(P) % 2 == 0, 1.0, 1e-4)
    oj = np.array([J - 1, J // 2, 3], np.int32)
    ooff = random_unit_quats(rng, (3,))
    ori = mc.OrientationErrorFunction(oj, ooff, np.array([1.0, 0.5, 2.0]), mc._qmul(mc.world_rotations(ch, ts, oj, ooff), small_rotation_quats(rng, (B, 3), 0.3)),
                                      weight=0.4)
    t, q, sc = mc.forward_kinematics(ch, ts)
    pw, rw = np.zeros(J), np.zeros(J)
    sj = np.array([2, J // 3, (2 * J) // 3, J - 2])
    pw[sj], rw[sj] = rng.uniform(0.5, 1.5, 4), rng.uniform(0.5, 1.5, 4)
    st = mc.StateErrorFunction(pw, rw, np.concatenate([t + 0.05 * rng.normal(size=t.shape), mc._qmul(q, small_rotation_quats(rng, (B, J), 0.3)), sc[..., None]], -1),
                               weight=0.7, pos_wgt=1.5, rot_wgt=0.8)
    theta = ts + rng.uniform(-0.05, 0.05, ts.shape)
    return _rounded(f"rig{J}_p{P}", "variant", ch, [pos, ori, st, mc.LimitErrorFunction(weight=0.5)], theta)


def cpu_fixtures():
    """Every family the sweep evaluates, each with small- and large-magnitude rows in one matrix, and the edges where float kernels go
    wrong. Small enough for the double oracle and the lane emulator."""
    F = []
    # Position: a shared block with a zero-weight constraint, an instanced block (offsets per instance) with per-instance weights, a
    # legacy-weight block (rows 1e-2 of the others)
    ch, efs, theta0, ts = chain_problem(J=8, B=3, seed=101, families=("position",))
    rng = np.random.default_rng(101)
    par = np.array([7, 5, 2, 6], np.int32)
    ioff = rng.uniform(-1, 1, (3, 4, 3))
    tg = np.stack([mc.world_points(ch, ts[b:b + 1], par, ioff[b])[0] for b in range(3)]) + 0.05 * rng.normal(size=(3, 4, 3))
    inst = mc.PositionErrorFunction(par, np.zeros((4, 3)), np.ones(4), tg, weight=1.0, instance_offsets=ioff)
    legacy = _position_block(ch, rng, ts, [3, 7], weight=mc.PositionErrorFunction.kLegacyWeight)
    iw = rng.uniform(0.2, 2.0, (3, 4)); iw[1, 2] = 0.0
    F.append(_rounded("position", "position", ch, efs + [inst, legacy], theta0, instance_weights={1: iw}))
    # Orientation: matrix and rot-diff forms, instanced offsets on one of them, next to a legacy-weight position block
    for rot_diff in (False, True):
        ch, efs, theta0, ts = chain_problem(J=7, B=2, seed=102 + rot_diff, families=("orientation",), rot_diff=rot_diff)
        rng = np.random.default_rng(110 + rot_diff)
        par = np.array([6, 3], np.int32)
        ioff = random_unit_quats(rng, (2, 2))
        tg = np.stack([mc._qmul(mc.world_rotations(ch, ts[b:b + 1], par, ioff[b])[0], small_rotation_quats(rng, (2,), 0.4)) for b in range(2)])
        inst = mc.OrientationErrorFunction(par, np.tile([0, 0, 0, 1.0], (2, 1)), np.array([0.7, 1.3]), tg, weight=0.5, rot_diff=rot_diff, instance_offsets=ioff)
        legacy = _position_block(ch, rng, ts, [6], weight=mc.PositionErrorFunction.kLegacyWeight)
        F.append(_rounded("orientation_rotdiff" if rot_diff else "orientation", "orientation", ch, efs + [inst, legacy], theta0))
    # State, both rotation error types
    for logmap in (False, True):
        ch, efs, theta0, _ = chain_problem(J=7, B=2, seed=104 + logmap, families=("state", "position"), logmap=logmap)
        F.append(_rounded("state_logmap" if logmap else "state_matrix", "state", ch, efs, theta0))
    # every limit type (MinMax, MinMaxJoint (+ passive), Linear, LinearJoint, HalfPlane, Ellipsoid) next to positions
    ch, efs, theta0, _ = chain_problem(J=8, B=2, seed=106, families=("limit", "position"))
    F.append(_rounded("limits", "limit", ch, efs, 1.5 * theta0))
    # Plane, both modes, points on both sides
    ch, efs, theta0, _ = chain_problem(J=7, B=3, seed=107, families=("plane", "halfplane", "position"))
    F.append(_rounded("planes", "plane", ch, efs, theta0))
    # ModelParameters with negative target weights (error-only units)
    ch, efs, theta0, _ = chain_problem(J=6, B=2, seed=108, families=("model_parameters", "position"))
    tw = np.asarray(efs[-1].target_weights, np.float64).copy(); tw[[0, 3, 7]] = [-0.7, -1.2, -0.4]
    efs[-1] = dataclasses.replace(efs[-1], target_weights=tw)
    F.append(_rounded("model_parameters", "model_parameters", ch, efs, theta0))
    # generalized losses
    for tag, alpha, c in (("l1", mc.LOSS_L1, 0.7), ("cauchy", mc.LOSS_CAUCHY, 1.3), ("welsch", mc.LOSS_WELSCH, 0.9), ("alpha-2", -2.0, 1.1), ("alpha1.5", 1.5, 0.8)):
        ch, efs, theta0, _ = chain_problem(J=6, B=2, seed=109, families=("position", "orientation", "limit", "plane"), loss=(alpha, c))
        F.append(_rounded(f"loss_{tag}", "loss", ch, efs, theta0))
    # an enabled subset
    ch, efs, theta0, _ = chain_problem(J=7, B=2, seed=112, families=("position", "orientation", "state", "limit", "plane"))
    en = np.ones(ch.num_params, bool); en[[0, 2, 5, 8, ch.num_params - 1]] = False
    F.append(_rounded("enabled_subset", "subset", ch, efs, theta0, enabled=en))
    # two roots
    ch = _two_roots()
    rng = np.random.default_rng(113)
    ts = rng.uniform(-0.5, 0.5, (2, ch.num_params))
    ori = mc.OrientationErrorFunction(np.array([4, 9], np.int32), random_unit_quats(rng, (2,)), np.ones(2),
                                      random_unit_quats(rng, (2, 2)), weight=0.3)
    F.append(_rounded("two_roots", "two_roots", ch, [_position_block(ch, rng, ts, [4, 9, 2, 7]), ori], rng.uniform(-0.4, 0.4, (2, ch.num_params))))
    # humanoid72 with the root and the targets 100 units out
    ch, efs, _, ts = humanoid_problem(2, seed=114, orientation=True, legacy_weights=True)
    ts[:, 0:3] += 100.0
    efs[0] = dataclasses.replace(efs[0], targets=mc.world_points(ch, ts, efs[0].parents, efs[0].offsets))
    th = ts + np.random.default_rng(114).normal(scale=0.02, size=ts.shape)
    F.append(_rounded("humanoid72_far", "humanoid", ch, efs, th))
    # a long chain: depth 299
    ch = mc.create_test_character(300)
    rng = np.random.default_rng(115)
    ts = rng.uniform(-0.3, 0.3, (1, ch.num_params))
    F.append(_rounded("chain300", "long_chain", ch, [_position_block(ch, rng, ts, [299, 150, 40], noise=0.5)], ts + rng.uniform(-0.05, 0.05, ts.shape)))
    # a random rig (random offsets and pre-rotations, 3-DOF joints, every limit type, Position / Orientation / State blocks): no two
    # joints share a table entry
    fx = _variant_fixture(12, 20, seed=150)
    F.append(dataclasses.replace(fx, name="random_rig12", family="random_rig"))
    F += edge_fixtures()
    return F


def edge_fixtures():
    """Exact zero rotation (LogMap and rot-diff), near pi, an Orientation target given as -q, an exactly zero residual, and theta exactly
    on a MinMax and a HalfPlane boundary (identity ParameterTransform rows: the comparison sees the same value in both precisions)."""
    F = []
    ch = mc.create_test_character(6)
    n, J = ch.num_params, ch.num_joints
    theta = np.zeros((2, n))
    q_id = np.tile([0.0, 0.0, 0.0, 1.0], (2, J, 1))
    t, q, s = mc.forward_kinematics(ch, theta)
    # state LogMap with target = the current orientation (identity) and, on the second instance, one joint near pi
    tg = np.concatenate([t, q_id, s[..., None]], -1)
    near_pi = np.pi - 1e-3
    tg[1, 4, 3:7] = [np.sin(near_pi / 2), 0.0, 0.0, np.cos(near_pi / 2)]
    st = mc.StateErrorFunction(np.ones(J), np.ones(J), tg, weight=0.7, rotation_error_type=mc.QUATERNION_LOG_MAP)
    rng = np.random.default_rng(120)
    off = random_unit_quats(rng, (3,))
    par = np.array([5, 2, 0], np.int32)
    cur = mc.world_rotations(ch, theta, par, off)
    tgr = cur.copy()
    tgr[1, 0] = mc._qmul(cur[1, 0], np.array([0.0, np.sin(near_pi / 2), 0.0, np.cos(near_pi / 2)]))
    rd = mc.OrientationErrorFunction(par, off, np.ones(3), tgr, weight=1.0, rot_diff=True)
    # -q targets (the same rotation): the matrix form must not care
    om = mc.OrientationErrorFunction(par, off, np.ones(3), -cur, weight=1.0)
    # zero residual: integer offsets at theta = 0 put the points exactly on their targets
    poff = np.array([[1.0, 0.0, 0.0], [0.0, 2.0, -1.0]])
    pos = mc.PositionErrorFunction(np.array([5, 3], np.int32), poff, np.ones(2), mc.world_points(ch, theta, np.array([5, 3]), poff), weight=1.0)
    F.append(_rounded("edges_zero_rotation_pi_negq", "edges", ch, [st, rd, om, pos], theta))
    # theta exactly on a MinMax boundary (parameter 0, limits +-0.1 as float) and on a HalfPlane boundary (0.5 p3 + 0.5 p5 = 0.25)
    ch = mc.create_test_character(6)
    lim = np.float32(0.1)
    ch.limits = [mc.ParameterLimit(mc.LIMIT_MINMAX, 1.0, (0,), (-0.1, 0.1)), mc.ParameterLimit(mc.LIMIT_MINMAX, 0.8, (1,), (-0.2, 0.3)),
                 mc.ParameterLimit(mc.LIMIT_HALFPLANE, 1.2, (3, 5), (0.5, 0.5, 0.25))]
    theta = np.random.default_rng(121).uniform(-0.1, 0.1, (2, ch.num_params))
    theta[0, 0], theta[1, 0] = lim, -lim
    theta[0, 1], theta[1, 1] = np.float32(0.3), np.float32(-0.2)
    theta[:, 3], theta[:, 5] = 0.25, 0.25
    rng = np.random.default_rng(122)
    F.append(_rounded("limits_on_boundary", "edges", ch, [mc.LimitErrorFunction(weight=0.5), _position_block(ch, rng, theta, [5, 2])], theta))
    return F


_CPU_FIXTURES = None


def fixtures():
    global _CPU_FIXTURES
    if _CPU_FIXTURES is None:
        _CPU_FIXTURES = cpu_fixtures()
    return _CPU_FIXTURES


def references(fx):
    """{b: SweepRef} of a fixture (per-instance weights folded in instance by instance)."""
    refs = {}
    for b in range(fx.theta.shape[0]):
        refs.update(R.sweep_reference(fx.ch, fx.efs_of(b), fx.theta, fx.enabled, instances=[b]))
    return refs


def device_function(fx, lib_path=None, B=None):
    B = fx.theta.shape[0] if B is None else B
    fn = ms.SkeletonSolverFunction(fx.ch, B, fx.efs, lib_path=lib_path)
    fn.upload_targets()
    for i, w in fx.instance_weights.items():
        fn.set_constraint_weights(i, w, per_instance=True)
    if fx.enabled is not None:
        fn.set_enabled_parameters(fx.enabled)
    return fn


def backend_ratios(fx, refs, lib_path=None, fn=None):
    """Worst k per output of the backend at ``lib_path`` (or of the handle ``fn``) over the fixture's instances: get_jacobian (K1),
    get_error and get_skeleton_state (K4)."""
    fn = fn or device_function(fx, lib_path)
    ej, J, r, _ = fn.get_jacobian(fx.theta)
    e4 = fn.get_error(fx.theta)
    st = fn.get_skeleton_state(fx.theta)
    # get_error is NOT float(get_jacobian's error) bit for bit: K4 evaluates each unit's error-only form (evalUnit<false>), which for
    # limits, the log map and the generalized losses is another float expression than the K1 form that also yields the residual, and
    # error-only units (negative ModelParameters weights) count in getError only. Both are held to their own double reference.
    worst = {}
    for b, ref in refs.items():
        ks = R.sweep_ratios(ref, J=J[b], r=r[b], e=ej[b], state=st[b], e_err=e4[b])
        for k, v in ks.items():
            worst[k] = max(worst.get(k, 0.0), v)
    return worst, fn


def oracle32_ratios(fx, refs):
    from oracle.binding import OracleFunction

    worst = {}
    for b, ref in refs.items():
        orc = OracleFunction(fx.ch, fx.efs_of(b), "float32", instance=b)
        xf, _, _ = orc.fk(fx.theta[b].astype(np.float64))
        if fx.enabled is not None:
            orc.set_enabled_parameters(fx.enabled)
        e, J, r, _ = orc.get_jacobian(fx.theta[b].astype(np.float64))
        e_err = orc.get_error(fx.theta[b].astype(np.float64))
        for k, v in R.sweep_ratios(ref, J=J, r=r, e=e, state=xf, e_err=e_err).items():
            worst[k] = max(worst.get(k, 0.0), v)
    return worst


# ------------------------------------------------------------------------------------------------------------------------------
# CPU: the bound is fair (float oracle, emulator) and tight (mutations)
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu():
    return emu_lib.build()


_CPU_NAMES = [f.name for f in fixtures()]


@pytest.mark.parametrize("name", _CPU_NAMES)
def test_float_oracle_passes_the_sweep_bound(name):
    fx = next(f for f in fixtures() if f.name == name)
    ks = oracle32_ratios(fx, references(fx))
    print(f"\n[float oracle] {name}: " + ", ".join(f"{k} {v:.3f}" for k, v in ks.items()))
    assert not R.sweep_failures(ks), (name, ks)


@pytest.mark.parametrize("name", _CPU_NAMES)
def test_emulator_passes_the_sweep_bound(name, emu):
    fx = next(f for f in fixtures() if f.name == name)
    ks, _ = backend_ratios(fx, references(fx), emu)
    print(f"\n[emulator] {name}: " + ", ".join(f"{k} {v:.3f}" for k, v in ks.items()))
    assert not R.sweep_failures(ks), (name, ks)


def branch_distances(fx):
    """Relative distance of every instance's inputs from every branch point the sweep evaluates: the MinMax / MinMaxJoint bounds, the
    range ends of a Linear / LinearJoint limit, the HalfPlane limit's and the half-plane Plane's zero. Distance |v - b| / max(1, |b|)."""
    ch = fx.ch
    out = []
    for b in range(fx.theta.shape[0]):
        th = fx.theta[b].astype(np.float64)
        rows = np.repeat(np.arange(7 * ch.num_joints), np.diff(ch.pt_outer))
        jp = np.asarray(ch.pt_offsets, np.float64).copy()
        np.add.at(jp, rows, np.asarray(ch.pt_vals, np.float64) * th[ch.pt_inner])
        lims = ch.limits if any(e.kind == mc.KIND_LIMIT and e.weight > 0 for e in fx.efs) else []
        for l in lims:
            f = np.asarray(l.f, np.float64)
            if l.type == mc.LIMIT_MINMAX:
                out += [(th[l.i[0]], f[0]), (th[l.i[0]], f[1])]
            elif l.type == mc.LIMIT_MINMAX_JOINT:
                out += [(jp[7 * l.i[0] + l.i[1]], f[0]), (jp[7 * l.i[0] + l.i[1]], f[1])]
            elif l.type in (mc.LIMIT_LINEAR, mc.LIMIT_LINEAR_JOINT) and not (f[2] == 0 and f[3] == 0):
                v = th[l.i[1]] if l.type == mc.LIMIT_LINEAR else jp[7 * l.i[2] + l.i[3]]
                out += [(v, f[2]), (v, f[3])]
            elif l.type == mc.LIMIT_HALFPLANE:
                out.append((th[l.i[0]] * f[0] + th[l.i[1]] * f[1] - f[2], 0.0))
        for e in fx.efs:
            if e.kind == mc.KIND_PLANE and e.above and e.weight > 0:
                tg = np.asarray(e.targets, np.float64)[b]
                unit = tg[:, :3] / np.linalg.norm(tg[:, :3], axis=-1, keepdims=True)
                p = mc.world_points(ch, th[None], e.parents, e.offsets)[0]
                out += [(v, 0.0) for v in np.sum(unit * p, -1) - tg[:, 3]]
    return np.array([abs(v - bp) / max(1.0, abs(bp)) for v, bp in out])


def test_fixtures_stay_away_from_branch_points():
    """Every fixture except the on-boundary one keeps its inputs at least 1e-3 relative from every limit / half-plane branch point, so
    that the float and double evaluations take the same branch and the bound compares like with like."""
    cases = [f for f in fixtures() if f.name != "limits_on_boundary"] + [_variant_fixture(*shape, seed=shape[0] + shape[1]) for shape, _ in VARIANTS]
    near = {f.name: float(branch_distances(f).min(initial=np.inf)) for f in cases}
    assert all(v >= 1e-3 for v in near.values()), {k: v for k, v in near.items() if v < 1e-3}
    # the on-boundary fixture is exactly on its MinMax and HalfPlane boundaries
    assert branch_distances(next(f for f in fixtures() if f.name == "limits_on_boundary")).min() == 0.0


def _jr_excess(ref, J, r):
    """How far a mutated (J, r) is beyond the bound: the larger of k_J / K_J and k_r / K_r (structural zeros included)."""
    try:
        ks = R.sweep_ratios(ref, J=J, r=r)
    except AssertionError:
        return np.inf
    return max(ks["J"] / R.SWEEP_K["J"], ks["r"] / R.SWEEP_K["r"])


def _oracle_jr(ch, efs, theta, b, enabled):
    from oracle.binding import OracleFunction

    orc = OracleFunction(ch, efs, "float64", instance=b)
    if enabled is not None:
        orc.set_enabled_parameters(enabled)
    _, J, r, _ = orc.get_jacobian(np.asarray(theta, np.float64))
    return J, r


def _bf16(x):
    a = np.ascontiguousarray(np.asarray(x, np.float32))
    return (a.view(np.uint32) & np.uint32(0xFFFF0000)).view(np.float32)


def mutations(fx, b, ref):
    """{name: (J, r)} for every mutation that applies to instance b of the fixture."""
    ch, efs, th = fx.ch, fx.efs_of(b), fx.theta[b].astype(np.float64)
    out = {}
    # a stale / misindexed theta read: one parameter moved by 2^-10 relative to max(1, |theta_p|); of the four columns with the largest
    # entries, the one whose move shows most
    en = np.ones(ch.num_params, bool) if fx.enabled is None else np.asarray(fx.enabled, bool)
    best = None
    for p in np.argsort(-(np.abs(ref.J).max(axis=0) * en))[:4]:
        t2 = th.copy(); t2[p] += 2.0 ** -10 * max(1.0, abs(t2[p]))
        J2, r2 = _oracle_jr(ch, efs, t2, b, fx.enabled)
        if best is None or _jr_excess(ref, J2, r2) > _jr_excess(ref, *best):
            best = (J2, r2)
    out["theta_read"] = best
    # a half-precision table: the joint whose offset / pre-rotation bf16 rounding changes most
    d_off = np.abs(_bf16(ch.offsets) - ch.offsets).max(axis=1) + np.abs(_bf16(ch.prerot) - ch.prerot).max(axis=1)
    if d_off.max() > 0:
        j = int(np.argmax(d_off))
        off, pre = ch.offsets.copy(), ch.prerot.copy()
        off[j], pre[j] = _bf16(off[j]), _bf16(pre[j])
        out["bf16_table"] = _oracle_jr(dataclasses.replace(ch, offsets=off, prerot=pre), efs, th, b, fx.enabled)
    # a table read off by one joint: the offset and pre-rotation of the joint where that changes most taken from its successor
    d_next = np.abs(np.diff(ch.offsets, axis=0)).max(axis=1) + np.abs(np.diff(ch.prerot, axis=0)).max(axis=1)
    if d_next.size and d_next.max() > 0:
        j = int(np.argmax(d_next))
        off, pre = ch.offsets.copy(), ch.prerot.copy()
        off[j], pre[j] = off[j + 1], pre[j + 1]
        out["table_off_by_one"] = _oracle_jr(dataclasses.replace(ch, offsets=off, prerot=pre), efs, th, b, fx.enabled)
    # two rotation DOFs of one joint swapped: the shallowest joint with two driven rotation rows of the ParameterTransform
    for j in np.argsort(ch.depth(), kind="stable"):
        live = [k for k in (3, 4, 5) if ch.pt_outer[7 * j + k + 1] > ch.pt_outer[7 * j + k]]
        if len(live) < 2:
            continue
        rows = np.repeat(np.arange(7 * ch.num_joints), np.diff(ch.pt_outer))
        a, c = 7 * j + live[0], 7 * j + live[1]
        rows2 = np.where(rows == a, c, np.where(rows == c, a, rows))
        outer, inner, vals = mc._csr_from_triplets(7 * ch.num_joints, ch.num_params, list(zip(rows2, ch.pt_inner, ch.pt_vals)))
        J2, r2 = _oracle_jr(dataclasses.replace(ch, pt_outer=outer, pt_inner=inner, pt_vals=vals), efs, th, b, fx.enabled)
        if np.abs(J2 - ref.J).max() > 0:
            out["dof_swap"] = (J2, r2)
            break
    # the scale column without its ln2
    scale_cols = {int(c) for j in range(ch.num_joints) for c in ch.pt_inner[ch.pt_outer[7 * j + 6]:ch.pt_outer[7 * j + 7]]}
    for c in sorted(scale_cols):
        if np.abs(ref.J[:, c]).max() > 0:
            J2 = ref.J.copy(); J2[:, c] /= np.log(2.0)
            out["scale_ln2"] = (J2, ref.r)
            break
    # a generalized loss evaluated as L2
    if any(float(getattr(e, "loss_alpha", 2.0)) != mc.LOSS_L2 for e in efs):
        efs2 = [dataclasses.replace(e, loss_alpha=mc.LOSS_L2) if hasattr(e, "loss_alpha") else e for e in efs]
        out["loss_as_l2"] = _oracle_jr(ch, efs2, th, b, fx.enabled)
    # one unit's rows from the neighbouring instance's targets
    B = fx.theta.shape[0]
    if B > 1:
        for i, e in enumerate(efs):
            tg = getattr(e, "targets", None)
            if tg is None or e.kind not in (mc.KIND_POSITION, mc.KIND_PLANE, mc.KIND_ORIENTATION, mc.KIND_ORIENTATION_ROTDIFF) or not e.weight > 0:
                continue
            tg2 = np.array(tg, copy=True)
            tg2[b, 0] = tg[(b + 1) % B, 0]
            efs2 = list(efs); efs2[i] = dataclasses.replace(e, targets=tg2)
            J2, r2 = _oracle_jr(ch, efs2, th, b, fx.enabled)
            if np.abs(r2 - ref.r).max() > 0:
                out["neighbour_targets"] = (J2, r2)
                break
    return out


def test_mutations_fail_the_sweep_bound_by_10x():
    seen, fails = {}, []
    for fx in fixtures():
        refs = references(fx)
        for b, ref in refs.items():
            for name, (J, r) in mutations(fx, b, ref).items():
                x = _jr_excess(ref, J, r)
                seen.setdefault(name, []).append((fx.name, b, x))
                # (the (D + 1) factor makes the bound of a row 300 joints deep 300x looser: a 2^-10 parameter error there stays within
                # 10x of it, so the long chain only has to fail it)
                if not x >= (1.0 if name == "theta_read" and ref.D.max() > 100 else 10.0):
                    fails.append((name, fx.name, b, x))
    for name, rows in sorted(seen.items()):
        print(f"\n[mutation] {name}: applies on {len(rows)} instances, smallest excess {min(x for _, _, x in rows):.1f}x")
    assert set(seen) == {"theta_read", "bf16_table", "table_off_by_one", "dof_swap", "scale_ln2", "loss_as_l2", "neighbour_targets"}, sorted(seen)
    assert not fails, fails


# ------------------------------------------------------------------------------------------------------------------------------
# GPU: every fixture, every launch variant
# ------------------------------------------------------------------------------------------------------------------------------
REPORT = {"variant": {}, "family": {}, "launch": []}


def _note(variant, family, ks):
    for table, key in (("variant", variant), ("family", family)):
        row = REPORT[table].setdefault(key, {})
        for k, v in ks.items():
            row[k] = max(row.get(k, 0.0), v)


def _variant_key(launch, jacobian, tag=""):
    return f"{'jacobian' if jacobian else 'error-only'} W={launch['warps']} stage={launch['stage']}" + (f" {tag}" if tag else "")


def _device_jacobian(fn, theta, rows):
    """get_jacobian_device's matrix as (J [B, rows, n], r [B, rows]) float32 on the host."""
    import torch

    from momentum_b200 import torch_ik as ti

    th = torch.as_tensor(np.ascontiguousarray(theta, np.float32), device="cuda")
    ptr, ld = fn.get_jacobian_device(th.data_ptr(), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    B, n = theta.shape
    Jall = ti._device_view(ptr, (B, n + 1, ld), th.device).clone().cpu().numpy()
    return Jall[:, :n, :rows].transpose(0, 2, 1), Jall[:, n, :rows]


def run_gpu_case(fx, label, refs=None, expect=None, tag="", strip_solve=False):
    """Every sweep entry on fixture ``fx``: bounds against the double reference, get_jacobian_device bitwise equal to get_jacobian, one
    solver step on the strip path judged by its recorded objective. ``expect(launch_jacobian, launch_error)`` asserts the variant;
    ``strip_solve``: the strip path must hold the system, and the solver's sweep must launch as get_jacobian's did."""
    refs = refs if refs is not None else references(fx)
    fn = device_function(fx)
    ks, _ = backend_ratios(fx, refs, fn=fn)
    lj, le = fn.get_sweep_launch(True), fn.get_sweep_launch(False)
    _, J, r, rows = fn.get_jacobian(fx.theta)
    Jd, rd = _device_jacobian(fn, fx.theta, rows)
    assert np.array_equal(Jd, J) and np.array_equal(rd, r), f"{label}: get_jacobian_device differs from get_jacobian"
    assert fn.get_sweep_launch(True) == lj
    print(f"\n[sweep] {label}: jacobian {lj}, error-only {le}; " + ", ".join(f"{k} {v:.3f}" for k, v in ks.items()))
    if expect is not None:
        expect(lj, le)
    # one Gauss-Newton step with the sweep writing the strip layout (where the tile path holds the system): its objective is
    # getJacobian's error at theta
    opts = ms.GaussNewtonSolverOptions(min_iterations=1, max_iterations=1, regularization=0.05, fused_mode=ms.FUSED_GRAM_CHOLESKY,
                                       cholesky_mode=ms.CHOLESKY_TILES_SPARSE)
    try:
        out = ms.GaussNewtonSolver(opts, fn).solve(fx.theta)
    except ms.MomentumB200Error as err:
        assert not strip_solve, (label, err)
        assert any(m in str(err) for m in ("does not fit", "do not fit", "needs the tile")), err
        out = None
        print(f"[sweep] {label}: no strip-path solve ({err})")
    ls = None
    if out is not None:
        ls = fn.get_sweep_launch(True)
        assert ls["grid"] > 0, f"{label}: the solver's Jacobian sweep recorded nothing"
        if strip_solve:
            assert {k: ls[k] for k in ("stage", "warps", "groups", "grid")} == {k: lj[k] for k in ("stage", "warps", "groups", "grid")}, (ls, lj)
        es = max(R._error_ratio(ref, (ref.D + 1) * R.EPS24 * ref.S, float(out["errors"][b]), ref.e, ref.l2) for b, ref in refs.items())
        print(f"[sweep] {label}: solver {ls}, objective k {es:.3f}")
        ks["e"] = max(ks["e"], es)
    REPORT["launch"].append((label, fx.family, lj, le, ls))
    REPORT["strip_solves"] = REPORT.get("strip_solves", 0) + (ls is not None)
    _note(_variant_key(lj, True, tag), fx.family, {k: v for k, v in ks.items() if k in ("J", "r", "e")})
    _note(_variant_key(le, False, tag), fx.family, {k: v for k, v in ks.items() if k in ("e", "t", "q")})
    assert not R.sweep_failures(ks), (label, ks)
    return fn


@pytest.mark.gpu
@pytest.mark.parametrize("name", _CPU_NAMES)
def test_gpu_sweep_bound_fixtures(name):
    """Batches of two or three instances: the small-batch spread (one one-warp instance per CTA, every table staged), and a strip-path
    solver step that launches the same sweep. The 300-joint chain needs four warps per instance and is too large for the tile path."""
    fx = next(f for f in fixtures() if f.name == name)
    if name == "chain300":
        run_gpu_case(fx, name, expect=_expect(1, 4, (4, 6)))
        return
    B = fx.theta.shape[0]

    def spread(lj, le):
        for l in (lj, le):
            assert (l["stage"], l["warps"], l["groups"], l["grid"]) == (1, 1, 1, B), l
    run_gpu_case(fx, name, expect=spread, tag="spread", strip_solve=True)


def _expect(stage, warps, groups):
    lo, hi = groups

    def check(lj, le):
        for l in (lj, le):
            assert l["stage"] == stage and l["warps"] == warps and lo <= l["groups"] <= hi, (l, stage, warps, groups)
    return check


# (J, P) of _variant_fixture -> (table staging, W, groups per CTA); sizes from the launch rule's shared-memory arithmetic on a 227 KB
# opt-in budget (per instance: joint state 17 J floats, + 7 J staged joint parameters when W > 1, 4 floats of evaluation record per
# Position unit), checked against the launches an H100 reports
VARIANTS = [
    ((16, 600), (2, 1, (13, 15))),    # large-rig branch: fewer than 16 one-warp instances fit, 13 * 2 > 24 warps: W stays 1
    ((150, 10), (1, 2, (7, 12))),
    ((200, 100), (2, 2, (7, 12))),
    ((16, 1900), (0, 2, (7, 12))),    # the unit table alone crowds out two instances: nothing staged
    ((250, 3), (1, 4, (4, 6))),
    ((300, 200), (2, 4, (4, 6))),
    ((12, 2200), (0, 4, (4, 6))),
    ((350, 3), (1, 8, (1, 3))),
    ((600, 100), (2, 8, (1, 3))),
    ((900, 100), (0, 8, (1, 3))),
]


@pytest.mark.gpu
@pytest.mark.parametrize("shape,variant", VARIANTS, ids=[f"rig{j}_p{p}" for (j, p), _ in VARIANTS])
def test_gpu_sweep_bound_launch_variants(shape, variant):
    fx = _variant_fixture(*shape, seed=shape[0] + shape[1])
    run_gpu_case(fx, fx.name, expect=_expect(*variant), tag="large-rig" if variant[1] == 1 else "")


@pytest.mark.gpu
def test_gpu_sweep_small_batch_spread_and_waves():
    """A small batch spread over the SMs (one instance per CTA) and a batch of three waves plus a remainder: a sampled instance's J, r,
    e and state are bitwise what it gives alone (the sweep has no cross-instance reduction)."""
    import torch

    sms = torch.cuda.get_device_properties(0).multi_processor_count
    ch, efs, _, ts = humanoid_problem(1, seed=130, orientation=False)
    # fewer instances than SMs: one per CTA; at least three rounds of every persistent CTA's groups (at most 24 per CTA)
    for B, label in ((sms - 32, "small batch spread"), (3 * sms * 24 + 17, "three waves + remainder")):
        rng = np.random.default_rng(B)
        theta_star = np.repeat(ts, B, 0) + rng.normal(scale=0.1, size=(B, ch.num_params))
        theta_star[:, 0:3] = rng.uniform(-10, 10, (B, 3))
        e2 = [dataclasses.replace(efs[0], targets=mc.world_points(ch, theta_star, efs[0].parents, efs[0].offsets))]
        theta = theta_star + rng.normal(scale=0.05, size=theta_star.shape)
        fx = _rounded(f"humanoid72_B{B}", "humanoid", ch, e2, theta)
        sample = [0, B // 2, B - 1]
        refs = {}
        for b in sample:
            refs.update(R.sweep_reference(fx.ch, fx.efs, fx.theta, instances=[b]))
        fn = device_function(fx)
        ej, J, r, _ = fn.get_jacobian(fx.theta)
        e4, st = fn.get_error(fx.theta), fn.get_skeleton_state(fx.theta)
        lj = fn.get_sweep_launch(True)
        REPORT["launch"].append((label, "humanoid", lj, fn.get_sweep_launch(False), None))
        print(f"\n[sweep] {label}: B={B} {lj}")
        if "spread" in label:
            assert lj["warps"] == 1 and lj["groups"] == 1 and lj["grid"] == B, lj
        else:
            assert lj["warps"] == 1 and lj["groups"] >= 12 and B > 3 * lj["grid"] * lj["groups"], lj
        worst = {}
        for b in sample:
            ks = R.sweep_ratios(refs[b], J=J[b], r=r[b], e=ej[b], state=st[b], e_err=e4[b])
            worst = {k: max(worst.get(k, 0.0), v) for k, v in ks.items()}
            sub = _slice_fixture(fx, b)
            f1 = device_function(sub)
            ej1, J1, r1, _ = f1.get_jacobian(sub.theta)
            assert np.array_equal(J1[0], J[b]) and np.array_equal(r1[0], r[b]) and ej1[0] == ej[b], (label, b)
            assert np.array_equal(f1.get_skeleton_state(sub.theta)[0], st[b]) and f1.get_error(sub.theta)[0] == e4[b], (label, b)
        _note(_variant_key(lj, True, "spread" if "spread" in label else "waves"), "humanoid", worst)
        assert not R.sweep_failures(worst), (label, worst)


def _slice_fixture(fx, b):
    efs = []
    for e in fx.efs:
        t = getattr(e, "targets", None)
        efs.append(dataclasses.replace(e, targets=np.asarray(t)[b:b + 1]) if t is not None and np.ndim(t) >= 2 else e)
    return Fixture(fx.name, fx.family, fx.ch, efs, fx.theta[b:b + 1], fx.enabled)


def _unstaged_chain(J, driven):
    """A chain of J joints of which only the first ``driven`` carry parameters (createTestCharacter(driven) extended by fixed joints)."""
    ch = mc.create_test_character(driven)
    extra = J - driven
    parents = np.arange(-1, J - 1, dtype=np.int32)
    offsets = np.concatenate([ch.offsets, np.tile([[0.0, 1.0, 0.0]], (extra, 1))]).astype(np.float32)
    prerot = np.concatenate([ch.prerot, np.tile([[0.0, 0.0, 0.0, 1.0]], (extra, 1))]).astype(np.float32)
    outer = np.concatenate([ch.pt_outer, np.full(7 * extra, ch.pt_outer[-1])]).astype(np.int32)
    return mc.Character(parents, offsets, prerot, ch.num_params, outer, ch.pt_inner, ch.pt_vals, np.zeros(7 * J, np.float32), [], f"chain{J}")


@pytest.mark.gpu
def test_gpu_sweep_rejects_an_instance_that_does_not_fit():
    """A rig whose single instance does not fit in shared memory (2600 joints: 24 floats of joint state and parameters per joint) is
    rejected with an error by every entry that sweeps; nothing is computed."""
    ch = _unstaged_chain(2600, 2000)
    rng = np.random.default_rng(140)
    ts = rng.uniform(-0.01, 0.01, (2, ch.num_params))
    fx = _rounded("chain2600", "reject", ch, [_position_block(ch, rng, ts, [2599, 1000])], ts)
    fn = device_function(fx)
    import torch

    th = torch.as_tensor(fx.theta, device="cuda")
    out = torch.zeros_like(th)
    calls = {"get_error": lambda: fn.get_error(fx.theta), "get_jacobian": lambda: fn.get_jacobian(fx.theta),
             "get_jacobian_device": lambda: fn.get_jacobian_device(th.data_ptr()), "get_jtjr": lambda: fn.get_jtjr(fx.theta),
             "get_skeleton_state": lambda: fn.get_skeleton_state(fx.theta),
             "implicit_direction_device": lambda: fn.implicit_direction_device(th.data_ptr(), th.data_ptr(), out.data_ptr()),
             "solve": lambda: ms.GaussNewtonSolver(ms.GaussNewtonSolverOptions(min_iterations=1, max_iterations=1, fused_mode=ms.FUSED_OFF,
                                                                               cholesky_mode=ms.CHOLESKY_DENSE_EIGEN), fn).solve(fx.theta)}
    for name, call in calls.items():
        # the sweep's own shared-memory check refused it (launchSweep returns cudaErrorInvalidConfiguration, before any launch)
        with pytest.raises(ms.MomentumB200Error, match=r"launchSweep\(.*invalid configuration") as err:
            call()
        print(f"\n[reject] {name}: {err.value}")
        # reached launchSweep (the message names it) and left the all-zero record a refused configuration leaves
        assert fn.get_sweep_launch(True) == fn.get_sweep_launch(False) == {"stage": 0, "warps": 0, "groups": 0, "grid": 0, "smem": 0}
    torch.cuda.synchronize()
    assert not out.any()


@pytest.mark.gpu
def test_zz_report_sweep_bounds():
    """Worst k per variant and per family over the GPU cases of this module, and the launches they reached."""
    print("\n[sweep bounds] pinned K:", R.SWEEP_K)
    for table in ("variant", "family"):
        print(f"[sweep bounds] worst k per {table}:")
        for key, ks in sorted(REPORT[table].items()):
            print(f"    {key:32s} " + ", ".join(f"{k} {v:.3f}" for k, v in sorted(ks.items())))
    worst = {}
    for ks in REPORT["family"].values():
        worst = {k: max(worst.get(k, 0.0), v) for k, v in {**worst, **ks}.items()}
    print("[sweep bounds] worst k overall:", {k: round(v, 3) for k, v in worst.items()})
    reached = {k for k in REPORT["variant"]}
    print("[sweep bounds] variants reached:", sorted(reached))
    print(f"[sweep bounds] strip-path solver steps: {REPORT.get('strip_solves', 0)} of {len(REPORT['launch'])} cases")
    for label, fam, lj, le, ls in REPORT["launch"]:
        print(f"    {label:32s} jacobian {lj} error-only {le}" + (f" solver {ls}" if ls else ""))
