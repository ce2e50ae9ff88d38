"""The QR step (qrSolveKernel, ik_qr.cuh) and the trust-region QR iteration (trustRegionQrKernel, ik_tr_qr.cuh) against float64 at their
width, chunk, zero-pivot and decision edges.

CPU (no device needed):
* the planner restated: qrSmemFloats, qrMaxChunkRows, trQrSmemFloats and the chunk loop of chooseSolvePath, checked against the path the
  CPU emulator plans at H100 SXM limits for every fixture below, so that each fixture is shown to sit on the edge it is named for;
* a float32 restatement of the online Householder fold and the triangular solve meets the QR backward-error bound on the fixtures, and
  four broken variants of it miss the bound by more than 100x: the bound is tight enough to catch what the GPU cases are there for;
* a float64 replay of the trust-region iteration from the double oracle's Jacobian shows that every accept / reject and damping decision
  the GPU cases rely on clears its threshold by a stated margin (a decision near its threshold may go either way in float).

GPU: one step from theta0 = 0 on each fixture. Every case asserts the path it ran (get_solve_path, fused profile), so that a change of
a launch rule fails here instead of silently dropping coverage, and prints its k (backward error over the bound without the K)."""
import dataclasses

import numpy as np
import pytest

from momentum_b200 import character as mc
from momentum_b200 import solver as ms
from momentum_b200.problems import humanoid_problem
from tests import emu_lib
from tests import f64ref as R
from tests.emu_lib import EMU_LIB

H100_SXM = (132, 227 * 1024, 228 * 1024)  # SMs, opt-in shared memory per block, shared memory per SM
QR_SMEM = 200 * 1024  # what chooseSolvePath gives R, y, x, g, the norms and the Jacobian chunk of the QR step
TR_SMEM = 220 * 1024  # ... and the trust-region kernel's R, damping rows and getError scratch
JOINT_STATE_STRIDE = 17  # kJointStateStride
FLT_EPSILON = 2.0 ** -23
MAX_RADIUS = 10.0  # the trust-region kernel's maxRadius (trust_region_qr.h:73)


# ------------------------------------------------------------------------------------------------------------------------------
# The planner, restated
# ------------------------------------------------------------------------------------------------------------------------------
def _r4(v):
    return (v + 3) & ~3


def qr_smem_floats(n, rows):
    return _r4(n * (n + 1) // 2) + 3 * _r4(n) + ((n + 4) & ~3) + (n + 1) * (rows | 1) + 8


def qr_max_chunk_rows(n, smem=QR_SMEM):
    """The most rows of a Jacobian chunk that fit beside R (even, at most 128); 0 when fewer than 8 fit."""
    fixed = qr_smem_floats(n, 0) - (n + 1)
    floats = smem // 4
    if floats <= fixed + (n + 1) * 9:
        return 0
    return min((floats - fixed) // (n + 1) - 1, 128) & ~1


def tr_qr_smem_floats(n, num_params, num_joints, rows):
    packed = _r4(n * (n + 1) // 2)
    chunk = _r4((n + 1) * (rows | 1))
    return packed + max(packed, chunk) + 7 * _r4(n) + ((n + 4) & ~3) + 2 * _r4(num_params) + _r4(num_joints * JOINT_STATE_STRIDE) + 64


def block_rows(ch, efs):
    """Jacobian rows of every block with a positive weight (jacobianBlockSize), in row order."""
    out = []
    for e in efs:
        if not e.weight > 0:
            continue
        if e.kind == mc.KIND_POSITION:
            out.append(3 * len(e.parents))
        elif e.kind in (mc.KIND_ORIENTATION, mc.KIND_ORIENTATION_ROTDIFF):
            out.append(9 * len(e.parents))
        elif e.kind == mc.KIND_PLANE:
            out.append(len(e.parents))
        elif e.kind == mc.KIND_MODEL_PARAMETERS:
            out.append(int(np.count_nonzero(np.asarray(e.target_weights) > 0)))
        else:
            raise ValueError(e.kind)
    return out


@dataclasses.dataclass
class QrPlan:
    rows: int           # qr_max_chunk_rows: 0 when refused
    chunks: list        # [(first row, rows)] in fold order
    refusal: str = None

    @property
    def widest(self):
        return max([p for _, p in self.chunks], default=1)


def plan_qr(ch, efs, ns, trust=False):
    """chooseSolvePath's QR branch: one chunk per block, split every ``rows`` rows."""
    rows = qr_max_chunk_rows(ns)
    if rows < 8:
        return QrPlan(0, [], "the QR step keeps R in shared memory")
    if trust:
        rows = min(rows, max(8, ns // 2))
        if tr_qr_smem_floats(ns, ch.num_params, ch.num_joints, rows) * 4 > TR_SMEM:
            return QrPlan(0, [], "the trust-region QR kernel keeps R and the damping rows in shared memory")
    chunks, r0 = [], 0
    for size in block_rows(ch, efs):
        chunks += [(r0 + done, min(rows, size - done)) for done in range(0, size, rows)]
        r0 += size
    return QrPlan(rows, chunks)


# ------------------------------------------------------------------------------------------------------------------------------
# Fixtures
# ------------------------------------------------------------------------------------------------------------------------------
def _chain(n, positions=24, planes=0):
    """chain_case's rig and constraint layout with the constraint points a chain's length away from their joints: every column then
    has Jacobian entries of the size of the largest (the lever arms of a deep joint and of the root differ by the chain's length at
    most, not by orders of magnitude), so that an error in the columns past 256 shows in the normwise bound."""
    J = n - 7
    rng = np.random.default_rng(n + 7 * positions + planes)
    ch = mc.create_test_character(J)
    pose = rng.uniform(-0.1, 0.1, (1, n))
    efs = []
    if positions:
        par = np.round(np.linspace(J - 1, 0, positions)).astype(np.int32)
        off = J * rng.uniform(-1, 1, (positions, 3))
        tg = mc.world_points(ch, pose, par, off) + 0.05 * rng.normal(size=(1, positions, 3))
        efs.append(mc.PositionErrorFunction(par, off, rng.uniform(0.5, 1.5, positions), tg, weight=1.0))
    if planes:
        par = np.round(np.linspace(0, J - 1, planes)).astype(np.int32)
        off = J * rng.uniform(-1, 1, (planes, 3))
        nrm = rng.normal(size=(1, planes, 3))
        unit = nrm / np.linalg.norm(nrm, axis=-1, keepdims=True)
        d = np.sum(unit * mc.world_points(ch, pose, par, off), -1) + 0.2 * rng.normal(size=(1, planes))
        efs.append(mc.PlaneErrorFunction(par, off, rng.uniform(0.5, 1.5, planes), np.concatenate([nrm, d[..., None]], -1), above=False, weight=1.0))
    return ch, efs


def _rooted_chain(n, K, seed):
    """createTestCharacter(n - 7) with one Position constraint on each of the joints 0 .. K - 1 and none below: 3K rows for the K + 7
    parameters of those joints (well determined), and the parameters of joints K .. n - 8 touched by no row."""
    J = n - 7
    rng = np.random.default_rng(seed)
    ch = mc.create_test_character(J)
    pose = rng.uniform(-0.1, 0.1, (1, n))
    joints = np.arange(K, dtype=np.int32)
    off = rng.uniform(-1, 1, (K, 3))
    tg = mc.world_points(ch, pose, joints, off) + 0.05 * rng.normal(size=(1, K, 3))
    return ch, [mc.PositionErrorFunction(joints, off, rng.uniform(0.5, 1.5, K), tg, weight=1.0)]


def _every_joint(ch, pose):
    """A Position and an Orientation constraint on every joint at ``pose`` (the reference's SanityCheck set): well determined."""
    J = ch.num_joints
    joints = np.arange(J, dtype=np.int32)
    ident = np.tile([0.0, 0.0, 0.0, 1.0], (J, 1))
    return [mc.PositionErrorFunction(joints, np.zeros((J, 3)), np.ones(J), mc.world_points(ch, pose, joints, np.zeros((J, 3))), weight=1.0),
            mc.OrientationErrorFunction(joints, ident, np.ones(J), mc.world_rotations(ch, pose, joints, ident), weight=1.0)]


def _subset_306():
    en = np.ones(306, bool)
    en[[3, 100, 250, 262, 280, 301]] = False  # compact column 256 is parameter 259: three disabled columns on each side
    return en


# name: (builder of (character, error functions), enabled parameters or None, the edge: a check of the restated plan, its description)
QR_CASES = {
    "n255": (lambda: _chain(255), None, lambda P, ns: ns == 255 and P.rows == 66 and [p for _, p in P.chunks] == [66, 6], "n = 255: one column per thread"),
    "n256": (lambda: _chain(256), None, lambda P, ns: ns == 256 and P.rows == 66, "n = 256: every thread owns one column"),
    "n257": (lambda: _chain(257), None, lambda P, ns: ns == 257 and P.rows == 64 and [p for _, p in P.chunks] == [64, 8], "n = 257: thread 0 takes columns 0 and 256"),
    "n288": (lambda: _chain(288), None, lambda P, ns: ns == 288 and P.rows == 28 and [p for _, p in P.chunks] == [28, 28, 16],
             "n = 288: the block split in three"),
    "n306": (lambda: _chain(306), None, lambda P, ns: ns == 306 and P.rows == 8 and [p for _, p in P.chunks] == [8] * 9,
             "n = 306: rows = 8, the minimum"),
    "n306_subset": (lambda: _chain(306), _subset_306(),
                    lambda P, ns: ns == 300 and P.rows == 14 and [p for _, p in P.chunks] == [14] * 5 + [2],
                    "306 parameters, 300 enabled: disabled columns on both sides of compact column 256"),
    "rows_exact": (lambda: _chain(255, positions=22), None, lambda P, ns: P.rows == 66 and [p for _, p in P.chunks] == [66],
                   "a block of exactly rows rows: one chunk"),
    "rows_plus_one": (lambda: _chain(255, positions=0, planes=67), None, lambda P, ns: P.rows == 66 and [p for _, p in P.chunks] == [66, 1],
                      "a block of rows + 1 rows: a second chunk of 1 row"),
    "odd_and_one_row_plane": (lambda: _chain(257, positions=11, planes=1), None,
                              lambda P, ns: P.rows == 64 and [p for _, p in P.chunks] == [33, 1],
                              "an odd-row block (p = ps = 33) and a 1-row Plane block"),
    "cap_128": (lambda: _chain(200, positions=50), None, lambda P, ns: ns == 200 and P.rows == 128 and [p for _, p in P.chunks] == [128, 22],
                "n = 200, a 150-row block: the 128-row cap"),
}
# lambda = 0, a well-determined step on the joints 0 .. K - 1 and enabled parameters no row touches: name: (n, K)
ZERO_CASES = {"zero_cols_n100": (100, 40), "zero_cols_n280": (280, 260)}
# the trust-region fixtures, well determined; radius: not reached / binding, both shown by the replay
TR_FIXTURES = {"humanoid": dict(free=10.0, binding=0.3), "chain223": dict(free=10.0, binding=0.3)}
# the trust-region iteration whose first trust step is rejected: a 13-parameter chain with a Position constraint on every joint (18 rows,
# well determined) towards a pose up to 1 radian away. The first trust step, damped from |x| 3.57 to the radius 3, overshoots (rho -0.34);
# the radius is quartered and the second trust step, starting from the damping R kept, is damped further and taken (rho 0.95).
REJECT_RADIUS = 3.0
# the trust-region iteration that takes no step: the humanoid constraints at the pose theta0 = 0 itself (g.x is far below its threshold)


def qr_fixture(name):
    """(character, error functions, enabled or None, lambda-free) of a QR-step fixture."""
    if name in ZERO_CASES:
        n, K = ZERO_CASES[name]
        ch, efs = _rooted_chain(n, K, seed=n)
        return ch, efs, None
    build, en, _, _ = QR_CASES[name]
    ch, efs = build()
    return ch, efs, en


def tr_fixture(name):
    if name == "reject_first":
        rng = np.random.default_rng(1)
        ch = mc.create_test_character(6)
        pose = rng.uniform(-1.0, 1.0, (1, ch.num_params))
        joints = np.arange(6, dtype=np.int32)
        off = rng.uniform(-1, 1, (6, 3))
        return ch, [mc.PositionErrorFunction(joints, off, np.ones(6), mc.world_points(ch, pose, joints, off), weight=1.0)]
    if name in ("humanoid", "at_solution"):
        ch, _, _, ts = humanoid_problem(1, orientation=True)
        return ch, _every_joint(ch, 0.3 * ts if name == "humanoid" else 0.0 * ts)
    n = int(name[5:])
    ch = mc.create_test_character(n - 7)
    return ch, _every_joint(ch, np.random.default_rng(n).uniform(-0.1, 0.1, (1, n)))


@pytest.fixture(scope="module")
def emu():
    emu_lib.build()
    return ms.load_library(EMU_LIB)


def _emu_fn(ch, efs, en):
    fn = ms.SkeletonSolverFunction(ch, 1, efs, lib_path=EMU_LIB)
    fn.upload_targets()
    if en is not None:
        fn.set_enabled_parameters(en)
    return fn


def _emu_path(emu, ch, efs, en, linear_solver, radius=1.0):
    """(record, error message) of the emulator's choice at H100 SXM limits"""
    emu.emu_set_device_limits(*H100_SXM)
    fn = _emu_fn(ch, efs, en)
    solver = ms.GaussNewtonSolver(_opts(linear_solver=linear_solver, trust_region_radius=radius), fn)
    if emu.emu_choose_solve_path(solver._h) != 0:
        return solver.get_solve_path(), emu.mb2_last_error().decode()
    return solver.get_solve_path(), None


def _opts(**kw):
    base = dict(min_iterations=1, max_iterations=1, threshold=1.0, regularization=0.05, fused_mode=ms.FUSED_OFF)
    base.update(kw)
    return ms.GaussNewtonSolverOptions(**base)


def _ns(ch, en):
    return ch.num_params if en is None else int(np.count_nonzero(en))


def _path_matches(rec, plan, kind):
    return (rec["kind"] == kind and rec["qr_max_chunk_rows"] == plan.rows and rec["qr_chunks"] == len(plan.chunks)
            and rec["qr_widest_chunk"] == plan.widest)


# ------------------------------------------------------------------------------------------------------------------------------
# CPU 1: the restated planner against the emulator's plan
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(QR_CASES) + list(ZERO_CASES))
def test_qr_fixture_sits_on_its_edge(name, emu):
    ch, efs, en = qr_fixture(name)
    ns = _ns(ch, en)
    plan = plan_qr(ch, efs, ns)
    if name in QR_CASES:
        assert QR_CASES[name][2](plan, ns), (name, QR_CASES[name][3], plan)
    rec, err = _emu_path(emu, ch, efs, en, ms.LINEAR_SOLVER_QR)
    assert err is None and _path_matches(rec, plan, "qr"), (name, rec, plan)


@pytest.mark.parametrize("name", list(TR_FIXTURES) + ["reject_first", "at_solution"])
def test_trust_region_fixture_path(name, emu):
    ch, efs = tr_fixture(name)
    plan = plan_qr(ch, efs, ch.num_params, trust=True)
    rec, err = _emu_path(emu, ch, efs, None, ms.LINEAR_SOLVER_TRUST_REGION_QR)
    assert err is None and _path_matches(rec, plan, "trust_region_qr"), (name, rec, plan)
    assert rec["tr_r_floats"] == _r4(ch.num_params * (ch.num_params + 1) // 2)
    if name == "chain223":  # the widest chain the trust-region kernel takes
        assert plan_qr(*_chain(224), 224, trust=True).refusal is not None


def test_planner_refuses_past_the_width_limits(emu):
    ch, efs = _chain(307)
    assert qr_max_chunk_rows(306) == 8 and qr_max_chunk_rows(307) == 0
    rec, err = _emu_path(emu, ch, efs, None, ms.LINEAR_SOLVER_QR)
    assert plan_qr(ch, efs, 307).refusal in err and rec["kind"] is None, err
    ch, efs = _chain(224)
    assert plan_qr(ch, efs, 224).refusal is None
    rec, err = _emu_path(emu, ch, efs, None, ms.LINEAR_SOLVER_TRUST_REGION_QR)
    assert plan_qr(ch, efs, 224, trust=True).refusal in err and rec["kind"] is None, err


# ------------------------------------------------------------------------------------------------------------------------------
# CPU 2: the bound against a float32 restatement of the fold and its broken variants
# ------------------------------------------------------------------------------------------------------------------------------
def qr_step32(A, b, chunks, diag0, mutant=None, chunk=0):
    """x with R x = y after folding [diag0 I; A | 0; b] chunk by chunk, in float32 as qrFoldJacobian and qrSolveUpperWarp do it.
    ``mutant`` breaks chunk ``chunk``: "no_fill" skips every column that is zero in the chunk even where R has entries, "drop_256"
    leaves the columns >= 256 out of it; "divide" makes the triangular solve divide 0 by a zero pivot."""
    f32 = np.float32
    n = A.shape[1]
    Rm = np.zeros((n, n + 1), f32)  # row i: R(i, i..n-1), then y(i)
    Rm[np.arange(n), np.arange(n)] = f32(diag0)
    for c, (r0, p) in enumerate(chunks):
        C = np.concatenate([A[r0:r0 + p], b[r0:r0 + p, None]], axis=1).astype(f32)
        if mutant == "drop_256" and c == chunk:
            C[:, 256:n] = 0
        norms = np.einsum("kj,kj->j", C, C)
        for i in range(n):
            sigma = norms[i]
            if sigma == 0:
                continue
            x1 = Rm[i, i]
            mu = np.sqrt(x1 * x1 + sigma)
            v1 = (x1 - mu) if x1 <= 0 else (-sigma / (x1 + mu))
            beta = f32(2) * v1 * v1 / (sigma + v1 * v1)
            inv = f32(1) / v1
            u = C[:, i]
            rr = Rm[i, i + 1:]
            keep = (norms[i + 1:] != 0) | (rr != 0)
            if mutant == "no_fill" and c == chunk:
                keep = norms[i + 1:] != 0
            s = np.where(keep, (rr + (u @ C[:, i + 1:]) * inv) * beta, f32(0)).astype(f32)
            Rm[i, i + 1:] = rr - s
            C[:, i + 1:] -= np.outer(u, s * inv)
            norms[i + 1:] = np.where(keep, np.einsum("kj,kj->j", C[:, i + 1:], C[:, i + 1:]), norms[i + 1:])
            Rm[i, i] = mu
    x = np.zeros(n, f32)
    with np.errstate(divide="ignore", invalid="ignore"):
        for i in range(n - 1, -1, -1):
            num, d = Rm[i, n] - Rm[i, i + 1:n] @ x[i + 1:], Rm[i, i]
            x[i] = f32(0) if (d == 0 and num == 0 and mutant != "divide") else num / d
    return x


def _cpu_step(name):
    """(J, r, cols, lambda, chunks, touched) of a fixture at theta0 = 0 from the emulator's float Jacobian."""
    ch, efs, en = qr_fixture(name)
    fn = _emu_fn(ch, efs, en)
    J, r = R.jacobian64(fn, np.zeros((1, ch.num_params)))
    cols = np.arange(ch.num_params) if en is None else np.nonzero(en)[0]
    plan = plan_qr(ch, efs, len(cols))
    Jc = J[0][:, cols]
    lam = 0.0 if name in ZERO_CASES else float(np.float32(max(0.05, 1e-5 * float(np.max(np.sum(Jc ** 2, axis=0))))))
    touched = np.any(Jc != 0, axis=0)
    return J[0], r[0], cols, lam, plan.chunks, touched


def _be(J, r, cols, x, lam, touched=None):
    t = np.ones(len(cols), bool) if touched is None else touched
    return R.backward_error(J, r, cols[t], np.asarray(x, np.float64)[t], lam)


CPU_WORST = {}


@pytest.mark.parametrize("name", ["n257", "n306", "n306_subset", "rows_plus_one", "odd_and_one_row_plane", "zero_cols_n280"])
def test_restated_fold_meets_the_qr_bound(name):
    J, r, cols, lam, chunks, touched = _cpu_step(name)
    x = qr_step32(J[:, cols], r, chunks, np.sqrt(np.float32(lam)))
    lim = R.solve_limit(len(cols), "qr")
    be = _be(J, r, cols, x, lam, touched if name in ZERO_CASES else None)
    k = be / lim * R.SOLVE_K["qr"]
    CPU_WORST[name] = k
    print(f"\n[restated fold {name}] n={len(cols)} chunks={len(chunks)} lambda={lam:.3e} backward error {be:.3e} limit {lim:.3e} k {k:.5f}")
    assert be <= lim
    if name in ZERO_CASES:
        assert not touched.all() and np.all(x[~touched] == 0)


def test_bound_rejects_the_broken_folds():
    """Each broken variant misses the bound by more than 100x (a NaN or Inf step misses it too)."""
    J, r, cols, lam, chunks, _ = _cpu_step("n306")
    A, d0, lim = J[:, cols], np.sqrt(np.float32(lam)), R.solve_limit(len(cols), "qr")
    assert len(chunks) == 9
    good = qr_step32(A, r, chunks, d0)
    out = {"no_fill": _be(J, r, cols, qr_step32(A, r, chunks, d0, "no_fill", chunk=2), lam),
           "drop_256": _be(J, r, cols, qr_step32(A, r, chunks, d0, "drop_256", chunk=1), lam)}
    lo, hi = np.arange(256), np.arange(256, len(cols))
    i, j = lo[np.argmax(good[lo])], hi[np.argmin(good[hi])]
    sw = good.copy(); sw[[i, j]] = sw[[j, i]]
    out["swap_across_256"] = _be(J, r, cols, sw, lam)
    J0, r0, cols0, _, chunks0, touched = _cpu_step("zero_cols_n280")
    x = qr_step32(J0[:, cols0], r0, chunks0, 0.0, "divide")
    out["divide_zero_pivot"] = _be(J0, r0, cols0, x, 0.0, touched) if np.all(np.isfinite(x)) else np.inf
    print(f"\n[broken folds] limit {lim:.3e}: " + ", ".join(f"{k} {v:.3e}" for k, v in out.items()))
    assert all(not v <= 100 * lim for v in out.values()), out


# ------------------------------------------------------------------------------------------------------------------------------
# CPU 3: the trust-region iteration replayed in float64
# ------------------------------------------------------------------------------------------------------------------------------
# How far from its threshold every decision of the replay must be: float rounding of the kernel (its J, its solves, its in-kernel
# getError) moves these quantities by far less, so the kernel takes the branch the replay takes.
MARGIN = {"xn": 0.01,       # |xn / (1.05 radius) - 1|
          "ql2": 2.0,       # ql2 / FLT_EPSILON outside [1/2, 2]
          "dlambda": 0.01,  # |(|p| - radius) / radius|: the sign of deltaLambda
          "gx": 2.0,        # g.x / (FLT_EPSILON (1 + e)) outside [1/2, 2]
          "rho": 0.05}      # |rho - t| for t = 0, 0.25, 0.75


@dataclasses.dataclass
class TrustStep:
    decisions: list   # (name, value, threshold)
    x: np.ndarray     # the step of the last trust step tried
    mu: float         # its damping: (J^T J + mu I) x = J^T r
    rho: float
    accepted: bool


def _qr_solves(J, mu):
    """x -> R^-1 x and x -> R^-T x for the R of [J; sqrt(mu) I] (float64 QR, as the kernel folds it: R^T R = J^T J + mu I)."""
    from scipy.linalg import solve_triangular

    Rm = np.linalg.qr(np.vstack([J, np.sqrt(mu) * np.eye(J.shape[1])]), mode="r")
    return (lambda v: solve_triangular(Rm, v)), (lambda v: solve_triangular(Rm, v, trans="T"))


def tr_replay(J, r, e, radius, error_at):
    """doIteration of trustRegionQrKernel in float64 from J [rows, n], r and the error e at theta0: the trust steps it tries, and the
    radius after it. ``error_at(x)``: the error at theta0 - x. The solves go through a QR of [J; sqrt(mu) I] like the kernel's (the
    normal equations of an under-determined J are indefinite in float64 at the kernel's 1e-20 damping)."""
    gJ = J.T @ r
    g = 2.0 * gJ
    mu, lam, steps = 1e-20, 1e-10, []  # mu: the damping R carries (the 1e-10 diagonal squared + the Newton increments)
    for _ in range(10):
        dec = []
        solve, solve_t = _qr_solves(J, mu)
        x = solve(solve_t(gJ))
        xg = float(x @ g)
        dec.append(("gx", xg, FLT_EPSILON * (1.0 + e)))
        if xg < FLT_EPSILON * (1.0 + e):
            steps.append(TrustStep(dec, x, mu, np.nan, False))
            break
        for _ in range(3):
            xn = float(np.linalg.norm(x))
            dec.append(("xn", xn, 1.05 * radius))
            if xn < 1.05 * radius:
                break
            q = solve_t(x)
            pl2, ql2 = xn * xn, float(q @ q)
            dec.append(("ql2", ql2, FLT_EPSILON))
            if ql2 < FLT_EPSILON:
                break
            dec.append(("dlambda", (xn - radius) / radius, 0.0))
            d = (pl2 / ql2) * ((xn - radius) / radius)
            if d <= 0:
                break
            lam, mu = lam + d, mu + d
            solve, solve_t = _qr_solves(J, mu)
            x = solve(solve_t(gJ))
        Jx = J @ x
        model = e - float(g @ x) + float(Jx @ Jx) + 1e-20 * float(x @ x)
        rho = (e - error_at(x)) / (e - model)
        dec.append(("rho", rho, (0.0, 0.25, 0.75)))
        if rho < 0.25:
            radius = 0.25 * radius
        elif rho > 0.75 and lam > 0:
            radius = min(2.0 * radius, MAX_RADIUS)
        steps.append(TrustStep(dec, x, mu, rho, rho > 0))
        if rho > 0:
            break
    return steps, radius


def margin_failures(steps):
    bad = []
    for s in steps:
        for name, v, t in s.decisions:
            if name == "rho":
                ok = all(abs(v - tt) >= MARGIN["rho"] for tt in t)
            elif name in ("ql2", "gx"):
                ok = not (t / MARGIN[name] <= v <= t * MARGIN[name])
            elif name == "xn":
                ok = abs(v / t - 1.0) >= MARGIN["xn"]
            else:
                ok = abs(v - t) >= MARGIN[name]
            if not ok:
                bad.append((name, v, t))
    return bad


def _oracle_replay(name, radius, iterations=1):
    """The replay from the double oracle at theta0 = 0 (float32-rounded inputs), iterations chained through the radius while every
    trust step is rejected. Returns the trust steps of every iteration and the final radius."""
    from oracle.binding import OracleFunction

    ch, efs = tr_fixture(name)
    ch, efs = R.rounded_inputs(ch, efs)
    orc = OracleFunction(ch, efs, "float64")
    th0 = np.zeros(ch.num_params)
    e, J, r, _ = orc.get_jacobian(th0)
    out = []
    for _ in range(iterations):
        steps, radius = tr_replay(J, r, e, radius, lambda x: orc.get_error(th0 - x))
        out.append(steps)
        if steps[-1].accepted:
            break
    return out, radius


@pytest.mark.parametrize("name", list(TR_FIXTURES))
@pytest.mark.parametrize("regime", ["free", "binding"])
def test_trust_region_replay_clears_its_thresholds(name, regime):
    (steps,), _ = _oracle_replay(name, TR_FIXTURES[name][regime])
    s = steps[0]
    print(f"\n[trust-region replay {name} {regime}] " + "; ".join(f"{d[0]} {d[1]:.4g}" for d in s.decisions) + f"; mu {s.mu:.3e}")
    assert not margin_failures(steps), margin_failures(steps)
    assert len(steps) == 1 and s.accepted  # the first trust step is taken
    names = [d[0] for d in s.decisions]
    if regime == "free":  # the radius is not reached: no damping
        assert names == ["gx", "xn", "rho"] and s.mu == 1e-20
    else:  # the radius binds: at least one damping iteration
        assert names.count("dlambda") >= 1 and s.mu > 1e-20


def test_trust_region_replay_rejects_the_first_trust_step():
    """rho of the first trust step is below 0 by the margin: the parameters are kept, the radius is quartered, R keeps its damping and
    the next trust step is damped to the smaller radius and taken."""
    (steps,), _ = _oracle_replay("reject_first", REJECT_RADIUS)
    print("\n[trust-region replay, rejection] " + " | ".join("; ".join(f"{d[0]} {d[1]:.4g}" for d in t.decisions) for t in steps))
    assert not margin_failures(steps), margin_failures(steps)
    assert len(steps) == 2 and steps[0].rho <= -MARGIN["rho"] and steps[1].accepted
    assert 1e-20 < steps[0].mu < steps[1].mu  # the rejected step was damped already, and the damping grows from there
    assert np.linalg.norm(steps[1].x) < 0.5 * np.linalg.norm(steps[0].x)


def test_trust_region_replay_takes_no_step_at_the_solution():
    """At the pose its targets come from, g.x is below FLT_EPSILON (1 + e) by far: the iteration stops before any trust step.

    (The under-determined cfg3 set is not used here: its float64 replay accepts the first trust step, rho = 0.48 at theta0 = 0, so
    the rejections the float kernel makes there come from rounding, not from a decision with a margin.)"""
    its, radius = _oracle_replay("at_solution", 1.0, 3)
    for steps in its:
        assert [d[0] for d in steps[0].decisions] == ["gx"] and not steps[0].accepted
        assert not margin_failures(steps), margin_failures(steps)
    assert len(its) == 3 and radius == 1.0
    print(f"\n[at the solution] g.x {its[0][0].decisions[0][1]:.3e} threshold {its[0][0].decisions[0][2]:.3e}")


# ------------------------------------------------------------------------------------------------------------------------------
# GPU: the kernels
# ------------------------------------------------------------------------------------------------------------------------------
GPU_WORST = {}


def _gpu_fn(ch, efs, B=1, en=None):
    fn = ms.SkeletonSolverFunction(ch, B, efs)
    fn.upload_targets()
    if en is not None:
        fn.set_enabled_parameters(en)
    return fn


def _k(family, label, be, n, folds=1):
    """The limit of a step whose R folded ``folds`` blocks of rows by Householder reflectors (the Jacobian, then each damping block of
    the trust-region search): the backward errors of successive orthogonal folds add up, so the limit is ``folds`` times one fold's.
    k is reported per fold."""
    lim = folds * R.solve_limit(n, "qr")
    k = be / lim * R.SOLVE_K["qr"]
    GPU_WORST[family] = max(GPU_WORST.get(family, 0.0), k)
    print(f"\n[{family}: {label}] n={n} folds={folds} backward error {be:.3e} limit {lim:.3e} k {k:.5f}")
    return lim


def _check_qr_path(solver, plan, kind="qr"):
    rec = solver.get_solve_path()
    assert _path_matches(rec, plan, kind), (rec, plan)
    assert solver.get_fused_profile()["fused"] == 0
    return rec


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(QR_CASES))
def test_qr_step_backward_error_at_its_edges(name):
    ch, efs, en = qr_fixture(name)
    th0 = np.zeros((1, ch.num_params))
    solver, out, J, r, cols, delta, lam = R.one_step(ch, efs, th0, _opts(linear_solver=ms.LINEAR_SOLVER_QR), enabled=en, rel_damping=1e-5)
    assert np.all(out["status"] == 0), out["status"]
    plan = plan_qr(ch, efs, len(cols))
    assert QR_CASES[name][2](plan, len(cols))
    _check_qr_path(solver, plan)
    be = R.backward_error(J[0], r[0], cols, delta[0], lam)
    assert be <= _k("qr step", f"{name} chunks {[p for _, p in plan.chunks]}", be, len(cols))


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(ZERO_CASES))
def test_qr_step_with_zero_damping_and_untouched_columns(name):
    """lambda = 0: R starts as 0 I. The columns no row touches keep a zero row of R (the sigma == 0 skip) and come out exactly 0 (the
    0 / 0 -> 0 rule of the triangular solve); the rest of the step solves the undamped normal equations."""
    n, K = ZERO_CASES[name]
    ch, efs, _ = qr_fixture(name)
    th0 = np.zeros((1, n))
    solver, out, J, r, cols, delta, lam = R.one_step(ch, efs, th0, _opts(linear_solver=ms.LINEAR_SOLVER_QR, regularization=0.0))
    assert lam == 0.0 and np.all(out["status"] == 0)
    _check_qr_path(solver, plan_qr(ch, efs, n))
    touched = np.any(J[0] != 0, axis=0)
    assert int(touched.sum()) == K + 7 and np.all(np.isfinite(out["params"]))
    assert np.all(out["params"][0][~touched] == 0), out["params"][0][~touched]
    be = R.backward_error(J[0], r[0], cols[touched], delta[0][touched], 0.0)
    assert be <= _k("qr step, lambda = 0", name, be, K + 7)


@pytest.mark.gpu
def test_qr_and_trust_region_refuse_past_their_width():
    for n, kind, msg in [(307, ms.LINEAR_SOLVER_QR, "the QR step keeps R in shared memory"),
                         (224, ms.LINEAR_SOLVER_TRUST_REGION_QR, "the trust-region QR kernel keeps R")]:
        ch, efs = _chain(n)
        solver = ms.GaussNewtonSolver(_opts(linear_solver=kind), _gpu_fn(ch, efs))
        with pytest.raises(ms.MomentumB200Error, match=msg):
            solver.solve(np.zeros((1, n), np.float32))
        assert solver.get_solve_path()["kind"] is None


def _slice(efs, idx):
    """The error functions of the instances ``idx`` (per-instance targets only; everything else is shared)."""
    out = []
    for e in efs:
        t = getattr(e, "targets", None)
        out.append(type(e)(**{**e.__dict__, "targets": np.asarray(t)[idx]}) if t is not None and np.ndim(t) >= 2 else e)
    return out


@pytest.mark.gpu
def test_qr_batch_past_256_columns_is_bitwise_per_instance():
    """300 instances of the 288-parameter chain (more CTAs than SMs), starting at, near and far from their solutions so that they stop
    at different iterations: later iterations skip the instances that are done. Every instance solved alone matches bit for bit."""
    B, n = 300, 288
    ch, efs, ts = R.chain_case(n, positions=24, B=B, seed=B)
    rng = np.random.default_rng(13)
    scale = rng.choice([0.0, 0.002, 0.05, 1.0], size=B)
    theta0 = (ts * (1.0 - scale[:, None]) + rng.normal(size=ts.shape) * 0.01 * (scale[:, None] > 0)).astype(np.float32)
    fn = _gpu_fn(ch, efs, B)
    J, _ = R.jacobian64(fn, theta0)
    lam = max(0.05, 1e-5 * float(np.max(np.sum(J ** 2, axis=1))))
    opts = ms.GaussNewtonSolverOptions(min_iterations=1, max_iterations=10, threshold=1e6, regularization=lam, linear_solver=ms.LINEAR_SOLVER_QR,
                                       fused_mode=ms.FUSED_OFF)
    solver = ms.GaussNewtonSolver(opts, fn)
    full = solver.solve(theta0)
    plan = plan_qr(ch, efs, n)
    assert plan.rows == 28 and len(plan.chunks) == 3
    _check_qr_path(solver, plan)
    assert np.all(full["status"] == 0) and len(np.unique(full["iterations"])) >= 3, np.unique(full["iterations"], return_counts=True)
    for b in range(B):
        one = ms.GaussNewtonSolver(opts, _gpu_fn(ch, _slice(efs, [b]), 1)).solve(theta0[b:b + 1])
        assert np.array_equal(one["params"][0], full["params"][b]), b
        assert one["errors"][0] == full["errors"][b] and one["iterations"][0] == full["iterations"][b] and one["status"][0] == full["status"][b]


def _tr_one_iteration(name, radius, iterations=1):
    """One trust-region iteration (or several) from theta0 = 0 on the device: (solver, out, J, r, e, fn) with the device's float J."""
    ch, efs = tr_fixture(name)
    fn = _gpu_fn(ch, efs)
    th0 = np.zeros((1, ch.num_params), np.float32)
    J, r = R.jacobian64(fn, th0)
    e = float(fn.get_error(th0)[0])
    opts = _opts(linear_solver=ms.LINEAR_SOLVER_TRUST_REGION_QR, trust_region_radius=radius, min_iterations=iterations, max_iterations=iterations,
                 store_error_history=True)
    solver = ms.GaussNewtonSolver(opts, fn)
    out = solver.solve(th0)
    rec = _check_qr_path(solver, plan_qr(ch, efs, ch.num_params, trust=True), "trust_region_qr")
    assert rec["tr_r_floats"] == _r4(ch.num_params * (ch.num_params + 1) // 2)
    return solver, out, J[0], r[0], e, fn


def _device_replay(J, r, e, radius, fn, trust_steps=1):
    """The replay from the device's own float J and error: its decisions clear their margins too. Returns its trust steps."""
    n = J.shape[1]
    steps, _ = tr_replay(J, r, e, radius, lambda x: float(fn.get_error(-x[None, :].astype(np.float32))[0]))
    assert not margin_failures(steps), margin_failures(steps)
    assert len(steps) == trust_steps and steps[-1].accepted and steps[-1].x.shape == (n,)
    return steps


def _check_damped_step(family, name, J, r, out, s, steps):
    """The device's accepted step x (theta0 = 0) against the replay's accepted trust step s: x solves (J^T J + lambda I) x = J^T r for
    the lambda recovered from x itself, lambda > 0, and |x| is the replay's to within a heuristic tolerance. R then holds the Jacobian
    and one diagonal block per damping increment of the replay's trust steps (``steps``; R keeps them across a rejection): the limit is
    the QR bound times the number of those folds.

    The tolerance, 10 kappa beta with beta the QR bound and kappa = cond(J^T J + mu I) at the replay's final damping mu: a float solve
    at that damping has a relative forward error of at most kappa beta; each of the at most three Newton updates of the damping is a
    product and quotient of |p|^2, |q|^2 and |p| - radius (about 3 kappa beta each, 9 for mu), |x(mu)| has a logarithmic derivative in
    [-1, 0] with respect to mu, and the last solve adds its own kappa beta. It is a heuristic, not a bound: the solves that set the
    earlier Newton updates run at smaller dampings, where kappa is larger (at the first one, cond(J^T J), 10 kappa beta exceeds 1 on the
    fixtures here and would check nothing). Both values are printed."""
    n = J.shape[1]
    assert np.all(out["status"] == 0) and np.any(out["params"][0] != 0)  # accepted
    x = -out["params"][0].astype(np.float64)
    H, g, _, _ = R.normal_equations64(J, r, np.arange(n))
    lam_hat = float(x @ (g - H @ x) / (x @ x))
    assert lam_hat > 0, lam_hat
    be = R.backward_error(J, r, np.arange(n), x, lam_hat)
    folds = 1 + sum(1 for t in steps for d in t.decisions if d[0] == "dlambda" and d[1] > 0)
    lim = _k(family, f"{name} lambda {lam_hat:.4g} (replay {s.mu:.4g})", be, n, folds)
    assert be <= lim
    w, beta = np.linalg.eigvalsh(H), R.solve_limit(n, "qr")
    tol = 10.0 * ((w[-1] + s.mu) / (w[0] + s.mu)) * beta
    rel = abs(np.linalg.norm(x) - np.linalg.norm(s.x)) / np.linalg.norm(s.x)
    print(f"    |x| {np.linalg.norm(x):.6g} replay {np.linalg.norm(s.x):.6g}: relative difference {rel:.3e}, tolerance {tol:.3e}"
          f" (10 kappa beta at the first solve's damping: {10.0 * w[-1] / max(w[0], 1e-20) * beta:.3e})")
    assert tol < 1 and rel <= tol
    return x


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(TR_FIXTURES))
def test_trust_region_step_with_the_radius_not_reached(name):
    """The undamped step: R^T R = J^T J + 1e-20 I, accepted."""
    radius = TR_FIXTURES[name]["free"]
    solver, out, J, r, e, fn = _tr_one_iteration(name, radius)
    n = J.shape[1]
    (s,) = _device_replay(J, r, e, radius, fn)
    assert [d[0] for d in s.decisions] == ["gx", "xn", "rho"]
    assert np.all(out["status"] == 0) and np.any(out["params"][0] != 0)  # accepted
    x = -out["params"][0].astype(np.float64)
    be = R.backward_error(J, r, np.arange(n), x, 1e-20)
    assert be <= _k("trust-region step, radius not reached", name, be, n)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(TR_FIXTURES))
def test_trust_region_step_with_a_binding_radius(name):
    """The damped step, taken at the first trust step (see _check_damped_step)."""
    radius = TR_FIXTURES[name]["binding"]
    solver, out, J, r, e, fn = _tr_one_iteration(name, radius)
    steps = _device_replay(J, r, e, radius, fn)
    s = steps[-1]
    assert "dlambda" in [d[0] for d in s.decisions] and s.mu > 1e-20
    _check_damped_step("trust-region step, binding radius", name, J, r, out, s, steps)


@pytest.mark.gpu
def test_trust_region_rejects_a_step_then_takes_one_at_the_quartered_radius():
    """The first trust step (damped to the radius 3) is rejected, rho < 0 by the margin; the parameters are kept, the radius is quartered
    and R keeps its damping. The step finally taken is the replay's second trust step, damped further from there."""
    solver, out, J, r, e, fn = _tr_one_iteration("reject_first", REJECT_RADIUS)
    steps = _device_replay(J, r, e, REJECT_RADIUS, fn, trust_steps=2)
    x = _check_damped_step("trust-region step after a rejection", "reject_first", J, r, out, steps[-1], steps)
    assert np.linalg.norm(x) < 0.5 * REJECT_RADIUS


@pytest.mark.gpu
def test_trust_region_takes_no_step_at_the_solution():
    """Every iteration stops at the g.x test: the parameters stay bitwise, the error history is constant."""
    solver, out, J, r, e, fn = _tr_one_iteration("at_solution", 1.0, iterations=4)
    steps, _ = tr_replay(J, r, e, 1.0, None)
    assert [d[0] for d in steps[0].decisions] == ["gx"] and not margin_failures(steps), steps[0].decisions
    assert np.all(out["params"].view(np.uint32) == 0) and np.all(out["status"] == 0)  # bitwise theta0 = +0
    hist = solver.get_error_history()[0]
    assert np.all(hist == hist[0]), hist


def test_zz_report_qr_bounds():
    print("\n[QR backward error] worst k per family:", GPU_WORST, " pinned:", R.SOLVE_K["qr"])
