"""Float64 references for the linear-algebra kernels, built from the backend's own float Jacobian.

The Jacobian and residual come from ``SkeletonSolverFunction.get_jacobian`` (the device's float values, promoted to float64), so FK and
Jacobian rounding drop out of every comparison and what remains is the error of the kernel under test:

* JtJ / Jtr kernels: elementwise ``|H - H64| <= c * E`` with ``E = |J|^T |J|`` (``|J|^T |r|`` for Jtr), the classical bound of a
  float dot product of length m; ``c`` depends on the kernel's arithmetic (``jtj_limit``).
* linear solves: the normwise backward error of one Gauss-Newton step, ``||A d - g||inf / ((||E||inf + lambda) ||d||inf + ||g||inf)``
  with ``A = H64 + lambda I`` over the enabled parameters. A correct factorisation keeps it at a small multiple of ``n 2^-24`` whatever
  the conditioning (``solve_limit``); a wrong tile, a missed update or a permuted step moves it by orders of magnitude.

No oracle is involved in those. Every helper takes a ``lib_path`` so that the CPU emulator (tests/emu) can run the same checks.

The sweep itself (FK + residual + Jacobian + error, the kernels that produce that float Jacobian) is held to the DOUBLE oracle on
float32-rounded inputs (``rounded_inputs``, ``sweep_reference``, ``sweep_ratios``), row by row:

* Jacobian and residual: ``|J_ij - J64_ij| <= K_J (D_i + 1) 2^-24 S_i`` and ``|r_i - r64_i| <= K_R (D_i + 1) 2^-24 S_i`` with D_i the depth
  of the row's joint (1 for limit and ModelParameters rows), ``S_i = max_j |J64_ij| + |r64_i| + rho c_i + g_i``, rho the instance's world radius
  ``max(1, max |t64|)``, c_i the row's largest |J64| over the roots' translation columns (all parameters enabled) and g_i the row's
  largest |J64| at two generic poses. The rho term keeps a rig far from the origin fair (a position is rounded relative to its distance
  from the origin, not to the residual) without loosening rotational rows, whose c_i is 0; the g term keeps a row at a stationary point
  (a rotation difference at zero rotation) at the size of what it differences. Entries outside every cell the plan can hold (columns
  that drive none of the row joint's ancestors, disabled columns, padding rows) must be exactly 0.
* error: from the residual bound when every block is an L2 block with rows for all of its terms (e = sum r_i^2),
  ``|e - e64| <= K_E (sum (2 |r64_i| beta_i + beta_i^2) + m 2^-24 e64)`` with ``beta_i = (D_i + 1) 2^-24 S_i``; else (generalized
  losses, error-only units) ``K_E (Dmax + 1) 2^-24 (e64 + sum |r64_i| S_i)``.
* skeleton state: t within ``K_T (D + 1) 2^-24 rho``, q and s within ``K_Q (D + 1) 2^-24 max(1, |s64|)``."""
import dataclasses

import numpy as np

from momentum_b200 import character as mc
from momentum_b200 import solver as ms

EPS24 = 2.0 ** -24

# Limits pinned from the worst ratios measured on an H100 80GB HBM3 (700 W power limit) over the cases of
# tests/test_gpu_kernel_bounds.py, which prints them; each about 4x above the worst measured k.
K_SIMT = 3.5          # |H - H64| <= K_SIMT * m * 2^-24 * E                 worst measured k 0.85 (m = 1)
K_TF32X3 = 4.0        # |H - H64| <= K_TF32X3 * (2^-21 + m * 2^-24) * E     worst measured k 0.91 (m = 2); lo*lo dropped
K_TF32 = 8.0          # |H - H64| <= K_TF32 * 2^-11 * E                     worst measured k 1.92
# The single-TF32 product fails the 3xTF32 limit by ~90x. The SIMT limit does NOT separate SIMT from 3xTF32: both are fp32-class (the
# split's error is ~2^-21 relative, below the classical m 2^-24 dot-product bound from m = 8 rows on), so a SIMT path that ran the
# 3xTF32 arithmetic would still pass it. Only the bitwise AUTO == SIMT check of the 513-column case tells the two kernels apart.

# Backward error of one step <= K * max(n, 16) * 2^-24, one K per linear-solve path (below one 16-wide tile the JtJ rounding, 2^-21
# for the 3xTF32 split, dominates the factorisation's own error).
SOLVE_K = {
    "dense": 1.0,            # dense Eigen-structured kernel     worst measured k 0.24 (n = 1, 3xTF32 JtJ)
    "tiles": 0.06,           # tile-scheduled kernel (FUSED_OFF) worst measured k 0.0148 (bodyhands300, 3xTF32 JtJ)
    "gram_cholesky": 0.004,  # Gram + Cholesky in one launch     worst measured k 0.00101 (humanoid72)
    "persistent": 0.0045,    # persistent whole-solve kernel     worst measured k 0.00113 (humanoid72 with a disabled subset)
    "qr": 0.006,             # QR step                           worst measured k 0.00154 (humanoid72, split block)
}


def jtj_limit(mode, m):
    """Elementwise JtJ / Jtr error limit relative to E for ``m`` Jacobian rows."""
    if mode == ms.JTJ_TF32:
        return K_TF32 * 2.0 ** -11
    if mode == ms.JTJ_TF32X3:
        return K_TF32X3 * (2.0 ** -21 + m * EPS24)
    return K_SIMT * m * EPS24


def jacobian64(fn, theta):
    """(J [B, rows, n], r [B, rows]) of the backend at ``theta`` in float64; padding rows are zero."""
    _, J, r, _ = fn.get_jacobian(np.asarray(theta, np.float32))
    return J.astype(np.float64), r.astype(np.float64)


def normal_equations64(J, r, cols):
    """H64 = Jc^T Jc, g64 = Jc^T r, E = |Jc|^T |Jc|, Eg = |Jc|^T |r| for the columns ``cols`` of one instance."""
    Jc = J[:, cols]
    A = np.abs(Jc)
    return Jc.T @ Jc, Jc.T @ r, A.T @ A, A.T @ np.abs(r)


def jtj_ratios(H, g, J, r):
    """Worst |H - H64| / E over the lower triangle and |g - g64| / Eg for one instance of get_jtjr (leading block of ``H.shape[0]``
    columns). An entry whose bound E is zero (a structurally zero product) must come out exactly zero."""
    ap = H.shape[0]
    H64, g64, E, Eg = normal_equations64(J, r, np.arange(ap))
    low = np.tril(np.ones((ap, ap), bool))
    dH = np.abs(H.astype(np.float64) - H64)[low]
    dg = np.abs(g.astype(np.float64) - g64)
    eH, eg = E[low], Eg
    assert np.all(dH[eH == 0] == 0) and np.all(dg[eg == 0] == 0), "non-zero result where every product is zero"
    with np.errstate(divide="ignore", invalid="ignore"):
        rh = np.where(eH > 0, dH / np.where(eH > 0, eH, 1), 0.0)
        rg = np.where(eg > 0, dg / np.where(eg > 0, eg, 1), 0.0)
    return float(max(rh.max(initial=0.0), rg.max(initial=0.0)))


def backward_error(J, r, cols, delta, lam):
    """Normwise backward error of ``delta`` as the solution of (Jc^T Jc + lam I) delta = Jc^T r, in float64."""
    H64, g64, E, _ = normal_equations64(J, r, cols)
    A = H64 + lam * np.eye(len(cols))
    res = np.max(np.abs(A @ delta - g64))
    den = (np.max(E.sum(axis=1)) + lam) * np.max(np.abs(delta)) + np.max(np.abs(g64))
    return float(res / den) if den > 0 else 0.0


def solve_limit(n, path="dense"):
    return SOLVE_K[path] * max(n, 16) * EPS24


def one_step(ch, efs, theta0, opts, lib_path=None, enabled=None, rel_damping=None):
    """One Gauss-Newton step without line search from ``theta0`` (float32, B instances) with ``opts`` (min = max = 1 iteration).
    ``rel_damping``: raise the damping to that fraction of the largest diagonal entry of JtJ, so that the float factorisation completes
    on long chains (their JtJ spans many orders of magnitude). Returns (solver, out, J, r, cols, delta, lam): the float64 Jacobian at
    theta0, the enabled columns, the step recovered as theta0 - theta1 (exact when theta0 = 0, else to the rounding of theta1) and the
    damping the kernels used."""
    import dataclasses

    theta0 = np.asarray(theta0, np.float32)
    B = theta0.shape[0]
    fn = ms.SkeletonSolverFunction(ch, B, efs, lib_path=lib_path)
    fn.upload_targets()
    if enabled is not None:
        fn.set_enabled_parameters(enabled)
    J, r = jacobian64(fn, theta0)
    cols = np.arange(ch.num_params) if enabled is None else np.nonzero(np.asarray(enabled, bool))[0]
    assert opts.min_iterations == 1 and opts.max_iterations == 1 and not opts.do_line_search
    if rel_damping is not None:
        diag = np.max(np.sum(J[:, :, cols] ** 2, axis=1))
        opts = dataclasses.replace(opts, regularization=max(opts.regularization, rel_damping * float(diag)))
    solver = ms.GaussNewtonSolver(opts, fn)
    out = solver.solve(theta0)
    delta = theta0.astype(np.float64)[:, cols] - out["params"].astype(np.float64)[:, cols]
    return solver, out, J, r, cols, delta, float(np.float32(opts.regularization))


def chain_case(n, positions, planes=0, B=1, seed=0, spread=0.1):
    """createTestCharacter(n - 7) with ``positions`` Position constraints spread along the chain (3 rows each) and ``planes`` Plane
    constraints (1 row each): m = 3 positions + planes. Targets are reachable points of a pose within +-spread of zero."""
    J = n - 7
    assert J >= 3
    rng = np.random.default_rng(seed)
    ch = mc.create_test_character(J)
    theta_star = rng.uniform(-spread, spread, (B, n))
    efs = []
    if positions:
        par = np.round(np.linspace(J - 1, 0, positions)).astype(np.int32)
        off = rng.uniform(-1, 1, (positions, 3))
        tg = mc.world_points(ch, theta_star, par, off) + 0.05 * rng.normal(size=(B, positions, 3))
        efs.append(mc.PositionErrorFunction(par, off, rng.uniform(0.5, 1.5, positions), tg, weight=1.0))
    if planes:
        par = np.round(np.linspace(0, J - 1, planes)).astype(np.int32)
        off = rng.uniform(-1, 1, (planes, 3))
        nrm = rng.normal(size=(B, planes, 3))
        unit = nrm / np.linalg.norm(nrm, axis=-1, keepdims=True)
        d = np.sum(unit * mc.world_points(ch, theta_star, par, off), -1) + 0.2 * rng.normal(size=(B, planes))
        efs.append(mc.PlaneErrorFunction(par, off, rng.uniform(0.5, 1.5, planes), np.concatenate([nrm, d[..., None]], -1), above=False, weight=1.0))
    return ch, efs, theta_star


# ------------------------------------------------------------------------------------------------------------------------------
# The sweep (FK + residual + Jacobian + error) against the double oracle
# ------------------------------------------------------------------------------------------------------------------------------
# Limits pinned from the worst ratios measured on an H100 80GB HBM3 over the GPU cases of tests/test_sweep_bounds.py (every fixture and
# launch variant; test_zz_report_sweep_bounds prints them; the same ratios on cards at 700 W and at 400 W power limit), about 4x above
# the worst measured k, and above the float oracle's and the lane emulator's worst k on the same fixtures.
SWEEP_K = {
    "J": 12.0,   # Jacobian entries      worst measured k 2.77 (exact zero rotation, rot-diff at identity)
    "r": 24.0,   # residual              worst measured k 6.05 (350-joint random rig, W = 8, all tables staged)
    "e": 0.5,    # error                 worst measured k 0.12 (Orientation rot-diff; the alpha = -2 loss)
    "t": 3.5,    # state translation     worst measured k 0.87 (random rig with 2200 Position constraints, W = 4, nothing staged)
    "q": 7.0,    # state rotation, scale worst measured k 1.97 (humanoid72, a batch of three waves + a remainder)
}


def _round32(v):
    if isinstance(v, (bool, np.bool_)) or isinstance(v, (int, np.integer)):
        return v
    if isinstance(v, (float, np.floating)):
        return float(np.float32(v))
    if isinstance(v, np.ndarray) and v.dtype.kind == "f":
        return v.astype(np.float32).astype(np.float64)
    return v


def rounded_inputs(ch, efs):
    """(character, error functions) with every real input rounded to float32: what the device holds, so that input rounding is not
    counted as kernel error. The character's tables are float32 already; the limit weights, the block weights, loss parameters,
    constraint weights, offsets and targets are rounded here. (The device normalises uploaded quaternions and plane normals in float,
    the double oracle in double: an ulp-level input difference the bound absorbs.)"""
    ch2 = dataclasses.replace(ch, offsets=np.asarray(ch.offsets, np.float32), prerot=np.asarray(ch.prerot, np.float32),
                              pt_vals=np.asarray(ch.pt_vals, np.float32), pt_offsets=np.asarray(ch.pt_offsets, np.float32),
                              limits=[dataclasses.replace(l, weight=float(np.float32(l.weight)), f=tuple(np.asarray(l.f, np.float32).astype(float)))
                                      for l in ch.limits])
    out = []
    for e in efs:
        vals = {f.name: _round32(getattr(e, f.name)) for f in dataclasses.fields(e)}
        vals = {k: (np.asarray(v, np.float32).astype(np.float64) if isinstance(v, np.ndarray) and v.dtype.kind == "f" else v) for k, v in vals.items()}
        out.append(dataclasses.replace(e, **vals))
    return ch2, out


def row_joints(ch, efs):
    """The joint behind every Jacobian row in the reference's row order (blocks in order, a block with weight <= 0 has no rows): the
    constraint's parent, the state joint, an Ellipsoid limit's parent; -1 for the other limit rows and ModelParameters rows. Padding rows
    are not included."""
    rows = []
    for e in efs:
        if not e.weight > 0:
            continue
        k = e.kind
        if k == mc.KIND_POSITION:
            rows += [int(p) for p in e.parents for _ in range(3)]
        elif k in (mc.KIND_ORIENTATION, mc.KIND_ORIENTATION_ROTDIFF):
            rows += [int(p) for p in e.parents for _ in range(9)]
        elif k == mc.KIND_PLANE:
            rows += [int(p) for p in e.parents]
        elif k == mc.KIND_STATE:
            per = 6 if e.rotation_error_type == mc.QUATERNION_LOG_MAP else 12
            active = (np.asarray(e.pos_weights) != 0) | (np.asarray(e.rot_weights) != 0)
            rows += [int(j) for j in np.nonzero(active)[0] for _ in range(per)]
        elif k == mc.KIND_LIMIT:
            for l in ch.limits:
                if l.type == mc.LIMIT_MINMAX_JOINT_PASSIVE:
                    continue
                rows += [-1] * (3 if l.type == mc.LIMIT_ELLIPSOID else 1)
        elif k == mc.KIND_MODEL_PARAMETERS:
            rows += [-1] * int(np.count_nonzero(np.asarray(e.target_weights) > 0))
        else:
            raise ValueError(k)
    return np.asarray(rows, np.int64)


def ancestor_columns(ch):
    """[J, n] bool: model parameter c drives joint j or one of its ancestors (the cells the plan can hold for a row of joint j)."""
    J, n = ch.num_joints, ch.num_params
    own = np.zeros((J, n), bool)
    for j in range(J):
        own[j, ch.pt_inner[ch.pt_outer[7 * j]:ch.pt_outer[7 * j + 7]]] = True
    anc = own.copy()
    for j, p in enumerate(ch.parents):
        if p >= 0:
            anc[j] |= anc[p]
    return anc


def root_translation_columns(ch):
    """Model parameters that drive a root joint's translation (ParameterTransform rows 7 root + 0..2)."""
    cols = set()
    for j in np.nonzero(np.asarray(ch.parents) < 0)[0]:
        for row in range(7 * j, 7 * j + 3):
            cols.update(int(c) for c in ch.pt_inner[ch.pt_outer[row]:ch.pt_outer[row + 1]])
    return np.array(sorted(cols), np.int64)


def l2_rows_cover_error(efs):
    """True when e = sum r_i^2 holds exactly for the double reference: every block has the L2 loss and every error term has a row
    (no ModelParameters term with a negative target weight)."""
    for e in efs:
        if float(getattr(e, "loss_alpha", mc.LOSS_L2)) != mc.LOSS_L2:
            return False
        if e.kind == mc.KIND_MODEL_PARAMETERS and np.any(np.asarray(e.target_weights) < 0):
            return False
    return True


@dataclasses.dataclass
class SweepRef:
    """Double-oracle reference of one instance at float32-rounded inputs."""
    J: np.ndarray       # [rows, n]
    r: np.ndarray       # [rows]
    e: float            # getJacobian's error
    e_err: float        # getError's (error-only units count here only)
    state: np.ndarray   # [joints, 8] t, q xyzw, s
    D: np.ndarray       # [rows] joint depth of each row (padding rows: 0)
    S: np.ndarray       # [rows] row scale
    zero: np.ndarray    # [rows, n] structural zeros (must come out exactly 0)
    rho: float
    l2: bool
    jdepth: np.ndarray  # [joints]


def sweep_reference(ch, efs, theta, enabled=None, instances=None):
    """SweepRef of every instance (``instances``: a subset) of theta [B, n] (float32 values) for the rounded inputs (ch, efs)."""
    from oracle.binding import OracleFunction

    theta = np.asarray(theta, np.float32).astype(np.float64)
    B = theta.shape[0]
    tcols = root_translation_columns(ch)
    rj = row_joints(ch, efs)
    depth = ch.depth().astype(np.int64)
    # limit and ModelParameters rows count as depth 1; an Ellipsoid limit's rows as its parent's depth would be the finer choice, but the
    # parameter-space limits dominate those blocks
    D0 = np.where(rj >= 0, depth[np.maximum(rj, 0)], 1)
    anc = ancestor_columns(ch)
    l2 = l2_rows_cover_error(efs)
    refs = {}
    for b in (range(B) if instances is None else instances):
        orc = OracleFunction(ch, efs, "float64", instance=b)
        _, Jall, _, rows = orc.get_jacobian(theta[b])
        state, _, _ = orc.fk(theta[b])
        if enabled is not None:
            orc.set_enabled_parameters(enabled)
        e, J, r, rows = orc.get_jacobian(theta[b])
        e_err = orc.get_error(theta[b])
        assert Jall.shape == J.shape and D0.size <= rows, (Jall.shape, J.shape, D0.size, rows)
        D = np.zeros(rows, np.int64)
        D[:D0.size] = D0
        rho = max(1.0, float(np.abs(state[:, :3]).max()))
        c = np.abs(Jall[:, tcols]).max(axis=1) if tcols.size else np.zeros(rows)
        # the row's scale at generic poses: a row at a stationary point (a rotation difference at zero rotation, whose diagonal entries
        # have a vanishing derivative there) keeps the size of the quantities it differences
        g = np.zeros(rows)
        rng = np.random.default_rng(1000 + b)
        generic = []
        for _ in range(2):
            _, Jg, _, _ = OracleFunction(ch, efs, "float64", instance=b).get_jacobian(rng.uniform(-0.9, 0.9, theta.shape[1]))
            g = np.maximum(g, np.abs(Jg).max(axis=1, initial=0.0))
            generic.append(Jg)
        S = np.abs(J).max(axis=1, initial=0.0) + np.abs(r) + rho * c + g
        # structural zeros: a joint row's columns that drive none of its ancestors, a parameter-space row's columns that are zero at
        # theta and at both generic poses, disabled columns, padding rows
        zero = np.zeros_like(J, bool)
        zero[:rj.size][rj >= 0] = ~anc[rj[rj >= 0]]
        lim = np.nonzero(rj < 0)[0]
        zero[lim] = (J[lim] == 0) & (generic[0][lim] == 0) & (generic[1][lim] == 0)
        if enabled is not None:
            zero[:, ~np.asarray(enabled, bool)] = True
        zero[rj.size:, :] = True
        refs[b] = SweepRef(J, r, float(e), float(e_err), state, D, S, zero, rho, l2, depth)
    return refs


def _error_ratio(ref, tol, e, e64, l2):
    de = abs(e - e64)
    if l2:  # e = sum r_i^2: |e - e64| <= sum (2 |r64_i| beta_i + beta_i^2) with beta_i = (D_i + 1) 2^-24 S_i, + m 2^-24 e64
        scale = float(np.sum(2 * np.abs(ref.r) * tol + tol ** 2)) + ref.r.size * EPS24 * abs(e64)
    else:
        scale = (int(ref.D.max(initial=1)) + 1) * EPS24 * (abs(e64) + float(np.sum(np.abs(ref.r) * ref.S)))
    return 0.0 if de == 0 else (de / scale if scale > 0 else np.inf)


def sweep_ratios(ref, J=None, r=None, e=None, state=None, e_err=None):
    """Worst measured k (|error| over its bound without the K) of each given output of one instance, as a dict: J, r, e (getJacobian's
    error ``e`` and getError's ``e_err``), t and q (skeleton state); raises AssertionError when a structural zero is not exactly 0."""
    out = {}
    tol = (ref.D + 1) * EPS24 * ref.S
    with np.errstate(divide="ignore", invalid="ignore"):
        if J is not None:
            J = np.asarray(J, np.float64)
            nz = J[ref.zero] != 0
            assert not np.any(nz), f"{int(nz.sum())} non-zero entries where the Jacobian is structurally zero"
            d = np.abs(J - ref.J)
            out["J"] = float(np.max(np.where(tol[:, None] > 0, d / tol[:, None], np.where(d > 0, np.inf, 0.0)), initial=0.0))
        if r is not None:
            d = np.abs(np.asarray(r, np.float64) - ref.r)
            out["r"] = float(np.max(np.where(tol > 0, d / tol, np.where(d > 0, np.inf, 0.0)), initial=0.0))
        if e is not None:
            out["e"] = _error_ratio(ref, tol, float(e), ref.e, ref.l2)
        if e_err is not None:  # error-only units (no rows) count in getError only: the residual-derived form does not cover them
            out["e"] = max(out.get("e", 0.0), _error_ratio(ref, tol, float(e_err), ref.e_err, ref.l2 and ref.e_err == ref.e))
        if state is not None:
            st = np.asarray(state, np.float64)
            dj = (ref.jdepth + 1) * EPS24
            out["t"] = float(np.max(np.abs(st[:, :3] - ref.state[:, :3]) / (dj[:, None] * ref.rho)))
            qs = np.maximum(1.0, np.abs(ref.state[:, 7:8]))
            out["q"] = float(np.max(np.abs(st[:, 3:] - ref.state[:, 3:]) / (dj[:, None] * qs)))
    return out


def sweep_failures(ks):
    """The entries of a ratio dict (sweep_ratios) above their pinned K."""
    return {k: v for k, v in ks.items() if not v <= SWEEP_K[k]}
