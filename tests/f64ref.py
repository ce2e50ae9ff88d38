"""Float64 references for the linear-algebra kernels, built from the backend's own float Jacobian.

The Jacobian and residual come from ``SkeletonSolverFunction.get_jacobian`` (the device's float values, promoted to float64), so FK and
Jacobian rounding drop out of every comparison and what remains is the error of the kernel under test:

* JtJ / Jtr kernels: elementwise ``|H - H64| <= c * E`` with ``E = |J|^T |J|`` (``|J|^T |r|`` for Jtr), the classical bound of a
  float dot product of length m; ``c`` depends on the kernel's arithmetic (``jtj_limit``).
* linear solves: the normwise backward error of one Gauss-Newton step, ``||A d - g||inf / ((||E||inf + lambda) ||d||inf + ||g||inf)``
  with ``A = H64 + lambda I`` over the enabled parameters. A correct factorisation keeps it at a small multiple of ``n 2^-24`` whatever
  the conditioning (``solve_limit``); a wrong tile, a missed update or a permuted step moves it by orders of magnitude.

No oracle is involved. Every helper takes a ``lib_path`` so that the CPU emulator (tests/emu) can run the same checks."""
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


def qr_max_chunk_rows(n, smem_bytes=200 * 1024):
    """Jacobian rows the QR step folds at once beside R (qrMaxChunkRows): a block with more rows is split into several chunks."""
    fixed = ((n * (n + 1) // 2 + 3) & ~3) + 3 * ((n + 3) & ~3) + ((n + 4) & ~3) + 8
    floats = smem_bytes // 4
    if floats <= fixed + (n + 1) * 9:
        return 0
    return min((floats - fixed) // (n + 1) - 1, 128) & ~1


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


def dense_cholesky_dispatch(n, smem_optin):
    """(NB, matrix in shared memory) of the dense Eigen-structured Cholesky for n unknowns, restating cholBlockSize / cholSmemBytes /
    launchCholesky. This is a recomputation, not an observation: no entry point reports which variant launched, so a change of the
    launcher's rule that this function does not follow goes unnoticed (the bound still holds on whichever variant ran)."""
    eig = n if n < 32 else min(max((n // 8) // 16 * 16, 8), 128)
    eig = max(eig, 1)
    NB = 8 if eig <= 8 else (16 if eig <= 16 else 32)
    ldp = ((n + 1 + 3) & ~3) + 4
    smem = 4 * (NB * ldp + ((n + 3) & ~3)) + 16 + 4 * (n + 1) * (n | 1)
    return NB, smem <= smem_optin


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
