"""JtJ and linear-solve kernels against float64 references built from the device's own float Jacobian (tests/f64ref.py), at the
dispatch edges of every launcher: wgmma work-item boundaries, the 32-row K block, leading-block stores, the dense Cholesky's block sizes
and shared / global branch, the tile schedule's 256 / 512-thread rule, the fused kernels, the QR step, and batches larger than one wave.

Every case asserts which path it ran (plan stats, fused profile, and the launch variants the solver reports with get_solve_path), so a
change of a launch rule that sends a case down another path fails here instead of silently losing coverage. No oracle is used."""
import numpy as np
import pytest

from momentum_b200 import character as mc
from momentum_b200 import solver as ms
from momentum_b200.problems import bodyhands_problem, humanoid_problem
from tests import f64ref as R

pytestmark = pytest.mark.gpu

def _device():
    import torch

    p = torch.cuda.get_device_properties(0)
    return p.shared_memory_per_block_optin, p.shared_memory_per_multiprocessor, p.multi_processor_count


def _fn(ch, efs, B, enabled=None):
    fn = ms.SkeletonSolverFunction(ch, B, efs)
    fn.upload_targets()
    if enabled is not None:
        fn.set_enabled_parameters(enabled)
    return fn


def _slice(efs, idx):
    """The error functions of the instances ``idx`` (per-instance targets only; everything else is shared)."""
    out = []
    for e in efs:
        t = getattr(e, "targets", None)
        out.append(type(e)(**{**e.__dict__, "targets": np.asarray(t)[idx]}) if t is not None and np.ndim(t) >= 2 else e)
    return out


def _report(title, rows):
    print(f"\n[{title}]")
    for r in rows:
        print("   ", r)


# ------------------------------------------------------------------------------------------------------------------------------
# 1. JtJ / Jtr kernels: elementwise bounds
# ------------------------------------------------------------------------------------------------------------------------------
MODES = {"SIMT": ms.JTJ_FP32_SIMT, "TF32X3": ms.JTJ_TF32X3, "TF32": ms.JTJ_TF32}


def _jtj_case(fn, theta, m, label, worst, rows, modes=MODES):
    J, r = R.jacobian64(fn, theta)
    out = {}
    for name, mode in modes.items():
        _, H, g = fn.get_jtjr(theta, mode)
        ratio = max(R.jtj_ratios(H[b], g[b], J[b], r[b]) for b in range(H.shape[0]))
        lim = R.jtj_limit(mode, m)
        k = ratio / (lim / {"SIMT": R.K_SIMT, "TF32X3": R.K_TF32X3, "TF32": R.K_TF32}[name])
        worst[name] = max(worst.get(name, 0.0), k)
        rows.append((label, name, m, f"ratio {ratio:.3e}", f"limit {lim:.3e}", f"k {k:.3f}"))
        out[name] = (ratio, lim, H, g)
    return out


def _theta(n, B=1, seed=1, scale=0.1):
    return np.random.default_rng(seed).uniform(-scale, scale, (B, n)).astype(np.float32)


# n + 1 = numCols + 1 of the wgmma shapes: row tiles at 128, N = 128 -> 256 box at 256, a far item from 385, the last supported 512
SHAPES = [16, 17, 127, 128, 129, 255, 256, 257, 383, 384, 385, 511, 512]


def test_jtj_elementwise_bounds_at_the_work_item_edges():
    worst, rows, fails, tf32_beyond_x3 = {}, [], [], 0.0
    # plus a single enabled column (ns = 1) of the smallest chain: get_jtjr keeps every model parameter as a device column, so this is a
    # one-column leading-block store from the numCols + 1 = 11 shape. The shape numCols + 1 = 2 itself is the compacted plan of the dense
    # solve at n = 1 with 3xTF32 JtJ (test_dense_cholesky_backward_error_at_every_block_size).
    cases = [(n1, None) for n1 in SHAPES] + [(11, 1)]
    for n1, ns in cases:
        n = n1 - 1
        ch, efs, _ = R.chain_case(n, positions=11, seed=n1)  # m = 33: two K blocks, one of them a single row
        enabled = None
        if ns is not None:
            enabled = np.zeros(n, bool); enabled[:ns] = True
        fn = _fn(ch, efs, 1, enabled)
        res = _jtj_case(fn, _theta(n, seed=n1), 33, f"numCols+1={n1}" + ("" if ns is None else f" ns={ns}"), worst, rows)
        for name, (ratio, lim, _, _) in res.items():
            if ratio > lim:
                fails.append((n1, ns, name, ratio, lim))
        tf32_beyond_x3 = max(tf32_beyond_x3, res["TF32"][0] / R.jtj_limit(ms.JTJ_TF32X3, 33))
    _report("JtJ elementwise, work-item edges", rows)
    print("    worst k per mode:", worst, " worst TF32 ratio / TF32X3 limit:", tf32_beyond_x3)
    assert not fails, fails
    # the 3xTF32 limit must be tight enough to reject the single-TF32 product
    assert tf32_beyond_x3 > 1.0, tf32_beyond_x3


@pytest.mark.parametrize("n1", [129, 385])
def test_jtj_elementwise_bounds_over_row_counts(n1):
    """1 - 3 rows (kRows rounds up to 4), both sides of the 32-row K block, and hundreds of rows (many K blocks, stage-ring wraps)."""
    n = n1 - 1
    worst, rows, fails = {}, [], []
    for P, Q in [(0, 1), (0, 2), (1, 0), (10, 1), (10, 2), (11, 0), (100, 0), (200, 0)]:
        m = 3 * P + Q
        ch, efs, _ = R.chain_case(n, positions=P, planes=Q, seed=m)
        fn = _fn(ch, efs, 1)
        assert fn.jacobian_rows == (m + 7) // 8 * 8
        for name, (ratio, lim, _, _) in _jtj_case(fn, _theta(n, seed=m), m, f"numCols={n} m={m}", worst, rows).items():
            if ratio > lim:
                fails.append((m, name, ratio, lim))
    _report(f"JtJ elementwise, row counts, n+1={n1}", rows)
    print("    worst k per mode:", worst)
    assert not fails, fails


def test_jtj_leading_block_stores():
    """get_jtjr with disabled parameters: the kernels store only the leading ns x ns block (ns = last enabled parameter + 1 < numCols),
    with zero columns inside it. ns itself crosses 128 and 256."""
    worst, rows, fails = {}, [], []
    cases = []
    for n1, ns in [(129, 127), (257, 128), (257, 129), (257, 255), (385, 256), (385, 257), (512, 384), (512, 385), (257, 5)]:
        ch, efs, _ = R.chain_case(n1 - 1, positions=12, seed=ns)
        en = np.zeros(ch.num_params, bool); en[:ns] = True
        en[[1, ns // 2, ns - 2]] = False
        cases.append((ch, efs, en, f"numCols+1={n1} ns={ns}", _theta(ch.num_params, seed=ns)))
    ch, efs, _, theta_star = bodyhands_problem(1)  # branching rig, m = 600, numCols = 424
    th = (0.3 * theta_star).astype(np.float32)
    for cut, holes in [(423, [2, 130, 257, 300]), (257, [0, 128, 200]), (129, [64, 127])]:
        en = np.zeros(ch.num_params, bool); en[:cut] = True; en[holes] = False
        cases.append((ch, efs, en, f"bodyhands ns={cut}", th))
    for ch, efs, en, label, th in cases:
        fn = _fn(ch, efs, 1, en)
        assert fn.actual_parameters == int(np.nonzero(en)[0].max()) + 1 < ch.num_params
        m = sum(3 * len(e.parents) for e in efs)
        for name, (ratio, lim, _, _) in _jtj_case(fn, th, m, label, worst, rows).items():
            if ratio > lim:
                fails.append((label, name, ratio, lim))
    _report("JtJ elementwise, leading-block stores", rows)
    print("    worst k per mode:", worst)
    assert not fails, fails


def test_jtj_past_512_columns_is_rejected_by_the_tensor_cores_and_auto_falls_back():
    n = 512  # numCols + 1 = 513: more than four row tiles
    ch, efs, _ = R.chain_case(n, positions=11, seed=513)
    fn = _fn(ch, efs, 1)
    th = _theta(n, seed=513)
    for mode in (ms.JTJ_TF32X3, ms.JTJ_TF32):
        with pytest.raises(ms.MomentumB200Error):
            fn.get_jtjr(th, mode)
    J, r = R.jacobian64(fn, th)
    _, H, g = fn.get_jtjr(th, ms.JTJ_AUTO)
    ratio = R.jtj_ratios(H[0], g[0], J[0], r[0])
    _, Hs, gs = fn.get_jtjr(th, ms.JTJ_FP32_SIMT)
    print(f"\n[JtJ n+1=513, AUTO] ratio {ratio:.3e} limit {R.jtj_limit(ms.JTJ_FP32_SIMT, 33):.3e}")
    assert ratio <= R.jtj_limit(ms.JTJ_FP32_SIMT, 33)
    assert np.array_equal(H, Hs) and np.array_equal(g, gs)  # AUTO is the SIMT kernel here


def test_jtj_batch_larger_than_the_sm_count_is_bitwise_per_instance():
    """B = 300 > 132 SMs: each wgmma CTA loops over several instances (the stage ring's phase carries across them). Every instance
    must come out bit for bit as when it is alone in the batch, in every mode."""
    B, n = 300, 256
    ch, efs, _ = R.chain_case(n, positions=40, B=B, seed=300)
    th = _theta(n, B=B, seed=300)
    fn = _fn(ch, efs, B)
    J, r = R.jacobian64(fn, th)
    full = {name: fn.get_jtjr(th, mode) for name, mode in MODES.items()}
    for b in np.random.default_rng(3).choice(B, 12, replace=False):
        one = _fn(ch, _slice(efs, [b]), 1)
        for name, mode in MODES.items():
            _, H1, g1 = one.get_jtjr(th[b:b + 1], mode)
            _, H, g = full[name][0], full[name][1], full[name][2]
            assert np.array_equal(H1[0], H[b]) and np.array_equal(g1[0], g[b]), (name, b)
            assert R.jtj_ratios(H[b], g[b], J[b], r[b]) <= R.jtj_limit(mode, 120), (name, b)


# ------------------------------------------------------------------------------------------------------------------------------
# 2. Linear-solve kernels: backward error of one Gauss-Newton step
# ------------------------------------------------------------------------------------------------------------------------------
def _opts(**kw):
    base = dict(min_iterations=1, max_iterations=1, threshold=1.0, regularization=0.05, fused_mode=ms.FUSED_OFF)
    base.update(kw)
    return ms.GaussNewtonSolverOptions(**base)


def _step_case(ch, efs, theta0, opts, enabled=None):
    solver, out, J, r, cols, delta, lam = R.one_step(ch, efs, theta0, opts, enabled=enabled, rel_damping=1e-5)
    assert np.all(out["status"] == 0), out["status"]
    be = max(R.backward_error(J[b], r[b], cols, delta[b], lam) for b in range(theta0.shape[0]))
    return solver, be, len(cols), (J, r, cols, delta, lam)


def _dense_case(n):
    """A chain with n enabled parameters: n < 10 is a leading subset of the smallest chain, n = 424 is bodyhands300."""
    if n == 424:
        ch, efs, _, _ = bodyhands_problem(1)
        return ch, efs, None
    if n < 10:
        ch, efs, _ = R.chain_case(10, positions=3, seed=n)
        en = np.zeros(10, bool); en[:n] = True
        return ch, efs, en
    ch, efs, _ = R.chain_case(n, positions=min(n - 7, 12), seed=n)
    return ch, efs, None


# n -> (NB, matrix in shared memory) on a device with 227 KB of opt-in shared memory per block, as the solver reports the variant it ran.
DENSE = {1: (8, True), 8: (8, True), 9: (16, True), 16: (16, True), 17: (32, True), 31: (32, True), 32: (8, True), 127: (8, True),
         128: (16, True), 231: (16, True), 232: (16, False), 255: (16, False), 256: (32, False), 424: (32, False)}
SOLVE_WORST = {}


@pytest.mark.parametrize("jtj", [ms.JTJ_FP32_SIMT, ms.JTJ_TF32X3])
def test_dense_cholesky_backward_error_at_every_block_size(jtj):
    rows, fails = [], []
    for n, expected in DENSE.items():
        ch, efs, en = _dense_case(n)
        solver, be, ns, _ = _step_case(ch, efs, np.zeros((1, ch.num_params)), _opts(cholesky_mode=ms.CHOLESKY_DENSE_EIGEN, jtj_mode=jtj), en)
        path = solver.get_solve_path()
        assert path["kind"] == "dense" and (path["dense_nb"], bool(path["dense_in_smem"])) == expected, (n, path)
        st = solver.get_plan_stats()
        assert ns == n and st["cholesky_tiles"] == 0 and st["strip_floats"] == 0 and solver.get_fused_profile()["fused"] == 0
        k = be / R.solve_limit(n) * R.SOLVE_K["dense"]
        SOLVE_WORST["dense"] = max(SOLVE_WORST.get("dense", 0.0), k)
        rows.append((n, expected, f"backward error {be:.3e}", f"limit {R.solve_limit(n):.3e}", f"k {k:.3f}"))
        if be > R.solve_limit(n):
            fails.append((n, be))
    _report(f"dense Cholesky, jtj mode {jtj}", rows)
    assert not fails, fails


def test_backward_error_rejects_a_swapped_or_tile_dropped_step():
    """Self-check of the bound: the step of a correct factorisation passes, the same step with two components swapped and the exact
    solution of a system with its off-diagonal 16 x 16 tile zeroed do not (n = 32: two tile columns)."""
    ch, efs, en = _dense_case(32)
    _, be, n, (J, r, cols, delta, lam) = _step_case(ch, efs, np.zeros((1, ch.num_params)), _opts(cholesky_mode=ms.CHOLESKY_DENSE_EIGEN), en)
    d = delta[0]
    lim = R.solve_limit(n)
    assert be <= lim
    i, j = int(np.argmax(d)), int(np.argmin(d))
    sw = d.copy(); sw[[i, j]] = sw[[j, i]]
    H64, g64, _, _ = R.normal_equations64(J[0], r[0], cols)
    A = H64 + lam * np.eye(n)
    A[16:32, 0:16] = 0.0; A[0:16, 16:32] = 0.0
    dropped = np.linalg.solve(A, g64)
    be_sw, be_tile = R.backward_error(J[0], r[0], cols, sw, lam), R.backward_error(J[0], r[0], cols, dropped, lam)
    print(f"\n[self-check] correct {be:.3e}, swapped {be_sw:.3e}, tile dropped {be_tile:.3e}, limit {lim:.3e}")
    assert be_sw > 100 * lim and be_tile > 100 * lim


def test_cholesky_auto_falls_back_to_the_dense_global_memory_kernel():
    """A chain with a constraint on its end effector couples every parameter pair: the dense tile schedule of n = 330 needs more than
    200 KB, so CHOLESKY_AUTO runs the dense kernel with the matrix in global memory, and an explicit tile request raises."""
    n = 330
    ch, efs, _ = R.chain_case(n, positions=12, seed=n)
    solver, be, ns, _ = _step_case(ch, efs, np.zeros((1, n)), _opts(cholesky_mode=ms.CHOLESKY_AUTO))
    path = solver.get_solve_path()
    assert path["kind"] == "dense" and (path["dense_nb"], path["dense_in_smem"]) == (32, 0), path
    assert solver.get_plan_stats()["cholesky_tiles"] == 0 and solver.get_fused_profile()["fused"] == 0
    print(f"\n[AUTO fallback n=330] backward error {be:.3e} limit {R.solve_limit(n):.3e} k {be / R.solve_limit(n) * R.SOLVE_K['dense']:.3f}")
    SOLVE_WORST["dense"] = max(SOLVE_WORST.get("dense", 0.0), be / R.solve_limit(n) * R.SOLVE_K["dense"])
    assert be <= R.solve_limit(n)
    fn = _fn(ch, efs, 1)
    for mode in (ms.CHOLESKY_TILES_DENSE,):
        with pytest.raises(ms.MomentumB200Error):
            ms.GaussNewtonSolver(_opts(cholesky_mode=mode), fn).solve(np.zeros((1, n)))


TILE_CASES = {  # name: (rig, cholesky mode, jtj mode, fused mode, 512-thread variants expected (None: not asserted))
    "humanoid_gram_sparse": ("humanoid", ms.CHOLESKY_TILES_SPARSE, ms.JTJ_AUTO, ms.FUSED_OFF, False),
    "humanoid_gram_dense": ("humanoid", ms.CHOLESKY_TILES_DENSE, ms.JTJ_AUTO, ms.FUSED_OFF, None),  # 105 tiles: next to the rule
    "humanoid_kmajor_simt": ("humanoid", ms.CHOLESKY_TILES_SPARSE, ms.JTJ_FP32_SIMT, ms.FUSED_OFF, False),
    "humanoid_kmajor_tf32x3": ("humanoid", ms.CHOLESKY_TILES_DENSE, ms.JTJ_TF32X3, ms.FUSED_OFF, None),
    "bodyhands_gram_sparse": ("bodyhands", ms.CHOLESKY_TILES_SPARSE, ms.JTJ_AUTO, ms.FUSED_OFF, True),
    "bodyhands_kmajor_tf32x3": ("bodyhands", ms.CHOLESKY_TILES_SPARSE, ms.JTJ_TF32X3, ms.FUSED_OFF, True),
    "humanoid_gram_cholesky": ("humanoid", ms.CHOLESKY_TILES_SPARSE, ms.JTJ_AUTO, ms.FUSED_GRAM_CHOLESKY, False),
    "humanoid_persistent": ("humanoid", ms.CHOLESKY_TILES_SPARSE, ms.JTJ_AUTO, ms.FUSED_PERSISTENT, False),
    "humanoid_subset_persistent": ("humanoid_subset", ms.CHOLESKY_TILES_SPARSE, ms.JTJ_AUTO, ms.FUSED_PERSISTENT, False),
}


def _rig(name, B=1):
    enabled = None
    if name == "bodyhands":
        ch, efs, _, ts = bodyhands_problem(B)
    else:
        ch, efs, _, ts = humanoid_problem(B, orientation=True)
        if name == "humanoid_subset":
            enabled = np.ones(ch.num_params, bool); enabled[[0, 5, 6, 40, 41, 42, 100, 219]] = False
    return ch, efs, ts, enabled


@pytest.mark.parametrize("case", list(TILE_CASES))
def test_tile_path_backward_error(case):
    rig, chol, jtj, fused, wide = TILE_CASES[case]
    ch, efs, _, en = _rig(rig)
    solver, be, n, _ = _step_case(ch, efs, np.zeros((1, ch.num_params)), _opts(cholesky_mode=chol, jtj_mode=jtj, fused_mode=fused), en)
    st, prof = solver.get_plan_stats(), solver.get_fused_profile()
    assert st["cholesky_tiles"] > 0
    assert prof["fused"] == {ms.FUSED_OFF: 0, ms.FUSED_PERSISTENT: 1, ms.FUSED_GRAM_CHOLESKY: 2}[fused]
    gram = jtj == ms.JTJ_AUTO
    assert (st["strip_floats"] > 0) == gram  # tile-sparse Gram on the strip layout, else K-major H through TMA
    if fused == ms.FUSED_OFF and wide is not None:  # choleskyScheduledKernel and gramTilesKernel: 512 threads when one CTA per SM fits
        path = solver.get_solve_path()
        assert path["chol_threads"] == (512 if wide else 256) and path["gram_threads"] == ((512 if wide else 256) if gram else 0), path
    if fused == ms.FUSED_GRAM_CHOLESKY:
        # Every Cholesky tile is dealt to one of the 8 warps (buildGramPlan), so the plan has at least ceil(tiles / 8) rounds per warp,
        # and the kernel launched, so at most kGramCholMaxRounds = 8: cfg3's plan sits within one round of the limit. A tile whose
        # storage overlaps the strips (t * 256 < strip floats + 64) is parked in an L2 scratch slot until the strips are dead.
        tiles = st["cholesky_tiles"]
        assert -(-tiles // 8) >= 7, tiles
        parked = min(tiles, -(-(st["strip_floats"] + 64) // 256))
        print(f"    Gram + Cholesky: >= {-(-tiles // 8)} rounds per warp, {parked} of {tiles} tiles parked")
        assert 0 < parked < tiles
    key = "tiles" if fused == ms.FUSED_OFF else ("gram_cholesky" if fused == ms.FUSED_GRAM_CHOLESKY else "persistent")
    lim = R.solve_limit(n, key)
    SOLVE_WORST[key] = max(SOLVE_WORST.get(key, 0.0), be / lim * R.SOLVE_K[key])
    print(f"\n[{case}] n={n} tiles={st['cholesky_tiles']} backward error {be:.3e} limit {lim:.3e} k {be / lim * R.SOLVE_K[key]:.5f}")
    assert be <= lim


@pytest.mark.parametrize("case", ["humanoid_split_block", "chain_subset"])
def test_qr_step_backward_error(case):
    """GaussNewtonSolverQRT's step solves the same damped normal equations. humanoid72 (n = 220, close to the kernel's limit) with a
    216-row Position block: more rows than fit beside R, so the block is folded in several chunks."""
    if case == "humanoid_split_block":
        ch, _, _, ts = humanoid_problem(1, orientation=False)
        joints = np.arange(ch.num_joints, dtype=np.int32)
        off = np.random.default_rng(9).uniform(-3, 3, (ch.num_joints, 3))
        efs = [mc.PositionErrorFunction(joints, off, np.ones(ch.num_joints), mc.world_points(ch, ts, joints, off), weight=mc.PositionErrorFunction.kLegacyWeight)]
        en = None
    else:
        ch, efs, _ = R.chain_case(60, positions=12, seed=60)
        en = np.ones(60, bool); en[[0, 7, 33]] = False
    th0 = np.zeros((1, ch.num_params))
    solver, be, n, _ = _step_case(ch, efs, th0, _opts(linear_solver=ms.LINEAR_SOLVER_QR), en)
    st = solver.get_plan_stats()
    assert solver.get_fused_profile()["fused"] == 0 and st["cholesky_tiles"] == 0 and st["strip_floats"] == 0  # dense Jacobian layout
    # the chunk rows the QR step ran with: the widest block must need more than one chunk on the split case
    path = solver.get_solve_path()
    chunk, widest = path["qr_max_chunk_rows"], max(3 * len(e.parents) for e in efs)
    assert path["kind"] == "qr" and chunk >= 8 and (widest > chunk) == (case == "humanoid_split_block"), (chunk, widest)
    assert (path["qr_chunks"] > len(efs)) == (case == "humanoid_split_block") and path["qr_widest_chunk"] == min(chunk, widest), path
    lim = R.solve_limit(n, "qr")
    SOLVE_WORST["qr"] = max(SOLVE_WORST.get("qr", 0.0), be / lim * R.SOLVE_K["qr"])
    print(f"\n[QR {case}] n={n} chunk rows {chunk}, widest block {widest}: backward error {be:.3e} limit {lim:.3e} k {be / lim * R.SOLVE_K['qr']:.5f}")
    assert be <= lim
    # a different solver ran: the dense Cholesky step on the same system is a different rounding of the same solution
    _, chol, *_ = R.one_step(ch, efs, th0, _opts(cholesky_mode=ms.CHOLESKY_DENSE_EIGEN), enabled=en, rel_damping=1e-5)
    _, qr, *_ = R.one_step(ch, efs, th0, _opts(linear_solver=ms.LINEAR_SOLVER_QR), enabled=en, rel_damping=1e-5)
    assert not np.array_equal(chol["params"], qr["params"])


def test_zz_report_solve_bounds():
    print("\n[backward error] worst k per path:", SOLVE_WORST, " pinned:", R.SOLVE_K)


# ------------------------------------------------------------------------------------------------------------------------------
# 3. An instance's result does not depend on its batch
# ------------------------------------------------------------------------------------------------------------------------------
DENSE_OFF = dict(fused_mode=ms.FUSED_OFF, cholesky_mode=ms.CHOLESKY_DENSE_EIGEN)
GRAM = dict(cholesky_mode=ms.CHOLESKY_TILES_SPARSE, jtj_mode=ms.JTJ_SPARSE_TILES)
BATCH_PATHS = {  # name: (rig, options that pin the kernels whatever the batch size, expected path)
    # dense kernel: NB = 16 with the matrix in shared memory (humanoid72), NB = 16 and NB = 32 in global memory (long chains), and the
    # CHOLESKY_AUTO fallback (its choice depends on the tile schedule's size only, never on the batch)
    "dense_simt": ("humanoid", dict(DENSE_OFF, jtj_mode=ms.JTJ_FP32_SIMT), "dense"),
    "dense_tf32x3": ("humanoid", dict(DENSE_OFF, jtj_mode=ms.JTJ_TF32X3), "dense"),
    "dense_global_nb16": ("chain240", dict(DENSE_OFF, jtj_mode=ms.JTJ_FP32_SIMT), "dense"),
    "dense_global_nb32_tf32x3": ("chain300", dict(DENSE_OFF, jtj_mode=ms.JTJ_TF32X3), "dense"),
    "auto_fallback_dense_global": ("chain330", dict(fused_mode=ms.FUSED_OFF, cholesky_mode=ms.CHOLESKY_AUTO), "dense"),
    # tile-scheduled kernel: 256-thread variants (humanoid72) and 512-thread variants of both the Gram and the Cholesky kernel (bodyhands300)
    "tiles_gram": ("humanoid", dict(GRAM, fused_mode=ms.FUSED_OFF), "tiles"),
    "tiles_kmajor_tf32x3": ("humanoid", dict(cholesky_mode=ms.CHOLESKY_TILES_DENSE, jtj_mode=ms.JTJ_TF32X3, fused_mode=ms.FUSED_OFF), "tiles"),
    "tiles_gram_wide": ("bodyhands", dict(GRAM, fused_mode=ms.FUSED_OFF), "tiles_wide"),
    "tiles_kmajor_tf32x3_wide": ("bodyhands", dict(cholesky_mode=ms.CHOLESKY_TILES_SPARSE, jtj_mode=ms.JTJ_TF32X3, fused_mode=ms.FUSED_OFF), "tiles_wide"),
    "gram_cholesky": ("humanoid", dict(GRAM, fused_mode=ms.FUSED_GRAM_CHOLESKY), "gram_cholesky"),
    "persistent": ("humanoid", dict(GRAM, fused_mode=ms.FUSED_PERSISTENT), "persistent"),
    "qr": ("humanoid", dict(linear_solver=ms.LINEAR_SOLVER_QR, fused_mode=ms.FUSED_OFF), "dense"),
}


def _batch_rig(rig, B):
    """(character, error functions, solutions, damping) of B instances; long chains get a damping relative to their JtJ diagonal so
    that every instance's factorisation completes in float."""
    if rig == "humanoid":
        ch, efs, _, ts = humanoid_problem(B, orientation=True)
        return ch, efs, ts, None
    if rig == "bodyhands":
        ch, efs, _, ts = bodyhands_problem(B)
        return ch, efs, ts, None
    ch, efs, ts = R.chain_case(int(rig[5:]), positions=12, B=B, seed=B)
    return ch, efs, ts, 1e-4


@pytest.mark.parametrize("path", list(BATCH_PATHS))
def test_instance_result_does_not_depend_on_the_batch(path):
    """About three waves plus a remainder (3 x SMs x 3 + 17 instances), instances starting at, near and far from their solution so that
    they stop at different iterations. A seeded sample re-solved alone must match its result inside the shuffled batch bit for bit."""
    rig, kw, expect = BATCH_PATHS[path]
    _, _, sms = _device()
    B = 3 * sms * 3 + 17
    ch, efs, ts, rel_damping = _batch_rig(rig, B)
    rng = np.random.default_rng(11)
    scale = rng.choice([0.0, 0.002, 0.05, 1.0], size=B)
    theta0 = (ts * (1.0 - scale[:, None]) + rng.normal(size=ts.shape) * 0.01 * (scale[:, None] > 0)).astype(np.float32)
    perm = rng.permutation(B)
    efs_p, th_p = _slice(efs, perm), theta0[perm]
    fn = _fn(ch, efs_p, B)
    lam = 0.05
    if rel_damping is not None:
        J, _ = R.jacobian64(fn, th_p)
        lam = max(lam, rel_damping * float(np.max(np.sum(J ** 2, axis=1))))
    opts = ms.GaussNewtonSolverOptions(min_iterations=1, max_iterations=10, threshold=1e4, regularization=lam, **kw)
    solver = ms.GaussNewtonSolver(opts, fn)
    full = solver.solve(th_p)
    st, fused, path = solver.get_plan_stats(), solver.get_fused_profile()["fused"], solver.get_solve_path()
    assert fused == {ms.FUSED_OFF: 0, ms.FUSED_PERSISTENT: 1, ms.FUSED_GRAM_CHOLESKY: 2}[opts.fused_mode]
    if expect == "dense":
        assert st["cholesky_tiles"] == 0 and st["strip_floats"] == 0
        if rig.startswith("chain"):  # the global-memory branch, NB from the block-size rule
            assert (path["dense_nb"], path["dense_in_smem"]) == ((16 if ch.num_params < 256 else 32), 0), path
    else:
        assert st["cholesky_tiles"] > 0 and (st["strip_floats"] > 0) == (opts.jtj_mode == ms.JTJ_SPARSE_TILES)
        if expect == "tiles_wide":
            assert path["chol_threads"] == 512 and path["gram_threads"] == (512 if st["strip_floats"] > 0 else 0), path
    assert np.all(full["status"] == 0), np.unique(full["status"], return_counts=True)
    assert len(np.unique(full["iterations"])) >= 2, np.unique(full["iterations"])
    for k in np.random.default_rng(12).choice(B, 16, replace=False):
        one = ms.GaussNewtonSolver(opts, _fn(ch, _slice(efs_p, [k]), 1)).solve(th_p[k:k + 1])
        assert np.array_equal(one["params"][0], full["params"][k]), (path, k)
        assert one["errors"][0] == full["errors"][k] and one["iterations"][0] == full["iterations"][k] and one["status"][0] == full["status"][k]
