"""GPU parity tests proper: the CUDA product path through the C-ABI vs the float oracle on the same
seeded inputs (small sizes), plus size-independent properties at BASELINE.json's full sizes."""
import numpy as np
import pytest

from momentum_b200 import character as mc
from momentum_b200 import solver as ms
from momentum_b200.problems import bodyhands_problem, chain_problem, chain22_problem, humanoid_problem
from tests import parity

pytestmark = pytest.mark.gpu

FAMS = [("position",), ("orientation",), ("state",), ("limit",), ("position", "orientation", "state", "limit")]


@pytest.mark.parametrize("fams", FAMS)
def test_single_iteration_families(fams):
    ch, efs, theta0, _ = chain_problem(J=6, B=5, seed=21, families=fams)
    parity.check_fk(ch, efs, theta0)
    parity.check_single_iteration(ch, efs, theta0)


@pytest.mark.parametrize("logmap,rot_diff", [(True, False), (False, True)])
def test_single_iteration_logmap_rotdiff(logmap, rot_diff):
    ch, efs, theta0, _ = chain_problem(J=7, B=3, seed=22, families=("orientation", "state"), logmap=logmap, rot_diff=rot_diff)
    parity.check_single_iteration(ch, efs, theta0)


@pytest.mark.parametrize("alpha,c", [(mc.LOSS_L1, 0.7), (mc.LOSS_CAUCHY, 1.3), (mc.LOSS_WELSCH, 0.9), (-2.0, 1.1), (1.5, 0.8)])
def test_single_iteration_generalized_loss(alpha, c):
    ch, efs, theta0, _ = chain_problem(J=5, B=3, seed=23, families=("position", "orientation", "limit"), loss=(alpha, c))
    parity.check_single_iteration(ch, efs, theta0)


def test_single_iteration_enabled_subset():
    ch, efs, theta0, _ = chain_problem(J=6, B=3, seed=24)
    en = np.ones(ch.num_params, bool); en[[0, 2, 5, 8, ch.num_params - 1]] = False
    parity.check_single_iteration(ch, efs, theta0, enabled=en)


def test_edge_cases_empty_and_degenerate_inputs():
    parity.check_edge_cases()


def test_humanoid_single_iteration():
    ch, efs, theta0, theta_star = humanoid_problem(40, orientation=True)
    th = (theta0 + 0.3 * theta_star).astype(np.float32)
    parity.check_single_iteration(ch, efs, th[:40])


@pytest.mark.parametrize("mode,rtol", [(ms.JTJ_TF32X3, 2e-5), (ms.JTJ_TF32, 5e-3)])
@pytest.mark.parametrize("case", ["humanoid", "chain22", "chain_all_families", "subset", "bodyhands", "bodyhands_subset"])
def test_jtj_tensor_core_modes(case, mode, rtol):
    """wgmma JtJ (3xTF32 split: fp32-class; single TF32: ~1e-3) vs the float oracle's getJtJR."""
    enabled = None
    if case.startswith("bodyhands"):  # cfg4 shape: 425 operand rows -> four row tiles, six work items (two with a separate A box), m = 600
        ch, efs, theta0, theta_star = bodyhands_problem(5)
        th = (theta0 + 0.3 * theta_star).astype(np.float32)
        if case == "bodyhands_subset":
            enabled = np.ones(ch.num_params, bool); enabled[[2, 130, 257, 300, 423]] = False
    elif case == "humanoid":    # rows = 221 -> two 128-row M tiles, N = 128 / 224
        ch, efs, theta0, theta_star = humanoid_problem(37, orientation=True)
        th = (theta0 + 0.3 * theta_star).astype(np.float32)
    elif case == "chain22":     # rows = 30 -> one M tile, N = 32
        ch, efs, th, _ = chain22_problem()
        th = th + 0.2
    elif case == "chain_all_families":
        ch, efs, th, _ = chain_problem(J=12, B=9, seed=41)
    else:
        ch, efs, th, _ = chain_problem(J=12, B=5, seed=42)
        enabled = np.ones(ch.num_params, bool); enabled[[3, 7, 18]] = False
    parity.check_single_iteration(ch, efs, th, enabled=enabled, rtol=rtol, jtj_mode=mode, check_jacobian=False)


def test_solve_with_tensor_core_jtj_matches_oracle():
    B = 64
    ch, efs, theta0, _ = humanoid_problem(B, orientation=True)
    opts = ms.GaussNewtonSolverOptions(min_iterations=1, max_iterations=50, threshold=1.0, regularization=0.05, jtj_mode=ms.JTJ_TF32X3)
    out, worst = parity.check_solve(ch, efs, theta0, opts, instances=range(0, B, 7))
    print("max rel param diff (3xTF32 JtJ)", worst)


def test_cfg4_solve_on_the_dense_wgmma_jtj():
    """BASELINE configs[3] "full JtJ tensor-core path": bodyhands300 (n = 424) with the dense wgmma JtJ (3xTF32) feeding the
    tile-scheduled Cholesky, against the oracle and against the default tile-sparse path."""
    ch, efs, theta0, _ = bodyhands_problem(8)
    opts = ms.GaussNewtonSolverOptions(min_iterations=10, max_iterations=10, threshold=1.0, regularization=0.05, jtj_mode=ms.JTJ_TF32X3)
    out, worst = parity.check_solve(ch, efs, theta0, opts, instances=range(0, 8, 3), param_tol=2e-4)
    ref = ms.GaussNewtonSolver(ms.GaussNewtonSolverOptions(min_iterations=10, max_iterations=10, threshold=1.0, regularization=0.05), parity.build_function(ch, efs, 8)).solve(theta0)
    assert np.all(out["status"] == 0) and np.max(np.abs(out["params"] - ref["params"])) <= 2e-3
    print("cfg4 on the dense wgmma JtJ: max rel param diff vs oracle", worst)


def test_plane_and_model_parameters_error_functions():
    """SURVEY 8(f) rank 1: PlaneErrorFunction (plain and half-plane) and ModelParametersErrorFunction on the device path."""
    ch, efs, theta0, _ = chain_problem(J=6, B=5, seed=31, families=("position", "limit", "plane", "halfplane", "model_parameters"))
    parity.check_single_iteration(ch, efs, theta0)
    en = np.ones(ch.num_params, bool); en[[1, 4, 9]] = False
    parity.check_single_iteration(ch, efs, theta0, enabled=en)
    # fixed iteration count: the relative-change stop (solver.cpp:98-101) sits at the float rounding floor on this fixture, so the
    # iteration at which it fires is not comparable between two float implementations
    opts = ms.GaussNewtonSolverOptions(min_iterations=8, max_iterations=8, threshold=10.0, regularization=0.05)
    parity.check_solve(ch, efs, theta0, opts, param_tol=2e-4)
    parity.check_solve(ch, efs, theta0, opts, enabled=en, param_tol=2e-4)
    # negative target weights: no Jacobian row but counted by getError (model_parameters_error_function.cpp:56-59 vs :113)
    tw = np.asarray(efs[-1].target_weights, np.float64).copy(); tw[[0, 3, 7]] = [-0.7, -1.2, -0.4]
    neg = efs[:-1] + [mc.ModelParametersErrorFunction(tw, efs[-1].targets, weight=0.6)]
    parity.check_single_iteration(ch, neg, theta0)
    ls = ms.GaussNewtonSolverOptions(min_iterations=4, max_iterations=4, threshold=10.0, regularization=0.05, do_line_search=True)
    parity.check_solve(ch, neg, theta0, ls, param_tol=2e-4)
    # on the tile-scheduled path (>= 48 parameters): floor planes + a pose prior on the humanoid
    ch, efs, theta0, theta_star = humanoid_problem(8, orientation=True)
    rng = np.random.default_rng(5)
    feet = np.array([60, 61, 65, 66], np.int32)
    off = rng.uniform(-1, 1, (4, 3))
    pts = mc.world_points(ch, theta_star, feet, off)
    nrm = np.tile(np.array([0.0, 1.0, 0.0]), (8, 4, 1))
    d = pts[..., 1] + 0.5 * rng.normal(size=(8, 4))
    efs.append(mc.PlaneErrorFunction(feet, off, np.ones(4), np.concatenate([nrm, d[..., None]], -1), above=True, weight=mc.PlaneErrorFunction.kLegacyWeight))
    efs.append(mc.ModelParametersErrorFunction(np.where(np.arange(ch.num_params) % 3 == 0, 1.0, 0.0), 0.9 * theta_star, weight=1e-3))
    opts = ms.GaussNewtonSolverOptions(min_iterations=1, max_iterations=8, threshold=1.0, regularization=0.05)
    parity.check_solve(ch, efs, theta0, opts, instances=[0, 3, 7])
    # every family at once on the tile path (one-row units share row quads)
    ch, efs, theta0, ts = chain_problem(J=20, B=3, seed=33, families=("position", "orientation", "state", "limit", "plane", "halfplane", "model_parameters"))
    theta0 = ts + 0.05 * theta0
    opts = ms.GaussNewtonSolverOptions(min_iterations=1, max_iterations=5, threshold=1.0, regularization=0.05, cholesky_mode=ms.CHOLESKY_TILES_SPARSE)
    parity.check_solve(ch, efs, theta0, opts, param_tol=3e-4)


def test_solve_jtj_paths_into_the_tile_cholesky():
    """The tile-scheduled Cholesky fed three ways: tile-sparse Gram (default and on request), dense SIMT JtJ through TMA boxes."""
    B = 16
    ch, efs, theta0, _ = humanoid_problem(B, orientation=True)
    for jtj in (ms.JTJ_SPARSE_TILES, ms.JTJ_FP32_SIMT):
        opts = ms.GaussNewtonSolverOptions(min_iterations=1, max_iterations=8, regularization=0.05, jtj_mode=jtj, cholesky_mode=ms.CHOLESKY_TILES_SPARSE)
        parity.check_solve(ch, efs, theta0, opts, instances=[0, 5, 15])
    # the strip layout only exists with the tile schedule
    opts = ms.GaussNewtonSolverOptions(min_iterations=1, max_iterations=2, jtj_mode=ms.JTJ_SPARSE_TILES, cholesky_mode=ms.CHOLESKY_DENSE_EIGEN)
    fn = parity.build_function(ch, efs, B)
    with pytest.raises(ms.MomentumB200Error):
        ms.GaussNewtonSolver(opts, fn).solve(theta0)


def test_bodyhands_single_iteration_wide_rig():
    # 300 joints / n = 424 / m = 600: multi-pass levels (>32 joints per depth level), matrix too big for smem Cholesky
    ch, efs, theta0, theta_star = bodyhands_problem(3)
    th = (theta0 + 0.3 * theta_star).astype(np.float32)
    parity.check_single_iteration(ch, efs, th, check_jacobian=True)


@pytest.mark.parametrize("line_search,subset", [(False, False), (True, False), (True, True)])
def test_solve_chain_all_families(line_search, subset):
    ch, efs, theta0, _ = chain_problem(J=6, B=7, seed=25)
    opts = ms.GaussNewtonSolverOptions(min_iterations=8 if line_search else 1, max_iterations=8 if line_search else 12, threshold=10.0,
                                       regularization=0.05, do_line_search=line_search, subset_line_search=subset)
    parity.check_solve(ch, efs, theta0, opts, param_tol=2e-4)


def test_solve_enabled_subset_and_block_sizes():
    ch, efs, theta0, theta_star = chain_problem(J=32, B=4, seed=26, families=("position", "state"))
    theta0 = theta_star + 0.1 * theta0
    en = np.ones(ch.num_params, bool); en[[1, 6, 9, 12, 30]] = False
    opts = ms.GaussNewtonSolverOptions(min_iterations=2, max_iterations=6, regularization=0.05)
    parity.check_solve(ch, efs, theta0, opts, enabled=en, param_tol=2e-4)


@pytest.mark.parametrize("mode", [ms.CHOLESKY_DENSE_EIGEN, ms.CHOLESKY_TILES_DENSE, ms.CHOLESKY_TILES_SPARSE])
@pytest.mark.parametrize("case", ["humanoid", "chain_state", "subset"])
def test_solve_cholesky_modes(case, mode):
    """Dense Eigen-structured LLT, and the level-scheduled tile Cholesky on the dense / min-degree sparse pattern."""
    enabled = None
    if case == "humanoid":
        ch, efs, theta0, _ = humanoid_problem(33, orientation=True)
        opts = ms.GaussNewtonSolverOptions(min_iterations=1, max_iterations=8, regularization=0.05, cholesky_mode=mode)
        inst = [0, 13, 32]
    elif case == "chain_state":
        ch, efs, theta0, theta_star = chain_problem(J=64, B=5, seed=51, families=("position", "state", "limit"))
        theta0 = theta_star + 0.02 * theta0  # a 64-joint chain is chaotic in float unless started near the targets
        opts = ms.GaussNewtonSolverOptions(min_iterations=2, max_iterations=5, regularization=0.05, cholesky_mode=mode)
        inst = [0, 1, 3, 4]  # instance 2 is chaotic: merely toggling FMA contraction on the CPU moves its objective by 0.4 %
    else:
        ch, efs, theta0, _ = humanoid_problem(9, orientation=True)
        enabled = np.ones(ch.num_params, bool); enabled[[0, 5, 6, 40, 41, 42, 100, 219]] = False
        opts = ms.GaussNewtonSolverOptions(min_iterations=1, max_iterations=6, regularization=0.05, cholesky_mode=mode)
        inst = [0, 8]
    out, worst = parity.check_solve(ch, efs, theta0, opts, enabled=enabled, param_tol=1e-4, instances=inst)
    assert np.all(out["status"] == 0)


def test_ka4_three_joint_ik_with_cholesky_breakdown():
    # momentum/test/character_solver/inverse_kinematics_test.cpp:38-123, float instantiation
    ch = mc.create_test_character(3)
    rng = np.random.default_rng(12345)
    tg = (rng.uniform(-1, 1, (10, 1, 3)) * 3).astype(np.float32)
    pos = mc.PositionErrorFunction(np.array([2], np.int32), np.array([[0.0, 1.0, 0.0]]), np.array([1.0]), tg)
    opts = ms.GaussNewtonSolverOptions(min_iterations=6, max_iterations=6, threshold=1.0, regularization=1e-7, use_block_jtj=True)
    out, _ = parity.check_solve(ch, [pos], np.zeros((10, ch.num_params), np.float32), opts, param_tol=5e-3)
    p = mc.world_points(ch, out["params"], [2], [[0, 1.0, 0]])[:, 0]
    assert np.all(np.linalg.norm(p - tg[:, 0], axis=1) <= 5e-5)
    assert np.all(out["errors"] <= 5e-7)


@pytest.mark.parametrize("mode", [ms.CHOLESKY_DENSE_EIGEN, ms.CHOLESKY_TILES_SPARSE])
def test_cholesky_breakdown_is_flagged_on_every_path(mode):
    """A pivot that is exactly zero (no damping, a parameter no constraint depends on). Eigen::LLT returns early and the reference ignores
    info() (gauss_newton_solver.cpp:251); the dense Eigen-structured kernel reproduces that and flags the instance; the tile schedule (the
    default from 48 unknowns) substitutes the damping for the pivot - zero here, so the step is not finite, the NaN guard of the batched
    caller (tensor_ik.cpp:168-173) restores the initial parameters. Either way the caller sees a non-zero status, never a silent wrong step."""
    ch, efs, theta0, _ = humanoid_problem(3, orientation=False)
    opts = ms.GaussNewtonSolverOptions(min_iterations=1, max_iterations=2, regularization=0.0, cholesky_mode=mode, fused_mode=ms.FUSED_OFF)
    out = ms.GaussNewtonSolver(opts, parity.build_function(ch, efs, 3)).solve(theta0)
    assert np.all(out["status"] != ms.INSTANCE_OK)
    if mode == ms.CHOLESKY_TILES_SPARSE:
        assert np.all(out["status"] == ms.INSTANCE_NON_FINITE) and np.array_equal(out["params"], theta0.astype(np.float32))
    else:
        # Eigen's early return leaves the trailing block unfactored; the substitutions then divide by the zero pivot, so an instance is either
        # flagged as a breakdown (finite step) or caught by the NaN guard (initial parameters restored)
        nf = out["status"] == ms.INSTANCE_NON_FINITE
        assert np.all((out["status"] == ms.INSTANCE_CHOLESKY_BREAKDOWN) | nf), out["status"]
        assert np.array_equal(out["params"][nf], theta0.astype(np.float32)[nf]) and np.all(np.isfinite(out["params"]))


def test_ka6_python_ik_basic_is_reached_and_deterministic():
    """pymomentum/test/test_solver2.py:135-199 on the CUDA path: joint positions reach the targets within 1e-4 and a second solve
    reproduces the error history and the parameters bit for bit (no atomics / no order-dependent sums on the data path)."""
    from tests.test_oracle_known_answers import _ka6_problem

    ch, ef, parents, offsets, targets = _ka6_problem()
    fn = parity.build_function(ch, [ef], 1)
    opts = ms.GaussNewtonSolverOptions(min_iterations=1, max_iterations=200, threshold=1.0, regularization=1e-5, store_error_history=True)
    solver = ms.GaussNewtonSolver(opts, fn)
    theta0 = np.zeros((1, ch.num_params))
    out = solver.solve(theta0)
    hist = solver.get_error_history()[0, : out["iterations"][0]]
    got = mc.world_points(ch, out["params"].astype(np.float64), parents, offsets)
    assert np.allclose(got, targets, rtol=1e-4, atol=1e-4)
    assert len(hist) > 1 and hist[-1] < hist[0]
    out2 = solver.solve(theta0)
    assert np.array_equal(solver.get_error_history()[0, : out2["iterations"][0]], hist) and np.array_equal(out["params"], out2["params"])
    # and on the tile-scheduled path (humanoid, Gram kernel + level-scheduled Cholesky)
    ch, efs, theta0, _ = humanoid_problem(16, orientation=True)
    fn = parity.build_function(ch, efs, 16)
    solver = ms.GaussNewtonSolver(ms.GaussNewtonSolverOptions(min_iterations=6, max_iterations=6, regularization=0.05, store_error_history=True), fn)
    a = solver.solve(theta0); ha = solver.get_error_history().copy()
    b = solver.solve(theta0); hb = solver.get_error_history()
    assert np.array_equal(a["params"], b["params"]) and np.array_equal(ha, hb)


@pytest.mark.parametrize("subset", [False, True])
def test_line_search_on_the_tile_scheduled_path(subset):
    """Armijo search with the strip layout / Gram kernel / tile Cholesky, with and without a disabled parameter subset."""
    ch, efs, theta0, _ = humanoid_problem(2, orientation=True)
    en = np.ones(ch.num_params, bool); en[[5, 17, 40, 41, 100, 150, 219]] = False
    opts = ms.GaussNewtonSolverOptions(min_iterations=5, max_iterations=5, threshold=1.0, regularization=0.05, do_line_search=True,
                                       subset_line_search=subset)
    parity.check_solve(ch, efs, theta0, opts)
    parity.check_solve(ch, efs, theta0, opts, enabled=en)


def test_cfg1_chain22():
    ch, efs, theta0, _ = chain22_problem()
    opts = ms.GaussNewtonSolverOptions(min_iterations=1, max_iterations=50, threshold=1.0, regularization=0.05)
    parity.check_solve(ch, efs, theta0, opts, param_tol=2e-4)


@pytest.mark.parametrize("orientation", [False, True])
def test_cfg2_cfg3_humanoid_converged_parameters(orientation):
    # cfg2 (24 Position, m=72) / cfg3 (+6 Orientation, m=126) at a size the oracle finishes in seconds
    # Every one of the 96 instances is compared at the stated 1e-4 against the FLOAT oracle. These under-determined problems (m < n)
    # are still creeping along their weakly constrained directions after 50 damped iterations, and on a few of them float rounding
    # alone moves the reference by ~1e-4 (scripts/parity_survey.py): such an instance must be as close to
    # the DOUBLE oracle as the reference's float build is, and at most 8 of the 96 may need that second look.
    B = 96
    ch, efs, theta0, _ = humanoid_problem(B, orientation=orientation)
    opts = ms.GaussNewtonSolverOptions(min_iterations=1, max_iterations=50, threshold=1.0, regularization=0.05)
    out, worst = parity.check_solve(ch, efs, theta0, opts, strict_double=True, max_calibrated=8)
    assert np.all(out["status"] == 0)
    print("max rel param diff", worst)


def test_cfg4_bodyhands_solve():
    # cfg4 (300 joints, n = 424, 200 markers): 32 instances, all compared at 1e-4 against the float oracle, convergence mode. None of them has converged
    # after 50 iterations, so rounding differences between two correct float implementations show at the 1e-4 level on a few instances: at
    # most 4 may need the strict second look of parity.check_solve (as close to the double oracle as the reference's float build is reproducible).
    ch, efs, theta0, _ = bodyhands_problem(32)
    opts = ms.GaussNewtonSolverOptions(min_iterations=1, max_iterations=50, threshold=1.0, regularization=0.05)
    out, worst = parity.check_solve(ch, efs, theta0, opts, strict_double=True, max_calibrated=4)
    assert np.all(out["status"] == 0)
    print("cfg4 max rel param diff", worst)


def test_cfg5_mixed_rigs_on_concurrent_streams():
    """cfg5: a mixed-rig batch is one solver function per rig; the handles are independent, so three rigs in flight on three CUDA
    streams must give bit-identical results to running them one after the other (no shared mutable state between handles)."""
    import torch

    groups = [chain22_problem(), humanoid_problem(40, orientation=True)[:4], bodyhands_problem(4)]
    opts = ms.GaussNewtonSolverOptions(min_iterations=1, max_iterations=6, threshold=1.0, regularization=0.05)
    runs = []
    for ch, efs, theta0, _ in groups:
        fn = parity.build_function(ch, efs, theta0.shape[0])
        runs.append((fn, ms.GaussNewtonSolver(opts, fn), theta0.astype(np.float32)))
    sequential = [solver.solve(theta0.copy()) for _, solver, theta0 in runs]
    streams = [torch.cuda.Stream() for _ in runs]
    dev = [torch.from_numpy(theta0).cuda() for _, _, theta0 in runs]
    torch.cuda.synchronize()
    for (fn, solver, _), st, th in zip(runs, streams, dev):
        solver.solve_device(th.data_ptr(), st.cuda_stream)  # no synchronisation in between: the three solves overlap
    torch.cuda.synchronize()
    for (fn, solver, _), th, ref in zip(runs, dev, sequential):
        res = solver.get_results()
        assert np.array_equal(th.cpu().numpy(), ref["params"])
        assert np.array_equal(res["errors"], ref["errors"]) and np.array_equal(res["iterations"], ref["iterations"])


@pytest.mark.parametrize("case", ["cfg3", "cfg2_odd_batch", "chain_all_families", "subset"])
def test_fused_kernels_match_the_three_kernel_path(case):
    """Gram + Cholesky in one launch (the default on the tile path) and the persistent whole-solve kernel run the same device functions
    as the three-kernel path. Gram + Cholesky is bit-identical to it (same code, only the tile hand-off differs: shared memory instead of HBM);
    the persistent kernel agrees to float rounding (its sweep is compiled in another context: different FMA contraction)."""
    enabled, kw = None, dict(min_iterations=6, max_iterations=6)
    if case == "cfg3":
        ch, efs, theta0, _ = humanoid_problem(70, orientation=True)
    elif case == "cfg2_odd_batch":  # fewer instances than one CTA's groups on some SMs, batch not a multiple of anything
        ch, efs, theta0, _ = humanoid_problem(5, orientation=False)
    elif case == "chain_all_families":
        ch, efs, theta0, ts = chain_problem(J=20, B=3, seed=33, families=("position", "orientation", "state", "limit", "plane", "halfplane", "model_parameters"))
        theta0 = ts + 0.05 * theta0
        kw = dict(min_iterations=1, max_iterations=5, cholesky_mode=ms.CHOLESKY_TILES_SPARSE)
    else:
        ch, efs, theta0, _ = humanoid_problem(9, orientation=True)
        enabled = np.ones(ch.num_params, bool); enabled[[0, 5, 6, 40, 41, 42, 100, 219]] = False
    fn = parity.build_function(ch, efs, theta0.shape[0], enabled=enabled)
    res = {}
    for fm, code in ((ms.FUSED_OFF, 0), (ms.FUSED_GRAM_CHOLESKY, 2), (ms.FUSED_AUTO, 1), (ms.FUSED_PERSISTENT, 1)):  # AUTO: these batches are a single wave
        solver = ms.GaussNewtonSolver(ms.GaussNewtonSolverOptions(regularization=0.05, fused_mode=fm, store_error_history=True, **kw), fn)
        out = solver.solve(theta0)
        assert solver.get_fused_profile()["fused"] == code
        res[fm] = (out, solver.get_error_history())
    (a, ha), (b, hb), (c, hc), (d, hd) = res[ms.FUSED_OFF], res[ms.FUSED_GRAM_CHOLESKY], res[ms.FUSED_AUTO], res[ms.FUSED_PERSISTENT]
    for x, hx, o, h in ((a, ha, b, hb), (d, hd, c, hc)):  # three kernels == Gram + Cholesky; AUTO == persistent
        assert np.array_equal(x["params"], o["params"]) and np.array_equal(x["iterations"], o["iterations"]) and np.array_equal(x["status"], o["status"])
        assert np.array_equal(x["errors"], o["errors"]) and np.array_equal(hx, h)
    assert np.array_equal(a["status"], d["status"]) and np.all(np.abs(a["iterations"].astype(int) - d["iterations"]) <= 1)
    scale = np.maximum(1.0, np.abs(a["params"]).max(axis=1, keepdims=True))
    assert np.max(np.abs(a["params"] - d["params"]) / scale) <= 5e-4   # a few GN iterations amplify rounding-level differences
    assert np.allclose(a["errors"], d["errors"], rtol=2e-3, atol=1e-9)


def test_persistent_kernel_against_the_oracle():
    """The whole-solve kernel through the same converged-parameter check as every other path (float oracle, 1e-4)."""
    ch, efs, theta0, _ = humanoid_problem(24, orientation=True)
    opts = ms.GaussNewtonSolverOptions(min_iterations=1, max_iterations=50, threshold=1.0, regularization=0.05, fused_mode=ms.FUSED_PERSISTENT)
    out, worst = parity.check_solve(ch, efs, theta0, opts, strict_double=True, max_calibrated=3)
    assert np.all(out["status"] == 0)
    ch, efs, theta0, ts = chain_problem(J=20, B=3, seed=33, families=("position", "orientation", "state", "limit", "plane", "halfplane", "model_parameters"))
    opts = ms.GaussNewtonSolverOptions(min_iterations=1, max_iterations=5, threshold=1.0, regularization=0.05, cholesky_mode=ms.CHOLESKY_TILES_SPARSE,
                                       fused_mode=ms.FUSED_PERSISTENT)
    parity.check_solve(ch, efs, ts + 0.05 * theta0, opts, param_tol=3e-4)


def test_fused_modes_reject_what_they_cannot_run():
    ch, efs, theta0, _ = humanoid_problem(4, orientation=True)
    fn = parity.build_function(ch, efs, 4)
    for fm in (ms.FUSED_PERSISTENT, ms.FUSED_GRAM_CHOLESKY):
        for kw in (dict(cholesky_mode=ms.CHOLESKY_DENSE_EIGEN), dict(jtj_mode=ms.JTJ_FP32_SIMT)):
            with pytest.raises(ms.MomentumB200Error):
                ms.GaussNewtonSolver(ms.GaussNewtonSolverOptions(max_iterations=3, fused_mode=fm, **kw), fn).solve(theta0)
    with pytest.raises(ms.MomentumB200Error):
        ms.GaussNewtonSolver(ms.GaussNewtonSolverOptions(max_iterations=3, fused_mode=ms.FUSED_PERSISTENT, do_line_search=True), fn).solve(theta0)
    ch, efs, theta0, _ = bodyhands_problem(2)  # 122 tiles + 155 KB of strips: neither fused kernel fits -> three kernels under AUTO
    fn = parity.build_function(ch, efs, 2)
    solver = ms.GaussNewtonSolver(ms.GaussNewtonSolverOptions(max_iterations=2), fn)
    solver.solve(theta0)
    assert solver.get_fused_profile()["fused"] == 0
    # AUTO at a batch larger than one wave of instance groups: Gram + Cholesky per iteration
    ch, efs, theta0, _ = humanoid_problem(600, orientation=True)
    fn = parity.build_function(ch, efs, 600)
    solver = ms.GaussNewtonSolver(ms.GaussNewtonSolverOptions(max_iterations=2), fn)
    solver.solve(theta0)
    assert solver.get_fused_profile()["fused"] == 2


@pytest.mark.parametrize("case", ["chain_all_families", "chain_subset_line_search", "humanoid", "bodyhands_too_wide"])
def test_gauss_newton_qr_step(case):
    """SURVEY 8(f) rank 3: GaussNewtonSolverQRT's step (online Householder QR of [sqrt(lambda) I; J], gauss_newton_solver_qr.cpp:50-150) as
    the device linear solver, against the oracle's restatement of that solver (oracle: KA-9 / KA-10)."""
    if case == "chain_all_families":
        ch, efs, theta0, ts = chain_problem(J=6, B=5, seed=81, families=("position", "orientation", "state", "limit", "plane", "halfplane", "model_parameters"))
        opts = ms.GaussNewtonSolverOptions(min_iterations=6, max_iterations=6, threshold=10.0, regularization=0.05, linear_solver=ms.LINEAR_SOLVER_QR)
        parity.check_solve(ch, efs, ts + 0.1 * theta0, opts, param_tol=2e-4)
    elif case == "chain_subset_line_search":
        ch, efs, theta0, _ = chain_problem(J=6, B=4, seed=82)
        en = np.ones(ch.num_params, bool); en[[0, 2, 5, 8]] = False
        opts = ms.GaussNewtonSolverOptions(min_iterations=6, max_iterations=6, threshold=10.0, regularization=0.05, do_line_search=True, subset_line_search=True,
                                           linear_solver=ms.LINEAR_SOLVER_QR)
        parity.check_solve(ch, efs, theta0, opts, enabled=en, param_tol=2e-4)
    elif case == "humanoid":
        ch, efs, theta0, _ = humanoid_problem(12, orientation=True)
        opts = ms.GaussNewtonSolverOptions(min_iterations=1, max_iterations=30, threshold=1.0, regularization=0.05, linear_solver=ms.LINEAR_SOLVER_QR)
        out, worst = parity.check_solve(ch, efs, theta0, opts, strict_double=True, max_calibrated=2)
        assert np.all(out["status"] == 0)
        # and the two linear solvers agree with each other (same normal equations)
        chol = ms.GaussNewtonSolver(ms.GaussNewtonSolverOptions(min_iterations=1, max_iterations=30, threshold=1.0, regularization=0.05), parity.build_function(ch, efs, 12)).solve(theta0)
        assert np.max(np.abs(chol["params"] - out["params"])) <= 1e-3
    else:
        ch, efs, theta0, _ = bodyhands_problem(2)  # n = 424: R alone is 360 KB
        fn = parity.build_function(ch, efs, 2)
        with pytest.raises(ms.MomentumB200Error):
            ms.GaussNewtonSolver(ms.GaussNewtonSolverOptions(max_iterations=2, linear_solver=ms.LINEAR_SOLVER_QR), fn).solve(theta0)


@pytest.mark.parametrize("case", ["chain_all_families", "chain_subset", "humanoid", "far_start"])
def test_trust_region_qr(case):
    """SURVEY 8(f) rank 3, second half: TrustRegionQRT (trust_region_qr.cpp:52-270) as a device iteration - QR of J, the damping search that
    keeps the step inside the radius, rho-driven radius, rejected steps - against the oracle's restatement (KA-11)."""
    TR = ms.LINEAR_SOLVER_TRUST_REGION_QR
    if case == "chain_all_families":
        ch, efs, theta0, ts = chain_problem(J=6, B=5, seed=81, families=("position", "orientation", "state", "limit", "plane", "halfplane", "model_parameters"))
        opts = ms.GaussNewtonSolverOptions(min_iterations=6, max_iterations=6, threshold=10.0, linear_solver=TR)
        parity.check_solve(ch, efs, ts + 0.1 * theta0, opts, param_tol=2e-4)
    elif case == "chain_subset":
        ch, efs, theta0, _ = chain_problem(J=6, B=4, seed=82)
        en = np.ones(ch.num_params, bool); en[[0, 2, 5, 8]] = False
        opts = ms.GaussNewtonSolverOptions(min_iterations=6, max_iterations=6, threshold=10.0, linear_solver=TR, trust_region_radius=0.5)
        parity.check_solve(ch, efs, theta0, opts, enabled=en, param_tol=2e-4)
    elif case == "humanoid":  # n = 220: R and the damping rows fill 194 KB of shared memory
        # (the cfg3 constraint set is under-determined, 126 rows for 220 parameters: with its 1e-10 diagonal the reference's trust-region
        # solver rejects every step there - oracle and device agree on that too; the reference's own tests are well-determined, as here)
        ch, _, theta0, theta_star = humanoid_problem(4, orientation=True)
        J = ch.num_joints
        joints = np.arange(J, dtype=np.int32)
        ident = np.tile([0.0, 0.0, 0.0, 1.0], (J, 1))
        pose = 0.5 * theta_star
        efs = [mc.PositionErrorFunction(joints, np.zeros((J, 3)), np.ones(J), mc.world_points(ch, pose, joints, np.zeros((J, 3))), weight=1.0),
               mc.OrientationErrorFunction(joints, ident, np.ones(J), mc.world_rotations(ch, pose, joints, ident), weight=1.0)]
        opts = ms.GaussNewtonSolverOptions(min_iterations=4, max_iterations=10, threshold=10.0, linear_solver=TR)
        out, worst = parity.check_solve(ch, efs, theta0[:4], opts, param_tol=2e-4)
        assert np.all(out["status"] == 0)
        # the reference's own property (solver_test.cpp:172-233, SanityCheck: a Position and an Orientation constraint on every joint):
        # the trust-region solver does at least as well as Gauss-Newton
        fn = parity.build_function(ch, efs, 4)
        gn = ms.GaussNewtonSolver(ms.GaussNewtonSolverOptions(min_iterations=4, max_iterations=10, threshold=10.0, regularization=0.05), fn).solve(theta0[:4])
        e_tr, e_gn = fn.get_error(out["params"]), fn.get_error(gn["params"])
        assert np.all(e_tr <= 1.001 * e_gn + 0.001), (e_tr, e_gn)
        assert np.all(e_tr < 0.05 * fn.get_error(theta0[:4]))
    else:  # a chain that starts far from its targets: the radius binds, steps get damped and some are rejected
        ch, efs, theta0, _ = chain_problem(J=8, B=6, seed=5, families=("position",))
        opts = ms.GaussNewtonSolverOptions(min_iterations=8, max_iterations=8, threshold=1.0, linear_solver=TR, store_error_history=True)
        fn = parity.build_function(ch, efs, 6)
        solver = ms.GaussNewtonSolver(opts, fn)
        out = solver.solve(theta0)
        hist = solver.get_error_history()
        assert np.all(hist[:, 1:] <= hist[:, :-1] * (1 + 1e-5) + 1e-9)  # a step that does not decrease the error is rejected
        # accept / reject decisions make this path discontinuous: here the reference's own float and double builds end O(1) apart (measured:
        # float-vs-double gap 0.004 - 1.25 in the parameters, already 0.1 after ONE iteration, which holds up to ten accept / reject
        # decisions), so the iterates are not comparable point by point; the progress both make is
        from oracle.binding import OracleFunction
        e_dev, e0 = fn.get_error(out["params"]), fn.get_error(theta0)
        for b in range(6):
            _, p, _, _ = OracleFunction(ch, efs, "float32", instance=b).solve(theta0[b], min_iterations=8, max_iterations=8, threshold=1.0, trust_region_qr=True)
            e_orc = OracleFunction(ch, efs, "float32", instance=b).get_error(p)
            print(f"far start, instance {b}: error {e0[b]:.4g} -> device {e_dev[b]:.4g}, oracle {e_orc:.4g}")
            assert e_dev[b] < 0.5 * e0[b] and e_dev[b] <= 10.0 * e_orc + 1e-2 * e0[b], (b, e_dev[b], e_orc, e0[b])


def test_full_size_properties_cfg3_shard():
    """BASELINE cfg3 per-GPU shard (8192 x humanoid72, m=126): properties that need no oracle."""
    B = 8192
    ch, efs, theta0, theta_star = humanoid_problem(B, orientation=True)
    fn = parity.build_function(ch, efs, B)
    e0 = fn.get_error(theta0)
    opts = ms.GaussNewtonSolverOptions(min_iterations=1, max_iterations=30, threshold=1.0, regularization=0.05, store_error_history=True)
    solver = ms.GaussNewtonSolver(opts, fn)
    out = solver.solve(theta0)
    assert np.all(out["status"] == 0) and np.all(np.isfinite(out["params"]))
    e1 = fn.get_error(out["params"])
    assert np.all(e1 < 0.5 * e0) and np.median(e1 / e0) < 1e-3   # reachable targets: objective collapses (damped GN: linear rate, a few slow instances)
    hist = solver.get_error_history()
    for b in range(0, B, 511):                                   # history is monotone for damped GN here
        h = hist[b, : out["iterations"][b]]
        assert np.all(np.diff(h) <= 1e-6 * h[:-1] + 1e-9)
    # idempotence: solving again from the solution changes nothing measurable
    out2 = ms.GaussNewtonSolver(ms.GaussNewtonSolverOptions(min_iterations=1, max_iterations=3, regularization=0.05), fn).solve(out["params"])
    e2 = fn.get_error(out2["params"])
    assert np.all(e2 <= e1 * (1 + 1e-3) + 1e-9)                  # continuing from the solution never makes it worse
    # permutation equivariance: instance b of a shuffled batch gives bit-identical parameters
    perm = np.random.default_rng(0).permutation(B)
    efs_p = [type(e)(**{**e.__dict__, "targets": np.asarray(e.targets)[perm]}) for e in efs]
    fn_p = parity.build_function(ch, efs_p, B)
    out_p = ms.GaussNewtonSolver(opts, fn_p).solve(theta0[perm])
    assert np.array_equal(out_p["params"], out["params"][perm])


def test_per_instance_constraint_weights_and_zero_weight_skip():
    ch, efs, theta0, _ = chain_problem(J=6, B=4, seed=31, families=("position",))
    fn = parity.build_function(ch, efs, 4)
    w = np.tile(np.asarray(efs[0].weights, np.float32), (4, 1))
    w[1, 0] = 0.0; w[2, :] *= 2.0
    fn.set_constraint_weights(0, w, per_instance=True)
    e = fn.get_error(theta0)
    from oracle.binding import OracleFunction
    import copy
    for b in range(4):
        ef = copy.copy(efs[0]); ef.weights = w[b]
        orc = OracleFunction(ch, [ef], "float32", instance=b)
        assert abs(orc.get_error(parity.f32(theta0[b])) - e[b]) <= 2e-5 * max(1, e[b])


def test_non_finite_input_reverts_to_initial_guess():
    # batched caller's guard, pymomentum/tensor_ik/tensor_ik.cpp:168-173
    ch, efs, theta0, _ = chain_problem(J=5, B=3, seed=33, families=("position",))
    efs[0].targets = np.asarray(efs[0].targets).copy(); efs[0].targets[1, 0, 0] = np.nan
    fn = parity.build_function(ch, efs, 3)
    out = ms.GaussNewtonSolver(ms.GaussNewtonSolverOptions(max_iterations=4), fn).solve(theta0)
    assert out["status"][1] == ms.INSTANCE_NON_FINITE and np.array_equal(out["params"][1], theta0[1].astype(np.float32))
    assert out["status"][0] == 0 and out["status"][2] == 0
