"""CPU lane-emulation of the device building blocks (tests/emu) vs the oracle.

Validates, without a GPU: the planner (units / cells / chain-rule contributions / gating), the
per-lane FK + residual + Jacobian code, the Eigen-structured blocked Cholesky phases and the batched
solve loop — i.e. everything in momentum_b200/csrc that is not CUDA launch glue."""
import numpy as np
import pytest

from momentum_b200 import character as mc
from momentum_b200 import solver as ms
from momentum_b200.problems import chain_problem, chain22_problem, humanoid_problem
from tests import emu_lib
from tests import parity
from tests.emu_lib import EMU_LIB


@pytest.fixture(scope="module", autouse=True)
def _build_emu():
    emu_lib.build()


FAMS = [("position",), ("orientation",), ("state",), ("limit",), ("position", "orientation", "state", "limit"), ("plane",), ("halfplane",),
        ("model_parameters",), ("position", "limit", "plane", "halfplane", "model_parameters")]


@pytest.mark.parametrize("fams", FAMS)
def test_single_iteration_families(fams):
    ch, efs, theta0, _ = chain_problem(J=6, B=3, seed=21, families=fams)
    parity.check_fk(ch, efs, theta0, EMU_LIB)
    parity.check_single_iteration(ch, efs, theta0, EMU_LIB)


@pytest.mark.parametrize("logmap,rot_diff", [(True, False), (False, True)])
def test_single_iteration_logmap_rotdiff(logmap, rot_diff):
    ch, efs, theta0, _ = chain_problem(J=7, B=2, seed=22, families=("orientation", "state"), logmap=logmap, rot_diff=rot_diff)
    parity.check_single_iteration(ch, efs, theta0, EMU_LIB)


@pytest.mark.parametrize("alpha,c", [(mc.LOSS_L1, 0.7), (mc.LOSS_CAUCHY, 1.3), (mc.LOSS_WELSCH, 0.9), (-2.0, 1.1), (1.5, 0.8)])
def test_single_iteration_generalized_loss(alpha, c):
    ch, efs, theta0, _ = chain_problem(J=5, B=2, seed=23, families=("position", "orientation", "limit"), loss=(alpha, c))
    parity.check_single_iteration(ch, efs, theta0, EMU_LIB)


def test_single_iteration_enabled_subset():
    ch, efs, theta0, _ = chain_problem(J=6, B=2, seed=24)
    en = np.ones(ch.num_params, bool); en[[0, 2, 5, 8, ch.num_params - 1]] = False
    parity.check_single_iteration(ch, efs, theta0, EMU_LIB, enabled=en)


def test_plane_and_model_parameters_with_enabled_subset_and_solve():
    """The two 'next' error functions of SURVEY 8(f): Plane (half-plane mode included) and ModelParameters, with a disabled
    parameter subset (ModelParameters packs its rows over the enabled parameters) and through a full solve."""
    ch, efs, theta0, _ = chain_problem(J=6, B=3, seed=31, families=("position", "plane", "halfplane", "model_parameters"))
    en = np.ones(ch.num_params, bool); en[[1, 4, 9]] = False
    parity.check_single_iteration(ch, efs, theta0, EMU_LIB, enabled=en)
    opts = ms.GaussNewtonSolverOptions(min_iterations=1, max_iterations=10, threshold=10.0, regularization=0.05)
    parity.check_solve(ch, efs, theta0, opts, EMU_LIB, param_tol=2e-4)
    parity.check_solve(ch, efs, theta0, opts, EMU_LIB, enabled=en, param_tol=2e-4)
    # negative target weights: no Jacobian row (model_parameters_error_function.cpp:113) but getError counts them (:56-59); the line
    # search is the consumer of that asymmetry
    tw = np.asarray(efs[-1].target_weights, np.float64).copy(); tw[[0, 3, 7]] = [-0.7, -1.2, -0.4]
    efs[-1] = mc.ModelParametersErrorFunction(tw, efs[-1].targets, weight=0.6)
    parity.check_single_iteration(ch, efs, theta0, EMU_LIB)
    parity.check_single_iteration(ch, efs, theta0, EMU_LIB, enabled=en)
    ls = ms.GaussNewtonSolverOptions(min_iterations=4, max_iterations=4, threshold=10.0, regularization=0.05, do_line_search=True)
    parity.check_solve(ch, efs, theta0, ls, EMU_LIB, param_tol=2e-4)


def test_all_families_on_the_tile_scheduled_path():
    """Every error-function family at once through the strip layout / tile-sparse Gram / tile Cholesky: multi-row units own their row
    quads, one-row units (limits, planes, model parameters) share quads without coupling each other's tile columns."""
    ch, efs, theta0, ts = chain_problem(J=20, B=2, seed=33, families=("position", "orientation", "state", "limit", "plane", "halfplane", "model_parameters"))
    theta0 = ts + 0.05 * theta0
    opts = ms.GaussNewtonSolverOptions(min_iterations=1, max_iterations=5, threshold=1.0, regularization=0.05, cholesky_mode=ms.CHOLESKY_TILES_SPARSE)
    parity.check_solve(ch, efs, theta0, opts, EMU_LIB, param_tol=3e-4)


def test_edge_cases_empty_and_degenerate_inputs():
    parity.check_edge_cases(EMU_LIB)


def test_ka6_python_ik_basic_through_the_device_code():
    """pymomentum/test/test_solver2.py:135-199 on the emulated device path: joint positions reach the targets within 1e-4 and a second
    solve reproduces the error history bit for bit."""
    from tests.test_oracle_known_answers import _ka6_problem

    ch, ef, parents, offsets, targets = _ka6_problem()
    fn = parity.build_function(ch, [ef], 1, EMU_LIB)
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


@pytest.mark.parametrize("subset", [False, True])
def test_line_search_on_the_tile_scheduled_path(subset):
    """Armijo search (gauss_newton_solver.cpp:283-313 / subset_gauss_newton_solver.cpp:119-141) with the strip layout: the step lives in
    device-column order with alignment gaps, the trial update maps it back through the column table."""
    ch, efs, theta0, _ = humanoid_problem(2, orientation=True)
    en = np.ones(ch.num_params, bool); en[[5, 17, 40, 41, 100, 150, 219]] = False
    opts = ms.GaussNewtonSolverOptions(min_iterations=5, max_iterations=5, threshold=1.0, regularization=0.05, do_line_search=True,
                                       subset_line_search=subset)
    parity.check_solve(ch, efs, theta0, opts, EMU_LIB)
    parity.check_solve(ch, efs, theta0, opts, EMU_LIB, enabled=en)


def test_humanoid_single_iteration():
    ch, efs, theta0, theta_star = humanoid_problem(2, orientation=True)
    th = (theta0 + 0.3 * theta_star).astype(np.float32)
    parity.check_single_iteration(ch, efs, th, EMU_LIB)


@pytest.mark.parametrize("line_search,subset", [(False, False), (True, False), (True, True)])
def test_solve_chain_all_families(line_search, subset):
    ch, efs, theta0, _ = chain_problem(J=6, B=3, seed=25)
    # fixed iteration count with line search: the relative-change stop (solver.cpp:98-101) sits at the
    # float rounding floor there, so iteration counts are only comparable without it
    opts = ms.GaussNewtonSolverOptions(min_iterations=8 if line_search else 1, max_iterations=8 if line_search else 12, threshold=10.0,
                                       regularization=0.05, do_line_search=line_search, subset_line_search=subset)
    parity.check_solve(ch, efs, theta0, opts, EMU_LIB, param_tol=2e-4)


def test_solve_enabled_subset_and_block_sizes():
    # n = 39 -> Eigen block size 8 (blocked LLT path), with a non-contiguous enabled set
    ch, efs, theta0, theta_star = chain_problem(J=32, B=2, seed=26, families=("position", "state"))
    theta0 = theta_star + 0.1 * theta0  # start near the targets: a 32-joint chain far from them is chaotic in float
    en = np.ones(ch.num_params, bool); en[[1, 6, 9, 12, 30]] = False
    opts = ms.GaussNewtonSolverOptions(min_iterations=2, max_iterations=6, regularization=0.05)
    parity.check_solve(ch, efs, theta0, opts, EMU_LIB, enabled=en, param_tol=2e-4)


def test_solve_humanoid_blocked_cholesky():
    ch, efs, theta0, _ = humanoid_problem(2, orientation=True)
    opts = ms.GaussNewtonSolverOptions(min_iterations=1, max_iterations=6, regularization=0.05)
    out, worst = parity.check_solve(ch, efs, theta0, opts, EMU_LIB)
    assert np.all(out["status"] == 0)


@pytest.mark.parametrize("mode", [ms.CHOLESKY_TILES_DENSE, ms.CHOLESKY_TILES_SPARSE])
@pytest.mark.parametrize("case", ["humanoid", "chain_state", "subset"])
def test_solve_tile_scheduled_cholesky(case, mode):
    """Level-scheduled tile Cholesky (dense pattern and min-degree sparse pattern) vs the oracle's Eigen-style LLT."""
    enabled = None
    if case == "humanoid":
        ch, efs, theta0, _ = humanoid_problem(2, orientation=True)
        opts = ms.GaussNewtonSolverOptions(min_iterations=1, max_iterations=6, regularization=0.05, cholesky_mode=mode)
    elif case == "chain_state":  # n = 71: dense-ish pattern (state terms couple every ancestor pair), 5 tile columns
        ch, efs, theta0, theta_star = chain_problem(J=64, B=2, seed=51, families=("position", "state", "limit"))
        theta0 = theta_star + 0.02 * theta0  # a 64-joint chain is chaotic in float unless started near the targets
        opts = ms.GaussNewtonSolverOptions(min_iterations=2, max_iterations=5, regularization=0.05, cholesky_mode=mode)
    else:
        ch, efs, theta0, _ = humanoid_problem(2, orientation=True)
        enabled = np.ones(ch.num_params, bool); enabled[[0, 5, 6, 40, 41, 42, 100, 219]] = False
        opts = ms.GaussNewtonSolverOptions(min_iterations=1, max_iterations=6, regularization=0.05, cholesky_mode=mode)
    out, worst = parity.check_solve(ch, efs, theta0, opts, EMU_LIB, enabled=enabled, param_tol=1e-4)
    assert np.all(out["status"] == 0)


def test_ka4_three_joint_ik_with_cholesky_breakdown():
    # inverse_kinematics_test.cpp:38-123 in float: regularization 1e-7 makes LLT hit a zero pivot;
    # the solver must behave like Eigen's early-exit LLT (status flags the breakdown, result still fine).
    ch = mc.create_test_character(3)
    rng = np.random.default_rng(12345)
    tg = (rng.uniform(-1, 1, (10, 1, 3)) * 3).astype(np.float32)
    pos = mc.PositionErrorFunction(np.array([2], np.int32), np.array([[0.0, 1.0, 0.0]]), np.array([1.0]), tg)
    opts = ms.GaussNewtonSolverOptions(min_iterations=6, max_iterations=6, threshold=1.0, regularization=1e-7, use_block_jtj=True)
    out, _ = parity.check_solve(ch, [pos], np.zeros((10, ch.num_params), np.float32), opts, EMU_LIB, param_tol=5e-3, compare_history=True)
    p = mc.world_points(ch, out["params"], [2], [[0, 1.0, 0]])[:, 0]
    assert np.all(np.linalg.norm(p - tg[:, 0], axis=1) <= 5e-5)
    assert np.all(out["errors"] <= 5e-7)


def test_chain22_cfg1():
    ch, efs, theta0, _ = chain22_problem()
    opts = ms.GaussNewtonSolverOptions(min_iterations=1, max_iterations=50, threshold=1.0, regularization=0.05)
    parity.check_solve(ch, efs, theta0, opts, EMU_LIB, param_tol=2e-4)


@pytest.mark.parametrize("n", [1, 8, 9, 16, 17, 31, 32, 127, 128, 231, 232, 255, 256])
def test_dense_cholesky_backward_error(n):
    """One Gauss-Newton step through the dense Eigen-structured Cholesky at every block size (tests/f64ref.py: normwise backward error
    against the float64 normal equations of the emulator's own float Jacobian). The emulator factors on the host, so the kernel's
    shared / global memory branch and the TF32 JtJ modes are GPU-only (tests/test_gpu_kernel_bounds.py). The emulator runs the path the
    library's chooseSolvePath picks (tests/test_solve_path.py asserts which); the explicit cholesky_mode pins it to the dense kernel."""
    from tests import f64ref as R

    if n < 10:
        ch, efs, _ = R.chain_case(10, positions=3, seed=n)
        en = np.zeros(10, bool); en[:n] = True
    else:
        ch, efs, _ = R.chain_case(n, positions=min(n - 7, 12), seed=n)
        en = None
    opts = ms.GaussNewtonSolverOptions(min_iterations=1, max_iterations=1, regularization=0.05, cholesky_mode=ms.CHOLESKY_DENSE_EIGEN)
    _, out, J, r, cols, delta, lam = R.one_step(ch, efs, np.zeros((1, ch.num_params)), opts, EMU_LIB, en, rel_damping=1e-5)
    assert np.all(out["status"] == 0) and len(cols) == n
    be = R.backward_error(J[0], r[0], cols, delta[0], lam)
    assert be <= R.solve_limit(n), (n, be, R.solve_limit(n))


@pytest.mark.parametrize("chol", [ms.CHOLESKY_TILES_DENSE, ms.CHOLESKY_TILES_SPARSE])
@pytest.mark.parametrize("jtj", [ms.JTJ_SPARSE_TILES, ms.JTJ_FP32_SIMT])
@pytest.mark.parametrize("rig", ["humanoid", "humanoid_subset", "chain240"])
def test_tile_cholesky_backward_error(rig, jtj, chol):
    """The level-scheduled tile Cholesky fed by the tile-sparse Gram and by the K-major JtJ, same bound as the dense kernel. The
    240-parameter chain is a long system whose dense tile schedule still fits in shared memory; the 330-parameter chain's does not,
    and the library, and with it the emulator, refuses the explicit tile modes there (tests/test_solve_path.py). The explicit modes decide the path;
    the 256 / 512-thread variants and the QR step are GPU-only."""
    from tests import f64ref as R

    en = None
    if rig == "chain240":
        ch, efs, _ = R.chain_case(240, positions=12, seed=240)
    else:
        ch, efs, _, _ = humanoid_problem(1, orientation=True)
        if rig == "humanoid_subset":
            en = np.ones(ch.num_params, bool); en[[0, 5, 6, 40, 41, 42, 100, 219]] = False
    opts = ms.GaussNewtonSolverOptions(min_iterations=1, max_iterations=1, regularization=0.05, cholesky_mode=chol, jtj_mode=jtj)
    _, out, J, r, cols, delta, lam = R.one_step(ch, efs, np.zeros((1, ch.num_params)), opts, EMU_LIB, en, rel_damping=1e-5)
    assert np.all(out["status"] == 0)
    be = R.backward_error(J[0], r[0], cols, delta[0], lam)
    assert be <= R.solve_limit(len(cols), "tiles"), (be, R.solve_limit(len(cols), "tiles"))


def test_solver_plan_figures_humanoid_and_bodyhands():
    """Host planning of the solver path: elimination order + tile schedule + device-column layout + Gram plan. Guards the
    structural invariants the kernels rely on and the schedule quality reached in round 1 (levels / tiles of humanoid72)."""
    import ctypes as C

    from momentum_b200.problems import bodyhands_problem

    for make, max_levels, max_tiles in ((lambda: humanoid_problem(2, orientation=True), 4, 55), (lambda: bodyhands_problem(2), 9, 130)):
        ch, efs, _, _ = make()
        fn = ms.SkeletonSolverFunction(ch, 2, efs, lib_path=EMU_LIB)
        out = (C.c_int64 * 10)()
        assert fn._L.emu_plan_figures(fn._h, out) == 0
        levels, tiles, tile_cols, n_pad, dev_cols, strips, pairs, misaligned, odd, outside = list(out)
        assert levels <= max_levels and tiles <= max_tiles, (levels, tiles)
        assert n_pad == 16 * tile_cols and dev_cols >= ch.num_params and dev_cols <= ch.num_params + 3 * tile_cols
        assert misaligned == 0  # every tile column starts on a device column that is a multiple of 4 (TMA box alignment)
        assert odd == 0         # pair lists are consumed two at a time
        assert outside == 0     # every Jacobian cell lands inside the strip of its (row quad, tile column)
        assert strips > 0 and pairs >= strips
        # what the sweep kernel's 16-byte strip stores rely on: joint units start on a row quad and own their padding rows, cells sit at
        # 16-byte aligned strip offsets in (kind, unit, device column) order
        inv = (C.c_int64 * 6)()
        assert fn._L.emu_store_invariants(fn._h, inv) == 0
        off_quad, overlap, unaligned, disorder, multi, cells = list(inv)
        assert multi > 0 and cells > 0 and off_quad == 0 and overlap == 0 and unaligned == 0 and disorder == 0, list(inv)
