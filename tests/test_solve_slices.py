"""Instance slices of a solve: on the Gram + Cholesky path a batch of at least kSliceMinWaves (4) waves of resident gramCholeskyKernel
CTAs runs as two slices, each with its own chain of sweep + gramCholeskyKernel launches on its own stream (SolvePath::slices, decided
by chooseSolvePath for the library and the CPU emulator alike).

CPU: the emulator's rule, with the limits of an H100 SXM, gives one slice just below the threshold and two at it.
GPU: a cfg3 batch at the threshold, solved sliced, gives bit for bit what each of its halves gives solved as a batch of its own (below
the threshold, one slice): parameters, errors, iterations, status and error history, with a fixed iteration count and in convergence
mode (threshold 1, and a loose threshold at which instances stop at different iterations)."""
import numpy as np
import pytest

from momentum_b200 import solver as ms
from momentum_b200.problems import humanoid_problem
from tests import emu_lib
from tests.emu_lib import EMU_LIB
from tests.test_solve_path import H100_SXM

CTAS_PER_SM = 4  # gramCholeskyKernel's launch bound (kGramCholCtasPerSm)
MIN_WAVES = 4    # kSliceMinWaves


def _threshold(sms):
    return MIN_WAVES * sms * CTAS_PER_SM


def _opts(**kw):
    base = dict(min_iterations=1, max_iterations=1, threshold=1.0, regularization=0.05)
    base.update(kw)
    return ms.GaussNewtonSolverOptions(**base)


@pytest.fixture(scope="module")
def emu():
    emu_lib.build()
    lib = ms.load_library(EMU_LIB)
    lib.emu_set_device_limits(*H100_SXM)
    return lib


def _emu_path(emu, B, orientation=True, **kw):
    ch, efs, _, _ = humanoid_problem(B, orientation=orientation)
    solver = ms.GaussNewtonSolver(_opts(**kw), ms.SkeletonSolverFunction(ch, B, efs, lib_path=EMU_LIB))
    assert emu.emu_choose_solve_path(solver._h) == 0, emu.mb2_last_error().decode()
    return solver.get_solve_path()


@pytest.mark.parametrize("orientation", [True, False], ids=["cfg3", "cfg2"])
def test_emulator_slices_from_four_waves(emu, orientation):
    T = _threshold(H100_SXM[0])
    below, at = _emu_path(emu, T - 1, orientation), _emu_path(emu, T, orientation)
    assert below["kind"] == at["kind"] == "gram_cholesky", (below, at)
    assert (below["slices"], at["slices"]) == (1, 2), (below, at)


def test_emulator_does_not_slice_the_line_search_or_the_persistent_kernel(emu):
    assert _emu_path(emu, 8192, do_line_search=True)["slices"] == 1
    small = _emu_path(emu, 256)
    assert small["kind"] == "persistent" and small["slices"] == 1, small


def _solve(ch, efs, theta, opts):
    B = theta.shape[0]
    fn = ms.SkeletonSolverFunction(ch, B, efs)
    fn.upload_targets()
    solver = ms.GaussNewtonSolver(opts, fn)
    out = solver.solve(theta)
    out["history"] = solver.get_error_history()
    return out, solver.get_solve_path()["slices"], solver.get_counters()[1]


def _half(efs, lo, hi):
    import dataclasses

    return [dataclasses.replace(e, targets=np.asarray(e.targets)[lo:hi]) for e in efs]


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [dict(min_iterations=10, max_iterations=10), dict(min_iterations=1, max_iterations=50),
                                  dict(min_iterations=1, max_iterations=50, threshold=1e6)], ids=["fixed", "convergence", "convergence_early_stops"])
def test_sliced_solve_equals_its_halves(mode):
    import torch

    B = _threshold(torch.cuda.get_device_properties(0).multi_processor_count)
    ch, efs, theta0, _ = humanoid_problem(B)
    theta = theta0.astype(np.float32)
    opts = _opts(store_error_history=True, **mode)
    whole, slices, launches = _solve(ch, efs, theta, opts)
    assert slices == 2
    if mode["min_iterations"] == mode["max_iterations"]:
        assert launches == 2 + 2 * 2 * mode["max_iterations"]  # init + finalize, and a sweep + gramCholeskyKernel per slice and iteration
    elif mode.get("threshold", 1.0) > 1.0:
        assert len(np.unique(whole["iterations"])) > 1  # instances stop at different iterations
    for lo, hi in ((0, B // 2), (B // 2, B)):
        half, half_slices, _ = _solve(ch, _half(efs, lo, hi), theta[lo:hi], opts)
        assert half_slices == 1
        for key in ("params", "errors", "iterations", "status", "history"):
            assert np.array_equal(whole[key][lo:hi], half[key]), (key, lo, hi)


@pytest.mark.gpu
def test_profiling_solve_runs_unsliced():
    import torch

    B = _threshold(torch.cuda.get_device_properties(0).multi_processor_count)
    ch, efs, theta0, _ = humanoid_problem(B)
    fn = ms.SkeletonSolverFunction(ch, B, efs)
    fn.upload_targets()
    solver = ms.GaussNewtonSolver(_opts(min_iterations=3, max_iterations=3), fn)
    solver.set_profiling(1)
    solver.solve(theta0.astype(np.float32))
    _, launches = solver.get_phase_times()
    assert solver.get_solve_path()["slices"] == 1 and launches[0] == launches[2] == 3, launches
    solver.set_profiling(0)
    solver.solve(theta0.astype(np.float32))
    assert solver.get_solve_path()["slices"] == 2
