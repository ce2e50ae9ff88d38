"""Which linear-solve path a solve runs: chooseSolvePath (momentum_b200/csrc/ik_solve_path.cpp) decides it once for the library and
for the CPU emulator, and mb2_solver_get_solve_path reports it.

CPU: the emulator evaluates the choice for every row of PATHS (planning only, no solve) with the limits of an H100 SXM, and runs the
chosen path. GPU: the library reports the same record as the emulator given the device's own limits, and refuses with the same message.
The runtime refusal "Gram + Cholesky fusion: no resident CTA" (the occupancy query finds no resident CTA) is not reached by any fixture."""
import numpy as np
import pytest

from momentum_b200 import solver as ms
from momentum_b200.problems import bodyhands_problem, humanoid_problem
from tests import emu_lib
from tests import f64ref as R
from tests.emu_lib import EMU_LIB

H100_SXM = (132, 227 * 1024, 228 * 1024)  # SMs, opt-in shared memory per block, shared memory per SM


@pytest.fixture(scope="module")
def emu():
    emu_lib.build()
    return ms.load_library(EMU_LIB)


def _rig(name, B):
    """(character, error functions, enabled parameters or None)"""
    if name == "humanoid":
        ch, efs, _, _ = humanoid_problem(B, orientation=True)
        return ch, efs, None
    if name == "humanoid_rows":  # ten copies of the Position block: the strips of an instance no longer fit in shared memory
        ch, efs, _, _ = humanoid_problem(B, orientation=True)
        return ch, efs + [efs[0]] * 9, None
    if name == "humanoid_none":
        ch, efs, _, _ = humanoid_problem(B, orientation=True)
        return ch, efs, np.zeros(ch.num_params, bool)
    if name == "bodyhands":
        ch, efs, _, _ = bodyhands_problem(B)
        return ch, efs, None
    n = int(name[5:])  # chainN: N parameters, all coupled through the end effector
    ch, efs, _ = R.chain_case(n, positions=12, B=B, seed=n)
    return ch, efs, None


def _opts(**kw):
    base = dict(min_iterations=1, max_iterations=1, threshold=1.0, regularization=0.05)
    base.update(kw)
    return ms.GaussNewtonSolverOptions(**base)


AUTO_OFF = dict(fused_mode=ms.FUSED_OFF)
GRAM = dict(cholesky_mode=ms.CHOLESKY_TILES_SPARSE, jtj_mode=ms.JTJ_SPARSE_TILES)
# name: (rig, options, batch ("wave": persistent groups x SMs, "wave+1": one more), expected fields of the record or (error, message part))
PATHS = {
    "dense_simt": ("humanoid", dict(cholesky_mode=ms.CHOLESKY_DENSE_EIGEN, jtj_mode=ms.JTJ_FP32_SIMT), 4,
                   dict(kind="dense", plan_mode=1, jtj_mode=ms.JTJ_FP32_SIMT, dense_nb=16, dense_in_smem=1)),
    "dense_auto_jtj": ("humanoid", dict(cholesky_mode=ms.CHOLESKY_DENSE_EIGEN), 4, dict(kind="dense", jtj_mode=ms.JTJ_TF32X3, dense_nb=16)),
    "auto_below_48": ("chain47", {}, 4, dict(kind="dense", plan_mode=1, dense_nb=8, dense_in_smem=1)),
    "auto_at_48": ("chain48", {}, 4, dict(kind="persistent", plan_mode=2, sched_dense=0, strips=1)),
    "auto_fallback_330": ("chain330", {}, 4, dict(kind="dense", plan_mode=1, strips=0, dense_nb=32, dense_in_smem=0)),
    "dense_global_nb16": ("chain240", dict(cholesky_mode=ms.CHOLESKY_DENSE_EIGEN), 4, dict(kind="dense", dense_nb=16, dense_in_smem=0)),
    "tiles_kmajor": ("humanoid", dict(cholesky_mode=ms.CHOLESKY_TILES_SPARSE, jtj_mode=ms.JTJ_TF32X3, **AUTO_OFF), 4,
                     dict(kind="tiles_kmajor", plan_mode=2, strips=0, jtj_mode=ms.JTJ_TF32X3, gram_threads=0, chol_threads=256)),
    "tiles_kmajor_dense_pattern": ("humanoid", dict(cholesky_mode=ms.CHOLESKY_TILES_DENSE, jtj_mode=ms.JTJ_FP32_SIMT), 4,
                                   dict(kind="tiles_kmajor", sched_dense=1, jtj_mode=ms.JTJ_FP32_SIMT)),
    "strips_fallback_kmajor": ("humanoid_rows", dict(cholesky_mode=ms.CHOLESKY_TILES_SPARSE), 4, dict(kind="tiles_kmajor", strips=0, jtj_mode=ms.JTJ_TF32X3)),
    "tiles": ("humanoid", dict(GRAM, **AUTO_OFF), 4, dict(kind="tiles", strips=1, jtj_mode=ms.JTJ_SPARSE_TILES, gram_threads=256, chol_threads=256)),
    "tiles_wide": ("bodyhands", dict(GRAM, **AUTO_OFF), 4, dict(kind="tiles", gram_threads=512, chol_threads=512)),
    "cfg4_bodyhands_auto": ("bodyhands", {}, 2048, dict(kind="tiles", strips=1, gram_threads=512, chol_threads=512)),
    "gram_cholesky": ("humanoid", dict(GRAM, fused_mode=ms.FUSED_GRAM_CHOLESKY), 4, dict(kind="gram_cholesky", strips=1)),
    "auto_one_wave": ("humanoid", {}, "wave", dict(kind="persistent", strips=1)),
    "auto_past_one_wave": ("humanoid", {}, "wave+1", dict(kind="gram_cholesky", strips=1)),
    "persistent": ("humanoid", dict(GRAM, fused_mode=ms.FUSED_PERSISTENT), 4096, dict(kind="persistent")),
    "line_search_not_persistent": ("humanoid", dict(do_line_search=True), 4, dict(kind="gram_cholesky")),
    "qr": ("humanoid", dict(linear_solver=ms.LINEAR_SOLVER_QR), 4, dict(kind="qr", plan_mode=1, jtj_mode=ms.JTJ_TF32X3, qr_max_chunk_rows=116)),
    "trust_region_qr": ("humanoid", dict(linear_solver=ms.LINEAR_SOLVER_TRUST_REGION_QR, trust_region_radius=1.0), 4,
                        dict(kind="trust_region_qr", qr_max_chunk_rows=110, tr_r_floats=24312)),
    # the twelve refusals of the choice, in the order it checks them
    "refuse_radius": ("humanoid", dict(linear_solver=ms.LINEAR_SOLVER_TRUST_REGION_QR, trust_region_radius=0.0), 4,
                      (ms.MomentumB200Error, "trust_region_radius must be positive")),
    "refuse_qr_tiles": ("humanoid", dict(linear_solver=ms.LINEAR_SOLVER_QR, cholesky_mode=ms.CHOLESKY_TILES_SPARSE), 4,
                        (ms.MomentumB200Error, "the QR step works on the dense Jacobian")),
    "refuse_sparse_tiles_dense": ("humanoid", dict(cholesky_mode=ms.CHOLESKY_DENSE_EIGEN, jtj_mode=ms.JTJ_SPARSE_TILES), 4,
                                  (ms.MomentumB200Error, "MB2_JTJ_SPARSE_TILES needs the tile-scheduled Cholesky")),
    "refuse_schedule_330": ("chain330", dict(cholesky_mode=ms.CHOLESKY_TILES_DENSE), 4, (ms.MomentumB200Error, "tile schedule does not fit")),
    "refuse_no_parameters": ("humanoid_none", {}, 4, (ms.MomentumB200Error, "no enabled parameters")),
    "refuse_strips": ("humanoid_rows", GRAM, 4, (ms.MomentumB200Error, "Jacobian strips do not fit")),
    "refuse_persistent_line_search": ("humanoid", dict(fused_mode=ms.FUSED_PERSISTENT, do_line_search=True), 4,
                                      (ms.MomentumB200Error, "the fused kernel needs")),
    "refuse_gram_cholesky_rounds": ("bodyhands", dict(fused_mode=ms.FUSED_GRAM_CHOLESKY), 4, (ms.MomentumB200Error, "do not fit in shared memory, or too many")),
    "refuse_gram_cholesky_dense": ("humanoid", dict(cholesky_mode=ms.CHOLESKY_DENSE_EIGEN, fused_mode=ms.FUSED_GRAM_CHOLESKY), 4,
                                   (ms.MomentumB200Error, "Gram + Cholesky fusion needs the tile-sparse Gram")),
    "refuse_tensor_shape": ("chain512", dict(cholesky_mode=ms.CHOLESKY_DENSE_EIGEN, jtj_mode=ms.JTJ_TF32X3), 4,
                            (ms.MomentumB200Error, "tensor-core JtJ does not support this shape")),
    "refuse_qr_size": ("chain330", dict(linear_solver=ms.LINEAR_SOLVER_QR), 4, (ms.MomentumB200Error, "the QR step keeps R in shared memory")),
    "refuse_trust_region_size": ("chain240", dict(linear_solver=ms.LINEAR_SOLVER_TRUST_REGION_QR, trust_region_radius=1.0), 4,
                                 (ms.MomentumB200Error, "the trust-region QR kernel keeps R")),
}


def _batch(emu, rig, kw, B, limits):
    if not isinstance(B, str):
        return B
    groups = _emu_path(emu, rig, kw, 4, limits)[0]["fused_groups"]  # a wave of persistent instance groups, from a small batch's plan
    assert groups >= 1
    return groups * limits[0] + (1 if B == "wave+1" else 0)


def _emu_path(emu, rig, kw, B, limits):
    """(record, error message) of the emulator's choice for one row"""
    emu.emu_set_device_limits(*limits)
    B = _batch(emu, rig, kw, B, limits)
    ch, efs, en = _rig(rig, B)
    fn = ms.SkeletonSolverFunction(ch, B, efs, lib_path=EMU_LIB)
    if en is not None:
        fn.set_enabled_parameters(en)
    solver = ms.GaussNewtonSolver(_opts(**kw), fn)
    if emu.emu_choose_solve_path(solver._h) != 0:
        return solver.get_solve_path(), emu.mb2_last_error().decode()
    return solver.get_solve_path(), None


def _check(name, rec, err):
    expect = PATHS[name][3]
    if isinstance(expect, tuple):
        assert err is not None and expect[1] in err, (name, err)
        assert rec["kind"] is None
        return
    assert err is None, (name, err)
    for k, v in expect.items():
        assert rec[k] == v, (name, k, rec[k], v, rec)
    kind = rec["kind"]
    assert (rec["dense_nb"] > 0) == (kind == "dense") and (rec["chol_threads"] > 0) == (kind in ("tiles", "tiles_kmajor"))
    assert (rec["qr_chunks"] > 0) == (kind in ("qr", "trust_region_qr"))
    assert rec["strips"] or rec["fused_groups"] == 0, rec  # the persistent kernel is sized for plans with strips only


@pytest.mark.parametrize("name", list(PATHS))
def test_emulator_chooses_the_path(name, emu):
    rig, kw, B, _ = PATHS[name]
    rec, err = _emu_path(emu, rig, kw, B, H100_SXM)
    _check(name, rec, err)


def test_no_path_before_the_first_solve(emu):
    ch, efs, _ = _rig("humanoid", 2)
    solver = ms.GaussNewtonSolver(_opts(), ms.SkeletonSolverFunction(ch, 2, efs, lib_path=EMU_LIB))
    assert solver.get_solve_path()["kind"] is None and not any(v for k, v in solver.get_solve_path().items() if k != "kind")


def test_emulator_refuses_qr_instead_of_solving_with_cholesky(emu):
    emu.emu_set_device_limits(*H100_SXM)
    ch, efs, _ = _rig("humanoid", 1)
    fn = ms.SkeletonSolverFunction(ch, 1, efs, lib_path=EMU_LIB)
    fn.upload_targets()
    solver = ms.GaussNewtonSolver(_opts(linear_solver=ms.LINEAR_SOLVER_QR), fn)
    with pytest.raises(ms.MomentumB200Error, match="does not emulate the QR"):
        solver.solve(np.zeros((1, ch.num_params), np.float32))
    assert solver.get_solve_path()["kind"] == "qr"


def test_emulated_auto_on_the_330_chain_is_the_dense_solve(emu):
    """CHOLESKY_AUTO on the 330-parameter chain falls back to the dense kernel (its tile schedule does not fit): the emulated AUTO
    solve is the explicitly dense one, bit for bit."""
    emu.emu_set_device_limits(*H100_SXM)
    ch, efs, _ = R.chain_case(330, positions=12, seed=330)
    th0 = np.zeros((1, ch.num_params))
    outs = []
    for mode in (ms.CHOLESKY_AUTO, ms.CHOLESKY_DENSE_EIGEN):
        solver, out, *_ = R.one_step(ch, efs, th0, _opts(cholesky_mode=mode, fused_mode=ms.FUSED_OFF), EMU_LIB, rel_damping=1e-5)
        assert solver.get_solve_path()["kind"] == "dense" and np.all(out["status"] == 0)
        outs.append(out)
    assert np.array_equal(outs[0]["params"], outs[1]["params"]) and np.array_equal(outs[0]["errors"], outs[1]["errors"])


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(PATHS))
def test_library_reports_the_emulators_path(name, emu):
    import torch

    p = torch.cuda.get_device_properties(0)
    limits = (p.multi_processor_count, p.shared_memory_per_block_optin, p.shared_memory_per_multiprocessor)
    rig, kw, B, expect = PATHS[name]
    want, want_err = _emu_path(emu, rig, kw, B, limits)
    B = _batch(emu, rig, kw, B, limits)
    ch, efs, en = _rig(rig, B)
    fn = ms.SkeletonSolverFunction(ch, B, efs)
    fn.upload_targets()
    if en is not None:
        fn.set_enabled_parameters(en)
    solver = ms.GaussNewtonSolver(_opts(**kw), fn)
    theta = np.zeros((B, ch.num_params), np.float32)
    if want_err is not None:
        with pytest.raises(ms.MomentumB200Error) as e:
            solver.solve(theta)
        assert str(e.value) == want_err
        assert solver.get_solve_path()["kind"] is None
        return
    solver.solve(theta)
    got = solver.get_solve_path()
    assert got == want, (name, got, want)
    _check(name, got, None)
    fused = {"persistent": 1, "gram_cholesky": 2}.get(got["kind"], 0)
    prof = solver.get_fused_profile()
    assert prof["fused"] == fused and prof["groups"] == (got["fused_groups"] if fused == 1 else 0)
    st = solver.get_plan_stats()
    assert (st["cholesky_tiles"] > 0) == (got["plan_mode"] == 2) and (st["strip_floats"] > 0) == bool(got["strips"])
    assert st["fused_groups"] == (got["fused_groups"] if got["strips"] else 0)
