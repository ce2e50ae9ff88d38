"""Part 1 of include/momentum_b200_adapters.hpp compiles as plain C++17 against the C-ABI and links the product library."""
import os
import subprocess
import tempfile

import numpy as np
import pytest

from momentum_b200 import solver as ms

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SRC = r"""
#include <cstdio>
#include <momentum_b200_adapters.hpp>
int main() {
  using namespace momentum_b200;
  // createTestCharacter(3): Y chain, 9 + 1 model parameters (character_helpers.cpp:106-149)
  std::vector<int32_t> parents{-1, 0, 1};
  std::vector<float> off{0,0,0, 0,1,0, 0,1,0}, pre{0,0,0,1, 0,0,0,1, 0,0,0,1};
  std::vector<int32_t> outer(22, 0), inner; std::vector<float> vals, offs(21, 0.f);
  int rows[] = {0,1,2,3,4,5,6, 10, 12, 19, 17};
  int cols[] = {0,1,2,3,4,5,6, 7, 8, 8, 9};
  float cf[] = {1,1,1,1,1,1,1, 1, .5f, .5f, 1};
  for (int r = 0; r < 21; ++r) { for (int k = 0; k < 11; ++k) if (rows[k] == r) { inner.push_back(cols[k]); vals.push_back(cf[k]); } outer[r + 1] = int(inner.size()); }
  try {
    Character ch(0, parents, off, pre, 10, outer, inner, vals, offs);
    BatchedSkeletonSolverFunction fn(ch, 4);
    GaussNewtonSolverOptions o; o.maxIterations = 6; o.minIterations = 6; o.regularization = 1e-7f; o.useBlockJtJ = true;
    int pos = fn.addPositionErrorFunction(1.f, {2}, {0.f, 1.f, 0.f}, {1.f});
    int pl = fn.addPlaneErrorFunction(1e-4f, {2}, {0.f, 0.5f, 0.f}, {1.f}, /*above=*/true);
    int mp = fn.addModelParametersErrorFunction(1e-3f, std::vector<float>(10, 1.f));
    // every block first, then the per-instance data (the record layout is fixed by the block list)
    std::vector<float> tg(4 * 3, 0.f); for (int b = 0; b < 4; ++b) { tg[3*b] = 0.3f * b; tg[3*b+1] = 2.5f; }
    fn.setTargets(pos, tg);
    std::vector<float> planes(4 * 4, 0.f); for (int b = 0; b < 4; ++b) { planes[4*b+1] = 1.f; planes[4*b+3] = -1.f; }
    fn.setTargets(pl, planes);
    fn.setTargets(mp, std::vector<float>(4 * 10, 0.f));
    BatchedGaussNewtonSolver solver(o, &fn);
    std::vector<float> params(4 * 10, 0.f);
    auto r = solver.solve(params);
    std::printf("solved: err0=%g it0=%d\n", r.errors[0], r.iterations[0]);
  } catch (const std::runtime_error& e) {
    std::printf("runtime_error: %s\n", e.what());
    return 3;
  }
  return 0;
}
"""


def _build_and_run():
    import __graft_entry__ as g

    g.build()
    with tempfile.TemporaryDirectory() as d:
        src = os.path.join(d, "t.cpp")
        exe = os.path.join(d, "t")
        open(src, "w").write(SRC)
        lib_dir = os.path.dirname(ms.DEFAULT_LIB)
        subprocess.check_call(["g++", "-std=c++17", "-I", os.path.join(ROOT, "include"), src, "-o", exe, "-L", lib_dir, "-lmomentum_b200",
                               f"-Wl,-rpath,{lib_dir}"])
        return subprocess.run([exe], capture_output=True, text=True)


def test_adapter_header_compiles_and_fails_loudly_without_gpu():
    p = _build_and_run()
    if ms.load_library().mb2_device_count() > 0:
        assert p.returncode == 0 and "solved" in p.stdout, p.stdout + p.stderr
    else:
        assert p.returncode == 3 and "no usable sm_90 CUDA device" in p.stdout, p.stdout + p.stderr


# ---- Part 2: subclasses of momentum's own interfaces, compiled against tests/mock_momentum (signature-level stand-ins) ----
def _fl(x):
    return repr(float(np.float32(x))) + "f"


def _part2_source(ch, efs, b, theta0, iterations, regularization):
    """C++ program that rebuilds `ch` / `efs` (instance b) as momentum:: objects, hands them to CudaSkeletonSolverFunction through
    addErrorFunction(shared_ptr<SkeletonErrorFunctionT<float>>) and solves three ways; prints one parameter vector per line."""
    from momentum_b200 import character as mc

    L = ["#include <cstdio>", "#include <momentum_b200_adapters.hpp>", "#ifndef MOMENTUM_B200_HAVE_MOMENTUM", "#error part 2 of the adapters header is not enabled",
         "#endif", "using namespace momentum;", "static void show(const char* tag, double e, const VectorXf& p) { std::printf(\"%s %.9g\", tag, e); for (Eigen::Index i = 0; i < p.size(); ++i) std::printf(\" %.9g\", p(i)); std::printf(\"\\n\"); }",
         "int main() {", "  Character ch;"]
    J, n = ch.num_joints, ch.num_params
    for j in range(J):
        par = "kInvalidIndex" if ch.parents[j] < 0 else f"size_t({int(ch.parents[j])})"
        o, q = ch.offsets[j], ch.prerot[j]
        L.append(f"  {{ Joint jt; jt.parent = {par}; jt.translationOffset = Vector3f({_fl(o[0])}, {_fl(o[1])}, {_fl(o[2])}); jt.preRotation = Quaternionf({_fl(q[3])}, {_fl(q[0])}, {_fl(q[1])}, {_fl(q[2])}); ch.skeleton.joints.push_back(jt); }}")
    L.append(f"  ch.parameterTransform.transform = SparseRowMatrix<float>({7 * J}, {n});")
    ent = []
    for r in range(7 * J):
        for k in range(ch.pt_outer[r], ch.pt_outer[r + 1]):
            ent.append(f"{{{r}, {int(ch.pt_inner[k])}, {_fl(ch.pt_vals[k])}}}")
    L.append("  ch.parameterTransform.transform.setFromEntries({" + ", ".join(ent) + "});")
    L.append(f"  ch.parameterTransform.offsets = VectorXf::Zero({7 * J});")
    for r in range(7 * J):
        if ch.pt_offsets[r] != 0:
            L.append(f"  ch.parameterTransform.offsets({r}) = {_fl(ch.pt_offsets[r])};")
    for lim in ch.limits:
        i, f = lim.packed()
        L.append(f"  {{ ParameterLimit l; l.type = LimitType({int(lim.type)}); l.weight = {_fl(lim.weight)};")
        t = int(lim.type)
        if t == mc.LIMIT_MINMAX:
            L.append(f"    l.data.minMax.parameterIndex = {i[0]}; l.data.minMax.limits = Vector2f({_fl(f[0])}, {_fl(f[1])});")
        elif t in (mc.LIMIT_MINMAX_JOINT, mc.LIMIT_MINMAX_JOINT_PASSIVE):
            L.append(f"    l.data.minMaxJoint.jointIndex = {i[0]}; l.data.minMaxJoint.jointParameter = {i[1]}; l.data.minMaxJoint.limits = Vector2f({_fl(f[0])}, {_fl(f[1])});")
        elif t == mc.LIMIT_LINEAR:
            L.append(f"    l.data.linear = LimitLinear{{{i[0]}, {i[1]}, {_fl(f[0])}, {_fl(f[1])}, {_fl(f[2])}, {_fl(f[3])}}};")
        elif t == mc.LIMIT_LINEAR_JOINT:
            L.append(f"    l.data.linearJoint = LimitLinearJoint{{{i[0]}, {i[1]}, {i[2]}, {i[3]}, {_fl(f[0])}, {_fl(f[1])}, {_fl(f[2])}, {_fl(f[3])}}};")
        elif t == mc.LIMIT_HALFPLANE:
            L.append(f"    l.data.halfPlane.param1 = {i[0]}; l.data.halfPlane.param2 = {i[1]}; l.data.halfPlane.normal = Vector2f({_fl(f[0])}, {_fl(f[1])}); l.data.halfPlane.offset = {_fl(f[2])};")
        elif t == mc.LIMIT_ELLIPSOID:
            L.append(f"    l.data.ellipsoid.ellipsoidParent = {i[0]}; l.data.ellipsoid.parent = {i[1]}; l.data.ellipsoid.offset = Vector3f({_fl(f[24])}, {_fl(f[25])}, {_fl(f[26])});")
            for r in range(3):
                for c in range(4):
                    L.append(f"    l.data.ellipsoid.ellipsoid.m[{r}][{c}] = {_fl(f[4 * r + c])}; l.data.ellipsoid.ellipsoidInv.m[{r}][{c}] = {_fl(f[12 + 4 * r + c])};")
        L.append("    ch.parameterLimits.push_back(l); }")
    L.append("  std::vector<std::shared_ptr<SkeletonErrorFunction>> efs;")
    for k, ef in enumerate(efs):
        v = f"ef{k}"
        if ef.kind == mc.KIND_POSITION:
            L.append(f"  auto {v} = std::make_shared<PositionErrorFunction>(ch, {_fl(ef.loss_alpha)}, {_fl(ef.loss_c)});")
            for c in range(len(ef.parents)):
                o, t = ef.offsets[c], ef.targets[b, c]
                L.append(f"  {v}->addConstraint(PositionData(Vector3f({_fl(o[0])}, {_fl(o[1])}, {_fl(o[2])}), Vector3f({_fl(t[0])}, {_fl(t[1])}, {_fl(t[2])}), {int(ef.parents[c])}, {_fl(ef.weights[c])}));")
        elif ef.kind in (mc.KIND_ORIENTATION, mc.KIND_ORIENTATION_ROTDIFF):
            cls = "OrientationRotDiffErrorFunctionT<float>" if ef.rot_diff else "OrientationErrorFunction"
            L.append(f"  auto {v} = std::make_shared<{cls}>(ch, {_fl(ef.loss_alpha)}, {_fl(ef.loss_c)});")
            for c in range(len(ef.parents)):
                o, t = ef.offsets[c], ef.targets[b, c]
                L.append(f"  {v}->addConstraint(OrientationData(Quaternionf({_fl(o[3])}, {_fl(o[0])}, {_fl(o[1])}, {_fl(o[2])}), Quaternionf({_fl(t[3])}, {_fl(t[0])}, {_fl(t[1])}, {_fl(t[2])}), {int(ef.parents[c])}, {_fl(ef.weights[c])}));")
        elif ef.kind == mc.KIND_PLANE:
            L.append(f"  auto {v} = std::make_shared<PlaneErrorFunction>(ch, {'true' if ef.above else 'false'}, {_fl(ef.loss_alpha)}, {_fl(ef.loss_c)});")
            for c in range(len(ef.parents)):
                o, t = ef.offsets[c], ef.targets[b, c]
                L.append(f"  {v}->addConstraint(PlaneData(Vector3f({_fl(o[0])}, {_fl(o[1])}, {_fl(o[2])}), Vector3f({_fl(t[0])}, {_fl(t[1])}, {_fl(t[2])}), {_fl(t[3])}, {int(ef.parents[c])}, {_fl(ef.weights[c])}));")
        elif ef.kind == mc.KIND_STATE:
            rt = "RotationErrorType::QuaternionLogMap" if ef.rotation_error_type == 1 else "RotationErrorType::RotationMatrixDifference"
            L.append(f"  auto {v} = std::make_shared<StateErrorFunction>(ch, {rt}); {v}->setWeights({_fl(ef.pos_wgt)}, {_fl(ef.rot_wgt)});")
            L.append(f"  {{ TransformListT<float> tg({J}); VectorXf pw({J}), rw({J});")
            for j in range(J):
                t = ef.targets[b, j]
                L.append(f"    tg[{j}].translation = Vector3f({_fl(t[0])}, {_fl(t[1])}, {_fl(t[2])}); tg[{j}].rotation = Quaternionf({_fl(t[6])}, {_fl(t[3])}, {_fl(t[4])}, {_fl(t[5])}); tg[{j}].scale = {_fl(t[7])}; pw({j}) = {_fl(ef.pos_weights[j])}; rw({j}) = {_fl(ef.rot_weights[j])};")
            L.append(f"    {v}->setTargetState(tg); {v}->setTargetWeights(pw, rw); }}")
        elif ef.kind == mc.KIND_LIMIT:
            L.append(f"  auto {v} = std::make_shared<LimitErrorFunction>(ch, {_fl(ef.loss_alpha)}, {_fl(ef.loss_c)});")
        elif ef.kind == mc.KIND_MODEL_PARAMETERS:
            L.append(f"  auto {v} = std::make_shared<ModelParametersErrorFunction>(ch);")
            L.append(f"  {{ VectorXf t({n}), w({n});")
            for i in range(n):
                L.append(f"    t({i}) = {_fl(ef.targets[b, i])}; w({i}) = {_fl(ef.target_weights[i])};")
            L.append(f"    {v}->setTargetParameters(ModelParameters(t), w); }}")
        L.append(f"  {v}->setWeight({_fl(ef.weight)}); efs.push_back({v});")
    L += ["  try {", "    momentum_b200::CudaSkeletonSolverFunction fn(ch, ch.parameterTransform, efs);",
          f"    GaussNewtonSolverOptions o; o.minIterations = {iterations}; o.maxIterations = {iterations}; o.threshold = 1.0f; o.regularization = {_fl(regularization)}; o.useBlockJtJ = true;",
          f"    VectorXf p0({n});"]
    L += [f"    p0({i}) = {_fl(theta0[i])};" for i in range(n)]
    L += ["    { GaussNewtonSolverT<float> stock(o, &fn); VectorXf p = p0; const double e = stock.solve(p); show(\"stock\", e, p); }   // momentum's solver loop, device getJtJR",
          "    { momentum_b200::CudaGaussNewtonSolver cuda(o, &fn); VectorXf p = p0; const double e = cuda.solve(p); show(\"solvert\", e, p);  // SolverT::solve, device doIteration",
          "      VectorXf q = p0; const double e2 = cuda.solveOnDevice(q); show(\"device\", e2, q); }                                            // whole loop on the device",
          "    { momentum_b200::CudaGaussNewtonSolver cuda(o, &fn); cuda.setLinearSolver(MB2_LINEAR_SOLVER_QR); VectorXf q = p0; const double e = cuda.solveOnDevice(q); show(\"qr\", e, q);  // GaussNewtonSolverQRT's step",
          "      cuda.setLinearSolver(MB2_LINEAR_SOLVER_TRUST_REGION_QR, 1.0f); VectorXf r = p0; const double e2 = cuda.solveOnDevice(r); show(\"trustregion\", e2, r); }                        // TrustRegionQRT's iteration",
          "    { VectorXf g; const double e = fn.getGradient(p0, g); show(\"gradient\", e, g); }",
          "    struct Other : SkeletonErrorFunctionT<float> { using SkeletonErrorFunctionT<float>::SkeletonErrorFunctionT; };",
          "    try { fn.addErrorFunction(std::make_shared<Other>(ch.skeleton, ch.parameterTransform)); std::printf(\"unsupported accepted\\n\"); } catch (const std::runtime_error&) { std::printf(\"unsupported rejected\\n\"); }",
          "  } catch (const std::runtime_error& ex) { std::printf(\"runtime_error: %s\\n\", ex.what()); return 3; }", "  return 0;", "}"]
    return "\n".join(L) + "\n"


def _build_and_run_part2(src_text):
    import __graft_entry__ as g

    g.build()
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "p2.cpp"), os.path.join(d, "p2")
        open(src, "w").write(src_text)
        lib_dir = os.path.dirname(ms.DEFAULT_LIB)
        subprocess.check_call(["g++", "-std=c++20", "-Wall", "-I", os.path.join(ROOT, "tests", "mock_momentum"), "-I", os.path.join(ROOT, "include"), src, "-o", exe,
                               "-L", lib_dir, "-lmomentum_b200", f"-Wl,-rpath,{lib_dir}"])
        return subprocess.run([exe], capture_output=True, text=True)


def _part2_problem():
    from momentum_b200.problems import chain_problem

    ch, efs, theta0, ts = chain_problem(J=6, B=2, seed=61, families=("position", "orientation", "state", "limit", "plane", "halfplane", "model_parameters"), rot_diff=False)
    return ch, efs, (ts + 0.1 * theta0).astype(np.float32)


def test_adapter_part2_compiles_against_the_momentum_interfaces():
    """CudaSkeletonSolverFunction : SolverFunctionT<float> and CudaGaussNewtonSolver : SolverT<float> compile against the (stand-in)
    momentum headers with every supported error-function class translated; without a GPU the first device call fails loudly."""
    ch, efs, theta0 = _part2_problem()
    p = _build_and_run_part2(_part2_source(ch, efs, 1, theta0[1], 5, 0.05))
    if ms.load_library().mb2_device_count() == 0:
        assert p.returncode == 3 and "no usable sm_90 CUDA device" in p.stdout, p.stdout + p.stderr


@pytest.mark.gpu
def test_adapter_part2_momentum_objects_solve_on_the_gpu_and_match_the_oracle():
    """Reference-shaped objects (Character, Position / Orientation / State / Limit / Plane / ModelParameters error functions) ->
    addErrorFunction -> three solve routes (momentum's own GaussNewtonSolverT loop over the device getJtJR; SolverT::solve over the device
    doIteration; the whole loop on the device) -> converged parameters against the float oracle on the same inputs."""
    from oracle.binding import OracleFunction

    ch, efs, theta0 = _part2_problem()
    its, reg, b = 5, 0.05, 1
    p = _build_and_run_part2(_part2_source(ch, efs, b, theta0[b], its, reg))
    assert p.returncode == 0, p.stdout + p.stderr
    got = {ln.split()[0]: np.array(ln.split()[1:], np.float64) for ln in p.stdout.splitlines() if ln and ln.split()[0] in ("stock", "solvert", "device", "gradient", "qr", "trustregion")}
    assert "unsupported rejected" in p.stdout
    orc = OracleFunction(ch, efs, "float32", instance=b)
    err, ref, _, _ = orc.solve(theta0[b].astype(np.float64), min_iterations=its, max_iterations=its, threshold=1.0, regularization=reg, use_block_jtj=True)
    for route in ("stock", "solvert", "device"):
        e, q = got[route][0], got[route][1:]
        assert np.max(np.abs(q - ref)) / max(1.0, np.max(np.abs(ref))) <= 2e-4, (route, np.max(np.abs(q - ref)))
        assert abs(e - err) <= 1e-3 * abs(err) + 1e-7, (route, e, err)
    # the other two solver classes through setLinearSolver, each against the oracle's restatement of that class
    for route, kw in (("qr", dict(regularization=reg, qr_solver=True)), ("trustregion", dict(trust_region_qr=True))):
        err_r, ref_r, _, _ = orc.solve(theta0[b].astype(np.float64), min_iterations=its, max_iterations=its, threshold=1.0, **kw)
        e, q = got[route][0], got[route][1:]
        assert np.max(np.abs(q - ref_r)) / max(1.0, np.max(np.abs(ref_r))) <= 5e-4, (route, np.max(np.abs(q - ref_r)))
        assert abs(e - err_r) <= 1e-3 * abs(err_r) + 1e-7, (route, e, err_r)
    _, Ho, go = orc.get_jtjr(theta0[b].astype(np.float64))
    g = got["gradient"][1:]
    assert g.shape[0] == ch.num_params and np.max(np.abs(g - 2 * go)) <= 2e-5 * max(1.0, np.abs(go).max())


@pytest.mark.gpu
def test_adapter_part1_solves_on_the_gpu():
    """The C++ host side (Part 1 of the adapters header) drives a real solve on the GPU under `pytest -m gpu`."""
    p = _build_and_run()
    assert p.returncode == 0 and "solved" in p.stdout, p.stdout + p.stderr
