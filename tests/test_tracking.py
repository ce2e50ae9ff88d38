"""SURVEY 8(f) rank 2: the trackPosesForFrames front end (include/momentum_b200_tracking.hpp) on a synthetic marker sequence,
against the oracle run frame by frame with the reference's schedule (rigid warm start, then the full solve)."""
import os
import subprocess
import tempfile

import numpy as np
import pytest

from momentum_b200 import character as mc
from momentum_b200 import solver as ms

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _sequence(F=10, seed=3):
    """humanoid72, 24 body locators + 2 floor locators on the feet, a smooth motion with a moving root, a few occluded markers."""
    ch, sets = mc.humanoid72()
    rng = np.random.default_rng(seed)
    n = ch.num_params
    pj = list(sets["position_joints"])
    locs = [dict(name=f"M{k}", parent=int(j), offset=rng.uniform(-3, 3, 3).astype(np.float32), weight=float(rng.uniform(0.8, 1.2))) for k, j in enumerate(pj)]
    feet = [int(j) for j in pj[-2:]]
    locs += [dict(name=f"Floor_{k}", parent=j, offset=rng.uniform(-1, 1, 3).astype(np.float32), weight=1.0) for k, j in enumerate(feet)]
    t = np.linspace(0, 1, F)[:, None]
    a, b = rng.uniform(-0.35, 0.35, (2, n))
    theta = a[None] * np.sin(2.0 * t) + b[None] * t
    theta[:, 6] = 0.0
    theta[:, 0:3] = np.array([5.0, 90.0, -3.0])[None] + 10.0 * t * np.array([1.0, 0.05, 0.5])[None]
    parents = np.array([l["parent"] for l in locs[:len(pj)]], np.int32)
    offs = np.stack([l["offset"] for l in locs[:len(pj)]])
    pos = mc.world_points(ch, theta, parents, offs) + 0.05 * rng.normal(size=(F, len(pj), 3))
    occl = rng.uniform(size=(F, len(pj))) < 0.12
    conf = rng.uniform(0.7, 1.0, (F, len(pj)))
    rigid = np.zeros(n, bool); rigid[:6] = True
    pose = np.ones(n, bool); pose[6] = False
    return ch, locs, len(pj), theta, pos, occl, conf, rigid, pose


def _source(ch, locs, nm, pos, occl, conf, rigid, pose, frames, continuous, max_iter, smoothing):
    F, n, J = pos.shape[0], ch.num_params, ch.num_joints
    fl = lambda x: repr(float(np.float32(x))) + "f"
    L = ["#include <cstdio>", "#include <momentum_b200_tracking.hpp>", "using namespace momentum_b200;", "int main() {"]
    L.append("  std::vector<int32_t> parents{" + ", ".join(str(int(p)) for p in ch.parents) + "};")
    L.append("  std::vector<float> off{" + ", ".join(fl(x) for x in ch.offsets.reshape(-1)) + "}, pre{" + ", ".join(fl(x) for x in ch.prerot.reshape(-1)) + "};")
    L.append("  std::vector<int32_t> outer{" + ", ".join(str(int(x)) for x in ch.pt_outer) + "}, inner{" + ", ".join(str(int(x)) for x in ch.pt_inner) + "};")
    L.append("  std::vector<float> vals{" + ", ".join(fl(x) for x in ch.pt_vals) + "}, offs(" + str(7 * J) + ", 0.f);")
    L.append("  std::vector<Locator> locators;")
    for l in locs:
        o = l["offset"]
        L.append(f"  {{ Locator l; l.name = \"{l['name']}\"; l.parent = {l['parent']}; l.offset[0] = {fl(o[0])}; l.offset[1] = {fl(o[1])}; l.offset[2] = {fl(o[2])}; l.weight = {fl(l['weight'])}; locators.push_back(l); }}")
    L.append(f"  std::vector<std::vector<Marker>> markers({F});")
    for f in range(F):
        for k in range(nm):
            p = pos[f, k]
            L.append(f"  {{ Marker m; m.name = \"M{k}\"; m.pos[0] = {float(p[0])!r}; m.pos[1] = {float(p[1])!r}; m.pos[2] = {float(p[2])!r}; m.occluded = {'true' if occl[f, k] else 'false'}; m.confidence = {fl(conf[f, k])}; markers[{f}].push_back(m); }}")
        L.append(f"  {{ Marker m; m.name = \"unmapped\"; m.occluded = false; markers[{f}].push_back(m); }}")  # no locator of that name: ignored
    L.append(f"  ParameterSet rigid, pose;")
    L += [f"  rigid.set({i});" for i in np.nonzero(rigid)[0]] + [f"  pose.set({i});" for i in np.nonzero(pose)[0]]
    L.append(f"  std::vector<float> init({F * n}, 0.f);")
    L.append("  std::vector<size_t> frames{" + ", ".join(str(int(x)) for x in frames) + "};")
    L += ["  try {", f"    Character ch(0, parents, off, pre, {n}, outer, inner, vals, offs);",
          f"    TrackingConfig cfg; cfg.maxIter = {max_iter}; cfg.minVisPercent = 0.5f; cfg.regularization = 0.05f; cfg.smoothing = {fl(smoothing)};",
          f"    const TrackingResult r = trackPosesForFrames(markers, ch, {n}, locators, init, cfg, frames, {'true' if continuous else 'false'}, rigid, pose);",
          "    std::printf(\"solved %zu\\n\", r.solvedFrames);",
          f"    for (size_t f = 0; f < {F}; ++f) {{ std::printf(\"frame\"); for (size_t i = 0; i < {n}; ++i) std::printf(\" %.9g\", r.motion[f * {n} + i]); std::printf(\"\\n\"); }}",
          "  } catch (const std::runtime_error& e) { std::printf(\"runtime_error: %s\\n\", e.what()); return 3; }", "  return 0;", "}"]
    return "\n".join(L) + "\n"


def _run(src_text):
    import __graft_entry__ as g

    g.build()
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "trk.cpp"), os.path.join(d, "trk")
        open(src, "w").write(src_text)
        lib_dir = os.path.dirname(ms.DEFAULT_LIB)
        subprocess.check_call(["g++", "-std=c++17", "-Wall", "-I", os.path.join(ROOT, "include"), src, "-o", exe, "-L", lib_dir, "-lmomentum_b200", f"-Wl,-rpath,{lib_dir}"])
        return subprocess.run([exe], capture_output=True, text=True)


def _oracle_frame(ch, locs, nm, pos, occl, conf, f, theta0, rigid, pose, max_iter, smooth_target=None, smoothing=0.0, rigid_init=True):
    from oracle.binding import OracleFunction

    parents = np.array([l["parent"] for l in locs[:nm]], np.int32)
    offs = np.stack([l["offset"] for l in locs[:nm]])
    w = np.array([0.0 if occl[f, k] else np.float32(locs[k]["weight"]) * np.float32(conf[f, k]) for k in range(nm)], np.float32)
    fl = locs[nm:]
    efs = [mc.LimitErrorFunction(weight=0.1), mc.PositionErrorFunction(parents, offs, w, pos[f][None].astype(np.float32), weight=mc.PositionErrorFunction.kLegacyWeight),
           mc.PlaneErrorFunction(np.array([l["parent"] for l in fl], np.int32), np.stack([l["offset"] for l in fl]), np.array([5.0 * l["weight"] for l in fl], np.float32),
                                 np.tile(np.array([0, 1.0, 0, 0], np.float32), (1, len(fl), 1)), above=True, weight=mc.PlaneErrorFunction.kLegacyWeight)]
    n = ch.num_params
    if smooth_target is not None:
        tw = (pose & ~rigid).astype(np.float32)
        efs.append(mc.ModelParametersErrorFunction(tw, smooth_target[None].astype(np.float32), weight=smoothing))
    th = theta0.astype(np.float64)
    if rigid_init:
        efs_r = efs[:3] + ([mc.ModelParametersErrorFunction(efs[3].target_weights, th[None].astype(np.float32), weight=0.0)] if smooth_target is not None else [])
        orc = OracleFunction(ch, efs_r, "float32")
        orc.set_enabled_parameters(rigid)
        _, th, _, _ = orc.solve(th, min_iterations=2, max_iterations=50, threshold=1.0, regularization=0.05)
        if smooth_target is not None:  # the smoothness target of the full solve is the pose after the rigid start
            efs[3] = mc.ModelParametersErrorFunction(efs[3].target_weights, th[None].astype(np.float32), weight=smoothing)
    orc = OracleFunction(ch, efs, "float32")
    orc.set_enabled_parameters(pose)
    _, th, _, _ = orc.solve(th, min_iterations=2, max_iterations=max_iter, threshold=1.0, regularization=0.05)
    return th


def test_tracking_front_end_compiles_and_fails_loudly_without_gpu():
    ch, locs, nm, theta, pos, occl, conf, rigid, pose = _sequence(F=3)
    p = _run(_source(ch, locs, nm, pos, occl, conf, rigid, pose, [0, 2], False, 5, 0.0))
    if ms.load_library().mb2_device_count() == 0:
        assert p.returncode == 3 and "no usable sm_90 CUDA device" in p.stdout, p.stdout + p.stderr


@pytest.mark.gpu
@pytest.mark.parametrize("continuous", [False, True])
def test_track_poses_for_frames_matches_the_oracle_frame_by_frame(continuous):
    F, max_iter, smoothing = 8, 12, (0.5 if continuous else 0.0)
    ch, locs, nm, theta, pos, occl, conf, rigid, pose = _sequence(F=F)
    occl[5, :] = True; occl[5, :3] = False          # frame 5: too few visible markers -> not solved (minVisPercent = 0.5)
    frames = [0, 1, 3, 5, 6]                        # a subset of the frames, unsorted order allowed
    p = _run(_source(ch, locs, nm, pos, occl, conf, rigid, pose, [3, 0, 1, 6, 5], continuous, max_iter, smoothing))
    assert p.returncode == 0, p.stdout + p.stderr
    got = np.array([ln.split()[1:] for ln in p.stdout.splitlines() if ln.startswith("frame")], np.float64)
    assert got.shape == (F, ch.num_params) and "solved 4" in p.stdout
    n = ch.num_params
    expect = np.zeros((F, n))
    if not continuous:
        sol = {f: _oracle_frame(ch, locs, nm, pos, occl, conf, f, np.zeros(n), rigid, pose, max_iter) for f in frames if f != 5}
        out, dof = 0, np.zeros(n)
        for f in frames:
            dof = sol.get(f, np.zeros(n))           # the unsolved frame keeps its initial column
            while out <= f:
                expect[out] = dof; out += 1
        expect[out:] = dof
    else:
        dof, need, out = np.zeros(n), True, 0
        for f in frames:
            if f != 5:
                dof = _oracle_frame(ch, locs, nm, pos, occl, conf, f, dof, rigid, pose, max_iter, smooth_target=dof, smoothing=smoothing, rigid_init=need)
                need = False
            while out <= f:
                expect[out] = dof; out += 1
        expect[out:] = dof
    scale = np.maximum(1.0, np.abs(expect).max(axis=1, keepdims=True))
    d = np.max(np.abs(got - expect) / scale)
    assert d <= 3e-4, d
