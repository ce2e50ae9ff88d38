"""Timing of find_closest_points_on_mesh on the device: the refit and the query kernel apart, queries per second, a chunked float32 torch
brute force with the same semantics as the baseline, and whether the tree built on the rest mesh stays good on posed meshes.

    python scripts/closest_points_bench.py [--reps 5] [--iters 10] [--json PATH]
    python scripts/closest_points_bench.py --visits     # nodes visited per query, from the CPU emulator (no GPU)

Meshes are synthetic_tube_mesh's (20 448 faces on humanoid72, 37 200 on bodyhands300), posed by skin_points at seeded random poses, one
per instance. Two query distributions per instance: "scan" samples the posed surface and offsets each sample along its face normal by 1 %
of the mean bone length (a scan-like correspondence search), "box" is uniform in the posed mesh's bounding box inflated by 20 % (the
worst case: most queries are far from the surface). Per case: microseconds per call (CUDA events around `iters` calls after a warm-up,
the median of `reps` windows with the fastest in brackets), the refit and query kernel times from torch.profiler in a run of their own,
queries per second, and the brute force where B N F <= 2^31. The tree-quality rows time the same batch at one pose (instance 0's,
repeated) with the tree built on the rest mesh and with a tree built by set_mesh_tree on that pose. The card and its power limit are read
in the same run. There is no CPU path for the timings: without a GPU they fail.
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from momentum_b200 import character as mc  # noqa: E402
from momentum_b200 import solver as ms  # noqa: E402
from momentum_b200 import torch_skeleton as tsk  # noqa: E402

TUBES = {"humanoid72": (mc.humanoid72, 12, 12), "bodyhands300": (mc.bodyhands300, 8, 8)}
BATCHES, POINTS = (1, 64, 1024), (1024, 10000)


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout
    return out.strip().splitlines()[0]


def timed(fn, reps, iters, warmup=2):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(iters):
            fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b) * 1e3 / iters)
    return float(np.median(times)), float(np.min(times))


def kernel_times(fn, calls=3):
    """Microseconds per call in meshTreeRefitKernel and in closestPointKernel, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile

    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            fn()
        torch.cuda.synchronize()
    out = {"refit": 0.0, "query": 0.0}
    for e in prof.key_averages():
        dt = getattr(e, "device_time_total", None)
        if dt is None:
            dt = e.cuda_time_total
        if "meshTreeRefitKernel" in e.key:
            out["refit"] += dt / calls
        elif "closestPointKernel" in e.key:
            out["query"] += dt / calls
    return out


def rig(name, seed=1):
    make, rings, segments = TUBES[name]
    ch = make()[0]
    ch.skinning = mc.synthetic_tube_mesh(ch, rings, segments, seed)
    return ch


def bone_length(ch):
    t, _, _ = mc.forward_kinematics(ch, np.zeros((1, ch.num_params)))
    p = np.asarray(ch.parents)
    d = np.linalg.norm(t[0][p >= 0] - t[0][p[p >= 0]], axis=-1)
    return float(d[d > 0].mean())


def posed(ch, B, seed, dev):
    theta = torch.from_numpy(np.random.default_rng(seed).uniform(-0.5, 0.5, (B, ch.num_params)).astype(np.float32)).to(dev)
    with torch.no_grad():
        return tsk.skin_points(ch, tsk.model_parameters_to_skeleton_state(ch, theta)).contiguous()


def queries(faces, x, N, kind, offset, seed):
    """[B, N, 3] queries on the device for posed vertices x [B, V, 3]."""
    B = x.shape[0]
    g = torch.Generator(device=x.device).manual_seed(seed)
    if kind == "box":
        lo, hi = x.amin(1, keepdim=True), x.amax(1, keepdim=True)
        pad = 0.2 * (hi - lo)
        return lo - pad + (hi - lo + 2 * pad) * torch.rand(B, N, 3, device=x.device, generator=g)
    fi = torch.randint(0, faces.shape[0], (B, N), device=x.device, generator=g)
    tri = faces[fi]  # [B, N, 3]
    c = torch.gather(x, 1, tri.reshape(B, -1, 1).expand(-1, -1, 3)).reshape(B, N, 3, 3)
    w = -torch.log(torch.rand(B, N, 3, device=x.device, generator=g))
    w = w / w.sum(-1, keepdim=True)
    n = torch.linalg.cross(c[:, :, 1] - c[:, :, 0], c[:, :, 2] - c[:, :, 0])
    n = n / n.norm(dim=-1, keepdim=True).clamp_min(1e-12)
    s = offset * (2 * torch.rand(B, N, 1, device=x.device, generator=g) - 1)
    return ((w[..., None] * c).sum(-2) + s * n).contiguous()


def brute_force(faces, x, p):
    """The same selection in float32 torch: per query every face's (Ericson) closest point, the smallest (d2, face); chunked."""
    B, N, _ = p.shape
    F = faces.shape[0]
    chunk = max(1, (1 << 24) // F)
    face_out = torch.empty(B, N, dtype=torch.int64, device=p.device)
    for b in range(B):
        a, bb, c = (x[b][faces[:, k]] for k in range(3))
        ab, ac = bb - a, c - a
        for s in range(0, N, chunk):
            pp = p[b, s:s + chunk, None, :]
            ap, bp, cp = pp - a, pp - bb, pp - c
            d1, d2, d3, d4, d5, d6 = ((u * v).sum(-1) for u, v in ((ab, ap), (ac, ap), (ab, bp), (ac, bp), (ab, cp), (ac, cp)))
            vc, vb, va = d1 * d4 - d3 * d2, d5 * d2 - d1 * d6, d3 * d6 - d5 * d4
            den = 1.0 / (va + vb + vc)
            v, w = vb * den, vc * den
            q = a + ab * v[..., None] + ac * w[..., None]
            for m, val in (((va <= 0) & (d4 - d3 >= 0) & (d5 - d6 >= 0), bb + ((d4 - d3) / ((d4 - d3) + (d5 - d6)))[..., None] * (c - bb)),
                           ((vb <= 0) & (d2 >= 0) & (d6 <= 0), a + (d2 / (d2 - d6))[..., None] * ac),
                           ((d6 >= 0) & (d5 <= d6), c.expand_as(q)),
                           ((vc <= 0) & (d1 >= 0) & (d3 <= 0), a + (d1 / (d1 - d3))[..., None] * ab),
                           ((d3 >= 0) & (d4 <= d3), bb.expand_as(q)), ((d1 <= 0) & (d2 <= 0), a.expand_as(q))):
                q = torch.where(m[..., None], val, q)
            d = ((q - pp) ** 2).sum(-1)
            d = torch.where(torch.isfinite(d), d, torch.full_like(d, float("inf")))
            face_out[b, s:s + chunk] = d.argmin(-1)  # the first index of the minimum: the lower face on ties
    return face_out


def visits():
    """Nodes visited per query from the CPU emulator (tests/emu/emu_closest_points.cu), rest tree against pose tree."""
    sys.path.insert(0, ROOT)
    from tests import test_closest_points_on_mesh as t

    d = tempfile.mkdtemp()
    lib = os.path.join(d, "libemu_closest_points.so")
    csrc = os.path.join(ROOT, "momentum_b200", "csrc")
    subprocess.check_call(["nvcc", "-O2", "-std=c++17", "-Xcompiler", "-fPIC,-ffp-contract=off", "--fmad=false", "-shared", "-o", lib,
                           os.path.join(ROOT, "tests", "emu", "emu_closest_points.cu"), os.path.join(csrc, "ik_plan.cpp"),
                           os.path.join(csrc, "ik_chol_sched.cpp")])
    L = ctypes.CDLL(lib)
    L.emu_closest_points_last_error.restype = ctypes.c_char_p
    L.emu_closest_points.argtypes = [ctypes.c_int32] * 2 + [ctypes.c_void_p] * 2 + [ctypes.c_int32] * 2 + [ctypes.c_void_p] * 2 + \
        [ctypes.c_float, ctypes.c_int32] + [ctypes.c_void_p] * 4
    print("| rig | queries | rest tree: mean / p99 nodes | pose tree: mean / p99 nodes | (CPU emulator) |")
    print("|---|---|---|---|---|")
    for name in TUBES:
        ch = rig(name)
        faces = ch.skinning.faces
        theta = np.random.default_rng(3).uniform(-0.5, 0.5, (4, ch.num_params))
        tt, q, s = mc.forward_kinematics(ch, theta)
        x = mc.skin_points(ch, np.concatenate([tt, q, s[..., None]], -1)).astype(np.float32)
        rng = np.random.default_rng(4)
        for kind in ("scan", "box"):
            res = []
            for ref in ("rest", "pose"):
                v = []
                for b in range(x.shape[0]):
                    if kind == "scan":
                        p = t._queries(ch, x[b], 512, 10 + b, scan_only=True)
                    else:
                        lo, hi = x[b].min(0), x[b].max(0)
                        pad = 0.2 * (hi - lo)
                        p = rng.uniform(lo - pad, hi + pad, (512, 3)).astype(np.float32)
                    r = ch.skinning.rest_vertices if ref == "rest" else x[b]
                    v.append(t._emu_run(L, faces, r, x[b:b + 1], p[None], visits=True)[3].ravel())
                v = np.concatenate(v)
                res.append(f"{v.mean():.0f} / {np.percentile(v, 99):.0f}")
            print(f"| {name} | {kind} | {res[0]} | {res[1]} | |", flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--json", default=None, help="also write the results here")
    ap.add_argument("--visits", action="store_true", help="print the emulator's nodes per query and exit")
    args = ap.parse_args()
    if args.visits:
        visits()
        return
    if not torch.cuda.is_available():
        raise SystemExit("closest_points_bench needs a CUDA device")
    gpu = card()
    print(f"card, power limit: {gpu}")
    dev = torch.device("cuda", 0)
    stream = torch.cuda.current_stream(dev).cuda_stream
    rows = []
    print("| rig | B | N | queries | call us | refit us | query us | Mqueries/s | brute force us | same faces as brute force |")
    print("|---|---|---|---|---|---|---|---|---|---|")
    tree_rows = []
    for name in TUBES:
        ch = rig(name)
        dc = ms.DeviceCharacter(ch, 0)
        faces = torch.from_numpy(ch.skinning.faces.astype(np.int64)).to(dev)
        F = faces.shape[0]
        off = 0.01 * bone_length(ch)
        for B in BATCHES:
            x = posed(ch, B, B, dev)
            for N in POINTS:
                for kind in ("scan", "box"):
                    p = queries(faces, x, N, kind, off, 7 * B + N)
                    q = torch.empty(B, N, 3, device=dev)
                    fo = torch.empty(B, N, dtype=torch.int32, device=dev)
                    bo = torch.empty(B, N, 3, device=dev)

                    def call(d=dc, x=x, p=p, B=B, N=N):
                        d.closest_points_on_mesh_device(B, N, x.data_ptr(), p.data_ptr(), float("inf"), q.data_ptr(), fo.data_ptr(), bo.data_ptr(), stream)

                    it = max(1, args.iters if B * N <= 1 << 20 else args.iters // 5)
                    t_call = timed(call, args.reps, it)
                    kt = kernel_times(call)
                    r = {"rig": name, "B": B, "N": N, "queries": kind, "call_us": t_call, "refit_us": kt["refit"], "query_us": kt["query"],
                         "Mqps": B * N / t_call[0]}
                    bf = ""
                    if B * N * F <= 1 << 31:
                        with torch.no_grad():
                            r["brute_us"] = timed(lambda: brute_force(faces, x, p), 1, 1, 1)
                            bfo = brute_force(faces, x, p)
                        call()
                        r["same_faces"] = float((bfo == fo.long()).float().mean())
                        bf = f"{r['brute_us'][0]:.0f} | {r['same_faces']:.4f}"
                    else:
                        bf = "not run | "
                    rows.append(r)
                    print(f"| {name} | {B} | {N} | {kind} | {t_call[0]:.1f} [{t_call[1]:.1f}] | {kt['refit']:.1f} | {kt['query']:.1f} | {r['Mqps']:.1f} | {bf} |",
                          flush=True)
            # tree quality: one pose for the batch, the rest tree against a tree built on that pose
            if B == 64:
                x0 = x[:1].expand(B, -1, -1).contiguous()
                dp = ms.DeviceCharacter(ch, 0)
                dp.set_mesh_tree(x0[0].cpu().numpy())
                for N in POINTS:
                    for kind in ("scan", "box"):
                        p = queries(faces, x0, N, kind, off, 11 * N)
                        q = torch.empty(B, N, 3, device=dev)
                        fo = torch.empty(B, N, dtype=torch.int32, device=dev)
                        bo = torch.empty(B, N, 3, device=dev)
                        res = []
                        outs = []
                        for d in (dc, dp):
                            def call(d=d, p=p, N=N):
                                d.closest_points_on_mesh_device(B, N, x0.data_ptr(), p.data_ptr(), float("inf"), q.data_ptr(), fo.data_ptr(), bo.data_ptr(),
                                                                stream)
                            res.append(kernel_times(call)["query"])
                            call()
                            outs.append((q.clone(), fo.clone(), bo.clone()))
                        same = all(torch.equal(u, w) for u, w in zip(*outs))
                        tree_rows.append({"rig": name, "B": B, "N": N, "queries": kind, "rest_tree_query_us": res[0], "pose_tree_query_us": res[1],
                                          "same_bits": same})
    print()
    print("| rig | B | N | queries | query us, rest tree | query us, pose tree | rest / pose | same bits |")
    print("|---|---|---|---|---|---|---|---|")
    for r in tree_rows:
        print(f"| {r['rig']} | {r['B']} | {r['N']} | {r['queries']} | {r['rest_tree_query_us']:.1f} | {r['pose_tree_query_us']:.1f} | "
              f"{r['rest_tree_query_us'] / r['pose_tree_query_us']:.2f} | {r['same_bits']} |")
    if args.json:
        with open(args.json, "w") as fh:
            json.dump({"card": gpu, "cases": rows, "tree_quality": tree_rows}, fh, indent=1)


if __name__ == "__main__":
    main()
