"""Timing of find_closest_points (point cloud, plain and normal variants) on the device: the per-call tree build and the query kernel
apart, queries per second, a chunked float32 torch brute force, and scipy's cKDTree on the host (the stand-in for pymomentum's CPU path).

    python scripts/closest_cloud_bench.py [--reps 5] [--iters 10] [--json PATH]

Sources are the posed vertices of synthetic_tube_mesh (10 368 on humanoid72, 19 200 on bodyhands300) with their vertex normals from
compute_vertex_normals, each instance at its own pose near the scan's (seeded model parameters, the scan's plus uniform +-0.05).
Targets are synthetic_scan clouds of 2 10^4 and 10^5 points of the same character at a seeded pose. "shared": one scan for the whole
batch (one tree per call); "batched": a scan per instance (four seeded scans, each instance's shifted by its own small offset, so every
instance builds its own tree). Per case: microseconds per call (CUDA events around `iters` calls after a warm-up, the median of `reps`
windows), the build (every cloud* kernel) and query (closestCloudKernel) kernel times from torch.profiler in a run of their own, and
queries per second. The brute force runs where B N M <= 2^32 and must agree on every index where its two best squared distances differ;
cKDTree (float64, one tree per instance and per call, queries on one core) runs for B <= 16. The card and its power limit are read in the
same run. There is no CPU path for the device timings: without a GPU they fail.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from momentum_b200 import character as mc  # noqa: E402
from momentum_b200 import solver as ms  # noqa: E402
from momentum_b200 import torch_skeleton as tsk  # noqa: E402

TUBES = {"humanoid72": (mc.humanoid72, 12, 12), "bodyhands300": (mc.bodyhands300, 8, 8)}
BATCHES, SCANS = (1, 16, 64, 256), (20_000, 100_000)


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
    return float(np.median(times))


def kernel_times(fn, calls=3):
    """Microseconds per call in the build kernels (cloud*) and in closestCloudKernel, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile

    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            fn()
        torch.cuda.synchronize()
    out = {"build": 0.0, "query": 0.0}
    for e in prof.key_averages():
        dt = getattr(e, "device_time_total", None)
        if dt is None:
            dt = e.cuda_time_total
        if "closestCloudKernel" in e.key:
            out["query"] += dt / calls
        elif "cloud" in e.key and "Kernel" in e.key:
            out["build"] += dt / calls
    return out


def rig(name):
    make, rings, segments = TUBES[name]
    ch = make()[0]
    ch.skinning = mc.synthetic_tube_mesh(ch, rings, segments, 1)
    return ch


def brute_force(p, x):
    """The nearest target by float32 torch: squared distances chunked, argmin (the lower index on ties), and whether the two best differ."""
    B, N, _ = p.shape
    idx = torch.empty(B, N, dtype=torch.int64, device=p.device)
    untied = torch.empty(B, N, dtype=torch.bool, device=p.device)
    chunk = max(1, (1 << 26) // x.shape[1])
    for b in range(B):
        xb = x[b if x.shape[0] > 1 else 0]
        for s in range(0, N, chunk):
            d = ((p[b, s:s + chunk, None, :] - xb[None]) ** 2).sum(-1)
            v, i = d.topk(2, dim=-1, largest=False)
            idx[b, s:s + chunk] = i[:, 0]
            untied[b, s:s + chunk] = v[:, 0] < v[:, 1]
    return idx, untied


def kdtree_us(p, x):
    """scipy cKDTree in float64 on the host: a tree per instance, then its queries; microseconds per call."""
    from scipy.spatial import cKDTree

    pc, xc = p.double().cpu().numpy(), x.double().cpu().numpy()
    t0 = time.perf_counter()
    for b in range(pc.shape[0]):
        cKDTree(xc[b if xc.shape[0] > 1 else 0]).query(pc[b], k=1)
    return (time.perf_counter() - t0) * 1e6


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--json", default=None, help="also write the results here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("closest_cloud_bench needs a CUDA device")
    gpu = card()
    print(f"card, power limit: {gpu}")
    dev = torch.device("cuda", 0)
    stream = torch.cuda.current_stream(dev).cuda_stream
    rows = []
    print("| rig | M | B | target | variant | call us | build us | query us | Mqueries/s | brute force us | same index (untied) | cKDTree us |")
    print("|---|---|---|---|---|---|---|---|---|---|---|---|")
    for name in TUBES:
        ch = rig(name)
        rng = np.random.default_rng(2)
        theta_s = rng.uniform(-0.3, 0.3, ch.num_params)
        for M in SCANS:
            scans = [mc.synthetic_scan(ch, M, theta=theta_s, seed=s) for s in range(4)]
            for B in BATCHES:
                theta = torch.from_numpy((theta_s + rng.uniform(-0.05, 0.05, (B, ch.num_params))).astype(np.float32)).to(dev)
                with torch.no_grad():
                    p = tsk.skin_points(ch, tsk.model_parameters_to_skeleton_state(ch, theta)).contiguous()
                    pn = tsk.compute_vertex_normals(ch, p).contiguous()
                N = p.shape[1]
                for kind in ("shared", "batched"):
                    if kind == "shared":
                        x = torch.from_numpy(scans[0][0]).to(dev)[None].contiguous()
                        xn = torch.from_numpy(scans[0][1]).to(dev)[None].contiguous()
                    else:
                        k = np.arange(B) % 4
                        shift = np.random.default_rng(B).uniform(-0.5, 0.5, (B, 1, 3)).astype(np.float32)
                        x = torch.from_numpy(np.stack([scans[i][0] for i in k]) + shift).to(dev)
                        xn = torch.from_numpy(np.stack([scans[i][1] for i in k])).to(dev)
                    q = torch.empty(B, N, 3, device=dev)
                    qn = torch.empty(B, N, 3, device=dev)
                    idx = torch.empty(B, N, dtype=torch.int32, device=dev)
                    for variant in ("plain", "normals"):
                        nrm = variant == "normals"

                        def call(x=x, xn=xn, nrm=nrm, kind=kind):
                            ms.closest_points_device(0, B, N, M, kind == "batched", p.data_ptr(), pn.data_ptr() if nrm else 0, x.data_ptr(),
                                                     xn.data_ptr() if nrm else 0, float("inf"), 0.0, q.data_ptr(), qn.data_ptr() if nrm else 0,
                                                     idx.data_ptr(), stream)

                        it = max(1, args.iters if B * N <= 1 << 20 else args.iters // 5)
                        t_call = timed(call, args.reps, it)
                        kt = kernel_times(call)
                        r = {"rig": name, "M": M, "B": B, "target": kind, "variant": variant, "N": N, "call_us": t_call, "build_us": kt["build"],
                             "query_us": kt["query"], "Mqps": B * N / t_call}
                        bf, kd = "not run | ", "not run"
                        if variant == "plain" and B * N * M <= 1 << 32:
                            with torch.no_grad():
                                t0 = torch.cuda.Event(enable_timing=True); t1 = torch.cuda.Event(enable_timing=True)
                                t0.record()
                                bi, untied = brute_force(p, x)
                                t1.record(); t1.synchronize()
                            r["brute_us"] = t0.elapsed_time(t1) * 1e3
                            call()
                            torch.cuda.synchronize()
                            r["same_untied"] = bool((bi == idx.long())[untied].all())
                            r["untied_fraction"] = float(untied.float().mean())
                            bf = f"{r['brute_us']:.0f} | {r['same_untied']} ({r['untied_fraction']:.4f})"
                        if variant == "plain" and B <= 16:
                            r["kdtree_us"] = kdtree_us(p, x)
                            kd = f"{r['kdtree_us']:.0f}"
                        rows.append(r)
                        print(f"| {name} | {M} | {B} | {kind} | {variant} | {t_call:.1f} | {kt['build']:.1f} | {kt['query']:.1f} | {r['Mqps']:.1f} | "
                              f"{bf} | {kd} |", flush=True)
                    del x, xn, q, qn, idx
                torch.cuda.empty_cache()
    if args.json:
        with open(args.json, "w") as fh:
            json.dump({"card": gpu, "cases": rows}, fh, indent=1)


if __name__ == "__main__":
    main()
