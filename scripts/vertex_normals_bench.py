"""Timing and memory of compute_vertex_normals on the device against the composition a user writes without it: pymomentum's
``compute_vertex_normals`` in torch (three index_selects, a cross, three index_add_s and normalize, with autograd), on the same GPU.

    python scripts/vertex_normals_bench.py [--reps 5] [--iters 20] [--json PATH]

Meshes are synthetic_tube_mesh's (10 368 vertices and 20 448 faces on humanoid72, 19 200 and 37 200 on bodyhands300); every instance has
its own positions (the rest mesh moved per vertex). Two layers are timed: the device layer (library calls into preallocated buffers,
against the composition's forward and its autograd backward) and the torch layer (torch_skeleton.compute_vertex_normals with autograd,
host dispatch included). Per case it prints microseconds per call for the forward and for forward + backward (CUDA events around
`iters` calls after a warm-up, the median of `reps` windows with the fastest in brackets), the peak device memory of one forward +
backward through the torch layer above what the inputs hold (torch.cuda.max_memory_allocated) with, beside it, the backward's
stream-ordered scratch, which torch's allocator does not see (the launcher's slicing rule), and the algorithmic bytes per second: 24 B
per vertex-instance forward (positions in, normals out) and 72 B more for the backward (positions and upstream in, h written and read,
the gradient out). The card and its power limit are read in the same run. There is no CPU path: without a GPU it fails.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from momentum_b200 import character as mc  # noqa: E402
from momentum_b200 import solver as ms  # noqa: E402
from momentum_b200 import torch_skeleton as tsk  # noqa: E402

CASES = [("humanoid72", 1), ("humanoid72", 64), ("humanoid72", 1024), ("humanoid72", 4096), ("bodyhands300", 512), ("bodyhands300", 2048)]
TUBES = {"humanoid72": (mc.humanoid72, 12, 12), "bodyhands300": (mc.bodyhands300, 8, 8)}
BUDGET = 256 << 20  # the backward's per-slice scratch budget (kSliceScratchBudget)
BYTES_FORWARD, BYTES_BACKWARD = 24, 72  # per vertex-instance: positions + normals; positions, upstream, h written and read, gradient


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout
    return out.strip().splitlines()[0]


def timed(fn, reps, iters, warmup):
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


def composition(faces, x):
    """pymomentum's compute_vertex_normals (tensor_skinning.cpp:354-383) in torch."""
    x0, x1, x2 = (x.index_select(-2, faces[:, k]) for k in range(3))
    n_f = torch.cross(x1 - x0, x2 - x0, dim=-1)
    n = torch.zeros_like(x)
    for k in range(3):
        n.index_add_(-2, faces[:, k], n_f)
    return torch.nn.functional.normalize(n, dim=-1)


def peak_above(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def run_case(rig, B, reps, iters, ch_cache):
    if rig not in ch_cache:
        make, rings, segments = TUBES[rig]
        ch = make()[0]
        ch.skinning = mc.synthetic_tube_mesh(ch, rings, segments, 1)
        ch_cache[rig] = (ch, ms.DeviceCharacter(ch, 0))
    ch, dc = ch_cache[rig]
    V, F = ch.skinning.num_vertices, ch.skinning.faces.shape[0]
    dev = torch.device("cuda", 0)
    gen = torch.Generator(device=dev).manual_seed(B)
    x = torch.from_numpy(ch.skinning.rest_vertices).to(dev)[None] + 0.1 * torch.randn(B, V, 3, device=dev, generator=gen)
    G = torch.randn(B, V, 3, device=dev, generator=gen)
    out, gx = torch.empty_like(x), torch.empty_like(x)
    faces = torch.from_numpy(ch.skinning.faces.astype(np.int64)).to(dev)
    stream = torch.cuda.current_stream(dev).cuda_stream
    warm = 3
    r = {"rig": rig, "B": B, "V": V, "F": F}

    # device layer
    def dev_fwd():
        dc.vertex_normals_device(B, x.data_ptr(), out.data_ptr(), stream)

    def dev_fwd_bwd():
        dc.vertex_normals_device(B, x.data_ptr(), out.data_ptr(), stream)
        dc.vertex_normals_backward_device(B, x.data_ptr(), G.data_ptr(), gx.data_ptr(), stream)

    xr = x.clone().requires_grad_(True)

    def comp_fwd():
        with torch.no_grad():
            composition(faces, x)

    def comp_fwd_bwd():
        composition(faces, xr).backward(G)
        xr.grad = None

    r["device_fwd_us"] = timed(dev_fwd, reps, iters, warm)
    r["device_fwd_bwd_us"] = timed(dev_fwd_bwd, reps, iters, warm)
    r["composition_fwd_us"] = timed(comp_fwd, reps, iters, warm)
    r["composition_fwd_bwd_us"] = timed(comp_fwd_bwd, reps, iters, warm)

    # torch layer
    xt = x.clone().requires_grad_(True)

    def torch_fwd():
        with torch.no_grad():
            tsk.compute_vertex_normals(ch, x)

    def torch_fwd_bwd():
        tsk.compute_vertex_normals(ch, xt).backward(G)
        xt.grad = None

    r["torch_fwd_us"] = timed(torch_fwd, reps, iters, warm)
    r["torch_fwd_bwd_us"] = timed(torch_fwd_bwd, reps, iters, warm)
    r["peak_torch_layer_MiB"] = peak_above(torch_fwd_bwd) / 2**20
    r["peak_composition_MiB"] = peak_above(comp_fwd_bwd) / 2**20
    slice_ = max(1, min(B, BUDGET // (V * 12)))
    r["backward_scratch_MiB"] = slice_ * V * 12 / 2**20
    # the two paths agree
    with torch.no_grad():
        tsk_out = tsk.compute_vertex_normals(ch, x)
        r["max_abs_diff_vs_composition"] = float((tsk_out - composition(faces, x)).abs().max())
    n = B * V
    r["device_fwd_GBps"] = n * BYTES_FORWARD / (r["device_fwd_us"][0] * 1e-6) / 1e9
    r["device_fwd_bwd_GBps"] = n * (BYTES_FORWARD + BYTES_BACKWARD) / (r["device_fwd_bwd_us"][0] * 1e-6) / 1e9
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--json", default=None, help="also write the results here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("vertex_normals_bench needs a CUDA device")
    gpu = card()
    print(f"card, power limit: {gpu}")
    cache, rows = {}, []
    hdr = ("rig", "B", "dev fwd us", "comp fwd us", "dev f+b us", "comp f+b us", "torch fwd us", "torch f+b us", "peak torch MiB (+scratch)",
           "peak comp MiB", "dev fwd GB/s", "dev f+b GB/s", "max|diff|")
    print("| " + " | ".join(hdr) + " |")
    print("|" + "---|" * len(hdr))
    for rig, B in CASES:
        r = run_case(rig, B, args.reps, args.iters, cache)
        rows.append(r)
        f = lambda t: f"{t[0]:.1f} [{t[1]:.1f}]"
        print(f"| {rig} | {B} | {f(r['device_fwd_us'])} | {f(r['composition_fwd_us'])} | {f(r['device_fwd_bwd_us'])} | {f(r['composition_fwd_bwd_us'])} | "
              f"{f(r['torch_fwd_us'])} | {f(r['torch_fwd_bwd_us'])} | {r['peak_torch_layer_MiB']:.0f} (+{r['backward_scratch_MiB']:.0f}) | "
              f"{r['peak_composition_MiB']:.0f} | {r['device_fwd_GBps']:.0f} | {r['device_fwd_bwd_GBps']:.0f} | {r['max_abs_diff_vs_composition']:.1e} |", flush=True)
    if args.json:
        with open(args.json, "w") as fh:
            json.dump({"card": gpu, "cases": rows}, fh, indent=1)


if __name__ == "__main__":
    main()
