"""Timing and memory of skin_with_blend_shapes on the device against the two-step composition it replaces: the shaped rest mesh
``base + w @ S`` in float32 torch, then skin_points with batched rest points, on the same GPU.

    python scripts/blend_skinning_bench.py [--reps 5] [--iters 20]

Meshes are synthetic_skinning's (about 10 k vertices on humanoid72, 20 k on bodyhands300) with synthetic_blend_shape's shape vectors,
every instance with its own weights [B, K]. Both paths are timed through the same layer, at two layers: the device layer (library calls
into preallocated buffers; the composition's GEMMs are torch calls with out=) and the torch layer (torch_skeleton's autograd functions,
host dispatch included). Per case it prints the card and its power limit, microseconds per call for the forward and for forward +
backward (the backward gives the skel-state and the weight gradients; CUDA events around `iters` calls after a warm-up, the median of
`reps` windows with the fastest in brackets), the peak device memory of one forward + backward through the torch layer above what the
inputs hold (torch.cuda.max_memory_allocated) with, beside it, the peak of each path's stream-ordered scratch, which torch's allocator
does not see (from the launchers' slicing rules),
and the algorithmic work: 3 K FMA per vertex-instance for the shape, and the skinning's bytes (32 J + 12 V per instance forward,
32 J + 12 V + 32 J + 4 K backward, the shape vectors read once). There is no CPU path: without a GPU it fails.
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
from momentum_b200 import torch_skeleton as tsk  # noqa: E402

# (rig, B, K): the throughput sizes and, last, a small batch for latency
CASES = [("humanoid72", 1024, 16), ("humanoid72", 1024, 64), ("humanoid72", 4096, 16), ("humanoid72", 4096, 64), ("bodyhands300", 512, 64),
         ("humanoid72", 32, 64)]
VERTICES_PER_JOINT = {"humanoid72": 139, "bodyhands300": 67}
BUDGET = 256 << 20  # the launchers' per-slice scratch budget (kSliceScratchBudget)


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


def peak_above(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("blend_skinning_bench: no CUDA device (there is no CPU path)")
    dev = torch.device("cuda", 0)
    name = card()
    print(f"card: {name} (name, power limit)")
    rigs = {}
    for rig, B, K in CASES:
        if (rig, K) not in rigs:
            ch = mc.humanoid72()[0] if rig == "humanoid72" else mc.bodyhands300()[0]
            ch.skinning = mc.synthetic_skinning(ch, VERTICES_PER_JOINT[rig], 0)
            ch.blend_shape = mc.synthetic_blend_shape(ch, ch.skinning, K, 0)
            rigs[(rig, K)] = ch
        ch = rigs[(rig, K)]
        J, V = ch.num_joints, ch.skinning.num_vertices
        rng = np.random.default_rng(0)
        t, q, s = mc.forward_kinematics(ch, rng.uniform(-0.5, 0.5, (B, ch.num_params)))
        st = torch.from_numpy(np.concatenate([t, q, s[..., None]], -1).astype(np.float32)).to(dev)
        w = torch.from_numpy(rng.normal(size=(B, K)).astype(np.float32)).to(dev)
        G = torch.from_numpy(rng.normal(size=(B, V, 3)).astype(np.float32)).to(dev)
        base = torch.from_numpy(ch.blend_shape.base_shape).to(dev)
        S = torch.from_numpy(ch.blend_shape.shape_vectors).to(dev).reshape(K, V * 3)
        dc = tsk._device_character(ch, dev)
        stream = torch.cuda.current_stream(dev).cuda_stream
        pts = torch.empty(B, V, 3, device=dev)
        gst = torch.empty(B, J, 8, device=dev)
        gw = torch.empty(B, K, device=dev)
        rest = torch.empty(B, V * 3, device=dev)
        grest = torch.empty(B, V * 3, device=dev)

        # the device layer: library calls into preallocated buffers, the composition's GEMMs as out= torch calls
        def fused_fwd():
            dc.skin_with_blend_shapes_device(B, st.data_ptr(), w.data_ptr(), K, pts.data_ptr(), stream)

        def fused_fwd_bwd():
            fused_fwd()
            dc.skin_with_blend_shapes_backward_device(B, st.data_ptr(), w.data_ptr(), K, G.data_ptr(), gst.data_ptr(), gw.data_ptr(), stream)

        def two_step_fwd():
            torch.addmm(base.reshape(1, -1), w, S, out=rest)
            dc.skin_points_device(B, st.data_ptr(), rest.data_ptr(), True, pts.data_ptr(), stream)

        def two_step_fwd_bwd():
            two_step_fwd()
            dc.skin_points_backward_device(B, st.data_ptr(), rest.data_ptr(), True, G.data_ptr(), gst.data_ptr(), grest.data_ptr(), stream)
            torch.mm(grest, S.t(), out=gw)

        # the torch layer: both through torch_skeleton's autograd functions
        st_req, w_req = st.clone().requires_grad_(True), w.clone().requires_grad_(True)

        def torch_fused_fwd():
            with torch.no_grad():
                tsk.skin_with_blend_shapes(ch, st, w)

        def torch_fused_fwd_bwd():
            torch.autograd.grad(tsk.skin_with_blend_shapes(ch, st_req, w_req), (st_req, w_req), G)

        def torch_two_step_fwd():
            with torch.no_grad():
                tsk.skin_points(ch, st, torch.addmm(base.reshape(1, -1), w, S).reshape(B, V, 3))

        def torch_two_step_fwd_bwd():
            p = tsk.skin_points(ch, st_req, torch.addmm(base.reshape(1, -1), w_req, S).reshape(B, V, 3))
            torch.autograd.grad(p, (st_req, w_req), G)

        fused_fwd_bwd()
        fp, fs, fw = pts.clone(), gst.clone(), gw.clone()
        two_step_fwd_bwd()
        torch.cuda.synchronize()
        agree = {"points_max_abs_diff_rel": float((fp - pts).abs().max() / pts.abs().max().clamp_min(1.0)),
                 "state_grad_max_abs_diff_rel": float((fs - gst).abs().max() / gst.abs().max().clamp_min(1.0)),
                 "weight_grad_max_abs_diff_rel": float((fw - gw).abs().max() / gw.abs().max().clamp_min(1.0))}
        del fp, fs, fw
        # stream-ordered scratch (cudaMallocAsync, not seen by torch), from the launchers' slicing rules. The fused backward holds the
        # shaped rest points of a slice together with the skin-points backward's per-segment partials, and frees both before it takes
        # the weight partials; the composition's skin-points backward takes the per-segment partials.
        act = np.cumprod(ch.skinning.skin_weight != 0.0, axis=1).astype(bool)
        per_joint = np.bincount(ch.skinning.skin_index[act], minlength=J)
        seg_bytes = 48 * int(np.sum((per_joint + 127) // 128))
        skin_partial = min(B, BUDGET // seg_bytes) * seg_bytes
        rest_slice = min(B, BUDGET // (12 * V))
        vblocks = (V + 255) // 256
        fused_scratch = max(rest_slice * 12 * V + min(rest_slice, BUDGET // seg_bytes) * seg_bytes, min(B, BUDGET // (4 * vblocks * K)) * 4 * vblocks * K)
        mem = {"fused_torch_peak_bytes": peak_above(torch_fused_fwd_bwd), "fused_scratch_peak_bytes": fused_scratch,
               "two_step_torch_peak_bytes": peak_above(torch_two_step_fwd_bwd), "two_step_scratch_peak_bytes": skin_partial}
        fma = 3 * K * V * B
        fwd_bytes = B * (32 * J + 12 * V + 4 * K) + 12 * K * V
        bwd_bytes = B * (32 * J + 12 * V + 32 * J + 4 * K) + 12 * K * V
        case = f"{B} x {rig} (V = {V}, K = {K})"
        for label, fn, nbytes, flops in (("device: fused forward", fused_fwd, fwd_bytes, 2 * fma),
                                         ("device: two-step forward", two_step_fwd, fwd_bytes, 2 * fma),
                                         ("device: fused forward+backward", fused_fwd_bwd, fwd_bytes + bwd_bytes, 6 * fma),
                                         ("device: two-step forward+backward", two_step_fwd_bwd, fwd_bytes + bwd_bytes, 6 * fma),
                                         ("torch: fused forward", torch_fused_fwd, fwd_bytes, 2 * fma),
                                         ("torch: two-step forward", torch_two_step_fwd, fwd_bytes, 2 * fma),
                                         ("torch: fused forward+backward", torch_fused_fwd_bwd, fwd_bytes + bwd_bytes, 6 * fma),
                                         ("torch: two-step forward+backward", torch_two_step_fwd_bwd, fwd_bytes + bwd_bytes, 6 * fma)):
            med, best = timed(fn, args.reps, args.iters, 3)
            rec = {"case": case, "impl": label, "us_per_call": round(med, 2), "us_best": round(best, 2), "algorithmic_bytes": nbytes,
                   "algorithmic_flops": flops, "GB_per_s": nbytes / (med * 1e-6) / 1e9, "TFLOP_per_s": flops / (med * 1e-6) / 1e12, "card": name}
            print(f"{case:>40} {label:<34} {med:10.1f} us [{best:10.1f}] {rec['GB_per_s']:8.1f} GB/s {rec['TFLOP_per_s']:6.2f} TFLOP/s")
            print(json.dumps(rec))
        print(json.dumps({"case": case, "memory": mem, "agreement_fused_vs_two_step": agree}))
        del rest, grest
        del pts, gst, gw, G
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
