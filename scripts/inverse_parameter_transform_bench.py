"""Timing of apply_inverse_parameter_transform on the device, forward and forward + backward, against pymomentum's own formulation in
float32 torch, (jp - o) @ pinv.T with a dense pseudo-inverse and its autograd backward, and beside apply_parameter_transform for scale.

    python scripts/inverse_parameter_transform_bench.py [--reps 5] [--iters 100] [--warmup 20]

Per case it prints the card and its power limit, microseconds per call, instances per second and the achieved HBM bytes per second
from the algorithmic bytes: the forward reads 7 J and writes n floats per instance, the backward reads n and writes 7 J (it does not
read the forward's input); apply_parameter_transform the other way round. The share of HBM bandwidth is that rate over the 3.35 TB/s
of NVIDIA's H100 SXM data sheet. Times are CUDA events around `iters` calls after a warm-up; the median of `reps` windows is reported,
with the fastest in brackets. There is no CPU path: without a GPU it fails.
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

CASES = [("humanoid72", 8192), ("bodyhands300", 2048), ("humanoid72", 256)]
HBM_PEAK = 3.35e12  # bytes/s, H100 SXM data sheet


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout
    return out.strip().splitlines()[0]


def dense_pinv(ch):
    """pymomentum's matrix: the dense pseudo-inverse of P with singular values > 1e-6 inverted (computed here in float64), as float32"""
    J = ch.num_joints
    P = np.zeros((7 * J, ch.num_params))
    rows = np.repeat(np.arange(7 * J), np.diff(ch.pt_outer))
    np.add.at(P, (rows, ch.pt_inner), ch.pt_vals.astype(np.float64))
    U, S, Vt = np.linalg.svd(P, full_matrices=False)
    return ((Vt.T * np.where(S > 1e-6, 1.0 / np.where(S > 1e-6, S, 1.0), 0.0)) @ U.T).astype(np.float32)


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("inverse_parameter_transform_bench: no CUDA device (there is no CPU path)")
    dev = torch.device("cuda", 0)
    name = card()
    print(f"card: {name} (name, power limit)")
    rigs = {"humanoid72": mc.humanoid72()[0], "bodyhands300": mc.bodyhands300()[0]}
    for rig, B in CASES:
        ch = rigs[rig]
        n, R = ch.num_params, 7 * ch.num_joints
        rng = np.random.default_rng(0)
        theta = torch.from_numpy(rng.uniform(-0.5, 0.5, (B, n)).astype(np.float32)).to(dev)
        dc = tsk._device_character(ch, dev)
        stream = torch.cuda.current_stream(dev).cuda_stream
        jp = tsk.apply_parameter_transform(ch, theta).contiguous()
        th_out, jp_out = torch.empty(B, n, device=dev), torch.empty(B, R, device=dev)
        g_theta = torch.from_numpy(rng.normal(size=(B, n)).astype(np.float32)).to(dev)
        g_jp = torch.from_numpy(rng.normal(size=(B, R)).astype(np.float32)).to(dev)
        g_jp_out, g_theta_out = torch.empty(B, R, device=dev), torch.empty(B, n, device=dev)
        pinv = torch.from_numpy(dense_pinv(ch)).to(dev)
        off = torch.from_numpy(ch.pt_offsets).to(dev)
        jp_req = jp.clone().requires_grad_(True)

        def inv_fwd():
            dc.joint_op_device("apply_inverse_parameter_transform", False, B, jp.data_ptr(), th_out.data_ptr(), stream=stream)

        def inv_fwd_bwd():
            inv_fwd()
            dc.joint_op_device("apply_inverse_parameter_transform", True, B, g_theta.data_ptr(), g_jp_out.data_ptr(), stream=stream)

        def pt_fwd():
            dc.joint_op_device("apply_parameter_transform", False, B, theta.data_ptr(), jp_out.data_ptr(), stream=stream)

        def pt_fwd_bwd():
            pt_fwd()
            dc.joint_op_device("apply_parameter_transform", True, B, g_jp.data_ptr(), g_theta_out.data_ptr(), stream=stream)

        def torch_fwd():
            with torch.no_grad():
                (jp - off) @ pinv.T

        def torch_fwd_bwd():
            torch.autograd.grad((((jp_req - off) @ pinv.T) * g_theta).sum(), jp_req)

        inv_fwd_bwd()
        ref_out = (jp - off) @ pinv.T
        ref_grad = torch.autograd.grad((((jp_req - off) @ pinv.T) * g_theta).sum(), jp_req)[0]
        torch.cuda.synchronize()
        agree = {"theta_max_abs_diff": float((th_out - ref_out).abs().max()), "theta_max_abs_err": float((th_out - theta).abs().max()),
                 "grad_max_abs_diff_rel": float((g_jp_out - ref_grad).abs().max() / ref_grad.abs().max().clamp_min(1.0))}
        inv_bytes = 4 * (R + n)  # either direction: 7 J and n floats per instance
        for label, f, nbytes in (("ours inverse forward", inv_fwd, inv_bytes), ("ours inverse forward+backward", inv_fwd_bwd, 2 * inv_bytes),
                                 ("torch dense pinv forward", torch_fwd, inv_bytes),
                                 ("torch dense pinv forward+backward", torch_fwd_bwd, 2 * inv_bytes),
                                 ("ours apply_parameter_transform forward", pt_fwd, inv_bytes),
                                 ("ours apply_parameter_transform forward+backward", pt_fwd_bwd, 2 * inv_bytes)):
            med, best = timed(f, args.reps, args.iters, args.warmup)
            rate = B * nbytes / (med * 1e-6)
            rec = {"case": f"{B} x {rig}", "impl": label, "us_per_call": round(med, 2), "us_best": round(best, 2), "instances_per_s": B / (med * 1e-6),
                   "hbm_GB_per_s": rate / 1e9, "hbm_share_of_3_35_TB_s": rate / HBM_PEAK, "card": name}
            print(f"{rec['case']:>18} {label:<50} {med:9.2f} us [{best:9.2f}] {rate / 1e9:8.1f} GB/s ({100 * rate / HBM_PEAK:5.1f} %)")
            print(json.dumps(rec))
        print(json.dumps({"case": f"{B} x {rig}", "agreement_with_torch_fp32": agree}))


if __name__ == "__main__":
    main()
