"""Timing of skin_points on the device (forward, and forward + backward to the skeleton state) against pymomentum's torch linear-blend
skinning (skel_state_backend.py:435-512: index_select of the skinning transforms and the rest points per influence, then index_add),
restated in float32 torch with its autograd backward, on the same GPU.

    python scripts/skinning_bench.py [--reps 5] [--iters 50] [--torch-iters 5]

Meshes are synthetic_skinning's: about 10 k vertices on humanoid72 and 20 k on bodyhands300, the rest mesh shared by the batch. Per
case it prints the card and its power limit, microseconds per call (CUDA events around `iters` calls after a warm-up, the median of
`reps` windows with the fastest in brackets), and the achieved HBM bytes per second from the algorithmic bytes with their share of the
H100 SXM's 3.35 TB/s: the forward reads the states and writes the points (32 J + 12 V bytes per instance); the backward reads the states
and the upstream gradient and writes the state gradient (32 J + 12 V + 32 J). The skin tables are shared by the batch and not counted.
There is no CPU path: without a GPU it fails.
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

# the three throughput sizes and, last, a small batch for latency
CASES = [("humanoid72", 1024), ("humanoid72", 4096), ("bodyhands300", 512), ("humanoid72", 32)]
VERTICES_PER_JOINT = {"humanoid72": 139, "bodyhands300": 67}
HBM_BYTES_PER_S = 3.35e12


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout
    return out.strip().splitlines()[0]


class TorchLBS:
    """pymomentum's skin_points_from_skel_state in float32 torch: one row per active influence."""

    def __init__(self, ch, dev):
        sk = ch.skinning
        act = np.cumprod(sk.skin_weight != 0.0, axis=1).astype(bool)
        v, k = np.nonzero(act)
        self.vert = torch.from_numpy(v.astype(np.int64)).to(dev)
        self.joint = torch.from_numpy(sk.skin_index[v, k].astype(np.int64)).to(dev)
        self.w = torch.from_numpy(sk.skin_weight[v, k]).to(dev)
        self.rest = torch.from_numpy(sk.rest_vertices).to(dev)
        self.ibp = torch.from_numpy(sk.inverse_bind_pose).to(dev)
        self.V = sk.num_vertices

    def __call__(self, st):
        q = st[..., 3:7]
        q = q / q.norm(dim=-1, keepdim=True)
        x, y, z, w = q.unbind(-1)
        R = torch.stack([torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)], -1),
                         torch.stack([2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)], -1),
                         torch.stack([2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)], -1)], -2) * st[..., 7, None, None]
        M = torch.cat([R @ self.ibp[..., :3], (R @ self.ibp[..., 3:]) + st[..., :3, None]], -1)  # [B, J, 3, 4]
        Mi = torch.index_select(M, 1, self.joint)
        xi = torch.index_select(self.rest, 0, self.vert)
        p = ((Mi[..., :3] @ xi[..., None])[..., 0] + Mi[..., 3]) * self.w[:, None]
        return torch.zeros(st.shape[0], self.V, 3, device=st.device, dtype=st.dtype).index_add(1, self.vert, p)


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
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--torch-iters", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("skinning_bench: no CUDA device (there is no CPU path)")
    dev = torch.device("cuda", 0)
    name = card()
    print(f"card: {name} (name, power limit)")
    rigs = {}
    for rig, B in CASES:
        if rig not in rigs:
            ch = mc.humanoid72()[0] if rig == "humanoid72" else mc.bodyhands300()[0]
            ch.skinning = mc.synthetic_skinning(ch, VERTICES_PER_JOINT[rig], 0)
            rigs[rig] = ch
        ch = rigs[rig]
        J, V = ch.num_joints, ch.skinning.num_vertices
        rng = np.random.default_rng(0)
        t, q, s = mc.forward_kinematics(ch, rng.uniform(-0.5, 0.5, (B, ch.num_params)))
        st = torch.from_numpy(np.concatenate([t, q, s[..., None]], -1).astype(np.float32)).to(dev)
        G = torch.from_numpy(rng.normal(size=(B, V, 3)).astype(np.float32)).to(dev)
        dc = tsk._device_character(ch, dev)
        pts = torch.empty(B, V, 3, device=dev)
        gst = torch.empty(B, J, 8, device=dev)
        stream = torch.cuda.current_stream(dev).cuda_stream

        def ours_fwd():
            dc.skin_points_device(B, st.data_ptr(), 0, False, pts.data_ptr(), stream)

        def ours_fwd_bwd():
            dc.skin_points_device(B, st.data_ptr(), 0, False, pts.data_ptr(), stream)
            dc.skin_points_backward_device(B, st.data_ptr(), 0, False, G.data_ptr(), gst.data_ptr(), 0, stream)

        lbs = TorchLBS(ch, dev)
        st_req = st.clone().requires_grad_(True)

        def torch_fwd():
            with torch.no_grad():
                lbs(st)

        def torch_fwd_bwd():
            torch.autograd.grad((lbs(st_req) * G).sum(), st_req)

        ours_fwd_bwd()
        ref_pts = lbs(st)
        ref_grad = torch.autograd.grad((lbs(st_req) * G).sum(), st_req)[0]
        torch.cuda.synchronize()
        agree = {"points_max_abs_diff_rel": float((pts - ref_pts).abs().max() / ref_pts.abs().max().clamp_min(1.0)),
                 "grad_max_abs_diff_rel": float((gst - ref_grad).abs().max() / ref_grad.abs().max().clamp_min(1.0))}
        del ref_pts, ref_grad
        fwd_bytes = 32 * J + 12 * V
        bwd_bytes = 32 * J + 12 * V + 32 * J
        for label, fn, nbytes, iters in (("ours forward", ours_fwd, fwd_bytes, args.iters), ("ours forward+backward", ours_fwd_bwd, fwd_bytes + bwd_bytes, args.iters),
                                         ("torch forward", torch_fwd, fwd_bytes, args.torch_iters),
                                         ("torch forward+backward", torch_fwd_bwd, fwd_bytes + bwd_bytes, args.torch_iters)):
            med, best = timed(fn, args.reps, iters, 2)
            rate = B * nbytes / (med * 1e-6)
            rec = {"case": f"{B} x {rig} (V = {V})", "impl": label, "us_per_call": round(med, 2), "us_best": round(best, 2),
                   "hbm_GB_per_s": rate / 1e9, "share_of_3.35TB_per_s": rate / HBM_BYTES_PER_S, "card": name}
            print(f"{rec['case']:>28} {label:<24} {med:11.2f} us [{best:10.2f}] {rate / 1e9:8.1f} GB/s {100 * rate / HBM_BYTES_PER_S:5.1f} %")
            print(json.dumps(rec))
        print(json.dumps({"case": f"{B} x {rig}", "agreement_with_torch_fp32": agree}))
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
