"""Timing of model_parameters_to_skeleton_state on the device (forward, and forward + backward) against the same forward kinematics
written in plain torch float32 with its autograd backward, on the same GPU.

    python scripts/skeleton_state_bench.py [--reps 5] [--iters 100] [--warmup 20]

Per case it prints the card and its power limit, microseconds per call, instances per second and the achieved HBM bytes per second
from the algorithmic bytes: the forward reads theta and writes the states (4 n + 32 J bytes per instance), the backward reads theta
and the upstream gradient and writes the parameter gradient (4 n + 32 J + 4 n). Times are CUDA events around `iters` calls after a
warm-up; the median of `reps` windows is reported, with the fastest in brackets. There is no CPU path: without a GPU it fails.
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
OP = "model_parameters_to_skeleton_state"


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout
    return out.strip().splitlines()[0]


class TorchFK:
    """The forward kinematics of character.forward_kinematics in float32 torch ops, vectorised over the joints of each tree level."""

    def __init__(self, ch, dev):
        J = ch.num_joints
        P = np.zeros((7 * J, ch.num_params), np.float32)
        rows = np.repeat(np.arange(7 * J), np.diff(ch.pt_outer))
        np.add.at(P, (rows, ch.pt_inner), ch.pt_vals)
        self.P = torch.from_numpy(P).to(dev)
        self.off = torch.from_numpy(ch.pt_offsets).to(dev)
        self.prerot = torch.from_numpy(ch.prerot).to(dev)
        self.offsets = torch.from_numpy(ch.offsets).to(dev)
        depth = ch.depth()
        self.levels = [np.nonzero(depth == d)[0] for d in range(depth.max() + 1)]
        pos = np.zeros(J, np.int64)
        for lv in self.levels:
            pos[lv] = np.arange(len(lv))
        self.lv_idx = [torch.from_numpy(lv).to(dev) for lv in self.levels]
        self.par_pos = [None] + [torch.from_numpy(pos[ch.parents[lv]]).to(dev) for lv in self.levels[1:]]
        self.order = torch.from_numpy(np.argsort(np.concatenate(self.levels))).to(dev)
        self.J = J

    @staticmethod
    def qmul(a, b):
        ax, ay, az, aw = a.unbind(-1)
        bx, by, bz, bw = b.unbind(-1)
        return torch.stack([aw * bx + ax * bw + ay * bz - az * by, aw * by + ay * bw + az * bx - ax * bz,
                            aw * bz + az * bw + ax * by - ay * bx, aw * bw - ax * bx - ay * by - az * bz], -1)

    @staticmethod
    def qrot(q, v):
        u = q[..., :3]
        uv = 2.0 * torch.linalg.cross(u, v)
        return v + q[..., 3:4] * uv + torch.linalg.cross(u, uv)

    def __call__(self, theta):
        B = theta.shape[0]
        jp = (theta @ self.P.T + self.off).reshape(B, self.J, 7)
        ql = self.prerot.expand(B, self.J, 4)
        zero = torch.zeros_like(jp[..., 0])
        for k in (2, 1, 0):
            h = 0.5 * jp[..., 3 + k]
            c = [zero, zero, zero, torch.cos(h)]
            c[k] = torch.sin(h)
            ql = self.qmul(ql, torch.stack(c, -1))
        tl = self.offsets + jp[..., :3]
        sl = torch.exp2(jp[..., 6])
        t, q, s = [], [], []
        for L, idx in enumerate(self.lv_idx):
            if L == 0:
                t.append(tl[:, idx]); q.append(ql[:, idx]); s.append(sl[:, idx])
            else:
                pp = self.par_pos[L]
                tp, qp, sp = t[-1][:, pp], q[-1][:, pp], s[-1][:, pp]
                t.append(tp + self.qrot(qp, sp[..., None] * tl[:, idx])); q.append(self.qmul(qp, ql[:, idx])); s.append(sp * sl[:, idx])
        st = torch.cat([torch.cat(t, 1), torch.cat(q, 1), torch.cat(s, 1)[..., None]], -1)
        return st[:, self.order]


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
        raise SystemExit("skeleton_state_bench: no CUDA device (there is no CPU path)")
    dev = torch.device("cuda", 0)
    name = card()
    print(f"card: {name} (name, power limit)")
    rigs = {"humanoid72": mc.humanoid72()[0], "bodyhands300": mc.bodyhands300()[0]}
    for rig, B in CASES:
        ch = rigs[rig]
        n, J = ch.num_params, ch.num_joints
        rng = np.random.default_rng(0)
        theta = torch.from_numpy(rng.uniform(-0.5, 0.5, (B, n)).astype(np.float32)).to(dev)
        G = torch.from_numpy(rng.normal(size=(B, J, 8)).astype(np.float32)).to(dev)
        dc = tsk._device_character(ch, dev)
        state = torch.empty(B, J, 8, device=dev)
        grad = torch.empty(B, n, device=dev)
        stream = torch.cuda.current_stream(dev).cuda_stream

        def ours_fwd():
            dc.joint_op_device(OP, False, B, theta.data_ptr(), state.data_ptr(), stream=stream)

        def ours_fwd_bwd():
            dc.joint_op_device(OP, False, B, theta.data_ptr(), state.data_ptr(), stream=stream)
            dc.joint_op_device(OP, True, B, theta.data_ptr(), G.data_ptr(), grad.data_ptr(), stream=stream)

        fk = TorchFK(ch, dev)
        th_req = theta.clone().requires_grad_(True)

        def torch_fwd():
            with torch.no_grad():
                fk(theta)

        def torch_fwd_bwd():
            torch.autograd.grad((fk(th_req) * G).sum(), th_req)

        ours_fwd_bwd()
        ref_state = fk(theta)
        ref_grad = torch.autograd.grad((fk(th_req) * G).sum(), th_req)[0]
        torch.cuda.synchronize()
        agree = {"state_max_abs_diff": float((state - ref_state).abs().max()),
                 "grad_max_abs_diff_rel": float((grad - ref_grad).abs().max() / ref_grad.abs().max().clamp_min(1.0))}
        fwd_bytes = 4 * n + 32 * J
        bwd_bytes = 4 * n + 32 * J + 4 * n
        for label, fn, nbytes in (("ours forward", ours_fwd, fwd_bytes), ("ours forward+backward", ours_fwd_bwd, fwd_bytes + bwd_bytes),
                                  ("torch forward", torch_fwd, fwd_bytes), ("torch forward+backward", torch_fwd_bwd, fwd_bytes + bwd_bytes)):
            med, best = timed(fn, args.reps, args.iters, args.warmup)
            rec = {"case": f"{B} x {rig}", "impl": label, "us_per_call": round(med, 2), "us_best": round(best, 2), "instances_per_s": B / (med * 1e-6),
                   "hbm_GB_per_s": B * nbytes / (med * 1e-6) / 1e9, "card": name}
            print(f"{rec['case']:>20} {label:<24} {med:10.2f} us [{best:9.2f}] {rec['instances_per_s'] / 1e6:9.3f} M inst/s {rec['hbm_GB_per_s']:8.1f} GB/s")
            print(json.dumps(rec))
        print(json.dumps({"case": f"{B} x {rig}", "agreement_with_torch_fp32": agree}))


if __name__ == "__main__":
    main()
