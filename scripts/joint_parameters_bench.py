"""Timing of the skeleton-state family on the device (apply_parameter_transform, joint_parameters_to_skeleton_state,
joint_parameters_to_local_skeleton_state, local_skeleton_state_to_joint_parameters, skeleton_state_to_joint_parameters), forward and
forward + backward, against float32 torch restatements of pymomentum's compositions with their autograd backward, on the same GPU.

    python scripts/joint_parameters_bench.py [--reps 5] [--iters 100] [--warmup 20]

Per case it prints the card and its power limit, microseconds per call, instances per second and the achieved HBM bytes per second
from the algorithmic bytes: a forward reads its input and writes its output; a backward reads the forward's input (except the
ParameterTransform's, which is linear) and the upstream gradient and writes the input gradient. The share of HBM bandwidth is that rate
over the 3.35 TB/s of NVIDIA's H100 SXM data sheet. Times are CUDA events around `iters` calls after a warm-up; the median of `reps`
windows is reported, with the fastest in brackets. joint_parameters_to_skeleton_state is also timed beside
model_parameters_to_skeleton_state. There is no CPU path: without a GPU it fails.
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
OPS = ["apply_parameter_transform", "joint_parameters_to_skeleton_state", "joint_parameters_to_local_skeleton_state",
       "local_skeleton_state_to_joint_parameters", "skeleton_state_to_joint_parameters"]


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout
    return out.strip().splitlines()[0]


def qmul(a, b):
    ax, ay, az, aw = a.unbind(-1)
    bx, by, bz, bw = b.unbind(-1)
    return torch.stack([aw * bx + ax * bw + ay * bz - az * by, aw * by + ay * bw + az * bx - ax * bz,
                        aw * bz + az * bw + ax * by - ay * bx, aw * bw - ax * bx - ay * by - az * bz], -1)


def qinverse(q):
    return torch.cat([-q[..., :3], q[..., 3:]], -1) / (q * q).sum(-1, keepdim=True)


def qrotate(q, v):  # quaternionRotateVector
    av = torch.linalg.cross(q[..., :3], v)
    return v + 2 * (av * q[..., 3:4] + torch.linalg.cross(q[..., :3], av))


class TorchOps:
    """pymomentum's compositions in float32 torch ops (the FK level by level, as scripts/skeleton_state_bench.py writes it)"""

    def __init__(self, ch, dev):
        J = ch.num_joints
        P = np.zeros((7 * J, ch.num_params), np.float32)
        rows = np.repeat(np.arange(7 * J), np.diff(ch.pt_outer))
        np.add.at(P, (rows, ch.pt_inner), ch.pt_vals)
        self.P = torch.from_numpy(P).to(dev)
        self.off = torch.from_numpy(ch.pt_offsets).to(dev)
        self.prerot = torch.from_numpy(ch.prerot).to(dev)
        self.offsets = torch.from_numpy(ch.offsets).to(dev)
        self.parents1 = torch.from_numpy(ch.parents.astype(np.int64) + 1).to(dev)
        depth = ch.depth()
        levels = [np.nonzero(depth == d)[0] for d in range(depth.max() + 1)]
        pos = np.zeros(J, np.int64)
        for lv in levels:
            pos[lv] = np.arange(len(lv))
        self.lv_idx = [torch.from_numpy(lv).to(dev) for lv in levels]
        self.par_pos = [None] + [torch.from_numpy(pos[ch.parents[lv]]).to(dev) for lv in levels[1:]]
        self.order = torch.from_numpy(np.argsort(np.concatenate(levels))).to(dev)
        self.J = J

    def apply_parameter_transform(self, theta):
        return theta @ self.P.T + self.off

    def joint_parameters_to_local_skeleton_state(self, jp):
        jp = jp.reshape(jp.shape[0], self.J, 7)
        ql = self.prerot.expand(jp.shape[0], self.J, 4)
        zero = torch.zeros_like(jp[..., 0])
        for k in (2, 1, 0):
            h = 0.5 * jp[..., 3 + k]
            c = [zero, zero, zero, torch.cos(h)]
            c[k] = torch.sin(h)
            ql = qmul(ql, torch.stack(c, -1))
        return torch.cat([self.offsets + jp[..., :3], ql, torch.exp2(jp[..., 6:7])], -1)

    def joint_parameters_to_skeleton_state(self, jp):
        loc = self.joint_parameters_to_local_skeleton_state(jp)
        t, q, s = [], [], []
        for L, idx in enumerate(self.lv_idx):
            tl, ql, sl = loc[:, idx, :3], loc[:, idx, 3:7], loc[:, idx, 7:]
            if L == 0:
                t.append(tl); q.append(ql); s.append(sl)
            else:
                pp = self.par_pos[L]
                tp, qp, sp = t[-1][:, pp], q[-1][:, pp], s[-1][:, pp]
                t.append(tp + qrotate(qp, sp * tl)); q.append(qmul(qp, ql)); s.append(sp * sl)
        return torch.cat([torch.cat(t, 1), torch.cat(q, 1), torch.cat(s, 1)], -1)[:, self.order]

    def local_skeleton_state_to_joint_parameters(self, ls):
        r = qmul(qinverse(self.prerot).expand_as(ls[..., 3:7]), ls[..., 3:7])
        x, y, z, w = r.unbind(-1)
        rx = torch.atan2(2 * (w * x + y * z), 1 - 2 * (x * x + y * y))
        ry = torch.asin((2 * (w * y - z * x)).clamp(-1.0, 1.0))
        rz = torch.atan2(2 * (w * z + x * y), 1 - 2 * (y * y + z * z))
        return torch.cat([ls[..., :3] - self.offsets, torch.stack([rx, ry, rz], -1), torch.log2(ls[..., 7:8])], -1)

    def skeleton_state_to_joint_parameters(self, X):
        ident = torch.zeros_like(X[:, :1])
        ident[..., 6:8] = 1.0
        P = torch.cat([ident, X], 1).index_select(1, self.parents1)
        qi, si = qinverse(P[..., 3:7]), 1.0 / P[..., 7:8]
        loc = torch.cat([-si * qrotate(qi, P[..., :3]) + qrotate(qi, si * X[..., :3]), qmul(qi, X[..., 3:7]), si * X[..., 7:8]], -1)
        return self.local_skeleton_state_to_joint_parameters(loc)


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
        raise SystemExit("joint_parameters_bench: no CUDA device (there is no CPU path)")
    dev = torch.device("cuda", 0)
    name = card()
    print(f"card: {name} (name, power limit)")
    rigs = {"humanoid72": mc.humanoid72()[0], "bodyhands300": mc.bodyhands300()[0]}
    for rig, B in CASES:
        ch = rigs[rig]
        n, J = ch.num_params, ch.num_joints
        rng = np.random.default_rng(0)
        theta = torch.from_numpy(rng.uniform(-0.5, 0.5, (B, n)).astype(np.float32)).to(dev)
        dc = tsk._device_character(ch, dev)
        ref = TorchOps(ch, dev)
        stream = torch.cuda.current_stream(dev).cuda_stream
        jp = tsk.apply_parameter_transform(ch, theta)
        inputs = {"apply_parameter_transform": theta, "joint_parameters_to_skeleton_state": jp, "joint_parameters_to_local_skeleton_state": jp,
                  "local_skeleton_state_to_joint_parameters": tsk.joint_parameters_to_local_skeleton_state(ch, jp).reshape(B, -1),
                  "skeleton_state_to_joint_parameters": tsk.joint_parameters_to_skeleton_state(ch, jp).reshape(B, -1)}
        outs = {"apply_parameter_transform": 7 * J, "joint_parameters_to_skeleton_state": 8 * J, "joint_parameters_to_local_skeleton_state": 8 * J,
                "local_skeleton_state_to_joint_parameters": 7 * J, "skeleton_state_to_joint_parameters": 7 * J}
        for op in OPS:
            x = inputs[op].contiguous()
            k_in, k_out = x.shape[1], outs[op]
            out = torch.empty(B, k_out, device=dev)
            G = torch.from_numpy(rng.normal(size=(B, k_out)).astype(np.float32)).to(dev)
            gx = torch.empty_like(x)
            bwd_ptrs = (G.data_ptr(), gx.data_ptr()) if op == "apply_parameter_transform" else (x.data_ptr(), G.data_ptr(), gx.data_ptr())

            def ours_fwd():
                dc.joint_op_device(op, False, B, x.data_ptr(), out.data_ptr(), stream=stream)

            def ours_fwd_bwd():
                ours_fwd()
                dc.joint_op_device(op, True, B, *bwd_ptrs, stream=stream)

            fn = getattr(ref, op)
            xs = x.reshape(B, J, 8) if op.endswith("to_joint_parameters") else x
            x_req = xs.clone().requires_grad_(True)
            Gs = G.reshape(fn(xs).shape)

            def torch_fwd():
                with torch.no_grad():
                    fn(xs)

            def torch_fwd_bwd():
                torch.autograd.grad((fn(x_req) * Gs).sum(), x_req)

            ours_fwd_bwd()
            ref_out = fn(xs).reshape(B, -1)
            ref_grad = torch.autograd.grad((fn(x_req) * Gs).sum(), x_req)[0].reshape(B, -1)
            torch.cuda.synchronize()
            agree = {"out_max_abs_diff": float((out - ref_out).abs().max()),
                     "grad_max_abs_diff_rel": float((gx - ref_grad).abs().max() / ref_grad.abs().max().clamp_min(1.0))}
            fwd_bytes = 4 * (k_in + k_out)
            bwd_bytes = 4 * (k_out + k_in) + (0 if op == "apply_parameter_transform" else 4 * k_in)
            for label, f, nbytes in (("ours forward", ours_fwd, fwd_bytes), ("ours forward+backward", ours_fwd_bwd, fwd_bytes + bwd_bytes),
                                     ("torch forward", torch_fwd, fwd_bytes), ("torch forward+backward", torch_fwd_bwd, fwd_bytes + bwd_bytes)):
                med, best = timed(f, args.reps, args.iters, args.warmup)
                rate = B * nbytes / (med * 1e-6)
                rec = {"case": f"{B} x {rig}", "op": op, "impl": label, "us_per_call": round(med, 2), "us_best": round(best, 2),
                       "instances_per_s": B / (med * 1e-6), "hbm_GB_per_s": rate / 1e9, "hbm_share_of_3_35_TB_s": rate / HBM_PEAK, "card": name}
                print(f"{rec['case']:>18} {op:<42} {label:<24} {med:9.2f} us [{best:9.2f}] {rate / 1e9:8.1f} GB/s ({100 * rate / HBM_PEAK:5.1f} %)")
                print(json.dumps(rec))
            print(json.dumps({"case": f"{B} x {rig}", "op": op, "agreement_with_torch_fp32": agree}))
        # the FK from joint parameters beside the FK from model parameters
        st = torch.empty(B, J, 8, device=dev)
        jpc = jp.contiguous()
        for label, f in (("model_parameters_to_skeleton_state", lambda: dc.joint_op_device("model_parameters_to_skeleton_state", False, B, theta.data_ptr(),
                                                                                          st.data_ptr(), stream=stream)),
                         ("joint_parameters_to_skeleton_state", lambda: dc.joint_op_device("joint_parameters_to_skeleton_state", False, B, jpc.data_ptr(),
                                                                                          st.data_ptr(), stream=stream))):
            med, best = timed(f, args.reps, args.iters, args.warmup)
            print(f"{B:>7} x {rig:<12} FK {label:<38} {med:9.2f} us [{best:9.2f}]")
            print(json.dumps({"case": f"{B} x {rig}", "fk": label, "us_per_call": round(med, 2), "us_best": round(best, 2), "card": name}))


if __name__ == "__main__":
    main()
