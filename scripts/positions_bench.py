"""Timing of model_parameters_to_positions and joint_parameters_to_positions on the device, forward and forward + backward, against two
compositions a user would otherwise write, on the same GPU:

  skel_state + torch   model_parameters_to_skeleton_state (joint_parameters_to_skeleton_state) on the device, then a torch gather,
                       quaternion rotation and add, with autograd through all of it;
  torch fp32           the whole op restated in float32 torch ops (the ParameterTransform, the FK level by level, the points), with
                       its autograd backward.

    python scripts/positions_bench.py [--reps 5] [--iters 100] [--warmup 20]

Cases: 8192 x humanoid72 with 24 points, 2048 x bodyhands300 with 200 points, 256 x humanoid72 with 24 points; the points are on
seeded random joints, with offsets shared by the batch. Every implementation is called through torch: the positions ops and the
skeleton-state op through their public functions, so each time includes the Python and autograd work a user pays. The forward +
backward differentiates with respect to the parameters and the offsets. Per case it prints the card and its power limit, microseconds
per call, and the achieved HBM bytes per second from the algorithmic bytes: a forward reads the parameters and the offsets and writes
the positions; a backward reads the parameters, the offsets and the upstream gradient and writes both gradients. The share of HBM
bandwidth is that rate over the 3.35 TB/s of NVIDIA's H100 SXM data sheet. Times are CUDA events around `iters` calls after a warm-up;
the median of `reps` windows is reported, with the fastest in brackets. There is no CPU path: without a GPU it fails.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for path in (ROOT, os.path.join(ROOT, "scripts")):
    if path not in sys.path:
        sys.path.insert(0, path)

from joint_parameters_bench import HBM_PEAK, TorchOps, card, qrotate, timed  # noqa: E402

from momentum_b200 import character as mc  # noqa: E402
from momentum_b200 import torch_skeleton as tsk  # noqa: E402

CASES = [("humanoid72", 8192, 24), ("bodyhands300", 2048, 200), ("humanoid72", 256, 24)]


def points_of(state, parents, offsets):
    """t_a + rot(q_a, s_a off) from skeleton states [B, J, 8] by a torch gather (qrotate is Eigen's rotation of a unit q)"""
    st = state.index_select(1, parents)
    return st[..., :3] + qrotate(st[..., 3:7], st[..., 7:8] * offsets)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("positions_bench: no CUDA device (there is no CPU path)")
    dev = torch.device("cuda", 0)
    name = card()
    print(f"card: {name} (name, power limit)")
    rigs = {"humanoid72": mc.humanoid72()[0], "bodyhands300": mc.bodyhands300()[0]}
    for rig, B, N in CASES:
        ch = rigs[rig]
        n, J = ch.num_params, ch.num_joints
        rng = np.random.default_rng(0)
        parents_np = rng.integers(0, J, N).astype(np.int32)
        parents = torch.from_numpy(parents_np.astype(np.int64)).to(dev)
        theta = torch.from_numpy(rng.uniform(-0.5, 0.5, (B, n)).astype(np.float32)).to(dev)
        offsets = torch.from_numpy(rng.normal(scale=0.1, size=(N, 3)).astype(np.float32)).to(dev)
        G = torch.from_numpy(rng.normal(size=(B, N, 3)).astype(np.float32)).to(dev)
        ref = TorchOps(ch, dev)
        jp = tsk.apply_parameter_transform(ch, theta).contiguous()
        for variant, x in (("model", theta), ("joint", jp)):
            ours = tsk.model_parameters_to_positions if variant == "model" else tsk.joint_parameters_to_positions
            state = tsk.model_parameters_to_skeleton_state if variant == "model" else tsk.joint_parameters_to_skeleton_state
            fk32 = (lambda t: ref.joint_parameters_to_skeleton_state(ref.apply_parameter_transform(t))) if variant == "model" \
                else ref.joint_parameters_to_skeleton_state
            impls = {"ours": lambda t, o: ours(ch, t, parents_np, o),
                     "skel_state + torch": lambda t, o: points_of(state(ch, t), parents, o),
                     "torch fp32": lambda t, o: points_of(fk32(t), parents, o)}
            k_in = x.shape[1]
            fwd_bytes = 4 * (B * k_in + 3 * N + 3 * B * N)
            bwd_bytes = 4 * (B * k_in + 3 * N + 3 * B * N) + 4 * (B * k_in + 3 * N)
            results = {}
            for label, f in impls.items():
                x_req, o_req = x.clone().requires_grad_(True), offsets.clone().requires_grad_(True)

                def fwd():
                    with torch.no_grad():
                        f(x, offsets)

                def fwd_bwd():
                    torch.autograd.grad((f(x_req, o_req) * G).sum(), (x_req, o_req))

                with torch.no_grad():
                    out = f(x, offsets)
                grads = torch.autograd.grad((f(x_req, o_req) * G).sum(), (x_req, o_req))
                results[label] = (out, grads)
                for mode, fn, nbytes in (("forward", fwd, fwd_bytes), ("forward+backward", fwd_bwd, fwd_bytes + bwd_bytes)):
                    med, best = timed(fn, args.reps, args.iters, args.warmup)
                    rate = nbytes / (med * 1e-6)
                    rec = {"case": f"{B} x {rig}, N = {N}", "variant": variant, "impl": label, "mode": mode, "us_per_call": round(med, 2),
                           "us_best": round(best, 2), "hbm_GB_per_s": rate / 1e9, "hbm_share_of_3_35_TB_s": rate / HBM_PEAK, "card": name}
                    print(f"{rec['case']:>28} {variant:<6} {label:<20} {mode:<17} {med:9.2f} us [{best:9.2f}] {rate / 1e9:8.1f} GB/s "
                          f"({100 * rate / HBM_PEAK:5.1f} %)")
                    print(json.dumps(rec))
            out, (gx, go) = results["ours"]
            agree = {}
            for label in ("skel_state + torch", "torch fp32"):
                o2, (gx2, go2) = results[label]
                agree[label] = {"positions_max_abs_diff": float((out - o2).abs().max()),
                                "grad_params_rel": float((gx - gx2).abs().max() / gx2.abs().max().clamp_min(1.0)),
                                "grad_offsets_rel": float((go - go2).abs().max() / go2.abs().max().clamp_min(1.0))}
            print(json.dumps({"case": f"{B} x {rig}, N = {N}", "variant": variant, "agreement": agree}))


if __name__ == "__main__":
    main()
