"""Timing of the input contraction of solve_ik's backward (mb2_solver_function_input_gradients_device) against the same contraction
written in float32 torch autograd on the same GPU, and of one whole solve_ik backward split into its parts.

    python scripts/input_gradients_bench.py [--reps 5] [--iters 50] [--warmup 10] [--batch 8192] [--backward-batch 1024 8192] [--no-svd]

1. Kernel: B x humanoid72 with cfg3's constraints (24 Position, 6 Orientation). Per block it prints microseconds per call, instances per
   second and the achieved HBM bytes per second from the algorithmic bytes per instance: theta and v (8 n), the block's records and
   weights, and the three outputs (4 nc (1 + 2 k) with k = 3 or 4). The torch side is grad_theta E . v by double autograd through the
   float32 FK of scripts/skeleton_state_bench.py, differentiated with respect to the same inputs.
2. Backward: one solve_ik backward (Position + Orientation, every input requiring grad) at each --backward-batch, split into the
   direction entry (mb2_solver_function_implicit_direction_device: Jacobian sweep + Jacobi kernel), the input kernels and the rest
   (total minus those). At 1024 one float64 torch.linalg.svd of the same Jacobian, the algorithm the entry replaced, is the comparison.
3. The direction entry alone on humanoid72 with Position + Orientation + Limit + Motion (k = 220) and on 32 x bodyhands300 cfg4
   (k = 424, the Gram matrix in global memory).
Times are CUDA events around `iters` calls after a warm-up; the median of `reps` windows is reported, with the fastest in brackets.
The card and its power limit are printed first. There is no CPU path: without a GPU it fails.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "scripts")):
    if p not in sys.path:
        sys.path.insert(0, p)

from momentum_b200 import character as mc  # noqa: E402
from momentum_b200 import solver as ms  # noqa: E402
from momentum_b200 import torch_ik as ti  # noqa: E402
from momentum_b200 import torch_skeleton as tsk  # noqa: E402
from momentum_b200.problems import add_test_limits, bodyhands_problem, humanoid_problem  # noqa: E402
from skeleton_state_bench import TorchFK, card, timed  # noqa: E402


def qmat(q):
    x, y, z, w = q.unbind(-1)
    return torch.stack([torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)], -1),
                        torch.stack([2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)], -1),
                        torch.stack([2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)], -1)], -2)


def kernel_case(args, dev, name):
    B = args.batch
    ch, efs, _, theta_star = humanoid_problem(B, orientation=True)
    n = ch.num_params
    rng = np.random.default_rng(0)
    theta = torch.from_numpy((theta_star + 0.05 * rng.normal(size=theta_star.shape)).astype(np.float32)).to(dev)
    v = torch.from_numpy(rng.normal(size=(B, n)).astype(np.float32)).to(dev)
    fn = ms.SkeletonSolverFunction(ch, B, efs, device=0)
    fn.upload_targets()
    stream = torch.cuda.current_stream(dev).cuda_stream
    fk = TorchFK(ch, dev)
    for idx, ef in enumerate(efs):
        k = 3 if idx == 0 else 4
        nc = len(ef.parents)
        outs = [torch.empty(B, nc, device=dev), torch.empty(B, nc, k, device=dev), torch.empty(B, nc, k, device=dev)]

        def ours():
            fn.input_gradients_device(idx, theta.data_ptr(), v.data_ptr(), *(o.data_ptr() for o in outs), stream=stream)

        par = torch.from_numpy(np.asarray(ef.parents, np.int64)).to(dev)
        tgt = torch.from_numpy(np.asarray(ef.targets, np.float32)).to(dev)
        off = torch.from_numpy(np.asarray(ef.offsets, np.float32)).to(dev)[None].expand(B, nc, k).contiguous()
        if k == 4:
            tgt, off = tgt / tgt.norm(dim=-1, keepdim=True), off / off.norm(dim=-1, keepdim=True)
        cw = torch.ones(B, nc, device=dev)

        def torch_contraction():
            leaves = [x.clone().requires_grad_(True) for x in (cw, off, tgt)]
            th = theta.clone().requires_grad_(True)
            st = fk(th)[:, par]
            if k == 3:
                f = st[..., :3] + fk.qrot(st[..., 3:7], st[..., 7:8] * leaves[1]) - leaves[2]
            else:
                f = (qmat(st[..., 3:7]) @ qmat(leaves[1]) - qmat(leaves[2])).flatten(2)
            E = (ef.weight * leaves[0] * (f * f).sum(-1)).sum()
            (g,) = torch.autograd.grad(E, th, create_graph=True)
            return torch.autograd.grad((g * v).sum(), leaves)

        ours()
        ref = torch_contraction()
        torch.cuda.synchronize()
        agree = max(float((a - b).abs().max() / b.abs().max().clamp_min(1.0)) for a, b in zip(outs, ref))
        nbytes = 8 * n + 4 * nc * k + 4 * nc + 4 * nc * (1 + 2 * k)
        block = "Position" if k == 3 else "Orientation"
        for label, f in (("ours kernel", ours), ("torch fp32 autograd", torch_contraction)):
            med, best = timed(f, args.reps, args.iters, args.warmup)
            rec = {"case": f"{B} x humanoid72 cfg3 {block} ({nc})", "impl": label, "us_per_call": round(med, 2), "us_best": round(best, 2),
                   "instances_per_s": B / (med * 1e-6), "hbm_GB_per_s": B * nbytes / (med * 1e-6) / 1e9, "bytes_per_instance": nbytes, "card": name}
            print(f"{rec['case']:>42} {label:<20} {med:10.2f} us [{best:9.2f}] {rec['instances_per_s'] / 1e6:8.3f} M inst/s {rec['hbm_GB_per_s']:7.1f} GB/s")
            print(json.dumps(rec))
        print(json.dumps({"case": f"{block}", "max_rel_diff_vs_torch_fp32": agree}))


def backward_case(args, dev, name, B, svd_column):
    """one solve_ik backward at B x humanoid72 cfg3: total, the direction entry (Jacobian sweep + Jacobi kernel), the input kernels and
    the rest; with ``svd_column`` also one float64 torch.linalg.svd of the same Jacobian, the algorithm the entry replaced"""
    ch, efs, _, theta_star = humanoid_problem(B, orientation=True)
    pos, ori = efs
    n = ch.num_params
    f64 = lambda a: torch.from_numpy(np.asarray(a, np.float64)).to(dev)
    opts = ti.SolverOptions(levmar_lambda=0.01, min_iter=4, max_iter=12, threshold=10.0, line_search=True)
    kinds = [ti.ErrorFunctionType.Position, ti.ErrorFunctionType.Orientation]
    active = np.ones(n, bool)
    gout = torch.from_numpy(np.random.default_rng(1).normal(size=(B, n))).to(dev)

    def forward():
        leaves = [f64(x).requires_grad_(True) for x in (pos.offsets, pos.targets, np.ones((B, len(pos.parents))), ori.offsets, ori.targets,
                                                         np.ones((B, len(ori.parents))))]
        out = ti.solve_ik(ch, active, torch.zeros(B, n, device=dev), kinds, torch.tensor([[pos.weight, ori.weight]] * B, device=dev), opts,
                          position_cons_parents=pos.parents, position_cons_offsets=leaves[0], position_cons_targets=leaves[1], position_cons_weights=leaves[2],
                          orientation_cons_parents=ori.parents, orientation_cons_offsets=leaves[3], orientation_cons_targets=leaves[4],
                          orientation_cons_weights=leaves[5])
        return (out.double() * gout).sum()

    def total():
        loss = forward()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        loss.backward()
        b.record()
        b.synchronize()
        return a.elapsed_time(b) * 1e3

    for _ in range(2):
        total()
    t_total = float(np.median([total() for _ in range(args.reps)]))
    [(fn, blocks)] = tsk._handle(ch, dev).solver_functions.values()  # the one solver function the solves above built
    theta = torch.from_numpy(theta_star.astype(np.float32)).to(dev)
    v = torch.from_numpy(np.random.default_rng(2).normal(size=(B, n)).astype(np.float32)).to(dev)
    stream = torch.cuda.current_stream(dev).cuda_stream
    parts = {"direction": direction_us(args, fn, theta, v, stream)}
    outs = {k: [torch.empty(B, len(e.parents), device=dev), torch.empty(B, len(e.parents), kk, device=dev), torch.empty(B, len(e.parents), kk, device=dev)]
            for k, e, kk in (("position", pos, 3), ("orientation", ori, 4))}

    def kernels():
        for k in ("position", "orientation"):
            fn.input_gradients_device(blocks[k], theta.data_ptr(), v.data_ptr(), *(o.data_ptr() for o in outs[k]), stream=stream)

    parts["input_kernels"] = timed(kernels, args.reps, max(1, args.iters // 10), 2)[0]
    parts["rest"] = t_total - sum(parts.values())
    rec = {"case": f"solve_ik backward, {B} x humanoid72 cfg3", "total_us": round(t_total, 1), **{k + "_us": round(x, 1) for k, x in parts.items()}}
    if svd_column:  # a single call: it takes seconds
        rows = 3 * len(pos.parents) + 9 * len(ori.parents)
        ptr, ld = fn.get_jacobian_device(theta.data_ptr(), stream)
        Jd = ti._device_view(ptr, (B, n + 1, ld), dev).clone()[:, :n, :rows].transpose(1, 2).double()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        torch.linalg.svd(Jd, full_matrices=False)
        b.record()
        b.synchronize()
        rec["torch_f64_svd_us"] = round(a.elapsed_time(b) * 1e3, 1)
    rec["card"] = name
    print(json.dumps(rec))


def direction_us(args, fn, theta, g, stream):
    """median microseconds of one mb2_solver_function_implicit_direction_device call (Jacobian sweep + Jacobi kernel)"""
    B, n = theta.shape
    out = [torch.empty(B, n, device=theta.device), torch.empty(B, fn.jacobian_rows, device=theta.device),
           torch.empty(B, fn.jacobian_rows, device=theta.device), torch.empty(B, device=theta.device)]
    f = lambda: fn.implicit_direction_device(theta.data_ptr(), g.data_ptr(), *(o.data_ptr() for o in out), stream=stream)
    return timed(f, args.reps, max(1, args.iters // 10), 2)[0]


def direction_case(args, dev, name, label, ch, efs, B, theta):
    """the direction entry alone on a larger k"""
    fn = ms.SkeletonSolverFunction(ch, B, efs, device=0)
    fn.upload_targets()
    th = torch.from_numpy(np.asarray(theta, np.float32)).to(dev)
    g = torch.from_numpy(np.random.default_rng(3).normal(size=th.shape).astype(np.float32)).to(dev)
    us = direction_us(args, fn, th, g, torch.cuda.current_stream(dev).cuda_stream)
    print(json.dumps({"case": f"implicit direction, {B} x {label}", "direction_us": round(us, 1), "card": name}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--batch", type=int, default=8192)
    ap.add_argument("--backward-batch", type=int, nargs="+", default=[1024, 8192])
    ap.add_argument("--no-svd", action="store_true", help="skip the float64 torch SVD column (seconds per call)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("input_gradients_bench: no CUDA device (there is no CPU path)")
    dev = torch.device("cuda", 0)
    name = card()
    print(f"card: {name} (name, power limit)")
    kernel_case(args, dev, name)
    for B in args.backward_batch:
        backward_case(args, dev, name, B, svd_column=B == 1024 and not args.no_svd)
    # Position + Orientation + Limit + Motion on humanoid72 (k = n_E = 220, the largest Gram matrix in shared memory)
    B = args.backward_batch[0]
    ch, efs, _, star = humanoid_problem(B, orientation=True)
    rng = np.random.default_rng(4)
    add_test_limits(ch, rng, ellipsoid=False)
    efs = efs + [mc.LimitErrorFunction(weight=1.0), mc.ModelParametersErrorFunction(rng.uniform(0.3, 1.0, ch.num_params), star, weight=1.0)]
    direction_case(args, dev, name, "humanoid72 Position + Orientation + Limit + Motion (k = 220)", ch, efs, B, star + 0.05 * rng.normal(size=star.shape))
    # cfg4 (k = 424: the Gram matrix in global memory)
    ch, efs, _, star = bodyhands_problem(32)
    direction_case(args, dev, name, "bodyhands300 cfg4 (k = 424)", ch, efs, 32, star + 0.05 * rng.normal(size=star.shape))


if __name__ == "__main__":
    main()
