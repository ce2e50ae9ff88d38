"""Timing of collision_residual on the device, forward and forward + backward, against a vectorised torch restatement of the same rows
(the world capsules by gathers over the skeleton states, closestPointsOnSegments over [B, P] pairs with ``torch.where`` for every branch),
with autograd for its backward.

    python scripts/collision_bench.py [--reps 5] [--iters 50] [--warmup 10]

Cases: 8192 x humanoid72 and 2048 x bodyhands300, each with ``character.synthetic_collision``; the states come from random model
parameters through ``model_parameters_to_skeleton_state``. Both implementations are called through torch, so each time includes the Python
and autograd work a user pays; the loss is the sum of squares. Per case it prints the card and its power limit, microseconds per call,
and the bytes the operation has to move (states in, rows out; backward: also the row gradient in and the state gradient out) over that
time. Times are CUDA events around `iters` calls after a warm-up; the median of `reps` windows is reported, with the fastest in brackets.
The outputs of the two implementations are compared. There is no CPU path: without a GPU it fails.
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

from joint_parameters_bench import card, qrotate, timed  # noqa: E402

from momentum_b200 import character as mc  # noqa: E402
from momentum_b200 import torch_skeleton as tsk  # noqa: E402

CASES = [("humanoid72", 8192), ("bodyhands300", 2048)]


class TorchCollision:
    """The rows of collision_residual restated in torch, float32, vectorised over [B, P]"""

    def __init__(self, caps, pairs, dev):
        par, L = mc._capsule_locals(caps)
        self.att = torch.from_numpy(np.nonzero(par >= 0)[0]).to(dev)
        self.par = torch.from_numpy(par[par >= 0]).to(dev)
        self.L = torch.from_numpy(L.astype(np.float32)).to(dev)
        self.i = torch.from_numpy(np.asarray(pairs)[:, 0]).to(dev)
        self.j = torch.from_numpy(np.asarray(pairs)[:, 1]).to(dev)

    def __call__(self, st):
        B = st.shape[0]
        ps = st[:, self.par]
        q = ps[..., 3:7] / ps[..., 3:7].norm(dim=-1, keepdim=True)
        s = ps[..., 7:8]
        La = self.L[self.att]
        geo = self.L.expand(B, -1, -1).clone()
        geo[:, self.att] = torch.cat([ps[..., :3] + qrotate(q, s * La[:, :3]), qrotate(q, s * La[:, 3:6]), La[:, 6:] * s], -1)
        A, Bc = geo[:, self.i], geo[:, self.j]
        zero, one = torch.zeros((), device=st.device), torch.ones((), device=st.device)
        maxd = A[..., 6:].amax(-1) + Bc[..., 6:].amax(-1)
        maxsq = maxd * maxd
        d1, d2 = A[..., 3:6], Bc[..., 3:6]
        w = A[..., :3] - Bc[..., :3]
        dot = lambda x, y: (x * y).sum(-1)  # noqa: E731
        a, b, c, d, e = dot(d1, d1), dot(d1, d2), dot(d2, d2), dot(d1, w), dot(d2, w)
        D = a * c - b * b
        par_ = D < 1e-7
        Dsafe = torch.where(par_, one, D)
        sN0, tN0 = b * e - c * d, a * e - b * d
        line = w + d1 * (sN0 / Dsafe)[..., None] - d2 * (tN0 / Dsafe)[..., None]
        far = torch.where(par_, dot(w, w) > maxsq, dot(line, line) > maxsq)
        sN = torch.where(par_, zero, sN0)
        sD = torch.where(par_, one, D)
        tN = torch.where(par_, e, tN0)
        tD = torch.where(par_, c, D)
        lo, hi = ~par_ & (sN0 < 0), ~par_ & ~(sN0 < 0) & (sN0 > D)
        sN = torch.where(lo, zero, torch.where(hi, sD, sN))
        tN = torch.where(lo, e, torch.where(hi, e + b, tN))
        tD = torch.where(lo | hi, c, tD)
        t0, t1 = tN < 0, ~(tN < 0) & (tN > tD)
        nd, ndb = -d, -d + b
        s_t0 = torch.where(nd < 0, zero, torch.where(nd > a, sD, nd))
        sD_t0 = torch.where((nd < 0) | (nd > a), sD, a)
        s_t1 = torch.where(ndb < 0, zero, torch.where(ndb > a, sD, ndb))
        sD_t1 = torch.where((ndb < 0) | (ndb > a), sD, a)
        sN, sD = torch.where(t0, s_t0, torch.where(t1, s_t1, sN)), torch.where(t0, sD_t0, torch.where(t1, sD_t1, sD))
        tN = torch.where(t0, zero, torch.where(t1, tD, tN))
        sv = torch.where((sN.abs() < 1e-7) | (sD.abs() < 1e-7), zero, sN / torch.where(sD == 0, one, sD))
        tv = torch.where((tN.abs() < 1e-7) | (tD.abs() < 1e-7), zero, tN / torch.where(tD == 0, one, tD))
        dP = w + d1 * sv[..., None] - d2 * tv[..., None]
        dsq = dot(dP, dP)
        dist = dsq.clamp_min(1e-30).sqrt()
        overlap = A[..., 6] + sv * (A[..., 7] - A[..., 6]) + Bc[..., 6] + tv * (Bc[..., 7] - Bc[..., 6]) - dist
        hit = ~far & ~(dsq > maxsq) & (overlap > 0) & (dist >= 1e-8)
        return torch.where(hit, np.sqrt(5e-3) * overlap, zero)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("collision_bench: no CUDA device (there is no CPU path)")
    dev = torch.device("cuda", 0)
    name = card()
    print(f"card: {name} (name, power limit)")
    for rig, B in CASES:
        ch = getattr(mc, rig)()[0]
        ch.collision = mc.synthetic_collision(ch, seed=0)
        pairs = tsk.collision_pairs(ch, dev).numpy()
        P, J = len(pairs), ch.num_joints
        theta = torch.from_numpy(np.random.default_rng(0).normal(scale=0.6, size=(B, ch.num_params)).astype(np.float32)).to(dev)
        st = tsk.model_parameters_to_skeleton_state(ch, theta).detach().contiguous()
        ref = TorchCollision(ch.collision, pairs, dev)
        impls = {"ours": lambda x: tsk.collision_residual(ch, x), "torch restatement": ref}
        bytes_fwd = 4 * (B * J * 8 + B * P)
        bytes_bwd = bytes_fwd + 4 * (B * J * 8 + B * P + B * J * 8)
        results = {}
        for label, f in impls.items():
            x_req = st.clone().requires_grad_(True)

            def fwd():
                with torch.no_grad():
                    f(st)

            def fwd_bwd():
                torch.autograd.grad(f(x_req).square().sum(), (x_req,))

            with torch.no_grad():
                rows = f(st)
            results[label] = (rows, torch.autograd.grad(f(x_req).square().sum(), (x_req,))[0])
            for mode, fn, nbytes in (("forward", fwd, bytes_fwd), ("forward+backward", fwd_bwd, bytes_bwd)):
                med, best = timed(fn, args.reps, args.iters, args.warmup)
                rec = {"case": f"{B} x {rig}", "pairs": P, "impl": label, "mode": mode, "us_per_call": round(med, 2), "us_best": round(best, 2),
                       "bytes": nbytes, "GB_per_s": round(nbytes / med / 1e3, 1), "card": name}
                print(f"{rec['case']:>20} {label:<18} {mode:<17} {med:9.2f} us [{best:9.2f}]  {rec['GB_per_s']:8.1f} GB/s")
                print(json.dumps(rec))
        (r0, g0), (r1, g1) = results["ours"], results["torch restatement"]
        differ = ((r0 != 0) != (r1 != 0)).sum().item()
        both = (r0 != 0) & (r1 != 0)
        print(json.dumps({"case": f"{B} x {rig}", "contacts": int((r0 != 0).sum()), "contact_flags_differ": differ,
                          "rows_max_abs_diff_where_both": float((r0 - r1)[both].abs().max()) if both.any() else 0.0,
                          "loss_rel_diff": float(((r0.double().square().sum() - r1.double().square().sum()) / r1.double().square().sum()).abs()),
                          "grad_rel": float((g0 - g1).abs().max() / g1.abs().max().clamp_min(1e-30))}))


if __name__ == "__main__":
    main()
