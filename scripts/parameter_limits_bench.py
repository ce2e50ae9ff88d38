"""Timing of parameter_limits_residual on the device, forward and forward + backward, against a torch restatement of pymomentum's
``pymomentum.torch.parameter_limits.ParameterLimits`` (rows grouped by limit type, gathers and ``torch.where``, the Ellipsoids through
skeleton-state inverses and point transforms), fed by the device ``apply_parameter_transform`` and ``model_parameters_to_skeleton_state``,
with autograd through all of it. The restatement reads a Linear / LinearJoint range (0, 0) as everywhere, as momentum does, so that its
sum of squares equals ours; pymomentum's module lacks that rule.

    python scripts/parameter_limits_bench.py [--reps 5] [--iters 100] [--warmup 20]

Cases: 8192 x humanoid72, 2048 x bodyhands300 and 256 x humanoid72, each with ``character.synthetic_limits``. Both implementations are
called through torch, so each time includes the Python and autograd work a user pays; the loss is the sum of squares. Per case it prints
the card and its power limit and microseconds per call. Times are CUDA events around `iters` calls after a warm-up; the median of `reps`
windows is reported, with the fastest in brackets. There is no CPU path: without a GPU it fails.
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

CASES = [("humanoid72", 8192), ("bodyhands300", 2048), ("humanoid72", 256)]


class TorchLimits:
    """pymomentum's ParameterLimits module restated (parameter_limits.py), float32, with momentum's (0, 0) range rule"""

    def __init__(self, limits, dev):
        f = lambda v: torch.tensor(v, dtype=torch.float32, device=dev)  # noqa: E731
        i = lambda v: torch.tensor(v, dtype=torch.long, device=dev)  # noqa: E731
        by = lambda t: [lim for lim in limits if lim.type == t]  # noqa: E731
        sw = lambda ls, k=10.0: f([np.sqrt(k * lim.weight) for lim in ls])  # noqa: E731

        def rng(ls):
            lo = [-np.inf if (lim.f[2] == 0 and lim.f[3] == 0) else lim.f[2] for lim in ls]
            hi = [np.inf if (lim.f[2] == 0 and lim.f[3] == 0) else lim.f[3] for lim in ls]
            return f(lo), f(hi)

        mm, mj, li, lj, hp, el = (by(t) for t in (mc.LIMIT_MINMAX, mc.LIMIT_MINMAX_JOINT, mc.LIMIT_LINEAR, mc.LIMIT_LINEAR_JOINT,
                                                  mc.LIMIT_HALFPLANE, mc.LIMIT_ELLIPSOID))
        self.mm = (i([lim.i[0] for lim in mm]), f([lim.f[0] for lim in mm]), f([lim.f[1] for lim in mm]), sw(mm))
        self.mj = (i([7 * lim.i[0] + lim.i[1] for lim in mj]), f([lim.f[0] for lim in mj]), f([lim.f[1] for lim in mj]), sw(mj))
        self.li = (i([lim.i[0] for lim in li]), i([lim.i[1] for lim in li]), f([lim.f[0] for lim in li]), f([lim.f[1] for lim in li]), *rng(li), sw(li))
        self.lj = (i([7 * lim.i[0] + lim.i[1] for lim in lj]), i([7 * lim.i[2] + lim.i[3] for lim in lj]), f([lim.f[0] for lim in lj]),
                   f([lim.f[1] for lim in lj]), *rng(lj), sw(lj))
        self.hp = (i([lim.i[0] for lim in hp]), i([lim.i[1] for lim in hp]), f([lim.f[:2] for lim in hp]), f([lim.f[2] for lim in hp]), sw(hp))
        E = np.array([lim.f for lim in el], np.float32).reshape(-1, 27)
        self.el = (i([lim.i[1] for lim in el]), i([lim.i[0] for lim in el]), f(E[:, 24:27]), f(E[:, :12].reshape(-1, 3, 4)),
                   f(E[:, 12:24].reshape(-1, 3, 4)), sw(el, 10.0 * 1e-4))

    @staticmethod
    def _minmax(x, lo, hi, w):
        return w * (torch.where(x < lo, lo - x, torch.zeros_like(x)) + torch.where(x > hi, x - hi, torch.zeros_like(x)))

    @staticmethod
    def _linear(x, ref, tgt, scale, off, lo, hi, w):
        t = x[:, tgt]
        res = w * (scale * t - off - x[:, ref])
        return torch.where((t >= lo) & (t < hi), res, torch.zeros_like(res))

    def __call__(self, theta, jp, state):
        idx, lo, hi, w = self.mm
        out = [self._minmax(theta[:, idx], lo, hi, w)]
        idx, lo, hi, w = self.mj
        out.append(self._minmax(jp[:, idx], lo, hi, w))
        out.append(self._linear(theta, *self.li))
        out.append(self._linear(jp, *self.lj))
        p1, p2, nrm, off, w = self.hp
        v = theta[:, p1] * nrm[:, 0] + theta[:, p2] * nrm[:, 1] - off
        out.append(w * torch.where(v < 0, v, torch.zeros_like(v)))
        par, epar, offs, M, Mi, w = self.el
        ps, es = state[:, par], state[:, epar]
        x = ps[..., :3] + qrotate(ps[..., 3:7], ps[..., 7:8] * offs)
        qi = es[..., 3:7] * torch.tensor([-1.0, -1.0, -1.0, 1.0], device=state.device)
        local = qrotate(qi, x - es[..., :3]) / es[..., 7:8]
        u = torch.einsum("eij,bej->bei", Mi[:, :, :3], local) + Mi[:, :, 3]
        ep = u / u.norm(dim=-1, keepdim=True)
        proj = torch.einsum("eij,bej->bei", M[:, :, :3], ep) + M[:, :, 3]
        diff = x - (es[..., :3] + qrotate(es[..., 3:7], es[..., 7:8] * proj))
        out.append((w[None, :, None] * diff).flatten(-2))
        return torch.cat(out, -1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("parameter_limits_bench: no CUDA device (there is no CPU path)")
    dev = torch.device("cuda", 0)
    name = card()
    print(f"card: {name} (name, power limit)")
    rigs = {}
    for rig in ("humanoid72", "bodyhands300"):
        ch = getattr(mc, rig)()[0]
        ch.limits = mc.synthetic_limits(ch, seed=0)
        rigs[rig] = ch
    for rig, B in CASES:
        ch = rigs[rig]
        n = ch.num_params
        theta = torch.from_numpy(np.random.default_rng(0).uniform(-1.0, 1.0, (B, n)).astype(np.float32)).to(dev)
        ref = TorchLimits(ch.limits, dev)
        impls = {"ours": lambda t: tsk.parameter_limits_residual(ch, t),
                 "torch ParameterLimits": lambda t: ref(t, tsk.apply_parameter_transform(ch, t), tsk.model_parameters_to_skeleton_state(ch, t))}
        results = {}
        for label, f in impls.items():
            x_req = theta.clone().requires_grad_(True)

            def fwd():
                with torch.no_grad():
                    f(theta)

            def fwd_bwd():
                torch.autograd.grad(f(x_req).square().sum(), (x_req,))

            with torch.no_grad():
                loss = f(theta).double().square().sum(-1)
            results[label] = (loss, torch.autograd.grad(f(x_req).square().sum(), (x_req,))[0])
            for mode, fn in (("forward", fwd), ("forward+backward", fwd_bwd)):
                med, best = timed(fn, args.reps, args.iters, args.warmup)
                rec = {"case": f"{B} x {rig}", "rows": int(f(theta[:1]).shape[1]), "impl": label, "mode": mode, "us_per_call": round(med, 2),
                       "us_best": round(best, 2), "card": name}
                print(f"{rec['case']:>20} {label:<22} {mode:<17} {med:9.2f} us [{best:9.2f}]")
                print(json.dumps(rec))
        (l0, g0), (l1, g1) = results["ours"], results["torch ParameterLimits"]
        print(json.dumps({"case": f"{B} x {rig}", "loss_max_rel_diff": float(((l0 - l1).abs() / l1.abs().clamp_min(1e-30)).max()),
                          "grad_rel": float((g0 - g1).abs().max() / g1.abs().max().clamp_min(1e-30))}))


if __name__ == "__main__":
    main()
