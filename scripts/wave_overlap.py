#!/usr/bin/env python
"""What a kernel boundary costs on the cfg3 problem (humanoid72, 24 Position + 6 Orientation, 10 GN iterations per solve).

For B = 528 k (k in 1, 2, 4, 8, 15, 16; 528 = the resident gramCholeskyKernel CTAs of an H100 SXM, four per SM on 132 SMs) and
B = 8192, it times
  * per launch, the sweep (FK + residual + Jacobian) and gramCholeskyKernel: a profiling solve (set_profiling(1): CUDA events around
    every launch, one stream, no instance slices) through get_phase_times;
  * per iteration, the solve as it runs without profiling (events around solve_device, L2 flushed before each solve; instance slices
    where the solve path takes them).
Each is fitted as time = a + b * waves with waves = B / resident CTAs (fractional). The intercept a is what a launch costs beyond its
share of steady-state work: the lock-step first wave, the last partial wave and the drain. Prints the card, its power limit and the
median SM clock over the timed solves. Run it from the repository root after build()."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from bench import ITERS, ClockSampler, make_problem  # noqa: E402
from momentum_b200 import solver as ms  # noqa: E402

GRAM_CHOL_CTAS_PER_SM = 4  # gramCholeskyKernel's launch bound (kGramCholCtasPerSm)


def card():
    import subprocess

    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout
    return out.strip().splitlines()[0]


def measure(B, reps, flush, stream):
    ch, efs, theta0, _ = make_problem("cfg3-shard", B)
    fn = ms.SkeletonSolverFunction(ch, B, efs, device=0)
    fn.upload_targets()
    opts = ms.GaussNewtonSolverOptions(min_iterations=ITERS, max_iterations=ITERS, threshold=1.0, regularization=0.05, fused_mode=ms.FUSED_GRAM_CHOLESKY)
    solver = ms.GaussNewtonSolver(opts, fn)
    theta0_dev = torch.from_numpy(theta0.astype(np.float32)).cuda()
    theta = torch.empty_like(theta0_dev)

    def solve():
        theta.copy_(theta0_dev)
        solver.solve_device(theta.data_ptr(), stream)

    for _ in range(2):
        solve()
    torch.cuda.synchronize()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    iteration_ms, sweep_ms, gc_ms = [], [], []
    slices = None
    for _ in range(reps):
        flush.zero_()
        torch.cuda.synchronize()
        ev0.record()
        solve()
        ev1.record()
        torch.cuda.synchronize()
        iteration_ms.append(ev0.elapsed_time(ev1) / ITERS)
        slices = solver.get_solve_path()["slices"]
        solver.set_profiling(1)
        flush.zero_()
        solve()
        torch.cuda.synchronize()
        solver.get_results()
        pm, pl = solver.get_phase_times()
        solver.set_profiling(0)
        sweep_ms.append(pm[0] / max(pl[0], 1))
        gc_ms.append(pm[2] / max(pl[2], 1))
    return {"B": B, "slices": slices, "sweep_ms": float(np.median(sweep_ms)), "gram_cholesky_ms": float(np.median(gc_ms)),
            "iteration_ms": float(np.median(iteration_ms))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5, help="solves per size (medians are reported)")
    ap.add_argument("--json", default=None, help="also write the rows and fits to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("wave_overlap.py needs a CUDA device")
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    resident = sms * GRAM_CHOL_CTAS_PER_SM
    sizes = [resident * k for k in (1, 2, 4, 8, 15, 16)] + [8192]
    flush = torch.empty(256 * 1024 * 1024 // 4, dtype=torch.float32, device="cuda")
    torch.cuda.set_stream(torch.cuda.Stream())  # a real (non-NULL) stream: NULL means "the handle's own stream" in the C-ABI
    stream = torch.cuda.current_stream().cuda_stream
    sampler = ClockSampler(0)
    sampler.start()
    rows = [measure(B, args.reps, flush, stream) for B in sorted(sizes)]
    clocks = sampler.stop()
    print(f"card: {card()} (name, power limit); median SM clock {clocks['sm_mhz']} MHz (max {clocks['sm_max_mhz']}), clock-event reasons {clocks['reasons']}")
    print(f"resident gramCholeskyKernel CTAs: {resident} ({sms} SMs x {GRAM_CHOL_CTAS_PER_SM})")
    print(f"{'B':>6} {'waves':>6} {'slices':>6} {'sweep ms':>9} {'gramChol ms':>11} {'iteration ms':>12}")
    for r in rows:
        print(f"{r['B']:>6} {r['B'] / resident:>6.2f} {r['slices']:>6} {r['sweep_ms']:>9.4f} {r['gram_cholesky_ms']:>11.4f} {r['iteration_ms']:>12.4f}")
    waves = np.array([r["B"] / resident for r in rows])
    fits = {}
    for key in ("sweep_ms", "gram_cholesky_ms", "iteration_ms"):
        b, a = np.polyfit(waves, np.array([r[key] for r in rows]), 1)
        fits[key] = {"a_us": 1e3 * a, "b_us_per_wave": 1e3 * b}
        per = "iteration" if key == "iteration_ms" else "launch"
        print(f"fit {key:>16}: a = {1e3 * a:7.1f} us per {per}, b = {1e3 * b:6.1f} us per wave")
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"card": card(), "clocks": clocks, "resident": resident, "rows": rows, "fits": fits}, f, indent=1)


if __name__ == "__main__":
    main()
