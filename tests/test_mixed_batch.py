"""cfg5: the mixed-rig bucketing front end (mb2_mixed_batch_*). Bucketing logic runs on the CPU; the solves need a GPU."""
import numpy as np
import pytest

from momentum_b200 import character as mc
from momentum_b200 import solver as ms
from momentum_b200.problems import mixed_problem, mixed_rigs


def _bucket_python(inst, granule=8):
    """Restatement of planBuckets (ik_mixed_batch.cpp): per rig, decreasing count; join the first bucket of the same size class whose
    parents start with the instance's own."""
    order = sorted(range(len(inst)), key=lambda i: (inst[i]["rig"], -len(inst[i]["parents"]), tuple(inst[i]["parents"])))
    buckets, index = [], {}
    for i in order:
        p = tuple(int(x) for x in inst[i]["parents"])
        key = (inst[i]["rig"], (len(p) + granule - 1) // granule)
        for b in index.get(key, []):
            if buckets[b]["parents"][: len(p)] == p:
                buckets[b]["members"].append(i)
                break
        else:
            buckets.append(dict(rig=inst[i]["rig"], parents=p, members=[i]))
            index.setdefault(key, []).append(len(buckets) - 1)
    return buckets


def test_mixed_problem_mix_and_bucketing_waste():
    rigs, inst = mixed_problem(1200, seed=7)
    share = {n: sum(1 for x in inst if x["rig"] == n) / len(inst) for n in rigs}
    assert abs(share["humanoid72"] - 0.5) < 0.06 and abs(share["chain22"] - 0.25) < 0.05 and abs(share["bodyhands300"] - 0.10) < 0.04
    buckets = _bucket_python(inst)
    rows = sum(3 * len(x["parents"]) for x in inst)
    padded = sum(3 * len(b["parents"]) * len(b["members"]) for b in buckets)
    assert padded >= rows and 1.0 - rows / padded < 0.15           # at most granule - 1 padded constraints per instance
    assert len(buckets) <= 4 * 26                                    # (rig, size class) pairs: canonical marker order keeps them few
    for b in buckets:
        for i in b["members"]:
            p = tuple(int(x) for x in inst[i]["parents"])
            assert b["parents"][: len(p)] == p and len(b["parents"]) - len(p) < 8


@pytest.mark.gpu
def test_mixed_batch_matches_the_oracle_instance_by_instance():
    """64 mixed instances through mb2_mixed_batch_solve vs one float-oracle solve per instance (its own rig, constraints, offsets)."""
    from oracle.binding import OracleFunction

    rigs, inst = mixed_problem(64, seed=11)
    mb = ms.MixedBatch()
    rid = {name: mb.add_rig(ch) for name, (ch, _) in rigs.items()}
    for x in inst:
        mb.add_instance(rid[x["rig"]], x["parents"], x["offsets"], x["weights"], x["targets"], x["theta0"])
    st = mb.stats()
    assert st["instances"] == 64 and st["buckets"] == len(_bucket_python(inst)) and st["padded_rows"] >= st["rows"]
    opts = ms.GaussNewtonSolverOptions(min_iterations=8, max_iterations=8, threshold=1.0, regularization=0.05)
    out = mb.solve(opts)
    assert np.all(out["status"] == 0) and np.all(out["iterations"] == 8)
    # Every instance is judged against the reference's float AND double builds on the same inputs: a 22-joint chain that starts far from
    # its targets amplifies rounding several hundred times per iteration, so on this mix the reference's own float result is more than
    # 1e-4 away from its double result on about a third of the instances (scripts/mixed_survey.py
    # measures both the reference's float-vs-double gap and the CUDA-vs-double distance on this mix). The rule: an instance either agrees with the float oracle to 2e-4 / 1e-3 in the
    # objective, or (second look) it stays within 4x the reference's own reproducibility on that instance - its float-vs-double gap and
    # its spread under 2^-21 relative perturbations of the targets (the size of the 3xTF32 rounding, include/momentum_b200.h) - and, over
    # the batch, the CUDA results are not farther from the exact (double) answers than the reference's float build is.
    kw = dict(min_iterations=8, max_iterations=8, threshold=1.0, regularization=0.05)
    worst, second_looks, d_cuda64, d_ref64 = 0.0, [], [], []
    for i, x in enumerate(inst):
        ch = rigs[x["rig"]][0]
        ef = mc.PositionErrorFunction(x["parents"], x["offsets"], x["weights"], x["targets"][None], weight=1.0)
        err, p, it, _ = OracleFunction(ch, [ef], "float32").solve(x["theta0"].astype(np.float64), **kw)
        e64, p64, _, _ = OracleFunction(ch, [ef], "float64").solve(x["theta0"].astype(np.float64), **kw)
        d = np.max(np.abs(out["params"][i] - p)) / max(1.0, np.max(np.abs(p)))
        gap, egap = np.max(np.abs(p - p64)) / max(1.0, np.max(np.abs(p))), abs(err - e64)
        d_cuda64.append(np.max(np.abs(out["params"][i] - p64)) / max(1.0, np.max(np.abs(p64))))
        d_ref64.append(gap)
        worst = max(worst, d)
        etol = 1e-3 * abs(err) + 1e-7
        if d > 2e-4 or abs(out["errors"][i] - err) > etol:
            rng = np.random.default_rng(1000 + i)
            for _ in range(8):
                tg = x["targets"] * (1.0 + 2.0 ** -21 * rng.uniform(-1, 1, x["targets"].shape))
                efp = mc.PositionErrorFunction(x["parents"], x["offsets"], x["weights"], tg[None], weight=1.0)
                ep, pp, _, _ = OracleFunction(ch, [efp], "float32").solve(x["theta0"].astype(np.float64), **kw)
                gap, egap = max(gap, np.max(np.abs(pp - p)) / max(1.0, np.max(np.abs(p)))), max(egap, abs(ep - err))
            second_looks.append((i, x["rig"], float(d), float(gap), float(abs(out["errors"][i] - err)), float(egap)))
            assert d <= max(2e-4, 4.0 * gap) and abs(out["errors"][i] - err) <= etol + 4.0 * egap, (i, x["rig"], len(x["parents"]), second_looks[-1])
    d_cuda64, d_ref64 = np.asarray(d_cuda64), np.asarray(d_ref64)
    print("mixed batch: buckets", st["buckets"], "padding waste %.1f %%" % (100 * st["padding_waste"]), "worst rel param diff", worst,
          "| distance to the double oracle: cuda median %.2e p90 %.2e, reference float median %.2e p90 %.2e" % (np.median(d_cuda64), np.quantile(d_cuda64, 0.9), np.median(d_ref64), np.quantile(d_ref64, 0.9)),
          "| second looks (instance, rig, d, reference spread, error diff, reference error spread)", second_looks)
    # the ill-conditioned instances are no noisier on the device than in the reference
    assert np.median(d_cuda64) <= 2.0 * np.median(d_ref64) + 1e-5
    assert int((d_cuda64 > 2e-4).sum()) <= int((d_ref64 > 2e-4).sum()) + 4, (int((d_cuda64 > 2e-4).sum()), int((d_ref64 > 2e-4).sum()))
    # a second solve from the solutions: bucket handles and plans are reused, nothing gets worse
    for i in range(len(inst)):
        mb.set_parameters(i, out["params"][i])
    out2 = mb.solve(ms.GaussNewtonSolverOptions(min_iterations=2, max_iterations=2, regularization=0.05))
    assert np.all(out2["errors"] <= out["errors"] * (1 + 1e-3) + 1e-9)


@pytest.mark.gpu
def test_instanced_position_offsets_single_bucket():
    """mb2_add_position_error_function_instanced: offsets per batch element, against per-instance oracles."""
    from momentum_b200.problems import humanoid_problem
    from oracle.binding import OracleFunction
    from tests import parity

    ch, efs, theta0, theta_star = humanoid_problem(6, orientation=False)
    rng = np.random.default_rng(3)
    e = efs[0]
    off = np.asarray(e.offsets)[None] + rng.uniform(-1, 1, (6, len(e.parents), 3))
    tg = np.stack([mc.world_points(ch, theta_star[b:b + 1], e.parents, off[b])[0] for b in range(6)])
    ef = mc.PositionErrorFunction(e.parents, e.offsets, e.weights, tg, weight=e.weight, instance_offsets=off)
    opts = ms.GaussNewtonSolverOptions(min_iterations=6, max_iterations=6, regularization=0.05)
    parity.check_solve(ch, [ef], theta0, opts, param_tol=2e-4)
