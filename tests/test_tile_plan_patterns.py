"""The tile-sparse Gram + Cholesky plan (ik_chol_sched.cpp) and the kernels that run it, on generated sparsity patterns.

A pattern is a rig, its error functions and an enabled set, built to hit a structure the planner has to get right: supernodes just
below, at and above one or two 16-wide tiles, many one-column supernodes, deep and wide elimination trees, forests, a parameter that
couples two limbs through the ParameterTransform, alignment gaps, enabled subsets with holes, parameters no constraint reaches, one-row
units that share a row quad with units of other columns, a diagonal-only system, and the sizes where the solve-path rules switch.

CPU (the emulator's plan, tests/emu emu_tile_plan):
* soundness: every structurally non-zero entry of the element-level Cholesky factor of J^T J (from the Jacobian cells, under the dumped
  permutation) lies in a planned tile; perm is a bijection; tile columns start on device columns that are multiples of 4; panels, update
  pairs and vector sources are exactly the ones the planned tiles imply; every dependency of a column sits in an earlier level; the Gram
  tile order deals every tile once;
* the Gram plan: each tile's quad-pair list covers exactly the row quads in which ONE unit touches both tile columns (from the cells);
* the 16-bit tables of the Gram + Cholesky kernel say the same as the schedule, entry for entry;
* a float64 replay of the plan, phase by phase (every item of a phase reads the values of the phase's start), solves (H + lambda I) x = g
  to 1e-10; dropping a fill tile, an update pair or a vector source, moving a column one level early or swapping two perm entries fails
  that replay and the normwise backward-error bound of the tile path by at least 10x;
* one emulated step on the sparse and the dense tile pattern, with the strip Gram and with the K-major JtJ, meets R.solve_limit(n, "tiles")
  and leaves the columns no constraint reaches exactly unchanged.

GPU (-m gpu): one step on every tile path a pattern reaches (the three kernels, K-major 3xTF32, Gram + Cholesky, persistent), each at the
path the emulator chooses under the device's limits and within its R.SOLVE_K bound; Gram + Cholesky bit for bit the three-kernel step;
the persistent kernel at 3, 2 and 1 instance groups on three waves plus a remainder, every instance within the bound and a sample of
instances bit for bit as when solved alone. test_zz_report prints the worst k per path and family.

Path-rule edges (H100 SXM limits, test_solve_path.H100_SXM): the Gram + Cholesky round limit kGramCholMaxRounds = 8 is reached at exactly
8 rounds and refused at 9; the tile kernels run 256 and 512 threads; the persistent kernel runs 3, 2 and 1 instance groups. The persistent
round limit kFusedMaxRounds = 32 is not reached by any generated plan: see test_persistent_round_limit_is_not_reached_by_the_generator."""
import ctypes
import dataclasses

import numpy as np
import pytest

from momentum_b200 import character as mc
from momentum_b200 import solver as ms
from tests import emu_lib
from tests import f64ref as R
from tests.emu_lib import EMU_LIB
from tests.test_solve_path import H100_SXM

GRAM_CHOL_MAX_ROUNDS = 8   # kGramCholMaxRounds (ik_chol_sched.h)
FUSED_MAX_ROUNDS = 32      # kFusedMaxRounds (ik_solve_path.h)
GRAM_WARPS = 8             # kGramWarps

# R.solve_limit(n, path) = SOLVE_K[path] * max(n, 16) * 2^-24 was pinned on humanoid72 and bodyhands300 (n = 212 - 424), where it is
# 13 - 25 ulp (2^-24) for the three tile kernels and about 1 ulp for Gram + Cholesky and persistent. The step's backward error also has a
# part that does not shrink with n: the rounding of each diagonal tile's elimination and of the reciprocal square roots and products with
# W = L^-1 it feeds (test_small_systems_exceed_the_pinned_limit_by_the_factorisation_rounding splits the emulated step into that
# factorisation part and the Gram rounding: the factorisation part alone is 1.1 ulp on a diagonal system of any size and up to 2.2 ulp on
# 15 columns in one tile; the Gram part stays below 0.7 ulp). Where the pinned limit is below that (tiles n <= 33, Gram + Cholesky and
# persistent n < ~2000) the patterns are held to TILE_ROUNDING ulp instead: about 4x the worst measured on an H100 80GB HBM3 (SXM),
# 2.07 ulp (the persistent kernel, 3 instance groups, a diagonal system of 320 columns); single steps measured up to 1.3 ulp there.
# Patterns with expect["pinned"] measured within the pinned limit on every path and stay on it.
TILE_ROUNDING = 8.0


def step_limit(n, key, pinned=False):
    return R.solve_limit(n, key) if pinned else max(R.solve_limit(n, key), TILE_ROUNDING * R.EPS24)


# ------------------------------------------------------------------------------------------------------------------------------
# Pattern generator
# ------------------------------------------------------------------------------------------------------------------------------
@dataclasses.dataclass
class Pattern:
    name: str
    family: str
    ch: object
    efs: list
    enabled: object = None
    expect: dict = dataclasses.field(default_factory=dict)  # plan / path facts the pattern was built for


def _character(parents, dofs, shared=(), seed=0, name="pattern"):
    """Joint j (parents[j], -1 = root) gets one model parameter of its own per joint-parameter row in dofs[j] (0-2 translation, 3-5
    rotation, 6 scale); each entry of `shared` is a list of (joint, row) driven by ONE further model parameter (weight 0.7). Random
    offsets and pre-rotations: no two joints share a table entry."""
    rng = np.random.default_rng(seed)
    parents = np.asarray(parents, np.int32)
    J = len(parents)
    d = rng.normal(size=(J, 3))
    offsets = (d / np.linalg.norm(d, axis=1, keepdims=True) * rng.uniform(0.3, 1.2, (J, 1))).astype(np.float32)
    offsets[parents < 0] = rng.uniform(-2.0, 2.0, (int(np.sum(parents < 0)), 3))
    prerot = np.stack([mc._random_prerot(rng) for _ in range(J)]).astype(np.float32)
    trip, p = [], 0
    for j in range(J):
        for row in dofs[j]:
            trip.append((7 * j + row, p, 1.0))
            p += 1
    for rows in shared:
        for j, row in rows:
            trip.append((7 * j + row, p, 0.7))
        p += 1
    outer, inner, vals = mc._csr_from_triplets(7 * J, p, trip)
    return mc.Character(parents, offsets, prerot, p, outer, inner, vals, np.zeros(7 * J, np.float32), [], name)


def _tree(limbs, root_dofs=(0, 1, 2), limb_dofs=(3,), roots=1):
    """parents + dofs of `roots` roots, each carrying the limbs (joint counts) listed in `limbs` (a list per root, or one list for all);
    returns (parents, dofs, ends, limb joint lists)."""
    parents, dofs, ends, chains = [], [], [], []
    per_root = limbs if isinstance(limbs[0], (list, tuple)) else [limbs] * roots
    for rl in per_root:
        r = len(parents)
        parents.append(-1); dofs.append(tuple(root_dofs))
        for length in rl:
            chain = []
            for k in range(length):
                parents.append(r if k == 0 else len(parents) - 1)
                dofs.append(tuple(limb_dofs))
                chain.append(len(parents) - 1)
            chains.append(chain)
            ends.append(chain[-1])
    return parents, dofs, ends, chains


class _Blocks:
    """Error functions with reachable targets (a pose within +-0.3 of zero) for B instances."""

    def __init__(self, ch, B, seed):
        self.ch, self.B = ch, B
        self.rng = np.random.default_rng(seed)
        self.ts = self.rng.uniform(-0.3, 0.3, (B, ch.num_params))
        self.efs = []

    def position(self, joints, weight=1.0, weights=None):
        joints = np.asarray(joints, np.int32)
        off = self.rng.uniform(-1, 1, (len(joints), 3))
        w = self.rng.uniform(0.5, 1.5, len(joints)) if weights is None else np.asarray(weights, np.float64)
        tg = mc.world_points(self.ch, self.ts, joints, off) + 0.05 * self.rng.normal(size=(self.B, len(joints), 3))
        self.efs.append(mc.PositionErrorFunction(joints, off, w, tg, weight=weight))
        return self

    def orientation(self, joints, weight=0.5):
        from momentum_b200.problems import random_unit_quats, small_rotation_quats

        joints = np.asarray(joints, np.int32)
        off = random_unit_quats(self.rng, (len(joints),))
        tg = mc._qmul(mc.world_rotations(self.ch, self.ts, joints, off), small_rotation_quats(self.rng, (self.B, len(joints)), 0.2))
        self.efs.append(mc.OrientationErrorFunction(joints, off, self.rng.uniform(0.5, 1.5, len(joints)), tg, weight=weight))
        return self

    def state(self, joints, weight=0.7):
        from momentum_b200.problems import small_rotation_quats

        J = self.ch.num_joints
        t, q, s = mc.forward_kinematics(self.ch, self.ts)
        pw, rw = np.zeros(J), np.zeros(J)
        pw[list(joints)], rw[list(joints)] = self.rng.uniform(0.5, 1.5, len(joints)), self.rng.uniform(0.5, 1.5, len(joints))
        tg = np.concatenate([t + 0.05 * self.rng.normal(size=t.shape), mc._qmul(q, small_rotation_quats(self.rng, (self.B, J), 0.2)), s[..., None]], -1)
        self.efs.append(mc.StateErrorFunction(pw, rw, tg, weight=weight, pos_wgt=1.5, rot_wgt=0.8))
        return self

    def plane(self, joints, weight=1.0):
        joints = np.asarray(joints, np.int32)
        off = self.rng.uniform(-1, 1, (len(joints), 3))
        nrm = self.rng.normal(size=(self.B, len(joints), 3))
        unit = nrm / np.linalg.norm(nrm, axis=-1, keepdims=True)
        d = np.sum(unit * mc.world_points(self.ch, self.ts, joints, off), -1) + 0.2 * self.rng.normal(size=(self.B, len(joints)))
        self.efs.append(mc.PlaneErrorFunction(joints, off, self.rng.uniform(0.5, 1.5, len(joints)), np.concatenate([nrm, d[..., None]], -1), weight=weight))
        return self

    def model_parameters(self, target_weights, weight=1.0):
        self.efs.append(mc.ModelParametersErrorFunction(np.asarray(target_weights, np.float64), self.ts + 0.1 * self.rng.normal(size=self.ts.shape), weight=weight))
        return self

    def limits(self, params, weight=0.5):
        """MinMax limits on `params` that theta = 0 violates (every limit row is active at the step's start)."""
        self.ch.limits = [mc.ParameterLimit(mc.LIMIT_MINMAX, 1.0, (int(p),), (0.1, 0.5)) for p in params]
        self.efs.append(mc.LimitErrorFunction(weight=weight))
        return self


def _supernode(w, B, seed):
    """A root (3 translations) with two limbs of w one-DOF joints, Position constraints at the limb ends and half-way: every limb is
    one supernode of w parameters."""
    parents, dofs, ends, chains = _tree([w, w])
    ch = _character(parents, dofs, seed=seed, name=f"limbs{w}")
    bl = _Blocks(ch, B, seed).position(ends + [c[len(c) // 2] for c in chains])
    return ch, bl.efs, chains


def _pattern_specs():
    """name -> (family, builder(B) -> (character, error functions, enabled or None), expected facts)"""
    S = {}

    for w in (15, 16, 17, 31, 32, 33):
        S[f"supernode{w}"] = ("supernode", lambda B, w=w: _supernode(w, B, 100 + w)[:2] + (None,), {})

    def enabled_n(n):
        def build(B):
            ch, efs, chains = _supernode(17, B, 200 + n)
            en = np.zeros(ch.num_params, bool)
            en[[3 + k for k in range(17)][17 - n:]] = True  # the n deepest parameters of the first limb
            return ch, efs, en
        return build
    for n in (1, 15, 16, 17):
        S[f"enabled{n}"] = ("enabled_count", enabled_n(n), dict(enabled=n))

    def star(B):  # 40 one-DOF leaves on a 3-DOF root: 40 one-column supernodes; Planes on four leaves share row quads
        parents, dofs, ends, _ = _tree([1] * 40)
        ch = _character(parents, dofs, seed=301, name="star40")
        return ch, _Blocks(ch, B, 301).position(ends).plane(ends[:4]).efs, None
    S["star40"] = ("star", star, {})

    def deep(B):  # one 72-joint chain, constraints along it: a long supernode, one tile column per level
        parents, dofs, ends, chains = _tree([72], root_dofs=(0, 1, 2, 3, 4, 5))
        ch = _character(parents, dofs, seed=302, name="deep72")
        return ch, _Blocks(ch, B, 302).position(chains[0][5::6]).efs, None
    S["deep72"] = ("deep", deep, dict(min_levels=5, pinned=True))

    def wide(B):  # 14 limbs of 3 two-DOF joints: six-column supernodes, two to a tile, two levels
        parents, dofs, ends, _ = _tree([3] * 14, root_dofs=(0, 1, 2, 3, 4, 5), limb_dofs=(3, 4))
        ch = _character(parents, dofs, seed=303, name="wide14x3")
        return ch, _Blocks(ch, B, 303).position(ends).efs, None
    S["wide14x3"] = ("wide", wide, dict(max_levels=3, pinned=True))

    def forest(B):  # three roots, independent elimination trees
        parents, dofs, ends, chains = _tree([[9, 6], [12], [5, 5, 4]], root_dofs=(0, 1, 2, 3))
        ch = _character(parents, dofs, seed=304, name="forest3")
        return ch, _Blocks(ch, B, 304).position(ends + [c[2] for c in chains]).orientation(ends[:2]).efs, None
    S["forest3"] = ("forest", forest, {})

    def cross(B):  # two parameters each drive joints of two different limbs: fill across the subtrees
        parents, dofs, ends, chains = _tree([8, 8, 8, 8])
        shared = [[(chains[0][3], 4), (chains[2][5], 4)], [(chains[1][6], 5), (chains[3][2], 5)]]
        ch = _character(parents, dofs, shared=shared, seed=305, name="cross4x8")
        return ch, _Blocks(ch, B, 305).position(ends + [c[4] for c in chains]).efs, None
    S["cross4x8"] = ("cross_limb", cross, {})

    def cycle(B):  # six groups of 16 parameters, group k driving limbs k and k - 1: the units' cliques form a 6-cycle of groups, which
        # no elimination order factors without element-level fill between groups that no unit couples (fill tiles)
        G, K, parents, J = 16, 6, [-1], 1
        limbs = []
        for _ in range(K):
            limbs.append(list(range(J, J + 2 * G)))
            parents += [0] + list(range(J, J + 2 * G - 1))
            J += 2 * G
        shared = [[(limbs[k][i], 3), (limbs[(k - 1) % K][G + i], 4)] for k in range(K) for i in range(G)]
        ch = _character(parents, [()] * J, shared=shared, seed=312, name="cycle6x16")
        return ch, _Blocks(ch, B, 312).position([l[-1] for l in limbs] + [l[G + 3] for l in limbs]).efs, None
    S["cycle6x16"] = ("cross_limb", cycle, dict(fill=True))

    def gaps(B):  # supernodes of 5, 7, 9, 6, 3 and 10 parameters: tile columns with 5, 7, 9 ... real columns -> alignment gaps
        parents, dofs, ends, chains = _tree([5, 7, 9, 6, 3, 10])
        ch = _character(parents, dofs, seed=306, name="gaps")
        return ch, _Blocks(ch, B, 306).position(ends).efs, None
    S["gaps"] = ("gaps", gaps, dict(gaps=True))

    def holes(B):  # an enabled subset with holes, one at the first parameter of a limb (a supernode boundary) and one at a limb end
        ch, efs, chains = _supernode(16, B, 307)
        en = np.ones(ch.num_params, bool)
        en[[3, 3 + 7, 3 + 15, 3 + 16, 3 + 16 + 9, 1]] = False
        return ch, efs, en
    S["holes16"] = ("subset", holes, {})

    def holes_rig(B):  # random_rig-style tree with a random 20 % disabled
        from tests.test_sweep_bounds import random_rig

        ch = random_rig(30, 308)
        ch.limits = []
        bl = _Blocks(ch, B, 308).position(np.arange(3, 30, 3))
        en = np.random.default_rng(308).uniform(size=ch.num_params) >= 0.2
        return ch, bl.efs, en
    S["rig30_subset"] = ("subset", holes_rig, {})

    def zero_cols(B):  # a limb that no constraint reaches: its columns are all zero
        parents, dofs, ends, chains = _tree([6, 6, 6], limb_dofs=(3, 5))
        ch = _character(parents, dofs, seed=309, name="zero_limb")
        return ch, _Blocks(ch, B, 309).position(ends[:2] + [chains[0][2]]).efs, None
    S["zero_limb"] = ("zero_columns", zero_cols, dict(zero_columns=True))

    def mix(B):  # 3-row Position, 9-row Orientation, 12-row State units next to one-row Plane / ModelParameters / limit units, zero weights
        parents, dofs, ends, chains = _tree([7, 6, 8, 5], limb_dofs=(3, 4))
        ch = _character(parents, dofs, seed=310, name="mix")
        n = ch.num_params
        bl = _Blocks(ch, B, 310)
        bl.position(ends + [chains[2][3]], weights=[1.0, 0.0, 1.2, 0.8, 0.0])  # two zero-weight constraints
        bl.orientation([ends[0], chains[1][2]]).state([chains[3][1], ends[2]])
        bl.plane([ends[0], ends[1], ends[2], ends[3], chains[0][1]])  # one-row units of different limbs in one row quad
        tw = np.zeros(n); tw[[5, 9, 17, n - 1]] = [0.5, 1.0, 2.0, 0.7]
        bl.model_parameters(tw).limits([4, 12, 20])
        bl.position([chains[1][4]], weight=0.0)  # a zero-weight block: no rows
        return ch, bl.efs, None
    S["mix"] = ("row_units", mix, {})

    def diagonal(B):  # ModelParameters only: every column alone, one level, no panels or updates
        parents, dofs, ends, _ = _tree([4, 4, 4], limb_dofs=(3, 4, 5))
        ch = _character(parents, dofs, seed=311, name="diagonal")
        return ch, _Blocks(ch, B, 311).model_parameters(np.random.default_rng(311).uniform(0.5, 2.0, ch.num_params)).efs, None
    S["diagonal"] = ("diagonal", diagonal, dict(levels=1))

    # ---- path-rule edges: diagonal systems of n parameters (n / 16 tiles of four row quads each, dealt evenly to the 8 Gram warps);
    # the sizes come from planning on the emulator with the H100 SXM limits ----
    def edge(n):
        def build(B):
            nj = (n + 6) // 7 + 1
            ch = _character([-1] + [0] * (nj - 1), [(0, 1, 2, 3, 4, 5, 6)] * nj, seed=n, name=f"diag{n}")
            tw = np.zeros(ch.num_params); tw[:n] = 1.0
            en = np.zeros(ch.num_params, bool); en[:n] = True
            return ch, _Blocks(ch, B, n).model_parameters(tw).efs, en
        return build
    for n, expect in EDGE_SPECS.items():
        S[f"edge{n}"] = ("path_edge", edge(n), dict(expect, levels=1))
    return S


# n -> expected plan / path facts under the H100 SXM limits: Gram tile-order rounds, persistent instance groups (0: the plan does not fit
# one group), whether Gram + Cholesky takes the plan (at most kGramCholMaxRounds = 8 rounds), threads of the tile kernels.
EDGE_SPECS = {
    320: dict(rounds=3, groups=3, gram_cholesky=True, threads=256),
    480: dict(rounds=4, groups=2, gram_cholesky=True, threads=256),
    720: dict(rounds=6, groups=1, gram_cholesky=True, threads=256),
    1024: dict(rounds=8, groups=0, gram_cholesky=True, threads=256),
    1025: dict(rounds=9, groups=0, gram_cholesky=False, threads=256),
    1400: dict(rounds=11, groups=0, gram_cholesky=False, threads=512),
}

_SPECS = None


def specs():
    global _SPECS
    if _SPECS is None:
        _SPECS = _pattern_specs()
    return _SPECS


def make_pattern(name, B=1):
    family, build, expect = specs()[name]
    ch, efs, en = build(B)
    return Pattern(name, family, ch, efs, en, expect)


# ------------------------------------------------------------------------------------------------------------------------------
# The plan as the emulator's planner makes it (emu_tile_plan)
# ------------------------------------------------------------------------------------------------------------------------------
SECTIONS = ["header", "perm", "pos", "device_cols", "tile_row", "tile_col", "tile_id", "diag_tile",
            "level_col_start", "level_cols", "level_panel_start", "panel_tile", "panel_diag", "panel_row",
            "level_task_start", "task_dst", "task_pair_start", "pair_a", "pair_b",
            "level_vtask_start", "vtask_row", "vtask_src_start", "vsrc_tile", "vsrc_col",
            "col_panel_start", "col_panel_tile", "col_panel_row",
            "level_order_start8", "task_order8", "level_order_start16", "task_order16",
            "strip_coord", "tile_pair_start", "gpair_a", "gpair_b", "tile_order", "tile_quad_start", "quad",
            "col_strip_start", "col_strip", "cell_strip_off", "cell_quad_stride", "tab", "cells"]
HEADER = ["n", "n_pad", "tile_cols", "tiles", "levels", "n_params", "rows", "strips", "stride", "resid_off", "park_tiles", "tables_valid",
          "L_gram", "L_quad", "L_col", "L_colEnt", "L_level", "L_diag", "L_panel", "L_order", "L_pair", "L_vtask", "L_vsrc", "L_colPanel"]


@pytest.fixture(scope="module")
def emu():
    emu_lib.build()
    L = ms.load_library(EMU_LIB)
    L.emu_tile_plan.argtypes = [ctypes.c_void_p, ctypes.c_int32, ctypes.c_void_p, ctypes.POINTER(ctypes.c_int64)]
    L.emu_gram_system.argtypes = [ctypes.c_void_p, ctypes.c_int32, ctypes.c_int32, ctypes.c_void_p, ctypes.c_void_p, ctypes.POINTER(ctypes.c_int64)]
    L.emu_set_device_limits(*H100_SXM)
    return L


def emu_function(p, B=1):
    fn = ms.SkeletonSolverFunction(p.ch, B, p.efs, lib_path=EMU_LIB)
    fn.upload_targets()
    if p.enabled is not None:
        fn.set_enabled_parameters(p.enabled)
    return fn


def tile_plan(emu, fn, chol_mode):
    """The dumped plan: a dict of int64 arrays by section name, the header's fields as ints."""
    words = ctypes.c_int64(0)
    assert emu.emu_tile_plan(fn._h, chol_mode, None, ctypes.byref(words)) == 0, emu.mb2_last_error()
    buf = np.zeros(words.value, np.int32)
    assert emu.emu_tile_plan(fn._h, chol_mode, buf.ctypes.data, ctypes.byref(words)) == 0, emu.mb2_last_error()
    out, k = {}, 0
    for name in SECTIONS:
        ln = int(buf[k])
        out[name] = buf[k + 1:k + 1 + ln].astype(np.int64)
        k += 1 + ln
    assert k == words.value
    out.update({h: int(v) for h, v in zip(HEADER, out.pop("header"))})
    out["cells"] = out["cells"].reshape(-1, 5)
    out["strip_coord"] = out["strip_coord"].reshape(-1, 2)
    out["tab"] = out["tab"] & 0xFFFF
    T = out["tile_cols"]
    out["tile_id"] = out["tile_id"].reshape(T, T)
    return out


def _tile_idx():
    """tileIdx (ik_chol_sched.cuh): float offset of X(r, c) in a tile's fragment layout, as a [16, 16] array"""
    out = np.zeros((16, 16), np.int64)
    for r in range(16):
        for c in range(16):
            lane = ((r & 7) << 2) | ((c & 7) >> 1)
            out[r, c] = ((c >> 3) << 7) + ((lane ^ (lane >> 3)) << 2) + (((r >> 3) << 1) | (c & 1))
    return out


TILE_IDX = _tile_idx()


def gram_system(emu, fn, P, chol_mode, theta, b=0):
    """(H, g) over device columns as the emulator's tile-sparse Gram rounds them (float32 values in float64; no damping) for instance b"""
    floats = ctypes.c_int64(0)
    assert emu.emu_gram_system(fn._h, chol_mode, b, None, None, ctypes.byref(floats)) == 0, emu.mb2_last_error()
    out = np.zeros(floats.value, np.float32)
    th = np.ascontiguousarray(theta, np.float32)
    assert emu.emu_gram_system(fn._h, chol_mode, b, th.ctypes.data, out.ctypes.data, ctypes.byref(floats)) == 0, emu.mb2_last_error()
    perm, n = P["perm"], P["n"]
    npad = len(perm)
    Hs = np.zeros((npad, npad))
    for t in range(P["tiles"]):
        I, J = int(P["tile_row"][t]), int(P["tile_col"][t])
        X = out[256 * t:256 * t + 256][TILE_IDX].astype(np.float64)
        Hs[16 * I:16 * I + 16, 16 * J:16 * J + 16] = X
        if I != J:
            Hs[16 * J:16 * J + 16, 16 * I:16 * I + 16] = X.T
    ys = out[256 * P["tiles"]:].astype(np.float64)
    idx = np.nonzero(perm >= 0)[0]
    H, g = np.zeros((n, n)), np.zeros(n)
    H[np.ix_(perm[idx], perm[idx])] = Hs[np.ix_(idx, idx)]
    g[perm[idx]] = ys[idx]
    return H, g


def gram_term(emu, fn, J, r, cols, lam, b=0, chol_mode=ms.CHOLESKY_TILES_SPARSE):
    """The Gram part of the backward error of a step from theta = 0 on instance b of the emulator function fn: the normwise backward
    error, against the float64 J^T J of (J, r), of the EXACT solution of the emulator's rounded Gram system. Also returns that system
    (damping not included) over `cols` (model parameters)."""
    P = tile_plan(emu, fn, chol_mode)
    Hd, gd = gram_system(emu, fn, P, chol_mode, np.zeros(fn.num_parameters), b)
    at = {int(c): d for d, c in enumerate(P["device_cols"]) if c >= 0}
    sel = [at[int(c)] for c in cols]
    Hc, gc = Hd[np.ix_(sel, sel)], gd[sel]
    x = np.linalg.solve(Hc + lam * np.eye(len(cols)), gc)
    return R.backward_error(J, r, cols, x, lam), Hc, gc


@dataclasses.dataclass
class View:
    """The schedule as lists: what the checks and the float64 replay read, and what the mutations edit."""
    n: int
    T: int
    perm: np.ndarray                 # [nPad] slot -> device column, -1 = padding
    tiles: dict                      # (I, J) -> tile id
    levels: list                     # per level: dict(cols, panels [(tile, diag, row)], tasks [(dst, [(a, b)])], vtasks [(row, [(tile, K)])])
    col_panels: dict                 # K -> [(tile, row)]
    diag: dict                       # K -> diagonal tile


def view_of(P):
    T = P["tile_cols"]
    tiles = {(int(P["tile_row"][t]), int(P["tile_col"][t])): t for t in range(P["tiles"])}
    levels = []
    for L in range(P["levels"]):
        cols = [int(K) for K in P["level_cols"][P["level_col_start"][L]:P["level_col_start"][L + 1]]]
        panels = [(int(P["panel_tile"][i]), int(P["panel_diag"][i]), int(P["panel_row"][i])) for i in range(P["level_panel_start"][L], P["level_panel_start"][L + 1])]
        tasks = [(int(P["task_dst"][t]), [(int(P["pair_a"][p]), int(P["pair_b"][p])) for p in range(P["task_pair_start"][t], P["task_pair_start"][t + 1])])
                 for t in range(P["level_task_start"][L], P["level_task_start"][L + 1])]
        vtasks = [(int(P["vtask_row"][v]), [(int(P["vsrc_tile"][s]), int(P["vsrc_col"][s])) for s in range(P["vtask_src_start"][v], P["vtask_src_start"][v + 1])])
                  for v in range(P["level_vtask_start"][L], P["level_vtask_start"][L + 1])]
        levels.append(dict(cols=cols, panels=panels, tasks=tasks, vtasks=vtasks))
    col_panels = {K: [(int(P["col_panel_tile"][i]), int(P["col_panel_row"][i])) for i in range(P["col_panel_start"][K], P["col_panel_start"][K + 1])] for K in range(T)}
    diag = {K: int(P["diag_tile"][K]) for K in range(T)}
    return View(P["n"], T, P["perm"].copy(), tiles, levels, col_panels, diag)


# ------------------------------------------------------------------------------------------------------------------------------
# Independent references: the pattern from the cells, its element-level fill, the Gram quads
# ------------------------------------------------------------------------------------------------------------------------------
def unit_columns(P):
    """unit -> (first row, row count, sorted device columns) from the cell list"""
    units = {}
    for r0, rows, col, unit, _ in P["cells"]:
        u = units.setdefault(int(unit), [int(r0), int(rows), set()])
        u[2].add(int(col))
    return {u: (r0, rows, sorted(c)) for u, (r0, rows, c) in units.items()}


def element_fill(P, perm):
    """[nPad, nPad] bool lower pattern of the Cholesky factor of J^T J (+ diagonal) under the slot order `perm`: the cliques of the units'
    columns, then symbolic elimination column by column in slot order."""
    npad = len(perm)
    slot_of = {int(d): s for s, d in enumerate(perm) if d >= 0}
    A = np.eye(npad, dtype=bool)
    for _, _, cols in unit_columns(P).values():
        s = [slot_of[c] for c in cols]
        A[np.ix_(s, s)] = True
    A = np.tril(A)
    for j in range(npad):  # column j's structure merges into its rows': L(i, k) != 0 for i, k in struct(j)
        below = np.nonzero(A[j + 1:, j])[0] + j + 1
        if below.size:
            A[np.ix_(below, below)] |= np.tril(np.ones((below.size, below.size), bool))
    return A


def tile_closure(P):
    """The tile set the planner must produce: the tile image of the units' cliques, then tile-level symbolic factorisation."""
    T = P["tile_cols"]
    pos = P["pos"]
    S = np.eye(T, dtype=bool)
    for _, _, cols in unit_columns(P).values():
        ks = sorted({int(pos[c]) >> 4 for c in cols})
        for a in ks:
            for b in ks:
                if a >= b:
                    S[a, b] = True
    for K in range(T):
        st = [I for I in range(K + 1, T) if S[I, K]]
        for a in st:
            for b in st:
                if a >= b:
                    S[a, b] = True
    return S


def required_quads(P):
    """(I, J) -> set of row quads q in which ONE unit has rows and cells in tile columns I and J (I >= J)"""
    pos = P["pos"]
    need = {}
    for r0, rows, cols in unit_columns(P).values():
        ks = sorted({int(pos[c]) >> 4 for c in cols})
        for q in range(r0 >> 2, ((r0 + rows - 1) >> 2) + 1):
            for a in ks:
                for b in ks:
                    if a >= b:
                        need.setdefault((a, b), set()).add(q)
    return need


# ------------------------------------------------------------------------------------------------------------------------------
# Checks of a plan
# ------------------------------------------------------------------------------------------------------------------------------
class PlanError(AssertionError):
    pass


def _need(cond, msg):
    if not cond:
        raise PlanError(msg)


def check_schedule(P, V):
    """Soundness of the schedule view V against the pattern of the dumped cells."""
    T, n = V.T, V.n
    perm = V.perm
    real = perm[perm >= 0]
    dev = P["device_cols"]
    _need(len(perm) == 16 * T, "perm length")
    _need(len(np.unique(real)) == len(real), "perm repeats a device column")
    _need(set(real.tolist()) == set(np.nonzero(dev >= 0)[0].tolist()), "perm is not a bijection onto the real device columns")
    _need(len(dev) == n, "device column count")
    for K in range(T):
        blk = perm[16 * K:16 * K + 16]
        v = int(np.sum(blk >= 0))
        _need(v >= 1 and np.all(blk[:v] >= 0) and np.all(blk[v:] < 0), f"tile column {K}: padding inside the tile")
        _need(blk[0] % 4 == 0, f"tile column {K} starts on device column {blk[0]}")
        _need(np.all(np.diff(blk[:v]) == 1), f"tile column {K}: device columns not contiguous")
    # every non-zero of the element-level factor in a planned tile
    F = element_fill(P, perm)
    r, c = np.nonzero(F)
    for I, J in {(int(a) >> 4, int(b) >> 4) for a, b in zip(r, c)}:
        _need((I, J) in V.tiles, f"factor entry in tile ({I},{J}) which is not planned")
    for K in range(T):
        _need(V.diag.get(K) == V.tiles.get((K, K)), f"diagonal tile of column {K}")
    # levels: each column once, dependencies earlier
    level = {}
    for L, lv in enumerate(V.levels):
        for K in lv["cols"]:
            _need(K not in level, f"column {K} in two levels")
            level[K] = L
    _need(sorted(level) == list(range(T)), "columns missing from the levels")
    for (I, J) in V.tiles:
        if I > J:
            _need(level[J] < level[I], f"column {I} depends on column {J} of level {level[J]} but sits in level {level[I]}")
    below = {K: sorted(I for (I, J) in V.tiles if J == K and I > K) for K in range(T)}
    for L, lv in enumerate(V.levels):
        cols = lv["cols"]
        want_panels = sorted((V.tiles[(I, K)], V.diag[K], I) for K in cols for I in below[K])
        _need(sorted(lv["panels"]) == want_panels, f"level {L}: panels")
        want_tasks = {}
        for K in cols:
            for a in below[K]:
                for b in below[K]:
                    if a >= b:
                        _need((a, b) in V.tiles, f"update destination ({a},{b}) not planned")
                        want_tasks.setdefault(V.tiles[(a, b)], []).append((V.tiles[(a, K)], V.tiles[(b, K)]))
        got = {}
        for dst, pairs in lv["tasks"]:
            _need(dst not in got, f"level {L}: two update tasks for tile {dst}")
            got[dst] = sorted(pairs)
        _need(got == {k: sorted(v) for k, v in want_tasks.items()}, f"level {L}: update pairs differ from {{(L(I,K), L(J,K))}}")
        sources = {V.tiles[(I, K)] for K in cols for I in below[K]} | {V.diag[K] for K in cols}
        _need(not (set(got) & sources), f"level {L}: an update writes a tile the level reads")
        want_v = {}
        for K in cols:
            for I in below[K]:
                want_v.setdefault(I, []).append((V.tiles[(I, K)], K))
        gotv = {}
        for row, srcs in lv["vtasks"]:
            _need(row not in gotv, f"level {L}: two vector tasks for block {row}")
            gotv[row] = sorted(srcs)
        _need(gotv == {k: sorted(v) for k, v in want_v.items()}, f"level {L}: vector-task sources")
    for K in range(T):
        _need(V.col_panels[K] == [(V.tiles[(I, K)], I) for I in below[K]], f"column {K}: backward-substitution panels")


def check_task_orders(P):
    for W in (8, 16):
        start, order = P[f"level_order_start{W}"], P[f"task_order{W}"]
        for L in range(P["levels"]):
            sec = order[start[L]:start[L + 1]]
            _need(len(sec) % W == 0, "task order section not whole rounds")
            got = sorted(int(t) for t in sec if t >= 0)
            _need(got == list(range(P["level_task_start"][L], P["level_task_start"][L + 1])), f"{W}-warp task order of level {L}")


def check_gram(P, sparse=True):
    """The Gram plan against the quads derived from the cells (sparse: the tile set is the tile-level fill of the units' cliques, dense:
    every lower tile)."""
    pos, perm = P["pos"], P["perm"]
    sc = P["strip_coord"]
    strip_qk = [(int(r) >> 2, int(pos[d]) >> 4) for r, d in sc]
    zero = P["stride"] // 64
    need = required_quads(P)
    tiles = {(int(P["tile_row"][t]), int(P["tile_col"][t])): t for t in range(P["tiles"])}
    closure = tile_closure(P) if sparse else np.tril(np.ones((P["tile_cols"], P["tile_cols"]), bool))
    _need(set(tiles) == {(int(a), int(b)) for a, b in zip(*np.nonzero(closure))}, "planned tiles differ from the tile-level fill of the unit cliques")
    for (I, J), t in tiles.items():
        pa = P["gpair_a"][P["tile_pair_start"][t]:P["tile_pair_start"][t + 1]]
        pb = P["gpair_b"][P["tile_pair_start"][t]:P["tile_pair_start"][t + 1]]
        _need(len(pa) % 2 == 0, f"tile {t}: odd pair list")
        quads = []
        for a, b in zip(pa, pb):
            if a == zero or b == zero:
                _need(a == zero and b == zero, f"tile {t}: half a padding pair")
                continue
            (qa, ka), (qb, kb) = strip_qk[a], strip_qk[b]
            _need(qa == qb and ka == I and kb == J, f"tile {t} ({I},{J}): pair of strips ({qa},{ka}) x ({qb},{kb})")
            quads.append(qa)
        _need(len(quads) == len(set(quads)), f"tile {t}: a quad twice")
        _need(set(quads) == need.get((I, J), set()), f"tile ({I},{J}): quads {sorted(quads)} != required {sorted(need.get((I, J), set()))}")
        q4 = P["quad"][4 * P["tile_quad_start"][t]:4 * P["tile_quad_start"][t + 1]].reshape(-1, 4)
        _need(np.array_equal(q4[:, [0, 2]].ravel(), pa * 64) and np.array_equal(q4[:, [1, 3]].ravel(), pb * 64), f"tile {t}: quad records")
    order = P["tile_order"]
    _need(len(order) % GRAM_WARPS == 0 and sorted(int(t) for t in order if t >= 0) == list(range(P["tiles"])), "tileOrder does not deal every tile once")
    for k in range(P["tile_cols"]):
        got = sorted(strip_qk[s] for s in P["col_strip"][P["col_strip_start"][k]:P["col_strip_start"][k + 1]])
        _need(got == sorted(sq for sq in strip_qk if sq[1] == k), f"strips of tile column {k}")
    for i, (r0, rows, col, _, _) in enumerate(P["cells"]):
        s, off = divmod(int(P["cell_strip_off"][i]), 64)
        _need(strip_qk[s] == (int(r0) >> 2, int(pos[col]) >> 4) and off // 4 == col - perm[16 * (int(pos[col]) >> 4)] and off % 4 == 0, f"cell {i} outside its strip")


def _valid(perm, K):
    return int(np.sum(perm[16 * K:16 * K + 16] >= 0))


def check_tables(P):
    """GramCholTables (16-bit, decoded here from its layout) entry for entry against the schedule and the Gram plan."""
    if P["tables_valid"] == 0:  # an entry past 16 bits: the solve path does not offer Gram + Cholesky (gramCholValid), which needs <= 8 rounds
        _need(len(P["tile_order"]) // GRAM_WARPS > GRAM_CHOL_MAX_ROUNDS, "16-bit tables refused for a plan within the Gram + Cholesky rounds")
        return
    tab, perm = P["tab"], P["perm"]

    def rec(sec, i, w):
        o = P["L_" + sec] + w * i
        return [int(x) for x in tab[o:o + w]]
    for i, t in enumerate(P["tile_order"]):
        r = rec("gram", i, 4)
        if t < 0:
            _need(r[0] == 0xFFFF, f"gram entry {i} should be idle")
            continue
        I, J = int(P["tile_row"][t]), int(P["tile_col"][t])
        _need(r == [int(t), _valid(perm, I) | _valid(perm, J) << 8 | (I == J) << 15, int(P["tile_quad_start"][t]), int(P["tile_quad_start"][t + 1])], f"gram entry {i}")
    for i, v in enumerate(P["quad"]):
        _need(rec("quad", i, 1)[0] == v, f"quad {i}")
    for i, v in enumerate(P["col_strip_start"]):
        _need(rec("col", i, 1)[0] == v, f"col {i}")
    for i, s in enumerate(P["col_strip"]):
        _need(rec("colEnt", i, 2) == [int(s) * 64, int(P["strip_coord"][s][0])], f"colEnt {i}")
    for L in range(P["levels"] + 1):
        _need(rec("level", L, 4) == [int(P["level_col_start"][L]), int(P["level_panel_start"][L]), int(P["level_order_start8"][L]), int(P["level_vtask_start"][L])], f"level {L}")
    for i, K in enumerate(P["level_cols"]):
        _need(rec("diag", i, 4) == [int(K), int(P["diag_tile"][K]), int(P["col_panel_start"][K]), int(P["col_panel_start"][K + 1])], f"diag {i}")
    for i in range(len(P["panel_tile"])):
        _need(rec("panel", i, 2) == [int(P["panel_tile"][i]), int(P["panel_diag"][i])], f"panel {i}")
    for i, t in enumerate(P["task_order8"]):
        r = rec("order", i, 4)
        want = [0xFFFF] if t < 0 else [int(P["task_dst"][t]), int(P["task_pair_start"][t]), int(P["task_pair_start"][t + 1]), 0]
        _need(r[:len(want)] == want, f"order {i}")
    for i in range(len(P["pair_a"])):
        _need(rec("pair", i, 2) == [int(P["pair_a"][i]), int(P["pair_b"][i])], f"pair {i}")
    for i in range(len(P["vtask_row"])):
        _need(rec("vtask", i, 4) == [int(P["vtask_row"][i]), int(P["vtask_src_start"][i]), int(P["vtask_src_start"][i + 1]), 0], f"vtask {i}")
    for i in range(len(P["vsrc_tile"])):
        _need(rec("vsrc", i, 2) == [int(P["vsrc_tile"][i]), int(P["vsrc_col"][i])], f"vsrc {i}")
    for i in range(len(P["col_panel_tile"])):
        _need(rec("colPanel", i, 2) == [int(P["col_panel_tile"][i]), int(P["col_panel_row"][i])], f"colPanel {i}")


# ------------------------------------------------------------------------------------------------------------------------------
# Float64 replay of the schedule
# ------------------------------------------------------------------------------------------------------------------------------
def _chol16(A, fallback):
    """Cholesky factor of a diagonal tile; a non-positive pivot is replaced by `fallback` as cholDiagTile does (a mutated plan can
    leave a tile indefinite)."""
    A = np.tril(A).copy()
    A = A + np.tril(A, -1).T
    L = np.zeros_like(A)
    for k in range(16):
        piv = A[k, k]
        if not piv > 0:
            piv = fallback
        L[k, k] = np.sqrt(piv)
        L[k + 1:, k] = A[k + 1:, k] / L[k, k]
        A[k + 1:, k + 1:] -= np.outer(L[k + 1:, k], L[k + 1:, k])
    return L


def replay(V, Hd, gd, fallback=0.05):
    """Solve (Hd) x = gd (device-column space, damping included) by running the schedule V in float64, phase by phase as the kernels do:
    every item of a phase reads the tiles / right-hand side as they were when the phase started. Entries of H outside the planned tiles
    are not loaded (the kernels never see them). Returns x over device columns (gaps 0) and the factor tiles."""
    perm = V.perm
    npad = len(perm)
    real = perm >= 0
    Hs = np.zeros((npad, npad))
    idx = np.nonzero(real)[0]
    Hs[np.ix_(idx, idx)] = Hd[np.ix_(perm[idx], perm[idx])]
    X = {}
    for (I, J), t in V.tiles.items():
        blk = Hs[16 * I:16 * I + 16, 16 * J:16 * J + 16].copy()
        if I == J:
            pad = ~real[16 * I:16 * I + 16]
            blk[pad, :] = 0.0; blk[:, pad] = 0.0
            blk[pad, pad] = 1.0
        X[t] = blk
    y = np.zeros(npad)
    y[idx] = gd[perm[idx]]
    for lv in V.levels:
        old = {k: v.copy() for k, v in X.items()}
        y0 = y.copy()
        for K in lv["cols"]:  # phase A: W = L(K,K)^-1 into the diagonal tile, y_K = W y_K
            d = V.diag[K]
            W = np.linalg.inv(_chol16(old[d], fallback))
            X[d] = W
            y[16 * K:16 * K + 16] = W @ y0[16 * K:16 * K + 16]
        old = {k: v.copy() for k, v in X.items()}
        for tile, diag, _ in lv["panels"]:  # phase B: L(I,K) = A(I,K) W^T
            if tile in old and diag in old:
                X[tile] = old[tile] @ old[diag].T
        old = {k: v.copy() for k, v in X.items()}
        y0 = y.copy()
        acc = {}
        for dst, pairs in lv["tasks"]:  # phase C: updates and vector tasks from the phase's start
            for a, b in pairs:
                if a in old and b in old and dst in old:
                    acc[dst] = acc.get(dst, 0.0) + old[a] @ old[b].T
        for dst, s in acc.items():
            X[dst] = old[dst] - s
        for row, srcs in lv["vtasks"]:
            s = np.zeros(16)
            for tile, K in srcs:
                if tile in old:
                    s += old[tile] @ y0[16 * K:16 * K + 16]
            y[16 * row:16 * row + 16] = y0[16 * row:16 * row + 16] - s
    for lv in reversed(V.levels):  # backward substitution, a level's columns from the level's start
        y0 = y.copy()
        for K in lv["cols"]:
            s = y0[16 * K:16 * K + 16].copy()
            for tile, I in V.col_panels[K]:
                if tile in X:
                    s -= X[tile].T @ y0[16 * I:16 * I + 16]
            y[16 * K:16 * K + 16] = X[V.diag[K]].T @ s
    x = np.zeros(len(gd))
    x[perm[idx]] = y[idx]
    return x, X


def normal_equations(fn, P, lam, theta):
    """(J [rows, n] float64 of the emulator at theta, r, H over device columns + lam I, g over device columns, device-column -> model
    parameter map)"""
    J, r = R.jacobian64(fn, theta)
    J, r = J[0], r[0]
    dev = P["device_cols"]
    Jd = np.zeros((J.shape[0], len(dev)))
    Jd[:, dev >= 0] = J[:, dev[dev >= 0]]
    Hd = Jd.T @ Jd + lam * np.diag((dev >= 0).astype(float))
    return J, r, Hd, Jd.T @ r, dev


def replay_case(fn, P, V, lam=0.05):
    """(relative error against np.linalg.solve, normwise backward error, n, limit) of the replayed step"""
    theta = np.zeros((1, fn.num_parameters), np.float32)
    J, r, Hd, gd, dev = normal_equations(fn, P, lam, theta)
    with np.errstate(all="ignore"):
        try:
            x, _ = replay(V, Hd, gd, lam)
        except np.linalg.LinAlgError:
            x = np.full(len(gd), np.nan)
    real = dev >= 0
    if not np.all(np.isfinite(x)):  # a broken plan can overflow: that fails every check
        return np.inf, np.inf, int(np.sum(real)), R.solve_limit(int(np.sum(real)), "tiles")
    ref = np.linalg.solve(Hd[np.ix_(real, real)], gd[real])
    rel = float(np.max(np.abs(x[real] - ref)) / max(np.max(np.abs(ref)), 1e-300))
    cols = dev[real]
    be = R.backward_error(J, r, cols, x[real], lam)
    return rel, be, len(cols), R.solve_limit(len(cols), "tiles")


# ------------------------------------------------------------------------------------------------------------------------------
# Mutations of the plan (each a plan bug the checks must see)
# ------------------------------------------------------------------------------------------------------------------------------
def _copy(V):
    return dataclasses.replace(V, perm=V.perm.copy(), tiles=dict(V.tiles),
                               levels=[dict(cols=list(l["cols"]), panels=list(l["panels"]), tasks=[(d, list(p)) for d, p in l["tasks"]],
                                            vtasks=[(r, list(s)) for r, s in l["vtasks"]]) for l in V.levels],
                               col_panels={k: list(v) for k, v in V.col_panels.items()}, diag=dict(V.diag))


def _factor(fn, P, V):
    theta = np.zeros((1, fn.num_parameters), np.float32)
    _, _, Hd, gd, _ = normal_equations(fn, P, 0.05, theta)
    x, X = replay(V, Hd, gd)
    return Hd, gd, X


def mutations(fn, P, V):
    """name -> mutated view (the most consequential candidate of each kind on this pattern), or absent when the kind does not apply"""
    Hd, gd, X = _factor(fn, P, V)
    nrm = {t: float(np.abs(v).max()) for t, v in X.items()}
    out = {}
    pattern_tiles = {(int(a), int(b)) for a, b in zip(*np.nonzero(_tile_image(P)))}
    fill = [(I, J) for (I, J) in V.tiles if (I, J) not in pattern_tiles]
    if fill:
        I, J = max(fill, key=lambda ij: nrm[V.tiles[ij]])
        t = V.tiles[(I, J)]
        M = _copy(V)
        del M.tiles[(I, J)]
        for lv in M.levels:
            lv["panels"] = [p for p in lv["panels"] if p[0] != t]
            lv["tasks"] = [(d, [(a, b) for a, b in ps if a != t and b != t]) for d, ps in lv["tasks"] if d != t]
            lv["vtasks"] = [(r, [s for s in ss if s[0] != t]) for r, ss in lv["vtasks"]]
        M.col_panels = {k: [p for p in v if p[0] != t] for k, v in M.col_panels.items()}
        out["drop_fill_tile"] = M
    pairs = [(L, i, j) for L, lv in enumerate(V.levels) for i, (_, ps) in enumerate(lv["tasks"]) for j in range(len(ps))]
    if pairs:
        def size(k):
            L, i, j = k
            a, b = V.levels[L]["tasks"][i][1][j]
            return float(np.abs(X[a] @ X[b].T).max())
        def dropped(k):
            M = _copy(V)
            del M.levels[k[0]]["tasks"][k[1]][1][k[2]]
            return M
        # of the six largest products, the one whose loss moves the replayed step most
        out["drop_update_pair"] = max((dropped(k) for k in sorted(pairs, key=size)[-6:]), key=lambda M: replay_case(fn, P, M)[1])
    if len(V.levels) > 1:
        # the column of level >= 1 with the largest incoming update
        level = {K: L for L, lv in enumerate(V.levels) for K in lv["cols"]}
        inc = {}
        for L, lv in enumerate(V.levels):
            for dst, ps in lv["tasks"]:
                inc[dst] = inc.get(dst, 0.0) + sum(float(np.abs(X[a] @ X[b].T).max()) for a, b in ps)
        K = max((K for K in level if level[K] >= 1), key=lambda K: inc.get(V.diag[K], 0.0))
        L = level[K]
        M = _copy(V)
        src = {V.tiles[(I, J)] for (I, J) in V.tiles if J == K}
        M.levels[L]["cols"].remove(K)
        M.levels[L - 1]["cols"].append(K)
        mv = [p for p in M.levels[L]["panels"] if p[1] == V.diag[K]]
        M.levels[L]["panels"] = [p for p in M.levels[L]["panels"] if p[1] != V.diag[K]]
        M.levels[L - 1]["panels"] += mv
        keep, move = [], []
        for d, ps in M.levels[L]["tasks"]:
            a = [pq for pq in ps if pq[0] not in src]
            b = [pq for pq in ps if pq[0] in src]
            if a:
                keep.append((d, a))
            if b:
                move.append((d, b))
        M.levels[L]["tasks"] = keep
        M.levels[L - 1]["tasks"] += move
        keepv, movev = [], []
        for r, ss in M.levels[L]["vtasks"]:
            a = [s for s in ss if s[1] != K]
            b = [s for s in ss if s[1] == K]
            if a:
                keepv.append((r, a))
            if b:
                movev.append((r, b))
        M.levels[L]["vtasks"] = keepv
        M.levels[L - 1]["vtasks"] += movev
        out["move_column_earlier"] = M
    srcs = [(L, i, j) for L, lv in enumerate(V.levels) for i, (_, ss) in enumerate(lv["vtasks"]) for j in range(len(ss))]
    if srcs:
        # the source with the largest L(I,K) y_K in the replay (y after the forward pass is enough to rank them)
        x, _ = replay(V, Hd, gd)
        def size(k):
            L, i, j = k
            t, K = V.levels[L]["vtasks"][i][1][j]
            return nrm[t] * float(np.abs(gd).max())
        L, i, j = max(srcs, key=size)
        M = _copy(V)
        del M.levels[L]["vtasks"][i][1][j]
        out["drop_vector_source"] = M
    # swap two perm entries: the real slot whose column, moved into another tile column, loses the largest coupling of H to tiles that
    # are not planned (swapped with that tile column's first slot)
    perm, T = V.perm, V.T
    real = np.nonzero(perm >= 0)[0]
    tile_of = np.full(Hd.shape[0], -1)
    tile_of[perm[real]] = real // 16
    dg = np.sqrt(np.abs(np.diag(Hd)))
    with np.errstate(all="ignore"):
        C = np.nan_to_num(np.abs(Hd) / np.outer(dg, dg))
    planned = np.zeros((T, T), bool)
    for (I, J) in V.tiles:
        planned[I, J] = planned[J, I] = True
    best = None
    for s in real:
        d = perm[s]
        nz = np.nonzero((C[d] > 0) & (tile_of >= 0))[0]
        nz = nz[nz != d]
        for Bc in range(T):
            if Bc == s // 16:
                continue
            lost = float(np.max(C[d, nz][~planned[Bc, tile_of[nz]]], initial=0.0))
            if best is None or lost > best[0]:
                best = (lost, s, 16 * Bc)
    if best is not None and best[0] > 0:
        M = _copy(V)
        _, sa, sb = best
        M.perm[[sa, sb]] = M.perm[[sb, sa]]
        out["swap_perm"] = M
    return out


def _tile_image(P):
    T = P["tile_cols"]
    pos = P["pos"]
    S = np.eye(T, dtype=bool)
    for _, _, cols in unit_columns(P).values():
        ks = sorted({int(pos[c]) >> 4 for c in cols})
        for a in ks:
            for b in ks:
                if a >= b:
                    S[a, b] = True
    return S


# ------------------------------------------------------------------------------------------------------------------------------
# CPU tests
# ------------------------------------------------------------------------------------------------------------------------------
PATTERNS = list(specs())
MODES = {"sparse": ms.CHOLESKY_TILES_SPARSE, "dense": ms.CHOLESKY_TILES_DENSE}
CPU_WORST = {}


def _note(table, key, family, k):
    table[(key, family)] = max(table.get((key, family), 0.0), k)


@pytest.mark.parametrize("name", PATTERNS)
def test_plan_is_sound_and_the_replay_solves(name, emu):
    p = make_pattern(name)
    fn = emu_function(p)
    for mode_name, mode in MODES.items():
        P = tile_plan(emu, fn, mode)
        V = view_of(P)
        check_schedule(P, V)
        check_task_orders(P)
        check_gram(P, mode_name == "sparse")
        check_tables(P)
        rel, be, n, lim = replay_case(fn, P, V)
        print(f"\n[{name} {mode_name}] n={n} tiles={P['tiles']} levels={P['levels']} gaps={int(np.sum(P['device_cols'] < 0))} "
              f"rounds={len(P['tile_order']) // GRAM_WARPS} replay rel {rel:.2e} backward error {be:.2e}")
        assert rel <= 1e-10, (name, mode_name, rel)
        assert be <= 1e-3 * lim, (name, mode_name, be)
        ex = p.expect
        if mode_name == "sparse":
            if "levels" in ex:
                assert P["levels"] == ex["levels"] and len(P["panel_tile"]) == 0 and len(P["task_dst"]) == 0
            if "min_levels" in ex:
                assert P["levels"] >= ex["min_levels"]
            if "max_levels" in ex:
                assert P["levels"] <= ex["max_levels"]
            if ex.get("gaps"):
                assert np.any(P["device_cols"] < 0)
            if "enabled" in ex:
                assert int(np.sum(P["device_cols"] >= 0)) == ex["enabled"]
            if "rounds" in ex:
                assert len(P["tile_order"]) // GRAM_WARPS == ex["rounds"], (name, len(P["tile_order"]) // GRAM_WARPS)
            fill = set(V.tiles) - {(int(a), int(b)) for a, b in zip(*np.nonzero(_tile_image(P)))}
            assert bool(fill) == bool(ex.get("fill")), (name, sorted(fill))
        else:
            assert len(P["tile_row"]) == P["tile_cols"] * (P["tile_cols"] + 1) // 2


@pytest.mark.parametrize("name", [n for n in PATTERNS if specs()[n][0] != "diagonal"])
def test_plan_mutations_fail_the_checks_by_10x(name, emu):
    p = make_pattern(name)
    fn = emu_function(p)
    P = tile_plan(emu, fn, ms.CHOLESKY_TILES_SPARSE)
    V = view_of(P)
    muts = mutations(fn, P, V)
    assert {"drop_update_pair", "move_column_earlier", "drop_vector_source"} <= set(muts) or P["levels"] == 1, (name, sorted(muts))
    if p.expect.get("fill"):  # the pattern with tile-level fill runs all five kinds
        assert set(muts) == set(MUTATION_KINDS), (name, sorted(muts))
    rows = []
    for kind, M in muts.items():
        with pytest.raises(PlanError):
            check_schedule(P, M)
        rel, be, n, lim = replay_case(fn, P, M)
        rows.append((kind, f"rel {rel:.2e}", f"be/limit {be / lim:.1f}"))
        _note(MUTATION_MARGIN, kind, name, be / lim)
        assert rel > 1e-10 and be > 10 * lim, (name, kind, rel, be, lim)
    print(f"\n[{name}] mutations:", rows)


MUTATION_MARGIN = {}
MUTATION_KINDS = ("drop_fill_tile", "drop_update_pair", "move_column_earlier", "drop_vector_source", "swap_perm")


STEP_CASES = {  # name: (cholesky mode, jtj mode)
    "sparse_gram": (ms.CHOLESKY_TILES_SPARSE, ms.JTJ_AUTO),
    "dense_gram": (ms.CHOLESKY_TILES_DENSE, ms.JTJ_AUTO),
    "sparse_kmajor": (ms.CHOLESKY_TILES_SPARSE, ms.JTJ_TF32X3),
    "dense_kmajor": (ms.CHOLESKY_TILES_DENSE, ms.JTJ_TF32X3),
}


def _opts(**kw):
    base = dict(min_iterations=1, max_iterations=1, threshold=1.0, regularization=0.05, fused_mode=ms.FUSED_OFF)
    base.update(kw)
    return ms.GaussNewtonSolverOptions(**base)


def _zero_columns(J, cols):
    return np.array([np.all(J[:, :, c] == 0) for c in cols], bool)


@pytest.mark.parametrize("name", PATTERNS)
def test_emulated_step_meets_the_tile_bound(name, emu):
    p = make_pattern(name)
    emu.emu_set_device_limits(*H100_SXM)
    for case, (chol, jtj) in STEP_CASES.items():
        if p.family == "path_edge" and chol == ms.CHOLESKY_TILES_DENSE:
            continue  # the dense pattern of these diagonal systems (20 - 88 tile columns) does not fit the tile schedule
        if jtj == ms.JTJ_TF32X3 and p.family == "path_edge" and p.expect["rounds"] >= 6:
            continue  # 720 columns and more: past the tensor-core JtJ's 512-column shape (the solver refuses the K-major request)
        solver, out, J, r, cols, delta, lam = R.one_step(p.ch, p.efs, np.zeros((1, p.ch.num_params)), _opts(cholesky_mode=chol, jtj_mode=jtj),
                                                         EMU_LIB, enabled=p.enabled, rel_damping=1e-5)
        path = solver.get_solve_path()
        assert path["kind"] == ("tiles" if jtj == ms.JTJ_AUTO else "tiles_kmajor"), (name, case, path)
        assert np.all(out["status"] == 0)
        be = R.backward_error(J[0], r[0], cols, delta[0], lam)
        lim = step_limit(len(cols), "tiles", p.expect.get("pinned", False))
        _note(CPU_WORST, "emu_" + case, p.family, be / R.solve_limit(len(cols), "tiles") * R.SOLVE_K["tiles"])
        assert be <= lim, (name, case, be, lim)
        z = _zero_columns(J, cols)
        assert np.all(delta[0][z] == 0.0), (name, case)
        if p.expect.get("zero_columns"):
            assert z.any()


GRAM_SPLIT = {}


@pytest.mark.parametrize("name", PATTERNS)
def test_small_systems_exceed_the_pinned_limit_by_the_factorisation_rounding(name, emu):
    """Where the excess over the pinned limit comes from. The emulated strip-Gram step d is split into its backward error against the
    emulator's own rounded Gram system (H~ + lambda I) d = g~ (the factorisation's part, normalised with the float64 |J|^T |J|) and the
    backward error of the exact solution of that rounded system (the Gram rounding, gram_term); the step's error is at most their sum.
    The Gram part stays below one ulp everywhere; the factorisation part is within the pinned tile limit wherever that limit is above
    TILE_ROUNDING, and within TILE_ROUNDING where it is not."""
    p = make_pattern(name)
    emu.emu_set_device_limits(*H100_SXM)
    for case in ("sparse_gram", "dense_gram"):
        chol, jtj = STEP_CASES[case]
        if p.family == "path_edge" and chol == ms.CHOLESKY_TILES_DENSE:
            continue
        _, out, J, r, cols, delta, lam = R.one_step(p.ch, p.efs, np.zeros((1, p.ch.num_params)), _opts(cholesky_mode=chol, jtj_mode=jtj),
                                                     EMU_LIB, enabled=p.enabled, rel_damping=1e-5)
        gram, Hc, gc = gram_term(emu, emu_function(p), J[0], r[0], cols, lam, chol_mode=chol)
        _, _, E, _ = R.normal_equations64(J[0], r[0], cols)
        d = delta[0]
        fact = float(np.max(np.abs((Hc + lam * np.eye(len(cols))) @ d - gc)) / ((np.max(E.sum(axis=1)) + lam) * np.max(np.abs(d)) + np.max(np.abs(gc))))
        be = R.backward_error(J[0], r[0], cols, d, lam)
        n = len(cols)
        GRAM_SPLIT[(name, case)] = (be / R.EPS24, fact / R.EPS24, gram / R.EPS24)
        print(f"\n[{name} {case}] n={n} step {be / R.EPS24:.2f} ulp = factorisation {fact / R.EPS24:.2f} + Gram {gram / R.EPS24:.2f}; pinned tile limit "
              f"{R.solve_limit(n, 'tiles') / R.EPS24:.2f} ulp")
        assert fact <= step_limit(n, "tiles"), (name, case, fact)
        assert gram <= R.EPS24, (name, case, gram)
        assert be <= 1.01 * (fact + gram) + 1e-3 * R.EPS24, (name, case, be, fact, gram)


# ------------------------------------------------------------------------------------------------------------------------------
# GPU: every tile path a pattern reaches
# ------------------------------------------------------------------------------------------------------------------------------
GPU_PATHS = {  # name: (options, SOLVE_K key)
    "tiles_sparse": (dict(cholesky_mode=ms.CHOLESKY_TILES_SPARSE, jtj_mode=ms.JTJ_AUTO, fused_mode=ms.FUSED_OFF), "tiles"),
    "tiles_dense": (dict(cholesky_mode=ms.CHOLESKY_TILES_DENSE, jtj_mode=ms.JTJ_AUTO, fused_mode=ms.FUSED_OFF), "tiles"),
    "kmajor_tf32x3": (dict(cholesky_mode=ms.CHOLESKY_TILES_SPARSE, jtj_mode=ms.JTJ_TF32X3, fused_mode=ms.FUSED_OFF), "tiles"),
    "gram_cholesky": (dict(cholesky_mode=ms.CHOLESKY_TILES_SPARSE, jtj_mode=ms.JTJ_AUTO, fused_mode=ms.FUSED_GRAM_CHOLESKY), "gram_cholesky"),
    "persistent": (dict(cholesky_mode=ms.CHOLESKY_TILES_SPARSE, jtj_mode=ms.JTJ_AUTO, fused_mode=ms.FUSED_PERSISTENT), "persistent"),
}
GPU_WORST = {}
REACHED = {}


def _device_limits():
    import torch

    q = torch.cuda.get_device_properties(0)
    return q.multi_processor_count, q.shared_memory_per_block_optin, q.shared_memory_per_multiprocessor


def _emu_choice(emu, p, opts, B, limits):
    emu.emu_set_device_limits(*limits)
    fn = emu_function(p, B)
    solver = ms.GaussNewtonSolver(opts, fn)
    rc = emu.emu_choose_solve_path(solver._h)
    return solver.get_solve_path(), (emu.mb2_last_error().decode() if rc != 0 else None)


def _reached(path):
    kind = path["kind"]
    if kind in ("tiles", "tiles_kmajor"):
        return f"{kind}_{path['chol_threads']}"
    if kind == "persistent":
        return f"persistent_{path['fused_groups']}_groups"
    return kind


@pytest.mark.gpu
@pytest.mark.parametrize("name", PATTERNS)
def test_gpu_tile_paths_on_the_pattern(name, emu):
    p = make_pattern(name)
    limits = _device_limits()
    th0 = np.zeros((1, p.ch.num_params))
    steps = {}
    for path_name, (kw, key) in GPU_PATHS.items():
        opts = _opts(**kw)
        want, err = _emu_choice(emu, p, opts, 1, limits)
        if err is not None:  # the library refuses with the emulator's message
            fn = ms.SkeletonSolverFunction(p.ch, 1, p.efs)
            fn.upload_targets()
            if p.enabled is not None:
                fn.set_enabled_parameters(p.enabled)
            with pytest.raises(ms.MomentumB200Error) as e:
                ms.GaussNewtonSolver(opts, fn).solve(th0.astype(np.float32))
            assert str(e.value) == err, (name, path_name, str(e.value), err)
            continue
        solver, out, J, r, cols, delta, lam = R.one_step(p.ch, p.efs, th0, opts, enabled=p.enabled, rel_damping=1e-5)
        got = solver.get_solve_path()
        assert got == want, (name, path_name, got, want)
        assert np.all(out["status"] == 0), out["status"]
        be = R.backward_error(J[0], r[0], cols, delta[0], lam)
        n = len(cols)
        k = be / R.solve_limit(n, key) * R.SOLVE_K[key]
        _note(GPU_WORST, _reached(got), p.family, k)
        REACHED.setdefault(_reached(got), []).append(name)
        lim = step_limit(n, key, p.expect.get("pinned", False))
        print(f"\n[{name} {path_name}] {_reached(got)} n={n} backward error {be:.3e} k {k:.5f} limit {lim:.3e}")
        assert be <= lim, (name, path_name, be, lim)
        prof = solver.get_fused_profile()
        fused = {"persistent": 1, "gram_cholesky": 2}.get(got["kind"], 0)
        assert prof["fused"] == fused and prof["groups"] == (got["fused_groups"] if fused == 1 else 0), (name, path_name, prof, got)
        z = _zero_columns(J, cols)
        assert np.all(delta[0][z] == 0.0), (name, path_name)
        steps[path_name] = out["params"]
    if "gram_cholesky" in steps:  # the Gram + Cholesky kernel runs the three-kernel arithmetic: bit for bit
        assert np.array_equal(steps["gram_cholesky"], steps["tiles_sparse"]), name
    ex = p.expect
    if "groups" in ex:
        assert ("persistent" in steps) == (ex["groups"] > 0) and ("gram_cholesky" in steps) == ex["gram_cholesky"], (name, sorted(steps))


def _instances(efs, idx):
    out = []
    for e in efs:
        t = getattr(e, "targets", None)
        out.append(dataclasses.replace(e, targets=np.asarray(t)[idx]) if t is not None and np.ndim(t) >= 2 else e)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("groups", [3, 2, 1])
def test_gpu_persistent_batch_at_each_group_count(groups, emu):
    """Three waves of instance groups plus a remainder on the persistent kernel: every instance within the bound, a seeded sample bit for
    bit as when solved alone."""
    n = {g: k for k, v in EDGE_SPECS.items() for g in [v["groups"]]}[groups]
    limits = _device_limits()
    B = 3 * groups * limits[0] + 17
    p = make_pattern(f"edge{n}", B)
    kw, key = GPU_PATHS["persistent"]
    opts = _opts(**kw)
    want, err = _emu_choice(emu, p, opts, B, limits)
    assert err is None and want["fused_groups"] == groups, (want, err)
    rng = np.random.default_rng(groups)
    th0 = np.zeros((B, p.ch.num_params), np.float32)
    fn = ms.SkeletonSolverFunction(p.ch, B, p.efs)
    fn.upload_targets()
    fn.set_enabled_parameters(p.enabled)
    solver = ms.GaussNewtonSolver(opts, fn)
    full = solver.solve(th0)
    assert solver.get_solve_path() == want and solver.get_fused_profile()["groups"] == groups
    assert np.all(full["status"] == 0)
    cols = np.nonzero(p.enabled)[0]
    lim = step_limit(len(cols), key)
    worst = 0.0
    for c0 in range(0, B, 128):  # every instance's step against its own float64 normal equations, 128 instances at a time
        idx = np.arange(c0, min(B, c0 + 128))
        f = ms.SkeletonSolverFunction(p.ch, len(idx), _instances(p.efs, idx))
        f.upload_targets()
        f.set_enabled_parameters(p.enabled)
        J, r = R.jacobian64(f, th0[idx])
        for k, b in enumerate(idx):
            be = R.backward_error(J[k], r[k], cols, -full["params"][b, cols].astype(np.float64), float(np.float32(0.05)))
            worst = max(worst, be)
            assert be <= lim, (groups, b, be, lim)
    _note(GPU_WORST, f"persistent_{groups}_groups_batch", "path_edge", worst / R.solve_limit(len(cols), key) * R.SOLVE_K[key])
    for b in rng.choice(B, 8, replace=False):
        one = ms.SkeletonSolverFunction(p.ch, 1, _instances(p.efs, [b]))
        one.upload_targets()
        one.set_enabled_parameters(p.enabled)
        alone = ms.GaussNewtonSolver(opts, one).solve(th0[b:b + 1])
        assert np.array_equal(alone["params"][0], full["params"][b]), (groups, b)


def test_persistent_round_limit_is_not_reached_by_the_generator(emu):
    """kFusedMaxRounds = 32 is not reached: the largest plan of the generator the persistent kernel takes has 6 rounds (edge720, one
    instance group); edge1024 (8 rounds), which Gram + Cholesky still takes, is refused by the persistent kernel because one instance
    group does not fit in shared memory, not because of its rounds. Plans of 32 rounds need many tiles or very uneven tile loads; none
    of the generated ones fits one group."""
    emu.emu_set_device_limits(*H100_SXM)
    p = make_pattern("edge720")
    want, err = _emu_choice(emu, p, _opts(**GPU_PATHS["persistent"][0]), 1, H100_SXM)
    assert err is None and want["fused_groups"] == 1
    p = make_pattern("edge1024")
    want, err = _emu_choice(emu, p, _opts(**GPU_PATHS["persistent"][0]), 1, H100_SXM)
    assert err is not None and "fits in shared memory" in err
    P = tile_plan(emu, emu_function(p), ms.CHOLESKY_TILES_SPARSE)
    assert len(P["tile_order"]) // GRAM_WARPS == 8 < FUSED_MAX_ROUNDS
    # the planner's figures: the union of the tiles alone is within the opt-in shared memory, the whole group (tables, strips,
    # per-instance vectors) is not
    assert P["tiles"] * 256 * 4 < H100_SXM[1]
    for name in PATTERNS:
        q = make_pattern(name)
        rounds = len(tile_plan(emu, emu_function(q), ms.CHOLESKY_TILES_SPARSE)["tile_order"]) // GRAM_WARPS
        assert rounds < FUSED_MAX_ROUNDS, (name, rounds)


def test_zz_report_emulator():
    print("\n[mutations] worst backward error / limit of each mutation kind (must exceed 10):")
    by_kind = {}
    for (kind, name), v in MUTATION_MARGIN.items():
        by_kind[kind] = min(by_kind.get(kind, np.inf), v)
    print("    weakest per kind:", {k: f"{v:.1f}" for k, v in by_kind.items()})
    if MUTATION_MARGIN:
        assert set(by_kind) == set(MUTATION_KINDS) and min(by_kind.values()) > 10, by_kind
    if GRAM_SPLIT:
        print("[emulator] step = factorisation + Gram (ulp), worst:", {k: round(max(v[k2] for v in GRAM_SPLIT.values()), 2)
                                                                    for k2, k in enumerate(("step", "factorisation", "gram"))})
    print("[emulator] worst k per path and family:", {f"{a}/{b}": round(v, 5) for (a, b), v in sorted(CPU_WORST.items())})


@pytest.mark.gpu
def test_zz_report():
    print("\n[gpu] worst k per path and family:", {f"{a}/{b}": round(v, 5) for (a, b), v in sorted(GPU_WORST.items())})
    print("[gpu] paths reached:", {k: sorted(set(v)) for k, v in sorted(REACHED.items())}, " pinned:", R.SOLVE_K)
    if GPU_WORST:
        want = {"tiles_256", "tiles_512", "tiles_kmajor_256", "gram_cholesky", "persistent_3_groups", "persistent_2_groups", "persistent_1_groups"}
        assert want <= set(REACHED), sorted(want - set(REACHED))
