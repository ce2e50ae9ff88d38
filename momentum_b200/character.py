"""Rig and objective descriptions (host side, numpy only).

These plain-data classes mirror the reference types that feed the Gauss-Newton hot path:

* ``Character``  = ``Skeleton`` (momentum/character/skeleton.h:22-77, joint.h:18-76) +
  ``ParameterTransform`` (character/parameter_transform.h:62-184, CSR 7J x n) +
  ``ParameterLimits`` (character/parameter_limits.h:20-138).
* ``PositionErrorFunction`` / ``OrientationErrorFunction`` / ``StateErrorFunction`` /
  ``LimitErrorFunction`` = the constraint data of the same-named reference classes
  (character_solver/position_error_function.h:16-73, orientation_error_function.h:16-108,
  state_error_function.h:35-117, limit_error_function.h:25-119), with a leading batch dimension on
  everything that differs per IK instance (targets, optionally constraint weights).

Synthetic generators follow SURVEY.md §8(d): ``create_test_character`` clones the reference test
fixture (momentum/test/character/character_helpers.cpp:38-55,106-149,213-220); ``humanoid72`` and
``bodyhands300`` are the named benchmark rigs.
"""
from __future__ import annotations

import dataclasses
from dataclasses import dataclass, field
from typing import List, Optional, Sequence

import numpy as np

PARAMETERS_PER_JOINT = 7  # character/types.h:21
MAX_MODEL_PARAMETERS = 2048  # ParameterSet = std::bitset<2048>, math/types.h:426-429

# character/parameter_limits.h:20-33
LIMIT_MINMAX, LIMIT_MINMAX_JOINT, LIMIT_MINMAX_JOINT_PASSIVE, LIMIT_LINEAR, LIMIT_LINEAR_JOINT, LIMIT_ELLIPSOID, LIMIT_HALFPLANE = range(7)

# generalized loss special alphas (math/generalized_loss.h:52-60)
LOSS_L2, LOSS_L1, LOSS_CAUCHY = 2.0, 1.0, 0.0
LOSS_WELSCH = float("-inf")

# state_error_function.h:17-32
ROTATION_MATRIX_DIFFERENCE, QUATERNION_LOG_MAP = 0, 1

# error-function kinds (shared numbering with include/momentum_b200.h and oracle/ik_oracle.hpp)
KIND_POSITION, KIND_ORIENTATION, KIND_ORIENTATION_ROTDIFF, KIND_STATE, KIND_LIMIT, KIND_PLANE, KIND_MODEL_PARAMETERS = range(7)


@dataclass
class ParameterLimit:
    """One ``ParameterLimit`` (character/parameter_limits.h:117-127). ``i``/``f`` packing:

    MinMax: i0=parameterIndex, f0,f1=limits. MinMaxJoint: i0=jointIndex, i1=jointParameter, f0,f1.
    Linear: i0=referenceIndex, i1=targetIndex, f0=scale, f1=offset, f2=rangeMin, f3=rangeMax.
    LinearJoint: i0,i1=reference joint/param, i2,i3=target joint/param, f0..f3 as Linear.
    HalfPlane: i0=param1, i1=param2, f0,f1=normal, f2=offset.
    Ellipsoid: i0=ellipsoidParent, i1=parent, f[0:12]=ellipsoid (3x4 row-major), f[12:24]=ellipsoidInv, f[24:27]=offset.
    """

    type: int = LIMIT_MINMAX
    weight: float = 1.0
    i: Sequence[int] = (0, 0, 0, 0)
    f: Sequence[float] = ()

    def packed(self):
        i = np.zeros(4, np.int32)
        i[: len(self.i)] = self.i
        f = np.zeros(27, np.float32)
        f[: len(self.f)] = np.asarray(self.f, np.float32)
        return i, f


MAX_SKIN_JOINTS = 8  # kMaxSkinJoints, skin_weights.h:19


@dataclass
class TaperedCapsule:
    """One ``TaperedCapsuleT`` (character/collision_geometry.h): the local ``transformation`` (translation, rotation xyzw, scale) in the
    ``parent`` joint's frame, -1 for a world-fixed capsule; the radii at its two ends and its length along the local x axis. The rotation is
    normalised when the geometry is uploaded (momentum composes a non-unit rotation as it is, so the two differ for one)."""

    parent: int = -1
    translation: Sequence[float] = (0.0, 0.0, 0.0)
    rotation: Sequence[float] = (0.0, 0.0, 0.0, 1.0)
    scale: float = 1.0
    radius: Sequence[float] = (0.0, 0.0)
    length: float = 0.0


# mb2_tapered_capsule, 48 bytes
CAPSULE_DTYPE = np.dtype([("parent", "<i4"), ("translation", "<f4", 3), ("rotation", "<f4", 4), ("scale", "<f4"), ("radius", "<f4", 2),
                          ("length", "<f4")])


def capsule_array(capsules: Sequence[TaperedCapsule]) -> np.ndarray:
    """The capsules as a contiguous mb2_tapered_capsule array."""
    a = np.zeros(len(capsules), CAPSULE_DTYPE)
    for k, c in enumerate(capsules):
        a[k] = (int(c.parent), tuple(c.translation), tuple(c.rotation), float(c.scale), tuple(c.radius), float(c.length))
    return a


@dataclass
class Skinning:
    """Linear-blend skinning of a character: ``SkinWeights`` (skin_weights.h:19-40) and ``Character::inverseBindPose``. A vertex's
    influences end at its first zero weight (linear_skinning.cpp:76-80); the slots after it are ignored."""

    rest_vertices: np.ndarray  # float32 [V,3]
    skin_index: np.ndarray  # int32 [V,8]
    skin_weight: np.ndarray  # float32 [V,8]
    inverse_bind_pose: np.ndarray  # float32 [J,3,4]: the top 3x4 of Affine3f::matrix()
    faces: Optional[np.ndarray] = None  # int32 [F,3]: the triangles over rest_vertices (Mesh::faces, mesh.h)

    @property
    def num_vertices(self) -> int:
        return int(self.rest_vertices.shape[0])


@dataclass
class BlendShape:
    """The identity blend shape of a character (``BlendShape``, blend_shape.h): the rest mesh of blend weights w is
    ``base_shape + sum_k w_k shape_vectors[k]`` over the first len(w) shape vectors (blend_shape_base.cpp:18-24)."""

    base_shape: np.ndarray  # float32 [V,3]
    shape_vectors: np.ndarray  # float32 [K,V,3]: shapeVectors_ (3V x K, column-major) as it lies in memory

    @property
    def num_shapes(self) -> int:
        return int(self.shape_vectors.shape[0])

    @property
    def num_vertices(self) -> int:
        return int(self.base_shape.shape[0])


@dataclass
class Character:
    parents: np.ndarray  # int32 [J], -1 = root, parents precede children
    offsets: np.ndarray  # float32 [J,3] translationOffset
    prerot: np.ndarray  # float32 [J,4] preRotation (x,y,z,w)
    num_params: int
    pt_outer: np.ndarray  # int32 [7J+1]
    pt_inner: np.ndarray  # int32 [nnz]
    pt_vals: np.ndarray  # float32 [nnz]
    pt_offsets: np.ndarray  # float32 [7J]
    limits: List[ParameterLimit] = field(default_factory=list)
    name: str = "character"
    skinning: Optional[Skinning] = None
    blend_shape: Optional["BlendShape"] = None
    collision: Optional[List[TaperedCapsule]] = None

    @property
    def num_joints(self) -> int:
        return int(self.parents.shape[0])

    def validate(self):
        J = self.num_joints
        assert self.offsets.shape == (J, 3) and self.prerot.shape == (J, 4)
        assert self.pt_outer.shape == (7 * J + 1,)
        assert self.num_params <= MAX_MODEL_PARAMETERS
        for j, p in enumerate(self.parents):
            assert -1 <= p < j, "skeleton must be topologically sorted (skeleton.h:23-24)"
        assert self.pt_inner.size == 0 or self.pt_inner.max() < self.num_params

    def depth(self) -> np.ndarray:
        d = np.zeros(self.num_joints, np.int32)
        for j, p in enumerate(self.parents):
            d[j] = 0 if p < 0 else d[p] + 1
        return d


def _csr_from_triplets(rows, n_params, triplets):
    trip = sorted(triplets, key=lambda t: (t[0], t[1]))
    outer = np.zeros(rows + 1, np.int32)
    for r, _, _ in trip:
        outer[r + 1] += 1
    outer = np.cumsum(outer).astype(np.int32)
    inner = np.array([t[1] for t in trip], np.int32)
    vals = np.array([t[2] for t in trip], np.float32)
    return outer, inner, vals


def create_test_character(num_joints: int = 3) -> Character:
    """Clone of ``createTestCharacter`` (momentum/test/character/character_helpers.cpp:224-244):
    Y-axis chain, unit offsets, identity pre-rotations, n = 9 + (J-2) model parameters
    {root tx,ty,tz,rx,ry,rz, scale_global, joint1_rx, shared_rz(0.5*j1.rz + 0.5*j2.rz), jointK_rx}
    and one MinMax limit on parameter 0 (:213-220)."""
    assert num_joints >= 3
    J = num_joints
    parents = np.arange(-1, J - 1, dtype=np.int32)
    offsets = np.zeros((J, 3), np.float32)
    offsets[1:, 1] = 1.0
    prerot = np.zeros((J, 4), np.float32)
    prerot[:, 3] = 1.0
    trip = [(k, k, 1.0) for k in range(7)]
    trip.append((1 * 7 + 3, 7, 1.0))
    trip.append((1 * 7 + 5, 8, 0.5))
    trip.append((2 * 7 + 5, 8, 0.5))
    for j in range(2, J):
        trip.append((j * 7 + 3, 9 + j - 2, 1.0))
    n = 9 + J - 2
    outer, inner, vals = _csr_from_triplets(7 * J, n, trip)
    limits = [ParameterLimit(LIMIT_MINMAX, 1.0, (0,), (-0.1, 0.1))]
    return Character(parents, offsets, prerot, n, outer, inner, vals, np.zeros(7 * J, np.float32), limits, f"chain{J}")


def _random_prerot(rng, max_angle_deg=30.0):
    axis = rng.normal(size=3)
    axis /= np.linalg.norm(axis)
    ang = np.deg2rad(rng.uniform(0, max_angle_deg))
    s = np.sin(ang / 2)
    return np.array([axis[0] * s, axis[1] * s, axis[2] * s, np.cos(ang / 2)], np.float32)


class _TreeBuilder:
    def __init__(self, rng):
        self.rng = rng
        self.parents, self.offsets, self.prerot, self.names = [], [], [], []

    def add(self, name, parent, length, direction=None):
        rng = self.rng
        if direction is None:
            direction = rng.normal(size=3)
        direction = np.asarray(direction, np.float64)
        direction = direction / np.linalg.norm(direction)
        self.parents.append(parent)
        self.offsets.append((direction * length).astype(np.float32))
        self.prerot.append(_random_prerot(rng) if parent >= 0 else np.array([0, 0, 0, 1], np.float32))
        self.names.append(name)
        return len(self.parents) - 1

    def chain(self, prefix, parent, lengths, direction):
        ids = []
        for k, L in enumerate(lengths):
            d = np.asarray(direction, np.float64) + 0.15 * self.rng.normal(size=3)
            parent = self.add(f"{prefix}{k}", parent, L, d)
            ids.append(parent)
        return ids


def humanoid72(seed: int = 12346) -> "tuple[Character, dict]":
    """72-joint humanoid, n = 220 (SURVEY.md §8d): pelvis root (6 DOF + global scale) and
    rx,ry,rz on each of the other 71 joints. Lengths are in centimetre-like units so that the
    reference's legacy weights (Position 1e-4, Orientation 1e-1) give O(1) normal-equation entries
    against the default damping 0.05. Returns (character, named joint sets)."""
    rng = np.random.default_rng(seed)
    tb = _TreeBuilder(rng)
    U = lambda a, b: float(rng.uniform(a, b))
    root = tb.add("pelvis", -1, 0.0, (0, 1, 0))
    tb.offsets[0][:] = 0
    spine = tb.chain("spine", root, [U(8, 14) for _ in range(4)], (0, 1, 0))
    neck = tb.add("neck", spine[-1], U(8, 12), (0, 1, 0))
    head = tb.add("head", neck, U(8, 12), (0, 1, 0))
    sets = {"pelvis": root, "head": head, "neck": neck}
    fingers_tips = []
    for side, sx in (("l", 1.0), ("r", -1.0)):
        clav = tb.add(f"{side}_clavicle", spine[-1], U(12, 18), (sx, 0.2, 0))
        sho = tb.add(f"{side}_shoulder", clav, U(5, 8), (sx, 0, 0))
        elb = tb.add(f"{side}_elbow", sho, U(25, 32), (sx, -0.2, 0))
        twist = tb.add(f"{side}_forearm_twist", elb, U(11, 14), (sx, 0, 0))
        wrist = tb.add(f"{side}_wrist", twist, U(11, 14), (sx, 0, 0))
        for fi in range(5):
            ids = tb.chain(f"{side}_finger{fi}_", wrist, [U(6, 9)] + [U(2, 4) for _ in range(3)], (sx, 0.1 * (fi - 2), 0.3 * (fi - 2)))
            fingers_tips.append(ids[-1])
        sets[f"{side}_shoulder"], sets[f"{side}_elbow"], sets[f"{side}_wrist"] = sho, elb, wrist
    for side, sx in (("l", 1.0), ("r", -1.0)):
        hip = tb.add(f"{side}_hip", root, U(9, 12), (sx, -0.3, 0))
        knee = tb.add(f"{side}_knee", hip, U(38, 46), (0, -1, 0))
        ankle = tb.add(f"{side}_ankle", knee, U(36, 44), (0, -1, 0))
        ball = tb.add(f"{side}_ball", ankle, U(10, 14), (0, -0.3, 1))
        toe = tb.add(f"{side}_toe", ball, U(5, 8), (0, 0, 1))
        sets[f"{side}_knee"], sets[f"{side}_ankle"], sets[f"{side}_toe"] = knee, ankle, toe
    helpers = [spine[1], spine[2], sets["l_elbow"], sets["r_elbow"], head]
    for k, h in enumerate(helpers):
        tb.add(f"helper{k}", h, U(4, 8))
    J = len(tb.parents)
    assert J == 72, J
    trip = [(k, k, 1.0) for k in range(7)]
    col = 7
    for j in range(1, J):
        for d in range(3):
            trip.append((j * 7 + 3 + d, col, 1.0))
            col += 1
    n = col
    assert n == 220
    outer, inner, vals = _csr_from_triplets(7 * J, n, trip)
    ch = Character(np.array(tb.parents, np.int32), np.stack(tb.offsets).astype(np.float32), np.stack(tb.prerot).astype(np.float32), n, outer, inner, vals, np.zeros(7 * J, np.float32), [], "humanoid72")
    sets["fingertips"] = fingers_tips
    pos_joints = [head, neck, sets["l_wrist"], sets["r_wrist"], sets["l_elbow"], sets["r_elbow"], sets["l_shoulder"], sets["r_shoulder"],
                  sets["l_ankle"], sets["r_ankle"], sets["l_knee"], sets["r_knee"], sets["l_toe"], sets["r_toe"]] + fingers_tips
    assert len(pos_joints) == 24
    sets["position_joints"] = pos_joints
    sets["orientation_joints"] = [root, head, sets["l_wrist"], sets["r_wrist"], sets["l_ankle"], sets["r_ankle"]]
    ch.validate()
    return ch, sets


def bodyhands_rig(num_chains: int = 60, chain_len: int = 4, seed: int = 12348, name: str = "bodyhands300") -> "tuple[Character, dict]":
    """Body + helper-chain rig: 60 body joints (root 6 DOF + scale, 3 rotation DOF on the other 59) + ``num_chains`` chains of
    ``chain_len`` one-DOF (rx) finger/helper joints; every 8th helper joint's rx row is additionally driven by its parent's parameter
    with weight 0.5 (mirrors ``shared_rz`` of the reference fixture, character_helpers.cpp:137-138).
    60 x 4 = the 300-joint body+hands rig with n = 424 of SURVEY.md §8d; 30 x 3 = the 150-joint rig of cfg5 (n = 274)."""
    rng = np.random.default_rng(seed)
    tb = _TreeBuilder(rng)
    U = lambda a, b: float(rng.uniform(a, b))
    root = tb.add("pelvis", -1, 0.0, (0, 1, 0))
    tb.offsets[0][:] = 0
    spine = tb.chain("spine", root, [U(7, 11) for _ in range(5)], (0, 1, 0))
    neck = tb.chain("neck", spine[-1], [U(5, 7), U(5, 7)], (0, 1, 0))
    head = tb.add("head", neck[-1], U(8, 12), (0, 1, 0))
    attach = []
    for side, sx in (("l", 1.0), ("r", -1.0)):
        arm = tb.chain(f"{side}_arm", spine[-1], [U(12, 18), U(5, 8), U(13, 16), U(13, 16), U(11, 14), U(11, 14)], (sx, 0, 0))
        leg = tb.chain(f"{side}_leg", root, [U(9, 12), U(19, 23), U(19, 23), U(18, 22), U(18, 22), U(10, 14), U(5, 8)], (0.2 * sx, -1, 0))
        attach += [arm[-1]] * 5 + [leg[-1]] * 3 + [leg[-2]] * 2
    body_leaf_parents = spine + neck + [head]
    k = 0
    while len(tb.parents) < 60:
        tb.add(f"body_helper{k}", body_leaf_parents[k % len(body_leaf_parents)], U(4, 9))
        k += 1
    n_body = len(tb.parents)
    assert n_body == 60
    attach += [head] * 4 + spine * 4
    body_all = list(range(1, n_body))
    k = 0
    while len(attach) < 60:  # remaining helper chains hang off body joints round-robin
        attach.append(body_all[(7 * k) % len(body_all)])
        k += 1
    chain_parents = attach[:num_chains]
    assert len(chain_parents) == num_chains
    helper_ids = []
    for ci, par in enumerate(chain_parents):
        ids = tb.chain(f"h{ci}_", par, [U(2, 6) for _ in range(chain_len)], rng.normal(size=3))
        helper_ids += ids
    J = len(tb.parents)
    assert J == 60 + num_chains * chain_len, J
    trip = [(k, k, 1.0) for k in range(7)]
    col = 7
    for j in range(1, n_body):
        for d in range(3):
            trip.append((j * 7 + 3 + d, col, 1.0))
            col += 1
    own = {}
    for j in helper_ids:
        own[j] = col
        trip.append((j * 7 + 3, col, 1.0))
        col += 1
    for idx, j in enumerate(helper_ids):
        p = tb.parents[j]
        if idx % 8 == 7 and p in own:
            trip.append((j * 7 + 3, own[p], 0.5))
    n = col
    assert n == 7 + 3 * 59 + num_chains * chain_len, n
    outer, inner, vals = _csr_from_triplets(7 * J, n, trip)
    ch = Character(np.array(tb.parents, np.int32), np.stack(tb.offsets).astype(np.float32), np.stack(tb.prerot).astype(np.float32), n, outer, inner, vals, np.zeros(7 * J, np.float32), [], name)
    ch.validate()
    sets = {"marker_joints": [int(j) for j in np.round(np.linspace(1, J - 1, min(200, J - 1))).astype(int)]}
    return ch, sets


def bodyhands300(seed: int = 12348) -> "tuple[Character, dict]":
    """300-joint body+hands rig, n = 424 (SURVEY.md §8d, cfg4)."""
    return bodyhands_rig(60, 4, seed, "bodyhands300")


def body150(seed: int = 12350) -> "tuple[Character, dict]":
    """150-joint rig of the cfg5 mix (60 body joints + 30 helper chains of three), n = 274."""
    return bodyhands_rig(30, 3, seed, "body150")


# ------------------------------------------------------------------------------------------------
# Error-function data (batched)
# ------------------------------------------------------------------------------------------------
@dataclass
class PositionErrorFunction:
    """PositionErrorFunctionT constraints (position_error_function.h:16-29): per constraint parent
    joint, offset in the parent frame, weight; ``targets`` carries the batch dimension [B, nc, 3]."""

    parents: np.ndarray
    offsets: np.ndarray  # [nc,3]
    weights: np.ndarray  # [nc] (shared) — ConstraintData::weight is float
    targets: np.ndarray  # [B,nc,3]
    weight: float = 1.0  # SkeletonErrorFunctionT::weight_
    loss_alpha: float = LOSS_L2
    loss_c: float = 1.0
    kind: int = KIND_POSITION
    instance_offsets: Optional[np.ndarray] = None  # [B,nc,3]: offsets per batch element (tensor_ik.cpp:136-140 builds them per element)
    kLegacyWeight = 1e-4  # position_error_function.h:64


@dataclass
class OrientationErrorFunction:
    """OrientationErrorFunctionT / OrientationRotDiffErrorFunctionT (orientation_error_function.h:16-108);
    quaternions are (x,y,z,w) and are normalised on entry as in OrientationDataT's constructor."""

    parents: np.ndarray
    offsets: np.ndarray  # [nc,4]
    weights: np.ndarray  # [nc]
    targets: np.ndarray  # [B,nc,4]
    weight: float = 1.0
    loss_alpha: float = LOSS_L2
    loss_c: float = 1.0
    rot_diff: bool = False
    instance_offsets: Optional[np.ndarray] = None  # [B,nc,4]: offsets per batch element (the instanced block)
    kLegacyWeight = 1e-1  # orientation_error_function.h:63

    @property
    def kind(self):
        return KIND_ORIENTATION_ROTDIFF if self.rot_diff else KIND_ORIENTATION


@dataclass
class StateErrorFunction:
    """StateErrorFunctionT (state_error_function.h:35-117): per-joint position/rotation target
    weights, global pos/rot weights; ``targets`` [B, J, 8] = (t, q xyzw, s) per joint."""

    pos_weights: np.ndarray  # [J]
    rot_weights: np.ndarray  # [J]
    targets: np.ndarray  # [B,J,8]
    weight: float = 1.0
    pos_wgt: float = 1.0
    rot_wgt: float = 1.0
    rotation_error_type: int = ROTATION_MATRIX_DIFFERENCE
    kind: int = KIND_STATE


@dataclass
class LimitErrorFunction:
    """LimitErrorFunctionT over the character's ParameterLimits (limit_error_function.h:25-119)."""

    weight: float = 1.0
    loss_alpha: float = LOSS_L2
    loss_c: float = 1.0
    kind: int = KIND_LIMIT


@dataclass
class PlaneErrorFunction:
    """PlaneErrorFunctionT (plane_error_function.h:20-101, .cpp:49-70): signed distance of T_parent * offset to the plane
    (normal, d), one row per constraint; ``above`` = half-plane mode (only penetration is penalised). ``targets`` [B, nc, 4] =
    (normal xyz, d) per instance; normals are normalised on entry as in PlaneDataT's constructor."""

    parents: np.ndarray
    offsets: np.ndarray  # [nc,3]
    weights: np.ndarray  # [nc]
    targets: np.ndarray  # [B,nc,4]
    above: bool = False
    weight: float = 1.0
    loss_alpha: float = LOSS_L2
    loss_c: float = 1.0
    kind: int = KIND_PLANE
    kLegacyWeight = 1e-4  # plane_error_function.h:83


@dataclass
class ModelParametersErrorFunction:
    """ModelParametersErrorFunctionT (model_parameters_error_function.h/.cpp): w_i (theta_i - target_i) on every enabled parameter
    with target weight > 0, scaled by weight * kMotionWeight (1e-1). ``targets`` [B, n] per instance, ``target_weights`` [n] shared."""

    target_weights: np.ndarray  # [n]
    targets: np.ndarray  # [B,n]
    weight: float = 1.0
    kind: int = KIND_MODEL_PARAMETERS
    kMotionWeight = 1e-1  # model_parameters_error_function.h:61


def jacobian_size(character: Character, ef) -> int:
    """getJacobianSize() of each family (joint_error_function-inl.h:300-302,
    state_error_function.cpp:394-404, limit_error_function.cpp:1138-1161)."""
    if ef.kind == KIND_POSITION:
        return 3 * len(ef.parents)
    if ef.kind in (KIND_ORIENTATION, KIND_ORIENTATION_ROTDIFF):
        return 9 * len(ef.parents)
    if ef.kind == KIND_STATE:
        active = int(np.count_nonzero((np.asarray(ef.pos_weights) != 0) | (np.asarray(ef.rot_weights) != 0)))
        return active * (6 if ef.rotation_error_type == QUATERNION_LOG_MAP else 12)
    if ef.kind == KIND_PLANE:
        return len(ef.parents)
    if ef.kind == KIND_MODEL_PARAMETERS:  # model_parameters_error_function.cpp:93-95
        return int(np.count_nonzero(np.asarray(ef.target_weights) > 0))
    if ef.kind == KIND_LIMIT:
        return sum(0 if l.type == LIMIT_MINMAX_JOINT_PASSIVE else (3 if l.type == LIMIT_ELLIPSOID else 1) for l in character.limits)
    raise ValueError(ef.kind)


# ------------------------------------------------------------------------------------------------
# numpy forward kinematics (float64) — used only to synthesise reachable targets for benchmarks/tests
# ------------------------------------------------------------------------------------------------
def _qmul(a, b):
    ax, ay, az, aw = a[..., 0], a[..., 1], a[..., 2], a[..., 3]
    bx, by, bz, bw = b[..., 0], b[..., 1], b[..., 2], b[..., 3]
    return np.stack([aw * bx + ax * bw + ay * bz - az * by, aw * by + ay * bw + az * bx - ax * bz,
                     aw * bz + az * bw + ax * by - ay * bx, aw * bw - ax * bx - ay * by - az * bz], -1)


def _qrot(q, v):
    u = q[..., :3]
    uv = np.cross(u, v)
    uv = uv + uv
    return v + q[..., 3:4] * uv + np.cross(u, uv)


def forward_kinematics(ch: Character, theta: np.ndarray):
    """Batched FK in float64 following joint_state.cpp:22-65 / transform.h:124-129.
    theta [B,n] -> (t [B,J,3], q [B,J,4], s [B,J])."""
    theta = np.asarray(theta, np.float64)
    B = theta.shape[0]
    J = ch.num_joints
    jp = np.zeros((B, 7 * J))
    rows = np.repeat(np.arange(7 * J), np.diff(ch.pt_outer))
    np.add.at(jp, (slice(None), rows), theta[:, ch.pt_inner] * ch.pt_vals.astype(np.float64))
    jp += ch.pt_offsets.astype(np.float64)
    jp = jp.reshape(B, J, 7)
    t = np.zeros((B, J, 3)); q = np.zeros((B, J, 4)); s = np.zeros((B, J))
    for j in range(J):
        p = jp[:, j]
        ql = np.broadcast_to(ch.prerot[j].astype(np.float64), (B, 4)).copy()
        for k in (2, 1, 0):
            r = np.zeros((B, 4)); r[:, k] = np.sin(0.5 * p[:, 3 + k]); r[:, 3] = np.cos(0.5 * p[:, 3 + k])
            ql = _qmul(ql, r)
        tl = ch.offsets[j].astype(np.float64) + p[:, :3]
        sl = np.exp2(p[:, 6])
        par = ch.parents[j]
        if par < 0:
            t[:, j], q[:, j], s[:, j] = tl, ql, sl
        else:
            t[:, j] = t[:, par] + _qrot(q[:, par], s[:, par, None] * tl)
            q[:, j] = _qmul(q[:, par], ql)
            s[:, j] = s[:, par] * sl
    return t, q, s


def world_points(ch: Character, theta, parents, offsets):
    """offsets [nc,3] (shared by the batch) or [B,nc,3] (per instance)."""
    t, q, s = forward_kinematics(ch, theta)
    parents = np.asarray(parents)
    off = np.asarray(offsets, np.float64)
    if off.ndim == 2:
        off = off[None]
    return t[:, parents] + _qrot(q[:, parents], s[:, parents, None] * off)


def _quat_matrix(q):
    """Eigen toRotationMatrix of (normalised) quaternions [..., 4] xyzw -> [..., 3, 3]."""
    x, y, z, w = q[..., 0], q[..., 1], q[..., 2], q[..., 3]
    return np.stack([np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)], -1),
                     np.stack([2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)], -1),
                     np.stack([2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)], -1)], -2)


def _rest_frames(ch: Character):
    """World positions of the joints at theta = 0, and the inverse bind pose (the inverse of the rest-pose world transform, as momentum
    builds it) as float64 [J,3,4]."""
    t, q, s = forward_kinematics(ch, np.zeros((1, ch.num_params)))
    t, q, s = t[0], q[0], s[0]
    R = _quat_matrix(q)
    Rt = np.swapaxes(R, -1, -2) / s[:, None, None]
    return t, np.concatenate([Rt, -(Rt @ t[:, :, None])], -1)


def _children(ch: Character):
    children = [[] for _ in range(ch.num_joints)]
    for j, p in enumerate(ch.parents):
        if p >= 0:
            children[p].append(j)
    return children


def _bone_skin_weights(ch: Character, t, children, j: int, length: float, x, rng):
    """The skin index and weights [n,8] of vertices x [n,3] around the bone of joint j: weights fall off with the distance to the joint,
    its parent, its children and its grandparent and are normalised; the smallest are dropped so that a vertex keeps 1 to 8 influences,
    largest first."""
    n = x.shape[0]
    p = int(ch.parents[j])
    cand = ([p] if p >= 0 else []) + [j] + children[j]
    if p >= 0 and ch.parents[p] >= 0 and len(cand) < MAX_SKIN_JOINTS:
        cand.append(int(ch.parents[p]))
    cand = np.array(cand[:MAX_SKIN_JOINTS])
    dist = np.linalg.norm(x[:, None, :] - t[cand][None], axis=-1)
    w = np.exp(-(dist / (0.5 * length + 2.0)) ** 2) + 1e-12
    w /= w.sum(1, keepdims=True)
    w[w < rng.uniform(0.02, 0.3, (n, 1))] = 0.0  # 1 to len(cand) influences per vertex
    w[np.arange(n), w.argmax(1)] = np.maximum(w.max(1), 1e-3)
    order = np.argsort(-w, axis=1, kind="stable")
    wi = np.zeros((n, MAX_SKIN_JOINTS))
    ii = np.zeros((n, MAX_SKIN_JOINTS), np.int32)
    wi[:, :len(cand)] = np.take_along_axis(w, order, 1)
    ii[:, :len(cand)] = cand[order]
    wi /= wi.sum(1, keepdims=True)
    ii[wi == 0.0] = 0
    return ii, wi


def synthetic_skinning(ch: Character, vertices_per_joint: int, seed: int = 0) -> Skinning:
    """A seeded mesh around the bones of ``ch`` at theta = 0: each joint gets ``vertices_per_joint`` vertices scattered around the
    segment from its parent to it (a blob for a root). Weights fall off with the distance to the joint, its parent and its children and
    are normalised; the smallest are dropped so that a vertex keeps 1 to 8 influences, largest first. The inverse bind pose is the
    inverse of the rest-pose world transform, as momentum builds it."""
    rng = np.random.default_rng(seed)
    t, ibp = _rest_frames(ch)
    children = _children(ch)
    verts, index, weight = [], [], []
    for j in range(ch.num_joints):
        p = int(ch.parents[j])
        start = t[p] if p >= 0 else t[j]
        length = float(np.linalg.norm(t[j] - start))
        radius = 0.2 * length + 1.0
        u = rng.uniform(0.0, 1.0, (vertices_per_joint, 1))
        d = rng.normal(size=(vertices_per_joint, 3))
        d *= (radius * rng.uniform(0.5, 1.0, (vertices_per_joint, 1))) / np.linalg.norm(d, axis=1, keepdims=True)
        x = start + u * (t[j] - start) + d
        ii, wi = _bone_skin_weights(ch, t, children, j, length, x, rng)
        verts.append(x); index.append(ii); weight.append(wi)
    return Skinning(np.concatenate(verts).astype(np.float32), np.concatenate(index).astype(np.int32), np.concatenate(weight).astype(np.float32),
                    ibp.astype(np.float32))


def synthetic_tube_mesh(ch: Character, rings: int, segments: int, seed: int = 0) -> Skinning:
    """A seeded, closed, triangulated mesh around the bones of ``ch`` at theta = 0, skinned by ``synthetic_skinning``'s weight rule: each
    joint gets a tube of ``rings`` x ``segments`` vertices along the segment from its parent to it (for a root or a zero-length bone, a
    tube along y as long as its diameter), with a seeded jitter of the radius per vertex so that face areas differ. Each quad is split
    into two triangles, and a fan closes each end; every triangle's (x1 - x0) x (x2 - x0) points out of its tube, so each edge of a tube
    appears once in each direction. rings = 12, segments = 12 gives 10 368 vertices on humanoid72; rings = segments = 8 gives 19 200 on
    bodyhands300."""
    assert rings >= 2 and segments >= 3
    rng = np.random.default_rng(seed)
    t, ibp = _rest_frames(ch)
    children = _children(ch)
    R, S = rings, segments
    ring_idx = np.arange(R)[:, None] * S
    k = np.arange(S)[None, :]
    k1 = (k + 1) % S
    a, b, c, d = (ring_idx[:-1] + k), (ring_idx[:-1] + k1), (ring_idx[1:] + k), (ring_idx[1:] + k1)
    quads = np.concatenate([np.stack([a, b, c], -1).reshape(-1, 3), np.stack([b, d, c], -1).reshape(-1, 3)])
    fan = np.arange(1, S - 1)
    cap0 = np.stack([np.zeros_like(fan), fan + 1, fan], -1)
    cap1 = (R - 1) * S + np.stack([np.zeros_like(fan), fan, fan + 1], -1)
    tube_faces = np.concatenate([quads, cap0, cap1]).astype(np.int64)
    theta = 2.0 * np.pi * np.arange(S) / S
    verts, index, weight, faces = [], [], [], []
    for j in range(ch.num_joints):
        p = int(ch.parents[j])
        start = t[p] if p >= 0 else t[j]
        length = float(np.linalg.norm(t[j] - start))
        radius = 0.2 * length + 1.0
        if length > 0.0:
            axis, end = (t[j] - start) / length, t[j]
        else:
            axis = np.array([0.0, 1.0, 0.0])
            start, end = t[j] - radius * axis, t[j] + radius * axis
        helper = np.array([1.0, 0.0, 0.0]) if abs(axis[0]) < 0.9 else np.array([0.0, 0.0, 1.0])
        b1 = np.cross(axis, helper)
        b1 /= np.linalg.norm(b1)
        b2 = np.cross(axis, b1)  # (b1, b2, axis) is right-handed
        r = radius * rng.uniform(0.7, 1.0, (R, S, 1))
        radial = np.cos(theta)[:, None] * b1 + np.sin(theta)[:, None] * b2
        s = (np.arange(R) / (R - 1))[:, None, None]
        x = (start + s * (end - start) + r * radial[None]).reshape(R * S, 3)
        ii, wi = _bone_skin_weights(ch, t, children, j, length, x, rng)
        faces.append(tube_faces + j * R * S)
        verts.append(x); index.append(ii); weight.append(wi)
    return Skinning(np.concatenate(verts).astype(np.float32), np.concatenate(index).astype(np.int32), np.concatenate(weight).astype(np.float32),
                    ibp.astype(np.float32), np.concatenate(faces).astype(np.int32))


def synthetic_scan(ch: Character, num_points: int, theta=None, noise: Optional[float] = None, seed: int = 0):
    """A seeded scan-like point cloud of ``ch``'s mesh (``ch.skinning``, e.g. a ``synthetic_tube_mesh``) posed at model parameters
    ``theta`` (default zero): ``num_points`` samples, uniform by area over the posed faces, each moved along its face's unit normal by a
    uniform offset in [-noise, noise] (default 1 % of the mean bone length). Returns (points, normals) float32 [num_points, 3], the normals
    those of the sampled faces."""
    sk = ch.skinning
    if sk is None or sk.faces is None or len(sk.faces) == 0:
        raise ValueError("synthetic_scan needs a skinned character with mesh faces")
    rng = np.random.default_rng(seed)
    th = np.zeros((1, ch.num_params)) if theta is None else np.asarray(theta, np.float64).reshape(1, ch.num_params)
    t, q, s = forward_kinematics(ch, th)
    x = skin_points(ch, np.concatenate([t, q, s[..., None]], -1))[0]
    if noise is None:
        t0, _, _ = forward_kinematics(ch, np.zeros((1, ch.num_params)))
        p = np.asarray(ch.parents)
        d = np.linalg.norm(t0[0][p >= 0] - t0[0][p[p >= 0]], axis=-1)
        noise = 0.01 * float(d[d > 0].mean()) if np.any(d > 0) else 0.0
    f = np.asarray(sk.faces, np.int64)
    n = np.cross(x[f[:, 1]] - x[f[:, 0]], x[f[:, 2]] - x[f[:, 0]])
    area = np.linalg.norm(n, axis=-1)
    fi = rng.choice(len(f), size=num_points, p=area / area.sum())
    r1, r2 = np.sqrt(rng.uniform(size=num_points)), rng.uniform(size=num_points)
    w = np.stack([1.0 - r1, r1 * (1.0 - r2), r1 * r2], -1)  # uniform over each triangle
    nf = n[fi] / np.maximum(area[fi], 1e-300)[:, None]
    pts = np.einsum("nk,nkc->nc", w, x[f[fi]]) + rng.uniform(-noise, noise, (num_points, 1)) * nf
    return pts.astype(np.float32), nf.astype(np.float32)


def vertex_normals(faces, positions):
    """Area-weighted vertex normals in float64 (pymomentum compute_vertex_normals, tensor_skinning.cpp:354-383): per vertex the sum of
    (x1 - x0) x (x2 - x0) over every corner of every face that is that vertex, faces ascending and corners in order, then
    n / max(|n|, 1e-12). positions [B,V,3] or [V,3]; non-finite positions propagate."""
    x = np.asarray(positions, np.float64)
    single = x.ndim == 2
    x = x.reshape((-1,) + x.shape[-2:])
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    n_f = np.cross(x[:, f[:, 1]] - x[:, f[:, 0]], x[:, f[:, 2]] - x[:, f[:, 0]])
    n = np.zeros_like(x)
    # ufunc.at applies the corners in the order given: face-major, corners in order
    np.add.at(n, (slice(None), f.reshape(-1)), np.repeat(n_f, 3, axis=1))
    out = n / np.maximum(np.linalg.norm(n, axis=-1, keepdims=True), 1e-12)
    return out[0] if single else out


def skin_points(ch: Character, skel_state, rest_points=None):
    """Linear-blend skinning in float64 (applySSD, linear_skinning.cpp:40-102, with q normalised): skel_state [B,J,8] or [J,8]
    (t, q xyzw, s) -> points [B,V,3] or [V,3]. rest_points: None = the rest mesh, [V,3] shared or [B,V,3]."""
    sk = ch.skinning
    st = np.asarray(skel_state, np.float64)
    single = st.ndim == 2
    st = st.reshape(-1, ch.num_joints, 8)
    x = np.asarray(sk.rest_vertices if rest_points is None else rest_points, np.float64)
    x = np.broadcast_to(x, (st.shape[0],) + x.shape[-2:])
    qn = st[..., 3:7] / np.linalg.norm(st[..., 3:7], axis=-1, keepdims=True)
    sR = _quat_matrix(qn) * st[..., 7, None, None]
    ibp = np.asarray(sk.inverse_bind_pose, np.float64)
    L = sR @ ibp[None, :, :, :3]
    c = (sR @ ibp[None, :, :, 3:])[..., 0] + st[..., :3]
    w = np.asarray(sk.skin_weight, np.float64)
    active = np.cumprod(w != 0.0, axis=1).astype(bool)
    out = np.zeros_like(x)
    for k in range(MAX_SKIN_JOINTS):
        j = np.where(active[:, k], sk.skin_index[:, k], 0)
        wk = np.where(active[:, k], w[:, k], 0.0)
        out += (np.einsum("bvrc,bvc->bvr", L[:, j], x) + c[:, j]) * wk[None, :, None]
    return out[0] if single else out


def synthetic_blend_shape(ch: Character, skinning: Skinning, num_shapes: int, seed: int = 0) -> BlendShape:
    """A seeded blend shape over ``skinning``'s mesh: ``base_shape`` is its rest mesh, and each shape vector is a smooth displacement
    field of three Gaussian bumps centred on random joints at theta = 0, each as wide as its bone and with an amplitude of 1 to 4 % of
    the bone length, in a random direction."""
    rng = np.random.default_rng(seed)
    t, _, _ = forward_kinematics(ch, np.zeros((1, ch.num_params)))
    t = t[0]
    parents = np.asarray(ch.parents)
    length = np.where(parents >= 0, np.linalg.norm(t - t[np.maximum(parents, 0)], axis=-1), 0.0)
    length = np.where(length > 0, length, max(float(length.max()), 1.0))
    x = np.asarray(skinning.rest_vertices, np.float64)
    S = np.zeros((num_shapes,) + x.shape)
    for k in range(num_shapes):
        for j in rng.integers(0, ch.num_joints, 3):
            d = rng.normal(size=3)
            d *= rng.uniform(0.01, 0.04) * length[j] / np.linalg.norm(d)
            sigma = length[j] + 1.0
            S[k] += np.exp(-0.5 * np.sum((x - t[j]) ** 2, axis=-1) / sigma ** 2)[:, None] * d
    return BlendShape(x.astype(np.float32), S.astype(np.float32))


def synthetic_limits(ch: Character, seed: int = 0) -> List[ParameterLimit]:
    """A seeded, realistic ParameterLimits set for any rig, in list order:

    * MinMax on every model parameter, sized by what it drives (rotation +-0.4..1.5 rad, translation +-0.5..2 bone lengths, scale
      +-0.05..0.3), and a second, tighter MinMax on every fifth parameter;
    * MinMaxJoint on a rotation row of every third joint, and a MinMaxJointPassive on every seventh;
    * Linear between pairs of parameters, LinearJoint between a joint's rotation row and its parent's, each with the (0, 0) range
      (everywhere) or a finite one;
    * HalfPlane on pairs of parameters with a random unit normal;
    * one Ellipsoid per limb: for each leaf joint at depth 2 or more, the leaf's point (an offset of up to 0.2 bone lengths) against an
      ellipsoid in its grandparent's frame around the point's rest position, with axes of 0.3 to 1 times the distance.

    The rig's own ``limits`` are not changed: assign the result to use it."""
    rng = np.random.default_rng(seed)
    J, n = ch.num_joints, ch.num_params
    parents = np.asarray(ch.parents)
    t, q, s = forward_kinematics(ch, np.zeros((1, n)))
    t, q, s = t[0], q[0], s[0]
    length = np.where(parents >= 0, np.linalg.norm(t - t[np.maximum(parents, 0)], axis=-1), 0.0)
    length = np.where(length > 0, length, max(float(length.max()), 1.0))
    # the joint-parameter rows each model parameter drives
    rows_of = [[] for _ in range(n)]
    for r in range(7 * J):
        for k in range(ch.pt_outer[r], ch.pt_outer[r + 1]):
            rows_of[int(ch.pt_inner[k])].append(r)
    driven = [r for r in range(7 * J) if ch.pt_outer[r + 1] > ch.pt_outer[r]]
    U = lambda a, b: float(rng.uniform(a, b))
    L = []
    for p in range(n):
        r = rows_of[p][0] if rows_of[p] else 3
        d = r % 7
        half = U(0.4, 1.5) if 3 <= d < 6 else (U(0.5, 2.0) * length[r // 7] if d < 3 else U(0.05, 0.3))
        L.append(ParameterLimit(LIMIT_MINMAX, U(0.5, 2.0), (p,), (-half * U(0.6, 1.0), half)))
    for p in range(0, n, 5):
        lo, hi = L[p].f
        L.append(ParameterLimit(LIMIT_MINMAX, U(0.5, 2.0), (p,), (0.7 * lo, 0.7 * hi)))
    rot_rows = [r for r in driven if 3 <= r % 7 < 6]
    for j in range(0, J, 3):
        rows = [r for r in rot_rows if r // 7 == j]
        if rows:
            h = U(0.3, 1.0)
            L.append(ParameterLimit(LIMIT_MINMAX_JOINT, U(0.5, 2.0), (j, int(rng.choice(rows)) % 7), (-h, h)))
    for j in range(0, J, 7):
        L.append(ParameterLimit(LIMIT_MINMAX_JOINT_PASSIVE, 1.0, (j, 3), (-0.5, 0.5)))
    rot_params = [p for p in range(n) if rows_of[p] and 3 <= rows_of[p][0] % 7 < 6]
    for k in range(max(2, len(rot_params) // 8)):
        ref, tgt = (int(x) for x in rng.choice(rot_params, 2, replace=False))
        rmin, rmax = (0.0, 0.0) if k % 2 == 0 else (-U(0.2, 1.0), U(0.2, 1.0))
        L.append(ParameterLimit(LIMIT_LINEAR, U(0.5, 2.0), (ref, tgt), (U(0.3, 1.0), U(-0.1, 0.1), rmin, rmax)))
    for k, r in enumerate(rot_rows[1::max(1, len(rot_rows) // 10)]):
        j = r // 7
        prows = [x for x in rot_rows if x // 7 == parents[j]] if parents[j] >= 0 else []
        if not prows:
            continue
        ref = int(rng.choice(prows))
        rmin, rmax = (0.0, 0.0) if k % 2 == 0 else (-U(0.2, 1.0), U(0.2, 1.0))
        L.append(ParameterLimit(LIMIT_LINEAR_JOINT, U(0.5, 2.0), (ref // 7, ref % 7, j, r % 7), (U(0.3, 1.0), U(-0.1, 0.1), rmin, rmax)))
    for _ in range(max(2, len(rot_params) // 10)):
        p1, p2 = (int(x) for x in rng.choice(rot_params, 2, replace=False))
        a = U(0, 2 * np.pi)
        L.append(ParameterLimit(LIMIT_HALFPLANE, U(0.5, 2.0), (p1, p2), (float(np.cos(a)), float(np.sin(a)), U(-0.5, 0.2))))
    depth = ch.depth()
    leaves = [j for j in range(J) if j not in set(int(p) for p in parents) and depth[j] >= 2]
    for leaf in leaves:
        e = int(parents[parents[leaf]])
        off = rng.uniform(-0.2, 0.2, 3) * length[leaf]
        x = t[leaf] + s[leaf] * _qrot(q[leaf], off)
        local = _qrot(q[e] * np.array([-1, -1, -1, 1]), x - t[e]) / s[e]
        dist = max(float(np.linalg.norm(local)), 1e-3)
        A = np.linalg.qr(rng.normal(size=(3, 3)))[0] @ np.diag(rng.uniform(0.3, 1.0, 3) * dist)
        c = local + rng.uniform(-0.1, 0.1, 3) * dist
        M = np.concatenate([A, c[:, None]], 1)
        Ai = np.linalg.inv(A)
        Mi = np.concatenate([Ai, (-Ai @ c)[:, None]], 1)
        L.append(ParameterLimit(LIMIT_ELLIPSOID, U(0.5, 2.0), (e, leaf), tuple(M.reshape(-1)) + tuple(Mi.reshape(-1)) + tuple(off)))
    return L


def skin_with_blend_shapes(ch: Character, skel_state, blend_weights):
    """skinWithBlendShapes in float64 (blend_shape_skinning.cpp:50-140): the rest mesh base_shape + sum_k w_k shape_vectors[k] over the
    first K' = len(w) shape vectors, skinned by ``skin_points``. skel_state [B,J,8] or [J,8]; blend_weights [K'] (shared) or [B,K']."""
    bs = ch.blend_shape
    w = np.asarray(blend_weights, np.float64)
    S = np.asarray(bs.shape_vectors[:w.shape[-1]], np.float64)
    rest = np.asarray(bs.base_shape, np.float64) + np.einsum("...k,kvc->...vc", w, S)
    return skin_points(ch, skel_state, rest)


def world_rotations(ch: Character, theta, parents, offsets_q):
    _, q, _ = forward_kinematics(ch, theta)
    parents = np.asarray(parents)
    return _qmul(q[:, parents], np.broadcast_to(np.asarray(offsets_q, np.float64)[None], (q.shape[0], len(parents), 4)))


# ---- Self-collision of tapered capsules (CollisionErrorFunction) in float64 ----------------------------------------------------------
COLLISION_WEIGHT = 5e-3  # kCollisionWeight, collision_error_function.h:139
SEG_CONST, SEG_INTERIOR, SEG_EDGE0, SEG_EDGE1 = range(4)  # which closed form a closest-point parameter came from (ik_device.cuh SegmentForm)


def _capsule_locals(capsules: Sequence[TaperedCapsule]):
    """[C] parents and [C, 8] local geometry in float64: origin, direction R(q^) e_x scale length (rotation normalised), r0, r1."""
    par = np.array([int(c.parent) for c in capsules], np.int64)
    L = np.zeros((len(capsules), 8))
    for k, c in enumerate(capsules):
        q = np.asarray(c.rotation, np.float64)
        q = q / np.linalg.norm(q)
        L[k, :3] = c.translation
        L[k, 3:6] = _qrot(q, np.array([float(c.scale) * float(c.length), 0.0, 0.0]))
        L[k, 6:] = c.radius
    return par, L


def capsule_world(capsules: Sequence[TaperedCapsule], skel_state) -> np.ndarray:
    """CollisionGeometryStateT::updatePrimitive in float64 for skeleton states [B, J, 8] (t, q xyzw, s; q normalised): [B, C, 8] world
    origin, direction, r0, r1. A world-fixed capsule keeps its local geometry."""
    st = np.asarray(skel_state, np.float64)
    par, L = _capsule_locals(capsules)
    B = st.shape[0]
    W = np.broadcast_to(L, (B,) + L.shape).copy()
    att = par >= 0
    if att.any():
        ps = st[:, par[att]]
        q = ps[..., 3:7] / np.linalg.norm(ps[..., 3:7], axis=-1, keepdims=True)
        s = ps[..., 7:8]
        W[:, att, :3] = ps[..., :3] + _qrot(q, s * L[att, :3])
        W[:, att, 3:6] = _qrot(q, s * L[att, 3:6])
        W[:, att, 6:] = L[att, 6:] * s
    return W


def capsule_contact(A, B, dist_eps: float = 1e-8, margins=None):
    """overlaps() over closestPointsOnSegments (collision_geometry_state.h:120-157, math/utility.cpp:443-552) branch for branch, in the
    precision of A and B [8]: (hit, s, t, dist, overlap, sForm, tForm). dist_eps is Eps (1e-8 in float, 1e-17 in double). ``margins``, a
    list, receives (what, relative margin) for every decision taken: "far" for the early-outs, "overlap" and "dist" for the contact
    test, "branch" for the rest, so that a caller can tell a sample within rounding of a branch boundary."""
    A = np.asarray(A)
    B = np.asarray(B)
    T = A.dtype.type
    m = margins if margins is not None else []

    def lt(x, y, what="branch"):
        m.append((what, abs(float(x) - float(y)) / (abs(float(x)) + abs(float(y)) + 1e-30)))
        return x < y

    miss = (False, T(0), T(0), T(0), T(0), SEG_CONST, SEG_CONST)
    maxA = A[7] if A[6] < A[7] else A[6]
    maxB = B[7] if B[6] < B[7] else B[6]
    maxDist = T(maxA + maxB)
    maxSq = T(maxDist * maxDist)
    d1, d2 = A[3:6], B[3:6]
    w = A[:3] - B[:3]
    dot = lambda x, y: T(x[0] * y[0] + x[1] * y[1] + x[2] * y[2])
    a, b, c, d, e = dot(d1, d1), dot(d1, d2), dot(d2, d2), dot(d1, w), dot(d2, w)
    D = T(a * c - b * b)
    sD, tD = D, D
    if lt(D, T(1e-7)):
        sN, sD, tN, tD = T(0), T(1), e, c
        sF, tF = SEG_CONST, SEG_EDGE0
        if lt(maxSq, dot(w, w), "far"):
            return miss
    else:
        sN, tN = T(b * e - c * d), T(a * e - b * d)
        sF = tF = SEG_INTERIOR
        q = w + d1 * sN / D - d2 * tN / D
        if lt(maxSq, dot(q, q), "far"):
            return miss
        if lt(sN, T(0)):
            sN, tN, tD, sF, tF = T(0), e, c, SEG_CONST, SEG_EDGE0
        elif lt(sD, sN):
            sN, tN, tD, sF, tF = sD, T(e + b), c, SEG_CONST, SEG_EDGE1
    if lt(tN, T(0)):
        tN, tF = T(0), SEG_CONST
        if lt(-d, T(0)):
            sN, sF = T(0), SEG_CONST
        elif lt(a, -d):
            sN, sF = sD, SEG_CONST
        else:
            sN, sD, sF = -d, a, SEG_EDGE0
    elif lt(tD, tN):
        tN, tF = tD, SEG_CONST
        if lt(T(-d + b), T(0)):
            sN, sF = T(0), SEG_CONST
        elif lt(a, T(-d + b)):
            sN, sF = sD, SEG_CONST
        else:
            sN, sD, sF = T(-d + b), a, SEG_EDGE1
    s_snap = lt(abs(sN), T(1e-7)) or lt(abs(sD), T(1e-7))
    t_snap = lt(abs(tN), T(1e-7)) or lt(abs(tD), T(1e-7))
    s = T(0) if s_snap else T(sN / sD)
    t = T(0) if t_snap else T(tN / tD)
    dP = w + d1 * s - d2 * t
    distSq = dot(dP, dP)
    if lt(maxSq, distSq, "far"):
        return miss
    dist = T(np.sqrt(distSq))
    overlap = T(A[6] + s * (A[7] - A[6]) + B[6] + t * (B[7] - B[6]) - dist)
    m.append(("overlap", abs(float(overlap)) / (float(A[6] + B[6]) + abs(float(A[7] - A[6])) + abs(float(B[7] - B[6])) + 1e-30)))
    m.append(("dist", float(dist) / (float(maxDist) + 1e-30)))
    hit = overlap > 0 and not dist < T(dist_eps)
    return (bool(hit), s, t, dist, overlap, SEG_CONST if s_snap else sF, SEG_CONST if t_snap else tF)


def collision_pairs(ch: Character, capsules: Sequence[TaperedCapsule]) -> np.ndarray:
    """updateCollisionPairs with isValidCollisionPair and filterRestPoseOverlaps (collision_geometry_state.h:526-557), the rest pose
    (model parameters zero) in float64: int64 [P, 2], i < j ascending."""
    t, q, s = forward_kinematics(ch, np.zeros((1, ch.num_params)))
    rest = capsule_world(capsules, np.concatenate([t, q, s[..., None]], -1))[0]
    parents = np.asarray(ch.parents)
    out = []
    for i in range(len(capsules)):
        for j in range(i + 1, len(capsules)):
            p0, p1 = int(capsules[i].parent), int(capsules[j].parent)
            if p0 < 0 or p1 < 0:
                ok = p0 != p1
            elif p0 == p1 or parents[p0] == p1 or parents[p1] == p0:
                ok = False
            else:
                ok = not capsule_contact(rest[i], rest[j], 1e-17)[0]
            if ok:
                out.append((i, j))
    return np.array(out, np.int64).reshape(-1, 2)


def collision_rows(capsules: Sequence[TaperedCapsule], pairs, skel_state) -> np.ndarray:
    """The rows of collision_residual in float64 for skeleton states [B, J, 8]: [B, P], sqrt(kCollisionWeight) overlap at a contact of
    capsule_contact (with float's thresholds), else 0."""
    geo = capsule_world(capsules, skel_state)
    pairs = np.asarray(pairs).reshape(-1, 2)
    out = np.zeros((geo.shape[0], len(pairs)))
    wgt = np.sqrt(COLLISION_WEIGHT)
    for b in range(geo.shape[0]):
        for k, (i, j) in enumerate(pairs):
            c = capsule_contact(geo[b, i], geo[b, j])
            out[b, k] = wgt * c[4] if c[0] else 0.0
    return out


def synthetic_collision(ch: Character, seed: int = 0) -> List[TaperedCapsule]:
    """A seeded tapered-capsule set for any rig: on every joint with a child (the spine and the limbs), one capsule along the bone to its
    first child, with radii of 0.2 to 0.45 bone lengths, tapered (r1 = 0.55 to 0.9 r0) on two capsules in three and untapered on the
    third; then two world-fixed capsules across the rest pose's bounding box. Radii this large put many pairs in contact under random
    poses. At the rest pose every pair that isValidCollisionPair tests is clearly overlapping (and so filtered out of the valid pairs) or clearly apart: the radii of a
    capsule whose rest-pose overlap with another lies within 1e-3 of their radii are shrunk by 3 % until none does.

    The rig's own ``collision`` is not changed: assign the result to use it."""
    rng = np.random.default_rng(seed)
    J = ch.num_joints
    parents = np.asarray(ch.parents)
    t, q, s = forward_kinematics(ch, np.zeros((1, ch.num_params)))
    rest = np.concatenate([t, q, s[..., None]], -1)
    jp0 = np.asarray(ch.pt_offsets, np.float64).reshape(J, 7)
    caps = []
    for j in range(J):
        kids = np.nonzero(parents == j)[0]
        if kids.size == 0:
            continue
        bone = np.asarray(ch.offsets[kids[0]], np.float64) + jp0[kids[0], :3]  # the child's origin in j's frame
        length = float(np.linalg.norm(bone))
        if length < 1e-6:
            continue
        x = bone / length
        axis = np.cross([1.0, 0.0, 0.0], x)
        sin, cos = np.linalg.norm(axis), x[0]
        if sin < 1e-9:
            rot = (0.0, 0.0, 0.0, 1.0) if cos > 0 else (0.0, 0.0, 1.0, 0.0)
        else:
            half = 0.5 * np.arctan2(sin, cos)
            rot = tuple(np.append(axis / sin * np.sin(half), np.cos(half)))
        r0 = float(rng.uniform(0.2, 0.45)) * length
        r1 = r0 if len(caps) % 3 == 2 else r0 * float(rng.uniform(0.55, 0.9))
        caps.append(TaperedCapsule(j, (0.0, 0.0, 0.0), rot, 1.0, (r0, r1), length))
    lo, hi = t[0].min(0), t[0].max(0)
    size = float(np.linalg.norm(hi - lo))
    for k in range(2):
        o = lo + rng.uniform(0.2, 0.8, 3) * (hi - lo) + rng.normal(size=3) * 0.05 * size  # off any line the rig lies on
        r = float(rng.uniform(0.04, 0.08)) * size
        rot = np.append(rng.normal(size=3) * 0.5, 1.0)
        caps.append(TaperedCapsule(-1, tuple(o), tuple(rot / np.linalg.norm(rot)), 1.0, (r, r * 0.7), 0.3 * size))
    for _ in range(200):  # clear every rest-pose pair of its boundary
        geo = capsule_world(caps, rest)[0]
        bad = set()
        for i in range(len(caps)):
            for j in range(i + 1, len(caps)):
                p0, p1 = caps[i].parent, caps[j].parent
                if (p0 < 0 and p1 < 0) or (p0 >= 0 and p1 >= 0 and (p0 == p1 or parents[p0] == p1 or parents[p1] == p0)):
                    continue  # never evaluated: not a valid pair whatever the pose
                margins = []
                capsule_contact(geo[i], geo[j], 1e-17, margins)
                if min(v for what, v in margins if what != "branch") < 1e-3:
                    bad.add(j)
        if not bad:
            return caps
        for j in bad:
            c = caps[j]
            caps[j] = dataclasses.replace(c, radius=(c.radius[0] * 0.97, c.radius[1] * 0.97))
    raise RuntimeError("synthetic_collision: could not clear the rest-pose pairs of their boundaries")
