// Shared host/device data model of the batched Gauss-Newton IK path.
//
// Vocabulary follows the reference (momentum/): a *character* is Skeleton + ParameterTransform +
// ParameterLimits; a *solver function* is a batch of SkeletonSolverFunctionT<float> sharing one
// character and one constraint topology; error functions contribute *units* (one constraint /
// state joint / limit = one group of residual rows) and *cells* (one (unit, model-parameter) block
// of the Jacobian, with the chain-rule contributions that the reference's ancestor walk would add
// into it, joint_error_function-inl.h:229-294).
#pragma once

#include <cstdint>

#if defined(__CUDACC__)
#define MB2_HD __host__ __device__ __forceinline__
#else
#define MB2_HD inline
#endif

namespace mb2 {

constexpr int kParametersPerJoint = 7; // character/types.h:21
constexpr int kJointStateStride = 17;  // t(3) q(4) s(1) rotationAxis(9); odd => bank-conflict-free per-joint access
constexpr int kSkelAccStride = 11;     // subtree sums of the skeleton-state backward (ik_device.cuh); odd: conflict-free with lanes = joints
constexpr int kTangentStride = 7;      // joint motion w(3) sigma tdot(3) of the input gradients (ik_device.cuh); odd: conflict-free with lanes = joints
constexpr float kLn2 = 0.69314718055994530942f; // math/constants.h:40
constexpr float kPi = 3.14159265358979323846f;

enum UnitKind : int32_t {
  kUnitPosition = 0,        // position_error_function.cpp:15-27
  kUnitOrientation = 1,     // orientation_error_function.cpp:15-40
  kUnitOrientationRotDiff = 2, // orientation_error_function.cpp:43-65
  kUnitStateMatrix = 3,     // state_error_function.cpp:407-558, RotationMatrixDifference
  kUnitStateLogMap = 4,     // ... QuaternionLogMap
  kUnitLimitMinMax = 5,     // limit_error_function.cpp:459-503
  kUnitLimitMinMaxJoint = 6, // :505-558
  kUnitLimitLinear = 7,     // :560-598
  kUnitLimitLinearJoint = 8, // :600-656
  kUnitLimitHalfPlane = 9,  // :658-699
  kUnitLimitEllipsoid = 10, // :701-785
  kUnitPlane = 11,          // plane_error_function.cpp:49-70 (one row; half-plane mode clamps)
  kUnitModelParameter = 12, // model_parameters_error_function.cpp:90-133 (one row per enabled parameter with target weight > 0)
};

enum LossType : int32_t { kLossL2 = 0, kLossL1 = 1, kLossCauchy = 2, kLossWelsch = 3, kLossGeneral = 4 };

// One error function block (SkeletonErrorFunctionT::weight_, GeneralizedLossT, StateErrorFunction weights)
struct EfDesc {
  float weight;
  int32_t lossType;
  float alpha;
  float invC2;
  float posWgt, rotWgt; // StateErrorFunctionT::posWgt_/rotWgt_
  int32_t kind;         // 0 pos, 1 ori, 2 rotdiff, 3 state, 4 limit, 5 plane, 6 model parameters
  int32_t halfPlane;    // PlaneErrorFunctionT(above)
};

struct UnitDesc {
  int32_t kind;      // UnitKind
  int32_t ef;        // index into EfDesc table
  int32_t joint;     // parent joint (pos/ori/ellipsoid), state joint
  int32_t row0;      // first residual row of this unit
  int32_t numRows;   // 3 / 9 / 12 / 6 / 1 / 3
  int32_t targetOff; // float offset into the per-instance target record (-1: none)
  int32_t weightIdx; // index into constraint-weight array (-1: none)
  int32_t recOff;    // float offset of this unit's evaluation record in the per-instance scratch
  int32_t i[4];      // limit indices (model parameter / joint-parameter rows), ellipsoidParent in i[0]
  float f[8];        // offset (3 or 4) | posW, rotW | limit floats f0..f3
  int32_t extra;     // float offset into limitData (ellipsoid matrices), -1 none
  int32_t pad[3];     // [0] limit gated off by the enabled set (zero rows); [1] error-only unit (ModelParameters with a negative target weight); [2] Position / Orientation: per-instance offset stored after the target
};

// One Jacobian cell: rows [unit.row0, +numRows) x column `col`
struct CellDesc {
  uint16_t unit;
  uint16_t col;           // device column of J (model parameter index, or its rank in the enabled list when compacted)
  uint32_t contribBegin;  // into ContribDesc table
  uint16_t contribCount;  // 0 for limit cells that only scale by coef
  uint16_t quadStride;    // strip layout: strips between consecutive row quads of this cell's unit (same tile column)
  float coef;             // static coefficient for limit cells
  uint32_t stripOff;      // strip layout: float offset of (first row quad, this column) in the instance's strip buffer
};

// One chain-rule contribution: joint-parameter (joint, dof) with ParameterTransform coefficient
struct ContribDesc {
  uint16_t joint;
  uint16_t dof; // 0-2 translation, 3-5 rotation, 6 scale
  float coef;
};

// The character as the FK reads it: skeleton, ParameterTransform (CSR) and the depth levels of the joint tree. Passed by value; the
// pointers are device addresses in the kernels' arguments (mb2_character::tables) and host addresses in the emulators
// (hostCharacterTables).
struct CharacterTables {
  int32_t numJoints, numParams;
  const int32_t* parent;     // [J]
  const float* offset;       // [J*3]
  const float* prerot;       // [J*4] xyzw
  const int32_t* ptOuter;    // [7J+1]
  const int32_t* ptInner;    // [nnz]
  const float* ptVals;       // [nnz]
  const float* ptOffsets;    // [7J]
  int32_t numLevels;         // depth levels of the joint tree
  const int32_t* levelStart; // [numLevels+1]
  const int32_t* levelJoints; // [J] joints sorted by depth
  int32_t ptNnz;             // entries of ptInner / ptVals
};

// Everything the FK / residual / Jacobian kernels need (device pointers), passed by value: the character, then the objective.
struct FunctionTables : CharacterTables {
  int32_t numEf, numUnits, numCells;
  const EfDesc* efs;
  const UnitDesc* units;
  const CellDesc* cells;
  const ContribDesc* contribs;
  const float* limitData;
  int32_t targetStride; // floats per instance
  int32_t recStride;    // floats per instance of evaluation records
  int32_t numRows;      // active residual rows m (unpadded)
  int32_t ldJ;          // row stride of a Jacobian column (m padded to 32)
  int32_t numCols;      // Jacobian columns held on the device (all n, or only the enabled ones when compacted);
                        // the device matrix has numCols + 1 columns: the last one is the residual vector
  int32_t weightsPerInstance; // 0: cweights [numWeights] shared, 1: [B][numWeights]
  int32_t numWeights;
  // table sizes (the sweep kernel stages every table in shared memory when they fit)
  int32_t numContribs, numLimitData;
  // Jacobian output layout. 0: K-major matrix [numCols + 1][ldJ] (column numCols = residual). 1: strips (GramPlan in
  // ik_chol_sched.h): [numStrips][16 columns][4 rows] then the residual at residOff, rows numbered with 4-aligned row groups.
  int32_t stripMode, residOff;
  size_t jacobianStride;     // floats per instance in the Jacobian buffer
};

// What the skeleton-state backward walks besides CharacterTables (HostCharacter::buildBackwardTables)
struct SkeletonTables {
  const int32_t* childStart; // [J+1]
  const int32_t* children;   // [J - roots], ascending within a joint
  const int32_t* ptColStart; // [n+1] ParameterTransform as CSC
  const int32_t* ptColRows;  // [nnz] ascending within a column
  const float* ptColVals;    // [nnz]
  // the inverse ParameterTransform W = P^+ (HostCharacter::buildInverseTables): by model parameter for its forward, by joint-parameter
  // row for its backward
  const int32_t* invStart;    // [n+1]
  const int32_t* invRows;     // [nnz W] ascending within a parameter
  const float* invVals;       // [nnz W]
  const int32_t* invRowStart; // [7J+1]
  const int32_t* invParams;   // [nnz W] ascending within a row
  const float* invRowVals;    // [nnz W]
  // apply_model_param_limits (makeLimitTables): per model parameter min, max and 1 when a MinMax limit names it (the last such limit in
  // list order), else 0, 0, 0
  const float* paramClamp;    // [n][3]
};

// character/parameter_limits.h:20-33 LimitType
enum LimitType : int32_t {
  kLimitMinMax = 0,
  kLimitMinMaxJoint = 1,
  kLimitMinMaxJointPassive = 2,
  kLimitLinear = 3,
  kLimitLinearJoint = 4,
  kLimitEllipsoid = 5,
  kLimitHalfPlane = 6,
};

// One live limit of parameter_limits_residual (makeLimitTables): its rows are the LimitErrorFunction rows at weight 1 and L2 loss.
//   MinMax       i0 parameter,            f0 f1 min max
//   MinMaxJoint  i0 joint-parameter row,  f0 f1 min max
//   Linear       i0 reference, i1 target parameter,   f0 scale, f1 offset, f2 f3 range
//   LinearJoint  i0 reference, i1 target row,         f0 .. f3 as Linear
//   HalfPlane    i0 i1 parameters, f0 f1 normal, f2 offset
//   Ellipsoid    i0 ellipsoidParent, i1 parent joint; its 27 floats (ellipsoid, ellipsoidInv, offset) at `data` in the ellipsoid array
struct LimitDesc {
  int32_t type;   // LimitType, never kLimitMinMaxJointPassive
  int32_t row;    // its first residual row
  int32_t i0, i1;
  float f[4];
  float w;        // the row scale sqrt(kLimitWeight weight), Ellipsoid sqrt(kLimitWeight kLimitPositionWeight weight), rounded once from double
  int32_t data;   // Ellipsoid: float offset into LimitTables::ellipsoidData; -1 otherwise
};

// The character's limits as parameter_limits_residual reads them (makeLimitTables), shared by the batch. The backward's gradient terms
// are grouped three ways, each a CSR in limit-list order within a group, so that every output is one lane's fixed-order sum:
//   by joint                Ellipsoid seeds: entry 2 l + role, role 0 the parent joint (the constrained point), 1 the ellipsoid parent
//   by joint-parameter row  MinMaxJoint and LinearJoint terms (target before reference), added before P^T
//   by model parameter      MinMax, Linear and HalfPlane terms (target / param1 first), added after P^T
struct LimitTables {
  int32_t numLimits;     // live limits (every type but MinMaxJointPassive)
  int32_t numRows;       // R
  int32_t ellipsoid;     // an Ellipsoid is among them: the operation runs the FK passes
  const LimitDesc* limits;       // [numLimits] in list order
  const float* ellipsoidData;    // [Ellipsoids][27]
  const int32_t* jointStart;     // [J+1]
  const int32_t* jointEntry;
  const int32_t* rowStart;       // [7J+1]
  const int32_t* rowLimit;
  const float* rowCoef;
  const int32_t* paramStart;     // [n+1]
  const int32_t* paramLimit;
  const float* paramCoef;
};

// Points fixed in joints' frames (model / joint_parameters_to_positions), shared by the batch (makePointTables): each point's joint, and
// the points grouped by joint (CSR), point indices ascending within a joint
struct PointTables {
  int32_t numPoints;
  const int32_t* parent;     // [N] in [0, J)
  const int32_t* pointStart; // [J+1] into pointIndex
  const int32_t* pointIndex; // [N]
};

// One tapered capsule of collision_residual (makeCollision), in its parent joint's frame: the world origin is T_parent(origin), the world
// direction s_parent R_parent dir and the world radii r0, r1 times s_parent, with T_parent the identity for a world-fixed capsule
// (CollisionGeometryStateT::updatePrimitive). origin and dir fold the capsule's local transformation and length, rounded once from double.
struct CapsuleDesc {
  int32_t parent;  // joint, or -1: world-fixed
  float origin[3]; // translation
  float dir[3];    // R(rotation) e_x scale length
  float r0, r1;    // radius
};

// The character's collision geometry as collision_residual reads it (makeCollision), shared by the batch: the capsules, the valid pairs
// (updateCollisionPairs, ascending), each capsule's pairs (CSR, pair indices ascending) and each joint's capsules (CSR, ascending).
struct CollisionTables {
  int32_t numCapsules;
  int32_t numPairs;
  const CapsuleDesc* capsules;   // [C]
  const int32_t* pairs;          // [P][2], i < j
  const int32_t* capsuleStart;   // [C+1] into capsulePair
  const int32_t* capsulePair;
  const int32_t* jointStart;     // [J+1] into jointCapsule
  const int32_t* jointCapsule;
};

// The flat joint-parameter operations (ik_device.cuh jointOpElement), forward / backward:
//   kJointOpParameterTransform  jp [7 J] = P theta + o (jointParameterRow)      /  g_theta [n] = P^T g_jp
//   kJointOpLocalState          local states [J][8] of jp [J][7]                /  g_jp [J][7] of g_local [J][8]
//   kJointOpFromLocal           jp [J][7] of local states [J][8]                /  g_local [J][8] of g_jp [J][7]
//   kJointOpFromWorld           jp [J][7] of world states [J][8]                /  g_world [J][8] of g_jp [J][7]
//   kJointOpInverseParameterTransform  theta [n] = W (jp - o), W = P^+          /  g_jp [7 J] = W^T g_theta
//   kJointOpClampParameters     theta [n] clamped by the MinMax limits          /  g_theta where min <= theta <= max, else 0
enum JointOp : int32_t {
  kJointOpParameterTransform = 0,
  kJointOpLocalState = 1,
  kJointOpFromLocal = 2,
  kJointOpFromWorld = 3,
  kJointOpInverseParameterTransform = 4,
  kJointOpClampParameters = 5,
};

// Linear-blend skinning tables (HostSkinning, makeSkinning), shared by the whole batch. The active influences of every vertex (the slots
// before its first zero weight) are stored twice: by vertex for the blend, and by joint for the reductions of the backward, where each
// joint's list is cut into segments of at most kSkinSegment influences that never cross a joint boundary.
constexpr int kSkinMaxInfluences = 8;  // kMaxSkinJoints (skin_weights.h:19)
constexpr int kSkinSegment = 128;      // influences per segment of the skel-state backward
constexpr int kSkinIbpStride = 12;     // inverse bind pose: the row-major top 3x4 of Affine3f::matrix()
struct SkinTables {
  int32_t numVertices, numSegments;
  const float* restVertices;    // [V][3]
  const int32_t* vertStart;     // [V+1] active influences by vertex (CSR)
  const int32_t* vertJoint;     // [nnz] slot order
  const float* vertWeight;      // [nnz]
  const float* inverseBindPose; // [J][12]
  const int32_t* infVertex;     // [nnz] by joint (CSC), vertices ascending within a joint
  const float* infWeight;       // [nnz]
  const int32_t* segStart;      // [S+1] into infVertex / infWeight
  const int32_t* segJoint;      // [S]
  const int32_t* jointSegStart; // [J+1] segments of each joint, in list order
};

// Blend-shape tables (HostBlendShape, makeBlendShape), shared by the whole batch; the mesh's V is the skinning's.
struct BlendShapeTables {
  int32_t numShapes;            // K; an instance uses the first K' <= K (computeDeltas' leftCols, blend_shape_base.cpp:18-24)
  const float* baseShape;       // [V][3]
  const float* shapeVectors;    // [K][V][3]
};

// Mesh-face tables (HostMeshFaces, makeMeshFaces), shared by the whole batch.
struct MeshFaceTables {
  int32_t numVertices, numFaces;
  const int32_t* faces;      // [F][3]
  const int32_t* vertStart;  // [V+1] into vertCorner
  const int32_t* vertCorner; // [3F]: 3 f + k of the corners that are the vertex, faces ascending, corners ascending
};

// Bounding-volume tree over the mesh faces (HostMeshTree, makeMeshTree): the topology only, shared by the whole batch; each instance's
// boxes are refitted to its vertices per call. Nodes are numbered level by level from the root (node 0); an internal node has its two
// children at nodeStart, nodeStart + 1 on the next level and nodeCount 0; a leaf holds the faces leafFaces[nodeStart .. + nodeCount),
// 1 <= nodeCount <= kLeafFaces.
constexpr int kLeafFaces = 4;  // faces per leaf (DESIGN §4, §7)
constexpr int kTreeStack = 32; // the traversal's stack: the tree's depth is at most this
struct MeshTreeTables {
  int32_t numNodes, depth;
  const int32_t* nodeStart;  // [numNodes]
  const int32_t* nodeCount;  // [numNodes]
  const int32_t* leafFaces;  // [F]: face indices, leaf by leaf
  const int32_t* levelStart; // [depth + 1]: the nodes of level L are levelStart[L] .. levelStart[L + 1)
};

// Point-cloud tree (find_closest_points), built per call and per target instance: the points sorted by Morton code, leaves of
// kLeafPoints consecutive sorted points, an implicit complete binary tree over the leaves padded to a power of two P (node 0 the root,
// the children of n at 2n + 1 and 2n + 2, leaf l at node P - 1 + l; a padding leaf has an empty box).
constexpr int kLeafPoints = 8;    // points per leaf (DESIGN §4, §7)
constexpr int kSortBits = 8;      // radix digit of the segmented LSD sort
constexpr int kSortPasses = 4;    // 32 bits: a code is at most 2^30
constexpr int kSortTile = 1024;   // points per (instance, tile) histogram
constexpr uint32_t kMortonNonFinite = 1u << 30; // the code of a point with a non-finite coordinate: after every finite one

} // namespace mb2
