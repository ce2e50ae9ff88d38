// sm_90a kernels of the batched Gauss-Newton iteration (declarations + launch parameter structs).
#pragma once

#include <cuda_runtime.h>

#include "ik_chol_sched.cuh"
#include "ik_chol_sched.h"
#include "ik_instance_launch.h"
#include "ik_solve_path.h"
#include "ik_types.h"

namespace mb2 {

struct SweepArgs {           // K1 (FK + residual + Jacobian) and K4 (FK + error only)
  FunctionTables T;
  int32_t batch;
  const float* theta;        // [B][ldTheta]
  int32_t ldTheta;
  const float* targets;      // [B][T.targetStride]
  const float* cweights;     // [numWeights] or [B][numWeights]
  float* jacobian;           // [B][numCols + 1][ldJ] (K1 only); column numCols is the residual vector
  double* errors;            // [B]
  const int32_t* active;     // optional per-instance mask
  float* stateOut;           // optional [B][J][8]
  int32_t planBatch;         // instances launchSweep plans the variant for (0: batch): the whole batch when this launch is one slice of it
  int32_t stageTables;       // set by launchSweep: 1 every read-only table in shared memory, 2 all but cells / contributions, 0 none
  int32_t warpsPerInstance;  // set by launchSweep: 1, 2, 4 or 8 warps share one instance (large rigs: few instances fit in shared memory)
  // the launch over instances b0 .. b0 + count - 1, with the variant planned for the whole batch
  SweepArgs slice(int b0, int count) const {
    SweepArgs a = *this;
    a.batch = count;
    a.planBatch = planBatch > 0 ? planBatch : batch;
    a.theta += size_t(b0) * ldTheta;
    a.targets += size_t(b0) * T.targetStride;
    if (T.weightsPerInstance) a.cweights += size_t(b0) * T.numWeights;
    if (jacobian != nullptr) a.jacobian += size_t(b0) * T.jacobianStride;
    a.errors += b0;
    if (active != nullptr) a.active += b0;
    if (stateOut != nullptr) a.stateOut += size_t(b0) * T.numJoints * 8;
    return a;
  }
};

struct JtJArgs {             // K2
  int32_t batch;
  const float* jacobian;     // [B][numCols + 1][ldJ]; column numCols = residual
  int32_t numCols, ldJ, kRows; // kRows = contraction length (rows rounded up to 4)
  int32_t ns;                // leading ns columns enter the normal equations (ns <= numCols)
  float* H;                  // [B][ns+1][ldH] symmetric matrix [J r]^T [J r] restricted to the leading ns columns + r, row-major;
                             // only the UPPER triangle H[i*ldH + j], j >= i, is guaranteed (column ns = J^T r: H[i*ldH + ns] = (J^T r)_i)
  int32_t ldH;               // multiple of 16, >= ns + 1
  size_t hStride;            // floats per instance in H
  const int32_t* active;
  float* g;                  // optional [B][ldG]: J^T r again, as a contiguous vector
  int32_t ldG;
};

struct CholArgs {            // K3: damped Cholesky + solve + update + SolverT bookkeeping
  int32_t batch;
  float* H;                  // [B][ns+1][ldH] full symmetric [JtJ, Jtr] (as written by K2); K3 never writes it unless it factors in place
  size_t hStride;            // floats per instance in H
  int32_t ns, ldH;
  float regularization;
  const int32_t* cols;       // [ns] subset -> full parameter index
  float* theta;              // [B][ldTheta], updated: theta[cols[a]] -= delta[a]   (no line search)
  int32_t ldTheta;
  float* delta;              // [B][ns] (always written)
  int32_t applyUpdate;       // 1: theta -= delta here
  SolveState state;          // the error of this iteration (from K1) and the SolverT bookkeeping
  int32_t bookkeeping;       // 1: run the SolverT convergence test here (no line search)
  float* gradDotDelta;       // optional [B]: Jtr . delta (SubsetGaussNewtonSolverT line search)
  const float* g;            // scheduled kernel: [B][ldG] J^T r as a contiguous vector (ldG = ns rounded up to 4)
  int32_t ldG;
  const float* tilesIn;      // scheduled kernel, optional: [B][tilesStride] tiles + slot-ordered J^T r from the Gram kernel (H, g unused)
  size_t tilesStride;
  int32_t profile;           // MB2_CHOL_PROFILE=1: block 0 prints per-phase cycles (debug aid)
  // the launch over instances b0 .. b0 + count - 1, which belong to instance slice k
  CholArgs slice(int k, int b0, int count) const {
    CholArgs a = *this;
    a.batch = count;
    if (H != nullptr) a.H += size_t(b0) * hStride;
    a.theta += size_t(b0) * ldTheta;
    a.delta += size_t(b0) * ns;
    a.state = state.slice(k, b0);
    if (gradDotDelta != nullptr) a.gradDotDelta += b0;
    if (g != nullptr) a.g += size_t(b0) * ldG;
    if (tilesIn != nullptr) a.tilesIn += size_t(b0) * tilesStride;
    return a;
  }
};

struct GramArgs {            // K2s: stored tiles of J^T J + lambda I and J^T r from the non-zero strips of the Jacobian (GramPlan)
  int32_t batch;
  const float* strips;       // [B][stripStride]: the Jacobian in strip layout + residual (FunctionTables::stripMode), written by the sweep kernel
  size_t stripStride;        // GramPlan::stride
  int32_t residOff;          // GramPlan::residOff
  const int32_t* active;
  int32_t numStrips, numTiles, numTileCols, nPad;
  int32_t numOrder;          // entries of the tile-order table ([rounds][kGramWarps], -1 = idle)
  // the GramPlan tables as one int32 blob (staged in shared memory by the kernel); offsets in ints
  const int32_t* blob;
  int32_t blobInts;
  int32_t offTileOrder, offTilePairStart, offPairA, offPairB, offColStripStart, offColStrip, offStripRow, offTileInfo;
  float regularization;
  float* out;                // [B][outStride]: numTiles x 256 floats in tile storage order, then the slot-ordered J^T r [nPad]
  size_t outStride;
  // the launch over instances b0 .. b0 + count - 1
  GramArgs slice(int b0, int count) const {
    GramArgs a = *this;
    a.batch = count;
    a.strips += size_t(b0) * stripStride;
    if (active != nullptr) a.active += b0;
    if (out != nullptr) a.out += size_t(b0) * outStride;
    return a;
  }
};
// threads: SolvePath::gramThreads
cudaError_t launchGramTiles(const GramArgs& a, int threads, cudaStream_t stream);

// K2s + K3 in one launch: strips in (bulk copy), tiles beyond the strips stored at once, the others parked in an L2-resident scratch
// slot and written over the strips once they are dead, tile Cholesky, update. No second launch; `g.out` is unused.
struct GramCholArgs {
  GramArgs g;
  CholArgs c;
  unsigned long long* phaseCycles; // optional [8], profiling instantiation: prologue, gram, parked tiles, diag, panel, update, backward, finish (block 0)
  // Parked tiles: a CTA takes one of 32 * parkSlotWords slots (a set bit of parkSlots = taken; all zero between launches) for the
  // Gram phase, and holds its tiles 0 .. parkTiles - 1 at park + (slot * parkTiles + tile) * 256 floats. At least as many slots as
  // CTAs can be resident (gramCholeskyParkSlots), so a free one always exists.
  float* park;
  uint32_t* parkSlots;
  int32_t parkSlotWords, parkTiles;
  // the launch over instances b0 .. b0 + count - 1, which belong to instance slice k
  GramCholArgs slice(int k, int b0, int count) const { GramCholArgs a = *this; a.g = g.slice(b0, count); a.c = c.slice(k, b0, count); return a; }
};
// gramCholeskyKernel's flattened tables (GramCholTables): in the kernel's parameter block (read through the constant cache) when
// they fit, else in global memory
constexpr int kGramCholParamEntries = 8192;
struct alignas(16) GramCholParamTables {
  GramCholLayout L;
  uint16_t tab[kGramCholParamEntries];
};
struct GramCholGlobalTables {
  GramCholLayout L;
  const uint16_t* tab;
};
// scratch slots for the parked tiles: resident CTAs of the launch on this device, rounded up to whole 32-bit words of parkSlots.
// The instance slices of a solve (SolvePath::slices) run concurrent gramCholeskyKernel grids on one bitmap: correct while the slots are
// at least all resident CTAs of every concurrent grid, which holds because the occupancy an SM allows this kernel bounds the CTAs of
// all its grids together.
int gramCholeskyParkSlots(const GramCholArgs& a, const CholSchedDev& sched, bool paramTables);
// tables: exactly one of inParams (non-null) or inGlobal is used
cudaError_t launchGramCholesky(const GramCholArgs& a, const CholSchedDev& sched, const GramCholParamTables* inParams, const GramCholGlobalTables& inGlobal, bool profile,
                               cudaStream_t stream);

// QR-accurate linear step (ik_qr.cu): Householder sweeps of the K-major Jacobian into a shared-memory R, replaces JtJ + Cholesky
struct QrArgs {
  CholArgs c;                // ns, regularization, cols, theta, delta, bookkeeping ... (H / tiles unused)
  const float* jacobian;     // [B][numCols + 1][ldJ], column numCols = residual (compact plan: numCols = ns)
  int32_t numCols, ldJ;
  const int32_t* chunkStart; // [numChunks + 1] first row of every chunk (device memory); a chunk never crosses an error-function block
  int32_t numChunks;
};
// TrustRegionQRT's iteration (ik_tr_qr.cuh): the QR arguments plus what getError needs inside the kernel and the solver's radius state
struct TrQrArgs {
  QrArgs q;
  FunctionTables T;
  const float* targets;
  const float* cweights;
  float* radius;      // [B] curTrustRegionRadius_ (in / out)
  float* rSaved;      // [B][packed upper triangle, rounded up to 4 floats] scratch for Rmatrix_
  float maxRadius;    // maxTrustRegionRadius_ = 10 (trust_region_qr.h:73)
  int32_t maxChunkRows;
};
cudaError_t launchTrustRegionQr(const TrQrArgs& a, cudaStream_t stream);
cudaError_t launchQrSolve(const QrArgs& a, int maxChunkRows, cudaStream_t stream);
// skeletonStateKernel<kBackward>: pymomentum's model_parameters_to_skeleton_state for a batch on the character alone (no solver
// function), and its backward
struct SkeletonStateArgs {
  CharacterTables T;
  SkeletonTables S;          // backward only
  int32_t numChildren;       // entries of S.children
  int32_t batch;
  const float* theta;        // [B][n], or [B][7 J] joint parameters when fromJointParameters
  const float* gradState;    // backward: [B][J][8] dLoss / d state
  float* out;                // forward: [B][J][8] (t, q xyzw, s); backward: [B][n] dLoss / d theta ([B][7 J] d joint parameters), overwritten
  int32_t fromJointParameters; // joint_parameters_to_skeleton_state: the FK from joint parameters, S.ptCol* unused
};
// What a per-instance kernel of the character operations launches (mb2_character_get_instance_launch,
// mb2_solver_function_get_input_gradient_launch): planInstanceOp's plan and the grid the device's occupancy gives it
struct InstanceLaunchQuery {
  InstanceLaunch launch;
  int32_t grid{0};
};
// `query` (optional): the launch is planned and reported there and nothing is enqueued; all zero for an empty batch
cudaError_t launchSkeletonState(const SkeletonStateArgs& a, bool backward, cudaStream_t stream, InstanceLaunchQuery* query = nullptr);
// positionsKernel<kBackward>: pymomentum's model_parameters_to_positions / joint_parameters_to_positions for a batch on the character
// alone, and their backward
struct PositionArgs {
  CharacterTables T;
  SkeletonTables S;          // backward only
  PointTables P;             // device memory
  int32_t numChildren;       // entries of S.children
  int32_t batch;
  const float* params;       // [B][n], or [B][7 J] joint parameters when fromJointParameters
  const float* offsets;      // [N][3] shared by the batch, or [B][N][3] when offsetsBatched
  int32_t offsetsBatched;
  float* positions;          // forward: [B][N][3]
  const float* gradPositions; // backward: [B][N][3] dLoss / d positions
  float* gradParams;         // backward, optional: [B][n] ([B][7 J]), overwritten
  float* gradOffsets;        // backward, optional: [N][3] (the batch sum) or [B][N][3], overwritten
  int32_t fromJointParameters;
};
// Both enqueue on `stream`. The backward of shared offsets takes stream-ordered scratch (cudaMallocAsync) for the per-instance offset
// gradients of a slice of instances (at most 256 MiB) and 128 x [N][3] floats for their chunk sums.
cudaError_t launchPositions(const PositionArgs& a, cudaStream_t stream);
cudaError_t launchPositionsBackward(const PositionArgs& a, cudaStream_t stream);
// the launch of positionsKernel over a.batch instances with a.P.numPoints points (a.P's arrays are not read); the shared-offset
// backward launches it per slice of whole batch-sum chunks, which is the whole batch unless the offset rows exceed the scratch bound
cudaError_t queryPositionsLaunch(const PositionArgs& a, bool backward, InstanceLaunchQuery* query);
// parameterLimitsKernel<kBackward>: the rows of the character's limits (LimitErrorFunction at weight 1, L2 loss) for a batch of model
// parameters, and their backward
struct ParameterLimitArgs {
  CharacterTables T;
  SkeletonTables S;           // backward only
  LimitTables L;              // device memory
  int32_t numChildren;        // entries of S.children
  int32_t batch;
  const float* theta;         // [B][n]
  float* residual;            // forward: [B][R]
  const float* gradResidual;  // backward: [B][R] dLoss / d residual
  float* gradTheta;           // backward: [B][n], overwritten
};
// Both enqueue on `stream` and take no scratch. R == 0: the forward writes nothing and the backward zeroes gradTheta. With `query`,
// the launch is reported there and nothing is enqueued.
cudaError_t launchParameterLimits(const ParameterLimitArgs& a, bool backward, cudaStream_t stream, InstanceLaunchQuery* query = nullptr);
// collisionKernel<kBackward>: the self-collision rows of the character's tapered capsules for a batch of skeleton states, and their
// backward
struct CollisionArgs {
  CharacterTables T;          // numJoints only
  CollisionTables L;          // device memory
  int32_t batch;
  const float* state;         // [B][J][8]
  float* residual;            // forward: [B][P]
  const float* gradResidual;  // backward: [B][P] dLoss / d residual
  float* gradState;           // backward: [B][J][8], overwritten
};
// Both enqueue on `stream` and take no scratch. P == 0: the forward writes nothing and the backward zeroes gradState. With `query`, the
// launch is reported there and nothing is enqueued.
cudaError_t launchCollision(const CollisionArgs& a, bool backward, cudaStream_t stream, InstanceLaunchQuery* query = nullptr);
// parameterTransformKernel ... clampParametersBackwardKernel: the flat joint-parameter operations of ik_device.cuh jointOpElement for a
// batch, forward or backward; arrays [B][...] dense, device memory
struct JointOpArgs {
  CharacterTables T;
  SkeletonTables S;          // the backward of kJointOpParameterTransform (ptCol*), of kJointOpFromWorld (children), both directions
                             // of kJointOpInverseParameterTransform (inv*) and of kJointOpClampParameters (paramClamp)
  int32_t batch;
  const float* in;           // the forward's input (backward: the forward's input, unused by the two linear ParameterTransform ops)
  const float* grad;         // backward: dLoss / d the forward's output
  float* out;                // forward: the output; backward: dLoss / d in, overwritten
};
cudaError_t launchJointOp(const JointOpArgs& a, JointOp op, bool backward, cudaStream_t stream);
// skinVertexKernel / skinStatePartialKernel / skinStateFinishKernel: linear-blend skinning of a batch (applySSD) and its backward
struct SkinArgs {
  SkinTables S;
  int32_t numJoints;
  int32_t batch;
  const float* skelState;    // [B][J][8] (t, q xyzw, s)
  const float* restPoints;   // [V][3] shared or [B][V][3]
  int32_t restBatched;
  const float* gradPoints;   // backward: [B][V][3] dLoss / d points
  float* points;             // forward: [B][V][3]
  float* gradState;          // backward, optional: [B][J][8]
  float* gradRest;           // backward, optional: [B][V][3] when batched, else [V][3] (the batch sum)
};
// Both enqueue on `stream`; the backward takes bounded stream-ordered scratch (cudaMallocAsync) for its partial sums.
cudaError_t launchSkinPoints(const SkinArgs& a, cudaStream_t stream);
cudaError_t launchSkinPointsBackward(const SkinArgs& a, cudaStream_t stream);
// blendSkinKernel / blendWeightPartialKernel / blendWeightFinishKernel: skinning with an identity blend shape (skinWithBlendShapes,
// blend_shape_skinning.cpp:50-140) and its backward
struct BlendSkinArgs {
  SkinArgs skin;             // S, numJoints, batch, skelState; forward: points; backward: gradPoints, gradState (optional). No rest points.
  BlendShapeTables Bs;
  int32_t numWeights;        // K', 1 <= K' <= K
  const float* blendWeights; // [B][K']
  float* gradWeights;        // backward, optional: [B][K']
};
// Both enqueue on `stream`; the backward takes bounded stream-ordered scratch (cudaMallocAsync): the shaped rest points of a slice of
// instances for the skel-state gradient (then launchSkinPointsBackward on them), and per-vertex-block partial sums of the weight gradient.
// Whether the narrowest tile's shared memory (its weights [K'][4] and the J transforms) fits on the device: K' and J bound it
bool blendSkinFits(const BlendSkinArgs& a);
cudaError_t launchSkinWithBlendShapes(const BlendSkinArgs& a, cudaStream_t stream);
cudaError_t launchSkinWithBlendShapesBackward(const BlendSkinArgs& a, cudaStream_t stream);
// vertexNormalKernel / vertexNormalGradKernel: area-weighted vertex normals of [B][V][3] positions over the mesh's faces
// (compute_vertex_normals, tensor_skinning.cpp:354-383) and their backward to the positions
struct NormalArgs {
  MeshFaceTables M;
  int32_t batch;
  const float* positions;   // [B][V][3]
  float* normals;           // forward: [B][V][3]
  const float* gradNormals; // backward: [B][V][3]
  float* gradPositions;     // backward: [B][V][3]
};
// Both enqueue on `stream`; the backward takes stream-ordered scratch (cudaMallocAsync) for h of a slice of instances, at most 256 MiB.
cudaError_t launchVertexNormals(const NormalArgs& a, cudaStream_t stream);
cudaError_t launchVertexNormalsBackward(const NormalArgs& a, cudaStream_t stream);
// meshTreeRefitKernel / closestPointKernel: the closest point on each instance's mesh of each of its query points (pymomentum
// find_closest_points_on_mesh), over the shared tree topology refitted to the instance's vertices
struct ClosestPointArgs {
  MeshFaceTables M;
  MeshTreeTables T;
  int32_t batch, numPoints;
  float maxDist2;        // max_dist * max_dist; +inf for no bound
  const float* vertices; // [B][V][3]
  const float* points;   // [B][N][3]
  float* outPoints;      // [B][N][3]
  int32_t* outFace;      // [B][N]
  float* outBary;        // [B][N][3]
};
// Enqueues on `stream`; the boxes of a slice of instances go to stream-ordered scratch (cudaMallocAsync), at most 256 MiB.
cudaError_t launchClosestPointsOnMesh(const ClosestPointArgs& a, cudaStream_t stream);
// cloud*Kernel / closestCloudKernel: the closest target point of each query point (pymomentum find_closest_points), over a tree built
// per call on the device for each target instance
struct ClosestCloudArgs {
  int32_t batch, numSource, numTarget;
  bool targetBatched;          // target [B][M][3], else [1][M][3]: one tree for the whole batch
  float maxDist2;              // max_dist * max_dist; +inf for no bound
  float maxNormalDot;          // the normal variant's lower bound on dot(n_p, n_t)
  const float* source;         // [B][N][3]
  const float* sourceNormals;  // [B][N][3], or null: the plain variant
  const float* target;         // [B or 1][M][3]
  const float* targetNormals;  // [B or 1][M][3] when sourceNormals is set
  float* outPoints;            // [B][N][3]
  float* outNormals;           // [B][N][3] when sourceNormals is set
  int32_t* outIndex;           // [B][N]
};
// Enqueues on `stream`; the trees of a slice of target instances go to stream-ordered scratch (cudaMallocAsync), at most 256 MiB.
cudaError_t launchClosestPointsOnCloud(const ClosestCloudArgs& a, cudaStream_t stream);
// inputGradientKernel: d/d input [grad_theta E . v] of one Position or Orientation (matrix difference) block with the L2 loss, per
// instance: the input contraction of solve_ik's implicit-function backward
struct InputGradientArgs {
  FunctionTables T;          // character part, units / efs, targetStride, weightsPerInstance, numWeights
  int32_t unitBegin;         // first unit of the block (its constraints are units unitBegin .. + numConstraints - 1)
  int32_t numConstraints;
  int32_t kind;              // kUnitPosition or kUnitOrientation
  int32_t batch;
  const float* theta;        // [B][n]
  const float* direction;    // [B][n] v; entries of disabled parameters are ignored
  const int32_t* enabledList; // [numEnabled]
  int32_t numEnabled;
  const float* targets;      // the handle's per-instance records [B][targetStride]
  const float* cweights;     // constraint weights [numWeights] or [B][numWeights]
  float* gradWeights;        // [B][nc] or null
  float* gradOffsets;        // [B][nc][3|4] or null
  float* gradTargets;        // [B][nc][3|4] or null
};
cudaError_t launchInputGradients(const InputGradientArgs& a, cudaStream_t stream, InstanceLaunchQuery* query = nullptr);
// implicitDirectionKernel: per instance v = (2 J_E^T J_E)^+ g (the reference's hessianInverseTimes, ik_jacobi.cuh), J v, the residual
// and the gradient RMS, from the K-major Jacobian [B][n + 1][ldJ] of a mode-0 plan
struct ImplicitDirectionArgs {
  int32_t batch;
  int32_t numParams;         // n
  int32_t rows;              // unpadded residual rows of the plan
  int32_t rowStride;         // floats per instance of jacobianDirection / residual (>= rows; the rows past `rows` are written 0)
  int32_t ldJ;
  const float* jacobian;     // [B][n + 1][ldJ], column n = residual
  const int32_t* enabledList; // E, ascending [numEnabled]
  int32_t numEnabled;
  const float* gradParameters; // [B][n] dLoss / d theta
  float* direction;          // [B][n] v, 0 on disabled parameters; or null
  float* jacobianDirection;  // [B][rowStride] J v; or null
  float* residual;           // [B][rowStride]; or null
  float* gradientRms;        // [B] sqrt(mean_E (2 J_E^T r)^2); or null
  double* scratch;           // [grid][slotDoubles]: the rotation log, then K when it does not fit in shared memory
  size_t slotDoubles;
  int32_t gramInShared;
};
struct ImplicitDirectionConfig {
  int grid{0};
  size_t smem{0};
  bool gramInShared{true};
  size_t slotDoubles{0};     // scratch per CTA; the launch needs grid x slotDoubles doubles
};
// sizes the persistent grid (shared memory, occupancy, the scratch budget) for a.rows / a.numEnabled / a.batch
cudaError_t implicitDirectionConfigure(const ImplicitDirectionArgs& a, ImplicitDirectionConfig& cfg);
cudaError_t launchImplicitDirection(const ImplicitDirectionArgs& a, const ImplicitDirectionConfig& cfg, cudaStream_t stream);
struct SweepLaunch {         // the variant and launch shape launchSweep chose (mb2_solver_function_get_sweep_launch)
  int32_t stageTables;       // 1 every read-only table in shared memory, 2 all but cells / contributions, 0 none
  int32_t warpsPerInstance;  // W: 1, 2, 4 or 8
  int32_t groupsPerCta;      // instances in flight per CTA
  int32_t grid;              // CTAs
  int64_t smemBytes;         // dynamic shared memory per CTA
};
// `out` (optional) receives the decision before the kernel is enqueued, all zero when no configuration fits
cudaError_t launchSweep(const SweepArgs& a, bool jacobian, cudaStream_t stream, SweepLaunch* out = nullptr);
size_t sweepSmemPerInstance(const FunctionTables& T, int warpsPerInstance);
cudaError_t launchJtJSimt(const JtJArgs& a, cudaStream_t stream);
// NB, inSmem: SolvePath::denseNb / denseInSmem
cudaError_t launchCholesky(const CholArgs& a, int NB, bool inSmem, cudaStream_t stream);
// level-scheduled tile-sparse variant (ik_chol_sched.h); returns cudaErrorInvalidConfiguration when the tiles do not fit in shared memory
// `a.H` is the full symmetric system in device-column (= elimination) order; threads: SolvePath::cholThreads
cudaError_t launchCholeskyScheduled(const CholArgs& a, const CholSchedDev& sched, int threads, cudaStream_t stream);
inline int cholGradientLd(int ns) { return (ns + 3) & ~3; }
cudaError_t initKernelAttributes();
DeviceLimits deviceLimits(); // of the device initKernelAttributes last read

// line-search helpers
cudaError_t launchTrialUpdate(int batch, const float* thetaOrig, int ldTheta, const float* delta, int ns, const int32_t* cols, const float* scale /*[B]*/,
                              float* thetaTrial, const int32_t* active, cudaStream_t stream);
struct LineSearchArgs {
  int32_t batch;
  const double* errors;      // error_ at theta (from the Jacobian pass)
  const double* trialErrors; // getError(theta - scale*delta)
  const float* gradDotDelta; // [B] (subset variant) or nullptr
  float* scale;              // [B] in/out line-search scale
  int32_t* searching;        // [B] 1 while the instance is still halving
  int32_t step;              // 0..9
  int32_t subsetVariant;
};
cudaError_t launchLineSearchStep(const LineSearchArgs& a, cudaStream_t stream);
// the SolverT bookkeeping of s.iteration for the active instances of a batch (after a line search)
cudaError_t launchBookkeeping(int batch, const SolveState& s, cudaStream_t stream);
cudaError_t launchScatterTargets(const float* packed, float* dst, int size, int strideFloats, int batch, cudaStream_t stream);
cudaError_t launchNormalizeQuats(float* base, int count, int strideFloats, int quatsPerRecord, int batch, cudaStream_t stream);

} // namespace mb2
