// C-ABI of momentum_b200 (include/momentum_b200.h): handle management, host<->device plumbing and
// the batched SolverT::solve driver. No CPU fallback: every compute entry fails with MB2_ERR_CUDA
// when no sm_90 device is usable.
#include "../../include/momentum_b200.h"

#include <cuda_runtime.h>
#include <nvtx3/nvToolsExt.h>

#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "ik_chol_sched.h"
#include "ik_fused.cuh"
#include "ik_jtj_tc.cuh"
#include "ik_kernels.cuh"
#include "ik_plan.h"
#include "ik_solve_path.h"

using namespace mb2;

namespace {

thread_local std::string g_lastError;

int fail(int code, const std::string& msg) {
  g_lastError = msg;
  return code;
}
#define MB2_CUDA(expr)                                                                                  \
  do {                                                                                                  \
    cudaError_t _e = (expr);                                                                            \
    if (_e != cudaSuccess) return fail(MB2_ERR_CUDA, std::string(#expr) + ": " + cudaGetErrorString(_e)); \
  } while (0)
#define MB2_CHECK(cond, msg)                                   \
  do {                                                         \
    if (!(cond)) return fail(MB2_ERR_INVALID_ARGUMENT, (msg)); \
  } while (0)

template <class T>
struct DeviceBuffer {
  T* p{nullptr};
  size_t n{0};
  ~DeviceBuffer() { release(); }
  void release() {
    if (p) cudaFree(p);
    p = nullptr;
    n = 0;
  }
  cudaError_t resize(size_t count) {
    if (count <= n && p) return cudaSuccess;
    release();
    if (count == 0) return cudaSuccess;
    cudaError_t e = cudaMalloc(&p, count * sizeof(T));
    if (e == cudaSuccess) n = count;
    return e;
  }
  cudaError_t upload(const std::vector<T>& v, cudaStream_t s) {
    cudaError_t e = resize(std::max<size_t>(v.size(), 1));
    if (e != cudaSuccess || v.empty()) return e;
    return cudaMemcpyAsync(p, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice, s);
  }
};

int roundUp(int v, int m) { return (v + m - 1) / m * m; }

int usableDevices();

// Every entry point that allocates or launches runs with the handle's device current and restores the caller's device on exit
// (a single process may drive several GPUs: one character / solver function per device).
struct DeviceGuard {
  int prev{-1};
  bool switched{false};
  cudaError_t err{cudaSuccess};
  explicit DeviceGuard(int device) {
    err = cudaGetDevice(&prev);
    if (err == cudaSuccess && prev != device) { err = cudaSetDevice(device); switched = err == cudaSuccess; }
  }
  ~DeviceGuard() { if (switched) cudaSetDevice(prev); }
  DeviceGuard(const DeviceGuard&) = delete;
  DeviceGuard& operator=(const DeviceGuard&) = delete;
};
#define MB2_DEVICE_GUARD(device)                                                                                      \
  if (usableDevices() <= 0) return fail(MB2_ERR_CUDA, "no usable sm_90 CUDA device: momentum_b200 has no CPU fallback"); \
  DeviceGuard _guard(device);                                                                                         \
  MB2_CUDA(_guard.err)

// NVTX ranges named like the reference's MT_PROFILE_FUNCTION zones (solver.cpp:51, gauss_newton_solver.cpp:225, skeleton_state.cpp:88)
struct NvtxRange {
  explicit NvtxRange(const char* name) { nvtxRangePushA(name); }
  ~NvtxRange() { nvtxRangePop(); }
};

} // namespace

// the device copy of a HostSkinning (SkinTables)
struct SkinBuffers {
  DeviceBuffer<float> rest, vertWeight, ibp, infWeight;
  DeviceBuffer<int32_t> vertStart, vertJoint, infVertex, segStart, segJoint, jointSegStart;
};
// the device copy of a HostBlendShape (BlendShapeTables)
struct BlendShapeBuffers {
  DeviceBuffer<float> baseShape, shapeVectors;
};
// the device copy of a HostMeshFaces (MeshFaceTables)
struct MeshFaceBuffers {
  DeviceBuffer<int32_t> faces, vertStart, vertCorner;
};
// the device copy of a HostMeshTree (MeshTreeTables)
struct MeshTreeBuffers {
  DeviceBuffer<int32_t> nodeStart, nodeCount, leafFaces, levelStart;
};
// the device copy of a HostLimitTables (LimitTables, SkeletonTables::paramClamp)
struct LimitBuffers {
  DeviceBuffer<LimitDesc> limits;
  DeviceBuffer<float> ellipsoidData, rowCoef, paramCoef, paramClamp;
  DeviceBuffer<int32_t> jointStart, jointEntry, rowStart, rowLimit, paramStart, paramLimit;
};

// the device copy of a HostCollision (CollisionTables)
struct CollisionBuffers {
  DeviceBuffer<CapsuleDesc> capsules;
  DeviceBuffer<int32_t> pairs, capsuleStart, capsulePair, jointStart, jointCapsule;
};

struct mb2_character {
  int device{0};
  HostCharacter host;
  DeviceBuffer<int32_t> parent, ptOuter, ptInner, levelStart, levelJoints;
  DeviceBuffer<float> offset, prerot, ptVals, ptOffsets;
  DeviceBuffer<int32_t> childStart, children, ptColStart, ptColRows; // skeleton-state backward (HostCharacter::buildBackwardTables)
  DeviceBuffer<float> ptColVals;
  DeviceBuffer<int32_t> invStart, invRows, invRowStart, invParams; // inverse ParameterTransform (HostCharacter::buildInverseTables)
  DeviceBuffer<float> invVals, invRowVals;
  uint64_t limitsVersion{0};
  // the limits as parameter_limits_residual and apply_model_param_limits read them, built and uploaded whenever the limits are set
  HostLimitTables limits;
  std::unique_ptr<LimitBuffers> limitsDev; // replaced whole by installLimitTables
  // the tapered capsules and their valid pairs (mb2_character_set_collision_geometry); collisionDev is null until a geometry is set
  HostCollision collision;
  std::unique_ptr<CollisionBuffers> collisionDev;
  // linear-blend skinning (mb2_character_set_skinning): numVertices == 0 when there is none
  HostSkinning skin;
  std::unique_ptr<SkinBuffers> skinDev; // replaced whole by mb2_character_set_skinning, never rewritten in place
  // identity blend shape (mb2_character_set_blend_shape): numShapes == 0 when there is none
  HostBlendShape blend;
  std::unique_ptr<BlendShapeBuffers> blendDev; // replaced whole by mb2_character_set_blend_shape
  // mesh faces (mb2_character_set_mesh_faces): numVertices == 0 when there are none
  HostMeshFaces faces;
  std::unique_ptr<MeshFaceBuffers> facesDev; // replaced whole by mb2_character_set_mesh_faces
  // bounding-volume tree over the faces (mb2_character_set_mesh_tree): numNodes == 0 when there is none
  HostMeshTree tree;
  std::unique_ptr<MeshTreeBuffers> treeDev; // replaced whole by mb2_character_set_mesh_tree, dropped by mb2_character_set_mesh_faces
  // the device copies above, as the kernels read them; each mesh table only while it is installed
  CharacterTables tables() const;
  SkeletonTables skeletonTables() const; // the skeleton-state backward's
  SkinTables skinTables() const;
  BlendShapeTables blendShapeTables() const;
  MeshFaceTables meshFaceTables() const;
  MeshTreeTables meshTreeTables() const;
  LimitTables limitTables() const;
  CollisionTables collisionTables() const;
};

struct DeviceSchedule {
  CholSchedule host;
  CholSchedDev dev{};
  DeviceBuffer<int32_t> blob;
  GramPlan gram;          // tile-sparse Gram tables of the same plan (rows aligned to quads), when the plan has strips
  DeviceBuffer<int32_t> gBlob;
  int32_t gBlobInts{0}, gOffsets[8]{};
  // gramCholeskyKernel's flattened tables: in its parameter block when they fit (gcParams), else in global memory (gcTab)
  GramCholTables gc;
  bool gcValid{false};
  std::unique_ptr<GramCholParamTables> gcParams;
  DeviceBuffer<uint16_t> gcTab;
  // fused persistent kernel (ik_fused.cuh): every table of the plan as one blob + how many instance groups fit beside it
  DeviceBuffer<int32_t> fBlob;
  FusedBlobLayout fLayout{};
  int fusedGroups{0}; // SolvePath::fused of the solve that requested this plan
};

struct mb2_solver_function {
  const mb2_character* ch{nullptr};
  int B{0};
  cudaStream_t stream{nullptr};
  HostFunction host;
  bool planDirty{true};
  int planMode{0};        // 0 full columns (API parity), 1 solver: enabled columns in natural order, 2 solver: elimination order + tile schedule
  bool planSchedDense{false};
  bool planAlignRows{false}; // row groups aligned to 4 (tile-sparse Gram reads the Jacobian in 4-row strips)
  uint64_t planLimitsVersion{~0ull};
  Plan plan;
  int ldJ{32};
  // device tables
  DeviceBuffer<EfDesc> dEfs;
  DeviceBuffer<UnitDesc> dUnits;
  DeviceBuffer<CellDesc> dCells;
  DeviceBuffer<ContribDesc> dContribs;
  DeviceBuffer<float> dLimitData;
  DeviceBuffer<int32_t> dEnabledList, dIdentity, dDeviceCols;
  // device data
  DeviceBuffer<float> dTargets, dWeights, dJ, dTheta, dState, dH, dTargetStage;
  DeviceBuffer<double> dErrors;
  DeviceBuffer<double> dJacobi;          // implicit direction: per-CTA rotation logs (and Gram matrices too large for shared memory)
  std::unique_ptr<DeviceSchedule> sched; // Cholesky schedule of the current (compact) plan
  SweepLaunch lastSweep[2]{};            // what launchSweep last chose: [0] error-only (K4), [1] Jacobian (K1)
  FunctionTables tables() const;
};

struct PhaseEvent {
  cudaEvent_t start, stop;
  int phase;
};

struct mb2_solver {
  mb2_solver_function* fn{nullptr};
  mb2_gauss_newton_options opt{};
  DeviceBuffer<float> dH, dDelta, dThetaOrig, dTheta0, dScale, dGradDotDelta, dThetaStage, dGrad, dTiles, dRadius, dRSaved;
  DeviceBuffer<double> dLastErrors, dTrialErrors, dHistory;
  DeviceBuffer<int32_t> dActive, dIterations, dStatus, dSearching, dActiveCount, dWorkCounter, dQrChunks;
  DeviceBuffer<unsigned long long> dPhaseCycles;
  DeviceBuffer<float> dPark;          // gramCholeskyKernel: parked Gram tiles, one slot per resident CTA
  DeviceBuffer<uint32_t> dParkSlots;  // its slot bitmap (zero between launches)
  SolvePath path; // what the last solve ran (chooseSolvePath)
  cudaEvent_t fusedStart{nullptr}, fusedStop{nullptr};
  double fusedMs{0};
  int* hActiveCount{nullptr}; // pinned, [kSolveSlices]: the active counter of every slice
  // the streams of slices 1 .. kSolveSlices - 1 (slice 0 runs on the caller's stream) and the events that fork them from, and join
  // them back to, the caller's stream; created by the first sliced solve
  cudaStream_t sliceStreams[kSolveSlices - 1]{};
  cudaEvent_t forkEvent{nullptr}, joinEvents[kSolveSlices - 1]{};
  // pinned staging of the per-instance results of an asynchronous host solve: [B] errors (double) | [B] iterations | [B] status, filled by
  // copies enqueued behind the solve so that mb2_solver_wait needs one stream synchronisation and no further device round trip
  char* hResults{nullptr};
  size_t hResultsBytes{0};
  bool resultsStaged{false};
  uint64_t totalIterations{0}, kernelLaunches{0};
  bool profiling{false};
  bool inKernelProfile{false}; // profiling level 2: the instrumented kernel instantiations (clock64 per phase; slower)
  std::vector<PhaseEvent> events;
  double phaseMs[4]{0, 0, 0, 0};
  uint64_t phaseLaunches[4]{0, 0, 0, 0};
  size_t historyStride{0};
  ~mb2_solver() {
    if (hActiveCount) cudaFreeHost(hActiveCount);
    if (hResults) cudaFreeHost(hResults);
    if (fusedStart) cudaEventDestroy(fusedStart);
    if (fusedStop) cudaEventDestroy(fusedStop);
    for (auto& e : events) { cudaEventDestroy(e.start); cudaEventDestroy(e.stop); }
    if (forkEvent) cudaEventDestroy(forkEvent);
    for (int i = 0; i < kSolveSlices - 1; ++i) {
      if (joinEvents[i]) cudaEventDestroy(joinEvents[i]);
      if (sliceStreams[i]) cudaStreamDestroy(sliceStreams[i]);
    }
  }
};

CharacterTables mb2_character::tables() const {
  CharacterTables C{};
  C.numJoints = host.numJoints;
  C.numParams = host.numParams;
  C.parent = parent.p;
  C.offset = offset.p;
  C.prerot = prerot.p;
  C.ptOuter = ptOuter.p;
  C.ptInner = ptInner.p;
  C.ptVals = ptVals.p;
  C.ptOffsets = ptOffsets.p;
  C.numLevels = int(host.levelStart.size()) - 1;
  C.ptNnz = int(host.ptInner.size());
  C.levelStart = levelStart.p;
  C.levelJoints = levelJoints.p;
  return C;
}

SkeletonTables mb2_character::skeletonTables() const {
  return SkeletonTables{childStart.p, children.p,  ptColStart.p, ptColRows.p, ptColVals.p, invStart.p,
                        invRows.p,    invVals.p,   invRowStart.p, invParams.p, invRowVals.p, limitsDev ? limitsDev->paramClamp.p : nullptr};
}

LimitTables mb2_character::limitTables() const {
  const LimitBuffers& d = *limitsDev;
  return LimitTables{int32_t(limits.limits.size()), limits.numRows, limits.ellipsoid ? 1 : 0, d.limits.p, d.ellipsoidData.p, d.jointStart.p,
                     d.jointEntry.p, d.rowStart.p, d.rowLimit.p, d.rowCoef.p, d.paramStart.p, d.paramLimit.p, d.paramCoef.p};
}

CollisionTables mb2_character::collisionTables() const {
  const CollisionBuffers& d = *collisionDev;
  return CollisionTables{int32_t(collision.capsules.size()), collision.numPairs(), d.capsules.p, d.pairs.p, d.capsuleStart.p, d.capsulePair.p,
                         d.jointStart.p, d.jointCapsule.p};
}

SkinTables mb2_character::skinTables() const {
  const SkinBuffers& d = *skinDev;
  return SkinTables{skin.numVertices, skin.numSegments(), d.rest.p, d.vertStart.p, d.vertJoint.p, d.vertWeight.p,
                    d.ibp.p, d.infVertex.p, d.infWeight.p, d.segStart.p, d.segJoint.p, d.jointSegStart.p};
}

BlendShapeTables mb2_character::blendShapeTables() const { return BlendShapeTables{blend.numShapes, blendDev->baseShape.p, blendDev->shapeVectors.p}; }

MeshFaceTables mb2_character::meshFaceTables() const {
  return MeshFaceTables{faces.numVertices, faces.numFaces, facesDev->faces.p, facesDev->vertStart.p, facesDev->vertCorner.p};
}

MeshTreeTables mb2_character::meshTreeTables() const {
  return MeshTreeTables{tree.numNodes, tree.depth, treeDev->nodeStart.p, treeDev->nodeCount.p, treeDev->leafFaces.p, treeDev->levelStart.p};
}

namespace {
// Replaces one of a character's mesh tables: fresh device buffers, filled by upload(buffers, fresh) when `present` (else none), so that a
// failed upload leaves the earlier table whole; the device is synchronised before the swap, so no work in flight on any stream still
// reads the buffers that are freed.
template <class Buffers, class Host, class Upload>
int installTables(int device, std::unique_ptr<Buffers>& dev, Host& host, Host&& fresh, Upload upload, bool present = true) {
  MB2_DEVICE_GUARD(device);
  std::unique_ptr<Buffers> d;
  if (present) {
    d = std::make_unique<Buffers>();
    const int rc = upload(*d, fresh);
    if (rc != MB2_OK) return rc;
  }
  MB2_CUDA(cudaDeviceSynchronize());
  dev = std::move(d);
  host = std::move(fresh);
  return MB2_OK;
}

// installs tree t (numNodes == 0: none)
int installMeshTree(mb2_character* c, HostMeshTree&& t) {
  const bool present = t.numNodes > 0;
  return installTables(c->device, c->treeDev, c->tree, std::move(t), [](MeshTreeBuffers& d, const HostMeshTree& t) -> int {
    MB2_CUDA(d.nodeStart.upload(t.nodeStart, nullptr));
    MB2_CUDA(d.nodeCount.upload(t.nodeCount, nullptr));
    MB2_CUDA(d.leafFaces.upload(t.leafFaces, nullptr));
    MB2_CUDA(d.levelStart.upload(t.levelStart, nullptr));
    return MB2_OK;
  }, present);
}

// installs the collision geometry h
int installCollision(mb2_character* c, HostCollision&& h) {
  return installTables(c->device, c->collisionDev, c->collision, std::move(h), [](CollisionBuffers& d, const HostCollision& h) -> int {
    MB2_CUDA(d.capsules.upload(h.capsules, nullptr));
    MB2_CUDA(d.pairs.upload(h.pairs, nullptr));
    MB2_CUDA(d.capsuleStart.upload(h.capsuleStart, nullptr));
    MB2_CUDA(d.capsulePair.upload(h.capsulePair, nullptr));
    MB2_CUDA(d.jointStart.upload(h.jointStart, nullptr));
    MB2_CUDA(d.jointCapsule.upload(h.jointCapsule, nullptr));
    return MB2_OK;
  });
}

// builds the limit tables of c's limits and installs them (rejected limits install empty tables and keep the reason)
int installLimitTables(mb2_character* c) {
  return installTables(c->device, c->limitsDev, c->limits, makeLimitTables(c->host), [](LimitBuffers& d, const HostLimitTables& t) -> int {
    MB2_CUDA(d.limits.upload(t.limits, nullptr));
    MB2_CUDA(d.ellipsoidData.upload(t.ellipsoidData, nullptr));
    MB2_CUDA(d.jointStart.upload(t.jointStart, nullptr));
    MB2_CUDA(d.jointEntry.upload(t.jointEntry, nullptr));
    MB2_CUDA(d.rowStart.upload(t.rowStart, nullptr));
    MB2_CUDA(d.rowLimit.upload(t.rowLimit, nullptr));
    MB2_CUDA(d.rowCoef.upload(t.rowCoef, nullptr));
    MB2_CUDA(d.paramStart.upload(t.paramStart, nullptr));
    MB2_CUDA(d.paramLimit.upload(t.paramLimit, nullptr));
    MB2_CUDA(d.paramCoef.upload(t.paramCoef, nullptr));
    MB2_CUDA(d.paramClamp.upload(t.paramClamp, nullptr));
    return MB2_OK;
  });
}
} // namespace

FunctionTables mb2_solver_function::tables() const {
  FunctionTables T{ch->tables()};
  T.numEf = int(plan.efs.size());
  T.numUnits = int(plan.units.size());
  T.numCells = int(plan.cells.size());
  T.efs = dEfs.p;
  T.units = dUnits.p;
  T.cells = dCells.p;
  T.contribs = dContribs.p;
  T.limitData = dLimitData.p;
  T.targetStride = host.targetStride;
  T.recStride = plan.recStride;
  T.numRows = plan.numRows;
  T.ldJ = ldJ;
  T.numCols = plan.numCols;
  T.weightsPerInstance = host.weightsPerInstance ? 1 : 0;
  T.numWeights = host.numWeights;
  T.numContribs = int(plan.contribs.size());
  T.numLimitData = int(plan.limitData.size());
  const bool strips = planMode == 2 && planAlignRows && sched;
  T.stripMode = strips ? 1 : 0;
  T.residOff = strips ? sched->gram.residOff : 0;
  T.jacobianStride = strips ? size_t(sched->gram.stride) : size_t(plan.numCols + 1) * ldJ;
  return T;
}

namespace {

bool g_deviceChecked = false;
int g_usableDevices = 0;
} // namespace
namespace {
int usableDevices() {
  if (!g_deviceChecked) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { n = 0; cudaGetLastError(); }
    int ok = 0;
    for (int d = 0; d < n; ++d) {
      int major = 0;
      if (cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, d) == cudaSuccess && major == 9) ++ok;
    }
    g_usableDevices = ok;
    g_deviceChecked = true;
  }
  return g_usableDevices;
}

int requireDevice(int device) {
  if (usableDevices() <= 0) return fail(MB2_ERR_CUDA, "no usable sm_90 CUDA device: momentum_b200 has no CPU fallback");
  MB2_CUDA(cudaSetDevice(device));
  MB2_CUDA(initKernelAttributes());
  return MB2_OK;
}

int ensureTargets(mb2_solver_function* f) {
  const size_t need = size_t(f->B) * std::max(f->host.targetStride, 1);
  if (f->dTargets.n < need) {
    DeviceBuffer<float> old;
    std::swap(old.p, f->dTargets.p);
    std::swap(old.n, f->dTargets.n);
    MB2_CUDA(f->dTargets.resize(need));
    MB2_CUDA(cudaMemsetAsync(f->dTargets.p, 0, need * sizeof(float), f->stream));
    // the next writer may be mb2_set_targets_device on a caller's stream: the zero fill must have landed first
    MB2_CUDA(cudaStreamSynchronize(f->stream));
    (void)old; // targets of blocks added earlier must be re-sent after adding blocks (documented)
  }
  return MB2_OK;
}

int uploadWeights(mb2_solver_function* f) {
  if (!f->host.weightsPerInstance) {
    std::vector<float> w = f->host.weights;
    if (w.empty()) w.push_back(0.f);
    MB2_CUDA(f->dWeights.upload(w, f->stream));
  }
  return MB2_OK;
}

// mode 0: every column at its model-parameter index (getJacobian / getJtJR parity);
// mode 1: solver, only the enabled columns, ascending (dense Eigen-structured Cholesky);
// mode 2: solver, enabled columns in the Cholesky elimination order + tile schedule (schedDense: dense pattern).
// Modes 0 and 1 coincide when every parameter is enabled.
int ensurePlan(mb2_solver_function* f, int mode, bool schedDense = false, bool alignRows = false) {
  bool allEnabled = true;
  for (uint8_t e : f->host.enabled) allEnabled = allEnabled && e;
  if (allEnabled && mode == 1) mode = 0;
  if (mode != 2) alignRows = false;
  if (!f->planDirty && f->planLimitsVersion == f->ch->limitsVersion && f->planMode == mode && (mode != 2 || (f->planSchedDense == schedDense && f->planAlignRows == alignRows)))
    return MB2_OK;
  MB2_DEVICE_GUARD(f->ch->device);
  cudaStream_t s = f->stream;
  f->sched.reset();
  std::unique_ptr<DeviceSchedule> ds;
  std::string err;
  if (mode == 2) {
    ds = std::make_unique<DeviceSchedule>();
    err = planSolverPath(f->ch->host, f->host.efs, f->host.enabled, schedDense, alignRows, f->plan, ds->host, ds->gram);
  } else {
    err = buildPlan(f->ch->host, f->host.efs, f->host.enabled, mode != 0, f->plan);
  }
  if (!err.empty()) return fail(MB2_ERR_INVALID_ARGUMENT, err);
  if (ds) {
    std::vector<int32_t> sblob, gblob;
    CholSchedDev hostView;
    makeScheduleBlob(ds->host, sblob, hostView);
    MB2_CUDA(ds->blob.upload(sblob, s));
    ds->dev = rebaseSchedule(hostView, ds->blob.p);
    if (alignRows) {
      makeGramBlob(ds->gram, ds->host, gblob, ds->gOffsets);
      ds->gBlobInts = int32_t(gblob.size());
      MB2_CUDA(ds->gBlob.upload(gblob, s));
      ds->gcValid = makeGramCholTables(ds->gram, ds->host, ds->gc).empty(); // else the three-kernel path
      if (ds->gcValid && ds->gc.tab.size() <= size_t(kGramCholParamEntries)) {
        ds->gcParams = std::make_unique<GramCholParamTables>();
        ds->gcParams->L = ds->gc.L;
        std::copy(ds->gc.tab.begin(), ds->gc.tab.end(), ds->gcParams->tab);
      } else if (ds->gcValid) {
        MB2_CUDA(ds->gcTab.upload(ds->gc.tab, s));
      }
      MB2_CUDA(ds->fBlob.upload(makeFusedBlob(f->ch->host, f->plan, gblob, sblob, ds->fLayout), s));
    }
    f->sched = std::move(ds);
  }
  f->planMode = mode;
  f->planSchedDense = schedDense;
  f->planAlignRows = alignRows;
  MB2_CUDA(f->dEfs.upload(f->plan.efs, s));
  MB2_CUDA(f->dUnits.upload(f->plan.units, s));
  MB2_CUDA(f->dCells.upload(f->plan.cells, s));
  MB2_CUDA(f->dContribs.upload(f->plan.contribs, s));
  MB2_CUDA(f->dLimitData.upload(f->plan.limitData, s));
  MB2_CUDA(f->dEnabledList.upload(f->plan.enabledList, s));
  MB2_CUDA(f->dDeviceCols.upload(f->plan.deviceCols, s));
  std::vector<int32_t> ident(f->ch->host.numParams);
  for (size_t i = 0; i < ident.size(); ++i) ident[i] = int32_t(i);
  MB2_CUDA(f->dIdentity.upload(ident, s));
  f->ldJ = std::max(32, roundUp(f->plan.numRows, 32));
  const bool stripLayout = mode == 2 && alignRows; // strips + residual instead of the K-major matrix
  const size_t jElems = stripLayout ? size_t(f->B) * size_t(f->sched->gram.stride) : size_t(f->B) * (f->plan.numCols + 1) * f->ldJ;
  MB2_CUDA(f->dJ.resize(jElems));
  // cells outside the plan are never written: zero once per plan (ResizeableMatrix::resizeAndSetZero
  // happens every iteration in the reference, solver_function.cpp:96)
  MB2_CUDA(cudaMemsetAsync(f->dJ.p, 0, jElems * sizeof(float), s));
  MB2_CUDA(f->dErrors.resize(f->B));
  MB2_CUDA(f->dTheta.resize(size_t(f->B) * f->ch->host.numParams));
  int rc = ensureTargets(f);
  if (rc != MB2_OK) return rc;
  rc = uploadWeights(f);
  if (rc != MB2_OK) return rc;
  // Plan tables, schedule / Gram blobs, weights and the Jacobian zero fill were issued on the handle's stream; the solve may run on a
  // caller's stream. A plan build is a rare host-side event: wait for it here instead of threading events through every launch.
  MB2_CUDA(cudaStreamSynchronize(s));
  f->planDirty = false;
  f->planLimitsVersion = f->ch->limitsVersion;
  return MB2_OK;
}

SweepArgs sweepArgs(mb2_solver_function* f, const float* theta, const int32_t* active) {
  SweepArgs a{};
  a.T = f->tables();
  a.batch = f->B;
  a.theta = theta;
  a.ldTheta = f->ch->host.numParams;
  a.targets = f->dTargets.p;
  a.cweights = f->dWeights.p;
  a.jacobian = f->dJ.p;
  a.errors = f->dErrors.p;
  a.active = active;
  a.stateOut = nullptr;
  return a;
}

// buildError: what the block's constructor said about the C-ABI arguments ef was built from
int addBlock(mb2_solver_function* f, const std::string& buildError, const HostErrorFunction& ef, int32_t* outIndex) {
  if (!buildError.empty()) return fail(MB2_ERR_INVALID_ARGUMENT, buildError);
  const std::string err = f->host.add(ef, outIndex);
  if (!err.empty()) return fail(MB2_ERR_UNSUPPORTED, err);
  f->planDirty = true;
  return MB2_OK;
}

void bitsToEnabled(const uint64_t* bits, int n, std::vector<uint8_t>& out) {
  out.assign(n, 0);
  for (int i = 0; i < n; ++i) out[i] = (bits[i >> 6] >> (i & 63)) & 1ull ? 1 : 0;
}

void recordPhaseStart(mb2_solver* s, int phase, cudaStream_t st) {
  s->kernelLaunches++;
  if (!s->profiling) return;
  PhaseEvent e;
  cudaEventCreate(&e.start);
  cudaEventCreate(&e.stop);
  e.phase = phase;
  cudaEventRecord(e.start, st);
  s->events.push_back(e);
}
void recordPhaseStop(mb2_solver* s, cudaStream_t st) {
  if (!s->profiling) return;
  cudaEventRecord(s->events.back().stop, st);
}

__global__ void initSolveStateKernel(int batch, const SolveState s) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= batch) return;
  s.active[b] = 1;
  s.iterations[b] = 0;
  s.status[b] = 0;
  s.lastErrors[b] = DBL_MAX; // solver.cpp:83-84
  s.errors[b] = DBL_MAX;
}
__global__ void initLineSearchKernel(int batch, const int32_t* active, int32_t* searching, float* scale) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= batch) return;
  searching[b] = active[b];
  scale[b] = 1.f;
}
// NaN/Inf guard of the batched caller (pymomentum/tensor_ik/tensor_ik.cpp:168-173): revert to the initial guess
__global__ void finalizeKernel(int batch, int n, float* theta, const float* theta0, int32_t* status) {
  const int b = blockIdx.x;
  __shared__ int bad;
  if (threadIdx.x == 0) bad = 0;
  __syncthreads();
  for (int i = threadIdx.x; i < n; i += blockDim.x)
    if (!isfinite(theta[size_t(b) * n + i])) bad = 1;
  __syncthreads();
  if (bad) {
    for (int i = threadIdx.x; i < n; i += blockDim.x) theta[size_t(b) * n + i] = theta0[size_t(b) * n + i];
    if (threadIdx.x == 0) status[b] = MB2_INSTANCE_NON_FINITE;
  }
}

int runJtJ(mb2_solver_function* f, int mode, int ns, float* H, int ldH, size_t hStride, const int32_t* active, cudaStream_t st, float* g = nullptr, int ldG = 0) {
  JtJArgs a{};
  a.batch = f->B;
  a.jacobian = f->dJ.p;
  a.numCols = f->plan.numCols;
  a.ldJ = f->ldJ;
  a.kRows = roundUp(std::max(f->plan.numRows, 1), 4);
  a.ns = ns;
  a.H = H;
  a.ldH = ldH;
  a.hStride = hStride;
  a.active = active;
  a.g = g;
  a.ldG = ldG;
  if (mode == MB2_JTJ_FP32_SIMT) { MB2_CUDA(launchJtJSimt(a, st)); }
  else { MB2_CUDA(launchJtJTensor(a, mode == MB2_JTJ_TF32X3 ? 3 : 1, st)); }
  return MB2_OK;
}

} // namespace

extern "C" {

const char* mb2_last_error(void) { return g_lastError.c_str(); }
int mb2_device_count(void) { return usableDevices(); }

void mb2_default_gauss_newton_options(mb2_gauss_newton_options* o) {
  if (!o) return;
  std::memset(o, 0, sizeof(*o));
  o->min_iterations = 1;  // solver.h:21
  o->max_iterations = 2;  // solver.h:24
  o->threshold = 1.0f;    // solver.h:27
  o->verbose = 0;
  o->regularization = 0.05f; // gauss_newton_solver.h:22
  o->do_line_search = 0;
  o->use_block_jtj = 0;
  o->target_rows_per_chunk = ~0ull;
  o->subset_line_search = 0;
  o->jtj_mode = MB2_JTJ_AUTO;
  o->store_error_history = 0;
  o->cholesky_mode = MB2_CHOLESKY_AUTO;
  o->fused_mode = MB2_FUSED_AUTO;
  o->linear_solver = MB2_LINEAR_SOLVER_CHOLESKY;
  o->trust_region_radius = 1.0f; // trust_region_qr.h:23
}

int mb2_character_create(int device, int32_t J, const int32_t* parents, const float* offsets, const float* prerot, int32_t n,
                         const int32_t* outer, const int32_t* inner, const float* vals, const float* ptoffsets, mb2_character** out) {
  MB2_CHECK(out != nullptr, "null argument");
  auto c = std::make_unique<mb2_character>();
  HostCharacter& h = c->host;
  const std::string err = makeCharacter(J, parents, offsets, prerot, n, outer, inner, vals, ptoffsets, h);
  if (!err.empty()) return fail(MB2_ERR_INVALID_ARGUMENT, err);
  MB2_DEVICE_GUARD(device);
  int rc = requireDevice(device);
  if (rc != MB2_OK) return rc;
  c->device = device;
  MB2_CUDA(c->parent.upload(h.parent, nullptr));
  MB2_CUDA(c->offset.upload(h.offset, nullptr));
  MB2_CUDA(c->prerot.upload(h.prerot, nullptr));
  MB2_CUDA(c->ptOuter.upload(h.ptOuter, nullptr));
  MB2_CUDA(c->ptInner.upload(h.ptInner, nullptr));
  MB2_CUDA(c->ptVals.upload(h.ptVals, nullptr));
  MB2_CUDA(c->ptOffsets.upload(h.ptOffsets, nullptr));
  MB2_CUDA(c->levelStart.upload(h.levelStart, nullptr));
  MB2_CUDA(c->levelJoints.upload(h.levelJoints, nullptr));
  MB2_CUDA(c->childStart.upload(h.childStart, nullptr));
  MB2_CUDA(c->children.upload(h.children, nullptr));
  MB2_CUDA(c->ptColStart.upload(h.ptColStart, nullptr));
  MB2_CUDA(c->ptColRows.upload(h.ptColRows, nullptr));
  MB2_CUDA(c->ptColVals.upload(h.ptColVals, nullptr));
  MB2_CUDA(c->invStart.upload(h.invStart, nullptr));
  MB2_CUDA(c->invRows.upload(h.invRows, nullptr));
  MB2_CUDA(c->invVals.upload(h.invVals, nullptr));
  MB2_CUDA(c->invRowStart.upload(h.invRowStart, nullptr));
  MB2_CUDA(c->invParams.upload(h.invParams, nullptr));
  MB2_CUDA(c->invRowVals.upload(h.invRowVals, nullptr));
  MB2_CUDA(cudaStreamSynchronize(nullptr));
  rc = installLimitTables(c.get()); // no limits yet: empty tables and a pass-through clamp
  if (rc != MB2_OK) return rc;
  *out = c.release();
  return MB2_OK;
}

int mb2_character_set_parameter_limits(mb2_character* c, int32_t count, const mb2_parameter_limit* limits) {
  MB2_CHECK(c != nullptr, "invalid limits");
  const std::string err = setParameterLimits(c->host, count, limits);
  if (!err.empty()) return fail(MB2_ERR_INVALID_ARGUMENT, err);
  c->limitsVersion++;
  return installLimitTables(c);
}

void mb2_character_destroy(mb2_character* c) { delete c; }

int mb2_solver_function_create(const mb2_character* c, int32_t batch, mb2_solver_function** out) {
  MB2_CHECK(c != nullptr && out != nullptr, "null argument");
  MB2_CHECK(batch > 0, "batch must be positive");
  MB2_DEVICE_GUARD(c->device);
  int rc = requireDevice(c->device);
  if (rc != MB2_OK) return rc;
  auto f = std::make_unique<mb2_solver_function>();
  f->ch = c;
  f->B = batch;
  f->host.enabled.assign(c->host.numParams, 1); // all parameters enabled by default (skeleton_error_function.h:27)
  MB2_CUDA(cudaStreamCreateWithFlags(&f->stream, cudaStreamNonBlocking));
  *out = f.release();
  return MB2_OK;
}

void mb2_solver_function_destroy(mb2_solver_function* f) {
  if (!f) return;
  if (f->stream) cudaStreamDestroy(f->stream);
  delete f;
}

// ---- replicas on other devices (single-process multi-GPU: ik_sharded.cpp) ----
// The rig (skeleton, parameter transform, parameter limits) on another device; independent of the original afterwards.
int mb2_character_clone(const mb2_character* c, int device, mb2_character** out) {
  MB2_CHECK(c != nullptr && out != nullptr, "null argument");
  const HostCharacter& h = c->host;
  mb2_character* copy = nullptr;
  int rc = mb2_character_create(device, h.numJoints, h.parent.data(), h.offset.data(), h.prerot.data(), h.numParams, h.ptOuter.data(), h.ptInner.data(), h.ptVals.data(),
                                h.ptOffsets.data(), &copy);
  if (rc != MB2_OK) return rc;
  copy->host.limits = h.limits;
  copy->limitsVersion = 1;
  rc = installLimitTables(copy);
  if (rc != MB2_OK) { mb2_character_destroy(copy); return rc; }
  const HostSkinning& s = c->skin;
  if (s.numVertices > 0) { // back to [V][8] slots: the active ones, then zero weights
    std::vector<int32_t> index(size_t(s.numVertices) * kSkinMaxInfluences, 0);
    std::vector<float> weight(index.size(), 0.f);
    for (int v = 0; v < s.numVertices; ++v)
      for (int k = s.vertStart[v]; k < s.vertStart[v + 1]; ++k) {
        index[size_t(v) * kSkinMaxInfluences + (k - s.vertStart[v])] = s.vertJoint[k];
        weight[size_t(v) * kSkinMaxInfluences + (k - s.vertStart[v])] = s.vertWeight[k];
      }
    rc = mb2_character_set_skinning(copy, s.numVertices, s.restVertices.data(), index.data(), weight.data(), s.inverseBindPose.data());
    if (rc != MB2_OK) { mb2_character_destroy(copy); return rc; }
  }
  const HostBlendShape& bs = c->blend;
  if (bs.numShapes > 0) {
    rc = mb2_character_set_blend_shape(copy, bs.numShapes, bs.numVertices, bs.baseShape.data(), bs.shapeVectors.data());
    if (rc != MB2_OK) { mb2_character_destroy(copy); return rc; }
  }
  const HostMeshFaces& mf = c->faces;
  if (mf.numVertices > 0) {
    rc = mb2_character_set_mesh_faces(copy, mf.numVertices, mf.numFaces, mf.faces.data());
    if (rc != MB2_OK) { mb2_character_destroy(copy); return rc; }
  }
  if (c->tree.numNodes > 0) {
    rc = installMeshTree(copy, HostMeshTree(c->tree));
    if (rc != MB2_OK) { mb2_character_destroy(copy); return rc; }
  }
  if (c->collisionDev) {
    rc = installCollision(copy, HostCollision(c->collision));
    if (rc != MB2_OK) { mb2_character_destroy(copy); return rc; }
  }
  *out = copy;
  return MB2_OK;
}

int mb2_character_set_skinning(mb2_character* c, int32_t num_vertices, const float* rest_vertices, const int32_t* skin_index, const float* skin_weight,
                               const float* inverse_bind_pose) {
  MB2_CHECK(c != nullptr, "null character");
  HostSkinning s;
  const std::string err = makeSkinning(c->host, num_vertices, rest_vertices, skin_index, skin_weight, inverse_bind_pose, s);
  if (!err.empty()) return fail(MB2_ERR_INVALID_ARGUMENT, err);
  return installTables(c->device, c->skinDev, c->skin, std::move(s), [](SkinBuffers& d, const HostSkinning& s) -> int {
    MB2_CUDA(d.rest.upload(s.restVertices, nullptr));
    MB2_CUDA(d.vertStart.upload(s.vertStart, nullptr));
    MB2_CUDA(d.vertJoint.upload(s.vertJoint, nullptr));
    MB2_CUDA(d.vertWeight.upload(s.vertWeight, nullptr));
    MB2_CUDA(d.ibp.upload(s.inverseBindPose, nullptr));
    MB2_CUDA(d.infVertex.upload(s.infVertex, nullptr));
    MB2_CUDA(d.infWeight.upload(s.infWeight, nullptr));
    MB2_CUDA(d.segStart.upload(s.segStart, nullptr));
    MB2_CUDA(d.segJoint.upload(s.segJoint, nullptr));
    MB2_CUDA(d.jointSegStart.upload(s.jointSegStart, nullptr));
    return MB2_OK;
  });
}

int32_t mb2_character_num_vertices(const mb2_character* c) { return c ? c->skin.numVertices : 0; }

int mb2_character_set_blend_shape(mb2_character* c, int32_t num_shapes, int32_t num_vertices, const float* base_shape, const float* shape_vectors) {
  MB2_CHECK(c != nullptr, "null character");
  HostBlendShape b;
  const std::string err = makeBlendShape(num_shapes, num_vertices, base_shape, shape_vectors, b);
  if (!err.empty()) return fail(MB2_ERR_INVALID_ARGUMENT, err);
  return installTables(c->device, c->blendDev, c->blend, std::move(b), [](BlendShapeBuffers& d, const HostBlendShape& b) -> int {
    MB2_CUDA(d.baseShape.upload(b.baseShape, nullptr));
    MB2_CUDA(d.shapeVectors.upload(b.shapeVectors, nullptr));
    return MB2_OK;
  });
}

int32_t mb2_character_num_blend_shapes(const mb2_character* c) { return c ? c->blend.numShapes : 0; }

int mb2_character_set_mesh_faces(mb2_character* c, int32_t num_vertices, int32_t num_faces, const int32_t* faces) {
  MB2_CHECK(c != nullptr, "null character");
  HostMeshFaces m;
  if (!(num_faces == 0 && faces == nullptr)) { // that pair removes the faces
    const std::string err = makeMeshFaces(num_vertices, num_faces, faces, m);
    if (!err.empty()) return fail(MB2_ERR_INVALID_ARGUMENT, err);
  }
  const bool present = m.numVertices > 0;
  const int rc = installTables(c->device, c->facesDev, c->faces, std::move(m), [](MeshFaceBuffers& d, const HostMeshFaces& m) -> int {
    MB2_CUDA(d.faces.upload(m.faces, nullptr));
    MB2_CUDA(d.vertStart.upload(m.vertStart, nullptr));
    MB2_CUDA(d.vertCorner.upload(m.vertCorner, nullptr));
    return MB2_OK;
  }, present);
  if (rc != MB2_OK) return rc;
  c->treeDev.reset(); // built over the faces it replaced; the swap above synchronised the device
  c->tree = HostMeshTree{};
  return MB2_OK;
}

int32_t mb2_character_num_faces(const mb2_character* c) { return c ? c->faces.numFaces : 0; }

int mb2_character_set_mesh_tree(mb2_character* c, int32_t num_vertices, const float* reference_positions) {
  MB2_CHECK(c != nullptr, "null character");
  HostMeshTree t;
  if (!(num_vertices == 0 && reference_positions == nullptr)) { // that pair removes the tree
    const std::string err = makeMeshTree(c->faces, num_vertices, reference_positions, t);
    if (!err.empty()) return fail(MB2_ERR_INVALID_ARGUMENT, err);
  }
  return installMeshTree(c, std::move(t));
}
// The DEFINITION of a solver function (error-function blocks with their shared constraint data and weights, block weights, enabled
// parameters) for `batch` instances of character `c` (normally a clone of f's character on another device). Per-instance data
// (targets, per-instance weights / offsets) is not copied: it belongs to the instances the new function will hold.
int mb2_solver_function_clone(const mb2_solver_function* f, const mb2_character* c, int32_t batch, mb2_solver_function** out) {
  MB2_CHECK(f != nullptr && c != nullptr && out != nullptr, "null argument");
  MB2_CHECK(c->host.numJoints == f->ch->host.numJoints && c->host.numParams == f->ch->host.numParams, "clone target character has a different shape");
  MB2_CHECK(!f->host.weightsPerInstance, "a function with per-instance constraint weights cannot be cloned (set them on the clone)");
  mb2_solver_function* g = nullptr;
  int rc = mb2_solver_function_create(c, batch, &g);
  if (rc != MB2_OK) return rc;
  g->host = f->host;
  g->planDirty = true;
  *out = g;
  return MB2_OK;
}
int mb2_character_device(const mb2_character* c) { return c ? c->device : -1; }
const mb2_character* mb2_solver_function_character(const mb2_solver_function* f) { return f ? f->ch : nullptr; }
int32_t mb2_solver_function_num_error_functions(const mb2_solver_function* f) { return f ? int32_t(f->host.efs.size()) : 0; }
int32_t mb2_solver_function_target_size(const mb2_solver_function* f, int32_t index) {
  return (f && index >= 0 && index < int32_t(f->host.efs.size())) ? f->host.efs[index].targetSize : -1;
}

int32_t mb2_solver_function_num_parameters(const mb2_solver_function* f) { return f ? f->ch->host.numParams : 0; }
int32_t mb2_solver_function_batch(const mb2_solver_function* f) { return f ? f->B : 0; }
int32_t mb2_solver_function_actual_parameters(const mb2_solver_function* f) { return f ? f->host.actualParameters() : 0; }
int32_t mb2_solver_function_jacobian_rows(const mb2_solver_function* f) { return f ? f->host.jacobianRows(f->ch->host) : 0; }
int32_t mb2_solver_function_jacobian_stride(const mb2_solver_function* f) { return f ? f->host.jacobianStride(f->ch->host) : 0; }

int mb2_add_position_error_function(mb2_solver_function* f, float weight, float alpha, float c, int32_t nc, const int32_t* parents,
                                    const float* offsets, const float* weights, int32_t* outIndex) {
  MB2_CHECK(f != nullptr, "null solver function");
  HostErrorFunction ef;
  return addBlock(f, positionErrorFunction(f->ch->host, weight, alpha, c, nc, parents, offsets, weights, ef), ef, outIndex);
}

int mb2_add_position_error_function_instanced(mb2_solver_function* f, float weight, float alpha, float c, int32_t nc, const int32_t* parents, const float* weights,
                                              int32_t* outIndex) {
  MB2_CHECK(f != nullptr, "null solver function");
  HostErrorFunction ef;
  return addBlock(f, instancedPositionErrorFunction(f->ch->host, weight, alpha, c, nc, parents, weights, ef), ef, outIndex);
}

int mb2_add_plane_error_function(mb2_solver_function* f, float weight, float alpha, float c, int32_t above, int32_t nc, const int32_t* parents,
                                 const float* offsets, const float* weights, int32_t* outIndex) {
  MB2_CHECK(f != nullptr, "null solver function");
  HostErrorFunction ef;
  return addBlock(f, planeErrorFunction(f->ch->host, weight, alpha, c, above, nc, parents, offsets, weights, ef), ef, outIndex);
}

int mb2_add_model_parameters_error_function(mb2_solver_function* f, float weight, const float* targetWeights, int32_t* outIndex) {
  MB2_CHECK(f != nullptr, "null solver function");
  HostErrorFunction ef;
  return addBlock(f, modelParametersErrorFunction(f->ch->host, weight, targetWeights, ef), ef, outIndex);
}

int mb2_add_orientation_error_function(mb2_solver_function* f, float weight, float alpha, float c, int32_t rotDiff, int32_t nc,
                                       const int32_t* parents, const float* offsets, const float* weights, int32_t* outIndex) {
  MB2_CHECK(f != nullptr, "null solver function");
  HostErrorFunction ef;
  return addBlock(f, orientationErrorFunction(f->ch->host, weight, alpha, c, rotDiff, nc, parents, offsets, weights, ef), ef, outIndex);
}

int mb2_add_orientation_error_function_instanced(mb2_solver_function* f, float weight, float alpha, float c, int32_t rotDiff, int32_t nc,
                                                 const int32_t* parents, const float* weights, int32_t* outIndex) {
  MB2_CHECK(f != nullptr, "null solver function");
  HostErrorFunction ef;
  return addBlock(f, instancedOrientationErrorFunction(f->ch->host, weight, alpha, c, rotDiff, nc, parents, weights, ef), ef, outIndex);
}

int mb2_add_state_error_function(mb2_solver_function* f, float weight, int32_t rotationErrorType, float posWgt, float rotWgt,
                                 const float* posW, const float* rotW, int32_t* outIndex) {
  MB2_CHECK(f != nullptr, "null solver function");
  HostErrorFunction ef;
  return addBlock(f, stateErrorFunction(f->ch->host, weight, rotationErrorType, posWgt, rotWgt, posW, rotW, ef), ef, outIndex);
}

int mb2_add_limit_error_function(mb2_solver_function* f, float weight, float alpha, float c, int32_t* outIndex) {
  MB2_CHECK(f != nullptr, "null solver function");
  HostErrorFunction ef;
  return addBlock(f, limitErrorFunction(weight, alpha, c, ef), ef, outIndex);
}

int mb2_set_error_function_weight(mb2_solver_function* f, int32_t index, float weight) {
  MB2_CHECK(f != nullptr && index >= 0 && index < int(f->host.efs.size()), "error function index out of range");
  f->host.efs[index].weight = weight;
  f->planDirty = true;
  return MB2_OK;
}

static int setTargetsImpl(mb2_solver_function* f, int32_t index, const float* targets, bool deviceSrc, cudaStream_t st) {
  MB2_CHECK(f != nullptr && index >= 0 && index < int(f->host.efs.size()) && targets, "invalid targets");
  const HostErrorFunction& ef = f->host.efs[index];
  if (ef.targetSize == 0 && ef.kind != 4) return MB2_OK; // a block without constraints: nothing to send (setConstraints({}) in the reference)
  MB2_CHECK(ef.targetSize > 0, "this error function has no per-instance targets");
  MB2_DEVICE_GUARD(f->ch->device);
  int rc = ensureTargets(f);
  if (rc != MB2_OK) return rc;
  float* dst = f->dTargets.p + ef.targetOff;
  const float* packed = targets;
  if (!deviceSrc) { // one contiguous transfer, then a kernel spreads it into the per-instance records
    MB2_CUDA(f->dTargetStage.resize(size_t(f->B) * ef.targetSize));
    MB2_CUDA(cudaMemcpyAsync(f->dTargetStage.p, targets, size_t(f->B) * ef.targetSize * sizeof(float), cudaMemcpyHostToDevice, st));
    packed = f->dTargetStage.p;
  }
  MB2_CUDA(launchScatterTargets(packed, dst, ef.targetSize, f->host.targetStride, f->B, st));
  if (ef.kind == 1 || ef.kind == 2) // targets (and the offsets of an instanced block, interleaved with them) are unit quaternions
    MB2_CUDA(launchNormalizeQuats(dst, 0, f->host.targetStride, (ef.instanceOffsets ? 2 : 1) * ef.numConstraints(), f->B, st));
  return MB2_OK;
}
int mb2_set_targets(mb2_solver_function* f, int32_t index, const float* targets) {
  if (!f) return fail(MB2_ERR_INVALID_ARGUMENT, "null solver function");
  int rc = setTargetsImpl(f, index, targets, false, f->stream);
  if (rc != MB2_OK) return rc;
  MB2_CUDA(cudaStreamSynchronize(f->stream)); // host buffer may be reused by the caller
  return MB2_OK;
}
int mb2_set_targets_device(mb2_solver_function* f, int32_t index, const float* targets, void* stream) {
  if (!f) return fail(MB2_ERR_INVALID_ARGUMENT, "null solver function");
  return setTargetsImpl(f, index, targets, true, stream ? (cudaStream_t)stream : f->stream);
}

int mb2_set_constraint_weights(mb2_solver_function* f, int32_t index, const float* weights, int32_t perInstance) {
  MB2_CHECK(f != nullptr && index >= 0 && index < int(f->host.efs.size()) && weights, "invalid constraint weights");
  HostErrorFunction& ef = f->host.efs[index];
  MB2_CHECK(ef.kind <= 2 || ef.kind == 5, "constraint weights apply to Position/Orientation/Plane error functions");
  MB2_DEVICE_GUARD(f->ch->device);
  const int nc = ef.numConstraints();
  if (!perInstance) {
    MB2_CHECK(!f->host.weightsPerInstance, "solver function already uses per-instance constraint weights");
    ef.weights.assign(weights, weights + nc);
    std::copy(weights, weights + nc, f->host.weights.begin() + ef.weightOff);
    return uploadWeights(f);
  }
  if (!f->host.weightsPerInstance) { // expand the shared array to [B][numWeights]
    std::vector<float> all(size_t(f->B) * f->host.numWeights);
    for (int b = 0; b < f->B; ++b) std::copy(f->host.weights.begin(), f->host.weights.end(), all.begin() + size_t(b) * f->host.numWeights);
    f->dWeights.release();
    MB2_CUDA(f->dWeights.upload(all, f->stream));
    f->host.weightsPerInstance = true;
  }
  MB2_CUDA(cudaMemcpy2DAsync(f->dWeights.p + ef.weightOff, size_t(f->host.numWeights) * sizeof(float), weights, size_t(nc) * sizeof(float),
                             size_t(nc) * sizeof(float), f->B, cudaMemcpyHostToDevice, f->stream));
  MB2_CUDA(cudaStreamSynchronize(f->stream));
  return MB2_OK;
}

// per-instance weights of one block from DEVICE memory [B][nc] (the torch binding's path: no host round trip)
int mb2_set_constraint_weights_device(mb2_solver_function* f, int32_t index, const float* weights_device, void* stream) {
  MB2_CHECK(f != nullptr && index >= 0 && index < int(f->host.efs.size()) && weights_device, "invalid constraint weights");
  HostErrorFunction& ef = f->host.efs[index];
  MB2_CHECK(ef.kind <= 2 || ef.kind == 5, "constraint weights apply to Position/Orientation/Plane error functions");
  MB2_DEVICE_GUARD(f->ch->device);
  const int nc = ef.numConstraints();
  if (!f->host.weightsPerInstance) { // expand the shared array to [B][numWeights]
    std::vector<float> all(size_t(f->B) * f->host.numWeights);
    for (int b = 0; b < f->B; ++b) std::copy(f->host.weights.begin(), f->host.weights.end(), all.begin() + size_t(b) * f->host.numWeights);
    f->dWeights.release();
    MB2_CUDA(f->dWeights.upload(all, f->stream));
    MB2_CUDA(cudaStreamSynchronize(f->stream));
    f->host.weightsPerInstance = true;
    f->planDirty = true; // tables() carries the per-instance flag
  }
  cudaStream_t st = stream ? (cudaStream_t)stream : f->stream;
  if (nc > 0)
    MB2_CUDA(cudaMemcpy2DAsync(f->dWeights.p + ef.weightOff, size_t(f->host.numWeights) * sizeof(float), weights_device, size_t(nc) * sizeof(float), size_t(nc) * sizeof(float), f->B,
                               cudaMemcpyDeviceToDevice, st));
  return MB2_OK;
}

int mb2_solver_function_set_enabled_parameters(mb2_solver_function* f, const uint64_t* bits) {
  MB2_CHECK(f != nullptr && bits != nullptr, "null argument");
  bitsToEnabled(bits, f->ch->host.numParams, f->host.enabled);
  f->planDirty = true;
  return MB2_OK;
}

int mb2_solver_function_get_error(mb2_solver_function* f, const float* params, double* errors) {
  MB2_CHECK(f != nullptr && params && errors, "null argument");
  MB2_DEVICE_GUARD(f->ch->device);
  int rc = ensurePlan(f, f->planMode, f->planSchedDense, f->planAlignRows);
  if (rc != MB2_OK) return rc;
  const size_t n = f->ch->host.numParams;
  MB2_CUDA(cudaMemcpyAsync(f->dTheta.p, params, size_t(f->B) * n * sizeof(float), cudaMemcpyHostToDevice, f->stream));
  MB2_CUDA(launchSweep(sweepArgs(f, f->dTheta.p, nullptr), false, f->stream, &f->lastSweep[0]));
  MB2_CUDA(cudaMemcpyAsync(errors, f->dErrors.p, size_t(f->B) * sizeof(double), cudaMemcpyDeviceToHost, f->stream));
  MB2_CUDA(cudaStreamSynchronize(f->stream));
  return MB2_OK;
}

int mb2_solver_function_get_jacobian(mb2_solver_function* f, const float* params, float* jac, float* residual, double* errors, int32_t* actualRows) {
  MB2_CHECK(f != nullptr && params, "null argument");
  MB2_DEVICE_GUARD(f->ch->device);
  int rc = ensurePlan(f, 0);
  if (rc != MB2_OK) return rc;
  const size_t n = f->ch->host.numParams;
  const int rows = mb2_solver_function_jacobian_rows(f);
  MB2_CUDA(cudaMemcpyAsync(f->dTheta.p, params, size_t(f->B) * n * sizeof(float), cudaMemcpyHostToDevice, f->stream));
  MB2_CUDA(launchSweep(sweepArgs(f, f->dTheta.p, nullptr), true, f->stream, &f->lastSweep[1]));
  for (int b = 0; b < f->B && rows > 0; ++b) { // parity/debug entry point: one strided copy per instance
    const float* Jb = f->dJ.p + size_t(b) * (n + 1) * f->ldJ;
    if (jac)
      MB2_CUDA(cudaMemcpy2DAsync(jac + size_t(b) * n * rows, size_t(rows) * sizeof(float), Jb, size_t(f->ldJ) * sizeof(float), size_t(rows) * sizeof(float), n,
                                 cudaMemcpyDeviceToHost, f->stream));
    if (residual)
      MB2_CUDA(cudaMemcpyAsync(residual + size_t(b) * rows, Jb + n * f->ldJ, size_t(rows) * sizeof(float), cudaMemcpyDeviceToHost, f->stream));
  }
  if (errors) MB2_CUDA(cudaMemcpyAsync(errors, f->dErrors.p, size_t(f->B) * sizeof(double), cudaMemcpyDeviceToHost, f->stream));
  MB2_CUDA(cudaStreamSynchronize(f->stream));
  if (actualRows) *actualRows = rows; // solver_function.cpp:50 actualRows = totalRows (padded)
  return MB2_OK;
}

// getJacobian with parameters and outputs resident on the device (backward pass of the torch binding): jacobian [B][n][ldJ] in the
// device layout (column c of instance b at (b * (n + 1) + c) * ldJ, ldJ = mb2_solver_function_jacobian_stride), residual = column n.
int mb2_solver_function_get_jacobian_device(mb2_solver_function* f, const float* params_device, const float** jacobian_device, int32_t* ld, void* stream) {
  MB2_CHECK(f != nullptr && params_device && jacobian_device, "null argument");
  MB2_DEVICE_GUARD(f->ch->device);
  int rc = ensurePlan(f, 0);
  if (rc != MB2_OK) return rc;
  cudaStream_t st = stream ? (cudaStream_t)stream : f->stream;
  MB2_CUDA(launchSweep(sweepArgs(f, params_device, nullptr), true, st, &f->lastSweep[1]));
  *jacobian_device = f->dJ.p;
  if (ld) *ld = f->ldJ;
  return MB2_OK;
}

int mb2_solver_function_get_jtjr(mb2_solver_function* f, const float* params, int32_t jtjMode, float* jtj, float* jtr, double* errors) {
  MB2_CHECK(f != nullptr && params, "null argument");
  MB2_DEVICE_GUARD(f->ch->device);
  int rc = ensurePlan(f, 0);
  if (rc != MB2_OK) return rc;
  const size_t n = f->ch->host.numParams;
  const int ap = f->plan.actualParameters;
  MB2_CHECK(ap > 0, "no enabled parameters");
  const int mode = resolveJtjMode(jtjMode, jtjTensorSupported(ap, f->plan.numCols, f->ldJ));
  if (mode < 0) return fail(MB2_ERR_UNSUPPORTED, "tensor-core JtJ does not support this shape");
  const int ldH = roundUp(ap + 1, 16);
  const size_t hElems = size_t(f->B) * (ap + 1) * ldH;
  MB2_CUDA(f->dH.resize(hElems));
  MB2_CUDA(cudaMemcpyAsync(f->dTheta.p, params, size_t(f->B) * n * sizeof(float), cudaMemcpyHostToDevice, f->stream));
  MB2_CUDA(launchSweep(sweepArgs(f, f->dTheta.p, nullptr), true, f->stream, &f->lastSweep[1]));
  MB2_CUDA(cudaMemsetAsync(f->dH.p, 0, hElems * sizeof(float), f->stream));
  rc = runJtJ(f, mode, ap, f->dH.p, ldH, size_t(ap + 1) * ldH, nullptr, f->stream);
  if (rc != MB2_OK) return rc;
  std::vector<float> h(hElems);
  MB2_CUDA(cudaMemcpyAsync(h.data(), f->dH.p, hElems * sizeof(float), cudaMemcpyDeviceToHost, f->stream));
  if (errors) MB2_CUDA(cudaMemcpyAsync(errors, f->dErrors.p, size_t(f->B) * sizeof(double), cudaMemcpyDeviceToHost, f->stream));
  MB2_CUDA(cudaStreamSynchronize(f->stream));
  for (int b = 0; b < f->B; ++b) { // device layout is the full symmetric [JtJ, Jtr]; the ABI returns the lower triangle + Jtr
    const float* Hb = h.data() + size_t(b) * (ap + 1) * ldH;
    for (int j = 0; j < ap; ++j) {
      if (jtj) for (int i = j; i < ap; ++i) jtj[(size_t(b) * ap + i) * ap + j] = Hb[size_t(j) * ldH + i];
      if (jtr) jtr[size_t(b) * ap + j] = Hb[size_t(j) * ldH + ap];
    }
  }
  return MB2_OK;
}

int mb2_solver_function_get_skeleton_state(mb2_solver_function* f, const float* params, float* state) {
  MB2_CHECK(f != nullptr && params && state, "null argument");
  MB2_DEVICE_GUARD(f->ch->device);
  int rc = ensurePlan(f, f->planMode, f->planSchedDense, f->planAlignRows);
  if (rc != MB2_OK) return rc;
  const size_t n = f->ch->host.numParams;
  const size_t sz = size_t(f->B) * f->ch->host.numJoints * 8;
  MB2_CUDA(f->dState.resize(sz));
  MB2_CUDA(cudaMemcpyAsync(f->dTheta.p, params, size_t(f->B) * n * sizeof(float), cudaMemcpyHostToDevice, f->stream));
  SweepArgs a = sweepArgs(f, f->dTheta.p, nullptr);
  a.stateOut = f->dState.p;
  MB2_CUDA(launchSweep(a, false, f->stream, &f->lastSweep[0]));
  MB2_CUDA(cudaMemcpyAsync(state, f->dState.p, sz * sizeof(float), cudaMemcpyDeviceToHost, f->stream));
  MB2_CUDA(cudaStreamSynchronize(f->stream));
  return MB2_OK;
}

namespace {
bool isDeviceMemoryOn(const void* p, int device) {
  cudaPointerAttributes attr{};
  if (cudaPointerGetAttributes(&attr, p) != cudaSuccess) { cudaGetLastError(); return false; }
  return attr.type == cudaMemoryTypeDevice && attr.device == device;
}

// every `required` array, and every non-null `optional` one, is device memory on `device`
bool onDevice(int device, std::initializer_list<const void*> required, std::initializer_list<const void*> optional = {}) {
  for (const void* p : required)
    if (!isDeviceMemoryOn(p, device)) return false;
  for (const void* p : optional)
    if (p != nullptr && !isDeviceMemoryOn(p, device)) return false;
  return true;
}

// both directions of mb2_character_skeleton_state*_device (gradState is read by the backward only)
int skeletonStateDevice(const mb2_character* c, int32_t batch, const float* theta, const float* gradState, float* out, void* stream, bool backward,
                        bool joint = false) {
  MB2_CHECK(c != nullptr, "null character");
  MB2_CHECK(batch >= 0, "batch must not be negative");
  if (batch == 0) return MB2_OK;
  MB2_CHECK(theta != nullptr && out != nullptr && (!backward || gradState != nullptr), "null argument");
  MB2_DEVICE_GUARD(c->device);
  MB2_CHECK(onDevice(c->device, {theta, out}, {gradState}), "skeleton state: every array must be device memory on the character's device");
  NvtxRange range(backward ? "skeletonStateBackward" : "skeletonState");
  SkeletonStateArgs a{};
  a.T = c->tables();
  a.S = c->skeletonTables();
  a.numChildren = int(c->host.children.size());
  a.batch = batch;
  a.theta = theta;
  a.gradState = gradState;
  a.out = out;
  a.fromJointParameters = joint;
  MB2_CUDA(launchSkeletonState(a, backward, (cudaStream_t)stream));
  return MB2_OK;
}

// both directions of the flat joint-parameter operations (launchJointOp); `in` is optional only for the backward of the two linear
// ParameterTransform ops, which do not read it
int jointOpDevice(const mb2_character* c, int32_t batch, JointOp op, const char* name, const float* in, const float* grad, float* out, void* stream,
                  bool backward) {
  MB2_CHECK(c != nullptr, "null character");
  MB2_CHECK(batch >= 0, "batch must not be negative");
  if (batch == 0) return MB2_OK;
  const bool needIn = !(backward && (op == kJointOpParameterTransform || op == kJointOpInverseParameterTransform));
  MB2_CHECK((in != nullptr || !needIn) && out != nullptr && (!backward || grad != nullptr), "null argument");
  MB2_CHECK(op != kJointOpClampParameters || c->limits.rejected.empty(), c->limits.rejected);
  MB2_DEVICE_GUARD(c->device);
  MB2_CHECK(onDevice(c->device, {out}, {in, grad}), std::string(name) + ": every array must be device memory on the character's device");
  NvtxRange range(name);
  JointOpArgs a{};
  a.T = c->tables();
  a.S = c->skeletonTables();
  a.batch = batch;
  a.in = in;
  a.grad = grad;
  a.out = out;
  MB2_CUDA(launchJointOp(a, op, backward, (cudaStream_t)stream));
  return MB2_OK;
}
} // namespace

int mb2_character_skeleton_state_device(const mb2_character* c, int32_t batch, const float* model_parameters_device, float* skeleton_state_device,
                                        void* cuda_stream) {
  return skeletonStateDevice(c, batch, model_parameters_device, nullptr, skeleton_state_device, cuda_stream, false);
}
int mb2_character_skeleton_state_backward_device(const mb2_character* c, int32_t batch, const float* model_parameters_device,
                                                 const float* grad_skeleton_state_device, float* grad_model_parameters_device, void* cuda_stream) {
  return skeletonStateDevice(c, batch, model_parameters_device, grad_skeleton_state_device, grad_model_parameters_device, cuda_stream, true);
}

int mb2_character_apply_parameter_transform_device(const mb2_character* c, int32_t batch, const float* model_parameters_device,
                                                   float* joint_parameters_device, void* cuda_stream) {
  return jointOpDevice(c, batch, kJointOpParameterTransform, "applyParameterTransform", model_parameters_device, nullptr, joint_parameters_device, cuda_stream, false);
}
int mb2_character_apply_parameter_transform_backward_device(const mb2_character* c, int32_t batch, const float* grad_joint_parameters_device,
                                                            float* grad_model_parameters_device, void* cuda_stream) {
  return jointOpDevice(c, batch, kJointOpParameterTransform, "applyParameterTransformBackward", nullptr, grad_joint_parameters_device, grad_model_parameters_device,
                       cuda_stream, true);
}
int mb2_character_apply_inverse_parameter_transform_device(const mb2_character* c, int32_t batch, const float* joint_parameters_device,
                                                           float* model_parameters_device, void* cuda_stream) {
  return jointOpDevice(c, batch, kJointOpInverseParameterTransform, "applyInverseParameterTransform", joint_parameters_device, nullptr,
                       model_parameters_device, cuda_stream, false);
}
int mb2_character_apply_inverse_parameter_transform_backward_device(const mb2_character* c, int32_t batch, const float* grad_model_parameters_device,
                                                                    float* grad_joint_parameters_device, void* cuda_stream) {
  return jointOpDevice(c, batch, kJointOpInverseParameterTransform, "applyInverseParameterTransformBackward", nullptr, grad_model_parameters_device,
                       grad_joint_parameters_device, cuda_stream, true);
}
int mb2_character_apply_model_parameter_limits_device(const mb2_character* c, int32_t batch, const float* model_parameters_device,
                                                      float* clamped_model_parameters_device, void* cuda_stream) {
  return jointOpDevice(c, batch, kJointOpClampParameters, "applyModelParameterLimits", model_parameters_device, nullptr, clamped_model_parameters_device,
                       cuda_stream, false);
}
int mb2_character_apply_model_parameter_limits_backward_device(const mb2_character* c, int32_t batch, const float* model_parameters_device,
                                                               const float* grad_clamped_device, float* grad_model_parameters_device, void* cuda_stream) {
  return jointOpDevice(c, batch, kJointOpClampParameters, "applyModelParameterLimitsBackward", model_parameters_device, grad_clamped_device,
                       grad_model_parameters_device, cuda_stream, true);
}

int mb2_character_num_limit_residuals(const mb2_character* c, int32_t* out) {
  MB2_CHECK(c != nullptr && out != nullptr, "null argument");
  MB2_CHECK(c->limits.rejected.empty(), c->limits.rejected);
  *out = c->limits.numRows;
  return MB2_OK;
}

namespace {
// both directions of mb2_character_parameter_limits_residual*_device: residual is the forward's output, gradResidual the backward's input
int parameterLimitsDevice(const mb2_character* c, int32_t batch, const float* theta, float* residual, const float* gradResidual, float* gradTheta,
                          void* stream, bool backward) {
  MB2_CHECK(c != nullptr, "null character");
  MB2_CHECK(batch >= 0, "batch must not be negative");
  MB2_CHECK(c->limits.rejected.empty(), c->limits.rejected);
  if (batch == 0) return MB2_OK;
  const bool rows = c->limits.numRows > 0;
  MB2_CHECK(theta != nullptr && (backward ? gradTheta != nullptr && (gradResidual != nullptr || !rows) : residual != nullptr || !rows), "null argument");
  MB2_DEVICE_GUARD(c->device);
  MB2_CHECK(onDevice(c->device, {theta}, {residual, gradResidual, gradTheta}), "parameter limits: every array must be device memory on the character's device");
  NvtxRange range(backward ? "parameterLimitsResidualBackward" : "parameterLimitsResidual");
  ParameterLimitArgs a{};
  a.T = c->tables();
  a.S = c->skeletonTables();
  a.L = c->limitTables();
  a.numChildren = int(c->host.children.size());
  a.batch = batch;
  a.theta = theta;
  a.residual = residual;
  a.gradResidual = gradResidual;
  a.gradTheta = gradTheta;
  MB2_CUDA(launchParameterLimits(a, backward, (cudaStream_t)stream));
  return MB2_OK;
}
} // namespace

int mb2_character_parameter_limits_residual_device(const mb2_character* c, int32_t batch, const float* model_parameters_device, float* residual_device,
                                                   void* cuda_stream) {
  return parameterLimitsDevice(c, batch, model_parameters_device, residual_device, nullptr, nullptr, cuda_stream, false);
}
int mb2_character_parameter_limits_residual_backward_device(const mb2_character* c, int32_t batch, const float* model_parameters_device,
                                                            const float* grad_residual_device, float* grad_model_parameters_device, void* cuda_stream) {
  return parameterLimitsDevice(c, batch, model_parameters_device, nullptr, grad_residual_device, grad_model_parameters_device, cuda_stream, true);
}

int mb2_character_set_collision_geometry(mb2_character* c, int32_t count, const mb2_tapered_capsule* capsules) {
  MB2_CHECK(c != nullptr, "null character");
  HostCollision h;
  const std::string err = makeCollision(c->host, count, capsules, h);
  if (!err.empty()) return fail(MB2_ERR_INVALID_ARGUMENT, err);
  return installCollision(c, std::move(h));
}

int mb2_character_num_collision_pairs(const mb2_character* c, int32_t* out) {
  MB2_CHECK(c != nullptr && out != nullptr, "null argument");
  MB2_CHECK(c->collisionDev != nullptr, "collision: the character has no collision geometry");
  *out = c->collision.numPairs();
  return MB2_OK;
}

int mb2_character_get_collision_pairs(const mb2_character* c, int32_t* pairs) {
  MB2_CHECK(c != nullptr, "null character");
  MB2_CHECK(c->collisionDev != nullptr, "collision: the character has no collision geometry");
  MB2_CHECK(pairs != nullptr || c->collision.pairs.empty(), "null argument");
  std::copy(c->collision.pairs.begin(), c->collision.pairs.end(), pairs);
  return MB2_OK;
}

namespace {
// both directions of mb2_character_collision_residual*_device: residual is the forward's output, gradResidual the backward's input
int collisionDevice(const mb2_character* c, int32_t batch, const float* state, float* residual, const float* gradResidual, float* gradState,
                    void* stream, bool backward) {
  MB2_CHECK(c != nullptr, "null character");
  MB2_CHECK(batch >= 0, "batch must not be negative");
  MB2_CHECK(c->collisionDev != nullptr, "collision: the character has no collision geometry");
  if (batch == 0) return MB2_OK;
  const bool rows = c->collision.numPairs() > 0;
  MB2_CHECK(state != nullptr && (backward ? gradState != nullptr && (gradResidual != nullptr || !rows) : residual != nullptr || !rows), "null argument");
  MB2_DEVICE_GUARD(c->device);
  MB2_CHECK(onDevice(c->device, {state}, {residual, gradResidual, gradState}), "collision: every array must be device memory on the character's device");
  NvtxRange range(backward ? "collisionResidualBackward" : "collisionResidual");
  CollisionArgs a{};
  a.T = c->tables();
  a.L = c->collisionTables();
  a.batch = batch;
  a.state = state;
  a.residual = residual;
  a.gradResidual = gradResidual;
  a.gradState = gradState;
  MB2_CUDA(launchCollision(a, backward, (cudaStream_t)stream));
  return MB2_OK;
}
} // namespace

int mb2_character_collision_residual_device(const mb2_character* c, int32_t batch, const float* skel_state_device, float* residual_device,
                                            void* cuda_stream) {
  return collisionDevice(c, batch, skel_state_device, residual_device, nullptr, nullptr, cuda_stream, false);
}
int mb2_character_collision_residual_backward_device(const mb2_character* c, int32_t batch, const float* skel_state_device,
                                                     const float* grad_residual_device, float* grad_skel_state_device, void* cuda_stream) {
  return collisionDevice(c, batch, skel_state_device, nullptr, grad_residual_device, grad_skel_state_device, cuda_stream, true);
}

int mb2_character_joint_parameters_to_skeleton_state_device(const mb2_character* c, int32_t batch, const float* joint_parameters_device,
                                                            float* skeleton_state_device, void* cuda_stream) {
  return skeletonStateDevice(c, batch, joint_parameters_device, nullptr, skeleton_state_device, cuda_stream, false, true);
}
int mb2_character_joint_parameters_to_skeleton_state_backward_device(const mb2_character* c, int32_t batch, const float* joint_parameters_device,
                                                                     const float* grad_skeleton_state_device, float* grad_joint_parameters_device,
                                                                     void* cuda_stream) {
  return skeletonStateDevice(c, batch, joint_parameters_device, grad_skeleton_state_device, grad_joint_parameters_device, cuda_stream, true, true);
}
int mb2_character_joint_parameters_to_local_skeleton_state_device(const mb2_character* c, int32_t batch, const float* joint_parameters_device,
                                                                  float* local_skeleton_state_device, void* cuda_stream) {
  return jointOpDevice(c, batch, kJointOpLocalState, "localSkeletonState", joint_parameters_device, nullptr, local_skeleton_state_device, cuda_stream, false);
}
int mb2_character_joint_parameters_to_local_skeleton_state_backward_device(const mb2_character* c, int32_t batch,
                                                                           const float* joint_parameters_device,
                                                                           const float* grad_local_skeleton_state_device,
                                                                           float* grad_joint_parameters_device, void* cuda_stream) {
  return jointOpDevice(c, batch, kJointOpLocalState, "localSkeletonStateBackward", joint_parameters_device, grad_local_skeleton_state_device,
                       grad_joint_parameters_device, cuda_stream, true);
}
int mb2_character_local_skeleton_state_to_joint_parameters_device(const mb2_character* c, int32_t batch, const float* local_skeleton_state_device,
                                                                  float* joint_parameters_device, void* cuda_stream) {
  return jointOpDevice(c, batch, kJointOpFromLocal, "localSkeletonStateToJointParameters", local_skeleton_state_device, nullptr, joint_parameters_device,
                       cuda_stream, false);
}
int mb2_character_local_skeleton_state_to_joint_parameters_backward_device(const mb2_character* c, int32_t batch,
                                                                           const float* local_skeleton_state_device,
                                                                           const float* grad_joint_parameters_device,
                                                                           float* grad_local_skeleton_state_device, void* cuda_stream) {
  return jointOpDevice(c, batch, kJointOpFromLocal, "localSkeletonStateToJointParametersBackward", local_skeleton_state_device, grad_joint_parameters_device,
                       grad_local_skeleton_state_device, cuda_stream, true);
}
int mb2_character_skeleton_state_to_joint_parameters_device(const mb2_character* c, int32_t batch, const float* skeleton_state_device,
                                                            float* joint_parameters_device, void* cuda_stream) {
  return jointOpDevice(c, batch, kJointOpFromWorld, "skeletonStateToJointParameters", skeleton_state_device, nullptr, joint_parameters_device, cuda_stream, false);
}
int mb2_character_skeleton_state_to_joint_parameters_backward_device(const mb2_character* c, int32_t batch, const float* skeleton_state_device,
                                                                     const float* grad_joint_parameters_device, float* grad_skeleton_state_device,
                                                                     void* cuda_stream) {
  return jointOpDevice(c, batch, kJointOpFromWorld, "skeletonStateToJointParametersBackward", skeleton_state_device, grad_joint_parameters_device,
                       grad_skeleton_state_device, cuda_stream, true);
}

namespace {
// both directions and both variants of mb2_character_*_parameters_to_positions*_device; positions is the forward's output, gradPositions
// the backward's input
int positionsDevice(const mb2_character* c, int32_t batch, const float* params, int32_t numPoints, const int32_t* parents, const float* offsets,
                    int32_t offsetsBatched, float* positions, const float* gradPositions, float* gradParams, float* gradOffsets, void* stream,
                    bool backward, bool joint) {
  MB2_CHECK(c != nullptr, "null character");
  MB2_CHECK(batch >= 0, "batch must not be negative");
  std::vector<int32_t> points;
  const std::string rejected = makePointTables(c->host.numJoints, numPoints, parents, points);
  MB2_CHECK(rejected.empty(), rejected);
  MB2_CHECK(!backward || gradParams != nullptr || gradOffsets != nullptr, "positions backward: grad_params and grad_offsets are both null");
  if (batch == 0) return MB2_OK;
  MB2_CHECK(params != nullptr && (numPoints == 0 || (offsets != nullptr && (backward ? gradPositions != nullptr : positions != nullptr))), "null argument");
  MB2_DEVICE_GUARD(c->device);
  MB2_CHECK(onDevice(c->device, {params}, {offsets, positions, gradPositions, gradParams, gradOffsets}),
            "positions: every array must be device memory on the character's device");
  NvtxRange range(joint ? (backward ? "jointParametersToPositionsBackward" : "jointParametersToPositions")
                        : (backward ? "modelParametersToPositionsBackward" : "modelParametersToPositions"));
  const cudaStream_t s = (cudaStream_t)stream;
  PositionArgs a{};
  a.T = c->tables();
  a.S = c->skeletonTables();
  a.numChildren = int(c->host.children.size());
  a.batch = batch;
  a.params = params;
  a.offsets = offsets;
  a.offsetsBatched = offsetsBatched != 0;
  a.positions = positions;
  a.gradPositions = gradPositions;
  a.gradParams = gradParams;
  a.gradOffsets = gradOffsets;
  a.fromJointParameters = joint;
  int32_t* dPoints = nullptr;
  if (numPoints > 0) MB2_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&dPoints), points.size() * sizeof(int32_t), s));
  a.P = pointTablesAt(dPoints, c->host.numJoints, numPoints);
  cudaError_t e = numPoints > 0 ? cudaMemcpyAsync(dPoints, points.data(), points.size() * sizeof(int32_t), cudaMemcpyHostToDevice, s) : cudaSuccess;
  if (e == cudaSuccess) e = backward ? launchPositionsBackward(a, s) : launchPositions(a, s);
  const cudaError_t f = numPoints > 0 ? cudaFreeAsync(dPoints, s) : cudaSuccess;
  MB2_CUDA(e != cudaSuccess ? e : f);
  return MB2_OK;
}
} // namespace

int mb2_character_model_parameters_to_positions_device(const mb2_character* c, int32_t batch, const float* model_parameters_device, int32_t num_points,
                                                       const int32_t* parents, const float* offsets_device, int32_t offsets_batched,
                                                       float* positions_device, void* cuda_stream) {
  return positionsDevice(c, batch, model_parameters_device, num_points, parents, offsets_device, offsets_batched, positions_device, nullptr, nullptr,
                         nullptr, cuda_stream, false, false);
}
int mb2_character_joint_parameters_to_positions_device(const mb2_character* c, int32_t batch, const float* joint_parameters_device, int32_t num_points,
                                                       const int32_t* parents, const float* offsets_device, int32_t offsets_batched,
                                                       float* positions_device, void* cuda_stream) {
  return positionsDevice(c, batch, joint_parameters_device, num_points, parents, offsets_device, offsets_batched, positions_device, nullptr, nullptr,
                         nullptr, cuda_stream, false, true);
}
int mb2_character_model_parameters_to_positions_backward_device(const mb2_character* c, int32_t batch, const float* model_parameters_device,
                                                                int32_t num_points, const int32_t* parents, const float* offsets_device,
                                                                int32_t offsets_batched, const float* grad_positions_device,
                                                                float* grad_model_parameters_device, float* grad_offsets_device, void* cuda_stream) {
  return positionsDevice(c, batch, model_parameters_device, num_points, parents, offsets_device, offsets_batched, nullptr, grad_positions_device,
                         grad_model_parameters_device, grad_offsets_device, cuda_stream, true, false);
}
int mb2_character_joint_parameters_to_positions_backward_device(const mb2_character* c, int32_t batch, const float* joint_parameters_device,
                                                                int32_t num_points, const int32_t* parents, const float* offsets_device,
                                                                int32_t offsets_batched, const float* grad_positions_device,
                                                                float* grad_joint_parameters_device, float* grad_offsets_device, void* cuda_stream) {
  return positionsDevice(c, batch, joint_parameters_device, num_points, parents, offsets_device, offsets_batched, nullptr, grad_positions_device,
                         grad_joint_parameters_device, grad_offsets_device, cuda_stream, true, true);
}

namespace {
// both directions of mb2_character_skin_points*_device: checks the arguments and fills the kernel arguments except the outputs
int skinArgs(const mb2_character* c, int32_t batch, const float* skelState, const float* restPoints, int32_t restBatched, SkinArgs& a) {
  MB2_CHECK(c != nullptr, "null character");
  MB2_CHECK(c->skin.numVertices > 0, "skin points: the character has no skinning (mb2_character_set_skinning)");
  MB2_CHECK(batch >= 0, "batch must not be negative");
  MB2_CHECK(batch == 0 || restPoints != nullptr || restBatched == 0, "skin points: batched rest points need a rest_points array");
  a = SkinArgs{};
  a.S = c->skinTables();
  a.numJoints = c->host.numJoints;
  a.batch = batch;
  a.skelState = skelState;
  a.restPoints = restPoints != nullptr ? restPoints : c->skinDev->rest.p;
  a.restBatched = restBatched != 0;
  return MB2_OK;
}
} // namespace

int mb2_character_skin_points_device(const mb2_character* c, int32_t batch, const float* skel_state_device, const float* rest_points_device,
                                     int32_t rest_points_batched, float* points_device, void* cuda_stream) {
  SkinArgs a;
  int rc = skinArgs(c, batch, skel_state_device, rest_points_device, rest_points_batched, a);
  if (rc != MB2_OK || batch == 0) return rc;
  MB2_CHECK(skel_state_device != nullptr && points_device != nullptr, "null argument");
  MB2_DEVICE_GUARD(c->device);
  MB2_CHECK(onDevice(c->device, {skel_state_device, points_device}, {rest_points_device}),
            "skin points: every array must be device memory on the character's device");
  NvtxRange range("skinPoints");
  a.points = points_device;
  MB2_CUDA(launchSkinPoints(a, (cudaStream_t)cuda_stream));
  return MB2_OK;
}

int mb2_character_skin_points_backward_device(const mb2_character* c, int32_t batch, const float* skel_state_device, const float* rest_points_device,
                                              int32_t rest_points_batched, const float* grad_points_device, float* grad_skel_state_device,
                                              float* grad_rest_points_device, void* cuda_stream) {
  SkinArgs a;
  int rc = skinArgs(c, batch, skel_state_device, rest_points_device, rest_points_batched, a);
  if (rc != MB2_OK) return rc;
  MB2_CHECK(rest_points_device != nullptr || grad_rest_points_device == nullptr,
            "skin points: grad_rest_points must be null when the character's rest mesh is skinned");
  if (batch == 0) return MB2_OK;
  MB2_CHECK(skel_state_device != nullptr && grad_points_device != nullptr, "null argument");
  MB2_DEVICE_GUARD(c->device);
  MB2_CHECK(onDevice(c->device, {skel_state_device, grad_points_device}, {rest_points_device, grad_skel_state_device, grad_rest_points_device}),
            "skin points: every array must be device memory on the character's device");
  NvtxRange range("skinPointsBackward");
  a.gradPoints = grad_points_device;
  a.gradState = grad_skel_state_device;
  a.gradRest = grad_rest_points_device;
  MB2_CUDA(launchSkinPointsBackward(a, (cudaStream_t)cuda_stream));
  return MB2_OK;
}

namespace {
// both directions of mb2_character_skin_with_blend_shapes*_device: checks the arguments and fills the kernel arguments except the outputs
int blendSkinArgs(const mb2_character* c, int32_t batch, const float* skelState, const float* blendWeights, int32_t numWeights, BlendSkinArgs& a) {
  MB2_CHECK(c != nullptr, "null character");
  MB2_CHECK(c->skin.numVertices > 0, "skin with blend shapes: the character has no skinning (mb2_character_set_skinning)");
  MB2_CHECK(c->blend.numShapes > 0, "skin with blend shapes: the character has no blend shape (mb2_character_set_blend_shape)");
  MB2_CHECK(c->blend.numVertices == c->skin.numVertices, "skin with blend shapes: the blend shape's vertex count differs from the skinning's");
  MB2_CHECK(numWeights >= 1 && numWeights <= c->blend.numShapes, "skin with blend shapes: num_weights must be in [1, number of shape vectors]");
  int rc = skinArgs(c, batch, skelState, nullptr, 0, a.skin);
  if (rc != MB2_OK) return rc;
  a.Bs = c->blendShapeTables();
  a.skin.restPoints = nullptr;
  a.numWeights = numWeights;
  a.blendWeights = blendWeights;
  a.gradWeights = nullptr;
  return MB2_OK;
}
} // namespace

int mb2_character_skin_with_blend_shapes_device(const mb2_character* c, int32_t batch, const float* skel_state_device, const float* blend_weights_device,
                                                int32_t num_weights, float* points_device, void* cuda_stream) {
  BlendSkinArgs a{};
  int rc = blendSkinArgs(c, batch, skel_state_device, blend_weights_device, num_weights, a);
  if (rc != MB2_OK || batch == 0) return rc;
  MB2_CHECK(skel_state_device != nullptr && blend_weights_device != nullptr && points_device != nullptr, "null argument");
  MB2_DEVICE_GUARD(c->device);
  MB2_CHECK(onDevice(c->device, {skel_state_device, blend_weights_device, points_device}),
            "skin with blend shapes: every array must be device memory on the character's device");
  MB2_CHECK(blendSkinFits(a), "skin with blend shapes: num_weights is too large for the device's shared memory");
  NvtxRange range("skinWithBlendShapes");
  a.skin.points = points_device;
  MB2_CUDA(launchSkinWithBlendShapes(a, (cudaStream_t)cuda_stream));
  return MB2_OK;
}

int mb2_character_skin_with_blend_shapes_backward_device(const mb2_character* c, int32_t batch, const float* skel_state_device,
                                                         const float* blend_weights_device, int32_t num_weights, const float* grad_points_device,
                                                         float* grad_skel_state_device, float* grad_blend_weights_device, void* cuda_stream) {
  BlendSkinArgs a{};
  int rc = blendSkinArgs(c, batch, skel_state_device, blend_weights_device, num_weights, a);
  if (rc != MB2_OK || batch == 0) return rc;
  MB2_CHECK(skel_state_device != nullptr && blend_weights_device != nullptr && grad_points_device != nullptr, "null argument");
  MB2_DEVICE_GUARD(c->device);
  MB2_CHECK(onDevice(c->device, {skel_state_device, blend_weights_device, grad_points_device}, {grad_skel_state_device, grad_blend_weights_device}),
            "skin with blend shapes: every array must be device memory on the character's device");
  MB2_CHECK(blendSkinFits(a), "skin with blend shapes: num_weights is too large for the device's shared memory");
  NvtxRange range("skinWithBlendShapesBackward");
  a.skin.gradPoints = grad_points_device;
  a.skin.gradState = grad_skel_state_device;
  a.gradWeights = grad_blend_weights_device;
  MB2_CUDA(launchSkinWithBlendShapesBackward(a, (cudaStream_t)cuda_stream));
  return MB2_OK;
}

namespace {
// both directions of mb2_character_vertex_normals*_device: checks the arguments and fills the tables
int normalArgs(const mb2_character* c, int32_t batch, NormalArgs& a) {
  MB2_CHECK(c != nullptr, "null character");
  MB2_CHECK(c->faces.numVertices > 0, "vertex normals: the character has no mesh faces (mb2_character_set_mesh_faces)");
  MB2_CHECK(batch >= 0, "batch must not be negative");
  a = NormalArgs{};
  a.M = c->meshFaceTables();
  a.batch = batch;
  return MB2_OK;
}
} // namespace

int mb2_character_vertex_normals_device(const mb2_character* c, int32_t batch, const float* positions_device, float* normals_device, void* cuda_stream) {
  NormalArgs a;
  int rc = normalArgs(c, batch, a);
  if (rc != MB2_OK || batch == 0) return rc;
  MB2_CHECK(positions_device != nullptr && normals_device != nullptr, "vertex normals: null argument");
  MB2_DEVICE_GUARD(c->device);
  MB2_CHECK(onDevice(c->device, {positions_device, normals_device}), "vertex normals: every array must be device memory on the character's device");
  NvtxRange range("vertexNormals");
  a.positions = positions_device;
  a.normals = normals_device;
  MB2_CUDA(launchVertexNormals(a, (cudaStream_t)cuda_stream));
  return MB2_OK;
}

int mb2_character_closest_points_on_mesh_device(const mb2_character* c, int32_t batch, int32_t num_points, const float* vertex_positions_device,
                                                const float* points_device, float max_dist, float* out_points_device, int32_t* out_face_device,
                                                float* out_bary_device, void* cuda_stream) {
  MB2_CHECK(c != nullptr, "null character");
  MB2_CHECK(c->faces.numVertices > 0, "closest points: the character has no mesh faces (mb2_character_set_mesh_faces)");
  MB2_CHECK(c->tree.numNodes > 0, "closest points: the character has no mesh tree (mb2_character_set_mesh_tree)");
  MB2_CHECK(batch >= 0 && num_points >= 0, "closest points: batch and num_points must not be negative");
  MB2_CHECK(max_dist >= 0.f, "closest points: max_dist must be >= 0 and not NaN (+inf for no bound)");
  if (batch == 0 || num_points == 0) return MB2_OK;
  MB2_CHECK(vertex_positions_device != nullptr && points_device != nullptr && out_points_device != nullptr && out_face_device != nullptr &&
                out_bary_device != nullptr,
            "closest points: null argument");
  MB2_DEVICE_GUARD(c->device);
  MB2_CHECK(onDevice(c->device, {vertex_positions_device, points_device, out_points_device, out_face_device, out_bary_device}),
            "closest points: every array must be device memory on the character's device");
  NvtxRange range("closestPointsOnMesh");
  ClosestPointArgs a{};
  a.M = c->meshFaceTables();
  a.T = c->meshTreeTables();
  a.batch = batch;
  a.numPoints = num_points;
  a.maxDist2 = max_dist * max_dist;
  a.vertices = vertex_positions_device;
  a.points = points_device;
  a.outPoints = out_points_device;
  a.outFace = out_face_device;
  a.outBary = out_bary_device;
  MB2_CUDA(launchClosestPointsOnMesh(a, (cudaStream_t)cuda_stream));
  return MB2_OK;
}

int mb2_closest_points_device(int device, int32_t batch, int32_t num_source, int32_t num_target, int32_t target_batched,
                              const float* source_device, const float* source_normals_device, const float* target_device,
                              const float* target_normals_device, float max_dist, float max_normal_dot, float* out_points_device,
                              float* out_normals_device, int32_t* out_index_device, void* cuda_stream) {
  MB2_CHECK(device >= 0, "closest points on cloud: device must not be negative");
  MB2_CHECK(batch >= 0 && num_source >= 0 && num_target >= 0, "closest points on cloud: batch, num_source and num_target must not be negative");
  MB2_CHECK(max_dist >= 0.f, "closest points on cloud: max_dist must be >= 0 and not NaN (+inf for no bound)");
  MB2_CHECK(max_normal_dot == max_normal_dot, "closest points on cloud: max_normal_dot must not be NaN");
  const bool normals = source_normals_device != nullptr;
  MB2_CHECK(num_target == 0 || normals == (target_normals_device != nullptr), // with no target, neither target array is read
            "closest points on cloud: source_normals and target_normals must be both null or both set");
  MB2_CHECK(normals == (out_normals_device != nullptr), "closest points on cloud: out_normals must be set exactly when normals are given");
  if (batch == 0 || num_source == 0) return MB2_OK;
  MB2_CHECK(source_device != nullptr && out_points_device != nullptr && out_index_device != nullptr && (num_target == 0 || target_device != nullptr),
            "closest points on cloud: null argument");
  MB2_DEVICE_GUARD(device);
  int rc = requireDevice(device);
  if (rc != MB2_OK) return rc;
  MB2_CHECK(onDevice(device, {source_device, out_points_device, out_index_device},
                     {source_normals_device, out_normals_device, num_target > 0 ? target_device : nullptr,
                      num_target > 0 ? target_normals_device : nullptr}),
            "closest points on cloud: every array must be device memory on the given device");
  NvtxRange range("closestPointsOnCloud");
  ClosestCloudArgs a{};
  a.batch = batch;
  a.numSource = num_source;
  a.numTarget = num_target;
  a.targetBatched = target_batched != 0;
  a.maxDist2 = max_dist * max_dist;
  a.maxNormalDot = max_normal_dot;
  a.source = source_device;
  a.sourceNormals = source_normals_device;
  a.target = target_device;
  a.targetNormals = target_normals_device;
  a.outPoints = out_points_device;
  a.outNormals = out_normals_device;
  a.outIndex = out_index_device;
  MB2_CUDA(launchClosestPointsOnCloud(a, (cudaStream_t)cuda_stream));
  return MB2_OK;
}

int mb2_character_vertex_normals_backward_device(const mb2_character* c, int32_t batch, const float* positions_device, const float* grad_normals_device,
                                                 float* grad_positions_device, void* cuda_stream) {
  NormalArgs a;
  int rc = normalArgs(c, batch, a);
  if (rc != MB2_OK || batch == 0) return rc;
  MB2_CHECK(positions_device != nullptr && grad_normals_device != nullptr && grad_positions_device != nullptr, "vertex normals: null argument");
  MB2_DEVICE_GUARD(c->device);
  MB2_CHECK(onDevice(c->device, {positions_device, grad_normals_device, grad_positions_device}),
            "vertex normals: every array must be device memory on the character's device");
  NvtxRange range("vertexNormalsBackward");
  a.positions = positions_device;
  a.gradNormals = grad_normals_device;
  a.gradPositions = grad_positions_device;
  MB2_CUDA(launchVertexNormalsBackward(a, (cudaStream_t)cuda_stream));
  return MB2_OK;
}

int mb2_solver_function_input_gradients_device(mb2_solver_function* f, int32_t index, const float* parameters_device, const float* direction_device,
                                               float* grad_weights_device, float* grad_offsets_device, float* grad_targets_device, void* cuda_stream) {
  MB2_CHECK(f != nullptr, "null solver function");
  MB2_CHECK(index >= 0 && index < int(f->host.efs.size()), "error function index out of range");
  const HostErrorFunction& ef = f->host.efs[index];
  MB2_CHECK(ef.kind == 0 || ef.kind == 1, "input gradients: only Position and Orientation (matrix difference) blocks are supported");
  const float kEps = 1e-9f; // the L2 snapping of GeneralizedLossT (makeEfDesc)
  MB2_CHECK(ef.lossAlpha >= 2.f - kEps && ef.lossAlpha <= 2.f + kEps, "input gradients: only the L2 loss is supported");
  MB2_CHECK(parameters_device != nullptr && direction_device != nullptr, "null parameters or direction");
  MB2_DEVICE_GUARD(f->ch->device);
  float* outs[3] = {grad_weights_device, grad_offsets_device, grad_targets_device};
  MB2_CHECK(onDevice(f->ch->device, {parameters_device, direction_device}, {grad_weights_device, grad_offsets_device, grad_targets_device}),
            "input gradients: every array must be device memory on the function's device");
  int rc = ensurePlan(f, f->planMode, f->planSchedDense, f->planAlignRows);
  if (rc != MB2_OK) return rc;
  NvtxRange range("inputGradients");
  cudaStream_t st = (cudaStream_t)cuda_stream;
  const int nc = ef.numConstraints(), per = ef.kind == 0 ? 3 : 4;
  int unitBegin = -1;
  for (size_t u = 0; u < f->plan.units.size() && unitBegin < 0; ++u)
    if (f->plan.units[u].ef == index) unitBegin = int(u);
  if (nc == 0) return MB2_OK;
  if (unitBegin < 0) { // a block with weight 0 has no rows: its gradient contribution is zero
    const size_t sizes[3] = {size_t(nc), size_t(nc) * per, size_t(nc) * per};
    for (int k = 0; k < 3; ++k)
      if (outs[k]) MB2_CUDA(cudaMemsetAsync(outs[k], 0, size_t(f->B) * sizes[k] * sizeof(float), st));
    return MB2_OK;
  }
  InputGradientArgs a{};
  a.T = f->tables();
  a.unitBegin = unitBegin;
  a.numConstraints = nc;
  a.kind = ef.kind == 0 ? kUnitPosition : kUnitOrientation;
  a.batch = f->B;
  a.theta = parameters_device;
  a.direction = direction_device;
  a.enabledList = f->dEnabledList.p;
  a.numEnabled = int(f->plan.enabledList.size());
  a.targets = f->dTargets.p;
  a.cweights = f->dWeights.p;
  a.gradWeights = grad_weights_device;
  a.gradOffsets = grad_offsets_device;
  a.gradTargets = grad_targets_device;
  MB2_CUDA(launchInputGradients(a, st));
  return MB2_OK;
}

int mb2_solver_function_implicit_direction_device(mb2_solver_function* f, const float* parameters_device, const float* grad_parameters_device,
                                                  float* direction_device, float* jacobian_direction_device, float* residual_device,
                                                  float* gradient_rms_device, void* cuda_stream) {
  MB2_CHECK(f != nullptr, "null solver function");
  MB2_CHECK(parameters_device != nullptr && grad_parameters_device != nullptr, "null parameters or gradient");
  MB2_CHECK(direction_device != nullptr, "null direction");
  MB2_DEVICE_GUARD(f->ch->device);
  MB2_CHECK(onDevice(f->ch->device, {parameters_device, grad_parameters_device},
                     {direction_device, jacobian_direction_device, residual_device, gradient_rms_device}),
            "implicit direction: every array must be device memory on the function's device");
  int rc = ensurePlan(f, 0); // the API-order Jacobian: column c = model parameter c
  if (rc != MB2_OK) return rc;
  NvtxRange range("implicitDirection");
  cudaStream_t st = (cudaStream_t)cuda_stream;
  MB2_CUDA(launchSweep(sweepArgs(f, parameters_device, nullptr), true, st, &f->lastSweep[1]));
  ImplicitDirectionArgs a{};
  a.batch = f->B;
  a.numParams = f->ch->host.numParams;
  a.rows = f->plan.numRows;
  a.rowStride = mb2_solver_function_jacobian_rows(f);
  a.ldJ = f->ldJ;
  a.jacobian = f->dJ.p;
  a.enabledList = f->dEnabledList.p;
  a.numEnabled = int(f->plan.enabledList.size());
  a.gradParameters = grad_parameters_device;
  a.direction = direction_device;
  a.jacobianDirection = jacobian_direction_device;
  a.residual = residual_device;
  a.gradientRms = gradient_rms_device;
  ImplicitDirectionConfig cfg;
  MB2_CUDA(implicitDirectionConfigure(a, cfg));
  MB2_CUDA(f->dJacobi.resize(std::max<size_t>(1, size_t(cfg.grid) * cfg.slotDoubles)));
  a.scratch = f->dJacobi.p;
  a.slotDoubles = cfg.slotDoubles;
  a.gramInShared = cfg.gramInShared ? 1 : 0;
  MB2_CUDA(launchImplicitDirection(a, cfg, st));
  return MB2_OK;
}

// ---------------------------------------------------------------------------------------------
// Solver
// ---------------------------------------------------------------------------------------------
int mb2_solver_create(mb2_solver_function* f, const mb2_gauss_newton_options* opt, mb2_solver** out) {
  MB2_CHECK(f != nullptr && out != nullptr, "null argument");
  auto s = std::make_unique<mb2_solver>();
  s->fn = f;
  if (opt) s->opt = *opt; else mb2_default_gauss_newton_options(&s->opt);
  MB2_DEVICE_GUARD(f->ch->device);
  MB2_CUDA(cudaMallocHost(&s->hActiveCount, kSolveSlices * sizeof(int)));
  *out = s.release();
  return MB2_OK;
}
void mb2_solver_destroy(mb2_solver* s) { delete s; }
int mb2_solver_set_options(mb2_solver* s, const mb2_gauss_newton_options* opt) {
  MB2_CHECK(s != nullptr && opt != nullptr, "null argument");
  s->opt = *opt;
  return MB2_OK;
}
int mb2_solver_set_enabled_parameters(mb2_solver* s, const uint64_t* bits) {
  MB2_CHECK(s != nullptr, "null solver");
  return mb2_solver_function_set_enabled_parameters(s->fn, bits);
}
int mb2_solver_set_profiling(mb2_solver* s, int32_t enabled) {
  MB2_CHECK(s != nullptr, "null solver");
  s->profiling = enabled != 0;
  s->inKernelProfile = enabled >= 2;
  return MB2_OK;
}

namespace {
// the figures chooseSolvePath weighs, of the plan ensurePlan builds (or keeps) for a request
int planFigures(mb2_solver_function* f, int mode, bool schedDense, bool strips, PlanFigures& F, std::string& msg) {
  const int rc = ensurePlan(f, mode, schedDense, strips);
  if (rc != MB2_OK) { msg = g_lastError; return rc; }
  F = PlanFigures{};
  F.numCols = f->plan.numCols;
  F.recStride = f->plan.recStride;
  F.jtjTensor = jtjTensorSupported(F.numCols, F.numCols, f->ldJ);
  if (const DeviceSchedule* ds = f->planMode == 2 ? f->sched.get() : nullptr) {
    F.nPad = ds->host.nPad;
    F.numTiles = ds->host.numTiles;
    F.schedBlobInts = ds->dev.blobInts;
    F.stripStride = ds->gram.stride;
    F.gramBlobInts = ds->gBlobInts;
    F.orderEntries = int(ds->gram.tileOrder.size());
    F.gramCholValid = ds->gcValid;
    F.fusedBlobWords = ds->fLayout.words;
  }
  return MB2_OK;
}

} // namespace

int mb2_solver_solve_device(mb2_solver* s, float* theta, void* cudaStream) {
  MB2_CHECK(s != nullptr && theta != nullptr, "null argument");
  mb2_solver_function* f = s->fn;
  MB2_DEVICE_GUARD(f->ch->device);
  NvtxRange nvtxSolve("mb2::SolverT::solve");
  const mb2_gauss_newton_options& o = s->opt;
  const DeviceLimits lim = deviceLimits();
  std::string msg;
  const PlanFiguresFn plan = [f](int mode, bool schedDense, bool strips, PlanFigures& F, std::string& m) { return planFigures(f, mode, schedDense, strips, F, m); };
  int rc = chooseSolvePath(o, f->B, f->ch->host, f->host, plan, lim, s->path, msg);
  if (s->path.planMode != 0 && f->sched) f->sched->fusedGroups = s->path.fused.groups;
  if (rc != MB2_OK) {
    s->path = SolvePath{};
    return fail(rc, msg);
  }
  if (s->profiling) s->path.slices = 1; // events around every launch on one stream: the per-kernel times keep their meaning
  const SolvePath& P = s->path;
  cudaStream_t st = cudaStream ? (cudaStream_t)cudaStream : f->stream;
  const int B = f->B, n = f->ch->host.numParams;
  const int ns = f->plan.numCols;
  const int maxIt = int(std::min<uint64_t>(o.max_iterations, 1u << 30));
  const int minIt = int(std::min<uint64_t>(o.min_iterations, 1u << 30));
  MB2_CUDA(s->dIterations.resize(B));
  MB2_CUDA(s->dStatus.resize(B));
  if (o.store_error_history) {
    MB2_CUDA(s->dHistory.resize(size_t(B) * std::max(maxIt, 1)));
    MB2_CUDA(cudaMemsetAsync(s->dHistory.p, 0, size_t(B) * std::max(maxIt, 1) * sizeof(double), st));
    s->historyStride = size_t(std::max(maxIt, 1));
  }
  // the per-instance state every launch takes (lastErrors, active, activeCount: below; the persistent kernel keeps them in shared memory)
  SolveState state{};
  state.errors = f->dErrors.p;
  state.iterations = s->dIterations.p;
  state.status = s->dStatus.p;
  state.history = o.store_error_history ? s->dHistory.p : nullptr;
  state.minIterations = minIt;
  state.maxIterations = maxIt;
  state.threshold = o.threshold;
  for (auto& e : s->events) { cudaEventDestroy(e.start); cudaEventDestroy(e.stop); }
  s->events.clear();
  if (s->profiling && (P.kind == kSolvePersistent || P.kind == kSolveGramCholesky)) {
    MB2_CUDA(s->dPhaseCycles.resize(16));
    MB2_CUDA(cudaMemsetAsync(s->dPhaseCycles.p, 0, 16 * sizeof(unsigned long long), st));
  }
  if (P.kind == kSolvePersistent) { // the whole solve in one launch
    const DeviceSchedule& ds = *f->sched;
    MB2_CUDA(s->dWorkCounter.resize(1));
    MB2_CUDA(cudaMemsetAsync(s->dWorkCounter.p, 0, sizeof(int32_t), st));
    FusedArgs fa{};
    fa.batch = B;
    fa.T = f->tables();
    fa.blob = ds.fBlob.p;
    fa.L = ds.fLayout;
    fa.S = ds.dev;
    fa.schedGlobal = ds.dev.blob;
    for (int k = 0; k < 8; ++k) fa.gramOff[k] = ds.gOffsets[k];
    fa.numStrips = ds.gram.numStrips;
    fa.stripStride = ds.gram.stride;
    fa.residOff = ds.gram.residOff;
    fa.numOrder = int32_t(ds.gram.tileOrder.size());
    fa.regularization = o.regularization;
    fa.theta = theta;
    fa.ldTheta = n;
    fa.targets = f->dTargets.p;
    fa.cweights = f->dWeights.p;
    fa.state = state;
    fa.workCounter = s->dWorkCounter.p;
    fa.phaseCycles = s->inKernelProfile ? s->dPhaseCycles.p : nullptr;
    if (s->profiling) {
      if (!s->fusedStart) { MB2_CUDA(cudaEventCreate(&s->fusedStart)); MB2_CUDA(cudaEventCreate(&s->fusedStop)); }
      MB2_CUDA(cudaEventRecord(s->fusedStart, st));
    }
    {
      NvtxRange nvtxIt("mb2::fusedSolveKernel (GaussNewtonSolverT::doIteration x maxIterations)");
      MB2_CUDA(launchFusedSolve(fa, P.fused, lim.numSms, s->inKernelProfile, st));
    }
    if (s->profiling) MB2_CUDA(cudaEventRecord(s->fusedStop, st));
    s->kernelLaunches = 1;
    return MB2_OK;
  }
  // normal equations of the JtJ kernels: full symmetric [ns+1][ldH] in device-column order (row/column ns = J^T r)
  const int ldH = roundUp(ns + 1, 16);
  const size_t hStride = size_t(ns + 1) * ldH;
  if (P.kind == kSolveDense || P.kind == kSolveTilesKMajor) MB2_CUDA(s->dH.resize(size_t(B) * hStride));
  const size_t tilesStride = P.strips ? size_t(f->sched->host.numTiles) * 256 + f->sched->host.nPad : 0;
  if (P.kind == kSolveTiles) MB2_CUDA(s->dTiles.resize(size_t(B) * tilesStride));
  const bool qr = P.kind == kSolveQr || P.kind == kSolveTrustRegionQr;
  if (qr) MB2_CUDA(s->dQrChunks.upload(P.qrChunkStarts, st));
  if (P.kind == kSolveTrustRegionQr) { // TrustRegionQRT::initializeSolver (trust_region_qr.cpp:38-40): the current radius starts at the option's value
    MB2_CUDA(s->dRadius.upload(std::vector<float>(size_t(B), o.trust_region_radius), st));
    MB2_CUDA(s->dRSaved.resize(size_t(B) * P.trRSavedFloats));
  }
  const int ldG = cholGradientLd(ns);
  MB2_CUDA(s->dGrad.resize(size_t(B) * ldG));
  MB2_CUDA(s->dDelta.resize(size_t(B) * ns));
  MB2_CUDA(s->dTheta0.resize(size_t(B) * n));
  MB2_CUDA(s->dLastErrors.resize(B));
  MB2_CUDA(s->dActive.resize(B));
  MB2_CUDA(s->dActiveCount.resize(size_t(P.slices)));
  state.lastErrors = s->dLastErrors.p; state.active = s->dActive.p; state.activeCount = s->dActiveCount.p;
  const bool lineSearch = o.do_line_search != 0 && P.kind != kSolveTrustRegionQr; // (TrustRegionQRT has no line search: steps are accepted or rejected by rho)
  if (lineSearch) {
    MB2_CUDA(s->dThetaOrig.resize(size_t(B) * n));
    MB2_CUDA(s->dTrialErrors.resize(B));
    MB2_CUDA(s->dScale.resize(B));
    MB2_CUDA(s->dSearching.resize(B));
    MB2_CUDA(s->dGradDotDelta.resize(B));
  }

  // ---- kernel arguments: only the iteration changes from one iteration to the next ----
  const SweepArgs sweep = sweepArgs(f, theta, s->dActive.p);
  GramArgs g{};
  if (P.strips) {
    const DeviceSchedule& ds = *f->sched;
    g.batch = B;
    g.strips = f->dJ.p;
    g.stripStride = size_t(ds.gram.stride);
    g.residOff = ds.gram.residOff;
    g.active = s->dActive.p;
    g.numStrips = ds.gram.numStrips;
    g.numTiles = ds.host.numTiles;
    g.numTileCols = ds.host.numTileCols;
    g.nPad = ds.host.nPad;
    g.numOrder = int32_t(ds.gram.tileOrder.size());
    g.blob = ds.gBlob.p;
    g.blobInts = ds.gBlobInts;
    g.offTileOrder = ds.gOffsets[0]; g.offTilePairStart = ds.gOffsets[1]; g.offPairA = ds.gOffsets[2]; g.offPairB = ds.gOffsets[3];
    g.offColStripStart = ds.gOffsets[4]; g.offColStrip = ds.gOffsets[5]; g.offStripRow = ds.gOffsets[6]; g.offTileInfo = ds.gOffsets[7];
    g.regularization = o.regularization;
    g.out = s->dTiles.p;
    g.outStride = tilesStride;
  }
  CholArgs c{};
  c.batch = B;
  c.H = s->dH.p;
  c.ns = ns;
  c.ldH = ldH;
  c.hStride = hStride;
  c.regularization = o.regularization;
  c.cols = f->dDeviceCols.p;
  c.theta = theta;
  c.ldTheta = n;
  c.delta = s->dDelta.p;
  c.applyUpdate = lineSearch ? 0 : 1;
  c.state = state;
  c.bookkeeping = lineSearch ? 0 : 1;
  c.gradDotDelta = lineSearch ? s->dGradDotDelta.p : nullptr;
  c.g = s->dGrad.p;
  c.ldG = ldG;
  c.tilesIn = P.strips ? s->dTiles.p : nullptr;
  c.tilesStride = tilesStride;
  TrQrArgs t{};
  t.q.c = c;
  t.q.jacobian = f->dJ.p;
  t.q.numCols = f->plan.numCols;
  t.q.ldJ = f->ldJ;
  t.q.chunkStart = s->dQrChunks.p;
  t.q.numChunks = int32_t(P.qrChunkStarts.size()) - 1;
  t.T = f->tables();
  t.targets = f->dTargets.p;
  t.cweights = f->dWeights.p;
  t.radius = s->dRadius.p;
  t.rSaved = s->dRSaved.p;
  t.maxRadius = 10.f; // trust_region_qr.h:73
  t.maxChunkRows = P.qrWidestChunk;
  GramCholArgs gc{};
  gc.g = g;
  gc.c = c;
  gc.c.tilesIn = nullptr;
  gc.phaseCycles = s->inKernelProfile ? s->dPhaseCycles.p : nullptr;
  GramCholGlobalTables gt{};
  if (P.kind == kSolveGramCholesky) {
    const DeviceSchedule& ds = *f->sched;
    gc.parkTiles = ds.gc.parkTiles;
    if (gc.parkTiles > 0) {
      const int slots = gramCholeskyParkSlots(gc, ds.dev, ds.gcParams != nullptr);
      if (slots < 1) {
        s->path = SolvePath{};
        return fail(MB2_ERR_CUDA, "Gram + Cholesky fusion: no resident CTA");
      }
      if (s->dParkSlots.n < size_t(slots / 32)) { // grown only here, and every launch leaves it all zero
        MB2_CUDA(s->dParkSlots.resize(size_t(slots / 32)));
        MB2_CUDA(cudaMemsetAsync(s->dParkSlots.p, 0, s->dParkSlots.n * sizeof(uint32_t), st));
      }
      MB2_CUDA(s->dPark.resize(size_t(slots) * size_t(gc.parkTiles) * 256));
      gc.park = s->dPark.p;
      gc.parkSlots = s->dParkSlots.p;
      gc.parkSlotWords = int32_t(slots / 32);
    }
    gt.L = ds.gc.L;
    gt.tab = ds.gcTab.p;
  }
  CholArgs& step = qr ? t.q.c : (P.kind == kSolveGramCholesky ? gc.c : c); // the arguments of the linear-solve launch
  SweepArgs trial = sweepArgs(f, theta, s->dSearching.p);
  trial.errors = s->dTrialErrors.p;
  LineSearchArgs la{};
  la.batch = B;
  la.errors = f->dErrors.p;
  la.trialErrors = s->dTrialErrors.p;
  la.gradDotDelta = s->dGradDotDelta.p;
  la.scale = s->dScale.p;
  la.searching = s->dSearching.p;
  la.subsetVariant = o.subset_line_search;

  // ---- instance slices (SolvePath::slices): slice k holds instances [B k / S, B (k + 1) / S) with its own active counter, and runs its
  // iteration chain on its own stream (slice 0 on the caller's). The arguments' slice functions offset its per-instance pointers.
  const int S = P.slices;
  auto sliceBegin = [&](int k) { return int(int64_t(B) * k / S); };
  auto sliceStream = [&](int k) { return k == 0 ? st : s->sliceStreams[k - 1]; };
  if (S > 1 && !s->forkEvent) {
    MB2_CUDA(cudaEventCreateWithFlags(&s->forkEvent, cudaEventDisableTiming));
    for (int i = 0; i < kSolveSlices - 1; ++i) {
      MB2_CUDA(cudaStreamCreateWithFlags(&s->sliceStreams[i], cudaStreamNonBlocking));
      MB2_CUDA(cudaEventCreateWithFlags(&s->joinEvents[i], cudaEventDisableTiming));
    }
  }
  auto fork = [&]() -> int {
    if (S == 1) return MB2_OK;
    MB2_CUDA(cudaEventRecord(s->forkEvent, st));
    for (int k = 1; k < S; ++k) MB2_CUDA(cudaStreamWaitEvent(sliceStream(k), s->forkEvent, 0));
    return MB2_OK;
  };
  auto join = [&]() -> int {
    for (int k = 1; k < S; ++k) {
      MB2_CUDA(cudaEventRecord(s->joinEvents[k - 1], sliceStream(k)));
      MB2_CUDA(cudaStreamWaitEvent(st, s->joinEvents[k - 1], 0));
    }
    return MB2_OK;
  };

  s->kernelLaunches = 0;
  initSolveStateKernel<<<(B + 127) / 128, 128, 0, st>>>(B, state);
  MB2_CUDA(cudaGetLastError());
  MB2_CUDA(cudaMemcpyAsync(s->dTheta0.p, theta, size_t(B) * n * sizeof(float), cudaMemcpyDeviceToDevice, st));
  if ((rc = fork()) != MB2_OK) return rc;

  static const bool cholProfile = getenv("MB2_CHOL_PROFILE") != nullptr;
  constexpr int kPollEvery = 4; // iterations between two reads of the device-side active counter (each read blocks the host on `st`)
  for (int it = 0; it < maxIt; ++it) {
    step.state.iteration = it;
    step.profile = (it == 0 && cholProfile) ? 1 : 0;
    // S > 1 only on the Gram + Cholesky path without line search: every other path runs the whole batch as slice 0
    for (int k = 0; k < S; ++k) {
      const cudaStream_t sk = sliceStream(k);
      const int b0 = sliceBegin(k), count = sliceBegin(k + 1) - b0;
      MB2_CUDA(cudaMemsetAsync(s->dActiveCount.p + k, 0, sizeof(int), sk));
      // --- doIteration (gauss_newton_solver.cpp:224-280) ---
      recordPhaseStart(s, 0, sk);
      MB2_CUDA(launchSweep(sweep.slice(b0, count), true, sk, &f->lastSweep[1]));
      recordPhaseStop(s, sk);
      switch (P.kind) {
        case kSolveDense:
        case kSolveTilesKMajor:
        case kSolveTiles: // the normal equations in a launch of their own, then the factorisation
          recordPhaseStart(s, 1, sk);
          if (P.kind == kSolveTiles) MB2_CUDA(launchGramTiles(g, P.gramThreads, sk));
          else if ((rc = runJtJ(f, P.jtjMode, ns, c.H, ldH, hStride, s->dActive.p, sk, s->dGrad.p, ldG)) != MB2_OK) return rc;
          recordPhaseStop(s, sk);
          recordPhaseStart(s, 2, sk);
          if (P.kind == kSolveDense) MB2_CUDA(launchCholesky(c, P.denseNb, P.denseInSmem, sk));
          else MB2_CUDA(launchCholeskyScheduled(c, f->sched->dev, P.cholThreads, sk));
          break;
        case kSolveGramCholesky:
          recordPhaseStart(s, 2, sk);
          MB2_CUDA(launchGramCholesky(gc.slice(k, b0, count), f->sched->dev, f->sched->gcParams.get(), gt, s->inKernelProfile, sk));
          break;
        case kSolveQr: // the QR kernels read the Jacobian directly
          recordPhaseStart(s, 2, sk);
          MB2_CUDA(launchQrSolve(t.q, P.qrWidestChunk, sk));
          break;
        default:
          recordPhaseStart(s, 2, sk);
          MB2_CUDA(launchTrustRegionQr(t, sk));
      }
      recordPhaseStop(s, sk);
    }
    if (lineSearch) { // gauss_newton_solver.cpp:283-313 / subset_gauss_newton_solver.cpp:119-141
      MB2_CUDA(cudaMemcpyAsync(s->dThetaOrig.p, theta, size_t(B) * n * sizeof(float), cudaMemcpyDeviceToDevice, st));
      initLineSearchKernel<<<(B + 127) / 128, 128, 0, st>>>(B, s->dActive.p, s->dSearching.p, s->dScale.p);
      MB2_CUDA(cudaGetLastError());
      for (int k = 0; k < 10; ++k) {
        MB2_CUDA(launchTrialUpdate(B, s->dThetaOrig.p, n, s->dDelta.p, ns, f->dDeviceCols.p, s->dScale.p, theta, s->dSearching.p, st));
        recordPhaseStart(s, 3, st);
        MB2_CUDA(launchSweep(trial, false, st, &f->lastSweep[0]));
        recordPhaseStop(s, st);
        la.step = k;
        MB2_CUDA(launchLineSearchStep(la, st));
        s->kernelLaunches += 2;
      }
      MB2_CUDA(launchBookkeeping(B, step.state, st));
      s->kernelLaunches += 1;
    }
    // Instances can only stop once iteration >= minIterations (solver.cpp:113): poll the device counter from then on (every
    // kPollEvery-th iteration: converged instances cost nothing on the device, the poll costs a host round trip) so that a
    // converged batch does not run to maxIterations.
    if (it + 1 < maxIt && it >= minIt && (it - minIt) % kPollEvery == kPollEvery - 1) {
      if ((rc = join()) != MB2_OK) return rc;
      MB2_CUDA(cudaMemcpyAsync(s->hActiveCount, s->dActiveCount.p, size_t(S) * sizeof(int), cudaMemcpyDeviceToHost, st));
      MB2_CUDA(cudaStreamSynchronize(st));
      int stillActive = 0;
      for (int k = 0; k < S; ++k) stillActive += s->hActiveCount[k];
      if (stillActive == 0) break;
      if ((rc = fork()) != MB2_OK) return rc;
    }
  }
  if ((rc = join()) != MB2_OK) return rc; // (after a break the slices are idle: an empty join)
  finalizeKernel<<<B, 128, 0, st>>>(B, n, theta, s->dTheta0.p, s->dStatus.p);
  MB2_CUDA(cudaGetLastError());
  s->kernelLaunches += 2;
  return MB2_OK;
}

static void collectProfile(mb2_solver* s) {
  if (s->profiling && s->path.kind == kSolvePersistent && s->fusedStart) {
    float ms = 0.f;
    s->fusedMs = cudaEventElapsedTime(&ms, s->fusedStart, s->fusedStop) == cudaSuccess ? double(ms) : 0.0;
  }
  if (s->profiling) {
    for (int k = 0; k < 4; ++k) { s->phaseMs[k] = 0; s->phaseLaunches[k] = 0; }
    for (auto& e : s->events) {
      float ms = 0.f;
      if (cudaEventElapsedTime(&ms, e.start, e.stop) == cudaSuccess) { s->phaseMs[e.phase] += ms; s->phaseLaunches[e.phase]++; }
    }
  }
}

int mb2_solver_get_results(mb2_solver* s, double* errors, int32_t* iterations, int32_t* status) {
  MB2_CHECK(s != nullptr, "null solver");
  mb2_solver_function* f = s->fn;
  const int B = f->B;
  MB2_DEVICE_GUARD(f->ch->device);
  MB2_CUDA(cudaDeviceSynchronize());
  if (errors) MB2_CUDA(cudaMemcpy(errors, f->dErrors.p, size_t(B) * sizeof(double), cudaMemcpyDeviceToHost));
  std::vector<int32_t> its(B);
  MB2_CUDA(cudaMemcpy(its.data(), s->dIterations.p, size_t(B) * sizeof(int32_t), cudaMemcpyDeviceToHost));
  s->totalIterations = 0;
  for (int v : its) s->totalIterations += uint64_t(v);
  if (iterations) std::copy(its.begin(), its.end(), iterations);
  if (status) MB2_CUDA(cudaMemcpy(status, s->dStatus.p, size_t(B) * sizeof(int32_t), cudaMemcpyDeviceToHost));
  collectProfile(s);
  return MB2_OK;
}

int mb2_solver_solve_async(mb2_solver* s, float* params) {
  MB2_CHECK(s != nullptr && params != nullptr, "null argument");
  mb2_solver_function* f = s->fn;
  MB2_DEVICE_GUARD(f->ch->device);
  const size_t B = size_t(f->B);
  const size_t bytes = B * f->ch->host.numParams * sizeof(float);
  MB2_CUDA(s->dThetaStage.resize(B * f->ch->host.numParams));
  MB2_CUDA(cudaMemcpyAsync(s->dThetaStage.p, params, bytes, cudaMemcpyHostToDevice, f->stream));
  s->resultsStaged = false;
  int rc = mb2_solver_solve_device(s, s->dThetaStage.p, f->stream);
  if (rc != MB2_OK) return rc;
  MB2_CUDA(cudaMemcpyAsync(params, s->dThetaStage.p, bytes, cudaMemcpyDeviceToHost, f->stream));
  // the per-instance results follow the parameters on the same stream into pinned staging (one synchronisation in mb2_solver_wait)
  const size_t need = B * (sizeof(double) + 2 * sizeof(int32_t));
  if (s->hResultsBytes < need) {
    if (s->hResults) cudaFreeHost(s->hResults);
    s->hResults = nullptr;
    s->hResultsBytes = 0;
    MB2_CUDA(cudaMallocHost(reinterpret_cast<void**>(&s->hResults), need));
    s->hResultsBytes = need;
  }
  MB2_CUDA(cudaMemcpyAsync(s->hResults, f->dErrors.p, B * sizeof(double), cudaMemcpyDeviceToHost, f->stream));
  MB2_CUDA(cudaMemcpyAsync(s->hResults + B * sizeof(double), s->dIterations.p, B * sizeof(int32_t), cudaMemcpyDeviceToHost, f->stream));
  MB2_CUDA(cudaMemcpyAsync(s->hResults + B * (sizeof(double) + sizeof(int32_t)), s->dStatus.p, B * sizeof(int32_t), cudaMemcpyDeviceToHost, f->stream));
  s->resultsStaged = true;
  return MB2_OK;
}

int mb2_solver_wait(mb2_solver* s, double* errors, int32_t* iterations, int32_t* status) {
  MB2_CHECK(s != nullptr, "null solver");
  MB2_DEVICE_GUARD(s->fn->ch->device);
  MB2_CUDA(cudaStreamSynchronize(s->fn->stream));
  if (!s->resultsStaged) return mb2_solver_get_results(s, errors, iterations, status);
  const size_t B = size_t(s->fn->B);
  const int32_t* its = reinterpret_cast<const int32_t*>(s->hResults + B * sizeof(double));
  if (errors) std::memcpy(errors, s->hResults, B * sizeof(double));
  s->totalIterations = 0;
  for (size_t b = 0; b < B; ++b) s->totalIterations += uint64_t(its[b]);
  if (iterations) std::memcpy(iterations, its, B * sizeof(int32_t));
  if (status) std::memcpy(status, s->hResults + B * (sizeof(double) + sizeof(int32_t)), B * sizeof(int32_t));
  s->resultsStaged = false;
  collectProfile(s);
  return MB2_OK;
}

int mb2_solver_solve(mb2_solver* s, float* params, double* errors, int32_t* iterations, int32_t* status) {
  const int rc = mb2_solver_solve_async(s, params);
  if (rc != MB2_OK) return rc;
  return mb2_solver_wait(s, errors, iterations, status);
}

int mb2_solver_get_error_history(mb2_solver* s, double* history) {
  MB2_CHECK(s != nullptr && history != nullptr, "null argument");
  MB2_CHECK(s->opt.store_error_history && s->dHistory.p, "error history was not stored (set store_error_history)");
  MB2_CUDA(cudaMemcpy(history, s->dHistory.p, size_t(s->fn->B) * s->historyStride * sizeof(double), cudaMemcpyDeviceToHost));
  return MB2_OK;
}

int mb2_solver_get_counters(mb2_solver* s, uint64_t* totalIterations, uint64_t* kernelLaunches) {
  MB2_CHECK(s != nullptr, "null solver");
  if (totalIterations) *totalIterations = s->totalIterations;
  if (kernelLaunches) *kernelLaunches = s->kernelLaunches;
  return MB2_OK;
}

int mb2_solver_get_plan_stats(mb2_solver* s, int64_t stats[12]) {
  MB2_CHECK(s != nullptr && stats != nullptr, "null argument");
  const mb2_solver_function* f = s->fn;
  int64_t nnz = 0;
  for (const CellDesc& c : f->plan.cells) nnz += f->plan.units[c.unit].numRows;
  const bool tiles = f->planMode == 2 && f->sched;
  stats[0] = nnz;
  stats[1] = f->plan.numCols;
  stats[2] = f->ldJ;
  stats[3] = f->planMode == 0 ? int64_t(f->plan.enabledList.size()) : int64_t(f->plan.numCols);
  stats[4] = tiles ? f->sched->host.numTiles : 0;
  stats[5] = tiles ? f->sched->host.tileOps : 0;
  stats[6] = tiles ? f->sched->host.numLevels : 0;
  stats[7] = f->plan.numRows;
  const bool gram = tiles && f->planAlignRows;
  stats[8] = gram ? f->sched->gram.stride : 0;
  stats[9] = gram ? f->sched->gram.macs : 0;
  stats[10] = gram ? int64_t(f->sched->gram.pairA.size()) : 0;
  stats[11] = gram ? f->sched->fusedGroups : 0;
  return MB2_OK;
}

int mb2_solver_get_fused_profile(mb2_solver* s, int32_t* fused, int32_t* groups, double* kernelMs, uint64_t phaseCycles[12]) {
  MB2_CHECK(s != nullptr, "null solver");
  const bool persistent = s->path.kind == kSolvePersistent, gramChol = s->path.kind == kSolveGramCholesky;
  if (fused) *fused = persistent ? 1 : (gramChol ? 2 : 0);
  if (groups) *groups = persistent ? s->path.fused.groups : 0;
  if (kernelMs) *kernelMs = persistent ? s->fusedMs : (gramChol ? s->phaseMs[2] : 0.0);
  if (phaseCycles) {
    for (int k = 0; k < 12; ++k) phaseCycles[k] = 0;
    if ((persistent || gramChol) && s->profiling && s->dPhaseCycles.p) {
      MB2_DEVICE_GUARD(s->fn->ch->device);
      unsigned long long h[12];
      MB2_CUDA(cudaMemcpy(h, s->dPhaseCycles.p, sizeof(h), cudaMemcpyDeviceToHost));
      if (persistent) {
        for (int k = 0; k < 12; ++k) phaseCycles[k] = h[k];
      } else { // gramCholeskyKernel (block 0, summed over the iterations): prologue, gram, parked tiles, diag, panel, update, backward, finish
        phaseCycles[0] = h[0];
        for (int k = 1; k < 8; ++k) phaseCycles[4 + k] = h[k];
      }
    }
  }
  return MB2_OK;
}

int mb2_solver_function_get_sweep_launch(mb2_solver_function* f, int32_t jacobian, int64_t out[5]) {
  MB2_CHECK(f != nullptr && out != nullptr, "null argument");
  const SweepLaunch& l = f->lastSweep[jacobian ? 1 : 0];
  out[0] = l.stageTables;
  out[1] = l.warpsPerInstance;
  out[2] = l.groupsPerCta;
  out[3] = l.grid;
  out[4] = l.smemBytes;
  return MB2_OK;
}

namespace {
void instanceLaunchWords(const InstanceLaunchQuery& q, int64_t out[6]) {
  out[0] = q.launch.warpsPerInstance;
  out[1] = q.launch.groupsPerCta;
  out[2] = q.launch.threads;
  out[3] = q.grid;
  out[4] = q.launch.smemBytes;
  out[5] = q.launch.stagedPoints;
}
} // namespace

int mb2_character_get_instance_launch(const mb2_character* c, int32_t op, int32_t backward, int32_t batch, int32_t num_points, int64_t out[6]) {
  MB2_CHECK(c != nullptr && out != nullptr, "null argument");
  MB2_CHECK((op >= kInstanceOpModelSkeletonState && op <= kInstanceOpJointPositions) || op == kInstanceOpParameterLimits || op == kInstanceOpCollision,
            "instance launch: op must be 0, 1, 2, 3, 5 or 6");
  MB2_CHECK(op != kInstanceOpCollision || c->collisionDev != nullptr, "collision: the character has no collision geometry");
  MB2_CHECK(batch >= 0 && num_points >= 0, "instance launch: batch and num_points must not be negative");
  MB2_CHECK(op != kInstanceOpParameterLimits || c->limits.rejected.empty(), c->limits.rejected);
  MB2_DEVICE_GUARD(c->device);
  InstanceLaunchQuery q;
  const bool joint = op == kInstanceOpJointSkeletonState || op == kInstanceOpJointPositions;
  if (op == kInstanceOpCollision) {
    CollisionArgs a{};
    a.T = c->tables();
    a.L = c->collisionTables();
    a.batch = batch;
    MB2_CUDA(launchCollision(a, backward != 0, nullptr, &q));
  } else if (op == kInstanceOpParameterLimits) {
    ParameterLimitArgs a{};
    a.T = c->tables();
    a.L = c->limitTables();
    a.numChildren = int(c->host.children.size());
    a.batch = batch;
    MB2_CUDA(launchParameterLimits(a, backward != 0, nullptr, &q));
  } else if (op == kInstanceOpModelSkeletonState || op == kInstanceOpJointSkeletonState) {
    SkeletonStateArgs a{};
    a.T = c->tables();
    a.numChildren = int(c->host.children.size());
    a.batch = batch;
    a.fromJointParameters = joint;
    MB2_CUDA(launchSkeletonState(a, backward != 0, nullptr, &q));
  } else {
    PositionArgs a{};
    a.T = c->tables();
    a.numChildren = int(c->host.children.size());
    a.batch = batch;
    a.P.numPoints = num_points;
    a.fromJointParameters = joint;
    MB2_CUDA(queryPositionsLaunch(a, backward != 0, &q));
  }
  instanceLaunchWords(q, out);
  return MB2_OK;
}

int mb2_solver_function_get_input_gradient_launch(mb2_solver_function* f, int64_t out[6]) {
  MB2_CHECK(f != nullptr && out != nullptr, "null argument");
  MB2_DEVICE_GUARD(f->ch->device);
  InputGradientArgs a{};
  a.T = f->tables();
  a.batch = f->B;
  InstanceLaunchQuery q;
  MB2_CUDA(launchInputGradients(a, nullptr, &q));
  instanceLaunchWords(q, out);
  return MB2_OK;
}

int mb2_solver_get_solve_path(mb2_solver* s, int64_t out[16]) {
  MB2_CHECK(s != nullptr && out != nullptr, "null argument");
  solvePathWords(s->path, out);
  return MB2_OK;
}

int mb2_solver_get_phase_times(mb2_solver* s, double ms[4], uint64_t launches[4]) {
  MB2_CHECK(s != nullptr, "null solver");
  for (int k = 0; k < 4; ++k) {
    if (ms) ms[k] = s->phaseMs[k];
    if (launches) launches[k] = s->phaseLaunches[k];
  }
  return MB2_OK;
}

} // extern "C"
