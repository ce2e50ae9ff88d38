// sm_90a kernels for one Gauss-Newton iteration over a batch of IK instances.
//
//   K1  sweepKernel<true, W>      FK sweep + residual + Jacobian cells (strip layout or K-major matrix)  (skeleton_solver_function.cpp:200-261)
//   K4  sweepKernel<false, W>     FK sweep + error only (line search)                                    (skeleton_solver_function.cpp:64-83)
//   K2s gramTilesKernel           stored tiles of JtJ + lambda I and Jtr from the non-zero strips of J (mma.sync, three-term TF32 split)
//   K2' jtjSimtKernel             dense JtJ and Jtr, fp32 CUDA cores (solver_function.cpp:113-116): validation path / wide systems
//   K3  choleskyScheduledKernel   level-scheduled tile-sparse damped Cholesky + solves + theta -= delta + SolverT bookkeeping
//   K3' choleskyKernel<NB>        dense blocked LLT with Eigen's block structure and early exit (gauss_newton_solver.cpp:248-259, solver.cpp:89-122)
//   small kernels                 line search, bookkeeping, target scatter / quaternion normalisation
//
// The dense tensor-core JtJ (wgmma, register accumulators, TMA-fed) lives in ik_jtj_tc.cu; PTX wrappers in ik_ptx.cuh.
#include "ik_kernels.cuh"

#include <algorithm>
#include <cstdio>
#include <type_traits>

#include "ik_chol.cuh"
#include "ik_chol_sched.h"
#include "ik_jtj_tc.cuh"
#include "ik_ptx.cuh"
#include "ik_device.cuh"
#include "ik_jacobi.cuh"

namespace mb2 {

// ------------------------------------------------------------------------------------------------
// K1 / K4: one warp per IK instance. Joint state lives in shared memory (17 floats / joint, odd
// stride => conflict-free when lanes own different joints); the joint tree is swept level by level
// with lanes = joints of one depth level; then lanes = units (constraints), then lanes = Jacobian cells.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ double warpSum(double v) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

size_t sweepSmemPerInstance(const FunctionTables& T, int warpsPerInstance) {
  const size_t nPad = (T.numParams + 3) & ~3;
  // several warps per instance (large rigs): the joint parameters [7 J] are staged too (lanes = rows: the lanes are plentiful there)
  const size_t jp = warpsPerInstance > 1 ? size_t((T.numJoints * kParametersPerJoint + 1) & ~1) : 0;
  return sizeof(float) * (nPad + jp + size_t((T.numJoints * kJointStateStride + 1) & ~1) + size_t((T.recStride + 1) & ~1) + 4 + 2 * size_t(warpsPerInstance));
}

// The read-only tables (character + plan) are walked by dependent loads (cell -> unit -> contributions -> joint);
// from L2 each hop costs several hundred cycles, so a persistent CTA copies them into shared memory once (the lists and their visitors:
// ik_instance_launch.h).
// mode 1: every table; mode 2: everything except the two big ones, cells and contributions (large rigs: those are streamed through
// L1 / L2, one sequential record per lane and iteration, while the tables walked by dependent loads - character, units, error functions -
// still sit in shared memory)
template <class V, class F>
MB2_HD void sweepTableList(V& v, F& T, int mode) {
  characterTableList(v, T);
  v(T.efs, T.numEf); v(T.units, T.numUnits); v(T.limitData, T.numLimitData);
  if (mode == 1) { v(T.cells, T.numCells); v(T.contribs, T.numContribs); }
}
size_t sweepTableBytes(const FunctionTables& T, int mode) {
  if (mode == 0) return 0;
  TableBytes tables;
  sweepTableList(tables, T, mode);
  return tables.bytes;
}

// kStage (1 all tables, 2 all but cells / contributions, 0 none): the tables live in shared memory for the whole kernel. A template parameter rather than a run-time branch so that every
// table pointer is PROVABLY a shared-memory address: with `if (a.stageTables)` the pointers could be either and all 273 table loads
// of the kernel were generic LD instructions (address-space check on every hop of the dependent chains cell -> unit -> record ->
// contributions).
constexpr int kSweepMaxWarps = 24; // up to 24 warps per CTA (80 registers per thread on sm_90a)
template <bool kJacobian, int W, int kStage>
__global__ void __launch_bounds__(32 * kSweepMaxWarps) sweepKernel(const SweepArgs a) {
  extern __shared__ __align__(16) float smem[];
  FunctionTables T = a.T;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const WarpLanes<W> g = WarpLanes<W>::of(warp, lane); // a group of W warps works on one instance
  const int groupsPerCta = (blockDim.x >> 5) / W;
  const int nPad = (T.numParams + 3) & ~3;
  // (kJointStateStride is odd: an odd joint count gets one float of padding so that the doubles below stay 8-byte aligned)
  const int jpFloats = W > 1 ? ((T.numJoints * kParametersPerJoint + 1) & ~1) : 0;
  const int perGroup = nPad + jpFloats + ((T.numJoints * kJointStateStride + 1) & ~1) + ((T.recStride + 1) & ~1) + 4 + 2 * W;
  float* th = smem + size_t(g.group) * perGroup;
  float* jp = W > 1 ? th + nPad : nullptr;
  float* js = th + nPad + jpFloats;
  float* rec = js + ((T.numJoints * kJointStateStride + 1) & ~1);
  double* errSlots = reinterpret_cast<double*>(rec + ((T.recStride + 1) & ~1)); // W partial sums (8-byte aligned: every preceding size is even)
  if constexpr (kStage != 0) {
    TableStager stager{reinterpret_cast<uint32_t*>(smem + ((size_t(groupsPerCta) * perGroup + 3) & ~size_t(3)))};
    sweepTableList(stager, T, kStage);
    __syncthreads();
  }

  for (int b = blockIdx.x * groupsPerCta + g.group; b < a.batch; b += gridDim.x * groupsPerCta) {
    if (a.active != nullptr && a.active[b] == 0) continue; // (the whole group skips together)
    const float* theta = a.theta + size_t(b) * a.ldTheta;
    for (int i = g.lane; i < T.numParams; i += g.size) th[i] = theta[i];
    g.sync();
    if (W == 1) { // touch the next instance's parameters now: by the time this one is done they sit in L1 / L2 (one warp = one 880-byte row)
      const int bn = b + gridDim.x * groupsPerCta;
      if (bn < a.batch) { const float* tn = a.theta + size_t(bn) * a.ldTheta; for (int i = g.lane * 8; i < T.numParams; i += g.size * 8) asm volatile("prefetch.global.L2 [%0];" ::"l"(tn + i)); }
    }
    // SkeletonState::set (fkPasses): one warp per instance takes each joint's seven parameters straight from theta (three rounds of
    // lanes = joints, each walking its seven rows); several warps per instance stage them first with lanes = rows
    if constexpr (W > 1) {
      for (int row = g.lane; row < T.numJoints * kParametersPerJoint; row += g.size) jp[row] = jointParameterRow(T, row, th);
      g.sync();
    }
    fkPasses<kJacobian, (W > 1)>(g, T, W > 1 ? jp : th, js);
    if constexpr (kJacobian) g.sync();
    if (a.stateOut != nullptr) {
      float* so = a.stateOut + size_t(b) * T.numJoints * 8;
      for (int i = g.lane; i < T.numJoints * 8; i += g.size) so[i] = js[(i >> 3) * kJointStateStride + (i & 7)];
    }
    const float* targets = a.targets + size_t(b) * T.targetStride;
    const float* cw = a.cweights + (T.weightsPerInstance ? size_t(b) * T.numWeights : 0);
    float* J = kJacobian ? a.jacobian + size_t(b) * T.jacobianStride : nullptr;
    // the residual is the last column of the device matrix, or follows the strips
    float* residual = kJacobian ? J + (T.stripMode ? size_t(T.residOff) : size_t(T.numCols) * T.ldJ) : nullptr;
    double err = 0.0;
    for (int u = g.lane; u < T.numUnits; u += g.size) err += (double)evalUnit<kJacobian>(T, u, th, jp, js, targets, cw, rec, residual);
    err = warpSum(err);
    if (W > 1 && lane == 0) errSlots[warp % W] = err;
    g.sync();
    if (kJacobian)
      for (int c = g.lane; c < T.numCells; c += g.size) jacobianCell(T, c, js, rec, targets, J);
    if (g.lane == 0) {
      if (W > 1) { err = 0.0; for (int w = 0; w < W; ++w) err += errSlots[w]; } // fixed order: deterministic
      // getError() rounds through float (skeleton_solver_function.cpp:82); the Jacobian pass keeps double
      a.errors[b] = kJacobian ? err : (double)(float)err;
    }
    g.sync();
  }
}

static int g_numSms = 0;
static int g_maxSmemOptin = 0;
static int g_maxSmemPerSm = 0;

cudaError_t launchSweep(const SweepArgs& a0, bool jacobian, cudaStream_t stream, SweepLaunch* out) {
  SweepArgs a = a0;
  if (out) *out = SweepLaunch{}; // a rejected configuration leaves an all-zero record
  const size_t budget = size_t(g_maxSmemOptin);
  // Persistent CTAs. As many instances in flight as shared memory holds next to the staged tables: all of them when they fit with at
  // least two instances, else all but the cell / contribution records (large rigs), else none. One warp per instance, up to
  // kSweepMaxWarps; when fewer than 16 instances fit, several warps share one instance (up to kSweepMaxWarps warps per CTA).
  const size_t per1 = sweepSmemPerInstance(a.T, 8);
  a.stageTables = (2 * per1 + sweepTableBytes(a.T, 1) + 16 <= budget) ? 1 : (2 * per1 + sweepTableBytes(a.T, 2) + 16 <= budget) ? 2 : 0;
  const size_t tableBytes = sweepTableBytes(a.T, a.stageTables) + 16;
  int groups = int((budget - tableBytes) / per1);
  if (groups < 1) return cudaErrorInvalidConfiguration;
  const int groupsOneWarp = int((budget - tableBytes) / sweepSmemPerInstance(a.T, 1)); // (no joint-parameter array)
  int W = 1;
  if (groupsOneWarp >= 16) {
    // The instances of an SM are dealt to its warps round by round, and from about a dozen warps on the kernel is throughput bound:
    // the time is rounds x warps, i.e. the padded instance count. Pick the warp count that wastes the fewest slots over the SMs of
    // this device (rounds x warps x SMs closest above the batch); more warps than kSweepMaxWarps spill registers.
    const int sms = std::max(g_numSms, 1);
    const int maxG = std::min(groupsOneWarp, kSweepMaxWarps), minG = std::min(12, maxG);
    const int planned = a.planBatch > 0 ? a.planBatch : a.batch;
    long best = -1;
    if (planned < sms * minG) { groups = std::max(1, (planned + sms - 1) / sms); best = 0; } // a small batch: spread it over the SMs
    for (int gcand = maxG; gcand >= minG && best != 0; --gcand) {
      const long rounds = (planned + long(sms) * gcand - 1) / (long(sms) * gcand);
      if (best < 0 || rounds * gcand < best) { best = rounds * gcand; groups = gcand; }
    }
  } else {
    if (groups > 15) groups = 15; // named barriers 1..15
    while (W < 8 && groups * W * 2 <= kSweepMaxWarps) W *= 2; // these instances wait on L1 / L2 and on each other's barriers: as many warps as fit
  }
  a.warpsPerInstance = W;
  const int warps = groups * W;
  const size_t per = sweepSmemPerInstance(a.T, W);
  const size_t smem = per * groups + tableBytes;
  if (smem > budget) return cudaErrorInvalidConfiguration;
  const int ctasNeeded = (a.batch + groups - 1) / groups;
  int ctasPerSm = (int)((size_t(g_maxSmemPerSm)) / (smem + 1024));
  if (ctasPerSm < 1) ctasPerSm = 1;
  if (ctasPerSm * warps > 32) ctasPerSm = 32 / warps > 0 ? 32 / warps : 1;
  int grid = g_numSms * ctasPerSm;
  if (grid > ctasNeeded) grid = ctasNeeded;
  if (grid < 1) grid = 1;
  if (out) *out = SweepLaunch{a.stageTables, W, groups, grid, int64_t(smem)};
  auto launch = [&](auto kernel) -> cudaError_t {
    const cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem));
    if (e != cudaSuccess) return e;
    kernel<<<grid, warps * 32, smem, stream>>>(a);
    return cudaGetLastError();
  };
  auto pick = [&](auto jac, auto staged) -> cudaError_t {
    constexpr bool kJ = decltype(jac)::value;
    constexpr int kS = decltype(staged)::value;
    switch (W) {
      case 1: return launch(sweepKernel<kJ, 1, kS>);
      case 2: return launch(sweepKernel<kJ, 2, kS>);
      case 4: return launch(sweepKernel<kJ, 4, kS>);
      default: return launch(sweepKernel<kJ, 8, kS>);
    }
  };
  auto pickStage = [&](auto jac) -> cudaError_t {
    switch (a.stageTables) {
      case 1: return pick(jac, std::integral_constant<int, 1>{});
      case 2: return pick(jac, std::integral_constant<int, 2>{});
      default: return pick(jac, std::integral_constant<int, 0>{});
    }
  };
  return jacobian ? pickStage(std::true_type{}) : pickStage(std::false_type{});
}

// ------------------------------------------------------------------------------------------------
// Skeleton state of a batch of model parameters, and its backward (ik_device.cuh skelGrad*).
// The per-instance frame, shared with the positions, limits, collision and input-gradient kernels: a persistent grid sized by
// launchInstanceGroups, one group of W warps per instance (WarpLanes<W>) with skeletonStateFrame's floats of shared memory, the kernel's
// table list staged once per CTA after the groups (TableStager), then per instance the pass functions of ik_device.cuh, which the CPU
// emulators run too.
//   forward:   fkPasses from theta, [J][8] out
//   backward:  fkPasses with the DOF axes, then skelGradPasses: lanes = joints seed their 11 subtree sums from G, levels from the
//              deepest up fold in their children, lanes = joint-parameter rows, lanes = model parameters over the CSC ParameterTransform.
// kJoint (joint_parameters_to_skeleton_state): the input is the joint parameters [7 J], staged where theta is staged otherwise; the
// backward writes the joint-parameter gradient straight out and stops before the ParameterTransform.
// Every output element is written by one lane in a fixed order: no atomics, the result does not depend on the launch shape.
// The frame's size, the staged tables and the choice of W: ik_instance_launch.h.
// ------------------------------------------------------------------------------------------------

template <bool kBackward, int W, bool kJoint>
__global__ void __launch_bounds__(32 * kSkelMaxWarps) skeletonStateKernel(const SkeletonStateArgs a) {
  extern __shared__ __align__(16) float smem[];
  CharacterTables T = a.T;
  SkeletonTables S = a.S;
  const WarpLanes<W> g = WarpLanes<W>::of(threadIdx.x >> 5, threadIdx.x & 31);
  const int groupsPerCta = (blockDim.x >> 5) / W;
  const int J = T.numJoints, n = T.numParams;
  const int inN = kJoint ? J * kParametersPerJoint : n; // floats per instance of the input
  const int thF = int(skelAligned(inN)), jsF = int(skelAligned(size_t(J) * kJointStateStride));
  const int accF = kBackward ? int(skelAligned(size_t(J) * kSkelAccStride)) : 0;
  const int perGroup = int(skeletonStateFrame(J, n, kBackward, kJoint).floats);
  float* th = smem + size_t(g.group) * perGroup;
  float* js = th + thF;
  float* acc = js + jsF;
  float* gjp = acc + accF;
  {
    TableStager stager{reinterpret_cast<uint32_t*>(smem + size_t(groupsPerCta) * perGroup)};
    skeletonTableList(stager, T, S, a.numChildren, kBackward, kBackward && !kJoint);
    __syncthreads();
  }
  for (int b = blockIdx.x * groupsPerCta + g.group; b < a.batch; b += gridDim.x * groupsPerCta) {
    const float* theta = a.theta + size_t(b) * inN;
    for (int i = g.lane; i < inN; i += g.size) th[i] = theta[i];
    g.sync();
    fkPasses<kBackward, kJoint>(g, T, th, js);
    if constexpr (!kBackward) {
      float* so = a.out + size_t(b) * J * 8;
      for (int i = g.lane; i < J * 8; i += g.size) so[i] = js[(i >> 3) * kJointStateStride + (i & 7)];
    } else if constexpr (kJoint) {
      skelGradPasses(g, T, S, js, a.gradState + size_t(b) * J * 8, acc, a.out + size_t(b) * inN, nullptr);
    } else {
      skelGradPasses(g, T, S, js, a.gradState + size_t(b) * J * 8, acc, gjp, a.out + size_t(b) * n);
    }
    g.sync(); // the next instance overwrites th / js / gjp
  }
}

namespace {
// Grid of a persistent kernel: what the SMs hold at once, capped by the work.
template <class K>
cudaError_t persistentGrid(K kernel, int threads, size_t smem, long work, int* grid) {
  if (smem > size_t(g_maxSmemOptin)) return cudaErrorInvalidConfiguration;
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem));
  if (e != cudaSuccess) return e;
  int perSm = 0;
  e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&perSm, kernel, threads, smem);
  if (e != cudaSuccess) return e;
  *grid = int(std::max(1L, std::min(long(std::max(g_numSms, 1)) * std::max(perSm, 1), work)));
  return cudaSuccess;
}

// f(std::true_type) or f(std::false_type): a run-time flag as a template argument
template <class F>
auto withFlag(bool flag, F&& f) { return flag ? f(std::true_type{}) : f(std::false_type{}); }

// A kernel in the per-instance frame, launched as planInstanceOp plans it (ik_instance_launch.cpp): kernelFor(W, plan) is its
// instantiation for the planned W (std::integral_constant<int, W>) and the plan's other choices. With `query`, the launch is reported
// there and nothing is enqueued.
template <class Args, class KernelFor>
cudaError_t launchInstanceGroups(const Args& a, int numChildren, int op, bool backward, int numPoints, cudaStream_t stream, InstanceLaunchQuery* query,
                                 bool limitsFk, KernelFor&& kernelFor) {
  if (query) *query = InstanceLaunchQuery{};
  if (a.batch <= 0) return cudaSuccess;
  const InstanceLaunch l = planInstanceOp(a.T, numChildren, op, backward, numPoints, a.batch, size_t(g_maxSmemOptin), g_numSms, limitsFk);
  if (l.warpsPerInstance == 0) return cudaErrorInvalidConfiguration; // not even one instance fits next to the tables
  const int W = l.warpsPerInstance;
  void (*const kernel)(Args) = W == 1 ? kernelFor(std::integral_constant<int, 1>{}, l) : W == 2 ? kernelFor(std::integral_constant<int, 2>{}, l)
                             : W == 4 ? kernelFor(std::integral_constant<int, 4>{}, l) : kernelFor(std::integral_constant<int, 8>{}, l);
  int grid = 0;
  const cudaError_t e = persistentGrid(kernel, l.threads, size_t(l.smemBytes), (long(a.batch) + l.groupsPerCta - 1) / l.groupsPerCta, &grid);
  if (e != cudaSuccess) return e;
  if (query) {
    *query = InstanceLaunchQuery{l, grid};
    return cudaSuccess;
  }
  kernel<<<grid, l.threads, size_t(l.smemBytes), stream>>>(a);
  return cudaGetLastError();
}
} // namespace

cudaError_t launchSkeletonState(const SkeletonStateArgs& a, bool backward, cudaStream_t stream, InstanceLaunchQuery* query) {
  const bool joint = a.fromJointParameters != 0;
  const int op = joint ? kInstanceOpJointSkeletonState : kInstanceOpModelSkeletonState;
  return launchInstanceGroups(a, a.numChildren, op, backward, 0, stream, query, false, [&](auto W, const InstanceLaunch&) {
    return withFlag(backward, [&](auto kB) { return withFlag(joint, [&](auto kJ) { return skeletonStateKernel<kB, W, kJ>; }); });
  });
}

// ------------------------------------------------------------------------------------------------
// Joint parameters <-> skeleton states, one element per thread (ik_device.cuh jointOpElement): flat grid-stride kernels over
// (instance, row), (instance, parameter) or (instance, joint). The character tables are read from global memory: they are shared by the
// batch and stay in L1 / L2. Each output element is written by one thread, so an instance gets the same bits in any batch.
// ------------------------------------------------------------------------------------------------
constexpr int kJointOpThreads = 256;
constexpr int kJointOpCtasPerSm = 8;

template <int kOp, bool kBackward>
__device__ __forceinline__ void jointOpGrid(const JointOpArgs& a) {
  const long items = long(a.batch) * jointOpItems<kOp, kBackward>(a.T);
  for (long i = blockIdx.x * long(blockDim.x) + threadIdx.x; i < items; i += long(gridDim.x) * blockDim.x)
    jointOpElement<kOp, kBackward>(a.T, a.S, i, a.in, a.grad, a.out);
}
__global__ void __launch_bounds__(kJointOpThreads) parameterTransformKernel(const JointOpArgs a) { jointOpGrid<kJointOpParameterTransform, false>(a); }
__global__ void __launch_bounds__(kJointOpThreads) parameterTransformBackwardKernel(const JointOpArgs a) { jointOpGrid<kJointOpParameterTransform, true>(a); }
__global__ void __launch_bounds__(kJointOpThreads) localStateKernel(const JointOpArgs a) { jointOpGrid<kJointOpLocalState, false>(a); }
__global__ void __launch_bounds__(kJointOpThreads) localStateBackwardKernel(const JointOpArgs a) { jointOpGrid<kJointOpLocalState, true>(a); }
__global__ void __launch_bounds__(kJointOpThreads) localToJointParametersKernel(const JointOpArgs a) { jointOpGrid<kJointOpFromLocal, false>(a); }
__global__ void __launch_bounds__(kJointOpThreads) localToJointParametersBackwardKernel(const JointOpArgs a) { jointOpGrid<kJointOpFromLocal, true>(a); }
__global__ void __launch_bounds__(kJointOpThreads) worldToJointParametersKernel(const JointOpArgs a) { jointOpGrid<kJointOpFromWorld, false>(a); }
__global__ void __launch_bounds__(kJointOpThreads) worldToJointParametersBackwardKernel(const JointOpArgs a) { jointOpGrid<kJointOpFromWorld, true>(a); }
__global__ void __launch_bounds__(kJointOpThreads) inverseParameterTransformKernel(const JointOpArgs a) {
  jointOpGrid<kJointOpInverseParameterTransform, false>(a);
}
__global__ void __launch_bounds__(kJointOpThreads) inverseParameterTransformBackwardKernel(const JointOpArgs a) {
  jointOpGrid<kJointOpInverseParameterTransform, true>(a);
}
__global__ void __launch_bounds__(kJointOpThreads) clampParametersKernel(const JointOpArgs a) { jointOpGrid<kJointOpClampParameters, false>(a); }
__global__ void __launch_bounds__(kJointOpThreads) clampParametersBackwardKernel(const JointOpArgs a) { jointOpGrid<kJointOpClampParameters, true>(a); }

cudaError_t launchJointOp(const JointOpArgs& a, JointOp op, bool backward, cudaStream_t stream) {
  using K = void (*)(JointOpArgs);
  static const K kernels[6][2] = {{parameterTransformKernel, parameterTransformBackwardKernel}, {localStateKernel, localStateBackwardKernel},
                                  {localToJointParametersKernel, localToJointParametersBackwardKernel},
                                  {worldToJointParametersKernel, worldToJointParametersBackwardKernel},
                                  {inverseParameterTransformKernel, inverseParameterTransformBackwardKernel},
                                  {clampParametersKernel, clampParametersBackwardKernel}};
  if (a.batch <= 0) return cudaSuccess;
  const long rows = long(a.T.numJoints) * kParametersPerJoint;
  const long per = op == kJointOpParameterTransform          ? (backward ? a.T.numParams : rows)
                   : op == kJointOpInverseParameterTransform ? (backward ? rows : a.T.numParams)
                   : op == kJointOpClampParameters           ? a.T.numParams
                                                             : a.T.numJoints;
  const long items = long(a.batch) * per;
  if (items == 0) return cudaSuccess;
  const int grid = int(std::min<long>((items + kJointOpThreads - 1) / kJointOpThreads, long(std::max(g_numSms, 1)) * kJointOpCtasPerSm));
  kernels[op][backward]<<<grid, kJointOpThreads, 0, stream>>>(a);
  return cudaGetLastError();
}

// The per-instance scratch of the skinning, blend-shape and normals backward passes, of the closest-point refit and of the point-cloud
// tree build: at most kSliceScratchBudget bytes at once, the instances run in slices that fit (at least one instance each). No
// instance's result depends on the slice it falls in.
constexpr size_t kSliceScratchBudget = size_t(256) << 20;

namespace {
// One stream-ordered allocation of slice x perInstance bytes, then body(scratch, slice, b0, nb) for the instances b0 .. b0 + nb of each
// slice in order; nb < slice for the last one. Returns the first error.
template <class Body>
cudaError_t forEachInstanceSlice(int batch, size_t perInstance, cudaStream_t stream, Body body) {
  const int slice = int(std::max<size_t>(1, std::min<size_t>(size_t(batch), kSliceScratchBudget / perInstance)));
  float* scratch = nullptr;
  cudaError_t e = cudaMallocAsync(reinterpret_cast<void**>(&scratch), perInstance * slice, stream);
  if (e != cudaSuccess) return e;
  for (int b0 = 0; e == cudaSuccess && b0 < batch; b0 += slice) e = body(scratch, slice, b0, std::min(slice, batch - b0));
  const cudaError_t f = cudaFreeAsync(scratch, stream);
  return e != cudaSuccess ? e : f;
}
} // namespace

// ------------------------------------------------------------------------------------------------
// Linear-blend skinning of a batch (ik_device.cuh skin*), three kernels. The skin tables are shared by the batch and stay in L2.
//   skinVertexKernel<kMode>  a persistent grid of work items (instances, vertex range): per instance the CTA writes the J skinning
//                            transforms M_j = T_j o IBP_j to shared memory, then lanes = vertices blend. kMode 0: points [B][V][3];
//                            1: rest-point gradient per instance; 2: rest-point gradient summed over a fixed chunk of instances, in
//                            instance order, into one row of bounded scratch (the chunks are summed in order by rowGroupSumKernel).
//   skinStatePartialKernel   one warp per (instance, segment of a joint's influence list): lanes = influences, then a butterfly sum
//                            of the 12 floats (a_j, E_j) to scratch.
//   skinStateFinishKernel    lanes = (instance, joint): the joint's segments summed in order, then skinStateGradient.
// No atomics: every output element is summed in a fixed order that depends on neither the batch size nor the launch shape.
// ------------------------------------------------------------------------------------------------
constexpr int kSkinThreads = 256;
constexpr int kSkinVertsPerThread = 4;                              // kMode 2 keeps their sums in registers
constexpr int kSkinChunkVerts = kSkinThreads * kSkinVertsPerThread; // vertex range of a kMode 2 work item

template <int kMode>
__global__ void __launch_bounds__(kSkinThreads) skinVertexKernel(const SkinArgs a, int perChunk, int numChunks, int vSplit, int vLen, float* out) {
  extern __shared__ __align__(16) float M[]; // [J][12]
  const SkinTables S = a.S;
  const int V = S.numVertices, J = a.numJoints;
  const long items = long(numChunks) * vSplit;
  for (long it = blockIdx.x; it < items; it += gridDim.x) {
    const int c = int(it / vSplit), v0 = int(it % vSplit) * vLen, v1 = min(V, v0 + vLen);
    F3 acc[kSkinVertsPerThread];
#pragma unroll
    for (int k = 0; k < kSkinVertsPerThread; ++k) acc[k] = f3(0.f, 0.f, 0.f);
    const int b1 = min(a.batch, (c + 1) * perChunk);
    for (int b = c * perChunk; b < b1; ++b) {
      __syncthreads(); // the previous instance's readers of M are done
      for (int j = threadIdx.x; j < J; j += blockDim.x)
        skinTransform(a.skelState + (size_t(b) * J + j) * 8, S.inverseBindPose + j * kSkinIbpStride, M + j * kSkinIbpStride);
      __syncthreads();
      const float* x = a.restPoints + (a.restBatched ? size_t(b) * V * 3 : 0);
      const size_t row = size_t(b) * V * 3;
      if constexpr (kMode == 0) {
        for (int v = v0 + threadIdx.x; v < v1; v += blockDim.x) {
          const F3 p = skinBlend(S, M, v, ld3(x + 3 * v));
          float* o = a.points + row + 3 * size_t(v);
          o[0] = p.x; o[1] = p.y; o[2] = p.z;
        }
      } else if constexpr (kMode == 1) {
        for (int v = v0 + threadIdx.x; v < v1; v += blockDim.x) {
          const F3 r = skinRestGradient(S, M, v, ld3(a.gradPoints + row + 3 * size_t(v)));
          float* o = out + row + 3 * size_t(v);
          o[0] = r.x; o[1] = r.y; o[2] = r.z;
        }
      } else {
#pragma unroll
        for (int k = 0; k < kSkinVertsPerThread; ++k) {
          const int v = v0 + threadIdx.x + k * kSkinThreads;
          if (v < v1) acc[k] = acc[k] + skinRestGradient(S, M, v, ld3(a.gradPoints + row + 3 * size_t(v)));
        }
      }
    }
    if constexpr (kMode == 2) {
#pragma unroll
      for (int k = 0; k < kSkinVertsPerThread; ++k) {
        const int v = v0 + threadIdx.x + k * kSkinThreads;
        if (v < v1) {
          float* o = out + size_t(c) * V * 3 + 3 * size_t(v);
          o[0] = acc[k].x; o[1] = acc[k].y; o[2] = acc[k].z;
        }
      }
    }
  }
}

// rows [numRows][n] summed over groups of rowsPerGroup consecutive rows, each group in row order, into out [groups][n]: the batch sums of
// a shared input's gradient (batchSumChunk), per chunk and then over the chunks
__global__ void rowGroupSumKernel(const float* rows, int numRows, int rowsPerGroup, size_t n, float* out) {
  const size_t total = size_t((numRows + rowsPerGroup - 1) / rowsPerGroup) * n;
  for (size_t i = size_t(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += size_t(gridDim.x) * blockDim.x) {
    const size_t r0 = i / n * rowsPerGroup, k = i % n, r1 = min(size_t(numRows), r0 + rowsPerGroup);
    float s = rows[r0 * n + k];
    for (size_t r = r0 + 1; r < r1; ++r) s += rows[r * n + k];
    out[i] = s;
  }
}
namespace {
cudaError_t launchRowGroupSum(const float* rows, int numRows, int rowsPerGroup, size_t n, float* out, cudaStream_t stream) {
  const size_t total = size_t((numRows + rowsPerGroup - 1) / rowsPerGroup) * n;
  rowGroupSumKernel<<<unsigned(std::min<size_t>((total + kSkinThreads - 1) / kSkinThreads, 4096)), kSkinThreads, 0, stream>>>(rows, numRows, rowsPerGroup, n, out);
  return cudaGetLastError();
}
} // namespace

__global__ void __launch_bounds__(kSkinThreads) skinStatePartialKernel(const SkinArgs a, int b0, int nb, float* partial) {
  const SkinTables S = a.S;
  const int lane = threadIdx.x & 31, V = S.numVertices, numSeg = S.numSegments;
  const long warps = long(gridDim.x) * (blockDim.x >> 5);
  for (long it = long(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5); it < long(nb) * numSeg; it += warps) {
    const int b = b0 + int(it / numSeg), s = int(it % numSeg);
    const float* ibp = S.inverseBindPose + S.segJoint[s] * kSkinIbpStride;
    const float* x = a.restPoints + (a.restBatched ? size_t(b) * V * 3 : 0);
    const float* g = a.gradPoints + size_t(b) * V * 3;
    float acc[kSkinAccFloats];
#pragma unroll
    for (int r = 0; r < kSkinAccFloats; ++r) acc[r] = 0.f;
    for (int k = S.segStart[s] + lane; k < S.segStart[s + 1]; k += 32) {
      const int v = S.infVertex[k];
      skinAccumulate(ibp, ld3(x + 3 * v), ld3(g + 3 * v), S.infWeight[k], acc);
    }
    float mine = 0.f;
#pragma unroll
    for (int r = 0; r < kSkinAccFloats; ++r) {
      float t = acc[r];
      for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o); // every lane ends with the same bits
      if (lane == r) mine = t;
    }
    if (lane < kSkinAccFloats) partial[size_t(it) * kSkinAccFloats + lane] = mine;
  }
}

__global__ void skinStateFinishKernel(const SkinArgs a, int b0, int nb, const float* partial) {
  const SkinTables S = a.S;
  const int J = a.numJoints;
  for (long it = long(blockIdx.x) * blockDim.x + threadIdx.x; it < long(nb) * J; it += long(gridDim.x) * blockDim.x) {
    const int bl = int(it / J), j = int(it % J);
    float acc[kSkinAccFloats];
#pragma unroll
    for (int r = 0; r < kSkinAccFloats; ++r) acc[r] = 0.f;
    for (int s = S.jointSegStart[j]; s < S.jointSegStart[j + 1]; ++s) {
      const float* p = partial + (size_t(bl) * S.numSegments + s) * kSkinAccFloats;
#pragma unroll
      for (int r = 0; r < kSkinAccFloats; ++r) acc[r] += p[r];
    }
    const size_t at = (size_t(b0 + bl) * J + j) * 8;
    skinStateGradient(acc, a.skelState + at, a.gradState + at);
  }
}

namespace {
// kMode 0 / 1: one work item per instance when the batch fills the grid, else each instance's vertices split over several
template <int kMode>
cudaError_t launchSkinPerInstance(const SkinArgs& a, float* out, cudaStream_t stream) {
  const size_t smem = size_t(a.numJoints) * kSkinIbpStride * sizeof(float);
  const int V = a.S.numVertices;
  int slots = 0;
  cudaError_t e = persistentGrid(skinVertexKernel<kMode>, kSkinThreads, smem, 1L << 30, &slots);
  if (e != cudaSuccess) return e;
  const int vSplit = a.batch >= slots ? 1 : std::min((slots + a.batch - 1) / a.batch, (V + kSkinThreads - 1) / kSkinThreads);
  const int vLen = (V + vSplit - 1) / vSplit;
  const int grid = int(std::min(long(slots), long(a.batch) * vSplit));
  skinVertexKernel<kMode><<<grid, kSkinThreads, smem, stream>>>(a, 1, a.batch, vSplit, vLen, out);
  return cudaGetLastError();
}
} // namespace

cudaError_t launchSkinPoints(const SkinArgs& a, cudaStream_t stream) {
  if (a.batch <= 0) return cudaSuccess;
  return launchSkinPerInstance<0>(a, nullptr, stream);
}

cudaError_t launchSkinPointsBackward(const SkinArgs& a, cudaStream_t stream) {
  if (a.batch <= 0) return cudaSuccess;
  const int V = a.S.numVertices, J = a.numJoints;
  cudaError_t e = cudaSuccess;
  if (a.gradState != nullptr && a.S.numSegments == 0) { // no influences at all: the gradient is zero
    e = cudaMemsetAsync(a.gradState, 0, size_t(a.batch) * J * 8 * sizeof(float), stream);
  } else if (a.gradState != nullptr) {
    e = forEachInstanceSlice(a.batch, size_t(a.S.numSegments) * kSkinAccFloats * sizeof(float), stream, [&](float* partial, int slice, int b0, int nb) {
      // grids sized for a whole slice, the last one included
      int g1 = 0, g2 = 0;
      cudaError_t r = persistentGrid(skinStatePartialKernel, kSkinThreads, 0, (long(slice) * a.S.numSegments + 7) / 8, &g1);
      if (r == cudaSuccess) r = persistentGrid(skinStateFinishKernel, kSkinThreads, 0, (long(slice) * J + kSkinThreads - 1) / kSkinThreads, &g2);
      if (r != cudaSuccess) return r;
      skinStatePartialKernel<<<g1, kSkinThreads, 0, stream>>>(a, b0, nb, partial);
      skinStateFinishKernel<<<g2, kSkinThreads, 0, stream>>>(a, b0, nb, partial);
      return cudaGetLastError();
    });
  }
  if (e != cudaSuccess || a.gradRest == nullptr) return e;
  if (a.restBatched) return launchSkinPerInstance<1>(a, a.gradRest, stream);
  // shared rest points: the batch sum over fixed chunks of instances (the chunking depends on the batch size only)
  const int perChunk = batchSumChunk(a.batch);
  const int numChunks = (a.batch + perChunk - 1) / perChunk;
  const int vSplit = (V + kSkinChunkVerts - 1) / kSkinChunkVerts;
  const size_t n = size_t(V) * 3, smem = size_t(J) * kSkinIbpStride * sizeof(float);
  float* partial = a.gradRest;
  if (numChunks > 1) {
    e = cudaMallocAsync(reinterpret_cast<void**>(&partial), n * numChunks * sizeof(float), stream);
    if (e != cudaSuccess) return e;
  }
  int grid = 0;
  e = persistentGrid(skinVertexKernel<2>, kSkinThreads, smem, long(numChunks) * vSplit, &grid);
  if (e == cudaSuccess) {
    skinVertexKernel<2><<<grid, kSkinThreads, smem, stream>>>(a, perChunk, numChunks, vSplit, kSkinChunkVerts, partial);
    e = cudaGetLastError();
  }
  if (numChunks > 1) {
    if (e == cudaSuccess) {
      e = launchRowGroupSum(partial, numChunks, numChunks, n, a.gradRest, stream);
    }
    const cudaError_t f = cudaFreeAsync(partial, stream);
    if (e == cudaSuccess) e = f;
  }
  return e;
}

// ------------------------------------------------------------------------------------------------
// Positions of points fixed in joints' frames (ik_device.cuh positionPasses / positionGradPasses), in the per-instance frame of
// skeletonStateKernel: its shared memory per instance, its tables and its launch (launchInstanceGroups), then lanes = points. The point
// tables (each point's joint; backward: the points by joint) follow the character tables in shared memory when staging them costs no
// instance per CTA, else they are read from global memory.
//   forward:   fkPasses, then lanes = points: p = t + rot(q, s off), [N][3] out
//   backward:  fkPasses with the DOF axes, then lanes = points write the per-instance offset gradient s rot(conj(q), g), and lanes =
//              joints seed their subtree sums from their own points in index order; then the tail of skelGradPasses.
// Shared offsets: their gradient is the batch sum of the per-instance rows, per chunk of batchSumChunk(B) instances in order and then
// over the chunks in order (rowGroupSumKernel). The rows of a slice of whole chunks go to bounded scratch. No atomics, and no result
// depends on the slicing or the launch shape.
// ------------------------------------------------------------------------------------------------
// kStagePoints: a template parameter rather than a run-time branch, so that the staged point tables are provably shared-memory addresses
template <bool kBackward, int W, bool kJoint, bool kStagePoints>
__global__ void __launch_bounds__(32 * kSkelMaxWarps, 1) positionsKernel(const PositionArgs a) {
  extern __shared__ __align__(16) float smem[];
  CharacterTables T = a.T;
  SkeletonTables S = a.S;
  PointTables P = a.P;
  const WarpLanes<W> g = WarpLanes<W>::of(threadIdx.x >> 5, threadIdx.x & 31);
  const int groupsPerCta = (blockDim.x >> 5) / W;
  const int J = T.numJoints, n = T.numParams, N = P.numPoints;
  const int inN = kJoint ? J * kParametersPerJoint : n; // floats per instance of the input
  const int thF = int(skelAligned(inN)), jsF = int(skelAligned(size_t(J) * kJointStateStride));
  const int accF = kBackward ? int(skelAligned(size_t(J) * kSkelAccStride)) : 0;
  const int perGroup = int(skeletonStateFrame(J, n, kBackward, kJoint).floats);
  float* th = smem + size_t(g.group) * perGroup;
  float* js = th + thF;
  float* acc = js + jsF;
  float* gjp = acc + accF;
  {
    TableStager stager{reinterpret_cast<uint32_t*>(smem + size_t(groupsPerCta) * perGroup)};
    // skeletonTableList(stager, T, S, a.numChildren, kBackward, kBackward && !kJoint) spelled out: through the list ptxas allocates
    // positionsKernel<true, 2, false, false> two more registers
    characterTableList(stager, T);
    if constexpr (kBackward) {
      stager(S.childStart, size_t(J) + 1); stager(S.children, a.numChildren);
      if constexpr (!kJoint) { stager(S.ptColStart, n + 1); stager(S.ptColRows, T.ptNnz); stager(S.ptColVals, T.ptNnz); }
    }
    if constexpr (kStagePoints) pointTableList(stager, P, J, kBackward);
    __syncthreads();
  }
  for (int b = blockIdx.x * groupsPerCta + g.group; b < a.batch; b += gridDim.x * groupsPerCta) {
    const float* src = a.params + size_t(b) * inN;
    for (int i = g.lane; i < inN; i += g.size) th[i] = src[i];
    g.sync();
    fkPasses<kBackward, kJoint>(g, T, th, js);
    const float* off = a.offsets + (a.offsetsBatched ? size_t(b) * N * 3 : 0);
    if constexpr (!kBackward) {
      positionPasses(g, P, js, off, a.positions + size_t(b) * N * 3);
    } else {
      // the joint-parameter gradient is the result from joint parameters, else the model-parameter gradient's intermediate
      float* gp = a.gradParams != nullptr ? a.gradParams + size_t(b) * inN : nullptr;
      float* gOff = a.gradOffsets != nullptr ? a.gradOffsets + size_t(b) * N * 3 : nullptr;
      positionGradPasses(g, T, S, P, js, off, a.gradPositions + size_t(b) * N * 3, acc, kJoint || gp == nullptr ? gp : gjp, kJoint ? nullptr : gp, gOff);
    }
    g.sync(); // the next instance overwrites th / js / gjp
  }
}

namespace {
// planInstanceOp decides the staging of the point tables
cudaError_t launchPositionsKernel(const PositionArgs& a, bool backward, cudaStream_t stream, InstanceLaunchQuery* query = nullptr) {
  const bool joint = a.fromJointParameters != 0;
  const int op = joint ? kInstanceOpJointPositions : kInstanceOpModelPositions;
  return launchInstanceGroups(a, a.numChildren, op, backward, a.P.numPoints, stream, query, false, [&](auto W, const InstanceLaunch& l) {
    return withFlag(backward, [&](auto kB) {
      return withFlag(joint, [&](auto kJ) { return withFlag(l.stagedPoints != 0, [&](auto kS) { return positionsKernel<kB, W, kJ, kS>; }); });
    });
  });
}
} // namespace

cudaError_t queryPositionsLaunch(const PositionArgs& a, bool backward, InstanceLaunchQuery* query) {
  *query = InstanceLaunchQuery{};
  if (a.P.numPoints == 0) return cudaSuccess; // nothing runs (the backward clears the parameter gradient)
  return launchPositionsKernel(a, backward, nullptr, query);
}

cudaError_t launchPositions(const PositionArgs& a, cudaStream_t stream) {
  if (a.batch <= 0 || a.P.numPoints == 0) return cudaSuccess;
  return launchPositionsKernel(a, false, stream);
}

cudaError_t launchPositionsBackward(const PositionArgs& a, cudaStream_t stream) {
  if (a.batch <= 0) return cudaSuccess;
  const size_t inN = a.fromJointParameters ? size_t(a.T.numJoints) * kParametersPerJoint : size_t(a.T.numParams);
  const size_t n3 = size_t(a.P.numPoints) * 3;
  if (n3 == 0) // no point: the parameter gradient is zero and the offset gradient empty
    return a.gradParams != nullptr ? cudaMemsetAsync(a.gradParams, 0, size_t(a.batch) * inN * sizeof(float), stream) : cudaSuccess;
  if (a.gradOffsets == nullptr || a.offsetsBatched) return launchPositionsKernel(a, true, stream);
  const int perChunk = batchSumChunk(a.batch);
  const int numChunks = (a.batch + perChunk - 1) / perChunk;
  float* partial = a.gradOffsets;
  cudaError_t e = cudaSuccess;
  if (numChunks > 1) {
    e = cudaMallocAsync(reinterpret_cast<void**>(&partial), n3 * numChunks * sizeof(float), stream);
    if (e != cudaSuccess) return e;
  }
  // slices of whole chunks: the instances b0 .. b0 + nb write their offset-gradient rows to scratch, summed per chunk into partial
  e = forEachInstanceSlice(numChunks, size_t(perChunk) * n3 * sizeof(float), stream, [&](float* rows, int, int c0, int nc) {
    const int b0 = c0 * perChunk, nb = std::min(nc * perChunk, a.batch - b0);
    PositionArgs s = a;
    s.batch = nb;
    s.params += size_t(b0) * inN;
    s.gradPositions += size_t(b0) * n3;
    if (s.gradParams != nullptr) s.gradParams += size_t(b0) * inN;
    s.gradOffsets = rows;
    cudaError_t r = launchPositionsKernel(s, true, stream);
    if (r == cudaSuccess) r = launchRowGroupSum(rows, nb, perChunk, n3, partial + size_t(c0) * n3, stream);
    return r;
  });
  if (numChunks > 1) {
    if (e == cudaSuccess) e = launchRowGroupSum(partial, numChunks, numChunks, n3, a.gradOffsets, stream);
    const cudaError_t f = cudaFreeAsync(partial, stream);
    if (e == cudaSuccess) e = f;
  }
  return e;
}

// ------------------------------------------------------------------------------------------------
// Parameter-limit residuals (ik_device.cuh limitPasses / limitGradPasses), in the per-instance frame of skeletonStateKernel: theta and the
// joint parameters P theta + o in shared memory, then lanes = limits write their rows. kEllipsoid (the character has an Ellipsoid limit,
// a fact of its limit tables): the FK passes from the joint parameters run before, with the DOF axes in the backward.
//   backward:  Ellipsoid seeds by joint (skelGradSeed's layout) and skelGradTail's fold when kEllipsoid; the joint-space terms added to
//              the joint-parameter gradient by row; P^T plus the parameter-space terms by model parameter. Each a host-planned CSR in
//              limit-list order: no atomics, and no result depends on the launch shape.
// The limit tables are read from global memory; they are small and shared by the batch.
// ------------------------------------------------------------------------------------------------
template <bool kBackward, int W, bool kEllipsoid>
__global__ void __launch_bounds__(32 * kSkelMaxWarps, 1) parameterLimitsKernel(const ParameterLimitArgs a) {
  extern __shared__ __align__(16) float smem[];
  CharacterTables T = a.T;
  SkeletonTables S = a.S;
  const LimitTables L = a.L;
  const WarpLanes<W> g = WarpLanes<W>::of(threadIdx.x >> 5, threadIdx.x & 31);
  const int groupsPerCta = (blockDim.x >> 5) / W;
  const int J = T.numJoints, n = T.numParams, R = L.numRows;
  const int perGroup = int(parameterLimitsFrame(J, n, kBackward, kEllipsoid).floats);
  float* th = smem + size_t(g.group) * perGroup;
  float* jp = th + skelAligned(size_t(n));
  float* js = jp + skelAligned(size_t(J) * kParametersPerJoint);
  float* gjp = js + (kEllipsoid ? skelAligned(size_t(J) * kJointStateStride) : 0);
  float* acc = gjp + (kBackward ? skelAligned(size_t(J) * kParametersPerJoint) : 0);
  {
    TableStager stager{reinterpret_cast<uint32_t*>(smem + size_t(groupsPerCta) * perGroup)};
    skeletonTableList(stager, T, S, a.numChildren, kBackward && kEllipsoid, kBackward);
    __syncthreads();
  }
  for (int b = blockIdx.x * groupsPerCta + g.group; b < a.batch; b += gridDim.x * groupsPerCta) {
    const float* src = a.theta + size_t(b) * n;
    for (int i = g.lane; i < n; i += g.size) th[i] = src[i];
    g.sync();
    if constexpr (!kBackward) limitPasses<kEllipsoid>(g, T, L, th, jp, js, a.residual + size_t(b) * R);
    else limitGradPasses<kEllipsoid>(g, T, S, L, th, jp, js, acc, gjp, a.gradResidual + size_t(b) * R, a.gradTheta + size_t(b) * n);
    g.sync(); // the next instance overwrites th / jp / js / gjp
  }
}

cudaError_t launchParameterLimits(const ParameterLimitArgs& a, bool backward, cudaStream_t stream, InstanceLaunchQuery* query) {
  if (query) *query = InstanceLaunchQuery{};
  if (a.batch <= 0) return cudaSuccess;
  if (a.L.numRows == 0) { // no live limit: nothing to write, and the gradient is zero
    if (query) return cudaSuccess;
    return backward ? cudaMemsetAsync(a.gradTheta, 0, size_t(a.batch) * a.T.numParams * sizeof(float), stream) : cudaSuccess;
  }
  const bool fk = a.L.ellipsoid != 0;
  return launchInstanceGroups(a, a.numChildren, kInstanceOpParameterLimits, backward, 0, stream, query, fk, [&](auto W, const InstanceLaunch&) {
    return withFlag(backward, [&](auto kB) { return withFlag(fk, [&](auto kE) { return parameterLimitsKernel<kB, W, kE>; }); });
  });
}

// ------------------------------------------------------------------------------------------------
// Self-collision rows of tapered capsules (ik_device.cuh collisionPasses / collisionGradPasses), in the per-instance frame of
// skeletonStateKernel: lanes = capsules build the world capsules in shared memory from their parents' states, then
//   forward:   lanes = pairs write the rows;
//   backward:  lanes = capsules walk their own pairs (a host-planned CSR, pairs ascending), recompute each contact and sum their own
//              side's gradient in shared memory; lanes = joints sum their capsules in CSR order into dLoss / d state.
// No atomics and no global scratch: every output is one lane's fixed-order sum, so no result depends on the launch shape. The collision
// tables are read from global memory; the states are read where a capsule or a joint with capsules needs them.
// ------------------------------------------------------------------------------------------------
template <bool kBackward, int W>
__global__ void __launch_bounds__(32 * kSkelMaxWarps, 1) collisionKernel(const CollisionArgs a) {
  extern __shared__ __align__(16) float smem[];
  const CollisionTables L = a.L;
  const WarpLanes<W> g = WarpLanes<W>::of(threadIdx.x >> 5, threadIdx.x & 31);
  const int groupsPerCta = (blockDim.x >> 5) / W;
  const int J = a.T.numJoints, P = L.numPairs;
  const int perGroup = int(collisionFrame(L.numCapsules, kBackward).floats);
  float* geo = smem + size_t(g.group) * perGroup;
  float* cg = geo + skelAligned(size_t(L.numCapsules) * kCapsuleFloats);
  for (int b = blockIdx.x * groupsPerCta + g.group; b < a.batch; b += gridDim.x * groupsPerCta) {
    const float* st = a.state + size_t(b) * J * 8;
    if constexpr (!kBackward) collisionPasses(g, L, st, geo, a.residual + size_t(b) * P);
    else collisionGradPasses(g, L, J, st, geo, cg, a.gradResidual + size_t(b) * P, a.gradState + size_t(b) * J * 8);
    g.sync(); // the next instance overwrites geo / cg
  }
}

cudaError_t launchCollision(const CollisionArgs& a, bool backward, cudaStream_t stream, InstanceLaunchQuery* query) {
  if (query) *query = InstanceLaunchQuery{};
  if (a.batch <= 0) return cudaSuccess;
  if (a.L.numPairs == 0) { // no pair: nothing to write, and the gradient is zero
    if (query) return cudaSuccess;
    return backward ? cudaMemsetAsync(a.gradState, 0, size_t(a.batch) * a.T.numJoints * 8 * sizeof(float), stream) : cudaSuccess;
  }
  return launchInstanceGroups(a, 0, kInstanceOpCollision, backward, a.L.numCapsules, stream, query, false, [&](auto W, const InstanceLaunch&) {
    return withFlag(backward, [&](auto kB) { return collisionKernel<kB, W>; });
  });
}

// ------------------------------------------------------------------------------------------------
// Skinning with an identity blend shape (ik_device.cuh blendShapeRest / blendWeightAccumulate), on the skinning's building blocks.
// A work item is (a tile of T instances, a block of kSkinThreads vertices, one per thread).
//   blendSkinKernel<T, kRestOnly>   the tile's weights [K'][T] in shared memory; each thread forms its vertex's rest points for the T
//                                   instances in registers (every shape-vector element it loads serves the whole tile), then per
//                                   instance the CTA writes the J skinning transforms to shared memory and blends. kRestOnly writes
//                                   the rest points instead (the backward's scratch for the skel-state gradient).
//   blendWeightPartialKernel<T>     per instance the rest-point gradient of the block's vertices (skinRestGradient) to shared memory,
//                                   then threads = (quarter of the block, k) sum <S_kv, r_tv> over their quarter's vertices in order;
//                                   the quarters are added in order into one partial sum per (vertex block, instance, k).
//   blendWeightFinishKernel         lanes = (instance, k): the vertex blocks summed in order.
// No atomics; an instance's sums run in an order fixed by V and K' alone, so neither the batch, the tile nor the grid changes a bit.
// ------------------------------------------------------------------------------------------------
constexpr int kBlendTileMax = 16;                        // instances per tile when the batch fills the grid with them
constexpr int kBlendTileMin = 4;                         // otherwise
constexpr int kBlendGroups = kSkinThreads / 64;          // blendWeightPartialKernel: thread = (group, k of a 64-wide block of K')
constexpr int kBlendGroupVerts = kSkinThreads / kBlendGroups;

template <int T, bool kRestOnly>
__global__ void __launch_bounds__(kSkinThreads, 2) blendSkinKernel(const BlendSkinArgs a, int b0, int nb, float* rest) {
  extern __shared__ __align__(16) float sm[];
  const SkinTables& S = a.skin.S;
  const int V = S.numVertices, J = a.skin.numJoints, Kp = a.numWeights;
  float* W = sm;                // [K'][T]
  float* M = sm + Kp * T;       // [J][12], one instance at a time
  const int vBlocks = (V + kSkinThreads - 1) / kSkinThreads;
  const long items = long((nb + T - 1) / T) * vBlocks;
  for (long it = blockIdx.x; it < items; it += gridDim.x) {
    const int tb = b0 + int(it / vBlocks) * T, nt = min(T, b0 + nb - tb);
    const int v = int(it % vBlocks) * kSkinThreads + threadIdx.x;
    __syncthreads(); // the previous item's readers of W and M are done
    for (int i = threadIdx.x; i < Kp * T; i += blockDim.x) {
      const int k = i / T, t = i % T;
      W[i] = t < nt ? a.blendWeights[size_t(tb + t) * Kp + k] : 0.f;
    }
    __syncthreads();
    F3 x[T];
    if (v < V) blendShapeRest<T>(a.Bs, V, v, W, Kp, x);
#pragma unroll
    for (int t = 0; t < T; ++t) {
      if (t >= nt) break;
      if constexpr (kRestOnly) {
        if (v < V) {
          float* o = rest + (size_t(tb - b0 + t) * V + v) * 3;
          o[0] = x[t].x; o[1] = x[t].y; o[2] = x[t].z;
        }
      } else {
        __syncthreads();
        for (int j = threadIdx.x; j < J; j += blockDim.x)
          skinTransform(a.skin.skelState + (size_t(tb + t) * J + j) * 8, S.inverseBindPose + j * kSkinIbpStride, M + j * kSkinIbpStride);
        __syncthreads();
        if (v < V) {
          const F3 p = skinBlend(S, M, v, x[t]);
          float* o = a.skin.points + (size_t(tb + t) * V + v) * 3;
          o[0] = p.x; o[1] = p.y; o[2] = p.z;
        }
      }
    }
  }
}

// partial: [vBlocks][nb][K']
template <int T>
__global__ void __launch_bounds__(kSkinThreads) blendWeightPartialKernel(const BlendSkinArgs a, int b0, int nb, float* partial) {
  extern __shared__ __align__(16) float sm[];
  constexpr int kStride = 3 * T + 4;                        // floats per vertex of R: 16-byte rows, fewer bank conflicts on the writes
  const SkinTables& S = a.skin.S;
  const int V = S.numVertices, J = a.skin.numJoints, Kp = a.numWeights;
  float* R = sm;                                             // [kSkinThreads][kStride]: r_tv at 3 t
  float* P = R + kSkinThreads * kStride;                     // [kBlendGroups][T][64]
  float* M = P + kBlendGroups * T * 64;                      // [J][12]
  const int vBlocks = (V + kSkinThreads - 1) / kSkinThreads;
  const long items = long((nb + T - 1) / T) * vBlocks;
  const int g = threadIdx.x / 64, kl = threadIdx.x % 64;
  for (long it = blockIdx.x; it < items; it += gridDim.x) {
    const int tb = b0 + int(it / vBlocks) * T, nt = min(T, b0 + nb - tb);
    const int vb = int(it % vBlocks), v = vb * kSkinThreads + threadIdx.x;
    float* mine = R + threadIdx.x * kStride;
    for (int t = 0; t < nt; ++t) {
      __syncthreads(); // the previous readers of M (and, at t = 0, of R and P) are done
      for (int j = threadIdx.x; j < J; j += blockDim.x)
        skinTransform(a.skin.skelState + (size_t(tb + t) * J + j) * 8, S.inverseBindPose + j * kSkinIbpStride, M + j * kSkinIbpStride);
      __syncthreads();
      const F3 r = v < V ? skinRestGradient(S, M, v, ld3(a.skin.gradPoints + (size_t(tb + t) * V + v) * 3)) : f3(0.f, 0.f, 0.f);
      mine[3 * t] = r.x; mine[3 * t + 1] = r.y; mine[3 * t + 2] = r.z;
    }
    for (int t = nt; t < T; ++t) mine[3 * t] = mine[3 * t + 1] = mine[3 * t + 2] = 0.f;
    const int vEnd = min(kBlendGroupVerts, V - vb * kSkinThreads - g * kBlendGroupVerts); // this group's vertices in the block
    for (int kb = 0; kb < Kp; kb += 64) {
      __syncthreads(); // R is complete; the previous k block's readers of P are done
      const int k = kb + kl;
      float acc[T];
#pragma unroll
      for (int t = 0; t < T; ++t) acc[t] = 0.f;
      if (k < Kp) {
        const float* sv = a.Bs.shapeVectors + (size_t(k) * V + vb * kSkinThreads + g * kBlendGroupVerts) * 3;
        const float* rv = R + g * kBlendGroupVerts * kStride;
        for (int i = 0; i < vEnd; ++i) {
          const F3 s = ld3(sv + 3 * i);
#pragma unroll
          for (int t = 0; t < T; ++t) acc[t] = blendWeightAccumulate(acc[t], s, ld3(rv + i * kStride + 3 * t));
        }
      }
#pragma unroll
      for (int t = 0; t < T; ++t) P[(g * T + t) * 64 + kl] = acc[t];
      __syncthreads();
      for (int i = threadIdx.x; i < nt * 64; i += blockDim.x) {
        const int t = i / 64, kk = i % 64;
        if (kb + kk >= Kp) continue;
        float s = P[t * 64 + kk];
        for (int q = 1; q < kBlendGroups; ++q) s += P[(q * T + t) * 64 + kk];
        partial[(size_t(vb) * nb + (tb - b0 + t)) * Kp + kb + kk] = s;
      }
    }
  }
}

__global__ void blendWeightFinishKernel(const float* partial, int vBlocks, int nb, int Kp, float* out) {
  const size_t n = size_t(nb) * Kp;
  for (size_t i = size_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += size_t(gridDim.x) * blockDim.x) {
    float s = partial[i];
    for (int c = 1; c < vBlocks; ++c) s += partial[size_t(c) * n + i];
    out[i] = s;
  }
}

namespace {
size_t blendSkinSmem(const BlendSkinArgs& a, int T) { return (size_t(a.numWeights) * T + size_t(a.skin.numJoints) * kSkinIbpStride) * sizeof(float); }
size_t blendWeightSmem(const BlendSkinArgs& a, int T) {
  return (size_t(kSkinThreads) * (3 * T + 4) + size_t(kBlendGroups) * T * 64 + size_t(a.skin.numJoints) * kSkinIbpStride) * sizeof(float);
}
} // namespace

bool blendSkinFits(const BlendSkinArgs& a) {
  return blendSkinSmem(a, kBlendTileMin) <= size_t(g_maxSmemOptin) && blendWeightSmem(a, kBlendTileMin) <= size_t(g_maxSmemOptin);
}

namespace {

// The widest tile that still gives every resident CTA a work item and fits in shared memory; the tile changes how often a shape vector
// is read, not the result.
template <class K16, class K4>
cudaError_t chooseBlendTile(K16 wide, size_t smemWide, K4 narrow, size_t smemNarrow, int V, int nb, int* T, int* grid) {
  const long vBlocks = (V + kSkinThreads - 1) / kSkinThreads;
  if (smemWide <= size_t(g_maxSmemOptin)) {
    int slots = 0;
    const cudaError_t e = persistentGrid(wide, kSkinThreads, smemWide, 1L << 30, &slots);
    if (e != cudaSuccess) return e;
    const long wideItems = (nb + kBlendTileMax - 1) / kBlendTileMax * vBlocks;
    if (wideItems >= slots) { *T = kBlendTileMax; *grid = slots; return cudaSuccess; }
  }
  *T = kBlendTileMin;
  return persistentGrid(narrow, kSkinThreads, smemNarrow, (nb + kBlendTileMin - 1) / kBlendTileMin * vBlocks, grid);
}

template <bool kRestOnly>
cudaError_t launchBlendSkin(const BlendSkinArgs& a, int b0, int nb, float* rest, cudaStream_t stream) {
  int T = 0, grid = 0;
  const size_t s16 = blendSkinSmem(a, kBlendTileMax), s4 = blendSkinSmem(a, kBlendTileMin);
  cudaError_t e = chooseBlendTile(blendSkinKernel<kBlendTileMax, kRestOnly>, s16, blendSkinKernel<kBlendTileMin, kRestOnly>, s4, a.skin.S.numVertices, nb, &T, &grid);
  if (e != cudaSuccess) return e;
  if (T == kBlendTileMax) blendSkinKernel<kBlendTileMax, kRestOnly><<<grid, kSkinThreads, s16, stream>>>(a, b0, nb, rest);
  else blendSkinKernel<kBlendTileMin, kRestOnly><<<grid, kSkinThreads, s4, stream>>>(a, b0, nb, rest);
  return cudaGetLastError();
}
} // namespace

cudaError_t launchSkinWithBlendShapes(const BlendSkinArgs& a, cudaStream_t stream) {
  if (a.skin.batch <= 0) return cudaSuccess;
  return launchBlendSkin<false>(a, 0, a.skin.batch, nullptr, stream);
}

cudaError_t launchSkinWithBlendShapesBackward(const BlendSkinArgs& a, cudaStream_t stream) {
  const int B = a.skin.batch, V = a.skin.S.numVertices, J = a.skin.numJoints, Kp = a.numWeights;
  if (B <= 0) return cudaSuccess;
  cudaError_t e = cudaSuccess;
  if (a.skin.gradState != nullptr) {
    // the shaped rest points of a slice of instances, then skin_points' own state-gradient path with them as batched rest points (its
    // partial sums are allocated while the slice's rest points are)
    e = forEachInstanceSlice(B, size_t(V) * 3 * sizeof(float), stream, [&](float* rest, int, int b0, int nb) {
      const cudaError_t r = launchBlendSkin<true>(a, b0, nb, rest, stream);
      if (r != cudaSuccess) return r;
      SkinArgs s = a.skin;
      s.batch = nb;
      s.skelState += size_t(b0) * J * 8;
      s.gradPoints += size_t(b0) * V * 3;
      s.gradState += size_t(b0) * J * 8;
      s.restPoints = rest;
      s.restBatched = 1;
      s.points = nullptr;
      s.gradRest = nullptr;
      return launchSkinPointsBackward(s, stream);
    });
  }
  if (e != cudaSuccess || a.gradWeights == nullptr) return e;
  const int vBlocks = (V + kSkinThreads - 1) / kSkinThreads;
  return forEachInstanceSlice(B, size_t(vBlocks) * Kp * sizeof(float), stream, [&](float* partial, int, int b0, int nb) {
    int T = 0, grid = 0;
    const size_t s16 = blendWeightSmem(a, kBlendTileMax), s4 = blendWeightSmem(a, kBlendTileMin);
    const cudaError_t r = chooseBlendTile(blendWeightPartialKernel<kBlendTileMax>, s16, blendWeightPartialKernel<kBlendTileMin>, s4, V, nb, &T, &grid);
    if (r != cudaSuccess) return r;
    if (T == kBlendTileMax) blendWeightPartialKernel<kBlendTileMax><<<grid, kSkinThreads, s16, stream>>>(a, b0, nb, partial);
    else blendWeightPartialKernel<kBlendTileMin><<<grid, kSkinThreads, s4, stream>>>(a, b0, nb, partial);
    const size_t n = size_t(nb) * Kp;
    blendWeightFinishKernel<<<unsigned(std::min<size_t>((n + kSkinThreads - 1) / kSkinThreads, 4096)), kSkinThreads, 0, stream>>>(
        partial, vBlocks, nb, Kp, a.gradWeights + size_t(b0) * Kp);
    return cudaGetLastError();
  });
}

// ------------------------------------------------------------------------------------------------
// Vertex normals (ik_device.cuh faceNormal / normalizeClamped / normalGradient / cornerGradient). A thread serves one vertex for a tile
// of kNormalTile instances: each entry of the vertex's corner list and its face are read once for the whole tile, then the positions of
// each instance are gathered. Work items are (tile, block of kNormalThreads vertices) with the vertex blocks fastest, so the CTAs in
// flight gather from the positions of a few instances, which stay in L2.
//   vertexNormalKernel<false>   n_v summed over the vertex's corner list in order, then normalised: the normals.
//   vertexNormalKernel<true>    the same n_v, then h_v = normalGradient(n_v, upstream) to scratch: the first pass of the backward.
//   vertexNormalGradKernel      per corner k of face f in the list, G_f = h_i0 + h_i1 + h_i2, then cornerGradient: the second pass.
// No atomics: every output is a sum in the order of the corner list, the same for any batch and launch shape.
// ------------------------------------------------------------------------------------------------
constexpr int kNormalThreads = 256;
constexpr int kNormalTile = 4;

template <bool kGrad>
__global__ void __launch_bounds__(kNormalThreads) vertexNormalKernel(const NormalArgs a, int b0, int nb, float* h) {
  const MeshFaceTables M = a.M;
  const int V = M.numVertices;
  const int vBlocks = (V + kNormalThreads - 1) / kNormalThreads;
  const long items = long((nb + kNormalTile - 1) / kNormalTile) * vBlocks;
  for (long it = blockIdx.x; it < items; it += gridDim.x) {
    const int v = int(it % vBlocks) * kNormalThreads + threadIdx.x;
    if (v >= V) continue;
    const int tb = b0 + int(it / vBlocks) * kNormalTile, nt = min(kNormalTile, b0 + nb - tb);
    F3 n[kNormalTile];
#pragma unroll
    for (int t = 0; t < kNormalTile; ++t) n[t] = f3(0.f, 0.f, 0.f);
    for (int c = M.vertStart[v]; c < M.vertStart[v + 1]; ++c) {
      const int* f = M.faces + (M.vertCorner[c] / 3) * 3;
      const int i0 = f[0], i1 = f[1], i2 = f[2];
#pragma unroll
      for (int t = 0; t < kNormalTile; ++t)
        if (t < nt) {
          const float* x = a.positions + size_t(tb + t) * V * 3;
          n[t] = n[t] + faceNormal(ld3(x + 3 * i0), ld3(x + 3 * i1), ld3(x + 3 * i2));
        }
    }
#pragma unroll
    for (int t = 0; t < kNormalTile; ++t)
      if (t < nt) {
        const size_t at = (size_t(tb + t) * V + v) * 3;
        F3 r;
        float* o;
        if constexpr (kGrad) {
          r = normalGradient(n[t], ld3(a.gradNormals + at));
          o = h + (size_t(tb + t - b0) * V + v) * 3;
        } else {
          r = normalizeClamped(n[t]);
          o = a.normals + at;
        }
        o[0] = r.x; o[1] = r.y; o[2] = r.z;
      }
  }
}

// h: [nb][V][3] of the instances b0 .. b0 + nb
__global__ void __launch_bounds__(kNormalThreads) vertexNormalGradKernel(const NormalArgs a, int b0, int nb, const float* h) {
  const MeshFaceTables M = a.M;
  const int V = M.numVertices;
  const int vBlocks = (V + kNormalThreads - 1) / kNormalThreads;
  const long items = long((nb + kNormalTile - 1) / kNormalTile) * vBlocks;
  for (long it = blockIdx.x; it < items; it += gridDim.x) {
    const int v = int(it % vBlocks) * kNormalThreads + threadIdx.x;
    if (v >= V) continue;
    const int tb = b0 + int(it / vBlocks) * kNormalTile, nt = min(kNormalTile, b0 + nb - tb);
    F3 g[kNormalTile];
#pragma unroll
    for (int t = 0; t < kNormalTile; ++t) g[t] = f3(0.f, 0.f, 0.f);
    for (int c = M.vertStart[v]; c < M.vertStart[v + 1]; ++c) {
      const int fc = M.vertCorner[c], k = fc % 3;
      const int* f = M.faces + (fc - k);
      const int i0 = f[0], i1 = f[1], i2 = f[2];
      const int next = k == 0 ? i1 : (k == 1 ? i2 : i0), prev = k == 0 ? i2 : (k == 1 ? i0 : i1);
#pragma unroll
      for (int t = 0; t < kNormalTile; ++t)
        if (t < nt) {
          const float* x = a.positions + size_t(tb + t) * V * 3;
          const float* hb = h + size_t(tb + t - b0) * V * 3;
          const F3 G = ld3(hb + 3 * i0) + ld3(hb + 3 * i1) + ld3(hb + 3 * i2);
          g[t] = g[t] + cornerGradient(ld3(x + 3 * next), ld3(x + 3 * prev), G);
        }
    }
#pragma unroll
    for (int t = 0; t < kNormalTile; ++t)
      if (t < nt) {
        float* o = a.gradPositions + (size_t(tb + t) * V + v) * 3;
        o[0] = g[t].x; o[1] = g[t].y; o[2] = g[t].z;
      }
  }
}

namespace {
template <class K, class P>
cudaError_t launchNormalPass(K kernel, const NormalArgs& a, int b0, int nb, P h, cudaStream_t stream) {
  const long vBlocks = (a.M.numVertices + kNormalThreads - 1) / kNormalThreads;
  int grid = 0;
  const cudaError_t e = persistentGrid(kernel, kNormalThreads, 0, (nb + kNormalTile - 1) / kNormalTile * vBlocks, &grid);
  if (e != cudaSuccess) return e;
  kernel<<<grid, kNormalThreads, 0, stream>>>(a, b0, nb, h);
  return cudaGetLastError();
}
} // namespace

cudaError_t launchVertexNormals(const NormalArgs& a, cudaStream_t stream) {
  if (a.batch <= 0) return cudaSuccess;
  return launchNormalPass(vertexNormalKernel<false>, a, 0, a.batch, static_cast<float*>(nullptr), stream);
}

cudaError_t launchVertexNormalsBackward(const NormalArgs& a, cudaStream_t stream) {
  if (a.batch <= 0) return cudaSuccess;
  return forEachInstanceSlice(a.batch, size_t(a.M.numVertices) * 3 * sizeof(float), stream, [&](float* h, int, int b0, int nb) {
    const cudaError_t r = launchNormalPass(vertexNormalKernel<true>, a, b0, nb, h, stream);
    return r != cudaSuccess ? r : launchNormalPass(vertexNormalGradKernel, a, b0, nb, static_cast<const float*>(h), stream);
  });
}

// ------------------------------------------------------------------------------------------------
// Closest points on the mesh (ik_device.cuh closestPointOnTriangle / faceDistance2 / closerFace / boxLowerBound / pruneBox / box*). The
// tree's topology is shared; each slice of instances gets its boxes [nb][numNodes][lo xyz, hi xyz] refitted in scratch, then queried.
//   meshTreeRefitKernel   one CTA per instance: the levels from the deepest up, a thread per node, __syncthreads between levels.
//   closestPointKernel    one thread per (instance, query): depth-first from the root, the nearer child first and the other on a stack
//                         of kTreeStack (node, lower bound) entries, re-checked when popped. The stack is indexed dynamically, so it
//                         lives in local memory.
// The result is the smallest (d2, face) over the candidates, whatever the tree and the visiting order: a subtree is skipped only when
// its lower bound is strictly above the best d2, which no face in it can then reach. No atomics.
// ------------------------------------------------------------------------------------------------
constexpr int kRefitThreads = 256;
constexpr int kClosestThreads = 128;

__global__ void __launch_bounds__(kRefitThreads) meshTreeRefitKernel(const ClosestPointArgs a, int b0, int nb, float* boxes) {
  const MeshTreeTables T = a.T;
  const int V = a.M.numVertices;
  for (int i = blockIdx.x; i < nb; i += gridDim.x) {
    const float* x = a.vertices + size_t(b0 + i) * V * 3;
    float* bx = boxes + size_t(i) * T.numNodes * 6;
    for (int L = T.depth - 1; L >= 0; --L) {
      const int end = T.levelStart[L + 1];
      for (int n = T.levelStart[L] + threadIdx.x; n < end; n += kRefitThreads) {
        const int start = T.nodeStart[n], count = T.nodeCount[n];
        float box[6];
        if (count == 0) {
          boxUnion(box, bx + size_t(start) * 6, bx + size_t(start + 1) * 6);
        } else {
          boxEmpty(box);
          for (int k = 0; k < count; ++k) {
            const int* f = a.M.faces + size_t(T.leafFaces[start + k]) * 3;
            boxGrow(box, ld3(x + 3 * size_t(f[0])));
            boxGrow(box, ld3(x + 3 * size_t(f[1])));
            boxGrow(box, ld3(x + 3 * size_t(f[2])));
          }
        }
        float* o = bx + size_t(n) * 6;
#pragma unroll
        for (int k = 0; k < 6; ++k) o[k] = box[k];
      }
      __syncthreads(); // the next level reads these boxes
    }
  }
}

// boxes: [nb][numNodes][6] of the instances b0 .. b0 + nb
__global__ void __launch_bounds__(kClosestThreads) closestPointKernel(const ClosestPointArgs a, int b0, int nb, const float* boxes) {
  const MeshTreeTables T = a.T;
  const int V = a.M.numVertices;
  const long N = a.numPoints, total = long(nb) * N;
  for (long it = long(blockIdx.x) * kClosestThreads + threadIdx.x; it < total; it += long(gridDim.x) * kClosestThreads) {
    const int i = int(it / N);
    const size_t qi = size_t(b0 + i) * N + size_t(it % N);
    const F3 p = ld3(a.points + 3 * qi);
    const float* x = a.vertices + size_t(b0 + i) * V * 3;
    const float* bx = boxes + size_t(i) * T.numNodes * 6;
    float best = a.maxDist2;
    int bestFace = INT_MAX;
    F3 bestQ = f3(0.f, 0.f, 0.f), bestBary = f3(0.f, 0.f, 0.f);
    int stackNode[kTreeStack];
    float stackLb[kTreeStack];
    int sp = 0, node = 0;
    bool go = finite3(p) && !pruneBox(boxLowerBound(bx, p), best);
    while (go) {
      const int start = T.nodeStart[node], count = T.nodeCount[node];
      if (count == 0) {
        const float lb0 = boxLowerBound(bx + size_t(start) * 6, p), lb1 = boxLowerBound(bx + size_t(start + 1) * 6, p);
        const bool in0 = !pruneBox(lb0, best), in1 = !pruneBox(lb1, best);
        if (in0 && in1) {
          const bool first1 = lb1 < lb0;
          stackNode[sp] = first1 ? start : start + 1;
          stackLb[sp] = first1 ? lb0 : lb1;
          ++sp;
          node = first1 ? start + 1 : start;
          continue;
        }
        if (in0 || in1) {
          node = in0 ? start : start + 1;
          continue;
        }
      } else {
        for (int k = 0; k < count; ++k) {
          const int f = T.leafFaces[start + k];
          const int* fv = a.M.faces + size_t(f) * 3;
          F3 q, bary;
          const float d2 = faceDistance2(p, ld3(x + 3 * size_t(fv[0])), ld3(x + 3 * size_t(fv[1])), ld3(x + 3 * size_t(fv[2])), q, bary);
          if (closerFace(d2, f, best, bestFace)) {
            best = d2; bestFace = f; bestQ = q; bestBary = bary;
          }
        }
      }
      go = false;
      while (sp > 0) {
        --sp;
        if (!pruneBox(stackLb[sp], best)) {
          node = stackNode[sp];
          go = true;
          break;
        }
      }
    }
    const bool found = bestFace != INT_MAX;
    float* oq = a.outPoints + 3 * qi;
    float* ob = a.outBary + 3 * qi;
    if (!found) bestQ = bestBary = f3(0.f, 0.f, 0.f);
    oq[0] = bestQ.x; oq[1] = bestQ.y; oq[2] = bestQ.z;
    ob[0] = bestBary.x; ob[1] = bestBary.y; ob[2] = bestBary.z;
    a.outFace[qi] = found ? bestFace : -1;
  }
}

cudaError_t launchClosestPointsOnMesh(const ClosestPointArgs& a, cudaStream_t stream) {
  if (a.batch <= 0 || a.numPoints <= 0) return cudaSuccess;
  return forEachInstanceSlice(a.batch, size_t(a.T.numNodes) * 6 * sizeof(float), stream, [&](float* boxes, int slice, int b0, int nb) {
    // grids sized for a whole slice, capped by the work of this one
    int refitGrid = 0, queryGrid = 0;
    cudaError_t r = persistentGrid(meshTreeRefitKernel, kRefitThreads, 0, slice, &refitGrid);
    if (r == cudaSuccess)
      r = persistentGrid(closestPointKernel, kClosestThreads, 0, (long(slice) * a.numPoints + kClosestThreads - 1) / kClosestThreads, &queryGrid);
    if (r != cudaSuccess) return r;
    meshTreeRefitKernel<<<std::min(refitGrid, nb), kRefitThreads, 0, stream>>>(a, b0, nb, boxes);
    r = cudaGetLastError();
    if (r != cudaSuccess) return r;
    const long blocks = (long(nb) * a.numPoints + kClosestThreads - 1) / kClosestThreads;
    closestPointKernel<<<int(std::min<long>(queryGrid, blocks)), kClosestThreads, 0, stream>>>(a, b0, nb, boxes);
    return cudaGetLastError();
  });
}

// ------------------------------------------------------------------------------------------------
// Closest points of a point cloud (ik_device.cuh pointDistance2 / normalCompatible / mortonCode / closerFace / boxLowerBound /
// pruneBox / box*). Per call, each target instance of a slice gets a tree built in scratch (CloudScratch), all on the call's stream:
//   cloudBoundsKernel        (instance, tile of kSortTile points): the box of the tile's finite points
//   cloudBoundsReduceKernel  one CTA per instance: the union of its tile boxes (min / max is exact: the order does not matter)
//   cloudCodeKernel          thread per point: (mortonCode, index)
//   kSortPasses x            a stable segmented LSD radix sort of (code, index), kSortBits per pass:
//     cloudSortCountKernel     (instance, tile): the tile's digit counts
//     cloudSortScanKernel      one CTA per instance: per digit the exclusive scan over the tiles, and each digit's start
//     cloudSortScatterKernel   (instance, tile): each point to start[d] + scan[tile][d] + its rank among the tile's points with digit d
//   cloudGatherKernel        thread per point: the sorted copy of the points (and normals)
//   cloudBoxKernel           groups of up to 256 nodes of one level: their boxes (the leaves' from the sorted points), then up to 8
//                            levels above them in shared memory; launched from the leaves up until the root is written
// then closestCloudKernel runs one thread per (instance, query), depth first as closestPointKernel. Ranks within a tile come from
// __match_any_sync and per-warp counts in shared memory: no atomics anywhere, so an instance gets the same bits alone as in any batch.
// ------------------------------------------------------------------------------------------------
constexpr int kCloudThreads = 256;
constexpr int kSortDigits = 1 << kSortBits;
constexpr int kSortGroups = kSortTile / 32; // warp-sized groups of a tile, in point order
static_assert(kSortDigits == kCloudThreads && kSortTile % kCloudThreads == 0, "a thread per digit, whole rounds per tile");

// The per-instance scratch of a tree over M points, each array [slice][its count]
struct CloudScratch {
  int M, tiles, P;
  float* tileBox;     // [tiles][6]
  float* bounds;      // [6]
  uint32_t* keys[2];  // [M]
  int32_t* index[2];  // [M]
  int32_t* tileScan;  // [tiles][kSortDigits]
  int32_t* digitStart; // [kSortDigits]
  float* sorted;      // [M][3]
  float* sortedNormals; // [M][3], when there are normals
  float* boxes;       // [2P - 1][6]
  size_t floats(bool normals) const { // per instance, in 4-byte words
    return size_t(tiles) * 6 + 6 + 4 * size_t(M) + size_t(tiles) * kSortDigits + kSortDigits + (normals ? 6 : 3) * size_t(M) +
           (2 * size_t(P) - 1) * 6;
  }
  void carve(float* base, int slice, bool normals) {
    float* p = base;
    auto take = [&](size_t n) { float* r = p; p += n * slice; return r; };
    tileBox = take(size_t(tiles) * 6);
    bounds = take(6);
    keys[0] = reinterpret_cast<uint32_t*>(take(M));
    keys[1] = reinterpret_cast<uint32_t*>(take(M));
    index[0] = reinterpret_cast<int32_t*>(take(M));
    index[1] = reinterpret_cast<int32_t*>(take(M));
    tileScan = reinterpret_cast<int32_t*>(take(size_t(tiles) * kSortDigits));
    digitStart = reinterpret_cast<int32_t*>(take(kSortDigits));
    sorted = take(size_t(M) * 3);
    sortedNormals = normals ? take(size_t(M) * 3) : nullptr;
    boxes = take((2 * size_t(P) - 1) * 6);
  }
};

// The instance's box over its finite points, tile by tile; tb0: the first target instance of the slice
__global__ void __launch_bounds__(kCloudThreads) cloudBoundsKernel(const ClosestCloudArgs a, int tb0, int nt, CloudScratch S) {
  __shared__ float red[6][kCloudThreads];
  const int M = S.M;
  for (long w = blockIdx.x; w < long(nt) * S.tiles; w += gridDim.x) {
    const int i = int(w / S.tiles), tile = int(w % S.tiles);
    const float* x = a.target + size_t(tb0 + i) * M * 3;
    float box[6];
    boxEmpty(box);
    for (int e = tile * kSortTile + threadIdx.x; e < min(M, (tile + 1) * kSortTile); e += kCloudThreads) {
      const F3 p = ld3(x + 3 * size_t(e));
      if (finite3(p)) boxGrow(box, p);
    }
#pragma unroll
    for (int k = 0; k < 6; ++k) red[k][threadIdx.x] = box[k];
    __syncthreads();
    for (int s = kCloudThreads / 2; s > 0; s >>= 1) {
      if (threadIdx.x < s)
        for (int k = 0; k < 6; ++k)
          red[k][threadIdx.x] = k < 3 ? fminf(red[k][threadIdx.x], red[k][threadIdx.x + s]) : fmaxf(red[k][threadIdx.x], red[k][threadIdx.x + s]);
      __syncthreads();
    }
    if (threadIdx.x < 6) S.tileBox[(size_t(i) * S.tiles + tile) * 6 + threadIdx.x] = red[threadIdx.x][0];
    __syncthreads(); // red is reused by the next tile
  }
}

__global__ void __launch_bounds__(kCloudThreads) cloudBoundsReduceKernel(int nt, CloudScratch S) {
  __shared__ float red[6][kCloudThreads];
  for (int i = blockIdx.x; i < nt; i += gridDim.x) {
    float box[6];
    boxEmpty(box);
    for (int t = threadIdx.x; t < S.tiles; t += kCloudThreads) {
      const float* b = S.tileBox + (size_t(i) * S.tiles + t) * 6;
      boxUnion(box, box, b);
    }
#pragma unroll
    for (int k = 0; k < 6; ++k) red[k][threadIdx.x] = box[k];
    __syncthreads();
    for (int s = kCloudThreads / 2; s > 0; s >>= 1) {
      if (threadIdx.x < s)
        for (int k = 0; k < 6; ++k)
          red[k][threadIdx.x] = k < 3 ? fminf(red[k][threadIdx.x], red[k][threadIdx.x + s]) : fmaxf(red[k][threadIdx.x], red[k][threadIdx.x + s]);
      __syncthreads();
    }
    if (threadIdx.x < 6) S.bounds[size_t(i) * 6 + threadIdx.x] = red[threadIdx.x][0];
    __syncthreads();
  }
}

__global__ void __launch_bounds__(kCloudThreads) cloudCodeKernel(const ClosestCloudArgs a, int tb0, int nt, CloudScratch S) {
  const long M = S.M;
  for (long it = long(blockIdx.x) * kCloudThreads + threadIdx.x; it < nt * M; it += long(gridDim.x) * kCloudThreads) {
    const int i = int(it / M);
    const int m = int(it % M);
    S.keys[0][size_t(i) * M + m] = mortonCode(ld3(a.target + (size_t(tb0 + i) * M + m) * 3), S.bounds + size_t(i) * 6);
    S.index[0][size_t(i) * M + m] = m;
  }
}

// The digit of each of the thread's kSortTile / kCloudThreads points of `tile` (point r * 256 + threadIdx.x of the tile in round r;
// kSortDigits for a point past M) and its rank among the tile's points with that digit, in point order. On return cnt[g][d] holds
// the number of points with digit d in the groups before g of the tile and total[d] the tile's count; the caller syncs before reuse.
__device__ __forceinline__ void cloudTileRanks(const uint32_t* keys, int M, int tile, int shift, uint16_t (*cnt)[kSortDigits], int* total,
                                               int* digit, int* rank) {
  constexpr int kRounds = kSortTile / kCloudThreads;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int g = 0; g < kSortGroups; ++g) cnt[g][threadIdx.x] = 0;
  __syncthreads();
#pragma unroll
  for (int r = 0; r < kRounds; ++r) {
    const int e = tile * kSortTile + r * kCloudThreads + threadIdx.x;
    const int d = e < M ? int((keys[e] >> shift) & (kSortDigits - 1)) : kSortDigits;
    const unsigned same = __match_any_sync(0xffffffffu, d);
    digit[r] = d;
    rank[r] = __popc(same & ((1u << lane) - 1));
    if (d < kSortDigits && lane == __ffs(same) - 1) cnt[r * (kCloudThreads / 32) + warp][d] = uint16_t(__popc(same));
  }
  __syncthreads();
  int run = 0; // thread = digit: the exclusive scan over the groups, in place
  for (int g = 0; g < kSortGroups; ++g) {
    const int c = cnt[g][threadIdx.x];
    cnt[g][threadIdx.x] = uint16_t(run);
    run += c;
  }
  total[threadIdx.x] = run;
  __syncthreads();
#pragma unroll
  for (int r = 0; r < kRounds; ++r)
    if (digit[r] < kSortDigits) rank[r] += cnt[r * (kCloudThreads / 32) + warp][digit[r]];
}

__global__ void __launch_bounds__(kCloudThreads) cloudSortCountKernel(int nt, CloudScratch S, int src, int shift) {
  __shared__ uint16_t cnt[kSortGroups][kSortDigits];
  __shared__ int total[kSortDigits];
  constexpr int kRounds = kSortTile / kCloudThreads;
  int digit[kRounds], rank[kRounds];
  for (long w = blockIdx.x; w < long(nt) * S.tiles; w += gridDim.x) {
    const int i = int(w / S.tiles), tile = int(w % S.tiles);
    cloudTileRanks((src ? S.keys[1] : S.keys[0]) + size_t(i) * S.M, S.M, tile, shift, cnt, total, digit, rank);
    S.tileScan[(size_t(i) * S.tiles + tile) * kSortDigits + threadIdx.x] = total[threadIdx.x];
    __syncthreads();
  }
}

// thread = digit: tileScan becomes the exclusive scan over the tiles, digitStart the exclusive scan of the digits' totals
__global__ void __launch_bounds__(kCloudThreads) cloudSortScanKernel(int nt, CloudScratch S) {
  __shared__ int tot[kSortDigits];
  for (int i = blockIdx.x; i < nt; i += gridDim.x) {
    int* h = S.tileScan + size_t(i) * S.tiles * kSortDigits + threadIdx.x;
    int run = 0;
    for (int t = 0; t < S.tiles; ++t) {
      const int c = h[size_t(t) * kSortDigits];
      h[size_t(t) * kSortDigits] = run;
      run += c;
    }
    tot[threadIdx.x] = run;
    __syncthreads();
    if (threadIdx.x == 0) {
      int s = 0;
      for (int d = 0; d < kSortDigits; ++d) {
        const int c = tot[d];
        tot[d] = s;
        s += c;
      }
    }
    __syncthreads();
    S.digitStart[size_t(i) * kSortDigits + threadIdx.x] = tot[threadIdx.x];
    __syncthreads();
  }
}

__global__ void __launch_bounds__(kCloudThreads) cloudSortScatterKernel(int nt, CloudScratch S, int src, int shift) {
  __shared__ uint16_t cnt[kSortGroups][kSortDigits];
  __shared__ int total[kSortDigits];
  __shared__ int start[kSortDigits];
  constexpr int kRounds = kSortTile / kCloudThreads;
  int digit[kRounds], rank[kRounds];
  const size_t M = S.M;
  for (long w = blockIdx.x; w < long(nt) * S.tiles; w += gridDim.x) {
    const int i = int(w / S.tiles), tile = int(w % S.tiles);
    // src selects by value: an indexed parameter array would go through local memory
    const uint32_t* kin = (src ? S.keys[1] : S.keys[0]) + i * M;
    const int32_t* xin = (src ? S.index[1] : S.index[0]) + i * M;
    uint32_t* kout = (src ? S.keys[0] : S.keys[1]) + i * M;
    int32_t* xout = (src ? S.index[0] : S.index[1]) + i * M;
    cloudTileRanks(kin, S.M, tile, shift, cnt, total, digit, rank);
    start[threadIdx.x] = S.digitStart[size_t(i) * kSortDigits + threadIdx.x] + S.tileScan[(size_t(i) * S.tiles + tile) * kSortDigits + threadIdx.x];
    __syncthreads();
#pragma unroll
    for (int r = 0; r < kRounds; ++r) {
      if (digit[r] == kSortDigits) continue;
      const int e = tile * kSortTile + r * kCloudThreads + threadIdx.x;
      const int o = start[digit[r]] + rank[r];
      kout[o] = kin[e];
      xout[o] = xin[e];
    }
    __syncthreads();
  }
}

__global__ void __launch_bounds__(kCloudThreads) cloudGatherKernel(const ClosestCloudArgs a, int tb0, int nt, CloudScratch S) {
  const long M = S.M;
  for (long it = long(blockIdx.x) * kCloudThreads + threadIdx.x; it < nt * M; it += long(gridDim.x) * kCloudThreads) {
    const size_t i = size_t(it / M);
    const size_t j = size_t(S.index[0][it]);
    const size_t from = ((tb0 + i) * M + j) * 3;
#pragma unroll
    for (int k = 0; k < 3; ++k) S.sorted[3 * it + k] = a.target[from + k];
    if (S.sortedNormals)
#pragma unroll
      for (int k = 0; k < 3; ++k) S.sortedNormals[3 * it + k] = a.targetNormals[from + k];
  }
}

// Groups of 2^h nodes of level `bottom` (2^bottom nodes, the first at heap index 2^bottom - 1): their boxes, from the sorted points when
// bottom is the leaf level (`leaves`), else as written by an earlier launch; then the h levels above them, each node the union of its
// two children.
__global__ void __launch_bounds__(kCloudThreads) cloudBoxKernel(int nt, CloudScratch S, int bottom, int h, bool leaves) {
  __shared__ float sb[kCloudThreads][6];
  const long groups = (1L << bottom) >> h;
  const int M = S.M;
  for (long w = blockIdx.x; w < nt * groups; w += gridDim.x) {
    const size_t i = size_t(w / groups);
    const long g = w % groups;
    float* bx = S.boxes + i * (2 * size_t(S.P) - 1) * 6;
    float box[6];
    if (threadIdx.x < (1 << h)) {
      const long j = (g << h) + threadIdx.x;
      const size_t n = size_t((1L << bottom) - 1 + j);
      if (leaves) {
        boxEmpty(box);
        const float* x = S.sorted + i * size_t(M) * 3;
        for (long m = j * kLeafPoints; m < min(long(M), (j + 1) * kLeafPoints); ++m) boxGrow(box, ld3(x + 3 * m));
#pragma unroll
        for (int k = 0; k < 6; ++k) bx[n * 6 + k] = box[k];
      } else {
#pragma unroll
        for (int k = 0; k < 6; ++k) box[k] = bx[n * 6 + k];
      }
#pragma unroll
      for (int k = 0; k < 6; ++k) sb[threadIdx.x][k] = box[k];
    }
    __syncthreads();
    for (int lev = 1; lev <= h; ++lev) {
      const int count = 1 << (h - lev);
      if (threadIdx.x < count) boxUnion(box, sb[2 * threadIdx.x], sb[2 * threadIdx.x + 1]);
      __syncthreads();
      if (threadIdx.x < count) {
        const size_t n = size_t((1L << (bottom - lev)) - 1 + g * count + threadIdx.x);
#pragma unroll
        for (int k = 0; k < 6; ++k) {
          sb[threadIdx.x][k] = box[k];
          bx[n * 6 + k] = box[k];
        }
      }
      __syncthreads();
    }
  }
}

// One thread per (instance, query) of the instances b0 .. b0 + nb; the trees in S are those of target instances tb0 .. (one when the
// target is not batched). Depth first from the root as closestPointKernel: both children's bounds, the nearer entered and the other
// pushed with its bound, re-checked when popped; a void box is never entered. The normal filter does not prune.
__global__ void __launch_bounds__(kClosestThreads) closestCloudKernel(const ClosestCloudArgs a, int b0, int nb, int tb0, CloudScratch S) {
  const long N = a.numSource, total = long(nb) * N;
  const int M = S.M, P = S.P;
  const bool normals = a.sourceNormals != nullptr;
  for (long it = long(blockIdx.x) * kClosestThreads + threadIdx.x; it < total; it += long(gridDim.x) * kClosestThreads) {
    const int i = int(it / N);
    const size_t qi = size_t(b0 + i) * N + size_t(it % N);
    const size_t ti = a.targetBatched ? size_t(b0 + i - tb0) : 0;
    const F3 p = ld3(a.source + 3 * qi);
    const F3 np = normals ? ld3(a.sourceNormals + 3 * qi) : f3(0.f, 0.f, 0.f);
    const float* x = S.sorted + ti * M * 3;
    const float* xn = normals ? S.sortedNormals + ti * M * 3 : nullptr;
    const int32_t* idx = S.index[0] + ti * M;
    const float* bx = S.boxes + ti * (2 * size_t(P) - 1) * 6;
    float best = a.maxDist2;
    int bestIndex = INT_MAX;
    int stackNode[kTreeStack];
    float stackLb[kTreeStack];
    int sp = 0, node = 0;
    bool go = finite3(p) && !boxVoid(bx) && !pruneBox(boxLowerBound(bx, p), best);
    while (go) {
      if (node < P - 1) {
        const int c0 = 2 * node + 1;
        const float* b0x = bx + size_t(c0) * 6;
        const float lb0 = boxLowerBound(b0x, p), lb1 = boxLowerBound(b0x + 6, p);
        const bool in0 = !boxVoid(b0x) && !pruneBox(lb0, best), in1 = !boxVoid(b0x + 6) && !pruneBox(lb1, best);
        if (in0 && in1) {
          const bool first1 = lb1 < lb0;
          stackNode[sp] = first1 ? c0 : c0 + 1;
          stackLb[sp] = first1 ? lb0 : lb1;
          ++sp;
          node = first1 ? c0 + 1 : c0;
          continue;
        }
        if (in0 || in1) {
          node = in0 ? c0 : c0 + 1;
          continue;
        }
      } else {
        const int m0 = (node - (P - 1)) * kLeafPoints, m1 = min(M, m0 + kLeafPoints);
        for (int m = m0; m < m1; ++m) {
          const float d2 = pointDistance2(p, ld3(x + 3 * size_t(m)));
          if (!(d2 <= best)) continue; // closerFace needs d2 <= best: the index is read only then
          const int j = idx[m];
          if (closerFace(d2, j, best, bestIndex) && (!normals || normalCompatible(np, ld3(xn + 3 * size_t(m)), a.maxNormalDot))) {
            best = d2;
            bestIndex = j;
          }
        }
      }
      go = false;
      while (sp > 0) {
        --sp;
        if (!pruneBox(stackLb[sp], best)) {
          node = stackNode[sp];
          go = true;
          break;
        }
      }
    }
    const bool found = bestIndex != INT_MAX;
    const size_t from = ((a.targetBatched ? size_t(b0 + i) : 0) * M + size_t(found ? bestIndex : 0)) * 3;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      a.outPoints[3 * qi + k] = found ? a.target[from + k] : 0.f;
      if (normals) a.outNormals[3 * qi + k] = found ? a.targetNormals[from + k] : 0.f;
    }
    a.outIndex[qi] = found ? bestIndex : -1;
  }
}

namespace {
// Builds the trees of target instances tb0 .. tb0 + nt into S (carved for at least nt instances)
cudaError_t buildCloudTrees(const ClosestCloudArgs& a, int tb0, int nt, int slice, const CloudScratch& S, cudaStream_t stream) {
  int g = 0;
  const long tileWork = long(slice) * S.tiles, pointWork = (long(slice) * S.M + kCloudThreads - 1) / kCloudThreads;
  auto grid = [&](auto kernel, long sliceWork, long work) -> cudaError_t { // sized for a whole slice, capped by this one's work
    const cudaError_t e = persistentGrid(kernel, kCloudThreads, 0, sliceWork, &g);
    g = int(std::max(1L, std::min<long>(g, work)));
    return e;
  };
  cudaError_t e = grid(cloudBoundsKernel, tileWork, long(nt) * S.tiles);
  if (e != cudaSuccess) return e;
  cloudBoundsKernel<<<g, kCloudThreads, 0, stream>>>(a, tb0, nt, S);
  if ((e = grid(cloudBoundsReduceKernel, slice, nt)) != cudaSuccess) return e;
  cloudBoundsReduceKernel<<<g, kCloudThreads, 0, stream>>>(nt, S);
  if ((e = grid(cloudCodeKernel, pointWork, (long(nt) * S.M + kCloudThreads - 1) / kCloudThreads)) != cudaSuccess) return e;
  cloudCodeKernel<<<g, kCloudThreads, 0, stream>>>(a, tb0, nt, S);
  for (int pass = 0; pass < kSortPasses; ++pass) {
    const int src = pass & 1;
    if ((e = grid(cloudSortCountKernel, tileWork, long(nt) * S.tiles)) != cudaSuccess) return e;
    cloudSortCountKernel<<<g, kCloudThreads, 0, stream>>>(nt, S, src, pass * kSortBits);
    if ((e = grid(cloudSortScanKernel, slice, nt)) != cudaSuccess) return e;
    cloudSortScanKernel<<<g, kCloudThreads, 0, stream>>>(nt, S);
    if ((e = grid(cloudSortScatterKernel, tileWork, long(nt) * S.tiles)) != cudaSuccess) return e;
    cloudSortScatterKernel<<<g, kCloudThreads, 0, stream>>>(nt, S, src, pass * kSortBits);
  }
  static_assert(kSortPasses % 2 == 0, "the sorted (code, index) end in keys[0] / index[0]");
  if ((e = grid(cloudGatherKernel, pointWork, (long(nt) * S.M + kCloudThreads - 1) / kCloudThreads)) != cudaSuccess) return e;
  cloudGatherKernel<<<g, kCloudThreads, 0, stream>>>(a, tb0, nt, S);
  int bottom = 0;
  while ((1 << bottom) < S.P) ++bottom;
  for (bool leaves = true; leaves || bottom > 0; leaves = false) {
    const int h = std::min(8, bottom);
    const long groups = (1L << bottom) >> h;
    if ((e = grid(cloudBoxKernel, long(slice) * groups, long(nt) * groups)) != cudaSuccess) return e;
    cloudBoxKernel<<<g, kCloudThreads, 0, stream>>>(nt, S, bottom, h, leaves);
    bottom -= h;
  }
  return cudaGetLastError();
}
} // namespace

cudaError_t launchClosestPointsOnCloud(const ClosestCloudArgs& a, cudaStream_t stream) {
  const long B = a.batch, N = a.numSource;
  if (B <= 0 || N <= 0) return cudaSuccess;
  const bool normals = a.sourceNormals != nullptr;
  if (a.numTarget <= 0) { // no target: index -1 and zeros everywhere
    cudaError_t e = cudaMemsetAsync(a.outIndex, 0xff, size_t(B) * N * sizeof(int32_t), stream);
    if (e == cudaSuccess) e = cudaMemsetAsync(a.outPoints, 0, size_t(B) * N * 3 * sizeof(float), stream);
    if (e == cudaSuccess && normals) e = cudaMemsetAsync(a.outNormals, 0, size_t(B) * N * 3 * sizeof(float), stream);
    return e;
  }
  CloudScratch S{};
  S.M = a.numTarget;
  S.tiles = (a.numTarget + kSortTile - 1) / kSortTile;
  S.P = cloudPadded(a.numTarget);
  const size_t perInstance = S.floats(normals) * sizeof(float);
  int queryGrid = 0;
  cudaError_t e = persistentGrid(closestCloudKernel, kClosestThreads, 0, (B * N + kClosestThreads - 1) / kClosestThreads, &queryGrid);
  if (e != cudaSuccess) return e;
  auto query = [&](int b0, int nb, int tb0, const CloudScratch& s) {
    const long blocks = (long(nb) * N + kClosestThreads - 1) / kClosestThreads;
    closestCloudKernel<<<int(std::min<long>(queryGrid, blocks)), kClosestThreads, 0, stream>>>(a, b0, nb, tb0, s);
    return cudaGetLastError();
  };
  // an unbatched target: one tree, then every instance's queries in one launch
  return forEachInstanceSlice(a.targetBatched ? int(B) : 1, perInstance, stream, [&](float* scratch, int slice, int b0, int nb) {
    CloudScratch s = S;
    s.carve(scratch, slice, normals);
    cudaError_t r = buildCloudTrees(a, a.targetBatched ? b0 : 0, nb, slice, s, stream);
    if (r != cudaSuccess) return r;
    return a.targetBatched ? query(b0, nb, b0, s) : query(0, int(B), 0, s);
  });
}

// ------------------------------------------------------------------------------------------------
// Input gradients of one Position / Orientation block, d/d input [grad_theta E . v] (ik_device.cuh tangent* / *InputGradient), in the
// per-instance frame of skeletonStateKernel:
//   lanes = parameters: theta, and v gated by the enabled set;  fkPasses with the DOF axes;  tangentPasses: each joint's own motion,
//   then level by level the parent's motion added;  lanes = constraints of the block.
// Every output element is written by one lane: no atomics, the result does not depend on the launch shape.
// ------------------------------------------------------------------------------------------------
template <int W>
__global__ void __launch_bounds__(32 * kSkelMaxWarps) inputGradientKernel(const InputGradientArgs a) {
  extern __shared__ __align__(16) float smem[];
  FunctionTables T = a.T;
  const WarpLanes<W> g = WarpLanes<W>::of(threadIdx.x >> 5, threadIdx.x & 31);
  const int groupsPerCta = (blockDim.x >> 5) / W;
  const int J = T.numJoints, n = T.numParams, nc = a.numConstraints;
  const int thF = int(skelAligned(n)), jsF = int(skelAligned(size_t(J) * kJointStateStride));
  const int perGroup = int(inputGradientFrame(J, n).floats);
  float* th = smem + size_t(g.group) * perGroup;
  float* vs = th + thF;
  float* js = vs + thF;
  float* tan = js + jsF;
  {
    TableStager stager{reinterpret_cast<uint32_t*>(smem + size_t(groupsPerCta) * perGroup)};
    characterTableList(stager, T);
    __syncthreads();
  }
  const EfDesc e = T.efs[T.units[a.unitBegin].ef];
  const bool position = a.kind == kUnitPosition;
  const int per = position ? 3 : 4;
  for (int b = blockIdx.x * groupsPerCta + g.group; b < a.batch; b += gridDim.x * groupsPerCta) {
    const float* theta = a.theta + size_t(b) * n;
    const float* dir = a.direction + size_t(b) * n;
    for (int i = g.lane; i < n; i += g.size) { th[i] = theta[i]; vs[i] = 0.f; }
    g.sync();
    for (int k = g.lane; k < a.numEnabled; k += g.size) { const int p = a.enabledList[k]; vs[p] = dir[p]; }
    fkPasses<true, false>(g, T, th, js);
    g.sync();
    tangentPasses(g, T, js, vs, tan);
    const float* targets = a.targets + size_t(b) * T.targetStride;
    const float* cweights = a.cweights + (T.weightsPerInstance ? size_t(b) * T.numWeights : 0);
    for (int c = g.lane; c < nc; c += g.size) {
      const UnitDesc& u = T.units[a.unitBegin + c];
      const size_t o = size_t(b) * nc + c;
      float* gW = a.gradWeights ? a.gradWeights + o : nullptr;
      float* gO = a.gradOffsets ? a.gradOffsets + o * per : nullptr;
      float* gT = a.gradTargets ? a.gradTargets + o * per : nullptr;
      if (position) positionInputGradient(u, e, js, tan, targets + u.targetOff, cweights[u.weightIdx], gW, gO, gT);
      else orientationInputGradient(u, e, js, tan, targets + u.targetOff, cweights[u.weightIdx], gW, gO, gT);
    }
    g.sync(); // the next instance overwrites th / vs / js / tan
  }
}

cudaError_t launchInputGradients(const InputGradientArgs& a, cudaStream_t stream, InstanceLaunchQuery* query) {
  return launchInstanceGroups(a, 0, kInstanceOpInputGradients, false, 0, stream, query, false,
                              [](auto W, const InstanceLaunch&) { return inputGradientKernel<W>; });
}

// ------------------------------------------------------------------------------------------------
// Implicit-function direction of solve_ik's backward (ik_jacobi.cuh): per instance v = (2 J_E^T J_E)^+ g, J v, the residual and the
// gradient RMS, from the K-major Jacobian the sweep wrote. A persistent grid with one CTA per instance in flight:
//   lanes = E: g, the gradient terms;  lanes = the triangle's columns, row by row: the float64 Gram K;  lanes = k: y
//   per sweep, per round-robin step: lanes = pairs: rotations, diagonal blocks, Q^T y, the log;  lanes = off-diagonal 2 x 2 blocks
//   lanes = k: the truncated inverse eigenvalues;  the log backwards, lanes = pairs;  lanes = E: v;  lanes = rows: J v
// K sits in shared memory when it fits, else in the CTA's global scratch slot (slot = blockIdx.x), which also holds the rotation log.
// Every sum is one lane's loop in a fixed order and there are no atomics: a result depends neither on the batch nor on the launch shape.
// ------------------------------------------------------------------------------------------------
constexpr int kJacobiThreads = 256;
constexpr size_t kJacobiScratchBudget = size_t(2) << 30; // the persistent grid is trimmed so that its scratch slots stay below 2 GiB

// shared memory besides K: y [k], g [n_E], v_E [n_E], c / s [h] (doubles), p / q [h] (ints)
static size_t implicitDirectionExtraBytes(int k, int nE) {
  const size_t h = size_t(jacobiPairs(k));
  return (sizeof(double) * (size_t(k) + 2 * size_t(nE) + 2 * h) + sizeof(int) * 2 * h + 15) / 16 * 16;
}

__global__ void __launch_bounds__(kJacobiThreads) implicitDirectionKernel(const ImplicitDirectionArgs a) {
  extern __shared__ __align__(16) double dsm[];
  __shared__ int rotated;
  __shared__ double floorK;
  const int tid = threadIdx.x, nt = blockDim.x;
  const int n = a.numParams, rows = a.rows, nE = a.numEnabled, ld = a.ldJ;
  const bool rowsSide = rows <= nE;
  const int k = rowsSide ? rows : nE, h = jacobiPairs(k), steps = jacobiSteps(k);
  const size_t kp = jacobiPackedSize(k);
  double* slot = a.scratch + size_t(blockIdx.x) * a.slotDoubles;
  double2* rlog = reinterpret_cast<double2*>(slot);
  double* K = a.gramInShared ? dsm : slot + jacobiLogDoubles(k);
  double* y = dsm + (a.gramInShared ? kp : 0);
  double* g = y + k;
  double* vE = g + nE;
  double* rc = vE + nE;
  double* rs = rc + h;
  int* rp = reinterpret_cast<int*>(rs + h);
  int* rq = rp + h;
  const int32_t* E = a.enabledList;
  for (int b = blockIdx.x; b < a.batch; b += gridDim.x) {
    const float* J = a.jacobian + size_t(b) * (n + 1) * ld;
    const float* res = J + size_t(n) * ld;
    for (int i = tid; i < nE; i += nt) g[i] = double(a.gradParameters[size_t(b) * n + E[i]]);
    if (a.residual)
      for (int r = tid; r < a.rowStride; r += nt) a.residual[size_t(b) * a.rowStride + r] = r < rows ? res[r] : 0.f;
    __syncthreads();
    for (int i = tid; i < nE; i += nt) {
      const double gi = jacobiGradient(J, ld, E, rows, res, i);
      vE[i] = gi * gi;
    }
    for (int r = 0; r < k; ++r)
      for (int c = r + tid; c < k; c += nt) K[jacobiPacked(r, c, k)] = jacobiGram(J, ld, E, nE, rows, rowsSide, r, c);
    for (int i = tid; i < k; i += nt) y[i] = jacobiRhs(J, ld, E, nE, rowsSide, g, i);
    __syncthreads();
    if (tid == 0) {
      double s = 0.0, d = 0.0;
      for (int i = 0; i < nE; ++i) s += vE[i];
      if (a.gradientRms) a.gradientRms[b] = nE > 0 ? float(sqrt(s / nE)) : 0.f;
      for (int i = 0; i < k; ++i) d = fmax(d, K[jacobiPacked(i, i, k)]);
      floorK = jacobiFloor(d);
    }
    __syncthreads();
    const double floor = floorK;
    int sweeps = 0;
    while (k > 1 && sweeps < kJacobiMaxSweeps) {
      if (tid == 0) rotated = 0;
      __syncthreads();
      for (int st = 0; st < steps; ++st) {
        double2* lg = rlog + (size_t(sweeps) * steps + st) * h;
        for (int t = tid; t < h; t += nt) {
          int p, q;
          jacobiPair(k, st, t, p, q);
          double c = 1.0, s = 0.0, tt = 0.0;
          if (q >= 0 && jacobiRotation(K[jacobiPacked(p, p, k)], K[jacobiPacked(q, q, k)], K[jacobiPacked(p, q, k)], floor, c, s, tt)) {
            jacobiRotateDiagonal(K, k, p, q, tt);
            jacobiRotateTransposed(y, p, q, c, s);
            rotated = 1;
          }
          rp[t] = p; rq[t] = q; rc[t] = c; rs[t] = s;
          lg[t] = make_double2(c, s);
        }
        __syncthreads();
        const int blocks = h * (h - 1) / 2;
        for (int L = tid; L < blocks; L += nt) {
          int i, j;
          jacobiBlock(L, i, j);
          if (rs[i] == 0.0 && rs[j] == 0.0) continue; // both identity
          jacobiRotateBlock(K, k, rp[i], rq[i], rc[i], rs[i], rp[j], rq[j], rc[j], rs[j]);
        }
        __syncthreads();
      }
      const bool any = rotated != 0;
      __syncthreads(); // every lane has read the flag before the next sweep clears it
      if (!any) break; // a sweep without a rotation: converged (its log entries are identities and are not replayed)
      ++sweeps;
    }
    for (int i = tid; i < k; i += nt) y[i] = jacobiScale(K[jacobiPacked(i, i, k)], y[i], rowsSide);
    __syncthreads();
    for (int st = sweeps * steps - 1; st >= 0; --st) { // z <- Q z: the rotations in reverse order
      const double2* lg = rlog + size_t(st) * h;
      const int step = st % steps;
      for (int t = tid; t < h; t += nt) {
        const double2 cs = lg[t];
        if (cs.y == 0.0) continue;
        int p, q;
        jacobiPair(k, step, t, p, q);
        jacobiRotateForward(y, p, q, cs.x, cs.y);
      }
      __syncthreads();
    }
    for (int i = tid; i < nE; i += nt) vE[i] = jacobiDirection(J, ld, E, rows, rowsSide, y, i);
    float* dir = a.direction ? a.direction + size_t(b) * n : nullptr;
    if (dir)
      for (int c = tid; c < n; c += nt) dir[c] = 0.f;
    __syncthreads();
    if (dir)
      for (int i = tid; i < nE; i += nt) dir[E[i]] = float(vE[i]);
    if (a.jacobianDirection)
      for (int r = tid; r < a.rowStride; r += nt)
        a.jacobianDirection[size_t(b) * a.rowStride + r] = r < rows ? float(jacobiJv(J, ld, E, nE, vE, r)) : 0.f;
    __syncthreads(); // the next instance overwrites g / v_E / y / K
  }
}

cudaError_t implicitDirectionConfigure(const ImplicitDirectionArgs& a, ImplicitDirectionConfig& cfg) {
  const int k = std::min(a.rows, a.numEnabled);
  const size_t extra = implicitDirectionExtraBytes(k, a.numEnabled), gram = sizeof(double) * jacobiPackedSize(k);
  cfg.gramInShared = extra + gram <= size_t(g_maxSmemOptin);
  cfg.smem = extra + (cfg.gramInShared ? gram : 0);
  cfg.slotDoubles = (jacobiLogDoubles(k) + (cfg.gramInShared ? 0 : jacobiPackedSize(k)) + 1) & ~size_t(1); // slots stay 16-byte aligned
  long work = std::max(a.batch, 1);
  if (cfg.slotDoubles > 0) work = std::min(work, long(std::max<size_t>(1, kJacobiScratchBudget / (sizeof(double) * cfg.slotDoubles))));
  return persistentGrid(implicitDirectionKernel, kJacobiThreads, cfg.smem, work, &cfg.grid);
}

cudaError_t launchImplicitDirection(const ImplicitDirectionArgs& a, const ImplicitDirectionConfig& cfg, cudaStream_t stream) {
  if (a.batch <= 0) return cudaSuccess;
  implicitDirectionKernel<<<cfg.grid, kJacobiThreads, cfg.smem, stream>>>(a);
  return cudaGetLastError();
}


// ------------------------------------------------------------------------------------------------
// K2 (SIMT validation path): H[i][j] = sum_k J[k][cols[i]] J[k][cols[j]] for i >= j; g = J^T r.
// grid = (lower-triangular 64x64 tile pairs, B); 256 threads, 4x4 outputs per thread.
// ------------------------------------------------------------------------------------------------
constexpr int kJtjTile = 64;
constexpr int kJtjKc = 32;

__global__ void __launch_bounds__(256) jtjSimtKernel(const JtJArgs a) {
  const int b = blockIdx.y;
  if (a.active != nullptr && a.active[b] == 0) return;
  // decode lower-triangular tile index
  int t = blockIdx.x, ti = 0;
  while ((ti + 1) * (ti + 2) / 2 <= t) ++ti;
  const int tj = t - ti * (ti + 1) / 2;
  __shared__ float As[kJtjTile][kJtjKc + 1];
  __shared__ float Bs[kJtjTile][kJtjKc + 1];
  __shared__ float rs[kJtjKc];
  const float* J = a.jacobian + size_t(b) * (a.numCols + 1) * a.ldJ;
  const float* r = J + size_t(a.numCols) * a.ldJ;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  float gacc = 0.f;
  const bool diag = (ti == tj);
  for (int k0 = 0; k0 < a.kRows; k0 += kJtjKc) {
    // load 64 columns x 32 rows for both operands (lane -> consecutive k: coalesced 128B per column)
    for (int idx = threadIdx.x; idx < kJtjTile * kJtjKc; idx += 256) {
      const int c = idx / kJtjKc, kk = idx % kJtjKc;
      const int ia = ti * kJtjTile + c, ib = tj * kJtjTile + c;
      const int k = k0 + kk;
      As[c][kk] = (ia < a.ns && k < a.kRows) ? J[size_t(ia) * a.ldJ + k] : 0.f;
      Bs[c][kk] = (ib < a.ns && k < a.kRows) ? J[size_t(ib) * a.ldJ + k] : 0.f;
    }
    if (threadIdx.x < kJtjKc) rs[threadIdx.x] = (k0 + threadIdx.x < a.kRows) ? r[k0 + threadIdx.x] : 0.f;
    __syncthreads();
#pragma unroll 8
    for (int kk = 0; kk < kJtjKc; ++kk) {
      float av[4], bv[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) av[i] = As[ty * 4 + i][kk];
#pragma unroll
      for (int j = 0; j < 4; ++j) bv[j] = Bs[tx * 4 + j][kk];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    if (diag && threadIdx.x < kJtjTile)
      for (int kk = 0; kk < kJtjKc; ++kk) gacc = fmaf(As[threadIdx.x][kk], rs[kk], gacc);
    __syncthreads();
  }
  float* H = a.H + size_t(b) * a.hStride;
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int gi = ti * kJtjTile + ty * 4 + i, gj = tj * kJtjTile + tx * 4 + j;
      if (gi < a.ns && gj <= gi) { H[size_t(gj) * a.ldH + gi] = acc[i][j]; H[size_t(gi) * a.ldH + gj] = acc[i][j]; }
    }
  if (diag && threadIdx.x < kJtjTile) {
    const int gi = ti * kJtjTile + threadIdx.x;
    if (gi < a.ns) {
      H[size_t(gi) * a.ldH + a.ns] = gacc; H[size_t(a.ns) * a.ldH + gi] = gacc;
      if (a.g != nullptr) a.g[size_t(b) * a.ldG + gi] = gacc;
    }
  }
}

cudaError_t launchJtJSimt(const JtJArgs& a, cudaStream_t stream) {
  const int tiles = (a.ns + kJtjTile - 1) / kJtjTile;
  dim3 grid(tiles * (tiles + 1) / 2, a.batch);
  jtjSimtKernel<<<grid, 256, 0, stream>>>(a);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// K3: one CTA per instance. Matrix A = [H + lambda I ; g^T] ((ns+1) x lda, row-major, lower part)
// is factored in place with Eigen's LLT structure (ik_chol.cuh); the appended row turns into
// y = L^-1 g for free; back substitution gives delta.
// ------------------------------------------------------------------------------------------------
// The SolverT bookkeeping of instance b after iteration s.iteration (solver.cpp:92-122), by one thread
__device__ __forceinline__ void finishIteration(const SolveState& s, int b) {
  const double error = s.errors[b], last = s.lastErrors[b];
  if (s.history != nullptr) s.history[size_t(b) * s.maxIterations + s.iteration] = error;
  const bool stop = solveStops(error, last, s.iteration, s.minIterations, s.maxIterations, s.threshold);
  s.iterations[b] = s.iteration + 1;
  if (stop) s.active[b] = 0;
  else { s.lastErrors[b] = error; atomicAdd(s.activeCount, 1); }
}

// Common tail of both Cholesky kernels: delta, parameter update (skeleton_solver_function.cpp:153-159),
// g.delta for the subset line search, status and the SolverT bookkeeping (solver.cpp:92-122).
// dsub / gsub are indexed by subset position. Every thread of the CTA must call it.
// dsub: the step per device column, or (slotOf != nullptr) per elimination slot with slotOf[i] = slot of device column i
__device__ void cholFinish(const CholArgs& a, int b, int n, const float* dsub, const float* gsub, bool failed, const int32_t* slotOf = nullptr) {
  const int tid = threadIdx.x;
  float* theta = a.theta + size_t(b) * a.ldTheta;
  float part = 0.f;
  for (int i = tid; i < n; i += blockDim.x) {
    const int c = a.cols[i];
    const float d = c >= 0 ? dsub[slotOf != nullptr ? slotOf[i] : i] : 0.f; // c < 0: all-zero alignment column of the scheduled layout (ik_chol_sched.h)
    a.delta[size_t(b) * n + i] = d;
    if (c >= 0) part += gsub[i] * d;
    if (a.applyUpdate && c >= 0) theta[c] -= d;
  }
  if (a.gradDotDelta != nullptr) {
    __shared__ float red[32];
    for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
    if ((tid & 31) == 0) red[tid >> 5] = part;
    __syncthreads();
    if (tid == 0) {
      float s = 0.f;
      for (int w = 0; w < int(blockDim.x >> 5); ++w) s += red[w];
      a.gradDotDelta[b] = s;
    }
  }
  if (tid == 0) {
    if (failed && a.state.status[b] == 0) a.state.status[b] = 1; // MB2_INSTANCE_CHOLESKY_BREAKDOWN
    if (a.bookkeeping) finishIteration(a.state, b);
  }
}

template <int NB>
__global__ void __launch_bounds__(kCholThreads) choleskyKernel(const CholArgs a, const int useSmemMatrix) {
  extern __shared__ float smem[];
  const int b = blockIdx.x;
  if (a.state.active[b] == 0) return;
  const int n = a.ns;
  const int tid = threadIdx.x;
  float* Hg = a.H + size_t(b) * a.hStride;
  CholCtx ctx;
  ctx.n = n;
  int ldp = ((n + 1 + 3) & ~3) + 4;
  float* P = smem;                       // [NB][ldp] transposed panel
  float* gsave = P + NB * ldp;           // [n] copy of Jtr (for g.delta)
  int* flags = reinterpret_cast<int*>(gsave + ((n + 3) & ~3)); // [0] = fail index+1
  float* As = reinterpret_cast<float*>(flags + 4);
  if (useSmemMatrix) {
    ctx.lda = n | 1;
    ctx.A = As;
    // source is column-major (coalesced along i); smem target is row-major with odd stride
    for (int idx = tid; idx < (n + 1) * n; idx += kCholThreads) {
      const int j = idx / (n + 1), i = idx - j * (n + 1);
      if (i >= j) {
        float v = Hg[size_t(j) * a.ldH + i];
        if (i == j) v += a.regularization; // gauss_newton_solver.cpp:248
        As[i * ctx.lda + j] = v;
      }
    }
  } else {
    // matrix too large for shared memory: factor in place in global memory (L2-resident). K2 wrote the lower
    // triangle column-major (element (i,j) at [j*ldH + i]); mirror it so that A(i,j) = Hg[i*ldH + j] reads row-major.
    ctx.lda = a.ldH;
    ctx.A = Hg;
    for (int idx = tid; idx < (n + 1) * n; idx += kCholThreads) {
      const int j = idx / (n + 1), i = idx - j * (n + 1);
      if (i > j) Hg[size_t(i) * a.ldH + j] = Hg[size_t(j) * a.ldH + i];
    }
    for (int i = tid; i < n; i += kCholThreads) Hg[size_t(i) * a.ldH + i] += a.regularization;
  }
  ctx.P = P;
  ctx.ldp = ldp;
  ctx.fail = flags;
  if (tid == 0) flags[0] = 0;
  for (int i = tid; i < n; i += kCholThreads) gsave[i] = Hg[size_t(i) * a.ldH + n];
  __syncthreads();

  const int blockSize = cholBlockSize(n, NB);
  for (int k = 0; k < n; k += blockSize) {
    const int bs = min(blockSize, n - k);
    if (tid < 32) { // unblocked LLT of the diagonal block by warp 0 (left-looking, Eigen llt_inplace::unblocked)
      for (int jj = 0; jj < bs; ++jj) {
        const float x = cholDiagPivot(ctx, k, jj);
        __syncwarp();
        if (!(x > 0.f)) { if (tid == 0) flags[0] = k + jj + 1; break; }
        cholDiagColumn(ctx, k, bs, jj, x, tid);
        __syncwarp();
      }
    }
    __syncthreads();
    if (flags[0] != 0) break; // Eigen returns early: the rest of the matrix stays as it is
    cholPanelSolve<NB>(ctx, k, bs, tid, kCholThreads);
    __syncthreads();
    cholTrailingUpdate<NB>(ctx, k, bs, tid, kCholThreads);
    __syncthreads();
  }
  float* y = ctx.A + size_t(n) * ctx.lda; // appended row
  if (flags[0] != 0) {
    // finish the forward substitution with whatever the lower triangle holds (LLT::solve after a failed compute)
    if (tid == 0) cholForwardFrom(ctx, cholCompletedColumns(flags[0] - 1, blockSize), y);
    __syncthreads();
  }
  // back substitution L^T x = y, 32 columns at a time from the bottom
  for (int i0 = ((n - 1) / 32) * 32; i0 >= 0; i0 -= 32) {
    const int nb = min(32, n - i0);
    if (tid < 32) {
      float yv = tid < nb ? y[i0 + tid] : 0.f;
      float dinv = tid < nb ? 1.f / ctx.A[size_t(i0 + tid) * ctx.lda + i0 + tid] : 0.f;
      for (int kk = nb - 1; kk >= 0; --kk) {
        const float xk = __shfl_sync(0xffffffffu, yv, kk) * __shfl_sync(0xffffffffu, dinv, kk);
        if (tid == kk) yv = xk;
        else if (tid < kk) yv -= ctx.A[size_t(i0 + kk) * ctx.lda + i0 + tid] * xk;
      }
      if (tid < nb) y[i0 + tid] = yv;
    }
    __syncthreads();
    for (int i = tid; i < i0; i += kCholThreads) {
      float s = y[i];
      for (int kk = 0; kk < nb; ++kk) s -= ctx.A[size_t(i0 + kk) * ctx.lda + i] * y[i0 + kk];
      y[i] = s;
    }
    __syncthreads();
  }
  cholFinish(a, b, n, y, gsave, flags[0] != 0);
}

cudaError_t launchCholesky(const CholArgs& a, int NB, bool inSmem, cudaStream_t stream) {
  const size_t smem = cholSmemBytes(a.ns, NB, inSmem);
  if (NB != 8 && NB != 16 && NB != 32) return cudaErrorInvalidConfiguration;
  cudaError_t e = cudaSuccess;
#define MB2_LAUNCH_CHOL(NBV)                                                                                   \
  e = cudaFuncSetAttribute(choleskyKernel<NBV>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem));       \
  if (e != cudaSuccess) return e;                                                                              \
  choleskyKernel<NBV><<<a.batch, kCholThreads, smem, stream>>>(a, inSmem ? 1 : 0);
  if (NB == 8) { MB2_LAUNCH_CHOL(8) } else if (NB == 16) { MB2_LAUNCH_CHOL(16) } else { MB2_LAUNCH_CHOL(32) }
#undef MB2_LAUNCH_CHOL
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// K2s: tile-sparse Gram. A skeleton Jacobian is mostly structural zeros (a row only touches the parameters of one
// root-to-constraint chain), so the stored 16x16 tiles of J^T J are accumulated from the non-zero 4-row x 16-column strips only
// (GramPlan): ~20x fewer multiply-adds than the dense product, fp32-class accuracy (three-term TF32 split on mma.sync, the lo*lo term dropped: ~2^-21 relative). One CTA per instance: every strip arrives as one
// TMA box of the K-major Jacobian, a warp owns a tile at a time, the output is already in the Cholesky kernel's tile layout.
// ------------------------------------------------------------------------------------------------
constexpr int kGramThreads = 32 * kGramWarps;

// kThreads = 256 (eight warps, the width the tile-order table is dealt for), or 512 when the strips of an instance leave room for only
// one CTA per SM anyway (bodyhands300: 155 KB): the sixteen warps then walk the same table two rounds at a time.
template <int kThreads>
__global__ void __launch_bounds__(kThreads) gramTilesKernel(const GramArgs a) {
  extern __shared__ __align__(16) float gramSmem[];
  const int b = blockIdx.x;
  if (a.active != nullptr && a.active[b] == 0) return;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, hw = tid >> 4, hl = tid & 15;
  float* strips = gramSmem + (((128u - (smemAddr(gramSmem) & 127u)) & 127u) >> 2);
  float* resid = strips + a.residOff;
  // smem: [strips | residual] as in global memory, then the all-zero strip that pads odd pair lists (index zeroStrip), barrier, tables
  float* zero = strips + a.stripStride;
  unsigned long long* bar = reinterpret_cast<unsigned long long*>(zero + 64);
  const uint32_t barAddr = smemAddr(bar);
  const uint32_t total = uint32_t(a.stripStride) * 4u;
  if (tid < 64) zero[tid] = 0.f;
  if (tid == 0) {
    mbarInit(barAddr, 1);
    fenceBarrierInit();
    mbarExpectTx(barAddr, total);
    const char* src = reinterpret_cast<const char*>(a.strips + size_t(b) * a.stripStride);
    for (uint32_t off = 0; off < total; off += 16384u) bulkLoad(smemAddr(strips) + off, src + off, total - off < 16384u ? total - off : 16384u, barAddr);
  }
  // the plan tables are read in dependent chains (tile -> pair range -> strips): stage them in shared memory while the copy is in flight
  int32_t* tab = reinterpret_cast<int32_t*>(bar + 2);
  for (int i = tid; i < a.blobInts; i += kThreads) tab[i] = __ldg(a.blob + i);
  __syncthreads();
  mbarWaitRelaxed(barAddr, 0);
  const int32_t* tileOrder = tab + a.offTileOrder, *tileQuadStart = tab + a.offTilePairStart, *quads = tab + a.offPairA; // (blob tables are 16-byte aligned)
  const int32_t* colStripStart = tab + a.offColStripStart, *colStrip = tab + a.offColStrip, *stripRow = tab + a.offStripRow, *tileInfo = tab + a.offTileInfo;
  float* out = a.out + size_t(b) * a.outStride;
  for (int ti = warp; ti < a.numOrder; ti += kThreads / 32) { // ([rounds][8] table: warp w + 8 takes the odd rounds of warp w's list)
    const int t = tileOrder[ti];
    if (t < 0) continue;
    float acc[2][4];
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
    gramTileAccumulate(strips, quads, tileQuadStart[t], tileQuadStart[t + 1], lane, acc);
    gramTileStore(out + size_t(t) * 256, acc, tileInfo[t], a.regularization, lane);
  }
  float* y = out + size_t(a.numTiles) * 256;
  for (int K = hw; K < a.numTileCols; K += kThreads / 16)
    y[16 * K + hl] = gramVectorEntry(strips, resid, colStrip, stripRow, colStripStart[K], colStripStart[K + 1], hl);
}

cudaError_t launchGramTiles(const GramArgs& a, int threads, cudaStream_t stream) {
  const size_t smem = gramTilesSmemBytes(a.stripStride, a.blobInts);
  if (smem > size_t(g_maxSmemOptin) || (a.stripStride & 3) != 0 || (threads != 256 && threads != 512)) return cudaErrorInvalidConfiguration;
  const bool wide = threads == 512;
  cudaError_t e = wide ? cudaFuncSetAttribute(gramTilesKernel<512>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem))
                       : cudaFuncSetAttribute(gramTilesKernel<kGramThreads>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem));
  if (e != cudaSuccess) return e;
  if (wide) gramTilesKernel<512><<<a.batch, 512, smem, stream>>>(a);
  else gramTilesKernel<kGramThreads><<<a.batch, kGramThreads, smem, stream>>>(a);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// K3 (scheduled): level-scheduled tile-sparse Cholesky of the permuted system (ik_chol_sched.h).
// One CTA per instance; tiles, right-hand side and scratch live in shared memory (<= ~64 KB for the
// humanoid rig => several CTAs per SM hide each other's latencies).
// ------------------------------------------------------------------------------------------------
// 256 threads and three CTAs per SM when the tiles of one instance take a third of shared memory (humanoid-size rigs); 512 threads in
// the single resident CTA when one instance needs more than half of it (body + hands)

// kProfile: per-phase cycle counters of block 0 (MB2_CHOL_PROFILE=1); a separate instantiation so that the production kernel does not
// carry the counters in its register budget
template <int kSchedThreads, bool kProfile>
__global__ void __launch_bounds__(kSchedThreads, kSchedThreads == 256 ? 3 : 1) choleskyScheduledKernel(const __grid_constant__ CUtensorMap hmap, const CholArgs a, const CholSchedDev Sg) {
  extern __shared__ __align__(16) float smemRaw[];
  const int b = blockIdx.x;
  if (a.state.active[b] == 0) return;
  const int n = a.ns, tid = threadIdx.x;
  const int warp = tid >> 5, lane = tid & 31, hw = tid >> 4, hl = tid & 15;
  const unsigned hmask = 0xFFFFu << (16 * ((tid >> 4) & 1));
  float* tiles = smemRaw + (((1024u - (smemAddr(smemRaw) & 1023u)) & 1023u) >> 2); // 1 KB aligned in the shared window (TMA swizzle atom)
  float* y = tiles + size_t(Sg.numTiles) * 256;
  float* gsub = y + Sg.nPad;
  float* dsub = gsub + ((n + 3) & ~3);
  int32_t* blob = reinterpret_cast<int32_t*>(dsub + ((n + 3) & ~3));
  int* flags = reinterpret_cast<int*>(blob + ((Sg.blobInts + 3) & ~3));
  unsigned long long* bar = reinterpret_cast<unsigned long long*>(flags + 2);
  long long pc[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0}, pt = clock64();
#define MB2_PROF(k) if constexpr (kProfile) { const long long now = clock64(); pc[k] += now - pt; pt = now; }
  // Prologue: everything this instance reads arrives asynchronously on one mbarrier -- the schedule tables and J^T r as 1-D
  // bulk copies, every stored tile as one TMA box (16 rows x 64 bytes of the row-major upper triangle of H, written
  // as swizzled 64-byte rows: SWIZZLE_64B, see tmaBoxIdx; cholConvertBox then rewrites each box in the fragment layout).
  const uint32_t barAddr = smemAddr(bar);
  const uint32_t blobBytes = uint32_t((Sg.blobInts + 3) & ~3) * 4u, gBytes = uint32_t(a.ldG) * 4u;
  const bool fromGram = a.tilesIn != nullptr; // tiles (+ lambda, identity extension) and the slot-ordered J^T r come ready-made from the Gram kernel
  const uint32_t tileBytes = uint32_t(Sg.numTiles) * 1024u, yBytes = uint32_t(Sg.nPad) * 4u;
  if (tid == 0) {
    flags[0] = 0;
    mbarInit(barAddr, 1);
    fenceBarrierInit();
    mbarExpectTx(barAddr, blobBytes + tileBytes + (fromGram ? yBytes : gBytes));
  }
  __syncthreads();
  if (fromGram) {
    if (tid == 0) {
      bulkLoad(smemAddr(blob), Sg.blob, blobBytes, barAddr);
      const float* src = a.tilesIn + size_t(b) * a.tilesStride;
      const uint32_t total = tileBytes + yBytes; // y follows the tiles in both layouts
      for (uint32_t off = 0; off < total; off += 16384u)
        bulkLoad(smemAddr(tiles) + off, reinterpret_cast<const char*>(src) + off, total - off < 16384u ? total - off : 16384u, barAddr);
    }
  } else {
    if (tid == 0) {
      bulkLoad(smemAddr(blob), Sg.blob, blobBytes, barAddr);
      bulkLoad(smemAddr(gsub), a.g + size_t(b) * a.ldG, gBytes, barAddr);
    }
    for (int t = tid; t < Sg.numTiles; t += kSchedThreads) { // one thread per tile: the table reads overlap, the compiler serialises the TMA issue per warp
      const int gi0 = __ldg(Sg.tileInfo + 3 * t), gj0 = __ldg(Sg.tileInfo + 3 * t + 1);
      tmaLoad3d(smemAddr(tiles + size_t(t) * 256), &hmap, gi0, gj0, b, barAddr);
    }
  }
  MB2_PROF(6)
  mbarWaitRelaxed(barAddr, 0); // 256 spinning threads would take issue slots from the other CTAs of the SM
  MB2_PROF(7)
  const CholSchedDev S = rebaseSchedule(Sg, blob);
  if (fromGram) {
    for (int s = tid; s < S.nPad; s += kSchedThreads) {
      const int p = S.perm[s];
      if (p >= 0) gsub[p] = y[s];
    }
  } else {
    // the boxes landed as swizzled 64-byte rows: a warp per tile turns them into the fragment layout (identity extension on padding)
    for (int t = warp; t < S.numTiles; t += kSchedThreads / 32) cholConvertBox(tiles + size_t(t) * 256, S.tileInfo[3 * t + 2], lane);
    for (int s = tid; s < S.nPad; s += kSchedThreads) {
      const int p = S.perm[s];
      y[s] = p >= 0 ? gsub[p] : 0.f;
    }
  }
  __syncthreads();
  MB2_PROF(8)
  if (!fromGram)
    for (int s = tid; s < S.nPad; s += kSchedThreads)
      if (S.perm[s] >= 0) tiles[size_t(S.diagTile[s >> 4]) * 256 + tileIdx(s & 15, s & 15)] += a.regularization; // gauss_newton_solver.cpp:248
  __syncthreads();
  MB2_PROF(0)

  for (int L = 0; L < S.numLevels; ++L) {
    // A: diagonal tiles of this level (one warp each) + forward solve of their rhs block
    for (int ci = S.levelColStart[L] + warp; ci < S.levelColStart[L + 1]; ci += kSchedThreads / 32) {
      const int K = S.levelCols[ci];
      cholDiagTile(tiles + size_t(S.diagTile[K]) * 256, y + 16 * K, lane, a.regularization, flags);
    }
    __syncthreads();
    MB2_PROF(1)
    // B: panel tiles
    for (int pi = S.levelPanelStart[L] + warp; pi < S.levelPanelStart[L + 1]; pi += kSchedThreads / 32) {
      float* ptile = tiles + size_t(S.panelTile[pi]) * 256;
      float x[2][4];
      cholPanelProduct(ptile, tiles + size_t(S.panelDiag[pi]) * 256, lane, x);
      cholPanelStore(ptile, lane, x);
    }
    __syncthreads();
    MB2_PROF(2)
    // C: update tasks (warp each) and rhs updates (half-warp each)
    {
      const int32_t* oStart = kSchedThreads == 256 ? S.levelOrderStart8 : S.levelOrderStart16, *order = kSchedThreads == 256 ? S.taskOrder8 : S.taskOrder16;
      for (int oi = oStart[L] + warp; oi < oStart[L + 1]; oi += kSchedThreads / 32) { const int ti = order[oi]; if (ti >= 0) cholUpdateTask(tiles, S, ti, lane); }
    }
    for (int vi = S.levelVTaskStart[L] + hw; vi < S.levelVTaskStart[L + 1]; vi += kSchedThreads / 16) cholVectorTask(tiles, y, S, vi, hl);
    __syncthreads();
    MB2_PROF(3)
  }
  for (int L = S.numLevels - 1; L >= 0; --L) {
    for (int ci = S.levelColStart[L] + warp; ci < S.levelColStart[L + 1]; ci += kSchedThreads / 32) cholBackwardColumn(tiles, y, S, S.levelCols[ci], lane);
    __syncthreads();
  }
  MB2_PROF(4)
  for (int i = tid; i < S.nPad; i += kSchedThreads) { const int p = S.perm[i]; if (p >= 0) dsub[p] = y[i]; }
  __syncthreads();
  cholFinish(a, b, n, dsub, gsub, flags[0] != 0);
  MB2_PROF(5)
  if (kProfile && b == 0 && tid == 0)
    printf("chol-profile (cycles, block 0): blob %lld issue %lld wait %lld lambda %lld diag %lld panel %lld update %lld backward %lld finish %lld | levels %d tiles %d\n", pc[6], pc[7],
           pc[8], pc[0], pc[1], pc[2], pc[3], pc[4], pc[5], S.numLevels, S.numTiles);
#undef MB2_PROF
}

cudaError_t launchCholeskyScheduled(const CholArgs& a, const CholSchedDev& sched, int threads, cudaStream_t stream) {
  const size_t smem = choleskyScheduledSmemBytes(a.ns, sched.nPad, sched.numTiles, sched.blobInts);
  if (smem > size_t(g_maxSmemOptin) || (threads != 256 && threads != 512)) return cudaErrorInvalidConfiguration;
  const bool wide = threads == 512;
  const bool prof = (a.profile & 1) != 0;
  cudaError_t e;
  if (wide) e = prof ? cudaFuncSetAttribute(choleskyScheduledKernel<512, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem))
                     : cudaFuncSetAttribute(choleskyScheduledKernel<512, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem));
  else e = prof ? cudaFuncSetAttribute(choleskyScheduledKernel<256, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem))
                : cudaFuncSetAttribute(choleskyScheduledKernel<256, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem));
  if (e != cudaSuccess) return e;
  if (a.tilesIn == nullptr && (a.g == nullptr || a.ldG != cholGradientLd(a.ns))) return cudaErrorInvalidValue;
  if ((a.ldH & 3) != 0 || (a.hStride & 3) != 0 || (a.tilesStride & 3) != 0) return cudaErrorInvalidValue;
  CUtensorMap hmap; // H as [batch][ns + 1][ldH]; one 16 x 16 box per stored tile (unused, but still a valid map, when the tiles come from the Gram kernel)
  const bool fromGram = a.tilesIn != nullptr;
  const uint64_t dims[3] = {uint64_t(fromGram ? 256 : a.ldH), uint64_t(fromGram ? sched.numTiles : a.ns + 1), uint64_t(a.batch)};
  const uint64_t strides[2] = {uint64_t(fromGram ? 256 : a.ldH) * sizeof(float), uint64_t(fromGram ? a.tilesStride : a.hStride) * sizeof(float)};
  const uint32_t box[3] = {16u, 16u, 1u};
  e = makeTensorMap3d(&hmap, fromGram ? a.tilesIn : a.H, dims, strides, box, 64);
  if (e != cudaSuccess) return e;
  if (wide && prof) choleskyScheduledKernel<512, true><<<a.batch, 512, smem, stream>>>(hmap, a, sched);
  else if (wide) choleskyScheduledKernel<512, false><<<a.batch, 512, smem, stream>>>(hmap, a, sched);
  else if (prof) choleskyScheduledKernel<256, true><<<a.batch, 256, smem, stream>>>(hmap, a, sched);
  else choleskyScheduledKernel<256, false><<<a.batch, 256, smem, stream>>>(hmap, a, sched);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// K2s + K3 fused (default on the tile path): one CTA per instance, four CTAs per SM.
//   prologue   strips + residual of the instance arrive as bulk copies on one mbarrier; the CTA takes a parking slot
//   Gram       a warp owns a tile at a time (longest-first assignment); a finished tile that lies beyond the strips is stored at
//              once, one that would overwrite strips still being read is parked in the CTA's scratch slot (L2-only stores)
//   restore    parked accumulators -> 16x16 tiles of J^T J + lambda I in the Cholesky layout, over the dead strips; slot released
//   Cholesky   level-scheduled tile factorisation, both substitutions, theta -= delta, SolverT bookkeeping (cholFinish)
// The stored tiles (0.45 GB per iteration on the cfg3 shard) never exist in HBM and the second launch is gone.
// ------------------------------------------------------------------------------------------------
// A free parking slot (see GramCholArgs): the search starts at a word that depends on the instance so that the CTAs of a wave do not
// all contend for the first word.
__device__ int acquireParkSlot(uint32_t* words, int numWords, int start) {
  for (int w = start % numWords;; w = (w + 1 == numWords) ? 0 : w + 1) {
    uint32_t freeBits = ~__ldcg(words + w);
    while (freeBits != 0u) {
      const int bit = __ffs(freeBits) - 1;
      if ((atomicOr(words + w, 1u << bit) & (1u << bit)) == 0u) return 32 * w + bit;
      freeBits &= freeBits - 1u;
    }
  }
}

// Shared memory holds only what is per instance: the strip / tile union, the right-hand side in slot order and J^T r per device column
// (cfg3: 54.9 KB), so that FOUR CTAs fit on an SM (with the 1 KB reserved per block, 64 registers per thread). That leaves ~28 KB of
// L1 per SM, so neither the plan nor the parked tiles go through it:
//   * the plan (GramCholTables: about 2 k entries on cfg3) is read from the kernel's parameter block through the constant cache (Tables =
//     GramCholParamTables), or from global memory when it does not fit there (GramCholGlobalTables). Every item of every phase is
//     one warp-uniform read of a pre-resolved record, where the schedule blob took a chain of two or three dependent reads;
//   * a parked tile goes to the CTA's scratch slot with L2-only stores and comes back with L2-only loads: no stack frame, and
//     the slots of the resident CTAs (cfg3: 544 x 30 KB) stay in L2.
// The per-instance critical path is a chain of dependent phases no wider than a few warps: instances in flight per SM are what
// buys throughput. The per-tile arithmetic is that of gramTilesKernel + choleskyScheduledKernel (the same device functions).
template <bool kProfile, class Tables>
__global__ void __launch_bounds__(kGramThreads, kGramCholCtasPerSm) gramCholeskyKernel(const GramCholArgs a, const CholSchedDev S, const __grid_constant__ Tables P) {
  extern __shared__ __align__(16) float gcSmem[];
  const GramArgs& g = a.g;
  const CholArgs& c = a.c;
  const int b = blockIdx.x;
  if (c.state.active[b] == 0) return;
  const int n = c.ns, tid = threadIdx.x;
  const int warp = tid >> 5, lane = tid & 31, hw = tid >> 4, hl = tid & 15;
  constexpr int kWarps = kGramThreads / 32;
  float* U = gcSmem + (((128u - (smemAddr(gcSmem) & 127u)) & 127u) >> 2); // strips | residual | zero strip, later the tiles
  const size_t tileFloats = size_t(S.numTiles) * 256, sweepFloats = g.stripStride + 64;
  const size_t uni = ((tileFloats > sweepFloats ? tileFloats : sweepFloats) + 3) & ~size_t(3);
  float* strips = U;
  float* resid = U + g.residOff;
  float* tiles = U;
  float* y = U + uni;
  float* gsub = y + S.nPad;
  int* flags = reinterpret_cast<int*>(gsub + ((n + 3) & ~3)); // [0] breakdown, [1] parking slot
  unsigned long long* bar = reinterpret_cast<unsigned long long*>(flags + 4);
  const uint16_t* tab = P.tab;
  const GramCholLayout& L = P.L;
  long long pc[8] = {0, 0, 0, 0, 0, 0, 0, 0}, pt = 0;
  if constexpr (kProfile) pt = clock64();
#define MB2_GC(k) if constexpr (kProfile) { const long long now = clock64(); pc[k] += now - pt; pt = now; }
  const uint32_t barAddr = smemAddr(bar);
  const uint32_t stripBytes = uint32_t(g.stripStride) * 4u;
  if (tid == 0) {
    flags[0] = 0;
    mbarInit(barAddr, 1);
    fenceBarrierInit();
    mbarExpectTx(barAddr, stripBytes);
    const char* src = reinterpret_cast<const char*>(g.strips + size_t(b) * g.stripStride);
    for (uint32_t off = 0; off < stripBytes; off += 16384u) bulkLoad(smemAddr(strips) + off, src + off, stripBytes - off < 16384u ? stripBytes - off : 16384u, barAddr);
    flags[1] = a.parkTiles > 0 ? acquireParkSlot(a.parkSlots, a.parkSlotWords, b) : 0; // (overlaps the copy)
  }
  if (tid >= 64 && tid < 128) strips[g.stripStride + (tid - 64)] = 0.f; // the all-zero strip that pads odd pair lists
  __syncthreads();
  mbarWaitRelaxed(barAddr, 0);
  MB2_GC(0)
  // this CTA's parked tile t, lane's two float4: park + t * 256 + {4 lane, 128 + 4 lane} (coalesced 512-byte warp accesses)
  float* park = a.park + size_t(flags[1]) * size_t(a.parkTiles) * 256 + 4 * lane;
  const int rounds = g.numOrder / kWarps;
  auto tileInfoOf = [](int packed) { return (packed & 0x7FFF) | ((packed >> 15) << 16); }; // GramCholTables::gram -> tileInfo
  // ---- Gram ----
  for (int r = 0; r < rounds; ++r) {
    const int4 rec = tableRecord4(tab + L.gram + 4 * (r * kWarps + warp)); // {tile, packed info, q0, q1}
    if (rec.x == 0xFFFF) continue;
    float acc[2][4];
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
    gramTileAccumulate(strips, tab + L.quad, rec.z, rec.w, lane, acc);
    if (rec.x >= a.parkTiles) gramTileStore(tiles + size_t(rec.x) * 256, acc, tileInfoOf(rec.y), g.regularization, lane);
    else {
      __stcg(reinterpret_cast<float4*>(park + size_t(rec.x) * 256), make_float4(acc[0][0], acc[0][1], acc[0][2], acc[0][3]));
      __stcg(reinterpret_cast<float4*>(park + size_t(rec.x) * 256 + 128), make_float4(acc[1][0], acc[1][1], acc[1][2], acc[1][3]));
    }
  }
  for (int K = hw; K < S.numTileCols; K += kGramThreads / 16)
    y[16 * K + hl] = gramVectorEntry(strips, resid, tab + L.colEnt, int(tab[L.col + K]), int(tab[L.col + K + 1]), hl);
  __syncthreads();
  MB2_GC(1)
  for (int r = 0; r < rounds; ++r) {
    const int4 rec = tableRecord4(tab + L.gram + 4 * (r * kWarps + warp));
    if (rec.x == 0xFFFF || rec.x >= a.parkTiles) continue;
    const float4 v0 = __ldcg(reinterpret_cast<const float4*>(park + size_t(rec.x) * 256));
    const float4 v1 = __ldcg(reinterpret_cast<const float4*>(park + size_t(rec.x) * 256 + 128));
    const float acc[2][4] = {{v0.x, v0.y, v0.z, v0.w}, {v1.x, v1.y, v1.z, v1.w}};
    gramTileStore(tiles + size_t(rec.x) * 256, acc, tileInfoOf(rec.y), g.regularization, lane);
  }
  for (int s2 = tid; s2 < S.nPad; s2 += kGramThreads) {
    const int p = S.perm[s2];
    if (p >= 0) gsub[p] = y[s2];
  }
  __syncthreads();
  // every parked value has been read (it sits in the tiles now): the slot is free for the next CTA
  if (tid == 0 && a.parkTiles > 0) atomicAnd(a.parkSlots + (flags[1] >> 5), ~(1u << (flags[1] & 31)));
  MB2_GC(2)
  // ---- level-scheduled Cholesky (same phases as choleskyScheduledKernel) ----
  for (int Lv = 0; Lv < S.numLevels; ++Lv) {
    const int4 l0 = tableRecord4(tab + L.level + 4 * Lv), l1 = tableRecord4(tab + L.level + 4 * (Lv + 1)); // {diag, panel, order, vtask}
    for (int ci = l0.x + warp; ci < l1.x; ci += kWarps) {
      const int4 d = tableRecord4(tab + L.diag + 4 * ci); // {K, diagonal tile, ...}
      cholDiagTile(tiles + size_t(d.y) * 256, y + 16 * d.x, lane, c.regularization, flags);
    }
    __syncthreads();
    MB2_GC(3)
    for (int pi = l0.y + warp; pi < l1.y; pi += kWarps) {
      const int2 pe = tableRecord2(tab + L.panel + 2 * pi);
      float* ptile = tiles + size_t(pe.x) * 256;
      float x[2][4];
      cholPanelProduct(ptile, tiles + size_t(pe.y) * 256, lane, x);
      cholPanelStore(ptile, lane, x);
    }
    __syncthreads();
    MB2_GC(4)
    for (int oi = l0.z + warp; oi < l1.z; oi += kWarps) {
      const int4 o = tableRecord4(tab + L.order + 4 * oi); // {destination, first pair, end pair}
      if (o.x != 0xFFFF) cholUpdateTile(tiles, tab + L.pair, tab + L.pair + 1, 2, o.y, o.z, o.x, lane);
    }
    for (int vi = l0.w + hw; vi < l1.w; vi += kGramThreads / 16) {
      const int4 v = tableRecord4(tab + L.vtask + 4 * vi); // {row block, first source, end source}
      cholVectorRows(tiles, y, tab + L.vsrc, tab + L.vsrc + 1, 2, v.y, v.z, v.x, hl);
    }
    __syncthreads();
    MB2_GC(5)
  }
  for (int Lv = S.numLevels - 1; Lv >= 0; --Lv) {
    const int c0 = tab[L.level + 4 * Lv], c1 = tab[L.level + 4 * (Lv + 1)];
    for (int ci = c0 + warp; ci < c1; ci += kWarps) {
      const int4 d = tableRecord4(tab + L.diag + 4 * ci); // {K, diagonal tile, first panel, end panel}
      cholBackwardPanels(tiles, y, tab + L.colPanel, tab + L.colPanel + 1, 2, d.z, d.w, d.x, d.y, lane);
    }
    __syncthreads();
  }
  MB2_GC(6)
  cholFinish(c, b, n, y, gsub, flags[0] != 0, S.pos); // y holds the step per elimination slot
  MB2_GC(7)
  if constexpr (kProfile) {
    // a block from the middle of the grid: its SM is in steady state (the other resident CTAs are at unrelated phases), unlike block 0,
    // whose whole first wave starts in lock step
    if (b == int(gridDim.x >> 1) && tid == 0 && a.phaseCycles != nullptr)
      for (int k = 0; k < 8; ++k) a.phaseCycles[k] += (unsigned long long)pc[k];
  }
#undef MB2_GC
}

template <bool kProfile, class Tables>
static cudaError_t prepareGramCholesky(size_t smem) {
  cudaError_t e = cudaFuncSetAttribute(gramCholeskyKernel<kProfile, Tables>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem));
  if (e != cudaSuccess) return e;
  return cudaFuncSetAttribute(gramCholeskyKernel<kProfile, Tables>, cudaFuncAttributePreferredSharedMemoryCarveout, int(cudaSharedmemCarveoutMaxShared));
}

int gramCholeskyParkSlots(const GramCholArgs& a, const CholSchedDev& sched, bool paramTables) {
  const size_t smem = gramCholeskySmemBytes(a.g.stripStride, a.c.ns, sched.nPad, sched.numTiles);
  // the profiling instantiations carry more registers: never more resident CTAs than the production ones
  cudaError_t e = paramTables ? prepareGramCholesky<false, GramCholParamTables>(smem) : prepareGramCholesky<false, GramCholGlobalTables>(smem);
  int perSm = 0;
  if (e == cudaSuccess)
    e = paramTables ? cudaOccupancyMaxActiveBlocksPerMultiprocessor(&perSm, gramCholeskyKernel<false, GramCholParamTables>, kGramThreads, smem)
                    : cudaOccupancyMaxActiveBlocksPerMultiprocessor(&perSm, gramCholeskyKernel<false, GramCholGlobalTables>, kGramThreads, smem);
  if (e != cudaSuccess || perSm < 1) return -1;
  return (g_numSms * perSm + 31) / 32 * 32;
}

cudaError_t launchGramCholesky(const GramCholArgs& a, const CholSchedDev& sched, const GramCholParamTables* inParams, const GramCholGlobalTables& inGlobal, bool profile,
                               cudaStream_t stream) {
  const size_t smem = gramCholeskySmemBytes(a.g.stripStride, a.c.ns, sched.nPad, sched.numTiles);
  if (smem > size_t(g_maxSmemOptin) || (a.g.stripStride & 3) != 0) return cudaErrorInvalidConfiguration;
  if (a.parkTiles > 0 && (a.park == nullptr || a.parkSlots == nullptr || a.parkSlotWords < 1)) return cudaErrorInvalidValue;
  cudaError_t e;
  if (inParams != nullptr) e = profile ? prepareGramCholesky<true, GramCholParamTables>(smem) : prepareGramCholesky<false, GramCholParamTables>(smem);
  else e = profile ? prepareGramCholesky<true, GramCholGlobalTables>(smem) : prepareGramCholesky<false, GramCholGlobalTables>(smem);
  if (e != cudaSuccess) return e;
  if (inParams != nullptr) {
    if (profile) gramCholeskyKernel<true, GramCholParamTables><<<a.c.batch, kGramThreads, smem, stream>>>(a, sched, *inParams);
    else gramCholeskyKernel<false, GramCholParamTables><<<a.c.batch, kGramThreads, smem, stream>>>(a, sched, *inParams);
  } else {
    if (profile) gramCholeskyKernel<true, GramCholGlobalTables><<<a.c.batch, kGramThreads, smem, stream>>>(a, sched, inGlobal);
    else gramCholeskyKernel<false, GramCholGlobalTables><<<a.c.batch, kGramThreads, smem, stream>>>(a, sched, inGlobal);
  }
  return cudaGetLastError();
}

} // namespace mb2
#include "ik_qr.cuh"
#include "ik_tr_qr.cuh"
namespace mb2 {

cudaError_t initKernelAttributes() {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  e = cudaDeviceGetAttribute(&g_numSms, cudaDevAttrMultiProcessorCount, dev);
  if (e != cudaSuccess) return e;
  e = cudaDeviceGetAttribute(&g_maxSmemPerSm, cudaDevAttrMaxSharedMemoryPerMultiprocessor, dev);
  if (e != cudaSuccess) return e;
  return cudaDeviceGetAttribute(&g_maxSmemOptin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
}

// ------------------------------------------------------------------------------------------------
// Small element-wise kernels: line search (gauss_newton_solver.cpp:283-313,
// subset_gauss_newton_solver.cpp:119-141), SolverT bookkeeping, target normalisation.
// ------------------------------------------------------------------------------------------------
__global__ void trialUpdateKernel(int batch, const float* thetaOrig, int ldTheta, const float* delta, int ns, const int32_t* cols, const float* scale,
                                  float* thetaTrial, const int32_t* active) {
  const int b = blockIdx.x;
  if (active[b] == 0) return;
  const float s = scale[b];
  for (int i = threadIdx.x; i < ns; i += blockDim.x) {
    const int c = cols[i];
    if (c >= 0) thetaTrial[size_t(b) * ldTheta + c] = thetaOrig[size_t(b) * ldTheta + c] - s * delta[size_t(b) * ns + i]; // c < 0: alignment column
  }
}
cudaError_t launchTrialUpdate(int batch, const float* thetaOrig, int ldTheta, const float* delta, int ns, const int32_t* cols, const float* scale,
                              float* thetaTrial, const int32_t* active, cudaStream_t stream) {
  trialUpdateKernel<<<batch, 128, 0, stream>>>(batch, thetaOrig, ldTheta, delta, ns, cols, scale, thetaTrial, active);
  return cudaGetLastError();
}

__global__ void lineSearchStepKernel(const LineSearchArgs a) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= a.batch || a.searching[b] == 0) return;
  const float scale = a.scale[b];
  if (lineSearchStops(a.errors[b], a.trialErrors[b], scale, a.subsetVariant, a.gradDotDelta + b, a.step)) a.searching[b] = 0;
  else a.scale[b] = scale * 0.5f;
}
cudaError_t launchLineSearchStep(const LineSearchArgs& a, cudaStream_t stream) {
  lineSearchStepKernel<<<(a.batch + 127) / 128, 128, 0, stream>>>(a);
  return cudaGetLastError();
}

__global__ void bookkeepingKernel(int batch, const SolveState s) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= batch || s.active[b] == 0) return;
  finishIteration(s, b);
}
cudaError_t launchBookkeeping(int batch, const SolveState& s, cudaStream_t stream) {
  bookkeepingKernel<<<(batch + 127) / 128, 128, 0, stream>>>(batch, s);
  return cudaGetLastError();
}

__global__ void normalizeQuatsKernel(float* base, int count, int strideFloats, int quatsPerRecord, int batch) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= batch * quatsPerRecord) return;
  const int b = idx / quatsPerRecord, q = idx % quatsPerRecord;
  float* p = base + size_t(b) * strideFloats + 4 * q;
  const float n = sqrtf(p[0] * p[0] + p[1] * p[1] + p[2] * p[2] + p[3] * p[3]);
  p[0] /= n; p[1] /= n; p[2] /= n; p[3] /= n;
}
// packed [batch][size] -> records [batch][strideFloats] at dst (a strided 2-D copy from the host takes one DMA descriptor per row)
__global__ void scatterTargetsKernel(const float* packed, float* dst, int size, int strideFloats, int batch) {
  const size_t idx = size_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= size_t(batch) * size) return;
  const size_t b = idx / size, k = idx % size;
  dst[b * strideFloats + k] = packed[idx];
}
cudaError_t launchScatterTargets(const float* packed, float* dst, int size, int strideFloats, int batch, cudaStream_t stream) {
  const size_t total = size_t(batch) * size;
  if (total == 0) return cudaSuccess;
  scatterTargetsKernel<<<unsigned((total + 255) / 256), 256, 0, stream>>>(packed, dst, size, strideFloats, batch);
  return cudaGetLastError();
}
cudaError_t launchNormalizeQuats(float* base, int count, int strideFloats, int quatsPerRecord, int batch, cudaStream_t stream) {
  const int total = batch * quatsPerRecord;
  if (total == 0) return cudaSuccess;
  normalizeQuatsKernel<<<(total + 127) / 128, 128, 0, stream>>>(base, count, strideFloats, quatsPerRecord, batch);
  return cudaGetLastError();
}

DeviceLimits deviceLimits() { return DeviceLimits{g_numSms, g_maxSmemOptin, g_maxSmemPerSm}; }

} // namespace mb2
