// The fused persistent Gauss-Newton kernel (see ik_fused.cuh for the data flow).
#include "ik_fused.cuh"

#include <algorithm>
#include <cfloat>
#include <cstdio>

#include "ik_chol_sched.h"
#include "ik_device.cuh"
#include "ik_ptx.cuh"

namespace mb2 {

namespace {

__device__ __forceinline__ double warpSumD(double v) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

static_assert(kFusedGroupThreads == 32 * kGramWarps, "the Gram tile-order table is laid out for kGramWarps warps per instance");
constexpr int kPhases = 12;
// phase ids of the profiling instantiation
enum { kPhFetch = 0, kPhJointParams, kPhFk, kPhUnits, kPhCells, kPhGram, kPhRestore, kPhDiag, kPhPanel, kPhUpdate, kPhBackward, kPhFinish };

template <int kGroups, bool kProfile>
__global__ void __launch_bounds__(kFusedGroupThreads* kGroups, 1) fusedSolveKernel(const FusedArgs a) {
  extern __shared__ __align__(128) uint8_t fusedSmem[];
  const int tid = threadIdx.x;
  const int group = tid / kFusedGroupThreads, gt = tid % kFusedGroupThreads;
  const int warp = gt >> 5, lane = gt & 31, hw = gt >> 4, hl = gt & 15;
  const unsigned hmask = 0xFFFFu << (16 * ((gt >> 4) & 1));
  uint8_t* base = fusedSmem + ((128u - (smemAddr(fusedSmem) & 127u)) & 127u);
  int32_t* tab = reinterpret_cast<int32_t*>(base);
  unsigned long long* bar = reinterpret_cast<unsigned long long*>(tab + a.L.words);
  float* groupBase = reinterpret_cast<float*>(bar + 2) + size_t(group) * a.groupFloats;

  // ---- once per CTA: every table by bulk copies on one mbarrier ----
  const uint32_t barAddr = smemAddr(bar);
  if (tid == 0) {
    mbarInit(barAddr, 1);
    fenceBarrierInit();
    const uint32_t total = uint32_t(a.L.words) * 4u;
    mbarExpectTx(barAddr, total);
    const char* src = reinterpret_cast<const char*>(a.blob);
    for (uint32_t off = 0; off < total; off += 32768u) bulkLoad(smemAddr(tab) + off, src + off, total - off < 32768u ? total - off : 32768u, barAddr);
  }
  __syncthreads();
  mbarWaitRelaxed(barAddr, 0);

  // table views on the staged copy (every pointer derived from the shared-memory base: see rebaseSchedule)
  FunctionTables T = a.T;
  T.parent = tab + a.L.parent;
  T.offset = reinterpret_cast<const float*>(tab + a.L.offset);
  T.prerot = reinterpret_cast<const float*>(tab + a.L.prerot);
  T.ptOuter = tab + a.L.ptOuter;
  T.ptInner = tab + a.L.ptInner;
  T.ptVals = reinterpret_cast<const float*>(tab + a.L.ptVals);
  T.ptOffsets = reinterpret_cast<const float*>(tab + a.L.ptOffsets);
  T.levelStart = tab + a.L.levelStart;
  T.levelJoints = tab + a.L.levelJoints;
  T.efs = reinterpret_cast<const EfDesc*>(tab + a.L.efs);
  T.units = reinterpret_cast<const UnitDesc*>(tab + a.L.units);
  T.cells = reinterpret_cast<const CellDesc*>(tab + a.L.cells);
  T.contribs = reinterpret_cast<const ContribDesc*>(tab + a.L.contribs);
  T.limitData = reinterpret_cast<const float*>(tab + a.L.limitData);
  const int32_t* cols = tab + a.L.cols;
  const int32_t* gtab = tab + a.L.gram;
  const int32_t* tileOrder = gtab + a.gramOff[0], *tileQuadStart = gtab + a.gramOff[1], *quads = gtab + a.gramOff[2];
  const int32_t* colStripStart = gtab + a.gramOff[4], *colStrip = gtab + a.gramOff[5], *stripRow = gtab + a.gramOff[6], *tileInfo = gtab + a.gramOff[7];
  const CholSchedDev S = rebaseSchedule(a.S, tab + a.L.sched);

  // ---- per-group shared memory ----
  const int n = S.n;                       // device columns (alignment gaps included)
  const int nc4 = (n + 3) & ~3, np4 = (T.numParams + 3) & ~3;
  float* U = groupBase;                    // union: [strips | residual | zero strip | joint states | joint parameters | records]  /  [tiles]
  float* strips = U;
  float* resid = U + a.residOff;
  float* js = U + a.stripStride + 64;
  float* jp = js + ((T.numJoints * kJointStateStride + 3) & ~3);
  float* rec = jp + ((T.numJoints * kParametersPerJoint + 3) & ~3);
  float* tiles = U;
  float* y = U + a.unionFloats;
  float* gsub = y + S.nPad;
  float* dsub = gsub + nc4;
  float* th = dsub + nc4;
  double* errSlots = reinterpret_cast<double*>(th + np4); // 8 warp partials, then [8] = error of this iteration, [9] = lastError
  int* flags = reinterpret_cast<int*>(errSlots + 10);     // [0] Cholesky breakdown, [1] stop, [2] next instance, [3] non-finite

  const WarpLanes<kFusedGroupThreads / 32> g{group, gt};
  const int numJointParams = T.numJoints * kParametersPerJoint;
  const size_t sweepStripFloats = size_t(a.stripStride) + 64; // strips | residual | zero strip: what the Gram phase reads
  float parked[kFusedMaxRounds][8]; // Gram tiles that would overwrite live strips, indexed by the round: thread-local memory

  unsigned long long pc[kPhases];
  long long pt = 0;
  if constexpr (kProfile) { for (int k = 0; k < kPhases; ++k) pc[k] = 0; pt = clock64(); }
  const bool profiler = kProfile && blockIdx.x == 0 && tid == 0;
#define MB2_PH(k) if constexpr (kProfile) { if (profiler) { const long long now = clock64(); pc[k] += (unsigned long long)(now - pt); pt = now; } }

  while (true) {
    if (gt == 0) flags[2] = atomicAdd(a.workCounter, 1);
    g.sync();
    const int b = flags[2];
    if (b >= a.batch) break;
    const float* targets = a.targets + size_t(b) * T.targetStride;
    const float* cw = a.cweights + (T.weightsPerInstance ? size_t(b) * T.numWeights : 0);
    float* thetaG = a.theta + size_t(b) * a.ldTheta;
    for (int i = gt; i < T.numParams; i += kFusedGroupThreads) th[i] = thetaG[i];
    if (gt == 0) { errSlots[8] = DBL_MAX; errSlots[9] = DBL_MAX; flags[0] = 0; flags[1] = 0; flags[3] = 0; } // solver.cpp:83-84
    int iterations = 0;
    MB2_PH(kPhFetch)
    for (int it = 0; it < a.state.maxIterations; ++it) {
      // ---- ParameterTransform::apply + zero background of the strips (ResizeableMatrix::resizeAndSetZero, solver_function.cpp:96) ----
      g.sync(); // theta (first iteration: the loads above; later: the update) is visible; the previous iteration is done with the tiles
      for (int row = gt; row < numJointParams; row += kFusedGroupThreads) jp[row] = jointParameterRow(T, row, th);
      for (int i = gt; i < (a.stripStride + 64) / 4; i += kFusedGroupThreads) reinterpret_cast<float4*>(strips)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
      g.sync();
      MB2_PH(kPhJointParams)
      // ---- SkeletonState::set, level by level (skeleton_state.cpp:87-121) ----
      fkPasses<true, true>(g, T, jp, js);
      g.sync();
      MB2_PH(kPhFk)
      // ---- residual + error (units), then the Jacobian cells into the strips ----
      double err = 0.0;
      for (int u = gt; u < T.numUnits; u += kFusedGroupThreads) err += (double)evalUnit<true>(T, u, th, jp, js, targets, cw, rec, resid);
      err = warpSumD(err);
      if (lane == 0) errSlots[warp] = err;
      g.sync();
      MB2_PH(kPhUnits)
      for (int c = gt; c < T.numCells; c += kFusedGroupThreads) jacobianCell(T, c, js, rec, targets, strips);
      if (gt == 0) { // fixed order: deterministic
        double e = 0.0;
        for (int w = 0; w < kFusedGroupThreads / 32; ++w) e += errSlots[w];
        errSlots[8] = e;
      }
      g.sync();
      MB2_PH(kPhCells)
      // ---- tile-sparse Gram: a warp owns a tile at a time; a finished tile beyond the strips is stored at once, one that would
      //      overwrite strips still being read waits in thread-local memory ----
      {
        int slot = 0;
        for (int ti = warp; ti < a.numOrder; ti += kFusedGroupThreads / 32, ++slot) {
          const int t = tileOrder[ti];
          if (t < 0) continue;
          float acc[2][4];
#pragma unroll
          for (int i = 0; i < 2; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
          gramTileAccumulate(strips, quads, tileQuadStart[t], tileQuadStart[t + 1], lane, acc);
          if (size_t(t) * 256 >= sweepStripFloats) gramTileStore(tiles + size_t(t) * 256, acc, tileInfo[t], a.regularization, lane);
          else {
#pragma unroll
            for (int i = 0; i < 8; ++i) parked[slot][i] = acc[i >> 2][i & 3];
          }
        }
        for (int K = hw; K < S.numTileCols; K += kFusedGroupThreads / 16)
          y[16 * K + hl] = gramVectorEntry(strips, resid, colStrip, stripRow, colStripStart[K], colStripStart[K + 1], hl);
      }
      g.sync();
      MB2_PH(kPhGram)
      {
        int slot = 0;
        for (int ti = warp; ti < a.numOrder; ti += kFusedGroupThreads / 32, ++slot) {
          const int t = tileOrder[ti];
          if (t < 0 || size_t(t) * 256 >= sweepStripFloats) continue;
          float acc[2][4];
#pragma unroll
          for (int i = 0; i < 8; ++i) acc[i >> 2][i & 3] = parked[slot][i];
          gramTileStore(tiles + size_t(t) * 256, acc, tileInfo[t], a.regularization, lane);
        }
        for (int s = gt; s < S.nPad; s += kFusedGroupThreads) {
          const int p = S.perm[s];
          if (p >= 0) gsub[p] = y[s];
        }
      }
      g.sync();
      MB2_PH(kPhRestore)
      // ---- level-scheduled Cholesky (ik_chol_sched.h) ----
      for (int Lv = 0; Lv < S.numLevels; ++Lv) {
        for (int ci = S.levelColStart[Lv] + warp; ci < S.levelColStart[Lv + 1]; ci += kFusedGroupThreads / 32) {
          const int K = S.levelCols[ci];
          cholDiagTile(tiles + size_t(S.diagTile[K]) * 256, y + 16 * K, lane, a.regularization, flags);
        }
        g.sync();
        MB2_PH(kPhDiag)
        for (int pi = S.levelPanelStart[Lv] + warp; pi < S.levelPanelStart[Lv + 1]; pi += kFusedGroupThreads / 32) {
          float* ptile = tiles + size_t(S.panelTile[pi]) * 256;
          float x[2][4];
          cholPanelProduct(ptile, tiles + size_t(S.panelDiag[pi]) * 256, lane, x);
          cholPanelStore(ptile, lane, x);
        }
        g.sync();
        MB2_PH(kPhPanel)
        for (int oi = S.levelOrderStart8[Lv] + warp; oi < S.levelOrderStart8[Lv + 1]; oi += kFusedGroupThreads / 32) { const int ti = S.taskOrder8[oi]; if (ti >= 0) cholUpdateTask(tiles, S, ti, lane); }
        for (int vi = S.levelVTaskStart[Lv] + hw; vi < S.levelVTaskStart[Lv + 1]; vi += kFusedGroupThreads / 16) cholVectorTask(tiles, y, S, vi, hl);
        g.sync();
        MB2_PH(kPhUpdate)
      }
      for (int Lv = S.numLevels - 1; Lv >= 0; --Lv) {
        for (int ci = S.levelColStart[Lv] + warp; ci < S.levelColStart[Lv + 1]; ci += kFusedGroupThreads / 32) cholBackwardColumn(tiles, y, S, S.levelCols[ci], lane);
        g.sync();
      }
      MB2_PH(kPhBackward)
      for (int i = gt; i < S.nPad; i += kFusedGroupThreads) { const int p = S.perm[i]; if (p >= 0) dsub[p] = y[i]; }
      g.sync();
      // ---- theta -= delta (skeleton_solver_function.cpp:153-159) and the SolverT bookkeeping (solver.cpp:92-122) ----
      for (int i = gt; i < n; i += kFusedGroupThreads) {
        const int c = cols[i];
        if (c >= 0) th[c] -= dsub[i];
      }
      iterations = it + 1;
      if (gt == 0) {
        const double error = errSlots[8], last = errSlots[9];
        if (a.state.history != nullptr) a.state.history[size_t(b) * a.state.maxIterations + it] = error;
        const bool stop = solveStops(error, last, it, a.state.minIterations, a.state.maxIterations, a.state.threshold);
        if (!stop) errSlots[9] = error;
        flags[1] = stop ? 1 : 0;
      }
      g.sync();
      MB2_PH(kPhFinish)
      if (flags[1] != 0) break;
    }
    // ---- NaN / Inf guard of the batched caller (tensor_ik.cpp:168-173): theta in global memory still holds the initial guess ----
    bool bad = false;
    for (int i = gt; i < T.numParams; i += kFusedGroupThreads) bad = bad || !isfinite(th[i]);
    if (bad) flags[3] = 1;
    g.sync();
    const bool nonFinite = flags[3] != 0;
    if (!nonFinite)
      for (int i = gt; i < T.numParams; i += kFusedGroupThreads) thetaG[i] = th[i];
    if (gt == 0) {
      a.state.errors[b] = errSlots[8];
      a.state.iterations[b] = iterations;
      a.state.status[b] = nonFinite ? 2 : (flags[0] != 0 ? 1 : 0);
    }
    MB2_PH(kPhFinish)
  }
#undef MB2_PH
  if constexpr (kProfile) {
    if (profiler && a.phaseCycles != nullptr)
      for (int k = 0; k < kPhases; ++k) a.phaseCycles[k] = pc[k];
  }
}

} // namespace

cudaError_t launchFusedSolve(const FusedArgs& a0, const FusedConfig& cfg, int numSms, bool profile, cudaStream_t stream) {
  if (cfg.groups < 1) return cudaErrorInvalidConfiguration;
  FusedArgs a = a0;
  a.groups = cfg.groups;
  a.groupFloats = cfg.groupFloats;
  a.unionFloats = cfg.unionFloats;
  int grid = (a.batch + cfg.groups - 1) / cfg.groups;
  if (grid > numSms) grid = numSms;
  if (grid < 1) grid = 1;
  auto launch = [&](auto kernel) -> cudaError_t {
    const cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, int(cfg.smemBytes));
    if (e != cudaSuccess) return e;
    kernel<<<grid, kFusedGroupThreads * cfg.groups, cfg.smemBytes, stream>>>(a);
    return cudaGetLastError();
  };
  if (profile) {
    switch (cfg.groups) {
      case 1: return launch(fusedSolveKernel<1, true>);
      case 2: return launch(fusedSolveKernel<2, true>);
      default: return launch(fusedSolveKernel<3, true>);
    }
  }
  switch (cfg.groups) {
    case 1: return launch(fusedSolveKernel<1, false>);
    case 2: return launch(fusedSolveKernel<2, false>);
    default: return launch(fusedSolveKernel<3, false>);
  }
}

} // namespace mb2
