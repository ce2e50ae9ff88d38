// TEST HARNESS ONLY — CPU lane-emulation of the device code, built into tests/emu/libmb2_emu.so.
//
// It exports the subset of include/momentum_b200.h that the parity tests use. Character and block setup and the solver-path planning
// are the library's own (ik_plan.cpp, ik_chol_sched.cpp); only the kernels' lane loops over the __host__ __device__ building blocks of
// momentum_b200/csrc (ik_device.cuh, ik_chol.cuh) run here, lane by lane on the CPU. Purpose: catch planner / indexing / semantics bugs
// without a GPU. It is not part of the product library and nothing in momentum_b200/ loads it.
#include <cfloat>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "../../include/momentum_b200.h"
#include "../../momentum_b200/csrc/ik_chol.cuh"
#include "../../momentum_b200/csrc/ik_chol_sched.cuh"
#include "../../momentum_b200/csrc/ik_chol_sched.h"
#include "../../momentum_b200/csrc/ik_device.cuh"
#include "../../momentum_b200/csrc/ik_plan.h"
#include "../../momentum_b200/csrc/ik_solve_path.h"
#include "emu_error.h"

using namespace mb2;

static thread_local std::string g_err;
static int fail(int c, const std::string& m) { g_err = m; return c; }

struct mb2_character { HostCharacter host; };
struct mb2_solver_function {
  const mb2_character* ch;
  int B;
  HostFunction host;
  std::vector<float> targets;         // [B][targetStride]
  std::vector<float> instanceWeights; // [B][numWeights] once the constraint weights are per instance
  Plan plan;
  int ldJ{32};
  std::vector<float> J;
  bool planCompact{false};
  bool stripMode{false};   // Jacobian buffer in strip layout (GramPlan) instead of the K-major matrix
  int residOff{0}, stripStride{0};
};
struct mb2_solver {
  mb2_solver_function* fn;
  mb2_gauss_newton_options opt;
  std::vector<double> errors, history;
  std::vector<int32_t> iterations, status;
  uint64_t totalIterations{0};
  SolvePath path;
};
// the device the solve path is chosen for (emu_set_device_limits): an H100 SXM by default
static DeviceLimits g_limits{132, 227 * 1024, 228 * 1024};

static int roundUp(int v, int m) { return (v + m - 1) / m * m; }

// Jacobian storage of f->plan: the strips of a Gram plan, or the K-major matrix
static void layoutJacobian(mb2_solver_function* f, const GramPlan* strips) {
  f->stripMode = strips != nullptr;
  f->residOff = strips ? strips->residOff : 0;
  f->stripStride = strips ? strips->stride : 0;
  f->ldJ = std::max(32, roundUp(f->plan.numRows, 32));
  f->J.assign(strips ? size_t(f->B) * strips->stride : size_t(f->B) * (f->plan.numCols + 1) * f->ldJ, 0.f);
}

static std::string plan(mb2_solver_function* f, bool compact) {
  const std::string e = buildPlan(f->ch->host, f->host.efs, f->host.enabled, compact, f->plan);
  if (!e.empty()) return e;
  f->planCompact = compact;
  layoutJacobian(f, nullptr);
  return "";
}

// the plan of the tile-scheduled solver path (cholMode 2: dense pattern, 3: sparse pattern), as the library plans it
static std::string planTiles(mb2_solver_function* f, int cholMode, bool strips, CholSchedule& s, GramPlan& g) {
  const std::string e = planSolverPath(f->ch->host, f->host.efs, f->host.enabled, cholMode == MB2_CHOLESKY_TILES_DENSE, strips, f->plan, s, g);
  if (!e.empty()) return e;
  f->planCompact = true;
  layoutJacobian(f, strips ? &g : nullptr);
  return "";
}

static FunctionTables tables(const mb2_solver_function* f) {
  FunctionTables T{hostCharacterTables(f->ch->host)};
  T.numEf = int(f->plan.efs.size()); T.numUnits = int(f->plan.units.size()); T.numCells = int(f->plan.cells.size());
  T.efs = f->plan.efs.data(); T.units = f->plan.units.data(); T.cells = f->plan.cells.data(); T.contribs = f->plan.contribs.data();
  T.limitData = f->plan.limitData.data();
  T.targetStride = f->host.targetStride; T.recStride = f->plan.recStride; T.numRows = f->plan.numRows; T.ldJ = f->ldJ; T.numCols = f->plan.numCols;
  T.weightsPerInstance = f->host.weightsPerInstance; T.numWeights = f->host.numWeights;
  T.stripMode = f->stripMode ? 1 : 0; T.residOff = f->residOff;
  T.jacobianStride = f->stripMode ? size_t(f->stripStride) : size_t(f->plan.numCols + 1) * f->ldJ;
  return T;
}

// emulation of sweepKernel<kJacobian> for one instance (the warp's lanes run in sequence)
template <bool kJacobian>
static void sweepOne(mb2_solver_function* f, const FunctionTables& T, int b, const float* theta, double* errOut, float* stateOut) {
  std::vector<float> jp(size_t(T.numJoints) * 7), js(size_t(T.numJoints) * kJointStateStride), rec(T.recStride + 4);
  for (int row = 0; row < T.numJoints * 7; ++row) jp[row] = jointParameterRow(T, row, theta);
  fkPasses<kJacobian, false>(HostLanes{}, T, theta, js.data()); // as sweepKernel with one warp: joint parameters straight from theta
  if (stateOut)
    for (int i = 0; i < T.numJoints * 8; ++i) stateOut[i] = js[(i >> 3) * kJointStateStride + (i & 7)];
  const float* tg = f->targets.data() + size_t(b) * T.targetStride;
  const float* cw = T.weightsPerInstance ? f->instanceWeights.data() + size_t(b) * T.numWeights : f->host.weights.data();
  float* Jb = f->J.data() + size_t(b) * T.jacobianStride;
  float* res = kJacobian ? Jb + (T.stripMode ? size_t(T.residOff) : size_t(T.numCols) * T.ldJ) : nullptr;
  // lanes accumulate in double, then a butterfly reduction: emulate the same association
  double lane[32];
  for (int l = 0; l < 32; ++l) lane[l] = 0.0;
  for (int u = 0; u < T.numUnits; ++u) lane[u & 31] += (double)evalUnit<kJacobian>(T, u, theta, (u & 1) ? jp.data() : nullptr, js.data(), tg, cw, rec.data(), res); // both forms of the joint-parameter access
  for (int o = 16; o > 0; o >>= 1) {
    double t[32];
    for (int l = 0; l < 32; ++l) t[l] = lane[l] + lane[l ^ o];
    for (int l = 0; l < 32; ++l) lane[l] = t[l];
  }
  if (kJacobian)
    for (int c = 0; c < T.numCells; ++c) jacobianCell(T, c, js.data(), rec.data(), tg, Jb);
  *errOut = kJacobian ? lane[0] : (double)(float)lane[0];
}

static void jtjOne(const mb2_solver_function* f, int b, int ns, float* H, int ldH) {
  const int nc = f->plan.numCols;
  const float* J = f->J.data() + size_t(b) * (nc + 1) * f->ldJ;
  const float* r = J + size_t(nc) * f->ldJ;
  const int K = roundUp(std::max(f->plan.numRows, 1), 4);
  for (int i = 0; i < ns; ++i) {
    for (int j = 0; j <= i; ++j) {
      float s = 0.f;
      for (int k = 0; k < K; ++k) s = fmaf(J[size_t(i) * f->ldJ + k], J[size_t(j) * f->ldJ + k], s);
      H[size_t(j) * ldH + i] = s; // upper triangle only (row j, column i >= j), like the tensor-core epilogue
    }
    float g = 0.f;
    for (int k = 0; k < K; ++k) g = fmaf(J[size_t(i) * f->ldJ + k], r[k], g);
    H[size_t(i) * ldH + ns] = g;
  }
}

// emulation of choleskyKernel<NB> for one instance; returns fail flag, writes delta and g.delta
template <int NB>
static int cholOne(float* Hg, int n, int ldH, float reg, float* delta, float* gdd) {
  const int lda = n | 1;
  std::vector<float> A(size_t(n + 1) * lda, 0.f);
  const int ldp = ((n + 1 + 3) & ~3) + 4;
  std::vector<float> P(size_t(NB) * ldp, 0.f), gsave(n);
  for (int i = 0; i <= n; ++i)
    for (int j = 0; j < n; ++j)
      if (j <= i) A[size_t(i) * lda + j] = Hg[size_t(j) * ldH + i] + ((i == j) ? reg : 0.f);
  for (int i = 0; i < n; ++i) gsave[i] = Hg[size_t(i) * ldH + n];
  int flag = 0;
  CholCtx ctx{A.data(), lda, n, P.data(), ldp, &flag};
  const int blockSize = cholBlockSize(n, NB);
  for (int k = 0; k < n && flag == 0; k += blockSize) {
    const int bs = std::min(blockSize, n - k);
    for (int jj = 0; jj < bs; ++jj) {
      const float x = cholDiagPivot(ctx, k, jj);
      if (!(x > 0.f)) { flag = k + jj + 1; break; }
      for (int lane = 0; lane < 32; ++lane) cholDiagColumn(ctx, k, bs, jj, x, lane);
    }
    if (flag) break;
    for (int t = 0; t < kCholThreads; ++t) cholPanelSolve<NB>(ctx, k, bs, t, kCholThreads);
    for (int t = 0; t < kCholThreads; ++t) cholTrailingUpdate<NB>(ctx, k, bs, t, kCholThreads);
  }
  float* y = A.data() + size_t(n) * lda;
  if (flag) cholForwardFrom(ctx, cholCompletedColumns(flag - 1, blockSize), y);
  for (int i = n - 1; i >= 0; --i) {
    float s = y[i];
    for (int k = i + 1; k < n; ++k) s -= A[size_t(k) * lda + i] * y[k];
    y[i] = s / A[size_t(i) * lda + i];
  }
  float gd = 0.f;
  for (int i = 0; i < n; ++i) { delta[i] = y[i]; gd += gsave[i] * y[i]; }
  *gdd = gd;
  return flag;
}

static int cholDispatch(int NB, float* Hg, int n, int ldH, float reg, float* delta, float* gdd) {
  if (NB == 8) return cholOne<8>(Hg, n, ldH, reg, delta, gdd);
  if (NB == 16) return cholOne<16>(Hg, n, ldH, reg, delta, gdd);
  return cholOne<32>(Hg, n, ldH, reg, delta, gdd);
}

// emulation of gramTilesKernel for one instance: strips = TMA boxes of the K-major Jacobian, warps / half-warps in sequence
static void gramOne(const mb2_solver_function* f, int b, const GramPlan& G, const CholSchedDev& S, float reg, float* out) {
  std::vector<float> store(size_t(G.stride) + 64 + 8, 0.f); // + the all-zero strip
  float* strips = store.data();
  while ((reinterpret_cast<uintptr_t>(strips) & 15) != 0) ++strips;
  std::copy(f->J.data() + size_t(b) * G.stride, f->J.data() + size_t(b + 1) * G.stride, strips); // the bulk copy
  float* resid = strips + G.residOff;
  std::vector<float> tileBuf(256 + 8);
  for (size_t ti = 0; ti < G.tileOrder.size(); ++ti) {
    const int t = G.tileOrder[ti];
    if (t < 0) continue;
    float* tile = out + size_t(t) * 256;
    for (int lane = 0; lane < 32; ++lane) {
      float acc[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
      gramTileAccumulate(strips, G.quad.data(), G.tileQuadStart[t], G.tileQuadStart[t + 1], lane, acc);
      gramTileStore(tile, acc, S.tileInfo[3 * t + 2], reg, lane);
    }
  }
  float* y = out + size_t(G.numTiles) * 256;
  std::vector<int32_t> stripRow(G.numStrips);
  for (int i = 0; i < G.numStrips; ++i) stripRow[i] = G.stripCoord[2 * i];
  for (int K = 0; K < G.numTileCols; ++K)
    for (int hl = 0; hl < 16; ++hl) y[16 * K + hl] = gramVectorEntry(strips, resid, G.colStrip.data(), stripRow.data(), G.colStripStart[K], G.colStripStart[K + 1], hl);
}

// emulation of choleskyScheduledKernel for one instance: phases in the same order, half-warps/warps in sequence
static int cholScheduledOne(const CholSchedDev& S, const float* Hs, int ldH, int n, float reg, float* delta, float* gdd, const float* gramOut = nullptr) {
  std::vector<float> store(size_t(S.numTiles) * 256 + S.nPad + 16, 0.f);
  float* tl = store.data();
  while ((reinterpret_cast<uintptr_t>(tl) & 15) != 0) ++tl; // float4 alignment
  float* y = tl + size_t(S.numTiles) * 256;
  std::vector<float> gsub(n, 0.f);
  std::fill(delta, delta + n, 0.f); // alignment columns keep a zero step
  if (gramOut != nullptr) { // tiles (+ lambda, identity extension) and the slot-ordered J^T r straight from the Gram kernel
    std::copy(gramOut, gramOut + size_t(S.numTiles) * 256 + S.nPad, tl);
    for (int s2 = 0; s2 < S.nPad; ++s2) { const int p = S.perm[s2]; if (p >= 0) gsub[p] = y[s2]; }
  } else {
  for (int t = 0; t < S.numTiles; ++t) { // the TMA box: 16 rows x 16 columns of H starting at (gj0, gi0), zero outside [ns+1] x [ldH]
    const int gi0 = S.tileInfo[3 * t], gj0 = S.tileInfo[3 * t + 1];
    auto boxAt = [&](int row, int col) { return (gj0 + row <= n && gi0 + col < ldH) ? Hs[size_t(gj0 + row) * ldH + gi0 + col] : 0.f; };
    for (int c = 0; c < 16; ++c)
      for (int r = 0; r < 16; ++r)
        tl[size_t(t) * 256 + tileIdx(r, c)] = cholPadElement(boxAt(((S.tileInfo[3 * t + 2] >> 16) & 1) && c > r ? r : c, ((S.tileInfo[3 * t + 2] >> 16) & 1) && c > r ? c : r), S.tileInfo[3 * t + 2], r, c); // cholConvertBox (diagonal boxes mirrored from the upper triangle)
  }
  for (int s2 = 0; s2 < S.nPad; ++s2) {
    const int p = S.perm[s2];
    const float g = p >= 0 ? Hs[size_t(p) * ldH + n] : 0.f;
    y[s2] = g;
    if (p >= 0) { gsub[p] = g; tl[size_t(S.diagTile[s2 >> 4]) * 256 + tileIdx(s2 & 15, s2 & 15)] += reg; }
  }
  }
  int flag = 0;
  for (int L = 0; L < S.numLevels; ++L) {
    for (int ci = S.levelColStart[L]; ci < S.levelColStart[L + 1]; ++ci) {
      const int K = S.levelCols[ci];
      for (int lane = 0; lane < 32; ++lane) cholDiagTile(tl + size_t(S.diagTile[K]) * 256, y + 16 * K, lane, reg, &flag);
    }
    for (int pi = S.levelPanelStart[L]; pi < S.levelPanelStart[L + 1]; ++pi)
    {
      float x[32][2][4];
      for (int lane = 0; lane < 32; ++lane) cholPanelProduct(tl + size_t(S.panelTile[pi]) * 256, tl + size_t(S.panelDiag[pi]) * 256, lane, x[lane]);
      for (int lane = 0; lane < 32; ++lane) cholPanelStore(tl + size_t(S.panelTile[pi]) * 256, lane, x[lane]);
    }
    for (int ti = S.levelTaskStart[L]; ti < S.levelTaskStart[L + 1]; ++ti)
      for (int lane = 0; lane < 32; ++lane) cholUpdateTask(tl, S, ti, lane);
    for (int vi = S.levelVTaskStart[L]; vi < S.levelVTaskStart[L + 1]; ++vi)
      for (int hl = 0; hl < 16; ++hl) cholVectorTask(tl, y, S, vi, hl);
  }
  for (int L = S.numLevels - 1; L >= 0; --L)
    for (int ci = S.levelColStart[L]; ci < S.levelColStart[L + 1]; ++ci)
      for (int lane = 0; lane < 32; ++lane) cholBackwardColumn(tl, y, S, S.levelCols[ci], lane);
  float gd = 0.f;
  for (int i = 0; i < S.nPad; ++i) { const int p = S.perm[i]; if (p >= 0) { delta[p] = y[i]; gd += gsub[p] * y[i]; } }
  *gdd = gd;
  return flag;
}

extern "C" {

const char* mb2_last_error(void) { return g_err.c_str(); }
int mb2_device_count(void) { return 0; }
void mb2_default_gauss_newton_options(mb2_gauss_newton_options* o) {
  std::memset(o, 0, sizeof(*o));
  o->min_iterations = 1; o->max_iterations = 2; o->threshold = 1.f; o->regularization = 0.05f; o->target_rows_per_chunk = ~0ull;
}

int mb2_character_create(int, int32_t J, const int32_t* parents, const float* offsets, const float* prerot, int32_t n, const int32_t* outer,
                         const int32_t* inner, const float* vals, const float* ptoffsets, mb2_character** out) {
  auto c = std::make_unique<mb2_character>();
  const std::string e = makeCharacter(J, parents, offsets, prerot, n, outer, inner, vals, ptoffsets, c->host);
  if (!e.empty()) return fail(MB2_ERR_INVALID_ARGUMENT, e);
  *out = c.release();
  return MB2_OK;
}
int mb2_character_set_parameter_limits(mb2_character* c, int32_t count, const mb2_parameter_limit* limits) {
  const std::string e = setParameterLimits(c->host, count, limits);
  return e.empty() ? MB2_OK : fail(MB2_ERR_INVALID_ARGUMENT, e);
}
void mb2_character_destroy(mb2_character* c) { delete c; }

int mb2_solver_function_create(const mb2_character* c, int32_t batch, mb2_solver_function** out) {
  auto f = std::make_unique<mb2_solver_function>();
  f->ch = c; f->B = batch;
  f->host.enabled.assign(c->host.numParams, 1);
  f->targets.assign(size_t(batch), 0.f);
  *out = f.release();
  return MB2_OK;
}
void mb2_solver_function_destroy(mb2_solver_function* f) { delete f; }
int32_t mb2_solver_function_num_parameters(const mb2_solver_function* f) { return f->ch->host.numParams; }
int32_t mb2_solver_function_batch(const mb2_solver_function* f) { return f->B; }
int32_t mb2_solver_function_actual_parameters(const mb2_solver_function* f) { return f->host.actualParameters(); }
int32_t mb2_solver_function_jacobian_rows(const mb2_solver_function* f) { return f->host.jacobianRows(f->ch->host); }
int32_t mb2_solver_function_jacobian_stride(const mb2_solver_function* f) { return f->host.jacobianStride(f->ch->host); }

static int addBlock(mb2_solver_function* f, const std::string& buildError, const HostErrorFunction& ef, int32_t* outIndex) {
  if (!buildError.empty()) return fail(MB2_ERR_INVALID_ARGUMENT, buildError);
  const std::string e = f->host.add(ef, outIndex);
  if (!e.empty()) return fail(MB2_ERR_UNSUPPORTED, e);
  f->targets.assign(size_t(f->B) * std::max(f->host.targetStride, 1), 0.f); // re-layout targets (tests add all blocks before setting targets)
  return MB2_OK;
}
int mb2_add_position_error_function(mb2_solver_function* f, float weight, float alpha, float c, int32_t nc, const int32_t* parents, const float* offsets,
                                    const float* weights, int32_t* outIndex) {
  HostErrorFunction ef;
  return addBlock(f, positionErrorFunction(f->ch->host, weight, alpha, c, nc, parents, offsets, weights, ef), ef, outIndex);
}
int mb2_add_position_error_function_instanced(mb2_solver_function* f, float weight, float alpha, float c, int32_t nc, const int32_t* parents, const float* weights,
                                              int32_t* outIndex) {
  HostErrorFunction ef;
  return addBlock(f, instancedPositionErrorFunction(f->ch->host, weight, alpha, c, nc, parents, weights, ef), ef, outIndex);
}
int mb2_add_plane_error_function(mb2_solver_function* f, float weight, float alpha, float c, int32_t above, int32_t nc, const int32_t* parents,
                                 const float* offsets, const float* weights, int32_t* outIndex) {
  HostErrorFunction ef;
  return addBlock(f, planeErrorFunction(f->ch->host, weight, alpha, c, above, nc, parents, offsets, weights, ef), ef, outIndex);
}
int mb2_add_model_parameters_error_function(mb2_solver_function* f, float weight, const float* targetWeights, int32_t* outIndex) {
  HostErrorFunction ef;
  return addBlock(f, modelParametersErrorFunction(f->ch->host, weight, targetWeights, ef), ef, outIndex);
}
int mb2_add_orientation_error_function(mb2_solver_function* f, float weight, float alpha, float c, int32_t rotDiff, int32_t nc, const int32_t* parents,
                                       const float* offsets, const float* weights, int32_t* outIndex) {
  HostErrorFunction ef;
  return addBlock(f, orientationErrorFunction(f->ch->host, weight, alpha, c, rotDiff, nc, parents, offsets, weights, ef), ef, outIndex);
}
int mb2_add_orientation_error_function_instanced(mb2_solver_function* f, float weight, float alpha, float c, int32_t rotDiff, int32_t nc,
                                                 const int32_t* parents, const float* weights, int32_t* outIndex) {
  HostErrorFunction ef;
  return addBlock(f, instancedOrientationErrorFunction(f->ch->host, weight, alpha, c, rotDiff, nc, parents, weights, ef), ef, outIndex);
}
int mb2_add_state_error_function(mb2_solver_function* f, float weight, int32_t rotationErrorType, float posWgt, float rotWgt, const float* posW,
                                 const float* rotW, int32_t* outIndex) {
  HostErrorFunction ef;
  return addBlock(f, stateErrorFunction(f->ch->host, weight, rotationErrorType, posWgt, rotWgt, posW, rotW, ef), ef, outIndex);
}
int mb2_add_limit_error_function(mb2_solver_function* f, float weight, float alpha, float c, int32_t* outIndex) {
  HostErrorFunction ef;
  return addBlock(f, limitErrorFunction(weight, alpha, c, ef), ef, outIndex);
}
int mb2_set_error_function_weight(mb2_solver_function* f, int32_t index, float weight) { f->host.efs[index].weight = weight; return MB2_OK; }
int mb2_set_targets(mb2_solver_function* f, int32_t index, const float* targets) {
  const HostErrorFunction& ef = f->host.efs[index];
  for (int b = 0; b < f->B; ++b) {
    float* dst = f->targets.data() + size_t(b) * f->host.targetStride + ef.targetOff;
    std::memcpy(dst, targets + size_t(b) * ef.targetSize, size_t(ef.targetSize) * sizeof(float));
    if (ef.kind == 1 || ef.kind == 2)
      for (int q = 0; q < (ef.instanceOffsets ? 2 : 1) * ef.numConstraints(); ++q) { // (an instanced block: target, then offset)
        float* p = dst + 4 * q;
        const float n = sqrtf(p[0] * p[0] + p[1] * p[1] + p[2] * p[2] + p[3] * p[3]);
        p[0] /= n; p[1] /= n; p[2] /= n; p[3] /= n;
      }
  }
  return MB2_OK;
}
int mb2_set_constraint_weights(mb2_solver_function* f, int32_t index, const float* weights, int32_t perInstance) {
  HostFunction& h = f->host;
  const HostErrorFunction& ef = h.efs[index];
  const int nc = ef.numConstraints();
  if (!perInstance) { std::copy(weights, weights + nc, h.weights.begin() + ef.weightOff); return MB2_OK; }
  if (!h.weightsPerInstance) {
    f->instanceWeights.resize(size_t(f->B) * h.numWeights);
    for (int b = 0; b < f->B; ++b) std::copy(h.weights.begin(), h.weights.end(), f->instanceWeights.begin() + size_t(b) * h.numWeights);
    h.weightsPerInstance = true;
  }
  for (int b = 0; b < f->B; ++b) std::copy(weights + size_t(b) * nc, weights + size_t(b + 1) * nc, f->instanceWeights.begin() + size_t(b) * h.numWeights + ef.weightOff);
  return MB2_OK;
}
int mb2_solver_function_set_enabled_parameters(mb2_solver_function* f, const uint64_t* bits) {
  for (int i = 0; i < f->ch->host.numParams; ++i) f->host.enabled[i] = (bits[i >> 6] >> (i & 63)) & 1ull ? 1 : 0;
  return MB2_OK;
}

int mb2_solver_function_get_error(mb2_solver_function* f, const float* params, double* errors) {
  const std::string e = plan(f, f->planCompact);
  if (!e.empty()) return fail(MB2_ERR_INVALID_ARGUMENT, e);
  const FunctionTables T = tables(f);
  for (int b = 0; b < f->B; ++b) sweepOne<false>(f, T, b, params + size_t(b) * T.numParams, &errors[b], nullptr);
  return MB2_OK;
}
int mb2_solver_function_get_skeleton_state(mb2_solver_function* f, const float* params, float* state) {
  const std::string e = plan(f, f->planCompact);
  if (!e.empty()) return fail(MB2_ERR_INVALID_ARGUMENT, e);
  const FunctionTables T = tables(f);
  double err;
  for (int b = 0; b < f->B; ++b) sweepOne<false>(f, T, b, params + size_t(b) * T.numParams, &err, state + size_t(b) * T.numJoints * 8);
  return MB2_OK;
}
int mb2_solver_function_get_jacobian(mb2_solver_function* f, const float* params, float* jac, float* residual, double* errors, int32_t* actualRows) {
  const std::string e = plan(f, false);
  if (!e.empty()) return fail(MB2_ERR_INVALID_ARGUMENT, e);
  const FunctionTables T = tables(f);
  const int rows = mb2_solver_function_jacobian_rows(f), n = T.numParams;
  for (int b = 0; b < f->B; ++b) {
    double err;
    sweepOne<true>(f, T, b, params + size_t(b) * n, &err, nullptr);
    if (errors) errors[b] = err;
    for (int c = 0; c < n && jac; ++c) std::memcpy(jac + (size_t(b) * n + c) * rows, f->J.data() + (size_t(b) * (n + 1) + c) * f->ldJ, size_t(rows) * sizeof(float));
    if (residual) std::memcpy(residual + size_t(b) * rows, f->J.data() + (size_t(b) * (n + 1) + n) * f->ldJ, size_t(rows) * sizeof(float));
  }
  if (actualRows) *actualRows = rows;
  return MB2_OK;
}
int mb2_solver_function_get_jtjr(mb2_solver_function* f, const float* params, int32_t, float* jtj, float* jtr, double* errors) {
  const std::string e = plan(f, false);
  if (!e.empty()) return fail(MB2_ERR_INVALID_ARGUMENT, e);
  const FunctionTables T = tables(f);
  const int ap = f->plan.actualParameters, n = T.numParams, ldH = roundUp(ap + 1, 16);
  std::vector<float> H(size_t(ap + 1) * ldH);
  for (int b = 0; b < f->B; ++b) {
    double err;
    sweepOne<true>(f, T, b, params + size_t(b) * n, &err, nullptr);
    if (errors) errors[b] = err;
    std::fill(H.begin(), H.end(), 0.f);
    jtjOne(f, b, ap, H.data(), ldH);
    for (int j = 0; j < ap; ++j) {
      if (jtj) for (int i = j; i < ap; ++i) jtj[(size_t(b) * ap + i) * ap + j] = H[size_t(j) * ldH + i];
      if (jtr) jtr[size_t(b) * ap + j] = H[size_t(j) * ldH + ap];
    }
  }
  return MB2_OK;
}

int mb2_solver_create(mb2_solver_function* f, const mb2_gauss_newton_options* opt, mb2_solver** out) {
  auto s = std::make_unique<mb2_solver>();
  s->fn = f;
  if (opt) s->opt = *opt; else mb2_default_gauss_newton_options(&s->opt);
  *out = s.release();
  return MB2_OK;
}
void mb2_solver_destroy(mb2_solver* s) { delete s; }
int mb2_solver_set_options(mb2_solver* s, const mb2_gauss_newton_options* opt) { s->opt = *opt; return MB2_OK; }
int mb2_solver_set_enabled_parameters(mb2_solver* s, const uint64_t* bits) { return mb2_solver_function_set_enabled_parameters(s->fn, bits); }

// the tile plan of a solve: schedule, Gram plan, and the schedule's tables as the kernels read them (S points into blob)
struct TilePlan {
  CholSchedule sched;
  GramPlan gram;
  std::vector<int32_t> blob;
  CholSchedDev S{};
};

// the plan of a solve-path request (PlanFiguresFn), with the figures the library reports for it
static int planFigures(mb2_solver_function* f, int mode, bool schedDense, bool strips, TilePlan& tp, PlanFigures& F, std::string& msg) {
  const CholSchedule& sched = tp.sched;
  const GramPlan& gram = tp.gram;
  msg = mode == 2 ? planTiles(f, schedDense ? MB2_CHOLESKY_TILES_DENSE : MB2_CHOLESKY_TILES_SPARSE, strips, tp.sched, tp.gram) : plan(f, true);
  if (!msg.empty()) return MB2_ERR_INVALID_ARGUMENT;
  F = PlanFigures{};
  F.numCols = f->plan.numCols;
  F.recStride = f->plan.recStride;
  F.jtjTensor = jtjTensorShape(F.numCols, F.numCols, f->ldJ);
  if (mode != 2) return MB2_OK;
  makeScheduleBlob(sched, tp.blob, tp.S);
  F.nPad = sched.nPad;
  F.numTiles = sched.numTiles;
  F.schedBlobInts = tp.S.blobInts;
  if (!strips) return MB2_OK;
  std::vector<int32_t> gblob;
  int32_t offsets[8];
  makeGramBlob(gram, sched, gblob, offsets);
  GramCholTables gc;
  FusedBlobLayout L;
  F.stripStride = gram.stride;
  F.gramBlobInts = int(gblob.size());
  F.orderEntries = int(gram.tileOrder.size());
  F.gramCholValid = makeGramCholTables(gram, sched, gc).empty();
  F.fusedBlobWords = int(makeFusedBlob(f->ch->host, f->plan, gblob, tp.blob, L).size());
  return MB2_OK;
}

// the library's choice of path (chooseSolvePath) for this solver, with the plan it leaves in f and tp
static int choosePath(mb2_solver* s, TilePlan& tp) {
  mb2_solver_function* f = s->fn;
  std::string msg;
  const PlanFiguresFn figures = [&](int mode, bool dense, bool strips, PlanFigures& F, std::string& m) { return planFigures(f, mode, dense, strips, tp, F, m); };
  const int rc = chooseSolvePath(s->opt, f->B, f->ch->host, f->host, figures, g_limits, s->path, msg);
  if (rc != MB2_OK) {
    s->path = SolvePath{};
    return fail(rc, msg);
  }
  return MB2_OK;
}

// emulation of mb2_solver_solve_device's launch sequence, instance by instance, on the path the library chooses. The Gram + Cholesky
// and persistent kernels run the arithmetic of the Gram and tile Cholesky kernels (bit-identical, respectively equal to float
// rounding on the device), so they are emulated as those two.
int mb2_solver_solve(mb2_solver* s, float* params, double* errors, int32_t* iterations, int32_t* status) {
  mb2_solver_function* f = s->fn;
  const auto& o = s->opt;
  TilePlan tp;
  const int rc = choosePath(s, tp);
  if (rc != MB2_OK) return rc;
  const SolvePath& P = s->path;
  if (P.kind == kSolveQr || P.kind == kSolveTrustRegionQr) return fail(MB2_ERR_UNSUPPORTED, "the CPU emulator does not emulate the QR solvers");
  const bool useGram = P.strips;
  const CholSchedule& sched = tp.sched;
  const GramPlan& gram = tp.gram;
  const CholSchedDev& S = tp.S;
  const FunctionTables T = tables(f);
  const int n = T.numParams, ns = f->plan.numCols, ldH = roundUp(ns + 1, 16);
  const int maxIt = int(o.max_iterations), minIt = int(o.min_iterations);
  s->errors.assign(f->B, DBL_MAX); s->iterations.assign(f->B, 0); s->status.assign(f->B, 0);
  s->history.assign(size_t(f->B) * std::max(maxIt, 1), 0.0);
  std::vector<float> H(size_t(ns + 1) * ldH, 0.f), delta(ns), orig(n), gramOut(useGram ? size_t(sched.numTiles) * 256 + sched.nPad : 1, 0.f);
  s->totalIterations = 0;
  for (int b = 0; b < f->B; ++b) {
    float* theta = params + size_t(b) * n;
    std::vector<float> theta0(theta, theta + n);
    double last = DBL_MAX, error = DBL_MAX;
    for (int it = 0; it < maxIt; ++it) {
      sweepOne<true>(f, T, b, theta, &error, nullptr);
      float gdd = 0.f;
      int failed;
      if (useGram) { // the strips hold no K-major matrix: the normal equations come from the Gram tiles only
        gramOne(f, b, gram, S, o.regularization, gramOut.data());
        failed = cholScheduledOne(S, nullptr, ldH, ns, o.regularization, delta.data(), &gdd, gramOut.data());
      } else {
        std::fill(H.begin(), H.end(), std::nanf("")); // entries the device never writes (lower triangle) are garbage there: poison them here
        jtjOne(f, b, ns, H.data(), ldH);
        failed = P.kind == kSolveDense ? cholDispatch(P.denseNb, H.data(), ns, ldH, o.regularization, delta.data(), &gdd)
                                       : cholScheduledOne(S, H.data(), ldH, ns, o.regularization, delta.data(), &gdd);
      }
      if (failed && s->status[b] == 0) s->status[b] = MB2_INSTANCE_CHOLESKY_BREAKDOWN;
      if (!o.do_line_search) {
        for (int a = 0; a < ns; ++a) if (f->plan.deviceCols[a] >= 0) theta[f->plan.deviceCols[a]] -= delta[a];
      } else {
        std::copy(theta, theta + n, orig.begin());
        float scale = 1.f;
        for (int step = 0; step < 10; ++step) {
          for (int a = 0; a < ns; ++a) { const int c = f->plan.deviceCols[a]; if (c >= 0) theta[c] = orig[c] - scale * delta[a]; }
          double en;
          sweepOne<false>(f, T, b, theta, &en, nullptr);
          if (lineSearchStops(error, en, scale, o.subset_line_search != 0, &gdd, step)) break;
          scale *= 0.5f;
        }
      }
      s->history[size_t(b) * std::max(maxIt, 1) + it] = error;
      s->iterations[b] = it + 1;
      if (solveStops(error, last, it, minIt, maxIt, o.threshold)) break;
      last = error;
    }
    bool bad = false;
    for (int i = 0; i < n; ++i) if (!std::isfinite(theta[i])) bad = true;
    if (bad) { std::copy(theta0.begin(), theta0.end(), theta); s->status[b] = MB2_INSTANCE_NON_FINITE; }
    s->errors[b] = error;
    s->totalIterations += s->iterations[b];
    if (errors) errors[b] = error;
    if (iterations) iterations[b] = s->iterations[b];
    if (status) status[b] = s->status[b];
  }
  return MB2_OK;
}
int mb2_solver_get_error_history(mb2_solver* s, double* history) {
  std::memcpy(history, s->history.data(), s->history.size() * sizeof(double));
  return MB2_OK;
}
int mb2_solver_get_counters(mb2_solver* s, uint64_t* totalIterations, uint64_t* kernelLaunches) {
  if (totalIterations) *totalIterations = s->totalIterations;
  if (kernelLaunches) *kernelLaunches = 0;
  return MB2_OK;
}
int mb2_solver_get_solve_path(mb2_solver* s, int64_t out[kSolvePathWords]) {
  solvePathWords(s->path, out);
  return MB2_OK;
}

} // extern "C"

// the message of the last emu_* entry of the other emulators (emu_*.cu) that failed on this thread
extern "C" const char* emu_last_error(void) { return g_emuErr.c_str(); }

// schedule / Gram-plan figures of the solver plan (cholesky_mode 3 with strips): out = {levels, tiles, tile columns, nPad, device
// columns, strips, pairs, misaligned tile starts, odd pair lists, cells outside their strip}
extern "C" int emu_plan_figures(mb2_solver_function* f, int64_t out[10]) {
  CholSchedule s;
  GramPlan g;
  const std::string e = planTiles(f, MB2_CHOLESKY_TILES_SPARSE, true, s, g);
  if (!e.empty()) return fail(MB2_ERR_INVALID_ARGUMENT, e);
  const Plan& p = f->plan;
  int64_t misaligned = 0, odd = 0, outside = 0;
  for (int K = 0; K < s.numTileCols; ++K) misaligned += (s.perm[16 * K] < 0 || (s.perm[16 * K] & 3) != 0) ? 1 : 0;
  for (int t = 0; t < s.numTiles; ++t) odd += (g.tilePairStart[t + 1] - g.tilePairStart[t]) & 1;
  for (size_t i = 0; i < p.cells.size(); ++i) {
    const int row0 = p.units[p.cells[i].unit].row0, col = p.cells[i].col;
    const int strip = int(g.cellStripOff[i] / 64), colInStrip = int(g.cellStripOff[i] % 64) / 4;
    if (strip >= g.numStrips || g.stripCoord[2 * strip] != (row0 & ~3) || g.stripCoord[2 * strip + 1] + colInStrip != col) ++outside;
  }
  out[0] = s.numLevels; out[1] = s.numTiles; out[2] = s.numTileCols; out[3] = s.nPad; out[4] = s.n; out[5] = g.numStrips; out[6] = int64_t(g.pairA.size());
  out[7] = misaligned; out[8] = odd; out[9] = outside;
  return MB2_OK;
}

// What the sweep kernel's 16-byte strip stores rely on (ik_device.cuh jacobianCell): in the solver (strip) layout every Position /
// Orientation unit starts on a row quad and owns whole quads (the rows up to the next multiple of four belong to no other unit), its
// cells sit at 16-byte aligned strip offsets, and cells are ordered by (kind, unit, device column).
// out: [0] units starting off a quad boundary, [1] units whose padding rows overlap another unit, [2] cells at unaligned strip offsets,
//      [3] cells out of (kind, unit, column) order, [4] multi-row units, [5] cells
extern "C" int emu_store_invariants(mb2_solver_function* f, int64_t out[6]) {
  CholSchedule s;
  GramPlan g;
  const std::string e = planTiles(f, MB2_CHOLESKY_TILES_SPARSE, true, s, g);
  if (!e.empty()) return fail(MB2_ERR_INVALID_ARGUMENT, e);
  const Plan& p = f->plan;
  std::vector<int> owner(size_t(p.numRows) + 8, -1);
  int64_t offQuad = 0, overlap = 0, multi = 0;
  for (size_t u = 0; u < p.units.size(); ++u) {
    const UnitDesc& d = p.units[u];
    const bool joint = d.kind == kUnitPosition || d.kind == kUnitOrientation || d.kind == kUnitOrientationRotDiff;
    if (joint) { ++multi; if ((d.row0 & 3) != 0) ++offQuad; }
    const int end = joint ? ((d.row0 + d.numRows + 3) & ~3) : d.row0 + d.numRows; // a joint unit claims its padding rows too
    for (int r = d.row0; r < end; ++r) { if (owner[size_t(r)] >= 0) ++overlap; owner[size_t(r)] = int(u); }
  }
  int64_t unaligned = 0, disorder = 0;
  for (size_t i = 0; i < p.cells.size(); ++i) {
    const CellDesc& c = p.cells[i];
    if ((g.cellStripOff[i] & 3u) != 0) ++unaligned;
    if (i > 0) {
      const CellDesc& a = p.cells[i - 1];
      const int ka = p.units[a.unit].kind, kb = p.units[c.unit].kind;
      const bool ok = ka < kb || (ka == kb && (a.unit < c.unit || (a.unit == c.unit && a.col < c.col)));
      if (!ok) ++disorder;
    }
  }
  out[0] = offQuad; out[1] = overlap; out[2] = unaligned; out[3] = disorder; out[4] = multi; out[5] = int64_t(p.cells.size());
  return MB2_OK;
}

// The tile plan of the solver function (cholesky mode 2: dense pattern, 3: sparse pattern; strips always planned) as a sequence of int32
// sections, each [length, values...], in this order:
//   header {n (device columns), nPad, numTileCols, numTiles, numLevels, nParams, numRows, numStrips, strip stride, residOff, parkTiles,
//           16-bit tables valid, then the 12 section offsets of GramCholLayout};
//   perm, pos, deviceCols (device column -> model parameter, -1 = gap), tileRow, tileCol, tileIdTable, diagTile,
//   levelColStart, levelCols, levelPanelStart, panelTile, panelDiag, panelRow, levelTaskStart, taskDst, taskPairStart, pairA, pairB,
//   levelVTaskStart, vtaskRow, vtaskSrcStart, vsrcTile, vsrcCol, colPanelStart, colPanelTile, colPanelRow,
//   levelOrderStart8, taskOrder8, levelOrderStart16, taskOrder16,
//   Gram plan: stripCoord, tilePairStart, pairA, pairB, tileOrder, tileQuadStart, quad, colStripStart, colStrip, cellStripOff, cellQuadStride,
//   GramCholTables::tab (undecoded), cells [numCells][5] {first row, row count, device column, unit, unit kind}.
// Called with out = nullptr it only returns the word count in *words; with a buffer of *words ints it fills it.
extern "C" int emu_tile_plan(mb2_solver_function* f, int32_t cholMode, int32_t* out, int64_t* words) {
  CholSchedule s;
  GramPlan g;
  const std::string e = planTiles(f, cholMode, true, s, g);
  if (!e.empty()) return fail(MB2_ERR_INVALID_ARGUMENT, e);
  GramCholTables gc;
  const bool valid = makeGramCholTables(g, s, gc).empty();
  const Plan& p = f->plan;
  std::vector<int32_t> blob;
  auto add = [&](auto first, auto last) { blob.push_back(int32_t(last - first)); for (auto it = first; it != last; ++it) blob.push_back(int32_t(*it)); };
  auto sec = [&](const auto& v) { add(v.begin(), v.end()); };
  const GramCholLayout& L = gc.L;
  const std::vector<int32_t> header = {s.n, s.nPad, s.numTileCols, s.numTiles, s.numLevels, s.nParams, p.numRows, g.numStrips, g.stride, g.residOff,
                                       gc.parkTiles, valid ? 1 : 0, L.gram, L.quad, L.col, L.colEnt, L.level, L.diag, L.panel, L.order, L.pair, L.vtask,
                                       L.vsrc, L.colPanel};
  sec(header);
  sec(s.perm); sec(s.pos); sec(p.deviceCols); sec(s.tileRow); sec(s.tileCol); sec(s.tileIdTable); sec(s.diagTile);
  sec(s.levelColStart); sec(s.levelCols); sec(s.levelPanelStart); sec(s.panelTile); sec(s.panelDiag); sec(s.panelRow);
  sec(s.levelTaskStart); sec(s.taskDst); sec(s.taskPairStart); sec(s.pairA); sec(s.pairB);
  sec(s.levelVTaskStart); sec(s.vtaskRow); sec(s.vtaskSrcStart); sec(s.vsrcTile); sec(s.vsrcCol);
  sec(s.colPanelStart); sec(s.colPanelTile); sec(s.colPanelRow);
  sec(s.levelOrderStart8); sec(s.taskOrder8); sec(s.levelOrderStart16); sec(s.taskOrder16);
  sec(g.stripCoord); sec(g.tilePairStart); sec(g.pairA); sec(g.pairB); sec(g.tileOrder); sec(g.tileQuadStart); sec(g.quad);
  sec(g.colStripStart); sec(g.colStrip); sec(g.cellStripOff); sec(g.cellQuadStride);
  sec(gc.tab);
  std::vector<int32_t> cells;
  for (const CellDesc& c : p.cells) {
    const UnitDesc& u = p.units[c.unit];
    cells.insert(cells.end(), {int32_t(u.row0), int32_t(u.numRows), int32_t(c.col), int32_t(c.unit), int32_t(u.kind)});
  }
  sec(cells);
  if (out != nullptr) {
    if (*words < int64_t(blob.size())) return fail(MB2_ERR_INVALID_ARGUMENT, "emu_tile_plan: buffer too small");
    std::copy(blob.begin(), blob.end(), out);
  }
  *words = int64_t(blob.size());
  return MB2_OK;
}

// The normal equations the tile-sparse Gram computes for instance b at params (the instance's theta, [numParams] floats), without
// damping: out = [numTiles][256] tiles in the fragment layout (tileIdx; padded rows / columns hold the identity extension) followed
// by J^T r in slot order [nPad]. *floats gets the count; out = nullptr only returns it.
extern "C" int emu_gram_system(mb2_solver_function* f, int32_t cholMode, int32_t b, const float* params, float* out, int64_t* floats) {
  TilePlan tp;
  const std::string e = planTiles(f, cholMode, true, tp.sched, tp.gram);
  if (!e.empty()) return fail(MB2_ERR_INVALID_ARGUMENT, e);
  const int64_t count = int64_t(tp.sched.numTiles) * 256 + tp.sched.nPad;
  if (out != nullptr) {
    if (*floats < count) return fail(MB2_ERR_INVALID_ARGUMENT, "emu_gram_system: buffer too small");
    makeScheduleBlob(tp.sched, tp.blob, tp.S);
    const FunctionTables T = tables(f);
    double err;
    sweepOne<true>(f, T, b, params, &err, nullptr);
    gramOne(f, b, tp.gram, tp.S, 0.f, out);
  }
  *floats = count;
  return MB2_OK;
}

// The device the solve path is chosen for (SM count, opt-in shared memory per block, shared memory per SM).
extern "C" void emu_set_device_limits(int32_t numSms, int32_t smemOptin, int32_t smemPerSm) { g_limits = DeviceLimits{numSms, smemOptin, smemPerSm}; }

// The solve path of the solver's next solve (mb2_solver_get_solve_path afterwards), without solving: planning only.
extern "C" int emu_choose_solve_path(mb2_solver* s) {
  TilePlan tp;
  return choosePath(s, tp);
}
