#include "ik_solve_path.h"

#include <algorithm>
#include <cstring>

#include "ik_chol.cuh"

namespace mb2 {

std::vector<int32_t> makeFusedBlob(const HostCharacter& h, const Plan& p, const std::vector<int32_t>& gramBlob, const std::vector<int32_t>& schedBlob, FusedBlobLayout& L) {
  std::vector<int32_t> blob;
  auto add = [&](const void* data, size_t bytes) {
    const int32_t off = int32_t(blob.size());
    const size_t words = (bytes + 3) / 4;
    blob.resize(blob.size() + words, 0);
    if (bytes) std::memcpy(blob.data() + off, data, bytes);
    while (blob.size() % 4) blob.push_back(0);
    return off;
  };
  L.parent = add(h.parent.data(), h.parent.size() * 4);
  L.offset = add(h.offset.data(), h.offset.size() * 4);
  L.prerot = add(h.prerot.data(), h.prerot.size() * 4);
  L.ptOuter = add(h.ptOuter.data(), h.ptOuter.size() * 4);
  L.ptInner = add(h.ptInner.data(), h.ptInner.size() * 4);
  L.ptVals = add(h.ptVals.data(), h.ptVals.size() * 4);
  L.ptOffsets = add(h.ptOffsets.data(), h.ptOffsets.size() * 4);
  L.levelStart = add(h.levelStart.data(), h.levelStart.size() * 4);
  L.levelJoints = add(h.levelJoints.data(), h.levelJoints.size() * 4);
  L.efs = add(p.efs.data(), p.efs.size() * sizeof(EfDesc));
  L.units = add(p.units.data(), p.units.size() * sizeof(UnitDesc));
  L.cells = add(p.cells.data(), p.cells.size() * sizeof(CellDesc));
  L.contribs = add(p.contribs.data(), p.contribs.size() * sizeof(ContribDesc));
  L.limitData = add(p.limitData.data(), p.limitData.size() * 4);
  L.cols = add(p.deviceCols.data(), p.deviceCols.size() * 4);
  L.gram = add(gramBlob.data(), gramBlob.size() * 4);
  L.sched = add(schedBlob.data(), schedBlob.size() * 4);
  if (blob.empty()) blob.push_back(0);
  while (blob.size() % 4) blob.push_back(0);
  L.words = int32_t(blob.size());
  return blob;
}

size_t cholSmemBytes(int n, int NB, bool matrixInSmem) {
  const size_t ldp = ((n + 1 + 3) & ~3) + 4;
  size_t s = sizeof(float) * (NB * ldp + ((n + 3) & ~3)) + 4 * sizeof(int);
  if (matrixInSmem) s += sizeof(float) * size_t(n + 1) * (n | 1);
  return s;
}

size_t gramTilesSmemBytes(size_t stripStride, int blobInts) { return 128 + sizeof(float) * (stripStride + 64) + 16 + sizeof(int32_t) * size_t((blobInts + 3) & ~3); }

size_t choleskyScheduledSmemBytes(int n, int nPad, int numTiles, int blobInts) {
  return 1024 /*tile storage is aligned to the TMA swizzle atom*/ + sizeof(float) * (size_t(numTiles) * 256 + size_t(nPad) + 2 * size_t((n + 3) & ~3)) +
         sizeof(int32_t) * size_t((blobInts + 3) & ~3) + 32;
}

// the plan tables are not staged in shared memory (gramCholeskyKernel reads them from its parameter block or global memory)
size_t gramCholeskySmemBytes(size_t stripStride, int n, int nPad, int numTiles) {
  const size_t uni = std::max<size_t>(size_t(numTiles) * 256, stripStride + 64);
  return 128 + sizeof(float) * (((uni + 3) & ~size_t(3)) + size_t(nPad) + size_t((n + 3) & ~3)) + 32;
}

size_t qrSmemFloats(int n, int maxChunkRows) {
  return (size_t(n) * (n + 1) / 2 + 3 & ~size_t(3)) + 3 * size_t((n + 3) & ~3) + size_t((n + 4) & ~3) + size_t(n + 1) * size_t(maxChunkRows | 1) + 8;
}
int qrMaxChunkRows(int n, size_t smemBytes) {
  const size_t fixed = qrSmemFloats(n, 0) - size_t(n + 1);
  const size_t floats = smemBytes / sizeof(float);
  if (floats <= fixed + size_t(n + 1) * 9) return 0;
  int p = int((floats - fixed) / size_t(n + 1)) - 1;
  p = std::min(p, 128) & ~1; // even: p | 1 = p + 1 stays inside the budget
  return p;
}

size_t trQrSmemFloats(int n, int numParams, int numJoints, int maxChunkRows) {
  const size_t packed = (size_t(n) * (n + 1) / 2 + 3) & ~size_t(3);
  const size_t n4 = size_t((n + 3) & ~3), np4 = size_t((numParams + 3) & ~3);
  const size_t chunk = (size_t(n + 1) * size_t(maxChunkRows | 1) + 3) & ~size_t(3);
  return packed + std::max(packed, chunk) + 7 * n4 + size_t((n + 4) & ~3) + 2 * np4 + size_t((numJoints * kJointStateStride + 3) & ~3) + 64;
}

bool jtjTensorShape(int ns, int numCols, int ldJ) { return ns >= 1 && ns <= numCols && numCols + 1 <= 512 && (ldJ % kJtjKBlock) == 0; }

int resolveJtjMode(int requested, bool tensorOk) {
  if (requested == MB2_JTJ_FP32_SIMT) return MB2_JTJ_FP32_SIMT;
  if (requested == MB2_JTJ_AUTO) return tensorOk ? MB2_JTJ_TF32X3 : MB2_JTJ_FP32_SIMT;
  return tensorOk ? requested : -1;
}

namespace {

// how many instance groups of the persistent kernel fit next to the staged tables (0: it cannot run this plan)
FusedConfig fusedConfigure(const PlanFigures& P, const HostCharacter& ch, int maxSmemOptin) {
  FusedConfig c;
  const int nc4 = (P.numCols + 3) & ~3, np4 = (ch.numParams + 3) & ~3;
  const int sweep = P.stripStride + 64 + ((ch.numJoints * kJointStateStride + 3) & ~3) + ((ch.numJoints * kParametersPerJoint + 3) & ~3) + ((P.recStride + 3) & ~3);
  c.unionFloats = (std::max(P.numTiles * 256, sweep) + 3) & ~3;
  c.groupFloats = c.unionFloats + P.nPad + 2 * nc4 + np4 + 32; // + 10 doubles and 4 ints of per-instance state
  if (P.orderEntries / kGramWarps > kFusedMaxRounds) return c; // more parked tiles per warp than the kernel holds
  const size_t fixed = 128 + size_t(P.fusedBlobWords) * 4 + 16;
  for (int g = kFusedMaxGroups; g >= 1; --g) {
    const size_t need = fixed + size_t(g) * c.groupFloats * sizeof(float);
    if (need <= size_t(maxSmemOptin)) {
      c.groups = g;
      c.smemBytes = need;
      break;
    }
  }
  return c;
}

// the tile kernels run 256 threads, or 512 when one CTA per SM is all that fits anyway
int tileThreads(size_t smem, const DeviceLimits& lim) { return 2 * (smem + 1024) > size_t(lim.smemPerSm) ? 512 : 256; }

} // namespace

int chooseSolvePath(const mb2_gauss_newton_options& o, int batch, const HostCharacter& ch, const HostFunction& fn, const PlanFiguresFn& plan,
                    const DeviceLimits& lim, SolvePath& P, std::string& msg) {
  P = SolvePath{};
  P.slices = 1;
  auto refuse = [&](int code, const char* m) { msg = m; return code; };
  PlanFigures F;
  auto request = [&](int mode, bool schedDense, bool strips) {
    P.planMode = mode;
    P.schedDense = schedDense;
    P.strips = strips;
    const int rc = plan(mode, schedDense, strips, F, msg);
    P.fused = rc == MB2_OK && strips ? fusedConfigure(F, ch, lim.smemOptin) : FusedConfig{};
    return rc;
  };
  // Cholesky path: 1 dense Eigen-structured kernel, 2 tile schedule on the dense pattern, 3 tile schedule on the sparse pattern
  int cholMode = resolveCholeskyMode(o.cholesky_mode, fn.enabled);
  // GaussNewtonSolverQRT's step: Householder QR of the K-major Jacobian (ik_qr.cuh); TrustRegionQRT's iteration builds on the same fold (ik_tr_qr.cuh)
  const bool useTr = o.linear_solver == MB2_LINEAR_SOLVER_TRUST_REGION_QR;
  const bool useQr = o.linear_solver == MB2_LINEAR_SOLVER_QR || useTr;
  if (useTr && !(o.trust_region_radius > 0.f)) return refuse(MB2_ERR_INVALID_ARGUMENT, "trust_region_radius must be positive");
  if (useQr) {
    if (o.jtj_mode == MB2_JTJ_SPARSE_TILES || o.cholesky_mode >= 2 || o.fused_mode >= MB2_FUSED_PERSISTENT)
      return refuse(MB2_ERR_UNSUPPORTED, "the QR step works on the dense Jacobian: it excludes the tile-sparse Gram, the tile Cholesky and the fused kernels");
    cholMode = 1;
  }
  // tile-sparse Gram: default whenever the tile-scheduled Cholesky runs (MB2_JTJ_AUTO), or on request
  bool useGram = cholMode >= 2 && (o.jtj_mode == MB2_JTJ_AUTO || o.jtj_mode == MB2_JTJ_SPARSE_TILES);
  if (o.jtj_mode == MB2_JTJ_SPARSE_TILES && cholMode < 2) return refuse(MB2_ERR_UNSUPPORTED, "MB2_JTJ_SPARSE_TILES needs the tile-scheduled Cholesky");
  int rc = request(cholMode >= 2 ? 2 : 1, cholMode == 2, useGram);
  if (rc != MB2_OK) return rc;
  bool useSchedule = cholMode >= 2;
  if (useSchedule && choleskyScheduledSmemBytes(F.numCols, F.nPad, F.numTiles, F.schedBlobInts) > size_t(200 * 1024)) {
    if (o.cholesky_mode >= 2) return refuse(MB2_ERR_UNSUPPORTED, "tile schedule does not fit in shared memory for this system");
    useSchedule = false; // fall back to the dense kernel (matrix in global memory)
    useGram = false;
    if ((rc = request(1, false, false)) != MB2_OK) return rc;
  }
  const int ns = F.numCols;
  if (ns <= 0) return refuse(MB2_ERR_INVALID_ARGUMENT, "no enabled parameters");
  if (useGram && gramTilesSmemBytes(size_t(F.stripStride), F.gramBlobInts) > size_t(200 * 1024)) {
    if (o.jtj_mode == MB2_JTJ_SPARSE_TILES) return refuse(MB2_ERR_UNSUPPORTED, "Jacobian strips do not fit in shared memory for this system");
    useGram = false;
    if ((rc = request(2, cholMode == 2, false)) != MB2_OK) return rc;
  }
  // ---- fused persistent kernel: the whole solve in one launch (ik_fused.cuh) ----
  const bool eligible = useGram && useSchedule && o.do_line_search == 0 && P.fused.groups >= 1;
  if (o.fused_mode == MB2_FUSED_PERSISTENT && !eligible)
    return refuse(MB2_ERR_UNSUPPORTED, "the fused kernel needs the tile-sparse Gram + tile-scheduled Cholesky path, no line search, and a plan that fits in shared memory");
  // AUTO takes the persistent kernel when the whole batch is one wave of instance groups: a single launch with no host round trip
  // saves ~2 launches per iteration there (H100 80GB HBM3 at 400 W, 256 x humanoid72 x 10 iterations: 0.68 - 0.71 vs 0.83 ms); at
  // thousands of instances the per-iteration kernels keep more instances in flight per SM (the persistent kernel holds at most three)
  // and AUTO keeps them (8192 instances: 13.0 vs 9.8 - 9.9 ms)
  if (eligible && (o.fused_mode == MB2_FUSED_PERSISTENT || (o.fused_mode == MB2_FUSED_AUTO && batch <= P.fused.groups * lim.numSms))) {
    P.kind = kSolvePersistent;
    P.jtjMode = MB2_JTJ_SPARSE_TILES;
    return MB2_OK;
  }
  // ---- Gram + Cholesky in one launch per iteration (gramCholeskyKernel): the default on the tile path ----
  bool useGramChol = false;
  if (useGram && useSchedule) {
    const int rounds = std::max(F.orderEntries / kGramWarps, 1);
    const bool fits = gramCholeskySmemBytes(size_t(F.stripStride), ns, F.nPad, F.numTiles) <= size_t(200 * 1024) && rounds <= kGramCholMaxRounds && F.gramCholValid;
    if (o.fused_mode == MB2_FUSED_GRAM_CHOLESKY && !fits) return refuse(MB2_ERR_UNSUPPORTED, "Gram + Cholesky fusion: strips / tiles of this plan do not fit in shared memory, or too many tiles per warp");
    useGramChol = fits && (o.fused_mode == MB2_FUSED_AUTO || o.fused_mode == MB2_FUSED_GRAM_CHOLESKY);
  } else if (o.fused_mode == MB2_FUSED_GRAM_CHOLESKY) {
    return refuse(MB2_ERR_UNSUPPORTED, "Gram + Cholesky fusion needs the tile-sparse Gram + tile-scheduled Cholesky path");
  }
  P.jtjMode = useGram ? MB2_JTJ_SPARSE_TILES : resolveJtjMode(o.jtj_mode == MB2_JTJ_SPARSE_TILES ? MB2_JTJ_AUTO : o.jtj_mode, F.jtjTensor);
  if (P.jtjMode < 0) return refuse(MB2_ERR_UNSUPPORTED, "tensor-core JtJ does not support this shape");
  if (useQr) { // row chunks: one per error-function block (the reference adds block by block), split when a block does not fit beside R
    int rows = qrMaxChunkRows(ns, size_t(200 * 1024));
    if (rows < 8) return refuse(MB2_ERR_UNSUPPORTED, "the QR step keeps R in shared memory: too many enabled parameters for this kernel");
    if (useTr) { // R and the damping rows D (both packed triangles) + the in-kernel getError scratch; the Jacobian chunk shares D's storage
      rows = std::min(rows, std::max(8, ns / 2));
      if (trQrSmemFloats(ns, ch.numParams, ch.numJoints, rows) * sizeof(float) > size_t(220 * 1024))
        return refuse(MB2_ERR_UNSUPPORTED, "the trust-region QR kernel keeps R and the damping rows in shared memory: too many enabled parameters / joints");
      P.trRSavedFloats = (size_t(ns) * (ns + 1) / 2 + 3) & ~size_t(3);
    }
    P.qrMaxChunkRows = rows;
    P.qrChunkStarts.assign(1, 0);
    int r0 = 0, widest = 0;
    for (const auto& ef : fn.efs) {
      if (!(ef.weight > 0.f)) continue;
      const int size = jacobianBlockSize(ch, ef);
      for (int done = 0; done < size; done += rows) { const int p = std::min(rows, size - done); P.qrChunkStarts.push_back(r0 + done + p); widest = std::max(widest, p); }
      r0 += size;
    }
    P.qrWidestChunk = std::max(widest, 1);
    P.kind = useTr ? kSolveTrustRegionQr : kSolveQr;
  } else if (useGramChol) {
    P.kind = kSolveGramCholesky;
    // resident gramCholeskyKernel CTAs on the device (1 KB of shared memory is reserved per CTA); the line search's launches run on
    // the whole batch, so only the plain iteration chain is sliced
    const size_t perCta = gramCholeskySmemBytes(size_t(F.stripStride), ns, F.nPad, F.numTiles) + 1024;
    const int resident = lim.numSms * std::min<int>(kGramCholCtasPerSm, int(size_t(lim.smemPerSm) / perCta));
    if (o.do_line_search == 0 && resident > 0 && batch >= kSliceMinWaves * resident) P.slices = kSolveSlices;
  } else if (useSchedule) {
    P.kind = useGram ? kSolveTiles : kSolveTilesKMajor;
    P.cholThreads = tileThreads(choleskyScheduledSmemBytes(ns, F.nPad, F.numTiles, F.schedBlobInts), lim);
    if (useGram) P.gramThreads = tileThreads(gramTilesSmemBytes(size_t(F.stripStride), F.gramBlobInts), lim);
  } else {
    P.kind = kSolveDense;
    const int eig = cholBlockSize(ns, 32);
    P.denseNb = eig <= 8 ? 8 : (eig <= 16 ? 16 : 32);
    P.denseInSmem = cholSmemBytes(ns, P.denseNb, true) <= size_t(lim.smemOptin);
  }
  return MB2_OK;
}

void solvePathWords(const SolvePath& p, int64_t out[kSolvePathWords]) {
  const int64_t w[kSolvePathWords] = {p.kind, p.planMode, p.schedDense, p.strips, p.jtjMode, p.denseNb, p.denseInSmem, p.gramThreads, p.cholThreads,
                                      p.qrMaxChunkRows, p.qrChunkStarts.empty() ? 0 : int64_t(p.qrChunkStarts.size()) - 1, p.qrWidestChunk,
                                      int64_t(p.trRSavedFloats), p.fused.groups, int64_t(p.fused.smemBytes), p.slices};
  std::copy(w, w + kSolvePathWords, out);
}

} // namespace mb2
