// How one solve runs its Gauss-Newton iterations: the choice between the linear-solve paths, the shared-memory size rules it rests
// on, and the launch variants that follow from them. Host code only, shared by the library (ik_capi.cu) and the CPU emulator
// (tests/emu), so that both run the path this decides.
#pragma once

#include <cstddef>
#include <cstdint>
#include <functional>
#include <string>
#include <vector>

#include "../../include/momentum_b200.h"
#include "ik_plan.h"

namespace mb2 {

constexpr int kFusedMaxGroups = 3;
constexpr int kFusedMaxRounds = 32; // rounds of the Gram tile-order table a warp can park (fusedConfigure refuses larger plans)

// word (4-byte) offsets of the tables inside the fused kernel's plan blob (every table starts on a 16-byte boundary)
struct FusedBlobLayout {
  int32_t parent, offset, prerot, ptOuter, ptInner, ptVals, ptOffsets, levelStart, levelJoints;
  int32_t efs, units, cells, contribs, limitData;
  int32_t cols;       // device column -> model parameter (-1: alignment column)
  int32_t gram;       // Gram plan blob (makeGramBlob), gramOff[] are relative to it
  int32_t sched;      // Cholesky schedule blob (makeScheduleBlob)
  int32_t words;      // total size, multiple of 4
};
// Every table the fused kernel walks, as one 16-byte-aligned blob (bulk-copied into shared memory once per CTA).
std::vector<int32_t> makeFusedBlob(const HostCharacter& h, const Plan& p, const std::vector<int32_t>& gramBlob, const std::vector<int32_t>& schedBlob, FusedBlobLayout& L);

struct FusedConfig {
  int groups{0};
  int groupFloats{0}, unionFloats{0};
  size_t smemBytes{0};
};

// Shared memory of the linear-solve kernels
size_t cholSmemBytes(int n, int NB, bool matrixInSmem); // dense Eigen-structured Cholesky
size_t gramTilesSmemBytes(size_t stripStride, int blobInts);
size_t choleskyScheduledSmemBytes(int n, int nPad, int numTiles, int blobInts);
size_t gramCholeskySmemBytes(size_t stripStride, int n, int nPad, int numTiles);
size_t qrSmemFloats(int n, int maxChunkRows);
int qrMaxChunkRows(int n, size_t smemBytes); // rows of Jacobian that fit beside R (0: the system is too large for this kernel)
size_t trQrSmemFloats(int n, int numParams, int numJoints, int maxChunkRows);
constexpr int kJtjKBlock = 32; // floats per K block of the tensor-core JtJ (one 128-byte swizzle row)
// the shapes the tensor-core JtJ handles: at most four row tiles, at most one far item per tile
bool jtjTensorShape(int ns, int numCols, int ldJ);
// the MB2_JTJ_* mode that runs for a request: AUTO takes the tensor cores where they can; -1 for a tensor-core request they cannot serve
int resolveJtjMode(int requested, bool tensorOk);

struct DeviceLimits {
  int numSms{0}, smemOptin{0}, smemPerSm{0};
};

// What a built plan weighs, as far as the size rules need it
struct PlanFigures {
  int numCols{0};                // device columns (the solve's ns)
  int recStride{0};
  bool jtjTensor{false};         // the tensor-core JtJ supports this plan (jtjTensorShape, and the device can build tensor maps)
  int nPad{0}, numTiles{0}, schedBlobInts{0};                   // tile schedule (plan mode 2)
  int stripStride{0}, gramBlobInts{0}, orderEntries{0};         // Gram plan (strips)
  bool gramCholValid{false};     // makeGramCholTables accepted the plan
  int fusedBlobWords{0};
};
// Builds (or keeps) the plan of a request and reports its figures: mode 1 compact columns in natural order, 2 the tile schedule
// (schedDense: on the dense pattern) with the Jacobian in strips when `strips`. Returns MB2_OK or an error code with `msg` set.
using PlanFiguresFn = std::function<int(int mode, bool schedDense, bool strips, PlanFigures& out, std::string& msg)>;

enum SolveKind : int32_t {
  kSolveNone = 0,
  kSolveDense = 1,        // JtJ (SIMT / tensor cores) + dense Eigen-structured Cholesky
  kSolveTilesKMajor = 2,  // JtJ on the K-major Jacobian + tile-scheduled Cholesky
  kSolveTiles = 3,        // sweep, gramTilesKernel, choleskyScheduledKernel
  kSolveGramCholesky = 4, // sweep, gramCholeskyKernel
  kSolvePersistent = 5,   // fusedSolveKernel: the whole solve in one launch
  kSolveQr = 6,
  kSolveTrustRegionQr = 7,
};

struct SolvePath {
  int32_t kind{kSolveNone};
  int32_t planMode{0};                // the plan request: 1 or 2 (see PlanFiguresFn)
  bool schedDense{false}, strips{false};
  int32_t jtjMode{0};                 // MB2_JTJ_* after AUTO resolution (MB2_JTJ_SPARSE_TILES on the strips)
  int32_t denseNb{0};                 // dense kernel: block size and where its matrix lives
  bool denseInSmem{false};
  int32_t gramThreads{0}, cholThreads{0}; // gramTilesKernel / choleskyScheduledKernel: 256, or 512 when one CTA per SM is all that fits
  int32_t qrMaxChunkRows{0};          // Jacobian rows the QR kernels fold at once (the limit; the widest chunk may be smaller)
  std::vector<int32_t> qrChunkStarts; // [chunks + 1] first row of every chunk: one per block, split at qrMaxChunkRows
  int32_t qrWidestChunk{0};
  size_t trRSavedFloats{0};           // trust-region QR: floats of the saved R per instance
  FusedConfig fused;                  // persistent kernel: instance groups per CTA next to the staged plan (every plan with strips it requested)
};

// The path of one solve of `batch` instances with options `o`. Every refusal returns its error code with `msg` set; plan builds go
// through `plan`, in the order the fallbacks need them.
int chooseSolvePath(const mb2_gauss_newton_options& o, int batch, const HostCharacter& ch, const HostFunction& fn, const PlanFiguresFn& plan,
                    const DeviceLimits& lim, SolvePath& out, std::string& msg);

constexpr int kSolvePathWords = 15;
// the record as mb2_solver_get_solve_path reports it (include/momentum_b200.h)
void solvePathWords(const SolvePath& p, int64_t out[kSolvePathWords]);

} // namespace mb2
