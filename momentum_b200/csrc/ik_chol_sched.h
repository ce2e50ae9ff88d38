// Level-scheduled, tile-sparse Cholesky: host-side symbolic analysis.
//
// The reference factors the dense normal matrix with Eigen::LLT (gauss_newton_solver.cpp:251). For a
// skeleton, (J^T J)(p,q) is structurally non-zero only when some residual row depends on both p and q,
// i.e. when their joints lie on one root-to-constraint path (joint_error_function-inl.h:229-294 walks
// exactly that path) — so the matrix of a branching rig is mostly zero blocks (the two arms never
// couple), and eliminating children before parents creates no fill outside that structure.
// This analysis (once per plan) turns the sparsity pattern into a static schedule for the device:
//   1. minimum-degree ordering of the enabled parameters (pattern = cliques of the Jacobian row groups),
//   2. 16x16 tiles over the permuted order, tile-level symbolic factorisation (fill included),
//   3. the tile elimination tree and its levels: all tile columns of one level are independent, so
//      a level costs three block-wide phases no matter how many columns it holds,
//   4. per level: diagonal tiles, panel tiles, and one update task per destination tile listing every
//      (L(I,K), L(J,K)) pair that contributes to it (deterministic summation order, no atomics).
// A dense matrix is the special case "every tile non-zero, elimination tree = chain".
// The solution of (H + lambda I) x = g is the same as Eigen's up to rounding.
#pragma once

#include <cstdint>
#include <string>
#include <vector>

namespace mb2 {

constexpr int kCholTile = 16;

struct CholSchedule {
  int32_t n{0}, nPad{0}, numTileCols{0}, numTiles{0}, numLevels{0};
  int32_t nParams{0};                   // parameters in the system (n also counts alignment gaps after layoutDeviceColumns)
  std::vector<int16_t> perm;            // [nPad] permuted position -> device column, -1 = padding
  std::vector<int16_t> pos;             // [n] device column -> permuted position (inverse of perm)
  std::vector<int16_t> tileIdTable;     // [numTileCols * numTileCols] tile id of (I,J), I >= J, or -1
  std::vector<int16_t> tileRow, tileCol; // [numTiles] block coordinates (I >= J)
  std::vector<int32_t> diagTile;        // [numTileCols]
  // per level
  std::vector<int32_t> levelColStart, levelCols;       // tile columns K of each level
  std::vector<int32_t> levelPanelStart, panelTile, panelDiag, panelRow; // panel tiles (I,K) of the level's columns; diag tile of K; block row I
  std::vector<int32_t> levelTaskStart, taskDst, taskPairStart, pairA, pairB; // matrix update tasks
  // which warp runs which update task: per level a [rounds][W] table (W = 8 or 16 warps per instance), -1 = idle; longest task first to
  // the least loaded warp (the root tile of a humanoid collects 12 pairs, the median task 4: dealing tasks round-robin made one warp do 17)
  std::vector<int32_t> levelOrderStart8, taskOrder8, levelOrderStart16, taskOrder16;
  std::vector<int32_t> levelVTaskStart, vtaskRow, vtaskSrcStart, vsrcTile, vsrcCol; // forward-substitution updates y_I -= L(I,K) y_K
  // per tile column (backward substitution): its panel tiles
  std::vector<int32_t> colPanelStart, colPanelTile, colPanelRow;
  std::vector<int> order;               // elimination order: order[i] = input column eliminated i-th
  // statistics
  int64_t tileOps{0};      // 16x16x16 multiply-accumulate blocks executed by update tasks
  int64_t denseTileOps{0}; // what a dense factorisation of the same size would execute
};

// `cliques`: for every Jacobian row group, the device columns it touches (each list is a clique of the
// pattern). n = number of device columns that enter the normal equations.
// `priority` (optional, per column): among columns of equal degree the ordering eliminates the larger priority first. Callers pass
// the depth of the joint a parameter drives: in the final cliques of a kinematic tree every order has the same fill, but only
// leaf-to-root orders keep independent limbs in separate subtrees of the tile elimination tree (= fewer levels).
std::string buildCholSchedule(int n, const std::vector<std::vector<int>>& cliques, bool forceDense, CholSchedule& out, const std::vector<int>* priority = nullptr);
// Device column layout of the solver plan: parameters in elimination order, and every tile column starting on a device column
// that is a multiple of 4 (TMA fetches a tile as one 16 x 16 box of the row-major H; the first byte of each box row must be
// 16-byte aligned). The up-to-3 skipped device columns before such a start are all-zero Jacobian columns ("gaps").
// deviceColumnOrder[d] = input column (as numbered in `cliques`) held by device column d, or -1 for a gap. Rewrites perm / pos
// to device columns (pos[d] = slot or -1) and sets n to the number of device columns (nParams keeps the original count).
void layoutDeviceColumns(CholSchedule& s, std::vector<int32_t>& deviceColumnOrder);

// Leading dimension of the row-major symmetric matrix [J r]^T [J r] the JtJ kernels write and the scheduled Cholesky reads.
inline int cholSchedLdH(int n) { return (n + 1 + 15) / 16 * 16; }
// tileInfo (3 ints per tile, in the device blob): {gi0, gj0, validI | validJ << 8 | diag << 16}: tile (I,J) is the 16x16 box of
// H with first row gj0 (device column of slot 16 J) and first column gi0 (slot 16 I); only its first validJ rows / validI columns
// are real (padding only closes a tile), the rest is overwritten by the padding pass.
// ---- Tile-sparse Gram plan: the stored tiles of J^T J straight from the non-zero pieces of the Jacobian ----
// Row quads: rows 4q..4q+3 of the (row-group aligned) Jacobian. A *strip* is (quad q, tile column K): the 4 x 16 piece
// J[4q..4q+3][gi0(K)..gi0(K)+15] -- one TMA box of the K-major device Jacobian, landing as [16 columns][4 rows]. A strip
// exists only where a unit with rows in q has a cell in tile column K. Tile (I,J) = sum over quads touching both I and J
// of strip(q,I)^T strip(q,J); block K of J^T r = sum over its strips of strip^T r[4q..4q+3].
constexpr int kGramWarps = 8; // warps that share the tiles of one instance (gramTilesKernel, gramCholeskyKernel, a group of the fused kernel)
// gramCholeskyKernel writes the tiles over the strips they are computed from: a finished tile that would land on strips still being
// read waits in its warp's registers' spill space (thread-local memory, served by L1 / L2) until every warp is done with the strips.
// Rounds of the tile-order table that one warp can hold that way.
constexpr int kGramCholMaxRounds = 8;
struct GramPlan {
  int32_t numStrips{0}, numTiles{0}, numTileCols{0};
  std::vector<int32_t> stripCoord;    // [numStrips][2] {first row 4q, first device column gi0(K)}; strips are ordered by (quad, tile column)
  std::vector<int32_t> tileOrder;     // [rounds][kGramWarps] tile of warp w in round r, -1 = none (longest-first / least-loaded assignment)
  std::vector<int32_t> tilePairStart; // [numTiles + 1] indexed by tile id
  std::vector<int32_t> pairA, pairB;  // strips of block row I / block column J of the tile
  std::vector<int32_t> tileQuadStart; // [numTiles + 1] the same lists, two pairs per entry, as the kernel consumes them:
  std::vector<int32_t> quad;          // [numQuads][4] float offsets {A0, B0, A1, B1} of the four strips (16-byte aligned records)
  std::vector<int32_t> colStripStart; // [numTileCols + 1]
  std::vector<int32_t> colStrip;      // strips of tile column K
  std::vector<uint32_t> cellStripOff; // per Jacobian cell: float offset of (first row quad, its column) in the strip buffer
  std::vector<uint16_t> cellQuadStride; // per cell: strips between consecutive row quads of its unit
  int32_t residOff{0};                // the residual (aligned row numbering) follows the strips
  int32_t stride{0};                  // floats per instance: residOff + rows rounded up to 4
  int64_t macs{0};                    // multiply-accumulates per instance (statistics)
};
// rowsOfCell[i] = {first row, row count, device column} of Jacobian cell i; needs layoutDeviceColumns() first.
std::string buildGramPlan(const CholSchedule& s, const std::vector<int32_t>& cellRow0, const std::vector<int32_t>& cellRows, const std::vector<int32_t>& cellCol,
                          int numRows, GramPlan& out);

// The Gram tables as one int32 blob; offsets[8] = {tileOrder, tileQuadStart, quad, (unused), colStripStart, colStrip, stripRow, tileInfo}
// (stripRow[s] = first row of strip s; tileInfo[t] = validI | validJ << 8 | diag << 16 of the schedule).
void makeGramBlob(const GramPlan& g, const CholSchedule& s, std::vector<int32_t>& blob, int32_t offsets[8]);

struct CholSchedDev;
// Concatenates every table into one int32 blob; `dev` gets pointers into blob.data() (rebase them after uploading).
void makeScheduleBlob(const CholSchedule& s, std::vector<int32_t>& blob, CholSchedDev& dev);

} // namespace mb2
