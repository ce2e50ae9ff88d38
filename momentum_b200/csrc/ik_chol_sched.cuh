// Device building blocks of the level-scheduled tile-sparse Cholesky (see ik_chol_sched.h).
//
// Storage: every structurally non-zero lower tile (I,J), I >= J, is a 16x16 fp32 block in shared memory holding X(r, c) =
// H(16 I + r, 16 J + c), later L(I,J), in the mma.sync fragment layout (see tileIdx below): products read and write tiles as the
// lanes' own fragments (two LDS.128 / STS.128), nothing is stored transposed.
//
// Diagonal tiles and the substitutions are mapped to half-warps (one 16-row tile each, width-16 shuffles); the 16x16x16
// products (panel tiles, update tasks, the Gram kernel) are one warp each on mma.sync with the three-term TF32 split.
// The host build (tests/emu) runs the same arithmetic lane by lane so that the schedule and the tile algebra are
// validated without a GPU.
#pragma once

#include <cmath>
#include <cstring>

#include "ik_types.h"

#include <vector_types.h> // float2 / float4 (CUDA toolkit header, usable from plain C++ too)

namespace mb2 {

struct CholSchedDev {
  int32_t n, nPad, numTileCols, numTiles, numLevels;
  // every table below lives in one contiguous int32 blob (copied to shared memory by the kernels)
  const int32_t* blob;
  int32_t blobInts;
  const int32_t* perm;        // [nPad] slot -> device column, -1 = padding
  const int32_t* pos;         // [n] device column -> slot (monotone: device columns are in elimination order)
  const int32_t* tileIdTable; // [numTileCols^2]
  const int32_t* tileRow;
  const int32_t* tileCol;
  const int32_t* diagTile;
  const int32_t* levelColStart;
  const int32_t* levelCols;
  const int32_t* levelPanelStart;
  const int32_t* panelTile;
  const int32_t* panelDiag;
  const int32_t* levelTaskStart;
  const int32_t* taskDst;
  const int32_t* taskPairStart;
  const int32_t* pairA;
  const int32_t* pairB;
  const int32_t* levelVTaskStart;
  const int32_t* vtaskRow;
  const int32_t* vtaskSrcStart;
  const int32_t* vsrcTile;
  const int32_t* vsrcCol;
  const int32_t* colPanelStart;
  const int32_t* colPanelTile;
  const int32_t* colPanelRow;
  const int32_t* levelOrderStart8;  // update-task assignment for 8 warps per instance: [numLevels + 1] into taskOrder8 ([rounds][8], -1 = idle)
  const int32_t* taskOrder8;
  const int32_t* levelOrderStart16; // ... for the 16-warp CTA of wide systems
  const int32_t* taskOrder16;
  const int32_t* tileInfo;    // [numTiles][3] {gi0, gj0, validI | validJ << 8 | diag << 16}, see ik_chol_sched.h
};
// view of the same schedule with every table pointer moved to a copy of the blob at `newBlob`
// Every pointer is re-derived FROM newBlob (newBlob + element offset): nvcc assumes kernel-parameter pointers address
// global memory, so "old pointer + delta" would still be loaded with ld.global even when the copy lives in shared memory.
MB2_HD CholSchedDev rebaseSchedule(const CholSchedDev& S, const int32_t* newBlob) {
  CholSchedDev R = S;
  const int32_t* o = S.blob;
  R.blob = newBlob;
#define MB2_RB(f) R.f = newBlob + (S.f - o);
  MB2_RB(perm) MB2_RB(pos) MB2_RB(tileIdTable) MB2_RB(tileRow) MB2_RB(tileCol) MB2_RB(diagTile) MB2_RB(levelColStart) MB2_RB(levelCols)
  MB2_RB(levelPanelStart) MB2_RB(panelTile) MB2_RB(panelDiag) MB2_RB(levelTaskStart) MB2_RB(taskDst) MB2_RB(taskPairStart) MB2_RB(pairA) MB2_RB(pairB)
  MB2_RB(levelVTaskStart) MB2_RB(vtaskRow) MB2_RB(vtaskSrcStart) MB2_RB(vsrcTile) MB2_RB(vsrcCol) MB2_RB(colPanelStart) MB2_RB(colPanelTile)
  MB2_RB(colPanelRow) MB2_RB(levelOrderStart8) MB2_RB(taskOrder8) MB2_RB(levelOrderStart16) MB2_RB(taskOrder16) MB2_RB(tileInfo)
#undef MB2_RB
  return R;
}

// Tile storage = the mma.sync FRAGMENT layout. Lane (g, t) = (lane >> 2, lane & 3) of a warp owns the eight elements
//   rows g, g + 8  x  columns 2t, 2t + 1 (first float4) and 8 + 2t, 9 + 2t (second float4)
// of a logical 16x16 tile X(r, c) -- exactly the C/D fragment of mma.m16n8k8 over two column halves. With the k index of a product
// permuted consistently (slot t <-> column 2t, slot t + 4 <-> column 2t + 1 of each column half) the SAME eight registers are the A
// fragment of X as a left operand (rows of X) and the B fragment of X as a right operand of  out(r, c) = sum_k A(r, k) B(c, k).  So
//   * every product in the factorisation (panel = A W^T, update = L L^T, the Gram tiles) reads an operand tile as two conflict-free
//     LDS.128 with one address register, and writes / updates its destination tile in place from its own accumulators;
//   * no tile is ever stored transposed: tile (I,J), I >= J, holds X(r, c) = H(16 I + r, 16 J + c) and later L(I,J).
// The float4 of lane l sits in slot l ^ (l >> 3) of its column half (a permutation inside each quarter-warp: LDS.128 stays
// conflict-free), which also makes the two scalar access shapes of the half-warp phases conflict-free: "lane r reads X(r, c)" for a
// fixed c (column access) and "lane r reads the pair X(r, 2j), X(r, 2j + 1)" (row access, 8-byte).
MB2_HD int tileSlotOffset(int lane) { return (lane ^ (lane >> 3)) << 2; } // float offset of the lane's float4 inside a column half
MB2_HD int tileIdx(int r, int c) {
  const int lane = ((r & 7) << 2) | ((c & 7) >> 1);
  return ((c >> 3) << 7) + ((lane ^ (lane >> 3)) << 2) + (((r >> 3) << 1) | (c & 1));
}
// the lane's element e (0..3) of column half h: row / column inside the tile
MB2_HD int fragRow(int lane, int e) { return (lane >> 2) + 8 * (e >> 1); }
MB2_HD int fragCol(int lane, int h, int e) { return 8 * h + 2 * (lane & 3) + (e & 1); }
MB2_HD void tileLoadFrag(const float* tile, int lane, float d[2][4]) {
  const int so = tileSlotOffset(lane);
#if defined(__CUDA_ARCH__)
  const float4 v0 = *reinterpret_cast<const float4*>(tile + so), v1 = *reinterpret_cast<const float4*>(tile + 128 + so);
  d[0][0] = v0.x; d[0][1] = v0.y; d[0][2] = v0.z; d[0][3] = v0.w; d[1][0] = v1.x; d[1][1] = v1.y; d[1][2] = v1.z; d[1][3] = v1.w;
#else
  for (int h = 0; h < 2; ++h) for (int e = 0; e < 4; ++e) d[h][e] = tile[128 * h + so + e];
#endif
}
MB2_HD void tileStoreFrag(float* tile, int lane, const float d[2][4]) {
  const int so = tileSlotOffset(lane);
#if defined(__CUDA_ARCH__)
  *reinterpret_cast<float4*>(tile + so) = make_float4(d[0][0], d[0][1], d[0][2], d[0][3]);
  *reinterpret_cast<float4*>(tile + 128 + so) = make_float4(d[1][0], d[1][1], d[1][2], d[1][3]);
#else
  for (int h = 0; h < 2; ++h) for (int e = 0; e < 4; ++e) tile[128 * h + so + e] = d[h][e];
#endif
}

// What a 16x16 box of H becomes as a tile: rows >= validI / columns >= validJ of the box belong to the NEXT parameters of the elimination
// order (padding only closes a tile): they are replaced by the identity extension (info = validI | validJ << 8 | diag << 16).
MB2_HD float cholPadElement(float v, int info, int r, int c) {
  const int vI = info & 0xFF, vJ = (info >> 8) & 0xFF, diag = (info >> 16) & 1;
  if (r < vI && c < vJ) return v;
  return (diag && r == c) ? 1.f : 0.f;
}
// K-major path: the TMA box of the row-major upper triangle of H lands as S[c][r] = H(gj0 + c, gi0 + r) in 64-byte rows with the
// SWIZZLE_64B pattern; one warp turns it into the fragment layout in place (every lane reads its eight elements, then all write).
MB2_HD int tmaBoxIdx(int c, int r) { return c * 16 + ((((r >> 2) ^ ((c >> 1) & 3)) << 2) | (r & 3)); }
MB2_HD void cholConvertBox(float* tile, int info, int lane) { // device only (a warp in lock step)
  float v[2][4];
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int r = fragRow(lane, e), c = fragCol(lane, h, e);
      // only the upper triangle of H is guaranteed: a diagonal box is mirrored from its row <= column half
      const bool mirror = ((info >> 16) & 1) != 0 && c > r;
      v[h][e] = cholPadElement(tile[mirror ? tmaBoxIdx(r, c) : tmaBoxIdx(c, r)], info, r, c);
    }
#if defined(__CUDA_ARCH__)
  __syncwarp();
#endif
  tileStoreFrag(tile, lane, v);
}

// ---- tile-sparse Gram (see GramPlan in ik_chol_sched.h): a warp owns one tile and accumulates it on the tensor cores ----
// strips: [strip][16 columns][4 rows] floats, so S[c][k] of a strip is float 4 c + k. Two pairs at a time form the
// 16 x 16 x 8 product out(r, c) += sum_k A[r][k] B[c][k] (k 0..3 from the first pair, 4..7 from the second; lists are padded
// to even length with an all-zero strip) = two mma.sync.m16n8k8 (column halves) per term of the three-term TF32 split
// hi*hi + hi*lo + lo*hi with fp32 accumulation (fp32-class accuracy). hi = nearest tf32 of x, lo = x - hi (exact; the tensor
// core reads its leading 10 mantissa bits: a 2^-22 relative perturbation). Every fragment is one conflict-free 128-byte warp read:
//   a0 = A[g][t], a1 = A[g + 8][t], b(h) = B[8 h + g][t]   with g = lane >> 2, t = lane & 3  ->  float index lane (+ 32).
// Accumulators d[h][0..3] follow the mma C layout: (row g, cols 8h + 2t, 8h + 2t + 1), (row g + 8, same cols) = the tile's fragment layout.
MB2_HD float tf32High(float x) { // nearest tf32 (ties away from zero), 10 mantissa bits: what cvt.rna.tf32.f32 returns for finite x, but on
                                  // the integer ALU (the conversion instruction runs on the quarter-rate XU pipe)
#if defined(__CUDA_ARCH__)
  return __uint_as_float((__float_as_uint(x) + 0x1000u) & 0xFFFFE000u);
#else
  uint32_t u;
  std::memcpy(&u, &x, 4);
  u = (u + 0x1000u) & 0xFFFFE000u;
  float r;
  std::memcpy(&r, &u, 4);
  return r;
#endif
}
#if defined(__CUDA_ARCH__)
__device__ __forceinline__ void mmaTf32K8(float d[4], float a0, float a1, float a2, float a3, float b0, float b1) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(__float_as_uint(a0)), "r"(__float_as_uint(a1)), "r"(__float_as_uint(a2)), "r"(__float_as_uint(a3)), "r"(__float_as_uint(b0)),
                 "r"(__float_as_uint(b1)));
}
// One k = 8 step of out += A B^T on the tensor cores with the three-term TF32 split: a0..a3 / b[h][0..1] are the raw fp32 fragment
// values of mma.m16n8k8 (A: rows g, g + 8 x k slots t, t + 4; B: n = 8 h + g).
//   d[h]     += hi*hi          -- added in fp32 registers (round to nearest) after EVERY step: the tensor core's own accumulator truncates;
//                                 letting it carry the leading term over just two steps moved converged cfg2 / cfg4 parameters past 1e-4
//   small[h] += lo*hi + hi*lo  -- inside the tensor core for the whole sum (2^-11 of the result: their truncation does not matter)
__device__ __forceinline__ void mma3xTf32Step(float d[2][4], float small[2][4], float a0, float a1, float a2, float a3, float b00, float b01, float b10, float b11) {
  const float a0h = tf32High(a0), a1h = tf32High(a1), a2h = tf32High(a2), a3h = tf32High(a3);
  const float b00h = tf32High(b00), b01h = tf32High(b01), b10h = tf32High(b10), b11h = tf32High(b11);
  const float a0l = a0 - a0h, a1l = a1 - a1h, a2l = a2 - a2h, a3l = a3 - a3h; // (the tensor core reads the leading bits of lo)
  const float b00l = b00 - b00h, b01l = b01 - b01h, b10l = b10 - b10h, b11l = b11 - b11h;
  mmaTf32K8(small[0], a0l, a1l, a2l, a3l, b00h, b01h); mmaTf32K8(small[1], a0l, a1l, a2l, a3l, b10h, b11h);
  mmaTf32K8(small[0], a0h, a1h, a2h, a3h, b00l, b01l); mmaTf32K8(small[1], a0h, a1h, a2h, a3h, b10l, b11l);
  float t0[4] = {0.f, 0.f, 0.f, 0.f}, t1[4] = {0.f, 0.f, 0.f, 0.f};
  mmaTf32K8(t0, a0h, a1h, a2h, a3h, b00h, b01h); mmaTf32K8(t1, a0h, a1h, a2h, a3h, b10h, b11h);
#pragma unroll
  for (int e = 0; e < 4; ++e) { d[0][e] += t0[e]; d[1][e] += t1[e]; }
}
#endif
// host emulation of the same step for one output: sum over the step's eight k of the split products
MB2_HD void mma3xEmulate(float& d, float& small, const float av[8], const float bv[8]) {
  float lo = 0.f, mid = 0.f, hi = 0.f;
  for (int k = 0; k < 8; ++k) {
    const float ah = tf32High(av[k]), bh = tf32High(bv[k]), al = av[k] - ah, bl = bv[k] - bh;
    lo += al * bh; mid += ah * bl; hi += ah * bh;
  }
  small += lo + mid;
  d += hi;
}

// one step = the four strips {A0, B0, A1, B1} (float offsets) of two pairs
MB2_HD void gramTilePairs(const float* strips, int oa0, int ob0, int oa1, int ob1, int lane, float d[2][4], float small[2][4]) {
  const float* A0 = strips + oa0;
  const float* B0 = strips + ob0;
  const float* A1 = strips + oa1;
  const float* B1 = strips + ob1;
#if defined(__CUDA_ARCH__)
  mma3xTf32Step(d, small, A0[lane], A0[32 + lane], A1[lane], A1[32 + lane], B0[lane], B1[lane], B0[32 + lane], B1[32 + lane]); // b[h][k half]
#else
  for (int h = 0; h < 2; ++h) // host emulation: the lane's eight outputs from the same three-term split
    for (int e = 0; e < 4; ++e) {
      const int r = fragRow(lane, e), c = fragCol(lane, h, e);
      float av[8], bv[8];
      for (int k = 0; k < 8; ++k) { av[k] = k < 4 ? A0[4 * r + k] : A1[4 * r + k - 4]; bv[k] = k < 4 ? B0[4 * c + k] : B1[4 * c + k - 4]; }
      mma3xEmulate(d[h][e], small[h][e], av, bv);
    }
#endif
}
// Four consecutive table entries (16-byte aligned int32 or 8-byte aligned uint16 records) as ONE warp-uniform read
MB2_HD int4 tableRecord4(const int32_t* p) {
#if defined(__CUDA_ARCH__)
  return *reinterpret_cast<const int4*>(p);
#else
  int4 r; r.x = p[0]; r.y = p[1]; r.z = p[2]; r.w = p[3];
  return r;
#endif
}
MB2_HD int4 tableRecord4(const uint16_t* p) {
  int4 r;
#if defined(__CUDA_ARCH__)
  const uint2 v = *reinterpret_cast<const uint2*>(p);
  r.x = int(v.x & 0xFFFFu); r.y = int(v.x >> 16); r.z = int(v.y & 0xFFFFu); r.w = int(v.y >> 16);
#else
  r.x = p[0]; r.y = p[1]; r.z = p[2]; r.w = p[3];
#endif
  return r;
}
MB2_HD int2 tableRecord2(const uint16_t* p) {
  int2 r;
#if defined(__CUDA_ARCH__)
  const uint32_t v = *reinterpret_cast<const uint32_t*>(p);
  r.x = int(v & 0xFFFFu); r.y = int(v >> 16);
#else
  r.x = p[0]; r.y = p[1];
#endif
  return r;
}
// quads: {A0, B0, A1, B1} float offsets per step (GramPlan::quad, pair lists padded to even length): the int32 blob staged in shared
// memory, or the 16-bit copy of gramCholeskyKernel's parameter block
template <class Q>
MB2_HD void gramTileAccumulate(const float* strips, const Q* quads, int q0, int q1, int lane, float d[2][4]) {
  float small[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
  for (int q = q0; q < q1; ++q) {
    const int4 o = tableRecord4(quads + 4 * q); // one broadcast read
    gramTilePairs(strips, o.x, o.y, o.z, o.w, lane, d, small);
  }
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int e = 0; e < 4; ++e) d[h][e] += small[h][e];
}
// writes the lane's accumulators (its fragment of the tile) with the identity extension on padded rows/columns and the damping added
// to the real diagonal (info = validI | validJ << 8 | diag << 16 as in tileInfo); full off-diagonal tiles take the plain path
MB2_HD void gramTileStore(float* tile, const float d[2][4], int info, float lambda, int lane) {
  const int vI = info & 0xFF, vJ = (info >> 8) & 0xFF, diag = (info >> 16) & 1;
  if (vI == 16 && vJ == 16 && !diag) { tileStoreFrag(tile, lane, d); return; }
  float v[2][4];
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int r = fragRow(lane, e), c = fragCol(lane, h, e);
      v[h][e] = cholPadElement((diag && r == c) ? d[h][e] + lambda : d[h][e], info, r, c);
    }
  tileStoreFrag(tile, lane, v);
}
// entry hl of block K of J^T r: sum over the strips of tile column K of strip[hl][0..3] . r[4q..4q+3]
MB2_HD void gramVectorTerm(const float* strip, const float* r4, int hl, float& g0, float& g1) {
  const float4 sv = *reinterpret_cast<const float4*>(strip + 4 * hl);
  const float4 rv = *reinterpret_cast<const float4*>(r4);
  g0 += sv.x * rv.x + sv.y * rv.y;
  g1 += sv.z * rv.z + sv.w * rv.w;
}
MB2_HD float gramVectorEntry(const float* strips, const float* resid, const int32_t* colStrip, const int32_t* stripRow, int s0, int s1, int hl) {
  float g0 = 0.f, g1 = 0.f;
  for (int k = s0; k < s1; ++k) {
    const int sidx = colStrip[k];
    gramVectorTerm(strips + size_t(sidx) * 64, resid + stripRow[sidx], hl, g0, g1);
  }
  return g0 + g1;
}
// the same sum over pre-resolved {strip float offset, first row} records (GramCholTables::colEnt)
MB2_HD float gramVectorEntry(const float* strips, const float* resid, const uint16_t* colEnt, int s0, int s1, int hl) {
  float g0 = 0.f, g1 = 0.f;
  for (int k = s0; k < s1; ++k) {
    const int2 e = tableRecord2(colEnt + 2 * k);
    gramVectorTerm(strips + e.x, resid + e.y, hl, g0, g1);
  }
  return g0 + g1;
}

// row r of a tile: 8-byte pieces (conflict-free when lane r of a half-warp handles row r)
MB2_HD void tileLoadRow(const float* tile, int r, float* a) {
#pragma unroll
  for (int j = 0; j < 16; j += 2) {
    const float2 v = *reinterpret_cast<const float2*>(tile + tileIdx(r, j));
    a[j] = v.x; a[j + 1] = v.y;
  }
}
MB2_HD void tileStoreRow(float* tile, int r, const float* a) {
#pragma unroll
  for (int j = 0; j < 16; j += 2) {
    float2 v;
    v.x = a[j]; v.y = a[j + 1];
    *reinterpret_cast<float2*>(tile + tileIdx(r, j)) = v;
  }
}

// ---- phase A: Cholesky of a diagonal tile, forward solve of its 16 right-hand-side entries, and W = L^-1; ONE WARP per tile ----
// A non-positive pivot is replaced by `fallback` (the damping) and reported through *fail.
// On return the tile holds W = L(K,K)^-1 (lower triangular, zeros above the diagonal): every later use of the diagonal
// block (panel solve, backward substitution) is then a 16x16 product with W — no dependent 16-step chain on the
// critical path of a level. L(K,K) itself is not needed again.
//
// Square-root-free elimination keeps the per-step dependency chain short (pivot broadcast -> reciprocal -> one multiply ->
// one fused multiply-add); the 1/sqrt(pivot) scalings and the right-hand side ride along off that chain:
//   A = U D U^T (U unit lower, U[r][k] = a_r[k] / d_k),  L = U D^1/2,  y = L^-1 g = D^-1/2 U^-1 g.
// W = L^-1 = D^-1/2 U^-1 comes out of the SAME sixteen steps (Gauss-Jordan on [A | I]): row_r -= U[r][k] row_k for r > k leaves E = U^-1.
// Lanes 0..15 hold ROW hl of A, lanes 16..31 hold COLUMN hl of E. With c_j = A[j][k] (lane j's element k) broadcast once, both halves
// execute the same instruction:   v[j] -= (v[k] / d_k) * c_j  for j > k
//   row hl of A:     a[j] -= U[hl][k] * A[k][j]             (A[k][j] = A[j][k] = c_j: the trailing block stays symmetric)
//   column hl of E:  E[j][hl] -= U[j][k] * E[k][hl] = c_j * (E[k][hl] / d_k)
// so a step costs one column broadcast and 15 - k FMAs for the whole tile: a warp is limited by its own issue rate, and a half-warp per
// tile with separate a / e loops and 33 shuffles per step would issue several times the instructions.
// The tile is symmetric (the Gram / update products compute both triangles; K-major boxes are mirrored by cholConvertBox) and only
// entries A[r][c], c <= r, are ever consumed.
MB2_HD void cholDiagTile(float* tile, float* y16, int lane, float fallback, int* fail) {
#if defined(__CUDA_ARCH__)
  const int hl = lane & 15;
  const bool isE = lane >= 16;
  float v[16];
#pragma unroll
  for (int k = 0; k < 16; ++k) v[k] = isE ? (k == hl ? 1.f : 0.f) : tile[tileIdx(k, hl)];
  float z = isE ? 0.f : y16[hl], rdSelf = 0.f;
  // Column k of A (c_j = lane j's element k) reaches every lane through shared memory: the row lanes store their element k with ONE
  // instruction and everyone reads the column back as broadcast LDS.128 instead of a chain of (17 - k) dependent shuffles per step.
  // The tile's own storage is the buffer (its contents live in registers until W is written at the end): two blocks of [16 column entries | 16 right-hand-side entries], alternating by step parity so that one
  // __syncwarp per step orders everything.
  __syncwarp(); // every lane has read its column before the buffer blocks are written
#pragma unroll
  for (int k = 0; k < 16; ++k) {
    float* blk = tile + 32 * (k & 1);
    if (!isE) { blk[hl] = v[k]; blk[16 + hl] = z; }
    __syncwarp();
    float c[16];
#pragma unroll
    for (int g4 = (k >> 2); g4 < 4; ++g4) {
      const float4 q = *reinterpret_cast<const float4*>(blk + 4 * g4);
      c[4 * g4] = q.x; c[4 * g4 + 1] = q.y; c[4 * g4 + 2] = q.z; c[4 * g4 + 3] = q.w;
    }
    float piv = c[k];
    const float zk = blk[16 + k];
    if (!(piv > 0.f)) { piv = fallback; if (lane == k) *fail = 1; }
    float inv;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(inv) : "f"(piv)); // one MUFU on the dependency chain (1 ulp; the step is damped Gauss-Newton)
    const float rdk = rsqrtf(piv);
    if (lane == k) rdSelf = rdk;
    const float m = v[k] * inv;                      // U[hl][k] (rows) / E[k][hl] / d_k (columns)
    const float tm = (!isE && hl > k) ? m : 0.f;     // rows <= k of the right-hand side are finished
#pragma unroll
    for (int j = k + 1; j < 16; ++j) v[j] -= m * c[j];
    z -= tm * zk;
    v[k] *= rdk;                                     // row k of W = D^-1/2 U^-1 is final (the row lanes no longer need their element k)
  }
  __syncwarp(); // the last buffer reads are done before W overwrites the blocks
  if (!isE) y16[hl] = z * rdSelf;
  else {
#pragma unroll
    for (int i = 0; i < 16; ++i) tile[tileIdx(i, hl)] = v[i]; // column hl of W (zero above the diagonal)
  }
#else
  if (lane != 0) return; // host emulation: one caller plays the thirty-two lanes in lock step with the same operation order
  float A[16][16], E[16][16], z[16], rd[16]; // A[row lane][k], E[i][column lane]
  for (int l = 0; l < 16; ++l) { for (int k = 0; k < 16; ++k) { A[l][k] = tile[tileIdx(k, l)]; E[k][l] = (k == l) ? 1.f : 0.f; } z[l] = y16[l]; }
  for (int k = 0; k < 16; ++k) {
    float piv = A[k][k];
    if (!(piv > 0.f)) { piv = fallback; *fail = 1; }
    const float inv = 1.f / piv;
    rd[k] = 1.f / sqrtf(piv);
    const float zk = z[k];
    float c[16];
    for (int j = 0; j < 16; ++j) c[j] = A[j][k]; // lane j's element k
    for (int l = 0; l < 16; ++l) { // row lanes
      const float m = c[l] * inv;
      for (int j = k + 1; j < 16; ++j) A[l][j] -= m * c[j];
      if (l > k) z[l] -= m * zk;
    }
    for (int l = 0; l < 16; ++l) { // column lanes
      const float m = E[k][l] * inv;
      for (int j = k + 1; j < 16; ++j) E[j][l] -= m * c[j];
      E[k][l] *= rd[k];
    }
  }
  for (int l = 0; l < 16; ++l) {
    y16[l] = z[l] * rd[l];
    for (int i = 0; i < 16; ++i) tile[tileIdx(i, l)] = E[i][l];
  }
#endif
}

// ---- 16x16x16 tile products on the tensor cores (mma.sync m16n8k8, three-term TF32 split, fp32 accumulate) ----
// d(r, c) += sum_k A(r, k) B(c, k) for two tiles in the fragment layout: four LDS.128, two k = 8 steps (column halves; the k slots of a
// step are that half's columns 2t, 2t + 1), the leading term added to d in fp32 registers after each step.
MB2_HD void tileProduct(const float* TA, const float* TB, int lane, float d[2][4], float small[2][4]) {
#if defined(__CUDA_ARCH__)
  const int so = tileSlotOffset(lane);
  const float4 a0 = *reinterpret_cast<const float4*>(TA + so), a1 = *reinterpret_cast<const float4*>(TA + 128 + so);
  const float4 b0 = *reinterpret_cast<const float4*>(TB + so), b1 = *reinterpret_cast<const float4*>(TB + 128 + so);
  mma3xTf32Step(d, small, a0.x, a0.z, a0.y, a0.w, b0.x, b0.y, b0.z, b0.w);
  mma3xTf32Step(d, small, a1.x, a1.z, a1.y, a1.w, b1.x, b1.y, b1.z, b1.w);
#else
  for (int h = 0; h < 2; ++h)
    for (int e = 0; e < 4; ++e) {
      const int r = fragRow(lane, e), c = fragCol(lane, h, e);
      for (int ks = 0; ks < 2; ++ks) {
        float av[8], bv[8];
        for (int k = 0; k < 8; ++k) { av[k] = TA[tileIdx(r, 8 * ks + k)]; bv[k] = TB[tileIdx(c, 8 * ks + k)]; }
        mma3xEmulate(d[h][e], small[h][e], av, bv);
      }
    }
#endif
}

// ---- phase B: X = A(I,K) L(K,K)^-T = A W^T for one panel tile, a warp per tile; the result replaces A ----
// (every lane reads and writes only its own fragment of the tile: no ordering needed between the product and the store)
MB2_HD void cholPanelProduct(const float* tile, const float* diagW, int lane, float out[2][4]) {
  float small[2][4];
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int e = 0; e < 4; ++e) { out[h][e] = 0.f; small[h][e] = 0.f; }
  tileProduct(tile, diagW, lane, out, small);
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int e = 0; e < 4; ++e) out[h][e] += small[h][e];
}
MB2_HD void cholPanelStore(float* tile, int lane, const float out[2][4]) { tileStoreFrag(tile, lane, out); }

// ---- phase C: one update task, D(I,J) -= sum_K L(I,K) L(J,K)^T; a warp per destination tile ----
// pairs p0 .. p1 - 1 of the task: source tiles pairA[p * stride], pairB[p * stride] (the schedule's two arrays, or the {A, B} records
// of GramCholTables with stride 2); dst = destination tile
template <class I>
MB2_HD void cholUpdateTile(float* tiles, const I* pairA, const I* pairB, int stride, int p0, int p1, int dst, int lane) {
  float d[2][4], small[2][4];
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int e = 0; e < 4; ++e) { d[h][e] = 0.f; small[h][e] = 0.f; }
  for (int p = p0; p < p1; ++p)
    tileProduct(tiles + size_t(pairA[p * stride]) * 256, tiles + size_t(pairB[p * stride]) * 256, lane, d, small);
  float* D = tiles + size_t(dst) * 256;
  float v[2][4];
  tileLoadFrag(D, lane, v);
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int e = 0; e < 4; ++e) v[h][e] -= d[h][e] + small[h][e];
  tileStoreFrag(D, lane, v);
}
MB2_HD void cholUpdateTask(float* tiles, const CholSchedDev& S, int task, int lane) {
  cholUpdateTile(tiles, S.pairA, S.pairB, 1, S.taskPairStart[task], S.taskPairStart[task + 1], S.taskDst[task], lane);
}

// ---- phase C (vector part): y_I -= sum L(I,K) y_K over this level's columns; lane hl = row ----
// sources p0 .. p1 - 1: tile srcTile[p * stride] times block srcCol[p * stride] of y; row = the block of y it updates
template <class I>
MB2_HD void cholVectorRows(const float* tiles, float* y, const I* srcTile, const I* srcCol, int stride, int p0, int p1, int row, int hl) {
  float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f; // four partial sums: the dependent chain is 4 deep instead of 16 per source tile
  for (int p = p0; p < p1; ++p) {
    float t[16];
    tileLoadRow(tiles + size_t(srcTile[p * stride]) * 256, hl, t);
    const float* yk = y + srcCol[p * stride] * 16;
#pragma unroll
    for (int c = 0; c < 16; c += 4) { s0 += t[c] * yk[c]; s1 += t[c + 1] * yk[c + 1]; s2 += t[c + 2] * yk[c + 2]; s3 += t[c + 3] * yk[c + 3]; }
  }
  y[row * 16 + hl] -= (s0 + s1) + (s2 + s3);
}
MB2_HD void cholVectorTask(const float* tiles, float* y, const CholSchedDev& S, int vtask, int hl) {
  cholVectorRows(tiles, y, S.vsrcTile, S.vsrcCol, 1, S.vtaskSrcStart[vtask], S.vtaskSrcStart[vtask + 1], S.vtaskRow[vtask], hl);
}

// ---- backward substitution for one tile column K: y_K <- L(K,K)^-T (y_K - sum_I L(I,K)^T y_I); ONE WARP per column ----
// Both parts are "column sums of a tile against a vector": sum_r X(r, c) v[r]. A lane reads its own fragment of the tile (two
// conflict-free LDS.128: rows g, g + 8 x columns 2t, 2t + 1, 8 + 2t, 9 + 2t), multiplies by v[g], v[g + 8] and keeps four partial
// column sums over all panel tiles of the column; ONE butterfly over the eight lanes that share t finishes them. (A half-warp per
// column with lane c reading X(r, c) scalar by scalar would replay on bank conflicts: a row of the fragment layout is not a
// conflict-free 4-byte access.)
// panels p0 .. p1 - 1 of column K: tile panelTile[p * stride] in block row panelRow[p * stride]; diag = the diagonal tile of K (holds W)
template <class I>
MB2_HD void cholBackwardPanels(const float* tiles, float* y, const I* panelTile, const I* panelRow, int stride, int p0, int p1, int K, int diag, int lane) {
#if defined(__CUDA_ARCH__)
  const int g = lane >> 2, t = lane & 3, so = tileSlotOffset(lane);
  float c0 = 0.f, c1 = 0.f, c2 = 0.f, c3 = 0.f;
  for (int p = p0; p < p1; ++p) {
    const float* T = tiles + size_t(panelTile[p * stride]) * 256;
    const float* yi = y + panelRow[p * stride] * 16;
    const float4 v0 = *reinterpret_cast<const float4*>(T + so), v1 = *reinterpret_cast<const float4*>(T + 128 + so);
    const float ya = yi[g], yb = yi[g + 8];
    c0 = fmaf(v0.x, ya, fmaf(v0.z, yb, c0)); c1 = fmaf(v0.y, ya, fmaf(v0.w, yb, c1));
    c2 = fmaf(v1.x, ya, fmaf(v1.z, yb, c2)); c3 = fmaf(v1.y, ya, fmaf(v1.w, yb, c3));
  }
#pragma unroll
  for (int o = 4; o < 32; o <<= 1) {
    c0 += __shfl_xor_sync(0xffffffffu, c0, o); c1 += __shfl_xor_sync(0xffffffffu, c1, o);
    c2 += __shfl_xor_sync(0xffffffffu, c2, o); c3 += __shfl_xor_sync(0xffffffffu, c3, o);
  }
  float* yk = y + K * 16;
  if (g == 0) { yk[2 * t] -= c0; yk[2 * t + 1] -= c1; yk[8 + 2 * t] -= c2; yk[9 + 2 * t] -= c3; } // s = y_K - sums
  __syncwarp();
  // x_K = W^T s with W = L(K,K)^-1 stored by phase A
  const float* W = tiles + size_t(diag) * 256;
  const float4 w0 = *reinterpret_cast<const float4*>(W + so), w1 = *reinterpret_cast<const float4*>(W + 128 + so);
  const float sa = yk[g], sb = yk[g + 8];
  float x0 = fmaf(w0.x, sa, w0.z * sb), x1 = fmaf(w0.y, sa, w0.w * sb), x2 = fmaf(w1.x, sa, w1.z * sb), x3 = fmaf(w1.y, sa, w1.w * sb);
#pragma unroll
  for (int o = 4; o < 32; o <<= 1) {
    x0 += __shfl_xor_sync(0xffffffffu, x0, o); x1 += __shfl_xor_sync(0xffffffffu, x1, o);
    x2 += __shfl_xor_sync(0xffffffffu, x2, o); x3 += __shfl_xor_sync(0xffffffffu, x3, o);
  }
  __syncwarp(); // every lane has read s before it is overwritten
  if (g == 0) { yk[2 * t] = x0; yk[2 * t + 1] = x1; yk[8 + 2 * t] = x2; yk[9 + 2 * t] = x3; }
#else
  if (lane != 0) return; // host emulation: one caller plays the warp
  float s[16];
  for (int c = 0; c < 16; ++c) s[c] = 0.f;
  for (int p = p0; p < p1; ++p) {
    const float* T = tiles + size_t(panelTile[p * stride]) * 256;
    const float* yi = y + panelRow[p * stride] * 16;
    for (int c = 0; c < 16; ++c) for (int r = 0; r < 16; ++r) s[c] += T[tileIdx(r, c)] * yi[r];
  }
  float* yk = y + K * 16;
  for (int c = 0; c < 16; ++c) s[c] = yk[c] - s[c];
  const float* W = tiles + size_t(diag) * 256;
  for (int c = 0; c < 16; ++c) {
    float x = 0.f;
    for (int r = 0; r < 16; ++r) x += W[tileIdx(r, c)] * s[r];
    yk[c] = x;
  }
#endif
}
MB2_HD void cholBackwardColumn(const float* tiles, float* y, const CholSchedDev& S, int K, int lane) {
  cholBackwardPanels(tiles, y, S.colPanelTile, S.colPanelRow, 1, S.colPanelStart[K], S.colPanelStart[K + 1], K, S.diagTile[K], lane);
}

} // namespace mb2
