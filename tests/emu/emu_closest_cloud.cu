// TEST HARNESS ONLY — CPU lane-emulation of the point-cloud closest-point kernels (mb2_closest_points_device), part of
// tests/emu/libmb2_emu.so.
//
// The build runs the kernels' steps with the __host__ __device__ blocks of ik_device.cuh: the bounds over the finite points, mortonCode,
// the segmented LSD radix sort of (code, index) with the device's tiles (kSortTile points, per-tile digit counts, the exclusive scan over
// the tiles, a stable scatter), the gather, and the boxes of the implicit tree (leaves of kLeafPoints sorted points, padded to a power of
// two) from the leaves up with boxGrow / boxUnion. Per query the depth-first traversal of closestCloudKernel uses boxVoid /
// boxLowerBound / pruneBox / pointDistance2 / normalCompatible / closerFace. A linear scan over the targets in ascending order with the
// same blocks is the definition the traversal must equal bit for bit. Three deliberately wrong variants (a prune on >=, a leaf that
// skips its last point, a strict > normal test) let the tests show that their checks catch them. It is not part of the product
// library and nothing in momentum_b200/ loads it.
#include <algorithm>
#include <climits>
#include <cstdint>
#include <vector>

#include "../../include/momentum_b200.h"
#include "../../momentum_b200/csrc/ik_device.cuh"
#include "emu_error.h"

using namespace mb2;

namespace {
enum Mode { kTraverse = 0, kScan = 1, kPruneOnEqual = 2, kDropLastLeafPoint = 3, kStrictNormal = 4 };

struct Tree {
  int M{0}, P{1};
  std::vector<uint32_t> codes;    // [M] by original index
  std::vector<int32_t> index;     // [M] original index of each sorted point
  std::vector<float> sorted, sortedNormals, boxes;
};

// cloudBoundsKernel + cloudBoundsReduceKernel: min / max is exact, so one pass over the finite points gives the same box
void bounds(const float* x, int M, float* box) {
  boxEmpty(box);
  for (int m = 0; m < M; ++m) {
    const F3 p = ld3(x + 3 * size_t(m));
    if (finite3(p)) boxGrow(box, p);
  }
}

// the kSortPasses passes of cloudSortCountKernel / cloudSortScanKernel / cloudSortScatterKernel
void radixSort(std::vector<uint32_t>& keys, std::vector<int32_t>& index) {
  const int M = int(keys.size()), tiles = (M + kSortTile - 1) / kSortTile, D = 1 << kSortBits;
  std::vector<uint32_t> k2(M);
  std::vector<int32_t> i2(M);
  std::vector<int32_t> scan(size_t(tiles) * D), start(D);
  for (int pass = 0; pass < kSortPasses; ++pass) {
    const int shift = pass * kSortBits;
    std::fill(scan.begin(), scan.end(), 0);
    for (int e = 0; e < M; ++e) ++scan[size_t(e / kSortTile) * D + ((keys[e] >> shift) & (D - 1))];
    std::vector<int32_t> total(D, 0);
    for (int d = 0; d < D; ++d)
      for (int t = 0; t < tiles; ++t) {
        const int c = scan[size_t(t) * D + d];
        scan[size_t(t) * D + d] = total[d];
        total[d] += c;
      }
    for (int d = 0, s = 0; d < D; ++d) { start[d] = s; s += total[d]; }
    for (int t = 0; t < tiles; ++t) {
      std::vector<int32_t> rank(D, 0);
      for (int e = t * kSortTile; e < std::min(M, (t + 1) * kSortTile); ++e) { // point order within the tile: stable
        const int d = int((keys[e] >> shift) & (D - 1));
        const size_t o = size_t(start[d] + scan[size_t(t) * D + d] + rank[d]++);
        k2[o] = keys[e];
        i2[o] = index[e];
      }
    }
    keys.swap(k2);
    index.swap(i2);
  }
}

Tree build(const float* x, const float* xn, int M) {
  Tree t;
  t.M = M;
  t.P = cloudPadded(M);
  float b[6];
  bounds(x, M, b);
  t.codes.resize(M);
  std::vector<int32_t> idx(M);
  for (int m = 0; m < M; ++m) { t.codes[m] = mortonCode(ld3(x + 3 * size_t(m)), b); idx[m] = m; }
  std::vector<uint32_t> keys = t.codes;
  radixSort(keys, idx);
  t.index = idx;
  t.sorted.resize(size_t(M) * 3);
  if (xn) t.sortedNormals.resize(size_t(M) * 3);
  for (int m = 0; m < M; ++m)
    for (int k = 0; k < 3; ++k) {
      t.sorted[3 * size_t(m) + k] = x[3 * size_t(idx[m]) + k];
      if (xn) t.sortedNormals[3 * size_t(m) + k] = xn[3 * size_t(idx[m]) + k];
    }
  // cloudBoxKernel: the leaves, then each level from the one below
  t.boxes.resize((2 * size_t(t.P) - 1) * 6);
  for (int l = 0; l < t.P; ++l) {
    float* box = t.boxes.data() + (size_t(t.P) - 1 + l) * 6;
    boxEmpty(box);
    for (int m = l * kLeafPoints; m < std::min(M, (l + 1) * kLeafPoints); ++m) boxGrow(box, ld3(t.sorted.data() + 3 * size_t(m)));
  }
  for (int n = t.P - 2; n >= 0; --n) boxUnion(t.boxes.data() + size_t(n) * 6, t.boxes.data() + size_t(2 * n + 1) * 6, t.boxes.data() + size_t(2 * n + 2) * 6);
  return t;
}

struct Query {
  F3 p, np;
  bool normals;
  float maxNormalDot;
  int mode;
};

bool compatible(const Query& q, F3 nt) {
  if (!q.normals) return true;
  if (q.mode == kStrictNormal) return fmaf(q.np.x, nt.x, fmaf(q.np.y, nt.y, q.np.z * nt.z)) > q.maxNormalDot;
  return normalCompatible(q.np, nt, q.maxNormalDot);
}

void tryPoint(const Query& q, F3 t, F3 nt, int j, float& best, int& bestIndex) {
  const float d2 = pointDistance2(q.p, t);
  if (closerFace(d2, j, best, bestIndex) && compatible(q, nt)) { best = d2; bestIndex = j; }
}

bool prune(float lb, float best, int mode) { return mode == kPruneOnEqual ? lb >= best : pruneBox(lb, best); }

// closestCloudKernel's loop for one query
void traverse(const Tree& t, const Query& q, float& best, int& bestIndex) {
  const float* bx = t.boxes.data();
  int stackNode[kTreeStack];
  float stackLb[kTreeStack];
  int sp = 0, node = 0;
  bool go = finite3(q.p) && !boxVoid(bx) && !prune(boxLowerBound(bx, q.p), best, q.mode);
  while (go) {
    if (node < t.P - 1) {
      const int c0 = 2 * node + 1;
      const float* b0 = bx + size_t(c0) * 6;
      const float lb0 = boxLowerBound(b0, q.p), lb1 = boxLowerBound(b0 + 6, q.p);
      const bool in0 = !boxVoid(b0) && !prune(lb0, best, q.mode), in1 = !boxVoid(b0 + 6) && !prune(lb1, best, q.mode);
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
      const int m0 = (node - (t.P - 1)) * kLeafPoints;
      int m1 = std::min(t.M, m0 + kLeafPoints);
      if (q.mode == kDropLastLeafPoint) m1 = std::max(m0, m1 - 1);
      for (int m = m0; m < m1; ++m)
        tryPoint(q, ld3(t.sorted.data() + 3 * size_t(m)), q.normals ? ld3(t.sortedNormals.data() + 3 * size_t(m)) : f3(0.f, 0.f, 0.f),
                 t.index[m], best, bestIndex);
    }
    go = false;
    while (sp > 0) {
      --sp;
      if (!prune(stackLb[sp], best, q.mode)) {
        node = stackNode[sp];
        go = true;
        break;
      }
    }
  }
}
} // namespace

// The emulated build over points [M][3]: codes [M] (by original index), perm [M] (the original index of each sorted point), boxes
// [2P - 1][6] of the implicit tree, sizes [2] = (P, number of real leaves).
extern "C" int emu_cloud_tree(int32_t M, const float* points, uint32_t* codes, int32_t* perm, float* boxes, int32_t* sizes) {
  if (M < 0) { g_emuErr = "cloud tree: M must not be negative"; return MB2_ERR_INVALID_ARGUMENT; }
  const Tree t = build(points, nullptr, M);
  std::copy(t.codes.begin(), t.codes.end(), codes);
  std::copy(t.index.begin(), t.index.end(), perm);
  std::copy(t.boxes.begin(), t.boxes.end(), boxes);
  sizes[0] = t.P;
  sizes[1] = cloudLeaves(M);
  return MB2_OK;
}

// mb2_closest_points_device on host arrays: source [B][N][3], target [B or 1][M][3], the normals null or both set. mode: 0 the kernels'
// traversal, 1 the linear scan, 2 / 3 / 4 the wrong variants.
extern "C" int emu_closest_cloud(int32_t B, int32_t N, int32_t M, int32_t targetBatched, const float* source, const float* sourceNormals,
                                 const float* target, const float* targetNormals, float maxDist, float maxNormalDot, int32_t mode,
                                 float* outPoints, float* outNormals, int32_t* outIndex) {
  if (B < 0 || N < 0 || M < 0) { g_emuErr = "closest points on cloud: negative size"; return MB2_ERR_INVALID_ARGUMENT; }
  if ((sourceNormals == nullptr) != (targetNormals == nullptr) || (sourceNormals == nullptr) != (outNormals == nullptr)) {
    g_emuErr = "closest points on cloud: mismatched normals";
    return MB2_ERR_INVALID_ARGUMENT;
  }
  const bool normals = sourceNormals != nullptr;
  Tree t;
  for (int b = 0; b < B; ++b) {
    const size_t tb = targetBatched ? size_t(b) : 0;
    const float* x = target + tb * M * 3;
    const float* xn = normals ? targetNormals + tb * M * 3 : nullptr;
    if (mode != kScan && (b == 0 || targetBatched)) t = build(x, xn, M);
    for (int n = 0; n < N; ++n) {
      const size_t qi = size_t(b) * N + n;
      Query q{ld3(source + 3 * qi), normals ? ld3(sourceNormals + 3 * qi) : f3(0.f, 0.f, 0.f), normals, maxNormalDot, mode};
      float best = maxDist * maxDist;
      int bestIndex = INT_MAX;
      if (mode == kScan) {
        for (int j = 0; j < M; ++j) tryPoint(q, ld3(x + 3 * size_t(j)), normals ? ld3(xn + 3 * size_t(j)) : f3(0.f, 0.f, 0.f), j, best, bestIndex);
      } else if (M > 0) {
        traverse(t, q, best, bestIndex);
      }
      const bool found = bestIndex != INT_MAX;
      for (int k = 0; k < 3; ++k) {
        outPoints[3 * qi + k] = found ? x[3 * size_t(bestIndex) + k] : 0.f;
        if (normals) outNormals[3 * qi + k] = found ? xn[3 * size_t(bestIndex) + k] : 0.f;
      }
      outIndex[qi] = found ? bestIndex : -1;
    }
  }
  return MB2_OK;
}
