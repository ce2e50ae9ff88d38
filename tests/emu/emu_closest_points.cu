// TEST HARNESS ONLY — CPU lane-emulation of the closest-point kernels (mb2_character_closest_points_on_mesh_device), built by
// tests/test_closest_points_on_mesh.py into a temporary directory together with ik_plan.cpp / ik_chol_sched.cpp.
//
// The face tables and the tree are made by the library's own makeMeshFaces / makeMeshTree; the __host__ __device__ building blocks of
// ik_device.cuh then run in the kernels' order: boxGrow / boxUnion level by level from the deepest (meshTreeRefitKernel), and per query
// the depth-first traversal of closestPointKernel with boxLowerBound / pruneBox / faceDistance2 / closerFace. A linear scan over the
// faces in ascending order with the same blocks is the definition the traversal must equal bit for bit. Two deliberately wrong
// traversals (a prune on >=, a leaf that skips its last face) let the tests show that their checks catch them. It is not part of the
// product library and nothing in momentum_b200/ loads it.
#include <algorithm>
#include <climits>
#include <cstdint>
#include <string>
#include <vector>

#include "../../include/momentum_b200.h"
#include "../../momentum_b200/csrc/ik_device.cuh"
#include "../../momentum_b200/csrc/ik_plan.h"

using namespace mb2;

static thread_local std::string g_err;

extern "C" const char* emu_closest_points_last_error(void) { return g_err.c_str(); }

namespace {
enum Mode { kTraverse = 0, kScan = 1, kPruneOnEqual = 2, kDropLastLeafFace = 3 };

int make(int32_t V, int32_t F, const int32_t* faces, const float* ref, HostMeshFaces& m, HostMeshTree& t) {
  g_err = makeMeshFaces(V, F, faces, m);
  if (g_err.empty()) g_err = makeMeshTree(m, V, ref, t);
  return g_err.empty() ? MB2_OK : MB2_ERR_INVALID_ARGUMENT;
}

// meshTreeRefitKernel for one instance: boxes [numNodes][6]
void refit(const HostMeshFaces& m, const HostMeshTree& t, const float* x, float* boxes) {
  for (int L = t.depth - 1; L >= 0; --L)
    for (int n = t.levelStart[L]; n < t.levelStart[L + 1]; ++n) {
      const int start = t.nodeStart[n], count = t.nodeCount[n];
      float box[6];
      if (count == 0) {
        boxUnion(box, boxes + size_t(start) * 6, boxes + size_t(start + 1) * 6);
      } else {
        boxEmpty(box);
        for (int k = 0; k < count; ++k) {
          const int* f = m.faces.data() + size_t(t.leafFaces[start + k]) * 3;
          for (int c = 0; c < 3; ++c) boxGrow(box, ld3(x + 3 * size_t(f[c])));
        }
      }
      std::copy(box, box + 6, boxes + size_t(n) * 6);
    }
}

struct Best {
  float d2;
  int face{INT_MAX};
  F3 q{0.f, 0.f, 0.f}, bary{0.f, 0.f, 0.f};
};

void tryFace(const HostMeshFaces& m, const float* x, F3 p, int f, Best& b) {
  const int* fv = m.faces.data() + size_t(f) * 3;
  F3 q, bary;
  const float d2 = faceDistance2(p, ld3(x + 3 * size_t(fv[0])), ld3(x + 3 * size_t(fv[1])), ld3(x + 3 * size_t(fv[2])), q, bary);
  if (closerFace(d2, f, b.d2, b.face)) { b.d2 = d2; b.face = f; b.q = q; b.bary = bary; }
}

bool prune(float lb, float best, int mode) { return mode == kPruneOnEqual ? lb >= best : pruneBox(lb, best); }

// closestPointKernel's loop for one query; returns the number of nodes visited
int traverse(const HostMeshFaces& m, const HostMeshTree& t, const float* x, const float* boxes, F3 p, int mode, Best& b) {
  int stackNode[kTreeStack];
  float stackLb[kTreeStack];
  int sp = 0, node = 0, visits = 0;
  bool go = finite3(p) && !prune(boxLowerBound(boxes, p), b.d2, mode);
  while (go) {
    ++visits;
    const int start = t.nodeStart[node], count = t.nodeCount[node];
    if (count == 0) {
      const float lb0 = boxLowerBound(boxes + size_t(start) * 6, p), lb1 = boxLowerBound(boxes + size_t(start + 1) * 6, p);
      const bool in0 = !prune(lb0, b.d2, mode), in1 = !prune(lb1, b.d2, mode);
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
      const int n = mode == kDropLastLeafFace ? count - 1 : count;
      for (int k = 0; k < n; ++k) tryFace(m, x, p, t.leafFaces[start + k], b);
    }
    go = false;
    while (sp > 0) {
      --sp;
      if (!prune(stackLb[sp], b.d2, mode)) {
        node = stackNode[sp];
        go = true;
        break;
      }
    }
  }
  return visits;
}
} // namespace

// makeMeshTree alone: its tables (nodeStart / nodeCount [2F], leafFaces [F], levelStart [kTreeStack + 1]) and sizes, or its message
// over Vt reference positions (makeMeshTree checks Vt against the faces' V)
extern "C" int emu_mesh_tree(int32_t V, int32_t F, const int32_t* faces, int32_t Vt, const float* ref, int32_t* sizes, int32_t* nodeStart,
                             int32_t* nodeCount, int32_t* leafFaces, int32_t* levelStart) {
  HostMeshFaces m;
  HostMeshTree t;
  g_err = makeMeshFaces(V, F, faces, m);
  if (g_err.empty()) g_err = makeMeshTree(m, Vt, ref, t);
  if (!g_err.empty()) return MB2_ERR_INVALID_ARGUMENT;
  sizes[0] = t.numNodes;
  sizes[1] = t.depth;
  std::copy(t.nodeStart.begin(), t.nodeStart.end(), nodeStart);
  std::copy(t.nodeCount.begin(), t.nodeCount.end(), nodeCount);
  std::copy(t.leafFaces.begin(), t.leafFaces.end(), leafFaces);
  std::copy(t.levelStart.begin(), t.levelStart.end(), levelStart);
  return MB2_OK;
}

// the refitted boxes [numNodes][6] of positions x [V][3] over the tree built from ref
extern "C" int emu_mesh_tree_boxes(int32_t V, int32_t F, const int32_t* faces, const float* ref, const float* x, float* boxes) {
  HostMeshFaces m;
  HostMeshTree t;
  if (make(V, F, faces, ref, m, t) != MB2_OK) return MB2_ERR_INVALID_ARGUMENT;
  refit(m, t, x, boxes);
  return MB2_OK;
}

// positions [B][V][3], points [B][N][3] -> outPoints [B][N][3], outFace [B][N], outBary [B][N][3] and, when not null, the nodes visited
// per query visits [B][N]. mode: 0 the kernels' traversal of the tree built from ref, 1 the linear scan (ref unused but checked),
// 2 / 3 the wrong traversals.
extern "C" int emu_closest_points(int32_t V, int32_t F, const int32_t* faces, const float* ref, int32_t batch, int32_t N, const float* positions,
                                  const float* points, float maxDist, int32_t mode, float* outPoints, int32_t* outFace, float* outBary, int32_t* visits) {
  HostMeshFaces m;
  HostMeshTree t;
  if (make(V, F, faces, ref, m, t) != MB2_OK) return MB2_ERR_INVALID_ARGUMENT;
  std::vector<float> boxes(size_t(t.numNodes) * 6);
  for (int b = 0; b < batch; ++b) {
    const float* x = positions + size_t(b) * V * 3;
    if (mode != kScan) refit(m, t, x, boxes.data());
    for (int n = 0; n < N; ++n) {
      const size_t qi = size_t(b) * N + n;
      const F3 p = ld3(points + 3 * qi);
      Best r;
      r.d2 = maxDist * maxDist;
      int v = 0;
      if (mode == kScan) {
        for (int f = 0; f < F; ++f) tryFace(m, x, p, f, r);
      } else {
        v = traverse(m, t, x, boxes.data(), p, mode, r);
      }
      const bool found = r.face != INT_MAX;
      const F3 q = found ? r.q : f3(0.f, 0.f, 0.f), bary = found ? r.bary : f3(0.f, 0.f, 0.f);
      outPoints[3 * qi] = q.x; outPoints[3 * qi + 1] = q.y; outPoints[3 * qi + 2] = q.z;
      outBary[3 * qi] = bary.x; outBary[3 * qi + 1] = bary.y; outBary[3 * qi + 2] = bary.z;
      outFace[qi] = found ? r.face : -1;
      if (visits) visits[qi] = v;
    }
  }
  return MB2_OK;
}
