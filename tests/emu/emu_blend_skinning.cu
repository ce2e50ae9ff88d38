// TEST HARNESS ONLY — CPU lane-emulation of the blend-shape skinning kernels (mb2_character_skin_with_blend_shapes*_device), part of
// tests/emu/libmb2_emu.so.
//
// The character, its skin tables and its blend shape are made by the library's own makeCharacter / makeSkinning / makeBlendShape; the
// __host__ __device__ building blocks of ik_device.cuh then run pass by pass in the kernels' order: the rest points (blendShapeRest), the
// skinning transforms and the vertex blend; for the skel-state gradient the shaped rest points, then the skinning's skel-state backward
// (emu_skin.cuh); for the weight gradient the rest-point gradient of each vertex, the sums of blendWeightPartialKernel over each quarter
// of a 256-vertex block, the quarters in order, then the blocks in order. It is not part of the product library and nothing in
// momentum_b200/ loads it.
#include <algorithm>
#include <cstdint>
#include <vector>

#include "../../include/momentum_b200.h"
#include "emu_error.h"
#include "emu_skin.cuh"

using namespace mb2;

namespace {
constexpr int kBlock = 256, kGroups = 4, kGroupVerts = kBlock / kGroups; // blendWeightPartialKernel's vertex block and its quarters

struct Emu {
  HostCharacter h;
  HostSkinning s;
  HostBlendShape b;
  SkinTables S{};
  BlendShapeTables Bs{};
};

// the rest points of one instance, [V][3]
void restPoints(const Emu& e, const float* w, int numWeights, std::vector<float>& x) {
  const int V = e.S.numVertices;
  x.resize(size_t(V) * 3);
  for (int v = 0; v < V; ++v) {
    F3 r[1];
    blendShapeRest<1>(e.Bs, V, v, w, numWeights, r);
    x[3 * v] = r[0].x; x[3 * v + 1] = r[0].y; x[3 * v + 2] = r[0].z;
  }
}
} // namespace

#define EMU_ARGS                                                                                                                          \
  int32_t J, const int32_t *parents, const float *offsets, const float *prerot, int32_t n, const int32_t *outer, const int32_t *inner, \
      const float *vals, const float *ptOffsets, int32_t V, const float *restVertices, const int32_t *skinIndex, const float *skinWeight,     \
      const float *inverseBindPose, int32_t K, int32_t BV, const float *baseShape, const float *shapeVectors
#define EMU_MAKE(e) make(J, parents, offsets, prerot, n, outer, inner, vals, ptOffsets, V, restVertices, skinIndex, skinWeight, inverseBindPose, K, BV, baseShape, shapeVectors, e)

static int make(EMU_ARGS, Emu& e) {
  g_emuErr = makeCharacter(J, parents, offsets, prerot, n, outer, inner, vals, ptOffsets, e.h);
  if (g_emuErr.empty()) g_emuErr = makeSkinning(e.h, V, restVertices, skinIndex, skinWeight, inverseBindPose, e.s);
  if (g_emuErr.empty()) g_emuErr = makeBlendShape(K, BV, baseShape, shapeVectors, e.b);
  if (g_emuErr.empty() && BV != V) g_emuErr = "skin with blend shapes: the blend shape's vertex count differs from the skinning's";
  if (!g_emuErr.empty()) return MB2_ERR_INVALID_ARGUMENT;
  e.S = emuSkinTables(e.s);
  e.Bs = BlendShapeTables{e.b.numShapes, e.b.baseShape.data(), e.b.shapeVectors.data()};
  return MB2_OK;
}

// makeBlendShape alone: a first blend shape (K1, V1), then a second into the same record; returns the second's code and the K the record
// holds afterwards
extern "C" int emu_blend_shape_replace(int32_t K1, int32_t V1, const float* base1, const float* vectors1, int32_t K2, int32_t V2, const float* base2,
                                       const float* vectors2, int32_t* kAfter) {
  HostBlendShape b;
  g_emuErr = makeBlendShape(K1, V1, base1, vectors1, b);
  if (!g_emuErr.empty()) return MB2_ERR_INVALID_ARGUMENT;
  g_emuErr = makeBlendShape(K2, V2, base2, vectors2, b);
  *kAfter = b.numShapes;
  return g_emuErr.empty() ? MB2_OK : MB2_ERR_INVALID_ARGUMENT;
}

// skel_state [B][J][8], blend weights [B][K'] -> points [B][V][3]
extern "C" int emu_skin_with_blend_shapes(EMU_ARGS, int32_t batch, const float* state, const float* weights, int32_t numWeights, float* points) {
  Emu e;
  if (EMU_MAKE(e) != MB2_OK) return MB2_ERR_INVALID_ARGUMENT;
  if (numWeights < 1 || numWeights > K) { g_emuErr = "num_weights out of range"; return MB2_ERR_INVALID_ARGUMENT; }
  std::vector<float> M, x;
  for (int b = 0; b < batch; ++b) {
    restPoints(e, weights + size_t(b) * numWeights, numWeights, x);
    emuSkinTransforms(e.S, J, state + size_t(b) * J * 8, M);
    for (int v = 0; v < V; ++v) {
      const F3 p = skinBlend(e.S, M.data(), v, ld3(x.data() + 3 * v));
      float* o = points + (size_t(b) * V + v) * 3;
      o[0] = p.x; o[1] = p.y; o[2] = p.z;
    }
  }
  return MB2_OK;
}

// the backward: gradState [B][J][8] and gradWeights [B][K'], either may be null
extern "C" int emu_skin_with_blend_shapes_backward(EMU_ARGS, int32_t batch, const float* state, const float* weights, int32_t numWeights,
                                                   const float* gradPoints, float* gradState, float* gradWeights) {
  Emu e;
  if (EMU_MAKE(e) != MB2_OK) return MB2_ERR_INVALID_ARGUMENT;
  if (numWeights < 1 || numWeights > K) { g_emuErr = "num_weights out of range"; return MB2_ERR_INVALID_ARGUMENT; }
  const SkinTables& S = e.S;
  std::vector<float> M, x;
  for (int b = 0; b < batch && gradState != nullptr; ++b) {
    restPoints(e, weights + size_t(b) * numWeights, numWeights, x);
    emuSkinStateBackward(S, J, state + size_t(b) * J * 8, x.data(), gradPoints + size_t(b) * V * 3, gradState + size_t(b) * J * 8);
  }
  if (gradWeights == nullptr) return MB2_OK;
  const int vBlocks = (V + kBlock - 1) / kBlock;
  std::vector<float> r(size_t(V) * 3);
  for (int b = 0; b < batch; ++b) {
    emuSkinTransforms(e.S, J, state + size_t(b) * J * 8, M);
    for (int v = 0; v < V; ++v) { // the rest-point gradient of every vertex
      const F3 q = skinRestGradient(S, M.data(), v, ld3(gradPoints + (size_t(b) * V + v) * 3));
      r[3 * v] = q.x; r[3 * v + 1] = q.y; r[3 * v + 2] = q.z;
    }
    for (int k = 0; k < numWeights; ++k) {
      float total = 0.f;
      for (int vb = 0; vb < vBlocks; ++vb) { // blendWeightPartialKernel: the quarters of the block in order; then the blocks in order
        float block = 0.f;
        for (int q = 0; q < kGroups; ++q) {
          float acc = 0.f;
          for (int v = vb * kBlock + q * kGroupVerts; v < std::min(V, vb * kBlock + (q + 1) * kGroupVerts); ++v)
            acc = blendWeightAccumulate(acc, ld3(e.Bs.shapeVectors + (size_t(k) * V + v) * 3), ld3(r.data() + 3 * v));
          block = q == 0 ? acc : block + acc;
        }
        total = vb == 0 ? block : total + block;
      }
      gradWeights[size_t(b) * numWeights + k] = total;
    }
  }
  return MB2_OK;
}
