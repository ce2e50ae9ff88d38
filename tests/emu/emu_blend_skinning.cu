// TEST HARNESS ONLY — CPU lane-emulation of the blend-shape skinning kernels (mb2_character_skin_with_blend_shapes*_device), built by
// tests/test_blend_shape_skinning.py into a temporary directory together with ik_plan.cpp / ik_chol_sched.cpp.
//
// The character, its skin tables and its blend shape are made by the library's own makeCharacter / makeSkinning / makeBlendShape; the
// __host__ __device__ building blocks of ik_device.cuh then run pass by pass in the kernels' order: the rest points (blendShapeRest), the
// skinning transforms and the vertex blend; for the skel-state gradient the shaped rest points, then skinStatePartialKernel's 32 lanes
// and butterfly and the segments of each joint in order; for the weight gradient the rest-point gradient of each vertex, the sums of
// blendWeightPartialKernel over each quarter of a 256-vertex block, the quarters in order, then the blocks in order. It is not part of
// the product library and nothing in momentum_b200/ loads it.
#include <algorithm>
#include <cstdint>
#include <string>
#include <vector>

#include "../../include/momentum_b200.h"
#include "../../momentum_b200/csrc/ik_device.cuh"
#include "../../momentum_b200/csrc/ik_plan.h"

using namespace mb2;

static thread_local std::string g_err;

extern "C" const char* emu_blend_skinning_last_error(void) { return g_err.c_str(); }

namespace {
constexpr int kBlock = 256, kGroups = 4, kGroupVerts = kBlock / kGroups; // blendWeightPartialKernel's vertex block and its quarters

struct Emu {
  HostCharacter h;
  HostSkinning s;
  HostBlendShape b;
  SkinTables S{};
  BlendShapeTables Bs{};
};

void transforms(const Emu& e, const float* state, std::vector<float>& M) {
  M.assign(size_t(e.h.numJoints) * kSkinIbpStride, 0.f);
  for (int j = 0; j < e.h.numJoints; ++j) skinTransform(state + 8 * j, e.S.inverseBindPose + j * kSkinIbpStride, M.data() + j * kSkinIbpStride);
}

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
  g_err = makeCharacter(J, parents, offsets, prerot, n, outer, inner, vals, ptOffsets, e.h);
  if (g_err.empty()) g_err = makeSkinning(e.h, V, restVertices, skinIndex, skinWeight, inverseBindPose, e.s);
  if (g_err.empty()) g_err = makeBlendShape(K, BV, baseShape, shapeVectors, e.b);
  if (g_err.empty() && BV != V) g_err = "skin with blend shapes: the blend shape's vertex count differs from the skinning's";
  if (!g_err.empty()) return MB2_ERR_INVALID_ARGUMENT;
  const HostSkinning& s = e.s;
  e.S = SkinTables{s.numVertices, s.numSegments(), s.restVertices.data(), s.vertStart.data(), s.vertJoint.data(), s.vertWeight.data(),
                   s.inverseBindPose.data(), s.infVertex.data(), s.infWeight.data(), s.segStart.data(), s.segJoint.data(), s.jointSegStart.data()};
  e.Bs = BlendShapeTables{e.b.numShapes, e.b.baseShape.data(), e.b.shapeVectors.data()};
  return MB2_OK;
}

// makeBlendShape alone: a first blend shape (K1, V1), then a second into the same record; returns the second's code and the K the record
// holds afterwards
extern "C" int emu_blend_shape_replace(int32_t K1, int32_t V1, const float* base1, const float* vectors1, int32_t K2, int32_t V2, const float* base2,
                                       const float* vectors2, int32_t* kAfter) {
  HostBlendShape b;
  g_err = makeBlendShape(K1, V1, base1, vectors1, b);
  if (!g_err.empty()) return MB2_ERR_INVALID_ARGUMENT;
  g_err = makeBlendShape(K2, V2, base2, vectors2, b);
  *kAfter = b.numShapes;
  return g_err.empty() ? MB2_OK : MB2_ERR_INVALID_ARGUMENT;
}

// skel_state [B][J][8], blend weights [B][K'] -> points [B][V][3]
extern "C" int emu_skin_with_blend_shapes(EMU_ARGS, int32_t batch, const float* state, const float* weights, int32_t numWeights, float* points) {
  Emu e;
  if (EMU_MAKE(e) != MB2_OK) return MB2_ERR_INVALID_ARGUMENT;
  if (numWeights < 1 || numWeights > K) { g_err = "num_weights out of range"; return MB2_ERR_INVALID_ARGUMENT; }
  std::vector<float> M, x;
  for (int b = 0; b < batch; ++b) {
    restPoints(e, weights + size_t(b) * numWeights, numWeights, x);
    transforms(e, state + size_t(b) * J * 8, M);
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
  if (numWeights < 1 || numWeights > K) { g_err = "num_weights out of range"; return MB2_ERR_INVALID_ARGUMENT; }
  const SkinTables& S = e.S;
  const int numSeg = S.numSegments;
  std::vector<float> partial(size_t(numSeg) * kSkinAccFloats), M, x;
  for (int b = 0; b < batch && gradState != nullptr; ++b) {
    restPoints(e, weights + size_t(b) * numWeights, numWeights, x);
    const float* g = gradPoints + size_t(b) * V * 3;
    for (int s = 0; s < numSeg; ++s) { // skinStatePartialKernel: 32 lanes, then the xor butterfly
      float lanes[32][kSkinAccFloats] = {};
      const float* ibp = S.inverseBindPose + S.segJoint[s] * kSkinIbpStride;
      for (int lane = 0; lane < 32; ++lane)
        for (int k = S.segStart[s] + lane; k < S.segStart[s + 1]; k += 32)
          skinAccumulate(ibp, ld3(x.data() + 3 * S.infVertex[k]), ld3(g + 3 * S.infVertex[k]), S.infWeight[k], lanes[lane]);
      for (int o = 16; o > 0; o >>= 1) {
        float next[32][kSkinAccFloats];
        for (int lane = 0; lane < 32; ++lane)
          for (int r = 0; r < kSkinAccFloats; ++r) next[lane][r] = lanes[lane][r] + lanes[lane ^ o][r];
        std::copy(&next[0][0], &next[0][0] + 32 * kSkinAccFloats, &lanes[0][0]);
      }
      std::copy(lanes[0], lanes[0] + kSkinAccFloats, partial.data() + size_t(s) * kSkinAccFloats);
    }
    for (int j = 0; j < J; ++j) { // skinStateFinishKernel
      float acc[kSkinAccFloats] = {};
      for (int s = S.jointSegStart[j]; s < S.jointSegStart[j + 1]; ++s)
        for (int r = 0; r < kSkinAccFloats; ++r) acc[r] += partial[size_t(s) * kSkinAccFloats + r];
      skinStateGradient(acc, state + (size_t(b) * J + j) * 8, gradState + (size_t(b) * J + j) * 8);
    }
  }
  if (gradWeights == nullptr) return MB2_OK;
  const int vBlocks = (V + kBlock - 1) / kBlock;
  std::vector<float> r(size_t(V) * 3);
  for (int b = 0; b < batch; ++b) {
    transforms(e, state + size_t(b) * J * 8, M);
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
