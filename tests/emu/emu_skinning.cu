// TEST HARNESS ONLY — CPU lane-emulation of the skinning kernels (mb2_character_skin_points*_device), built by tests/test_skinning.py
// into a temporary directory together with ik_plan.cpp / ik_chol_sched.cpp.
//
// The character and its skin tables are made by the library's own makeCharacter / makeSkinning; the __host__ __device__ building blocks
// of ik_device.cuh then run pass by pass in the kernels' order: the skinning transforms, the vertex blend, the per-segment sums with 32
// lanes and the butterfly of skinStatePartialKernel, the segments of each joint in order, and the rest-point gradient summed over the
// same fixed chunks of instances. It is not part of the product library and nothing in momentum_b200/ loads it.
#include <algorithm>
#include <cstdint>
#include <string>
#include <vector>

#include "../../include/momentum_b200.h"
#include "../../momentum_b200/csrc/ik_device.cuh"
#include "../../momentum_b200/csrc/ik_plan.h"

using namespace mb2;

static thread_local std::string g_err;

extern "C" const char* emu_skinning_last_error(void) { return g_err.c_str(); }

namespace {
struct Emu {
  HostCharacter h;
  HostSkinning s;
  SkinTables S{};
};

int make(int32_t J, const int32_t* parents, const float* offsets, const float* prerot, int32_t n, const int32_t* outer, const int32_t* inner,
         const float* vals, const float* ptOffsets, int32_t V, const float* rest, const int32_t* index, const float* weight, const float* ibp, Emu& e) {
  g_err = makeCharacter(J, parents, offsets, prerot, n, outer, inner, vals, ptOffsets, e.h);
  if (g_err.empty()) g_err = makeSkinning(e.h, V, rest, index, weight, ibp, e.s);
  if (!g_err.empty()) return MB2_ERR_INVALID_ARGUMENT;
  const HostSkinning& s = e.s;
  e.S = SkinTables{s.numVertices, s.numSegments(), s.restVertices.data(), s.vertStart.data(), s.vertJoint.data(), s.vertWeight.data(),
                   s.inverseBindPose.data(), s.infVertex.data(), s.infWeight.data(), s.segStart.data(), s.segJoint.data(), s.jointSegStart.data()};
  return MB2_OK;
}

void transforms(const Emu& e, const float* state, std::vector<float>& M) {
  M.assign(size_t(e.h.numJoints) * kSkinIbpStride, 0.f);
  for (int j = 0; j < e.h.numJoints; ++j) skinTransform(state + 8 * j, e.S.inverseBindPose + j * kSkinIbpStride, M.data() + j * kSkinIbpStride);
}
} // namespace

#define EMU_CHARACTER_ARGS                                                                                                                       \
  int32_t J, const int32_t *parents, const float *offsets, const float *prerot, int32_t n, const int32_t *outer, const int32_t *inner, \
      const float *vals, const float *ptOffsets, int32_t V, const float *restVertices, const int32_t *skinIndex, const float *skinWeight,     \
      const float *inverseBindPose
#define EMU_MAKE(e) make(J, parents, offsets, prerot, n, outer, inner, vals, ptOffsets, V, restVertices, skinIndex, skinWeight, inverseBindPose, e)

// the number of active influences per vertex [V] and the by-joint list (jointStart [J+1], infVertex [nnz]) as the library built them
extern "C" int emu_skinning_tables(EMU_CHARACTER_ARGS, int32_t* counts, int32_t* numInfluences) {
  Emu e;
  if (EMU_MAKE(e) != MB2_OK) return MB2_ERR_INVALID_ARGUMENT;
  for (int v = 0; v < V; ++v) counts[v] = e.s.vertStart[v + 1] - e.s.vertStart[v];
  *numInfluences = e.s.numInfluences();
  return MB2_OK;
}

// skel_state [B][J][8], rest points (null: the rest mesh; else [V][3] or [B][V][3]) -> points [B][V][3]
extern "C" int emu_skin_points(EMU_CHARACTER_ARGS, int32_t batch, const float* state, const float* restPoints, int32_t restBatched, float* points) {
  Emu e;
  if (EMU_MAKE(e) != MB2_OK) return MB2_ERR_INVALID_ARGUMENT;
  std::vector<float> M;
  for (int b = 0; b < batch; ++b) {
    transforms(e, state + size_t(b) * J * 8, M);
    const float* x = restPoints == nullptr ? e.S.restVertices : restPoints + (restBatched ? size_t(b) * V * 3 : 0);
    for (int v = 0; v < V; ++v) {
      const F3 p = skinBlend(e.S, M.data(), v, ld3(x + 3 * v));
      float* o = points + (size_t(b) * V + v) * 3;
      o[0] = p.x; o[1] = p.y; o[2] = p.z;
    }
  }
  return MB2_OK;
}

// the backward: gradState [B][J][8] and gradRest ([B][V][3] batched, [V][3] shared), either may be null
extern "C" int emu_skin_points_backward(EMU_CHARACTER_ARGS, int32_t batch, const float* state, const float* restPoints, int32_t restBatched,
                                        const float* gradPoints, float* gradState, float* gradRest) {
  Emu e;
  if (EMU_MAKE(e) != MB2_OK) return MB2_ERR_INVALID_ARGUMENT;
  const SkinTables& S = e.S;
  const int numSeg = S.numSegments;
  std::vector<float> partial(size_t(numSeg) * kSkinAccFloats), M;
  for (int b = 0; b < batch && gradState != nullptr; ++b) {
    const float* x = restPoints == nullptr ? S.restVertices : restPoints + (restBatched ? size_t(b) * V * 3 : 0);
    const float* g = gradPoints + size_t(b) * V * 3;
    for (int s = 0; s < numSeg; ++s) { // skinStatePartialKernel: 32 lanes, then the xor butterfly
      float lanes[32][kSkinAccFloats] = {};
      const float* ibp = S.inverseBindPose + S.segJoint[s] * kSkinIbpStride;
      for (int lane = 0; lane < 32; ++lane)
        for (int k = S.segStart[s] + lane; k < S.segStart[s + 1]; k += 32)
          skinAccumulate(ibp, ld3(x + 3 * S.infVertex[k]), ld3(g + 3 * S.infVertex[k]), S.infWeight[k], lanes[lane]);
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
  if (gradRest == nullptr) return MB2_OK;
  if (restPoints == nullptr) { g_err = "grad_rest_points must be null when the rest mesh is skinned"; return MB2_ERR_INVALID_ARGUMENT; }
  // shared: fixed chunks of max(8, ceil(B / 128)) instances summed in instance order, then the chunks in order
  const int perChunk = restBatched ? 1 : std::max(8, (batch + 127) / 128);
  std::vector<float> chunk(size_t(V) * 3), total(size_t(V) * 3, 0.f);
  for (int c0 = 0; c0 < batch; c0 += perChunk) {
    std::fill(chunk.begin(), chunk.end(), 0.f);
    for (int b = c0; b < std::min(batch, c0 + perChunk); ++b) {
      transforms(e, state + size_t(b) * J * 8, M);
      for (int v = 0; v < V; ++v) {
        const F3 r = skinRestGradient(S, M.data(), v, ld3(gradPoints + (size_t(b) * V + v) * 3));
        chunk[3 * v] += r.x; chunk[3 * v + 1] += r.y; chunk[3 * v + 2] += r.z;
      }
    }
    if (restBatched) std::copy(chunk.begin(), chunk.end(), gradRest + size_t(c0) * V * 3);
    else if (c0 == 0) total = chunk;
    else for (size_t i = 0; i < total.size(); ++i) total[i] += chunk[i];
  }
  if (!restBatched) std::copy(total.begin(), total.end(), gradRest);
  return MB2_OK;
}
