// TEST HARNESS ONLY — CPU lane-emulation of the skinning kernels (mb2_character_skin_points*_device), part of tests/emu/libmb2_emu.so.
//
// The character and its skin tables are made by the library's own makeCharacter / makeSkinning; the __host__ __device__ building blocks
// of ik_device.cuh then run pass by pass in the kernels' order: the skinning transforms, the vertex blend, the skel-state backward of
// emu_skin.cuh, and the rest-point gradient summed over the same fixed chunks of instances. It is not part of the product library and
// nothing in momentum_b200/ loads it.
#include <algorithm>
#include <cstdint>
#include <vector>

#include "../../include/momentum_b200.h"
#include "emu_error.h"
#include "emu_skin.cuh"

using namespace mb2;

namespace {
struct Emu {
  HostCharacter h;
  HostSkinning s;
  SkinTables S{};
};

int make(int32_t J, const int32_t* parents, const float* offsets, const float* prerot, int32_t n, const int32_t* outer, const int32_t* inner,
         const float* vals, const float* ptOffsets, int32_t V, const float* rest, const int32_t* index, const float* weight, const float* ibp, Emu& e) {
  g_emuErr = makeCharacter(J, parents, offsets, prerot, n, outer, inner, vals, ptOffsets, e.h);
  if (g_emuErr.empty()) g_emuErr = makeSkinning(e.h, V, rest, index, weight, ibp, e.s);
  if (!g_emuErr.empty()) return MB2_ERR_INVALID_ARGUMENT;
  e.S = emuSkinTables(e.s);
  return MB2_OK;
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
    emuSkinTransforms(e.S, J, state + size_t(b) * J * 8, M);
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
  for (int b = 0; b < batch && gradState != nullptr; ++b) {
    const float* x = restPoints == nullptr ? S.restVertices : restPoints + (restBatched ? size_t(b) * V * 3 : 0);
    emuSkinStateBackward(S, J, state + size_t(b) * J * 8, x, gradPoints + size_t(b) * V * 3, gradState + size_t(b) * J * 8);
  }
  if (gradRest == nullptr) return MB2_OK;
  if (restPoints == nullptr) { g_emuErr = "grad_rest_points must be null when the rest mesh is skinned"; return MB2_ERR_INVALID_ARGUMENT; }
  // shared: fixed chunks of max(8, ceil(B / 128)) instances summed in instance order, then the chunks in order
  const int perChunk = restBatched ? 1 : std::max(8, (batch + 127) / 128);
  std::vector<float> M, chunk(size_t(V) * 3), total(size_t(V) * 3, 0.f);
  for (int c0 = 0; c0 < batch; c0 += perChunk) {
    std::fill(chunk.begin(), chunk.end(), 0.f);
    for (int b = c0; b < std::min(batch, c0 + perChunk); ++b) {
      emuSkinTransforms(S, J, state + size_t(b) * J * 8, M);
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
