// TEST HARNESS ONLY — CPU lane-emulation of positionsKernel (mb2_character_{model,joint}_parameters_to_positions*_device), part of
// tests/emu/libmb2_emu.so.
//
// The character and the point tables are made by the library's own makeCharacter and makePointTables; the kernel's own pass functions of
// ik_device.cuh (fkPasses, positionPasses, positionGradPasses) then run with HostLanes, the lanes of each pass in sequence. A shared
// offset gradient is summed as the device sums it: in instance order within chunks of batchSumChunk(B) instances, then chunk by chunk. It
// is not part of the product library and nothing in momentum_b200/ loads it.
#include <algorithm>
#include <cstdint>
#include <vector>

#include "../../include/momentum_b200.h"
#include "../../momentum_b200/csrc/ik_device.cuh"
#include "../../momentum_b200/csrc/ik_plan.h"
#include "emu_error.h"

using namespace mb2;

namespace {
struct Emulated {
  HostCharacter h;
  std::vector<int32_t> points;
  CharacterTables C;
  SkeletonTables S;
  PointTables P;
  size_t inN;
};

int setUp(int32_t numJoints, const int32_t* parents, const float* offsets, const float* prerot, int32_t numParams, const int32_t* outer,
          const int32_t* inner, const float* vals, const float* ptOffsets, int32_t joint, int32_t numPoints, const int32_t* pointParents, Emulated& e) {
  g_emuErr = makeCharacter(numJoints, parents, offsets, prerot, numParams, outer, inner, vals, ptOffsets, e.h);
  if (g_emuErr.empty()) g_emuErr = makePointTables(e.h.numJoints, numPoints, pointParents, e.points);
  if (!g_emuErr.empty()) return MB2_ERR_INVALID_ARGUMENT;
  e.C = hostCharacterTables(e.h);
  e.S = SkeletonTables{e.h.childStart.data(), e.h.children.data(), e.h.ptColStart.data(), e.h.ptColRows.data(), e.h.ptColVals.data()};
  e.P = pointTablesAt(e.points.data(), e.C.numJoints, numPoints);
  e.inN = joint ? size_t(e.C.numJoints) * kParametersPerJoint : size_t(e.C.numParams);
  return MB2_OK;
}
} // namespace

// character arrays as mb2_character_create takes them; joint: params are [B][7 J] joint parameters, else [B][n] model parameters;
// parents [N], offsets [N][3] shared or [B][N][3] (offsetsBatched) -> positions [B][N][3] (host memory)
extern "C" int emu_positions(int32_t numJoints, const int32_t* parents, const float* offsets, const float* prerot, int32_t numParams, const int32_t* outer,
                             const int32_t* inner, const float* vals, const float* ptOffsets, int32_t joint, int32_t batch, const float* params,
                             int32_t numPoints, const int32_t* pointParents, const float* pointOffsets, int32_t offsetsBatched, float* positions) {
  Emulated e;
  if (setUp(numJoints, parents, offsets, prerot, numParams, outer, inner, vals, ptOffsets, joint, numPoints, pointParents, e) != MB2_OK)
    return MB2_ERR_INVALID_ARGUMENT;
  const size_t n3 = size_t(numPoints) * 3;
  std::vector<float> js(size_t(e.C.numJoints) * kJointStateStride);
  for (int b = 0; b < batch; ++b) {
    const float* p = params + size_t(b) * e.inN;
    if (joint) fkPasses<false, true>(HostLanes{}, e.C, p, js.data());
    else fkPasses<false, false>(HostLanes{}, e.C, p, js.data());
    positionPasses(HostLanes{}, e.P, js.data(), pointOffsets + (offsetsBatched ? size_t(b) * n3 : 0), positions + size_t(b) * n3);
  }
  return MB2_OK;
}

// its backward from gradPositions [B][N][3]: gradParams [B][n] ([B][7 J]) and gradOffsets ([N][3] the batch sum when shared, else
// [B][N][3]), each skipped when null
extern "C" int emu_positions_backward(int32_t numJoints, const int32_t* parents, const float* offsets, const float* prerot, int32_t numParams,
                                      const int32_t* outer, const int32_t* inner, const float* vals, const float* ptOffsets, int32_t joint, int32_t batch,
                                      const float* params, int32_t numPoints, const int32_t* pointParents, const float* pointOffsets,
                                      int32_t offsetsBatched, const float* gradPositions, float* gradParams, float* gradOffsets) {
  Emulated e;
  if (setUp(numJoints, parents, offsets, prerot, numParams, outer, inner, vals, ptOffsets, joint, numPoints, pointParents, e) != MB2_OK)
    return MB2_ERR_INVALID_ARGUMENT;
  const int J = e.C.numJoints;
  const size_t n3 = size_t(numPoints) * 3;
  std::vector<float> js(size_t(J) * kJointStateStride), acc(size_t(J) * kSkelAccStride), gjp(size_t(J) * kParametersPerJoint);
  std::vector<float> rows(gradOffsets != nullptr && !offsetsBatched ? size_t(batch) * n3 : 0);
  for (int b = 0; b < batch; ++b) {
    const float* p = params + size_t(b) * e.inN;
    if (joint) fkPasses<true, true>(HostLanes{}, e.C, p, js.data());
    else fkPasses<true, false>(HostLanes{}, e.C, p, js.data());
    float* gp = gradParams != nullptr ? gradParams + size_t(b) * e.inN : nullptr;
    float* gOff = gradOffsets == nullptr ? nullptr : (offsetsBatched ? gradOffsets + size_t(b) * n3 : rows.data() + size_t(b) * n3);
    positionGradPasses(HostLanes{}, e.C, e.S, e.P, js.data(), pointOffsets + (offsetsBatched ? size_t(b) * n3 : 0), gradPositions + size_t(b) * n3,
                       acc.data(), joint || gp == nullptr ? gp : gjp.data(), joint ? nullptr : gp, gOff);
  }
  if (gradOffsets != nullptr && !offsetsBatched) {
    const int perChunk = batchSumChunk(batch);
    for (size_t k = 0; k < n3; ++k) {
      float total = 0.f;
      for (int c0 = 0; c0 < batch; c0 += perChunk) {
        float s = rows[size_t(c0) * n3 + k];
        for (int b = c0 + 1; b < std::min(batch, c0 + perChunk); ++b) s += rows[size_t(b) * n3 + k];
        total = c0 == 0 ? s : total + s;
      }
      gradOffsets[k] = total;
    }
  }
  return MB2_OK;
}
