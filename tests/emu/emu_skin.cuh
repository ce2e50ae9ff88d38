// TEST HARNESS ONLY — the skinning passes that emu_skinning.cu and emu_blend_skinning.cu share, as the device's blend-shape backward
// runs the skinning backward unchanged (launchSkinPointsBackward): the skin tables, the skinning transforms and the skel-state backward.
#pragma once
#include <algorithm>
#include <vector>

#include "../../momentum_b200/csrc/ik_device.cuh"
#include "../../momentum_b200/csrc/ik_plan.h"

namespace mb2 {

inline SkinTables emuSkinTables(const HostSkinning& s) {
  return SkinTables{s.numVertices, s.numSegments(), s.restVertices.data(), s.vertStart.data(), s.vertJoint.data(), s.vertWeight.data(),
                    s.inverseBindPose.data(), s.infVertex.data(), s.infWeight.data(), s.segStart.data(), s.segJoint.data(), s.jointSegStart.data()};
}

// the skinning transforms M [J][kSkinIbpStride] of one instance's skel_state [J][8]
inline void emuSkinTransforms(const SkinTables& S, int numJoints, const float* state, std::vector<float>& M) {
  M.assign(size_t(numJoints) * kSkinIbpStride, 0.f);
  for (int j = 0; j < numJoints; ++j) skinTransform(state + 8 * j, S.inverseBindPose + j * kSkinIbpStride, M.data() + j * kSkinIbpStride);
}

// the skel-state gradient [J][8] of one instance from its rest points x [V][3] and gradPoints g [V][3]
inline void emuSkinStateBackward(const SkinTables& S, int numJoints, const float* state, const float* x, const float* g, float* gradState) {
  std::vector<float> partial(size_t(S.numSegments) * kSkinAccFloats);
  for (int s = 0; s < S.numSegments; ++s) { // skinStatePartialKernel: 32 lanes, then the xor butterfly
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
  for (int j = 0; j < numJoints; ++j) { // skinStateFinishKernel
    float acc[kSkinAccFloats] = {};
    for (int s = S.jointSegStart[j]; s < S.jointSegStart[j + 1]; ++s)
      for (int r = 0; r < kSkinAccFloats; ++r) acc[r] += partial[size_t(s) * kSkinAccFloats + r];
    skinStateGradient(acc, state + size_t(j) * 8, gradState + size_t(j) * 8);
  }
}

} // namespace mb2
