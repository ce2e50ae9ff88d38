// TEST HARNESS ONLY — CPU lane-emulation of skeletonStateKernel<true> (mb2_character_skeleton_state_backward_device), part of
// tests/emu/libmb2_emu.so.
//
// The character is made by the library's own makeCharacter, which builds the tables the kernel walks (levels, children in CSR, the
// ParameterTransform in CSC); the kernel's own pass functions of ik_device.cuh (fkPasses, skelGradPasses) then run with HostLanes, the
// lanes of each pass in sequence. It is not part of the product library and nothing in momentum_b200/ loads it.
#include <cstdint>
#include <vector>

#include "../../include/momentum_b200.h"
#include "../../momentum_b200/csrc/ik_device.cuh"
#include "../../momentum_b200/csrc/ik_plan.h"
#include "emu_error.h"

using namespace mb2;

// character arrays as mb2_character_create takes them; theta [B][n], grad_state [B][J][8] -> grad_theta [B][n] (host memory)
extern "C" int emu_skeleton_state_backward(int32_t numJoints, const int32_t* parents, const float* offsets, const float* prerot, int32_t numParams,
                                           const int32_t* outer, const int32_t* inner, const float* vals, const float* ptOffsets, int32_t batch,
                                           const float* theta, const float* gradState, float* gradTheta) {
  HostCharacter h;
  g_emuErr = makeCharacter(numJoints, parents, offsets, prerot, numParams, outer, inner, vals, ptOffsets, h);
  if (!g_emuErr.empty()) return MB2_ERR_INVALID_ARGUMENT;
  if (batch < 0 || (batch > 0 && !(theta && gradState && gradTheta))) { g_emuErr = "null argument"; return MB2_ERR_INVALID_ARGUMENT; }
  const CharacterTables C = hostCharacterTables(h);
  const SkeletonTables S{h.childStart.data(), h.children.data(), h.ptColStart.data(), h.ptColRows.data(), h.ptColVals.data()};
  const int J = C.numJoints, n = C.numParams;
  std::vector<float> js(size_t(J) * kJointStateStride), acc(size_t(J) * kSkelAccStride), gjp(size_t(J) * kParametersPerJoint);
  for (int b = 0; b < batch; ++b) {
    fkPasses<true, false>(HostLanes{}, C, theta + size_t(b) * n, js.data());
    skelGradPasses(HostLanes{}, C, S, js.data(), gradState + size_t(b) * J * 8, acc.data(), gjp.data(), gradTheta + size_t(b) * n);
  }
  return MB2_OK;
}
