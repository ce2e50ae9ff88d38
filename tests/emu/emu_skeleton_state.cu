// TEST HARNESS ONLY — CPU lane-emulation of skeletonStateKernel<true> (mb2_character_skeleton_state_backward_device), part of
// tests/emu/libmb2_emu.so.
//
// The character is made by the library's own makeCharacter, which builds the tables the kernel walks (levels, children in CSR, the
// ParameterTransform in CSC); the kernel's own pass functions of ik_device.cuh (fkPasses, skelGradPasses) then run with HostLanes, the
// lanes of each pass in sequence. It is not part of the product library and nothing in momentum_b200/ loads it.
#include <cstdint>

#include "../../include/momentum_b200.h"
#include "../../momentum_b200/csrc/ik_device.cuh"
#include "../../momentum_b200/csrc/ik_plan.h"
#include "emu_error.h"
#include "emu_frame.h"

using namespace mb2;

// character arrays as mb2_character_create takes them; theta [B][n], grad_state [B][J][8] -> grad_theta [B][n] (host memory). shortFloats:
// the frame is that many floats shorter than skeletonStateFrame's (0 for the kernel's frame; > 0 shows that an overrun is caught).
extern "C" int emu_skeleton_state_backward_frame(int32_t numJoints, const int32_t* parents, const float* offsets, const float* prerot, int32_t numParams,
                                                 const int32_t* outer, const int32_t* inner, const float* vals, const float* ptOffsets, int32_t batch,
                                                 const float* theta, const float* gradState, float* gradTheta, int32_t shortFloats) {
  HostCharacter h;
  g_emuErr = makeCharacter(numJoints, parents, offsets, prerot, numParams, outer, inner, vals, ptOffsets, h);
  if (!g_emuErr.empty()) return MB2_ERR_INVALID_ARGUMENT;
  if (batch < 0 || (batch > 0 && !(theta && gradState && gradTheta))) { g_emuErr = "null argument"; return MB2_ERR_INVALID_ARGUMENT; }
  const CharacterTables C = hostCharacterTables(h);
  const SkeletonTables S{h.childStart.data(), h.children.data(), h.ptColStart.data(), h.ptColRows.data(), h.ptColVals.data()};
  const int J = C.numJoints, n = C.numParams;
  const auto f = skeletonStateFrame(J, n, true, false);
  EmuFrame fr{f.floats - size_t(shortFloats)};
  for (int b = 0; b < batch; ++b) {
    fkPasses<true, false>(HostLanes{}, C, fr.load(f.in, theta + size_t(b) * n, n), fr.at(f.js));
    skelGradPasses(HostLanes{}, C, S, fr.at(f.js), gradState + size_t(b) * J * 8, fr.at(f.acc), fr.at(f.gjp), gradTheta + size_t(b) * n);
  }
  return fr.check("skeletonStateKernel");
}

extern "C" int emu_skeleton_state_backward(int32_t numJoints, const int32_t* parents, const float* offsets, const float* prerot, int32_t numParams,
                                           const int32_t* outer, const int32_t* inner, const float* vals, const float* ptOffsets, int32_t batch,
                                           const float* theta, const float* gradState, float* gradTheta) {
  return emu_skeleton_state_backward_frame(numJoints, parents, offsets, prerot, numParams, outer, inner, vals, ptOffsets, batch, theta, gradState,
                                           gradTheta, 0);
}
