// TEST HARNESS ONLY — CPU emulation of the inverse ParameterTransform, part of tests/emu/libmb2_emu.so: the flat kernels
// inverseParameterTransformKernel / inverseParameterTransformBackwardKernel of launchJointOp
// (mb2_character_apply_inverse_parameter_transform*_device).
//
// The character, with its pseudo-inverse tables, is made by the library's own makeCharacter; the kernels' own element function of
// ik_device.cuh (jointOpElement) then runs element by element in order. It is not part of the product library and nothing in
// momentum_b200/ loads it.
#include <cstdint>

#include "../../include/momentum_b200.h"
#include "../../momentum_b200/csrc/ik_device.cuh"
#include "../../momentum_b200/csrc/ik_plan.h"
#include "emu_error.h"

using namespace mb2;

// character arrays as mb2_character_create takes them. Forward: out [B][n] = W (in [B][7 J] - o); backward: out [B][7 J] = W^T grad
// [B][n] (in is not read). batch == 0 only makes the character, tables included. Arrays dense, host memory.
extern "C" int emu_inverse_parameter_transform(int32_t numJoints, const int32_t* parents, const float* offsets, const float* prerot, int32_t numParams,
                                               const int32_t* outer, const int32_t* inner, const float* vals, const float* ptOffsets, int32_t backward,
                                               int32_t batch, const float* in, const float* grad, float* out) {
  HostCharacter h;
  g_emuErr = makeCharacter(numJoints, parents, offsets, prerot, numParams, outer, inner, vals, ptOffsets, h);
  if (!g_emuErr.empty()) return MB2_ERR_INVALID_ARGUMENT;
  if (batch < 0 || (batch > 0 && !((in || backward) && out && (!backward || grad)))) { g_emuErr = "null argument"; return MB2_ERR_INVALID_ARGUMENT; }
  const CharacterTables C = hostCharacterTables(h);
  const SkeletonTables S{h.childStart.data(),  h.children.data(), h.ptColStart.data(), h.ptColRows.data(), h.ptColVals.data(), h.invStart.data(),
                         h.invRows.data(),     h.invVals.data(),  h.invRowStart.data(), h.invParams.data(), h.invRowVals.data()};
  if (backward) {
    const long items = long(batch) * jointOpItems<kJointOpInverseParameterTransform, true>(C);
    for (long i = 0; i < items; ++i) jointOpElement<kJointOpInverseParameterTransform, true>(C, S, i, in, grad, out);
  } else {
    const long items = long(batch) * jointOpItems<kJointOpInverseParameterTransform, false>(C);
    for (long i = 0; i < items; ++i) jointOpElement<kJointOpInverseParameterTransform, false>(C, S, i, in, grad, out);
  }
  return MB2_OK;
}
