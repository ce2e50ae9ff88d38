// TEST HARNESS ONLY — CPU lane-emulation of the joint-parameter operations, part of tests/emu/libmb2_emu.so:
// skeletonStateKernel<kBackward, W, true> (mb2_character_joint_parameters_to_skeleton_state*_device) and the flat kernels of
// launchJointOp (mb2_character_apply_parameter_transform*, *_local_skeleton_state*, *_to_joint_parameters*).
//
// The character is made by the library's own makeCharacter; the kernels' own pass and element functions of ik_device.cuh (fkPasses,
// skelGradPasses, jointOpElement) then run with HostLanes or element by element in order. It is not part of the product library and
// nothing in momentum_b200/ loads it.
#include <cstdint>

#include "../../include/momentum_b200.h"
#include "../../momentum_b200/csrc/ik_device.cuh"
#include "../../momentum_b200/csrc/ik_plan.h"
#include "emu_error.h"
#include "emu_frame.h"

using namespace mb2;

namespace {
template <int kOp, bool kBackward>
void runElements(const CharacterTables& C, const SkeletonTables& S, int batch, const float* in, const float* grad, float* out) {
  const long items = long(batch) * jointOpItems<kOp, kBackward>(C);
  for (long i = 0; i < items; ++i) jointOpElement<kOp, kBackward>(C, S, i, in, grad, out);
}
} // namespace

// character arrays as mb2_character_create takes them; op: 0 apply_parameter_transform, 1 joint_parameters_to_local_skeleton_state,
// 2 local_skeleton_state_to_joint_parameters, 3 skeleton_state_to_joint_parameters, 4 joint_parameters_to_skeleton_state. Forward:
// out = op(in); backward: out = dLoss / d in from grad = dLoss / d op(in). Arrays [B][...] dense, host memory.
extern "C" int emu_joint_parameters(int32_t numJoints, const int32_t* parents, const float* offsets, const float* prerot, int32_t numParams,
                                    const int32_t* outer, const int32_t* inner, const float* vals, const float* ptOffsets, int32_t op,
                                    int32_t backward, int32_t batch, const float* in, const float* grad, float* out) {
  HostCharacter h;
  g_emuErr = makeCharacter(numJoints, parents, offsets, prerot, numParams, outer, inner, vals, ptOffsets, h);
  if (!g_emuErr.empty()) return MB2_ERR_INVALID_ARGUMENT;
  if (op < 0 || op > 4) { g_emuErr = "unknown operation"; return MB2_ERR_INVALID_ARGUMENT; }
  if (batch < 0 || (batch > 0 && !((in || (op == 0 && backward)) && out && (!backward || grad)))) { g_emuErr = "null argument"; return MB2_ERR_INVALID_ARGUMENT; }
  const CharacterTables C = hostCharacterTables(h);
  const SkeletonTables S{h.childStart.data(), h.children.data(), h.ptColStart.data(), h.ptColRows.data(), h.ptColVals.data()};
  const int J = C.numJoints;
  if (op == 4) {
    const size_t inN = size_t(J) * kParametersPerJoint;
    const auto f = skeletonStateFrame(J, C.numParams, backward != 0, true);
    EmuFrame fr{f.floats};
    float* js = fr.at(f.js);
    for (int b = 0; b < batch; ++b) {
      const float* jp = fr.load(f.in, in + size_t(b) * inN, inN);
      if (backward) {
        fkPasses<true, true>(HostLanes{}, C, jp, js);
        skelGradPasses(HostLanes{}, C, S, js, grad + size_t(b) * J * 8, fr.at(f.acc), out + size_t(b) * inN, nullptr);
      } else {
        fkPasses<false, true>(HostLanes{}, C, jp, js);
        for (int i = 0; i < J * 8; ++i) out[size_t(b) * J * 8 + i] = js[(i >> 3) * kJointStateStride + (i & 7)];
      }
    }
    return fr.check("skeletonStateKernel");
  }
  switch (op * 2 + (backward ? 1 : 0)) {
    case 0: runElements<kJointOpParameterTransform, false>(C, S, batch, in, grad, out); break;
    case 1: runElements<kJointOpParameterTransform, true>(C, S, batch, in, grad, out); break;
    case 2: runElements<kJointOpLocalState, false>(C, S, batch, in, grad, out); break;
    case 3: runElements<kJointOpLocalState, true>(C, S, batch, in, grad, out); break;
    case 4: runElements<kJointOpFromLocal, false>(C, S, batch, in, grad, out); break;
    case 5: runElements<kJointOpFromLocal, true>(C, S, batch, in, grad, out); break;
    case 6: runElements<kJointOpFromWorld, false>(C, S, batch, in, grad, out); break;
    default: runElements<kJointOpFromWorld, true>(C, S, batch, in, grad, out); break;
  }
  return MB2_OK;
}
