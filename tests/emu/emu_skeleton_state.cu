// TEST HARNESS ONLY — CPU lane-emulation of skeletonStateKernel<true> (mb2_character_skeleton_state_backward_device), built by
// tests/test_skeleton_state.py into a temporary directory together with ik_plan.cpp / ik_chol_sched.cpp.
//
// The character is made by the library's own makeCharacter, which builds the tables the kernel walks (levels, children in CSR, the
// ParameterTransform in CSC); the __host__ __device__ building blocks of ik_device.cuh then run pass by pass, the lanes of each pass in
// sequence. It is not part of the product library and nothing in momentum_b200/ loads it.
#include <cstdint>
#include <string>
#include <vector>

#include "../../include/momentum_b200.h"
#include "../../momentum_b200/csrc/ik_device.cuh"
#include "../../momentum_b200/csrc/ik_plan.h"

using namespace mb2;

static thread_local std::string g_err;

extern "C" const char* emu_skeleton_state_last_error(void) { return g_err.c_str(); }

// character arrays as mb2_character_create takes them; theta [B][n], grad_state [B][J][8] -> grad_theta [B][n] (host memory)
extern "C" int emu_skeleton_state_backward(int32_t numJoints, const int32_t* parents, const float* offsets, const float* prerot, int32_t numParams,
                                           const int32_t* outer, const int32_t* inner, const float* vals, const float* ptOffsets, int32_t batch,
                                           const float* theta, const float* gradState, float* gradTheta) {
  HostCharacter h;
  g_err = makeCharacter(numJoints, parents, offsets, prerot, numParams, outer, inner, vals, ptOffsets, h);
  if (!g_err.empty()) return MB2_ERR_INVALID_ARGUMENT;
  if (batch < 0 || (batch > 0 && !(theta && gradState && gradTheta))) { g_err = "null argument"; return MB2_ERR_INVALID_ARGUMENT; }
  FunctionTables T{};
  T.numJoints = h.numJoints; T.numParams = h.numParams;
  T.parent = h.parent.data(); T.offset = h.offset.data(); T.prerot = h.prerot.data();
  T.ptOuter = h.ptOuter.data(); T.ptInner = h.ptInner.data(); T.ptVals = h.ptVals.data(); T.ptOffsets = h.ptOffsets.data();
  T.numLevels = int(h.levelStart.size()) - 1; T.levelStart = h.levelStart.data(); T.levelJoints = h.levelJoints.data();
  T.ptNnz = int(h.ptInner.size());
  const SkeletonTables S{h.childStart.data(), h.children.data(), h.ptColStart.data(), h.ptColRows.data(), h.ptColVals.data()};
  const int J = T.numJoints, n = T.numParams;
  std::vector<float> js(size_t(J) * kJointStateStride), acc(size_t(J) * kSkelAccStride), gjp(size_t(J) * kParametersPerJoint);
  for (int b = 0; b < batch; ++b) {
    const float* th = theta + size_t(b) * n;
    for (int j = 0; j < J; ++j) fkLocalFromTheta<true>(T, j, th, js.data());
    for (int lvl = 1; lvl < T.numLevels; ++lvl)
      for (int k = T.levelStart[lvl]; k < T.levelStart[lvl + 1]; ++k) fkCompose(T, T.levelJoints[k], js.data());
    for (int i = 0; i < 3 * J; ++i) fkAxis(T, i / 3, i % 3, js.data());
    const float* G = gradState + size_t(b) * J * 8;
    for (int i = 0; i < J; ++i) skelGradSeed(js.data(), i, G + 8 * i, acc.data());
    for (int lvl = T.numLevels - 2; lvl >= 0; --lvl)
      for (int k = T.levelStart[lvl]; k < T.levelStart[lvl + 1]; ++k) skelGradFold(S, js.data(), T.levelJoints[k], acc.data());
    for (int row = 0; row < J * kParametersPerJoint; ++row) gjp[row] = skelGradJointParameter(T, js.data(), acc.data(), row);
    for (int p = 0; p < n; ++p) gradTheta[size_t(b) * n + p] = skelGradModelParameter(S, gjp.data(), p);
  }
  return MB2_OK;
}
