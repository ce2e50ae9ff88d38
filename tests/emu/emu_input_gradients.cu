// TEST HARNESS ONLY — CPU lane-emulation of inputGradientKernel (mb2_solver_function_input_gradients_device), built by
// tests/test_solve_ik_input_gradients.py into a temporary directory together with ik_plan.cpp / ik_chol_sched.cpp.
//
// The character is made by the library's own makeCharacter and the block by the library's own error-function constructors and planner
// (the units the kernel reads); the __host__ __device__ building blocks of ik_device.cuh then run pass by pass, the lanes of each pass in
// sequence. It is not part of the product library and nothing in momentum_b200/ loads it.
#include <cmath>
#include <cstdint>
#include <string>
#include <vector>

#include "../../include/momentum_b200.h"
#include "../../momentum_b200/csrc/ik_device.cuh"
#include "../../momentum_b200/csrc/ik_plan.h"

using namespace mb2;

static thread_local std::string g_err;

extern "C" const char* emu_input_gradients_last_error(void) { return g_err.c_str(); }

// character arrays as mb2_character_create takes them; one block: kind 0 Position / 1 Orientation (matrix difference), shared offsets
// [nc][3|4] or (instanced) none; records [B][targetSize] as mb2_set_targets takes them, constraint weights [B][nc], enabled [n];
// theta, direction [B][n] -> grad_weights [B][nc], grad_offsets / grad_targets [B][nc][3|4] (host memory; null outputs skipped)
extern "C" int emu_input_gradients(int32_t numJoints, const int32_t* parents, const float* offsets, const float* prerot, int32_t numParams,
                                   const int32_t* outer, const int32_t* inner, const float* vals, const float* ptOffsets, int32_t kind,
                                   int32_t instanced, int32_t nc, const int32_t* cparents, const float* coffsets, float weight, float lossC,
                                   const uint8_t* enabled, int32_t batch, const float* records, const float* cweights, const float* theta,
                                   const float* direction, float* gradWeights, float* gradOffsets, float* gradTargets) {
  HostCharacter h;
  g_err = makeCharacter(numJoints, parents, offsets, prerot, numParams, outer, inner, vals, ptOffsets, h);
  if (!g_err.empty()) return MB2_ERR_INVALID_ARGUMENT;
  std::vector<float> ones(size_t(nc), 1.f);
  HostErrorFunction ef;
  if (kind == 0) g_err = instanced ? instancedPositionErrorFunction(h, weight, 2.f, lossC, nc, cparents, ones.data(), ef)
                                   : positionErrorFunction(h, weight, 2.f, lossC, nc, cparents, coffsets, ones.data(), ef);
  else g_err = instanced ? instancedOrientationErrorFunction(h, weight, 2.f, lossC, 0, nc, cparents, ones.data(), ef)
                         : orientationErrorFunction(h, weight, 2.f, lossC, 0, nc, cparents, coffsets, ones.data(), ef);
  if (!g_err.empty()) return MB2_ERR_INVALID_ARGUMENT;
  HostFunction hf;
  hf.enabled.assign(enabled, enabled + numParams);
  hf.add(ef, nullptr);
  Plan plan;
  g_err = buildPlan(h, hf.efs, hf.enabled, false, plan);
  if (!g_err.empty()) return MB2_ERR_INVALID_ARGUMENT;
  const int stride = hf.targetStride, per = kind == 0 ? 3 : 4;
  std::vector<float> rec(records, records + size_t(batch) * stride);
  if (kind == 1) // what the upload does (launchNormalizeQuats): every quaternion of the record normalised
    for (int b = 0; b < batch; ++b)
      for (int q = 0; q < stride / 4; ++q) {
        float* p = rec.data() + size_t(b) * stride + 4 * q;
        const float n = sqrtf(p[0] * p[0] + p[1] * p[1] + p[2] * p[2] + p[3] * p[3]);
        p[0] /= n; p[1] /= n; p[2] /= n; p[3] /= n;
      }
  FunctionTables T{};
  T.numJoints = h.numJoints; T.numParams = h.numParams;
  T.parent = h.parent.data(); T.offset = h.offset.data(); T.prerot = h.prerot.data();
  T.ptOuter = h.ptOuter.data(); T.ptInner = h.ptInner.data(); T.ptVals = h.ptVals.data(); T.ptOffsets = h.ptOffsets.data();
  T.numLevels = int(h.levelStart.size()) - 1; T.levelStart = h.levelStart.data(); T.levelJoints = h.levelJoints.data();
  T.ptNnz = int(h.ptInner.size());
  T.efs = plan.efs.data(); T.units = plan.units.data();
  T.targetStride = stride;
  T.weightsPerInstance = 1; T.numWeights = nc;
  const int J = T.numJoints, n = T.numParams;
  std::vector<float> vs(n), js(size_t(J) * kJointStateStride), tan(size_t(J) * kTangentStride);
  for (int b = 0; b < batch; ++b) {
    const float* th = theta + size_t(b) * n;
    for (int i = 0; i < n; ++i) vs[i] = 0.f;
    for (int p : plan.enabledList) vs[p] = direction[size_t(b) * n + p];
    for (int j = 0; j < J; ++j) fkLocalFromTheta<true>(T, j, th, js.data());
    for (int lvl = 1; lvl < T.numLevels; ++lvl)
      for (int k = T.levelStart[lvl]; k < T.levelStart[lvl + 1]; ++k) fkCompose(T, T.levelJoints[k], js.data());
    for (int i = 0; i < 3 * J; ++i) fkAxis(T, i / 3, i % 3, js.data());
    for (int j = 0; j < J; ++j) tangentLocal(T, js.data(), j, vs.data(), tan.data());
    for (int lvl = 1; lvl < T.numLevels; ++lvl)
      for (int k = T.levelStart[lvl]; k < T.levelStart[lvl + 1]; ++k) tangentCompose(T, js.data(), T.levelJoints[k], tan.data());
    const float* tg = rec.data() + size_t(b) * stride;
    const float* cw = cweights + size_t(b) * nc;
    for (int c = 0; c < nc; ++c) {
      const UnitDesc& u = T.units[c];
      const size_t o = size_t(b) * nc + c;
      float* gW = gradWeights ? gradWeights + o : nullptr;
      float* gO = gradOffsets ? gradOffsets + o * per : nullptr;
      float* gT = gradTargets ? gradTargets + o * per : nullptr;
      if (kind == 0) positionInputGradient(u, T.efs[u.ef], js.data(), tan.data(), tg + u.targetOff, cw[u.weightIdx], gW, gO, gT);
      else orientationInputGradient(u, T.efs[u.ef], js.data(), tan.data(), tg + u.targetOff, cw[u.weightIdx], gW, gO, gT);
    }
  }
  return MB2_OK;
}
