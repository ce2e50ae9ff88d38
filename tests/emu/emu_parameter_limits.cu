// TEST HARNESS ONLY — CPU lane-emulation of parameterLimitsKernel (mb2_character_parameter_limits_residual*_device) and of the clamp
// kernels of launchJointOp (mb2_character_apply_model_parameter_limits*_device), part of tests/emu/libmb2_emu.so.
//
// The character and its limit tables are made by the library's own makeCharacter, setParameterLimits and makeLimitTables; the kernels'
// own pass and element functions of ik_device.cuh (limitPasses, limitGradPasses, jointOpElement) then run with HostLanes, the lanes of
// each pass in sequence. The launch is planned by the library's planInstanceOp. It is not part of the product library and nothing in
// momentum_b200/ loads it.
#include <cstdint>
#include <vector>

#include "../../include/momentum_b200.h"
#include "../../momentum_b200/csrc/ik_device.cuh"
#include "../../momentum_b200/csrc/ik_plan.h"
#include "emu_error.h"
#include "emu_frame.h"

using namespace mb2;

namespace {
struct Emulated {
  HostCharacter h;
  HostLimitTables t;
  CharacterTables C;
  SkeletonTables S;
  LimitTables L;
};

// limits as mb2_parameter_limit arrays: types [K], weights [K], ints [K][4], floats [K][27]
int setUp(int32_t numJoints, const int32_t* parents, const float* offsets, const float* prerot, int32_t numParams, const int32_t* outer,
          const int32_t* inner, const float* vals, const float* ptOffsets, int32_t numLimits, const int32_t* types, const float* weights,
          const int32_t* ints, const float* floats, Emulated& e) {
  g_emuErr = makeCharacter(numJoints, parents, offsets, prerot, numParams, outer, inner, vals, ptOffsets, e.h);
  if (!g_emuErr.empty()) return MB2_ERR_INVALID_ARGUMENT;
  std::vector<mb2_parameter_limit> limits(numLimits > 0 ? size_t(numLimits) : 0);
  for (size_t k = 0; k < limits.size(); ++k) {
    limits[k].type = types[k];
    limits[k].weight = weights[k];
    for (int i = 0; i < 4; ++i) limits[k].i[i] = ints[4 * k + i];
    for (int i = 0; i < 27; ++i) limits[k].f[i] = floats[27 * k + i];
  }
  g_emuErr = setParameterLimits(e.h, numLimits, limits.data());
  if (!g_emuErr.empty()) return MB2_ERR_INVALID_ARGUMENT;
  e.t = makeLimitTables(e.h);
  if (!e.t.rejected.empty()) { g_emuErr = e.t.rejected; return MB2_ERR_INVALID_ARGUMENT; }
  e.C = hostCharacterTables(e.h);
  e.S = SkeletonTables{e.h.childStart.data(), e.h.children.data(), e.h.ptColStart.data(), e.h.ptColRows.data(), e.h.ptColVals.data(),
                       nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, e.t.paramClamp.data()};
  e.L = hostLimitTables(e.t);
  return MB2_OK;
}
} // namespace

#define MB2_EMU_CHARACTER                                                                                                                 \
  int32_t numJoints, const int32_t *parents, const float *offsets, const float *prerot, int32_t numParams, const int32_t *outer,         \
      const int32_t *inner, const float *vals, const float *ptOffsets, int32_t numLimits, const int32_t *types, const float *weights,   \
      const int32_t *ints, const float *floats
#define MB2_EMU_SETUP(e) setUp(numJoints, parents, offsets, prerot, numParams, outer, inner, vals, ptOffsets, numLimits, types, weights, ints, floats, e)

// character arrays as mb2_character_create takes them, then the limits; *rows = R and *ellipsoid = whether the FK runs, or the rejection
extern "C" int emu_parameter_limits_tables(MB2_EMU_CHARACTER, int32_t* rows, int32_t* ellipsoid) {
  Emulated e;
  if (MB2_EMU_SETUP(e) != MB2_OK) return MB2_ERR_INVALID_ARGUMENT;
  *rows = e.t.numRows;
  *ellipsoid = e.t.ellipsoid;
  return MB2_OK;
}

// forward: out [B][R] from theta [B][n]; backward: out [B][n] = dLoss / d theta from grad [B][R]
extern "C" int emu_parameter_limits(MB2_EMU_CHARACTER, int32_t backward, int32_t batch, const float* theta, const float* grad, float* out) {
  Emulated e;
  if (MB2_EMU_SETUP(e) != MB2_OK) return MB2_ERR_INVALID_ARGUMENT;
  const int n = e.C.numParams, R = e.t.numRows;
  const auto f = parameterLimitsFrame(e.C.numJoints, n, backward != 0, e.t.ellipsoid != 0);
  EmuFrame fr{f.floats};
  float *jp = fr.at(f.jp), *js = fr.at(f.js), *gjp = fr.at(f.gjp), *acc = fr.at(f.acc);
  for (int b = 0; b < batch; ++b) {
    if (R == 0) { // the library's launcher: nothing to write, a zero gradient
      if (backward) for (int p = 0; p < n; ++p) out[size_t(b) * n + p] = 0.f;
      continue;
    }
    const float* th = fr.load(f.th, theta + size_t(b) * n, n);
    if (!backward) {
      if (e.t.ellipsoid) limitPasses<true>(HostLanes{}, e.C, e.L, th, jp, js, out + size_t(b) * R);
      else limitPasses<false>(HostLanes{}, e.C, e.L, th, jp, js, out + size_t(b) * R);
    } else if (e.t.ellipsoid) {
      limitGradPasses<true>(HostLanes{}, e.C, e.S, e.L, th, jp, js, acc, gjp, grad + size_t(b) * R, out + size_t(b) * n);
    } else {
      limitGradPasses<false>(HostLanes{}, e.C, e.S, e.L, th, jp, js, acc, gjp, grad + size_t(b) * R, out + size_t(b) * n);
    }
  }
  return fr.check("parameterLimitsKernel");
}

// apply_model_param_limits: forward out [B][n] = the clamp of theta; backward out [B][n] from grad [B][n]
extern "C" int emu_apply_model_parameter_limits(MB2_EMU_CHARACTER, int32_t backward, int32_t batch, const float* theta, const float* grad, float* out) {
  Emulated e;
  if (MB2_EMU_SETUP(e) != MB2_OK) return MB2_ERR_INVALID_ARGUMENT;
  const long items = long(batch) * e.C.numParams;
  for (long i = 0; i < items; ++i) {
    if (backward) jointOpElement<kJointOpClampParameters, true>(e.C, e.S, i, theta, grad, out);
    else jointOpElement<kJointOpClampParameters, false>(e.C, e.S, i, theta, grad, out);
  }
  return MB2_OK;
}

// planInstanceOp of kInstanceOpParameterLimits: out = [W, groups per CTA, threads, smem bytes, 0], all zero when refused
extern "C" int emu_parameter_limits_launch(MB2_EMU_CHARACTER, int32_t backward, int64_t batch, int64_t smemBudget, int32_t numSms, int64_t out[5]) {
  Emulated e;
  if (MB2_EMU_SETUP(e) != MB2_OK) return MB2_ERR_INVALID_ARGUMENT;
  const InstanceLaunch l = planInstanceOp(e.C, int(e.h.children.size()), kInstanceOpParameterLimits, backward != 0, 0, long(batch),
                                          size_t(smemBudget), numSms, e.t.ellipsoid);
  launchWords(l, out);
  return MB2_OK;
}
