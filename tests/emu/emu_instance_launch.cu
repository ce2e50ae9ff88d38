// TEST HARNESS ONLY — the launch planning of the per-instance character kernels (ik_instance_launch.cpp), as the library runs it, part
// of tests/emu/libmb2_emu.so. Tests size rigs for a launch variant with it before any device runs them. It is not part of the product
// library and nothing in momentum_b200/ loads it.
#include <cstdint>

#include "../../include/momentum_b200.h"
#include "../../momentum_b200/csrc/ik_plan.h"
#include "emu_error.h"
#include "emu_frame.h"

using namespace mb2;

// planInstanceGroups: out = [W, groups per CTA, threads, smem bytes, 0], all zero when refused
extern "C" int emu_plan_instance_groups(int64_t perInstance, int64_t tableBytes, int64_t batch, int64_t smemBudget, int32_t numSms, int64_t out[5]) {
  if (perInstance < 0 || tableBytes < 0 || smemBudget < 0 || out == nullptr) { g_emuErr = "bad argument"; return MB2_ERR_INVALID_ARGUMENT; }
  launchWords(planInstanceGroups(size_t(perInstance), size_t(tableBytes), long(batch), size_t(smemBudget), numSms), out);
  return MB2_OK;
}

// planInstanceOp for the character made from mb2_character_create's arguments: op as mb2_character_get_instance_launch takes it, 4 the
// input gradients; out = [W, groups per CTA, threads, smem bytes, staged point tables], all zero when refused
extern "C" int emu_instance_launch(int32_t numJoints, const int32_t* parents, const float* offsets, const float* prerot, int32_t numParams,
                                   const int32_t* outer, const int32_t* inner, const float* vals, const float* ptOffsets, int32_t op, int32_t backward,
                                   int64_t batch, int32_t numPoints, int64_t smemBudget, int32_t numSms, int64_t out[5]) {
  HostCharacter h;
  g_emuErr = makeCharacter(numJoints, parents, offsets, prerot, numParams, outer, inner, vals, ptOffsets, h);
  if (!g_emuErr.empty()) return MB2_ERR_INVALID_ARGUMENT;
  if (op < 0 || op > kInstanceOpInputGradients || numPoints < 0 || smemBudget < 0 || out == nullptr) { g_emuErr = "bad argument"; return MB2_ERR_INVALID_ARGUMENT; }
  launchWords(planInstanceOp(hostCharacterTables(h), int(h.children.size()), op, backward != 0, numPoints, long(batch), size_t(smemBudget), numSms), out);
  return MB2_OK;
}
