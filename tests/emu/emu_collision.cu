// TEST HARNESS ONLY — CPU lane-emulation of collisionKernel (mb2_character_collision_residual*_device), part of tests/emu/libmb2_emu.so.
//
// The character and its collision tables are made by the library's own makeCharacter and makeCollision; the kernel's own pass functions
// of ik_device.cuh (collisionPasses, collisionGradPasses) then run with HostLanes, the lanes of each pass in sequence. The launch is
// planned by the library's planInstanceOp. It is not part of the product library and nothing in momentum_b200/ loads it.
#include <cstdint>

#include "../../include/momentum_b200.h"
#include "../../momentum_b200/csrc/ik_device.cuh"
#include "../../momentum_b200/csrc/ik_plan.h"
#include "emu_error.h"
#include "emu_frame.h"

using namespace mb2;

namespace {
struct Emulated {
  HostCharacter h;
  HostCollision c;
  CollisionTables L;
};

int setUp(int32_t numJoints, const int32_t* parents, const float* offsets, const float* prerot, int32_t numParams, const int32_t* outer,
          const int32_t* inner, const float* vals, const float* ptOffsets, int32_t count, const mb2_tapered_capsule* capsules, Emulated& e) {
  g_emuErr = makeCharacter(numJoints, parents, offsets, prerot, numParams, outer, inner, vals, ptOffsets, e.h);
  if (!g_emuErr.empty()) return MB2_ERR_INVALID_ARGUMENT;
  g_emuErr = makeCollision(e.h, count, capsules, e.c);
  if (!g_emuErr.empty()) return MB2_ERR_INVALID_ARGUMENT;
  e.L = hostCollisionTables(e.c);
  return MB2_OK;
}
} // namespace

#define MB2_EMU_CHARACTER                                                                                                                 \
  int32_t numJoints, const int32_t *parents, const float *offsets, const float *prerot, int32_t numParams, const int32_t *outer,         \
      const int32_t *inner, const float *vals, const float *ptOffsets, int32_t count, const mb2_tapered_capsule *capsules
#define MB2_EMU_SETUP(e) setUp(numJoints, parents, offsets, prerot, numParams, outer, inner, vals, ptOffsets, count, capsules, e)

// character arrays as mb2_character_create takes them, then the capsules; *numPairs = P and, when pairs is set, pairs [P][2]
extern "C" int emu_collision_pairs(MB2_EMU_CHARACTER, int32_t* numPairs, int32_t* pairs) {
  Emulated e;
  if (MB2_EMU_SETUP(e) != MB2_OK) return MB2_ERR_INVALID_ARGUMENT;
  *numPairs = e.c.numPairs();
  if (pairs) for (size_t k = 0; k < e.c.pairs.size(); ++k) pairs[k] = e.c.pairs[k];
  return MB2_OK;
}

// forward: out [B][P] from states [B][J][8]; backward: out [B][J][8] = dLoss / d state from grad [B][P]
extern "C" int emu_collision(MB2_EMU_CHARACTER, int32_t backward, int32_t batch, const float* state, const float* grad, float* out) {
  Emulated e;
  if (MB2_EMU_SETUP(e) != MB2_OK) return MB2_ERR_INVALID_ARGUMENT;
  const int J = e.h.numJoints, P = e.c.numPairs();
  const auto f = collisionFrame(int(e.c.capsules.size()), backward != 0);
  EmuFrame fr{f.floats};
  for (int b = 0; b < batch; ++b) {
    const float* st = state + size_t(b) * J * 8;
    if (P == 0) { // the library's launcher: nothing to write, a zero gradient
      if (backward) for (int i = 0; i < J * 8; ++i) out[size_t(b) * J * 8 + i] = 0.f;
      continue;
    }
    if (!backward) collisionPasses(HostLanes{}, e.L, st, fr.at(f.geo), out + size_t(b) * P);
    else collisionGradPasses(HostLanes{}, e.L, J, st, fr.at(f.geo), fr.at(f.cg), grad + size_t(b) * P, out + size_t(b) * J * 8);
  }
  return fr.check("collisionKernel");
}

// One pair of world capsules A, B [8] (origin, direction, r0, r1) through capsuleContact<float>: out = [hit, s, t, dist, overlap, sForm,
// tForm]; with a contact, gA and gB [8] = d overlap / d A, d B (capsuleContactGrad), else zero
extern "C" void emu_capsule_contact(const float* A, const float* B, float* out, float* gA, float* gB) {
  const CapsuleContact<float> c = capsuleContact(A, B);
  out[0] = c.hit ? 1.f : 0.f;
  out[1] = c.s; out[2] = c.t; out[3] = c.dist; out[4] = c.overlap;
  out[5] = float(c.sForm); out[6] = float(c.tForm);
  for (int i = 0; i < kCapsuleFloats; ++i) gA[i] = gB[i] = 0.f;
  if (c.hit) capsuleContactGrad(A, B, c, 1.f, gA, gB);
}

// planInstanceOp of kInstanceOpCollision: out = [W, groups per CTA, threads, smem bytes, 0], all zero when refused
extern "C" int emu_collision_launch(MB2_EMU_CHARACTER, int32_t backward, int64_t batch, int64_t smemBudget, int32_t numSms, int64_t out[5]) {
  Emulated e;
  if (MB2_EMU_SETUP(e) != MB2_OK) return MB2_ERR_INVALID_ARGUMENT;
  const InstanceLaunch l = planInstanceOp(hostCharacterTables(e.h), int(e.h.children.size()), kInstanceOpCollision, backward != 0,
                                          int(e.c.capsules.size()), long(batch), size_t(smemBudget), numSms);
  launchWords(l, out);
  return MB2_OK;
}
