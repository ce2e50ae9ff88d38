// The launch of the per-instance kernels of the character operations (skeletonStateKernel, positionsKernel, inputGradientKernel): their
// shared memory per instance and per CTA, and the one rule that picks the warps per instance W and the instance groups per CTA from it.
// Host code shared by the library (ik_kernels.cu) and the CPU emulator (tests/emu), so that the launch a test sizes a rig for is the
// launch that runs.
#pragma once

#include <cstddef>
#include <cstdint>

#include "ik_types.h"

namespace mb2 {

constexpr int kSkelMaxWarps = 16; // warps per CTA, and instance groups per CTA (named barriers 1..groups when W > 1)

// words (4 bytes) of a table of `count` elements staged in shared memory: every table starts on a 16-byte boundary
MB2_HD size_t tableWords(size_t count, size_t elemBytes) { return (count * elemBytes + 15) / 16 * 4; }
// the character tables, staged first by every kernel that stages tables (stageCharacterTables)
inline size_t characterTableWords(const CharacterTables& C) {
  const size_t J = C.numJoints;
  size_t w = tableWords(J, 4) + tableWords(3 * J, 4) + tableWords(4 * J, 4);                 // parent, offset, prerot
  w += tableWords(7 * J + 1, 4) + tableWords(C.ptNnz, 4) * 2 + tableWords(7 * J, 4);         // ptOuter, ptInner, ptVals, ptOffsets
  w += tableWords(C.numLevels + 1, 4) + tableWords(J, 4);                                    // levelStart, levelJoints
  return w;
}

MB2_HD size_t skelAligned(size_t floats) { return (floats + 3) & ~size_t(3); } // 16-byte aligned regions
// skeletonStateKernel and positionsKernel, per instance: the input (theta [n], or the joint parameters [7 J]), joint states [J][17],
// backward: subtree sums [J][11] and, from theta, the joint-parameter gradient [7 J]
MB2_HD size_t skeletonStateSmemPerInstanceFloats(int J, int n, bool backward, bool joint) {
  size_t f = skelAligned(joint ? size_t(J) * kParametersPerJoint : size_t(n)) + skelAligned(size_t(J) * kJointStateStride);
  if (backward) f += skelAligned(size_t(J) * kSkelAccStride) + (joint ? 0 : skelAligned(size_t(J) * kParametersPerJoint));
  return f;
}
// their tables: the character's; backward: the children in CSR and, from theta, the ParameterTransform in CSC
inline size_t skeletonStateTableBytes(const CharacterTables& C, int numChildren, bool backward, bool joint) {
  size_t w = characterTableWords(C);
  if (backward) w += tableWords(size_t(C.numJoints) + 1, 4) + tableWords(size_t(numChildren), 4);
  if (backward && !joint) w += tableWords(size_t(C.numParams) + 1, 4) + tableWords(size_t(C.ptNnz), 4) * 2;
  return w * 4;
}
// positionsKernel's point tables: each point's joint; backward: the points by joint
inline size_t pointTableBytes(int numPoints, int J, bool backward) {
  size_t w = tableWords(size_t(numPoints), 4);
  if (backward) w += tableWords(size_t(J) + 1, 4) + tableWords(size_t(numPoints), 4);
  return w * 4;
}
// inputGradientKernel, per instance: theta [n], v [n], joint states [J][17], joint motions [J][7]; its tables are the character's
MB2_HD size_t inputGradientSmemPerInstanceFloats(int J, int n) {
  return 2 * skelAligned(size_t(n)) + skelAligned(size_t(J) * kJointStateStride) + skelAligned(size_t(J) * kTangentStride);
}

// What a per-instance kernel runs with; all zero when one instance does not fit next to the tables.
struct InstanceLaunch {
  int32_t warpsPerInstance{0}; // W: 1, 2, 4 or 8
  int32_t groupsPerCta{0};     // instances in flight per CTA
  int32_t threads{0};          // groupsPerCta x W x 32
  int64_t smemBytes{0};        // dynamic shared memory per CTA: the instances, the tables, 16 bytes of slack
  int32_t stagedPoints{0};     // positionsKernel: the point tables sit in shared memory after the character tables
};

// Instance groups per CTA before a small batch is spread: as many instances as fit next to the tables, at most kSkelMaxWarps; 0 when
// not even one fits.
int instanceGroupsFit(size_t perInstance, size_t tableBytes, size_t smemBudget);
// The rule: one warp per instance when at least eight fit, else as many warps per instance as kSkelMaxWarps allows, up to eight (fit
// 5-7: W = 2, 3-4: W = 4, 1-2: W = 8). A batch smaller than one group per SM is spread over the SMs.
InstanceLaunch planInstanceGroups(size_t perInstance, size_t tableBytes, long batch, size_t smemBudget, int numSms);

enum InstanceOp : int32_t { // the operations whose kernels run in this frame (mb2_character_get_instance_launch's op, then the solver's)
  kInstanceOpModelSkeletonState = 0, // skeletonStateKernel<kBackward, W, false>
  kInstanceOpJointSkeletonState = 1, // skeletonStateKernel<kBackward, W, true>
  kInstanceOpModelPositions = 2,     // positionsKernel<kBackward, W, false, kStagePoints>
  kInstanceOpJointPositions = 3,     // positionsKernel<kBackward, W, true, kStagePoints>
  kInstanceOpInputGradients = 4,     // inputGradientKernel<W> (forward only)
};
// The launch of one operation over `batch` instances of the character C (numChildren: entries of its children table), with numPoints
// points for the positions, whose tables are staged when that costs no instance per CTA.
InstanceLaunch planInstanceOp(const CharacterTables& C, int numChildren, int op, bool backward, int numPoints, long batch, size_t smemBudget,
                              int numSms);

} // namespace mb2
