// The frame of the per-instance kernels of the character operations (skeletonStateKernel, positionsKernel, inputGradientKernel,
// parameterLimitsKernel, collisionKernel): the regions of an instance's shared memory, the tables each kernel stages, and the one rule
// that picks the warps per instance W and the instance groups per CTA from them.
// Shared by the library's kernels and launch planning (ik_kernels.cu, ik_instance_launch.cpp) and the CPU emulator (tests/emu), so that
// the frame and tables a kernel takes are those its launch was sized for and those the emulated passes run in.
#pragma once

#include <cstddef>
#include <cstdint>

#include "ik_types.h"

namespace mb2 {

constexpr int kSkelMaxWarps = 16; // warps per CTA, and instance groups per CTA (named barriers 1..groups when W > 1)

// ---- The regions of one instance group, in floats from the group's base: every region starts on a 16-byte boundary and an empty one
// takes no space. `floats` is the group's total; the CTA holds groupsPerCta of them, then the staged tables. The kernels size their groups
// with `floats`, whose sum keeps the grouping they have always compiled with: a regrouped sum moves ptxas's register allocation.
MB2_HD size_t skelAligned(size_t floats) { return (floats + 3) & ~size_t(3); }
// skeletonStateKernel and positionsKernel: the input (theta [n], or the joint parameters [7 J]), joint states [J][17]; backward: subtree
// sums [J][11] and, from theta, the joint-parameter gradient [7 J]
struct SkeletonStateFrame { size_t in, js, acc, gjp, floats; };
MB2_HD SkeletonStateFrame skeletonStateFrame(int J, int n, bool backward, bool joint) {
  const size_t in = skelAligned(joint ? size_t(J) * kParametersPerJoint : size_t(n)), js = skelAligned(size_t(J) * kJointStateStride);
  const size_t acc = backward ? skelAligned(size_t(J) * kSkelAccStride) : 0, gjp = backward && !joint ? skelAligned(size_t(J) * kParametersPerJoint) : 0;
  return {0, in, in + js, in + js + acc, in + js + (acc + gjp)};
}
// parameterLimitsKernel: theta [n], the joint parameters [7 J], with the FK (an Ellipsoid among the limits) the joint states [J][17];
// backward: the joint-parameter gradient [7 J] and, with the FK, the subtree sums [J][11]
struct ParameterLimitsFrame { size_t th, jp, js, gjp, acc, floats; };
MB2_HD ParameterLimitsFrame parameterLimitsFrame(int J, int n, bool backward, bool fk) {
  const size_t th = skelAligned(size_t(n)), jp = skelAligned(size_t(J) * kParametersPerJoint), js = fk ? skelAligned(size_t(J) * kJointStateStride) : 0;
  ParameterLimitsFrame f{0, th, th + jp, th + jp + js, th + jp + js + (backward ? jp : 0), th + jp};
  if (fk) f.floats += skelAligned(size_t(J) * kJointStateStride);
  if (backward) f.floats += skelAligned(size_t(J) * kParametersPerJoint) + (fk ? skelAligned(size_t(J) * kSkelAccStride) : 0);
  return f;
}
// collisionKernel: the world capsules [C][8]; backward: their gradients [C][8]. The skeleton states are read from global memory where a
// capsule needs its parent's.
struct CollisionFrame { size_t geo, cg, floats; };
MB2_HD CollisionFrame collisionFrame(int numCapsules, bool backward) {
  const size_t geo = skelAligned(size_t(numCapsules) * kCapsuleFloats);
  return {0, geo, geo * (backward ? 2 : 1)};
}
// inputGradientKernel: theta [n], v [n], joint states [J][17], joint motions [J][7]
struct InputGradientFrame { size_t th, vs, js, tan, floats; };
MB2_HD InputGradientFrame inputGradientFrame(int J, int n) {
  const size_t th = skelAligned(size_t(n)), js = skelAligned(size_t(J) * kJointStateStride), tan = skelAligned(size_t(J) * kTangentStride);
  return {0, th, 2 * th, 2 * th + js, 2 * th + js + tan};
}

// ---- The tables a kernel stages in shared memory once per CTA, as lists walked by a visitor v(table, count): on the device
// TableStager copies each table and points it at the copy, on the host TableBytes adds up the bytes the copies take. Every table
// starts on a 16-byte boundary.
MB2_HD size_t tableWords(size_t count, size_t elemBytes) { return (count * elemBytes + 15) / 16 * 4; }
struct TableBytes {
  size_t bytes = 0;
  template <class E> MB2_HD void operator()(const E*, size_t count) { bytes += 4 * tableWords(count, sizeof(E)); }
};
#if defined(__CUDACC__)
// The CTA's threads copy each table to `cursor` word by word and move the table's pointer there; the caller syncs the CTA before the
// copies are read.
struct TableStager {
  uint32_t* cursor;
  template <class E> __device__ __forceinline__ void operator()(const E*& table, size_t count) {
    static_assert(sizeof(E) % 4 == 0, "tables are staged word by word");
    const uint32_t* src = reinterpret_cast<const uint32_t*>(table);
    const size_t words = count * (sizeof(E) / 4);
    // eight loads in flight per thread (a word-by-word loop is a chain of global-load latencies: 23 of them for the 40 KB of cfg3)
    const int nt = int(blockDim.x);
    size_t i = threadIdx.x;
    for (; i + 7 * size_t(nt) < words; i += 8 * size_t(nt)) {
      uint32_t v[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) v[k] = src[i + size_t(k) * nt];
#pragma unroll
      for (int k = 0; k < 8; ++k) cursor[i + size_t(k) * nt] = v[k];
    }
    for (; i < words; i += nt) cursor[i] = src[i];
    table = reinterpret_cast<const E*>(cursor);
    cursor += tableWords(count, sizeof(E));
  }
};
#endif

// The character's tables, first in every kernel that stages tables (C: CharacterTables or FunctionTables)
template <class V, class C>
MB2_HD void characterTableList(V& v, C& T) {
  const size_t J = T.numJoints;
  v(T.parent, J); v(T.offset, 3 * J); v(T.prerot, 4 * J);
  v(T.ptOuter, 7 * J + 1); v(T.ptInner, T.ptNnz); v(T.ptVals, T.ptNnz); v(T.ptOffsets, 7 * J);
  v(T.levelStart, T.numLevels + 1); v(T.levelJoints, J);
}
// skeletonStateKernel, positionsKernel and parameterLimitsKernel: the character's; then for a backward the children in CSR where it
// folds subtree sums (`children`), and the ParameterTransform in CSC where it ends in model parameters (`csc`)
template <class V, class C, class S>
MB2_HD void skeletonTableList(V& v, C& T, S& Sk, int numChildren, bool children, bool csc) {
  const int J = T.numJoints, n = T.numParams;
  characterTableList(v, T);
  if (children) { v(Sk.childStart, size_t(J) + 1); v(Sk.children, numChildren); }
  if (csc) { v(Sk.ptColStart, n + 1); v(Sk.ptColRows, T.ptNnz); v(Sk.ptColVals, T.ptNnz); }
}
// positionsKernel's point tables, after skeletonTableList's when staged: each point's joint; backward: the points by joint
template <class V, class P>
MB2_HD void pointTableList(V& v, P& Pt, int J, bool backward) {
  v(Pt.parent, Pt.numPoints);
  if (backward) { v(Pt.pointStart, size_t(J) + 1); v(Pt.pointIndex, Pt.numPoints); }
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
  kInstanceOpParameterLimits = 5,    // parameterLimitsKernel<kBackward, W, kEllipsoid>
  kInstanceOpCollision = 6,          // collisionKernel<kBackward, W>
};
// The launch of one operation over `batch` instances of the character C (numChildren: entries of its children table), with numPoints
// points for the positions (for the collision: numPoints capsules), whose tables are staged when that costs no instance per CTA. limitsFk: for the parameter limits, that the
// character has an Ellipsoid limit, so the kernel runs the FK passes (LimitTables::ellipsoid).
InstanceLaunch planInstanceOp(const CharacterTables& C, int numChildren, int op, bool backward, int numPoints, long batch, size_t smemBudget,
                              int numSms, bool limitsFk = false);

} // namespace mb2
