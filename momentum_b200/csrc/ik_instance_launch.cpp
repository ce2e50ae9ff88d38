#include "ik_instance_launch.h"

#include <algorithm>

namespace mb2 {

int instanceGroupsFit(size_t perInstance, size_t tableBytes, size_t smemBudget) {
  tableBytes += 16;
  if (perInstance == 0 || tableBytes + perInstance > smemBudget) return 0;
  return int(std::min<size_t>((smemBudget - tableBytes) / perInstance, kSkelMaxWarps));
}

InstanceLaunch planInstanceGroups(size_t perInstance, size_t tableBytes, long batch, size_t smemBudget, int numSms) {
  InstanceLaunch l;
  int groups = instanceGroupsFit(perInstance, tableBytes, smemBudget);
  if (groups == 0 || batch <= 0) return l;
  int W = 1;
  if (groups < 8)
    while (W < 8 && groups * W * 2 <= kSkelMaxWarps) W *= 2;
  const long sms = std::max(numSms, 1);
  if (batch < sms * groups) groups = int(std::max(1L, (batch + sms - 1) / sms));
  l.warpsPerInstance = W;
  l.groupsPerCta = groups;
  l.threads = groups * W * 32;
  l.smemBytes = int64_t(perInstance * groups + tableBytes + 16);
  return l;
}

InstanceLaunch planInstanceOp(const CharacterTables& C, int numChildren, int op, bool backward, int numPoints, long batch, size_t smemBudget,
                              int numSms) {
  if (op == kInstanceOpInputGradients)
    return planInstanceGroups(sizeof(float) * inputGradientSmemPerInstanceFloats(C.numJoints, C.numParams), characterTableWords(C) * 4, batch,
                              smemBudget, numSms);
  const bool joint = op == kInstanceOpJointSkeletonState || op == kInstanceOpJointPositions;
  const size_t per = sizeof(float) * skeletonStateSmemPerInstanceFloats(C.numJoints, C.numParams, backward, joint);
  const size_t tables = skeletonStateTableBytes(C, numChildren, backward, joint);
  if (op != kInstanceOpModelPositions && op != kInstanceOpJointPositions) return planInstanceGroups(per, tables, batch, smemBudget, numSms);
  const size_t points = pointTableBytes(numPoints, C.numJoints, backward);
  const bool stage = instanceGroupsFit(per, tables + points, smemBudget) >= instanceGroupsFit(per, tables, smemBudget);
  InstanceLaunch l = planInstanceGroups(per, tables + (stage ? points : 0), batch, smemBudget, numSms);
  if (l.warpsPerInstance != 0) l.stagedPoints = stage;
  return l;
}

} // namespace mb2
