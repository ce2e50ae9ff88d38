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
                              int numSms, bool limitsFk) {
  const int J = C.numJoints, n = C.numParams;
  const SkeletonTables S{}; // the lists read only the counts
  const PointTables P{numPoints};
  const bool joint = op == kInstanceOpJointSkeletonState || op == kInstanceOpJointPositions;
  size_t per = 0; // floats, then bytes per instance
  TableBytes tables, points;
  if (op == kInstanceOpInputGradients) { per = inputGradientFrame(J, n).floats; characterTableList(tables, C); }
  else if (op == kInstanceOpCollision) per = collisionFrame(numPoints, backward).floats;
  else if (op != kInstanceOpParameterLimits) { per = skeletonStateFrame(J, n, backward, joint).floats; skeletonTableList(tables, C, S, numChildren, backward, backward && !joint); }
  else { per = parameterLimitsFrame(J, n, backward, limitsFk).floats; skeletonTableList(tables, C, S, numChildren, backward && limitsFk, backward); }
  per *= sizeof(float);
  if (op != kInstanceOpModelPositions && op != kInstanceOpJointPositions) return planInstanceGroups(per, tables.bytes, batch, smemBudget, numSms);
  pointTableList(points, P, J, backward);
  const bool stage = instanceGroupsFit(per, tables.bytes + points.bytes, smemBudget) >= instanceGroupsFit(per, tables.bytes, smemBudget);
  InstanceLaunch l = planInstanceGroups(per, tables.bytes + (stage ? points.bytes : 0), batch, smemBudget, numSms);
  if (l.warpsPerInstance != 0) l.stagedPoints = stage;
  return l;
}

} // namespace mb2
