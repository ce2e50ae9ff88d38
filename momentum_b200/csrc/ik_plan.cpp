#include "ik_plan.h"

#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstring>
#include <map>

namespace mb2 {

std::string HostCharacter::validate() const {
  const int J = numJoints;
  if (J <= 0) return "skeleton has no joints";
  if (numParams <= 0 || numParams > 2048) return "number of model parameters must be in [1, 2048] (ParameterSet is bitset<2048>)";
  if (int(parent.size()) != J || int(offset.size()) != 3 * J || int(prerot.size()) != 4 * J) return "joint array sizes do not match the joint count";
  for (int j = 0; j < J; ++j)
    if (parent[j] >= j || parent[j] < -1) return "skeleton is not topologically sorted: parent index must precede child (skeleton.h:23-24)";
  const int rows = J * kParametersPerJoint;
  if (int(ptOuter.size()) != rows + 1 || int(ptOffsets.size()) != rows) return "parameter transform must have 7 * numJoints rows";
  if (ptOuter[0] != 0) return "parameter transform outer index must start at 0";
  for (int r = 0; r < rows; ++r)
    if (ptOuter[r + 1] < ptOuter[r]) return "parameter transform outer index must be non-decreasing";
  if (ptOuter[rows] != int(ptInner.size()) || ptInner.size() != ptVals.size()) return "parameter transform nnz mismatch";
  for (int c : ptInner)
    if (c < 0 || c >= numParams) return "parameter transform column out of range";
  return "";
}

void HostCharacter::buildLevels() {
  std::vector<int> depth(numJoints, 0);
  int maxDepth = 0;
  for (int j = 0; j < numJoints; ++j) {
    depth[j] = parent[j] < 0 ? 0 : depth[parent[j]] + 1;
    maxDepth = std::max(maxDepth, depth[j]);
  }
  levelStart.assign(maxDepth + 2, 0);
  for (int j = 0; j < numJoints; ++j) levelStart[depth[j] + 1]++;
  for (int l = 0; l <= maxDepth; ++l) levelStart[l + 1] += levelStart[l];
  levelJoints.resize(numJoints);
  std::vector<int> cursor(levelStart.begin(), levelStart.end() - 1);
  for (int j = 0; j < numJoints; ++j) levelJoints[cursor[depth[j]]++] = j;
}

void HostCharacter::buildBackwardTables() {
  childStart.assign(numJoints + 1, 0);
  for (int j = 0; j < numJoints; ++j)
    if (parent[j] >= 0) childStart[parent[j] + 1]++;
  for (int j = 0; j < numJoints; ++j) childStart[j + 1] += childStart[j];
  children.resize(childStart[numJoints]);
  std::vector<int32_t> cursor(childStart.begin(), childStart.end() - 1);
  for (int j = 0; j < numJoints; ++j) // ascending j: each joint's children in increasing index order
    if (parent[j] >= 0) children[cursor[parent[j]]++] = j;
  const int rows = numJoints * kParametersPerJoint;
  ptColStart.assign(numParams + 1, 0);
  for (int c : ptInner) ptColStart[c + 1]++;
  for (int p = 0; p < numParams; ++p) ptColStart[p + 1] += ptColStart[p];
  ptColRows.resize(ptInner.size());
  ptColVals.resize(ptInner.size());
  cursor.assign(ptColStart.begin(), ptColStart.end() - 1);
  for (int r = 0; r < rows; ++r) // ascending rows: each column's rows in increasing order
    for (int k = ptOuter[r]; k < ptOuter[r + 1]; ++k) {
      const int at = cursor[ptInner[k]]++;
      ptColRows[at] = r;
      ptColVals[at] = ptVals[k];
    }
}

std::vector<uint8_t> HostCharacter::computeActiveJointParams(const std::vector<uint8_t>& enabled) const {
  std::vector<uint8_t> r(size_t(numJoints) * kParametersPerJoint, 0);
  for (int row = 0; row < numJoints * kParametersPerJoint; ++row)
    for (int k = ptOuter[row]; k < ptOuter[row + 1]; ++k)
      if (enabled[ptInner[k]]) r[row] = 1;
  return r;
}

int32_t jacobianBlockSize(const HostCharacter& ch, const HostErrorFunction& ef) {
  switch (ef.kind) {
    case 0: return 3 * ef.numConstraints();
    case 1:
    case 2: return 9 * ef.numConstraints();
    case 3: {
      int n = 0;
      for (int j = 0; j < ch.numJoints; ++j) n += (ef.posW[j] != 0.f || ef.rotW[j] != 0.f) ? 1 : 0;
      return n * (ef.rotationErrorType == 1 ? 6 : 12);
    }
    case 5: return ef.numConstraints(); // joint_error_function-inl.h:300-302 with FuncDim = 1
    case 6: { // model_parameters_error_function.cpp:93-95
      int n = 0;
      for (float w : ef.paramWeights) n += w > 0.f ? 1 : 0;
      return n;
    }
    case 4: {
      int n = 0;
      for (const auto& l : ch.limits) {
        if (l.type == 2) continue; // MinMaxJointPassive
        n += (l.type == 5) ? 3 : 1;
      }
      return n;
    }
  }
  return 0;
}

std::string makeCharacter(int32_t numJoints, const int32_t* parents, const float* offsets, const float* prerot, int32_t numParams, const int32_t* outer,
                          const int32_t* inner, const float* vals, const float* ptOffsets, HostCharacter& out) {
  if (!(parents && offsets && prerot && outer && ptOffsets)) return "null argument";
  if (!(numJoints > 0 && numParams > 0)) return "numJoints and numModelParameters must be positive";
  const int J = numJoints;
  out = HostCharacter();
  out.numJoints = J;
  out.numParams = numParams;
  out.parent.assign(parents, parents + J);
  out.offset.assign(offsets, offsets + 3 * J);
  out.prerot.assign(prerot, prerot + 4 * J);
  out.ptOuter.assign(outer, outer + 7 * J + 1);
  const int nnz = outer[7 * J];
  if (!(nnz >= 0 && (nnz == 0 || (inner && vals)))) return "parameter transform nnz invalid";
  out.ptInner.assign(inner, inner + nnz);
  out.ptVals.assign(vals, vals + nnz);
  out.ptOffsets.assign(ptOffsets, ptOffsets + 7 * J);
  const std::string err = out.validate();
  if (!err.empty()) return err;
  out.buildLevels();
  out.buildBackwardTables();
  return "";
}

std::string makeSkinning(const HostCharacter& ch, int32_t numVertices, const float* restVertices, const int32_t* skinIndex, const float* skinWeight,
                         const float* inverseBindPose, HostSkinning& out) {
  if (!(restVertices && skinIndex && skinWeight && inverseBindPose)) return "skinning: null argument";
  if (numVertices < 1) return "skinning: the mesh must have at least one vertex";
  const int J = ch.numJoints, V = numVertices;
  for (size_t k = 0; k < size_t(V) * 3; ++k)
    if (!std::isfinite(restVertices[k])) return "skinning: rest vertices must be finite";
  for (size_t k = 0; k < size_t(J) * kSkinIbpStride; ++k)
    if (!std::isfinite(inverseBindPose[k])) return "skinning: inverse bind poses must be finite";
  HostSkinning s;
  s.numVertices = V;
  s.restVertices.assign(restVertices, restVertices + size_t(V) * 3);
  s.inverseBindPose.assign(inverseBindPose, inverseBindPose + size_t(J) * kSkinIbpStride);
  s.vertStart.assign(V + 1, 0);
  for (int v = 0; v < V; ++v) {
    for (int k = 0; k < kSkinMaxInfluences; ++k) {
      const size_t at = size_t(v) * kSkinMaxInfluences + k;
      if (skinWeight[at] == 0.f) break; // linear_skinning.cpp:76-80: the slots after it are not read, whatever they hold
      if (!std::isfinite(skinWeight[at])) return "skinning: skin weights must be finite";
      if (skinIndex[at] < 0 || skinIndex[at] >= J) return "skinning: skin index out of range [0, numJoints)";
      s.vertJoint.push_back(skinIndex[at]);
      s.vertWeight.push_back(skinWeight[at]);
    }
    s.vertStart[v + 1] = int32_t(s.vertJoint.size());
  }
  // by joint: a counting sort over ascending vertices keeps each joint's list in vertex (then slot) order
  s.jointStart.assign(J + 1, 0);
  for (int j : s.vertJoint) s.jointStart[j + 1]++;
  for (int j = 0; j < J; ++j) s.jointStart[j + 1] += s.jointStart[j];
  s.infVertex.resize(s.vertJoint.size());
  s.infWeight.resize(s.vertJoint.size());
  std::vector<int32_t> cursor(s.jointStart.begin(), s.jointStart.end() - 1);
  for (int v = 0; v < V; ++v)
    for (int k = s.vertStart[v]; k < s.vertStart[v + 1]; ++k) {
      const int at = cursor[s.vertJoint[k]]++;
      s.infVertex[at] = v;
      s.infWeight[at] = s.vertWeight[k];
    }
  s.jointSegStart.assign(J + 1, 0);
  for (int j = 0; j < J; ++j) {
    for (int b = s.jointStart[j]; b < s.jointStart[j + 1]; b += kSkinSegment) {
      s.segStart.push_back(b);
      s.segJoint.push_back(j);
    }
    s.jointSegStart[j + 1] = int32_t(s.segJoint.size());
  }
  s.segStart.push_back(s.jointStart[J]);
  out = std::move(s);
  return "";
}

CharacterTables hostCharacterTables(const HostCharacter& ch) {
  CharacterTables C{};
  C.numJoints = ch.numJoints;
  C.numParams = ch.numParams;
  C.parent = ch.parent.data();
  C.offset = ch.offset.data();
  C.prerot = ch.prerot.data();
  C.ptOuter = ch.ptOuter.data();
  C.ptInner = ch.ptInner.data();
  C.ptVals = ch.ptVals.data();
  C.ptOffsets = ch.ptOffsets.data();
  C.numLevels = int32_t(ch.levelStart.size()) - 1;
  C.ptNnz = int32_t(ch.ptInner.size());
  C.levelStart = ch.levelStart.data();
  C.levelJoints = ch.levelJoints.data();
  return C;
}

std::string setParameterLimits(HostCharacter& ch, int32_t count, const mb2_parameter_limit* limits) {
  if (!(count >= 0 && (count == 0 || limits))) return "invalid limits";
  ch.limits.clear();
  for (int i = 0; i < count; ++i) {
    HostLimit l;
    l.type = limits[i].type;
    l.weight = limits[i].weight;
    std::memcpy(l.i, limits[i].i, sizeof(l.i));
    std::memcpy(l.f, limits[i].f, sizeof(l.f));
    if (!(l.type >= 0 && l.type <= 6)) return "Unknown parameter type for joint limit";
    ch.limits.push_back(l);
  }
  return "";
}

// What Position, Plane and Orientation blocks share: the generalized loss, and the parent joint and weight of each constraint.
static std::string jointConstraints(const HostCharacter& ch, int32_t kind, float weight, float alpha, float c, int32_t nc, const int32_t* parents,
                                    const float* weights, HostErrorFunction& ef) {
  if (!(c > 0.f)) return "Parameter c should be positive"; // generalized_loss.cpp:83
  ef.kind = kind;
  ef.weight = weight;
  ef.lossAlpha = alpha;
  ef.lossC = c;
  ef.parents.assign(parents, parents + nc);
  for (int p : ef.parents)
    if (p < 0 || p >= ch.numJoints) return "constraint parent joint out of range";
  ef.weights.assign(weights, weights + nc);
  return "";
}

std::string positionErrorFunction(const HostCharacter& ch, float weight, float alpha, float c, int32_t nc, const int32_t* parents, const float* offsets,
                                  const float* weights, HostErrorFunction& ef) {
  if (!(nc >= 0 && (nc == 0 || (parents && offsets && weights)))) return "invalid position constraints";
  ef.offsets.assign(offsets, offsets + 3 * size_t(nc));
  ef.targetSize = 3 * nc;
  return jointConstraints(ch, 0, weight, alpha, c, nc, parents, weights, ef);
}

std::string instancedPositionErrorFunction(const HostCharacter& ch, float weight, float alpha, float c, int32_t nc, const int32_t* parents, const float* weights,
                                           HostErrorFunction& ef) {
  if (!(nc >= 0 && (nc == 0 || (parents && weights)))) return "invalid position constraints";
  ef.instanceOffsets = true;
  ef.offsets.assign(3 * size_t(nc), 0.f);
  ef.targetSize = 6 * nc;
  return jointConstraints(ch, 0, weight, alpha, c, nc, parents, weights, ef);
}

std::string planeErrorFunction(const HostCharacter& ch, float weight, float alpha, float c, int32_t above, int32_t nc, const int32_t* parents, const float* offsets,
                               const float* weights, HostErrorFunction& ef) {
  if (!(nc >= 0 && (nc == 0 || (parents && offsets && weights)))) return "invalid plane constraints";
  ef.halfPlane = above != 0;
  ef.offsets.assign(offsets, offsets + 3 * size_t(nc));
  ef.targetSize = 4 * nc;
  return jointConstraints(ch, 5, weight, alpha, c, nc, parents, weights, ef);
}

std::string modelParametersErrorFunction(const HostCharacter& ch, float weight, const float* targetWeights, HostErrorFunction& ef) {
  if (targetWeights == nullptr) return "invalid model-parameter weights";
  ef.kind = 6;
  ef.weight = weight;
  ef.paramWeights.assign(targetWeights, targetWeights + ch.numParams);
  ef.targetSize = ch.numParams;
  return "";
}

std::string orientationErrorFunction(const HostCharacter& ch, float weight, float alpha, float c, int32_t rotDiff, int32_t nc, const int32_t* parents,
                                     const float* offsets, const float* weights, HostErrorFunction& ef) {
  if (!(nc >= 0 && (nc == 0 || (parents && offsets && weights)))) return "invalid orientation constraints";
  ef.offsets.assign(offsets, offsets + 4 * size_t(nc));
  for (int i = 0; i < nc; ++i) { // OrientationDataT ctor: offset(inOffset.normalized()) (orientation_error_function.h:33-35)
    float* q = &ef.offsets[4 * size_t(i)];
    const float nrm = std::sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
    for (int k = 0; k < 4; ++k) q[k] /= nrm;
  }
  ef.targetSize = 4 * nc;
  return jointConstraints(ch, rotDiff ? 2 : 1, weight, alpha, c, nc, parents, weights, ef);
}

std::string instancedOrientationErrorFunction(const HostCharacter& ch, float weight, float alpha, float c, int32_t rotDiff, int32_t nc, const int32_t* parents,
                                              const float* weights, HostErrorFunction& ef) {
  if (!(nc >= 0 && (nc == 0 || (parents && weights)))) return "invalid orientation constraints";
  ef.instanceOffsets = true;
  ef.offsets.assign(4 * size_t(nc), 0.f);
  ef.targetSize = 8 * nc;
  return jointConstraints(ch, rotDiff ? 2 : 1, weight, alpha, c, nc, parents, weights, ef);
}

std::string stateErrorFunction(const HostCharacter& ch, float weight, int32_t rotationErrorType, float posWgt, float rotWgt, const float* posW, const float* rotW,
                               HostErrorFunction& ef) {
  if (!(posW && rotW)) return "invalid state error function";
  if (!(rotationErrorType == 0 || rotationErrorType == 1)) return "unknown rotation error type";
  ef.kind = 3;
  ef.weight = weight;
  ef.rotationErrorType = rotationErrorType;
  ef.posWgt = posWgt;
  ef.rotWgt = rotWgt;
  ef.posW.assign(posW, posW + ch.numJoints);
  ef.rotW.assign(rotW, rotW + ch.numJoints);
  ef.targetSize = 8 * ch.numJoints;
  return "";
}

std::string limitErrorFunction(float weight, float alpha, float c, HostErrorFunction& ef) {
  if (!(c > 0.f)) return "Parameter c should be positive";
  ef.kind = 4;
  ef.weight = weight;
  ef.lossAlpha = alpha;
  ef.lossC = c;
  ef.targetSize = 0;
  return "";
}

std::string HostFunction::add(const HostErrorFunction& block, int32_t* index) {
  const bool hasWeights = block.kind <= 2 || block.kind == 5;
  if (hasWeights && weightsPerInstance) return "add all error functions before setting per-instance constraint weights";
  HostErrorFunction ef = block;
  ef.targetOff = targetStride;
  ef.weightOff = numWeights;
  targetStride += ef.targetSize;
  if (hasWeights) {
    numWeights += ef.numConstraints();
    weights.insert(weights.end(), ef.weights.begin(), ef.weights.end());
  }
  efs.push_back(std::move(ef));
  if (index) *index = int32_t(efs.size()) - 1;
  return "";
}

int32_t HostFunction::actualParameters() const {
  int32_t ap = 0;
  for (size_t i = 0; i < enabled.size(); ++i)
    if (enabled[i]) ap = int32_t(i) + 1;
  return ap;
}

static int32_t unpaddedRows(const HostCharacter& ch, const std::vector<HostErrorFunction>& efs) {
  int32_t total = 0;
  for (const auto& ef : efs)
    if (ef.weight > 0.f) total += jacobianBlockSize(ch, ef);
  return total;
}
int32_t HostFunction::jacobianRows(const HostCharacter& ch) const { return (unpaddedRows(ch, efs) + 7) / 8 * 8; }
int32_t HostFunction::jacobianStride(const HostCharacter& ch) const { return std::max(32, (unpaddedRows(ch, efs) + 31) / 32 * 32); }

static EfDesc makeEfDesc(const HostErrorFunction& ef) {
  EfDesc d{};
  d.weight = ef.weight;
  d.alpha = ef.lossAlpha;
  d.invC2 = 1.f / (ef.lossC * ef.lossC);
  // GeneralizedLossT ctor snapping (math/generalized_loss.cpp:81-101), kEps = 1e-9
  const float kEps = 1e-9f;
  const float a = ef.lossAlpha;
  if (a >= 2.f - kEps && a <= 2.f + kEps) d.lossType = kLossL2;
  else if (a >= 1.f - kEps && a <= 1.f + kEps) d.lossType = kLossL1;
  else if (a >= 0.f - kEps && a <= 0.f + kEps) d.lossType = kLossCauchy;
  else if (a == -FLT_MAX || (std::isinf(a) && a < 0)) d.lossType = kLossWelsch;
  else d.lossType = kLossGeneral;
  d.posWgt = ef.posWgt;
  d.rotWgt = ef.rotWgt;
  d.kind = ef.kind;
  d.halfPlane = ef.halfPlane ? 1 : 0;
  return d;
}

namespace {
struct CellBuilder {
  // column -> contributions in walk order
  std::map<int, std::vector<ContribDesc>> m;
  void add(const HostCharacter& ch, int jointParam, int joint, int dof, const std::vector<uint8_t>* enabledGate) {
    for (int k = ch.ptOuter[jointParam]; k < ch.ptOuter[jointParam + 1]; ++k) {
      const int col = ch.ptInner[k];
      if (enabledGate != nullptr && !(*enabledGate)[col]) continue;
      ContribDesc c;
      c.joint = uint16_t(joint);
      c.dof = uint16_t(dof);
      c.coef = ch.ptVals[k];
      m[col].push_back(c);
    }
  }
};
} // namespace

std::string buildPlan(const HostCharacter& ch, const std::vector<HostErrorFunction>& efs, const std::vector<uint8_t>& enabled, bool compact, Plan& out,
                      const std::vector<int32_t>* columnOrder, bool alignRowGroups) {
  out = Plan();
  out.compact = compact;
  const int n = ch.numParams;
  if (int(enabled.size()) != n) return "enabled parameter set size mismatch";
  for (int i = 0; i < n; ++i)
    if (enabled[i]) { out.actualParameters = i + 1; out.enabledList.push_back(i); }
  const std::vector<uint8_t> active = ch.computeActiveJointParams(enabled);
  std::vector<int> colMap(n, -1); // model parameter -> device column
  if (compact) {
    out.deviceCols = out.enabledList;
    if (columnOrder != nullptr) out.deviceCols = *columnOrder; // may hold -1 entries: all-zero alignment columns (ik_chol_sched.h)
    size_t listed = 0;
    for (size_t a = 0; a < out.deviceCols.size(); ++a) {
      const int p = out.deviceCols[a];
      if (p == -1 && columnOrder != nullptr) continue;
      if (p < 0 || p >= n || !enabled[p] || colMap[p] >= 0) return "column order must list every enabled parameter once";
      colMap[p] = int(a);
      ++listed;
    }
    if (listed != out.enabledList.size()) return "column order must list every enabled parameter once";
    out.numCols = int(out.deviceCols.size());
  } else {
    for (int i = 0; i < n; ++i) colMap[i] = i;
    out.numCols = n;
    out.deviceCols.resize(n);
    for (int i = 0; i < n; ++i) out.deviceCols[i] = i;
  }

  int row = 0, rec = 0;
  auto flushCells = [&](int unitIndex, CellBuilder& cb) {
    for (auto& kv : cb.m) {
      if (colMap[kv.first] < 0) continue; // column of a disabled parameter: not held on the device
      CellDesc c{};
      c.unit = uint16_t(unitIndex);
      c.col = uint16_t(colMap[kv.first]);
      c.contribBegin = uint32_t(out.contribs.size());
      c.contribCount = uint16_t(kv.second.size());
      c.coef = 0.f;
      out.contribs.insert(out.contribs.end(), kv.second.begin(), kv.second.end());
      out.cells.push_back(c);
    }
  };
  auto staticCell = [&](int unitIndex, int col, float coef) {
    if (colMap[col] < 0) return;
    CellDesc c{};
    c.unit = uint16_t(unitIndex);
    c.col = uint16_t(colMap[col]);
    c.contribBegin = 0;
    c.contribCount = 0;
    c.coef = coef;
    out.cells.push_back(c);
  };

  for (size_t e = 0; e < efs.size(); ++e) {
    const HostErrorFunction& ef = efs[e];
    out.efs.push_back(makeEfDesc(ef));
    if (!(ef.weight > 0.f)) continue; // skeleton_solver_function.cpp:228-230: disabled block has no rows
    if (ef.kind <= 2) {
      const bool isPos = ef.kind == 0;
      const int per = isPos ? 3 : 4;
      for (int c = 0; c < ef.numConstraints(); ++c) {
        if (ef.parents[c] < 0 || ef.parents[c] >= ch.numJoints) return "constraint parent joint out of range";
        UnitDesc u{};
        u.kind = isPos ? kUnitPosition : (ef.kind == 1 ? kUnitOrientation : kUnitOrientationRotDiff);
        u.ef = int32_t(e);
        u.joint = ef.parents[c];
        if (alignRowGroups) row = (row + 3) & ~3;
        u.row0 = row;
        u.numRows = isPos ? 3 : 9;
        const bool instanced = ef.instanceOffsets; // record per constraint: target, then its offset
        u.targetOff = ef.targetOff + (instanced ? 2 * per : per) * c;
        u.weightIdx = ef.weightOff + c;
        u.recOff = rec;
        u.extra = -1;
        u.pad[2] = instanced ? 1 : 0;
        if (!instanced) for (int k = 0; k < per; ++k) u.f[k] = ef.offsets[size_t(per) * c + k];
        const int ui = int(out.units.size());
        out.units.push_back(u);
        row += u.numRows;
        if (alignRowGroups) row = (row + 3) & ~3; // a multi-row unit owns its row quads (one-row units pack among themselves)
        rec += isPos ? 4 : 10;
        CellBuilder cb;
        for (int jnt = ef.parents[c]; jnt >= 0; jnt = ch.parent[jnt]) { // joint_error_function-inl.h:229-294
          const int pb = jnt * kParametersPerJoint;
          if (isPos)
            for (int d = 0; d < 3; ++d)
              if (active[pb + d]) cb.add(ch, pb + d, jnt, d, &enabled);
          for (int d = 0; d < 3; ++d)
            if (active[pb + 3 + d]) cb.add(ch, pb + 3 + d, jnt, 3 + d, &enabled);
          if (isPos && active[pb + 6]) cb.add(ch, pb + 6, jnt, 6, &enabled);
        }
        flushCells(ui, cb);
      }
    } else if (ef.kind == 3) {
      const bool lm = ef.rotationErrorType == 1;
      for (int i = 0; i < ch.numJoints; ++i) {
        if (ef.rotW[i] == 0.f && ef.posW[i] == 0.f) continue; // state_error_function.cpp:424-426
        UnitDesc u{};
        u.kind = lm ? kUnitStateLogMap : kUnitStateMatrix;
        u.ef = int32_t(e);
        u.joint = i;
        if (alignRowGroups) row = (row + 3) & ~3;
        u.row0 = row;
        u.numRows = lm ? 6 : 12;
        u.targetOff = ef.targetOff + 8 * i;
        u.weightIdx = -1;
        u.recOff = rec;
        u.extra = -1;
        u.f[0] = ef.posW[i];
        u.f[1] = ef.rotW[i];
        const int ui = int(out.units.size());
        out.units.push_back(u);
        row += u.numRows;
        if (alignRowGroups) row = (row + 3) & ~3;
        rec += lm ? 14 : 2;
        CellBuilder cb;
        for (int jnt = i; jnt >= 0; jnt = ch.parent[jnt]) { // state_error_function.cpp:486-555 (no enabledParameters gate)
          const int pb = jnt * kParametersPerJoint;
          for (int d = 0; d < 3; ++d) {
            if (active[pb + d]) cb.add(ch, pb + d, jnt, d, nullptr);
            if (active[pb + 3 + d]) cb.add(ch, pb + 3 + d, jnt, 3 + d, nullptr);
          }
          if (active[pb + 6]) cb.add(ch, pb + 6, jnt, 6, nullptr);
        }
        flushCells(ui, cb);
      }
    } else if (ef.kind == 5) { // Plane: a one-row position-type constraint (JointErrorFunctionT<T, PlaneDataT<T>, 1>)
      for (int c = 0; c < ef.numConstraints(); ++c) {
        if (ef.parents[c] < 0 || ef.parents[c] >= ch.numJoints) return "constraint parent joint out of range";
        UnitDesc u{};
        u.kind = kUnitPlane;
        u.ef = int32_t(e);
        u.joint = ef.parents[c];
        u.row0 = row;
        u.numRows = 1;
        u.targetOff = ef.targetOff + 4 * c;
        u.weightIdx = ef.weightOff + c;
        u.recOff = rec;
        u.extra = -1;
        for (int k = 0; k < 3; ++k) u.f[k] = ef.offsets[size_t(3) * c + k];
        const int ui = int(out.units.size());
        out.units.push_back(u);
        row += 1;
        rec += 6; // world point, scaled normal
        CellBuilder cb;
        for (int jnt = ef.parents[c]; jnt >= 0; jnt = ch.parent[jnt]) { // joint_error_function-inl.h:229-294, NumPos = 1
          const int pb = jnt * kParametersPerJoint;
          for (int d = 0; d < 3; ++d)
            if (active[pb + d]) cb.add(ch, pb + d, jnt, d, &enabled);
          for (int d = 0; d < 3; ++d)
            if (active[pb + 3 + d]) cb.add(ch, pb + 3 + d, jnt, 3 + d, &enabled);
          if (active[pb + 6]) cb.add(ch, pb + 6, jnt, 6, &enabled);
        }
        flushCells(ui, cb);
      }
    } else if (ef.kind == 6) { // ModelParameters: rows are packed over the enabled parameters with weight > 0 (:113-123); the block
      if (int(ef.paramWeights.size()) != n) return "model-parameter target weights must have one entry per parameter"; // keeps getJacobianSize rows
      const int blockStart = row;
      for (int i = 0; i < n; ++i) {
        if (!enabled[i] || ef.paramWeights[i] == 0.f) continue;
        if (ef.paramWeights[i] < 0.f) { // no Jacobian row (:113 tests weight > 0) but getError still counts it (:56-59): an error-only unit
          UnitDesc u{};
          u.kind = kUnitModelParameter;
          u.ef = int32_t(e);
          u.joint = -1;
          u.row0 = row;
          u.numRows = 0;
          u.targetOff = ef.targetOff + i;
          u.weightIdx = -1;
          u.recOff = rec;
          u.extra = -1;
          u.i[0] = i;
          u.f[0] = ef.paramWeights[i];
          u.pad[1] = 1;
          out.units.push_back(u);
          continue;
        }
        UnitDesc u{};
        u.kind = kUnitModelParameter;
        u.ef = int32_t(e);
        u.joint = -1;
        u.row0 = row;
        u.numRows = 1;
        u.targetOff = ef.targetOff + i;
        u.weightIdx = -1;
        u.recOff = rec;
        u.extra = -1;
        u.i[0] = i;
        u.f[0] = ef.paramWeights[i];
        const int ui = int(out.units.size());
        out.units.push_back(u);
        row += 1;
        rec += 1;
        staticCell(ui, i, ef.paramWeights[i]);
      }
      row = blockStart + jacobianBlockSize(ch, ef);
    } else if (ef.kind == 4) {
      for (const HostLimit& l : ch.limits) {
        if (l.type == 2) continue; // MinMaxJointPassive: no rows (limit_error_function.cpp:1051-1052)
        UnitDesc u{};
        u.ef = int32_t(e);
        u.row0 = row;
        u.numRows = 1;
        u.targetOff = -1;
        u.weightIdx = -1;
        u.recOff = rec;
        u.extra = -1;
        u.f[7] = l.weight;
        const int ui = int(out.units.size());
        bool disabled = false;
        switch (l.type) {
          case 0: { // MinMax :459-503
            u.kind = kUnitLimitMinMax;
            u.i[0] = l.i[0];
            u.f[0] = l.f[0]; u.f[1] = l.f[1];
            if (l.i[0] < 0 || l.i[0] >= n) return "MinMax limit parameter index out of range";
            disabled = !enabled[l.i[0]];
            out.units.push_back(u);
            if (!disabled) staticCell(ui, l.i[0], 1.f);
            break;
          }
          case 1: { // MinMaxJoint :505-558
            u.kind = kUnitLimitMinMaxJoint;
            const int jpi = l.i[0] * kParametersPerJoint + l.i[1];
            if (l.i[0] < 0 || l.i[0] >= ch.numJoints || l.i[1] < 0 || l.i[1] > 6) return "MinMaxJoint limit index out of range";
            u.i[0] = jpi;
            u.f[0] = l.f[0]; u.f[1] = l.f[1];
            disabled = !active[jpi];
            out.units.push_back(u);
            if (!disabled)
              for (int k = ch.ptOuter[jpi]; k < ch.ptOuter[jpi + 1]; ++k) staticCell(ui, ch.ptInner[k], ch.ptVals[k]);
            break;
          }
          case 3: { // Linear :560-598
            u.kind = kUnitLimitLinear;
            const int ref = l.i[0], tgt = l.i[1];
            if (ref < 0 || ref >= n || tgt < 0 || tgt >= n) return "Linear limit parameter index out of range";
            u.i[0] = ref; u.i[1] = tgt;
            for (int k = 0; k < 4; ++k) u.f[k] = l.f[k];
            disabled = !enabled[tgt] && !enabled[ref];
            out.units.push_back(u);
            if (!disabled) {
              // assignments, target first then reference: the later one wins if both name the same column
              if (enabled[tgt] && !(enabled[ref] && ref == tgt)) staticCell(ui, tgt, l.f[0]);
              if (enabled[ref]) staticCell(ui, ref, -1.f);
            }
            break;
          }
          case 4: { // LinearJoint :600-656
            u.kind = kUnitLimitLinearJoint;
            const int ri = l.i[0] * kParametersPerJoint + l.i[1];
            const int ti = l.i[2] * kParametersPerJoint + l.i[3];
            if (l.i[0] < 0 || l.i[0] >= ch.numJoints || l.i[2] < 0 || l.i[2] >= ch.numJoints || l.i[1] < 0 || l.i[1] > 6 || l.i[3] < 0 || l.i[3] > 6)
              return "LinearJoint limit index out of range";
            u.i[0] = ri; u.i[1] = ti;
            for (int k = 0; k < 4; ++k) u.f[k] = l.f[k];
            disabled = !active[ri] && !active[ti];
            out.units.push_back(u);
            if (!disabled) {
              std::map<int, float> acc;
              if (active[ti]) for (int k = ch.ptOuter[ti]; k < ch.ptOuter[ti + 1]; ++k) acc[ch.ptInner[k]] += l.f[0] * ch.ptVals[k];
              if (active[ri]) for (int k = ch.ptOuter[ri]; k < ch.ptOuter[ri + 1]; ++k) acc[ch.ptInner[k]] += -ch.ptVals[k];
              for (auto& kv : acc) staticCell(ui, kv.first, kv.second);
            }
            break;
          }
          case 6: { // HalfPlane :658-699
            u.kind = kUnitLimitHalfPlane;
            const int p1 = l.i[0], p2 = l.i[1];
            if (p1 < 0 || p1 >= n || p2 < 0 || p2 >= n) return "HalfPlane limit parameter index out of range";
            u.i[0] = p1; u.i[1] = p2;
            u.f[0] = l.f[0]; u.f[1] = l.f[1]; u.f[2] = l.f[2];
            disabled = !enabled[p1] && !enabled[p2];
            out.units.push_back(u);
            if (!disabled) {
              if (enabled[p1] && !(enabled[p2] && p1 == p2)) staticCell(ui, p1, l.f[0]);
              if (enabled[p2]) staticCell(ui, p2, l.f[1]);
            }
            break;
          }
          case 5: { // Ellipsoid :701-785
            u.kind = kUnitLimitEllipsoid;
            u.numRows = 3;
            if (alignRowGroups) { row = (row + 3) & ~3; u.row0 = row; }
            u.i[0] = l.i[0]; // ellipsoidParent
            u.joint = l.i[1]; // parent
            if (l.i[0] < 0 || l.i[0] >= ch.numJoints || l.i[1] < 0 || l.i[1] >= ch.numJoints) return "Ellipsoid limit joint index out of range";
            u.extra = int32_t(out.limitData.size());
            out.limitData.insert(out.limitData.end(), l.f, l.f + 27);
            out.limitData.push_back(0.f);
            out.units.push_back(u);
            CellBuilder cb;
            for (int jnt = l.i[1]; jnt != l.i[0] && jnt >= 0; jnt = ch.parent[jnt]) { // :740-777
              const int pb = jnt * kParametersPerJoint;
              for (int d = 0; d < 3; ++d) {
                if (active[pb + d]) cb.add(ch, pb + d, jnt, d, nullptr);
                if (active[pb + 3 + d]) cb.add(ch, pb + 3 + d, jnt, 3 + d, nullptr);
              }
              if (active[pb + 6]) cb.add(ch, pb + 6, jnt, 6, nullptr);
            }
            flushCells(ui, cb);
            break;
          }
          default: return "Unknown parameter type for joint limit";
        }
        out.units[ui].pad[0] = disabled ? 1 : 0;
        row += out.units[ui].numRows;
        if (alignRowGroups && out.units[ui].numRows > 1) row = (row + 3) & ~3;
        rec += (l.type == 5) ? 4 : 1;
      }
    } else {
      return "unknown error function kind";
    }
  }
  if (out.units.size() > 65535) return "too many constraints in one solver function (limit 65535 units)";
  out.numRows = row;
  out.recStride = std::max(rec, 1);
  // Group cells so that neighbouring lanes run the same code path and store next to each other. K-major matrix: same column, consecutive
  // units = consecutive rows of that column. Strip layout (alignRowGroups): same unit, consecutive device columns = consecutive 16-byte
  // pieces of the unit's strip (a row quad x 16 columns is 256 contiguous bytes), so a warp's stores fill whole sectors and lines, and
  // the unit / record reads of a warp are broadcasts.
  std::stable_sort(out.cells.begin(), out.cells.end(), [&](const CellDesc& a, const CellDesc& b) {
    const int ka = out.units[a.unit].kind, kb = out.units[b.unit].kind;
    if (ka != kb) return ka < kb;
    if (alignRowGroups) return a.unit != b.unit ? a.unit < b.unit : a.col < b.col;
    if (a.col != b.col) return a.col < b.col;
    return a.unit < b.unit;
  });
  return "";
}

int resolveCholeskyMode(int requested, const std::vector<uint8_t>& enabled) {
  if (requested != MB2_CHOLESKY_AUTO) return requested;
  int numEnabled = 0;
  for (uint8_t e : enabled) numEnabled += e ? 1 : 0;
  return numEnabled >= 48 ? MB2_CHOLESKY_TILES_SPARSE : MB2_CHOLESKY_DENSE_EIGEN;
}

// depth (in the joint tree) of the deepest joint each enabled parameter drives: tie-break priority of the elimination order
static std::vector<int> columnDepthPriority(const HostCharacter& h, const std::vector<int32_t>& enabledList) {
  std::vector<int> jointDepth(h.numJoints, 0);
  for (int j = 0; j < h.numJoints; ++j) { int d = 0; for (int a = h.parent[j]; a >= 0; a = h.parent[a]) ++d; jointDepth[j] = d; }
  std::vector<int> paramDepth(h.numParams, 0);
  for (int r = 0; r < kParametersPerJoint * h.numJoints; ++r)
    for (int k = h.ptOuter[r]; k < h.ptOuter[r + 1]; ++k) paramDepth[h.ptInner[k]] = std::max(paramDepth[h.ptInner[k]], jointDepth[r / kParametersPerJoint]);
  std::vector<int> prio(enabledList.size());
  for (size_t a = 0; a < enabledList.size(); ++a) prio[a] = paramDepth[enabledList[a]];
  return prio;
}

std::string planSolverPath(const HostCharacter& ch, const std::vector<HostErrorFunction>& efs, const std::vector<uint8_t>& enabled, bool densePattern, bool strips,
                           Plan& plan, CholSchedule& sched, GramPlan& gram) {
  gram = GramPlan();
  std::string err = buildPlan(ch, efs, enabled, true, plan);
  if (!err.empty()) return err;
  std::vector<std::vector<int>> cliques(plan.units.size());
  for (const CellDesc& c : plan.cells) cliques[c.unit].push_back(int(c.col));
  const std::vector<int> prio = columnDepthPriority(ch, plan.enabledList);
  err = buildCholSchedule(plan.numCols, cliques, densePattern, sched, &prio);
  if (!err.empty()) return err;
  // re-plan with the device columns in elimination order (tile starts aligned to 4 columns), the schedule expressed in them
  std::vector<int32_t> colOrder;
  layoutDeviceColumns(sched, colOrder);
  for (int32_t& c : colOrder) if (c >= 0) c = plan.enabledList[c];
  err = buildPlan(ch, efs, enabled, true, plan, &colOrder, strips);
  if (!err.empty() || !strips) return err;
  std::vector<int32_t> cr0, crn, cc;
  for (const CellDesc& c : plan.cells) { cr0.push_back(plan.units[c.unit].row0); crn.push_back(plan.units[c.unit].numRows); cc.push_back(int32_t(c.col)); }
  err = buildGramPlan(sched, cr0, crn, cc, plan.numRows, gram);
  if (!err.empty()) return err;
  for (size_t i = 0; i < plan.cells.size(); ++i) { plan.cells[i].stripOff = gram.cellStripOff[i]; plan.cells[i].quadStride = gram.cellQuadStride[i]; }
  return "";
}

} // namespace mb2
