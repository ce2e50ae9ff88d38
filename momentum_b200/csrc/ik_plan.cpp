#include "ik_plan.h"

#include "ik_device.cuh" // capsuleContact, shared with the kernels

#include <algorithm>
#include <array>
#include <cfloat>
#include <cmath>
#include <cstring>
#include <map>
#include <numeric>

#include "ik_jacobi.cuh"

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

namespace {
constexpr double kInverseSigmaTol = 1e-6;  // utility.cpp:423-435: a singular value is inverted when > 1e-6 (absolute), else 0
constexpr int kInverseMaxSweeps = 64;      // cyclic Jacobi sweeps of one component's Gram matrix (it stops at the first sweep without a rotation)

// W = A^+ [c][m] of the dense block A [m][c] (row-major), through the eigen-decomposition K = Q Lambda Q^T of the Gram matrix on A's
// smaller side: c <= m: K = A^T A, W = Q Lambda^+ Q^T A^T; m < c: K = A A^T, W = A^T Q Lambda^+ Q^T. lambda = sigma^2 is inverted when
// sigma > 1e-6, i.e. lambda > 1e-12. The rotations are ik_jacobi.cuh's (jacobiRotation, its skip floor), applied cyclically by rows.
void blockPseudoInverse(const std::vector<double>& A, int m, int c, std::vector<double>& W) {
  const bool colSide = c <= m;
  const int k = colSide ? c : m;
  std::vector<double> K(size_t(k) * k), Q(size_t(k) * k, 0.0);
  for (int a = 0; a < k; ++a)
    for (int b = a; b < k; ++b) {
      double s = 0.0;
      if (colSide)
        for (int r = 0; r < m; ++r) s += A[size_t(r) * c + a] * A[size_t(r) * c + b];
      else
        for (int p = 0; p < c; ++p) s += A[size_t(a) * c + p] * A[size_t(b) * c + p];
      K[size_t(a) * k + b] = K[size_t(b) * k + a] = s;
    }
  double maxDiagonal = 0.0;
  for (int a = 0; a < k; ++a) {
    Q[size_t(a) * k + a] = 1.0;
    maxDiagonal = std::max(maxDiagonal, K[size_t(a) * k + a]);
  }
  const double floor = jacobiFloor(maxDiagonal);
  for (int sweep = 0; sweep < kInverseMaxSweeps; ++sweep) {
    bool rotated = false;
    for (int p = 0; p < k; ++p)
      for (int q = p + 1; q < k; ++q) {
        double cs, sn, t;
        if (!jacobiRotation(K[size_t(p) * k + p], K[size_t(q) * k + q], K[size_t(p) * k + q], floor, cs, sn, t)) continue;
        rotated = true;
        // K <- R^T K R (R_pp = R_qq = c, R_pq = s, R_qp = -s), Q <- Q R
        const double apq = K[size_t(p) * k + q];
        K[size_t(p) * k + p] -= t * apq;
        K[size_t(q) * k + q] += t * apq;
        K[size_t(p) * k + q] = K[size_t(q) * k + p] = 0.0;
        for (int i = 0; i < k; ++i) {
          if (i != p && i != q) {
            const double kip = K[size_t(i) * k + p], kiq = K[size_t(i) * k + q];
            K[size_t(i) * k + p] = K[size_t(p) * k + i] = cs * kip - sn * kiq;
            K[size_t(i) * k + q] = K[size_t(q) * k + i] = sn * kip + cs * kiq;
          }
          const double qip = Q[size_t(i) * k + p], qiq = Q[size_t(i) * k + q];
          Q[size_t(i) * k + p] = cs * qip - sn * qiq;
          Q[size_t(i) * k + q] = sn * qip + cs * qiq;
        }
      }
    if (!rotated) break;
  }
  // M = Q Lambda^+ Q^T [k][k]
  std::vector<double> inv(k), M(size_t(k) * k, 0.0);
  for (int a = 0; a < k; ++a) {
    const double lambda = K[size_t(a) * k + a];
    inv[a] = lambda > kInverseSigmaTol * kInverseSigmaTol ? 1.0 / lambda : 0.0;
  }
  for (int i = 0; i < k; ++i)
    for (int j = 0; j < k; ++j) {
      double s = 0.0;
      for (int a = 0; a < k; ++a) s += Q[size_t(i) * k + a] * inv[a] * Q[size_t(j) * k + a];
      M[size_t(i) * k + j] = s;
    }
  W.assign(size_t(c) * m, 0.0);
  for (int p = 0; p < c; ++p)
    for (int r = 0; r < m; ++r) {
      double s = 0.0;
      if (colSide)
        for (int a = 0; a < c; ++a) s += M[size_t(p) * k + a] * A[size_t(r) * c + a]; // (M A^T)_pr
      else
        for (int a = 0; a < m; ++a) s += A[size_t(a) * c + p] * M[size_t(a) * k + r]; // (A^T M)_pr
      W[size_t(p) * m + r] = s;
    }
}
} // namespace

// P is block-diagonal under the permutation that groups the connected components of its sparsity graph (joint-parameter rows and model
// parameters, joined by every stored entry, stored zeros included). The pseudo-inverse of a block-diagonal matrix is the block-diagonal
// matrix of the blocks' pseudo-inverses, and P's singular values are the union of the blocks', so the absolute 1e-6 rule truncates the
// same values per block as for the whole matrix: W is the reference's matrix, computed per component. A parameter without entries is a
// component of its own with an empty row of W. Entries that round to 0 are not stored.
void HostCharacter::buildInverseTables() {
  const int rows = numJoints * kParametersPerJoint, n = numParams;
  std::vector<int32_t> root(size_t(rows) + n);
  std::iota(root.begin(), root.end(), 0);
  auto find = [&](int32_t x) {
    while (root[x] != x) x = root[x] = root[root[x]];
    return x;
  };
  for (int r = 0; r < rows; ++r)
    for (int k = ptOuter[r]; k < ptOuter[r + 1]; ++k) {
      const int32_t a = find(r), b = find(rows + ptInner[k]);
      if (a != b) root[std::max(a, b)] = std::min(a, b);
    }
  // the rows and parameters of each component, both ascending
  std::map<int32_t, std::pair<std::vector<int32_t>, std::vector<int32_t>>> comps;
  for (int r = 0; r < rows; ++r) comps[find(r)].first.push_back(r);
  for (int p = 0; p < n; ++p) comps[find(rows + p)].second.push_back(p);
  std::vector<std::vector<std::pair<int32_t, float>>> byParam(n);
  std::vector<double> A, W;
  std::vector<int32_t> local(rows, -1);
  for (const auto& kv : comps) {
    const std::vector<int32_t>& cr = kv.second.first;
    const std::vector<int32_t>& cp = kv.second.second;
    const int m = int(cr.size()), c = int(cp.size());
    if (m == 0 || c == 0) continue; // a parameter without entries, or rows no parameter drives
    for (int i = 0; i < m; ++i) local[cr[i]] = i;
    std::map<int32_t, int32_t> col;
    for (int j = 0; j < c; ++j) col[cp[j]] = j;
    A.assign(size_t(m) * c, 0.0);
    for (int i = 0; i < m; ++i)
      for (int k = ptOuter[cr[i]]; k < ptOuter[cr[i] + 1]; ++k) A[size_t(i) * c + col[ptInner[k]]] += double(ptVals[k]);
    blockPseudoInverse(A, m, c, W);
    for (int j = 0; j < c; ++j)
      for (int i = 0; i < m; ++i) {
        const float w = float(W[size_t(j) * m + i]);
        if (w != 0.f) byParam[cp[j]].push_back({cr[i], w});
      }
  }
  invStart.assign(n + 1, 0);
  invRows.clear();
  invVals.clear();
  for (int p = 0; p < n; ++p) {
    for (const auto& e : byParam[p]) {
      invRows.push_back(e.first);
      invVals.push_back(e.second);
    }
    invStart[p + 1] = int32_t(invRows.size());
  }
  invRowStart.assign(rows + 1, 0);
  for (int32_t r : invRows) invRowStart[r + 1]++;
  for (int r = 0; r < rows; ++r) invRowStart[r + 1] += invRowStart[r];
  invParams.resize(invRows.size());
  invRowVals.resize(invRows.size());
  std::vector<int32_t> cursor(invRowStart.begin(), invRowStart.end() - 1);
  for (int p = 0; p < n; ++p) // ascending parameters: each row's parameters in increasing order
    for (int k = invStart[p]; k < invStart[p + 1]; ++k) {
      const int at = cursor[invRows[k]]++;
      invParams[at] = p;
      invRowVals[at] = invVals[k];
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
  out.buildInverseTables();
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

std::string makeBlendShape(int32_t numShapes, int32_t numVertices, const float* baseShape, const float* shapeVectors, HostBlendShape& out) {
  if (numVertices < 1) return "blend shape: the mesh must have at least one vertex";
  if (numShapes < 1) return "blend shape: there must be at least one shape vector";
  if (!(baseShape && shapeVectors)) return "blend shape: null argument";
  const size_t n = size_t(numVertices) * 3;
  for (size_t k = 0; k < n; ++k)
    if (!std::isfinite(baseShape[k])) return "blend shape: the base shape must be finite";
  for (size_t k = 0; k < n * size_t(numShapes); ++k)
    if (!std::isfinite(shapeVectors[k])) return "blend shape: shape vectors must be finite";
  HostBlendShape b;
  b.numShapes = numShapes;
  b.numVertices = numVertices;
  b.baseShape.assign(baseShape, baseShape + n);
  b.shapeVectors.assign(shapeVectors, shapeVectors + n * size_t(numShapes));
  out = std::move(b);
  return "";
}

std::string makeMeshFaces(int32_t numVertices, int32_t numFaces, const int32_t* faces, HostMeshFaces& out) {
  if (numVertices < 1) return "mesh faces: the mesh must have at least one vertex";
  if (numFaces < 0) return "mesh faces: the number of faces must not be negative";
  if (numFaces > INT32_MAX / 3) return "mesh faces: too many faces (3 x num_faces must fit in int32)";
  if (numFaces > 0 && faces == nullptr) return "mesh faces: null argument";
  const size_t corners = size_t(numFaces) * 3;
  for (size_t c = 0; c < corners; ++c)
    if (faces[c] < 0 || faces[c] >= numVertices) return "mesh faces: a face index is outside [0, num_vertices)";
  HostMeshFaces m;
  m.numVertices = numVertices;
  m.numFaces = numFaces;
  m.faces.assign(faces, faces + corners);
  m.vertStart.assign(size_t(numVertices) + 1, 0);
  for (size_t c = 0; c < corners; ++c) ++m.vertStart[size_t(m.faces[c]) + 1];
  for (int32_t v = 0; v < numVertices; ++v) m.vertStart[v + 1] += m.vertStart[v];
  m.vertCorner.resize(corners);
  std::vector<int32_t> fill(m.vertStart.begin(), m.vertStart.end() - 1);
  for (size_t c = 0; c < corners; ++c) m.vertCorner[size_t(fill[m.faces[c]]++)] = int32_t(c); // c = 3 f + k ascending
  out = std::move(m);
  return "";
}

std::string makePointTables(int32_t numJoints, int32_t numPoints, const int32_t* parents, std::vector<int32_t>& out) {
  if (numPoints < 0) return "positions: the number of points must not be negative";
  if (numPoints > 0 && parents == nullptr) return "positions: null parents";
  for (int32_t i = 0; i < numPoints; ++i)
    if (parents[i] < 0 || parents[i] >= numJoints) return "positions: a parent is outside [0, num_joints)";
  const size_t N = size_t(numPoints), J = size_t(numJoints);
  std::vector<int32_t> t(2 * N + J + 1, 0);
  int32_t* start = t.data() + N;
  int32_t* index = start + J + 1;
  std::copy(parents, parents + N, t.begin());
  for (size_t i = 0; i < N; ++i) ++start[parents[i] + 1];
  for (size_t j = 0; j < J; ++j) start[j + 1] += start[j];
  std::vector<int32_t> fill(start, start + J);
  for (size_t i = 0; i < N; ++i) index[fill[parents[i]]++] = int32_t(i); // i ascending within a joint
  out = std::move(t);
  return "";
}

std::string makeMeshTree(const HostMeshFaces& faces, int32_t numVertices, const float* referencePositions, HostMeshTree& out) {
  if (faces.numFaces < 1) return "mesh tree: the mesh has no faces";
  if (numVertices != faces.numVertices) return "mesh tree: num_vertices differs from the mesh faces' num_vertices";
  if (referencePositions == nullptr) return "mesh tree: null argument";
  const int32_t F = faces.numFaces;
  for (size_t i = 0; i < size_t(numVertices) * 3; ++i)
    if (!std::isfinite(referencePositions[i])) return "mesh tree: a reference position is not finite";
  std::vector<double> centroid(size_t(F) * 3);
  for (int32_t f = 0; f < F; ++f)
    for (int k = 0; k < 3; ++k) {
      double s = 0.0;
      for (int c = 0; c < 3; ++c) s += referencePositions[size_t(faces.faces[size_t(f) * 3 + c]) * 3 + k];
      centroid[size_t(f) * 3 + k] = s / 3.0;
    }
  HostMeshTree t;
  t.numVertices = numVertices;
  t.numFaces = F;
  t.leafFaces.resize(size_t(F));
  for (int32_t f = 0; f < F; ++f) t.leafFaces[f] = f;
  // level by level: the nodes of a level are face ranges [lo, hi) of leafFaces; the children of a split node are appended to the next
  // level in order, so the two are adjacent
  std::vector<std::pair<int32_t, int32_t>> level{{0, F}}, next;
  while (!level.empty()) {
    if (t.depth == kTreeStack) return "mesh tree: the tree is deeper than the traversal stack";
    t.levelStart.push_back(t.numNodes);
    const int32_t nextFirst = t.numNodes + int32_t(level.size());
    next.clear();
    for (const auto& r : level) {
      const int32_t lo = r.first, hi = r.second, n = hi - lo;
      if (n <= kLeafFaces) {
        t.nodeStart.push_back(lo);
        t.nodeCount.push_back(n);
        continue;
      }
      double bmin[3] = {DBL_MAX, DBL_MAX, DBL_MAX}, bmax[3] = {-DBL_MAX, -DBL_MAX, -DBL_MAX};
      for (int32_t i = lo; i < hi; ++i)
        for (int k = 0; k < 3; ++k) {
          const double c = centroid[size_t(t.leafFaces[i]) * 3 + k];
          bmin[k] = std::min(bmin[k], c);
          bmax[k] = std::max(bmax[k], c);
        }
      int axis = 0;
      for (int k = 1; k < 3; ++k)
        if (bmax[k] - bmin[k] > bmax[axis] - bmin[axis]) axis = k;
      std::sort(t.leafFaces.begin() + lo, t.leafFaces.begin() + hi, [&](int32_t a, int32_t b) {
        const double ca = centroid[size_t(a) * 3 + axis], cb = centroid[size_t(b) * 3 + axis];
        return ca < cb || (ca == cb && a < b);
      });
      t.nodeStart.push_back(nextFirst + int32_t(next.size()));
      t.nodeCount.push_back(0);
      const int32_t groups = (n + kLeafFaces - 1) / kLeafFaces; // the median rounded to whole leaves: all leaves but one are full
      const int32_t mid = lo + (groups + 1) / 2 * kLeafFaces;
      next.push_back({lo, mid});
      next.push_back({mid, hi});
    }
    t.numNodes += int32_t(level.size());
    ++t.depth;
    level.swap(next);
  }
  t.levelStart.push_back(t.numNodes);
  out = std::move(t);
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

namespace {
const char* limitTypeName(int type) {
  static const char* names[] = {"MinMax", "MinMaxJoint", "MinMaxJointPassive", "Linear", "LinearJoint", "Ellipsoid", "HalfPlane"};
  return type >= 0 && type <= 6 ? names[type] : "unknown";
}
// CSR of (key, limit, coef) triples: keys in [0, count), the triples of a key in the order given
void limitCsr(int count, const std::vector<std::array<double, 3>>& t, std::vector<int32_t>& start, std::vector<int32_t>& limit,
              std::vector<float>* coef) {
  start.assign(size_t(count) + 1, 0);
  for (const auto& e : t) ++start[size_t(e[0]) + 1];
  for (int k = 0; k < count; ++k) start[k + 1] += start[k];
  std::vector<int32_t> fill(start.begin(), start.end() - 1);
  limit.assign(t.size(), 0);
  if (coef) coef->assign(t.size(), 0.f);
  for (const auto& e : t) { // stable: the triples of one key keep their order
    const int32_t at = fill[size_t(e[0])]++;
    limit[at] = int32_t(e[1]);
    if (coef) (*coef)[at] = float(e[2]);
  }
}
} // namespace

HostLimitTables makeLimitTables(const HostCharacter& ch) {
  HostLimitTables t;
  const int J = ch.numJoints, n = ch.numParams, rows = J * kParametersPerJoint;
  std::vector<std::array<double, 3>> byJoint, byRow, byParam;
  t.paramClamp.assign(size_t(n) * 3, 0.f);
  for (size_t k = 0; k < ch.limits.size(); ++k) {
    const HostLimit& l = ch.limits[k];
    if (l.type == kLimitMinMaxJointPassive) continue; // no rows (limit_error_function.cpp:1051-1052)
    const std::string name = "parameter limits: limit " + std::to_string(k) + " (" + limitTypeName(l.type) + ")";
    auto param = [&](int p) { return p >= 0 && p < n; };
    auto joint = [&](int j) { return j >= 0 && j < J; };
    auto jointRow = [&](int j, int d) { return joint(j) && d >= 0 && d < kParametersPerJoint; };
    LimitDesc D{};
    D.type = l.type;
    D.row = t.numRows;
    D.data = -1;
    const int l32 = int(t.limits.size());
    const double w = std::sqrt(10.0 * double(l.weight)); // kLimitWeight
    D.w = float(w);
    for (int i = 0; i < 4; ++i) D.f[i] = l.f[i];
    switch (l.type) {
      case kLimitMinMax:
        if (!param(l.i[0])) { t = HostLimitTables{}; t.rejected = name + ": parameter index " + std::to_string(l.i[0]) + " is outside [0, n)"; return t; }
        D.i0 = l.i[0];
        byParam.push_back({double(D.i0), double(l32), w});
        t.paramClamp[3 * D.i0] = l.f[0];
        t.paramClamp[3 * D.i0 + 1] = l.f[1];
        t.paramClamp[3 * D.i0 + 2] = 1.f;
        break;
      case kLimitMinMaxJoint:
        if (!jointRow(l.i[0], l.i[1])) { t = HostLimitTables{}; t.rejected = name + ": joint " + std::to_string(l.i[0]) + " parameter " + std::to_string(l.i[1]) + " is out of range"; return t; }
        D.i0 = l.i[0] * kParametersPerJoint + l.i[1];
        byRow.push_back({double(D.i0), double(l32), w});
        break;
      case kLimitLinear:
        if (!param(l.i[0]) || !param(l.i[1])) { t = HostLimitTables{}; t.rejected = name + ": a parameter index is outside [0, n)"; return t; }
        D.i0 = l.i[0];
        D.i1 = l.i[1];
        byParam.push_back({double(D.i1), double(l32), w * double(l.f[0])});
        byParam.push_back({double(D.i0), double(l32), -w});
        break;
      case kLimitLinearJoint:
        if (!jointRow(l.i[0], l.i[1]) || !jointRow(l.i[2], l.i[3])) { t = HostLimitTables{}; t.rejected = name + ": a joint or joint parameter is out of range"; return t; }
        D.i0 = l.i[0] * kParametersPerJoint + l.i[1];
        D.i1 = l.i[2] * kParametersPerJoint + l.i[3];
        byRow.push_back({double(D.i1), double(l32), w * double(l.f[0])});
        byRow.push_back({double(D.i0), double(l32), -w});
        break;
      case kLimitHalfPlane:
        if (!param(l.i[0]) || !param(l.i[1])) { t = HostLimitTables{}; t.rejected = name + ": a parameter index is outside [0, n)"; return t; }
        D.i0 = l.i[0];
        D.i1 = l.i[1];
        byParam.push_back({double(D.i0), double(l32), w * double(l.f[0])});
        byParam.push_back({double(D.i1), double(l32), w * double(l.f[1])});
        break;
      case kLimitEllipsoid:
        if (!joint(l.i[0]) || !joint(l.i[1])) { t = HostLimitTables{}; t.rejected = name + ": a joint index is outside [0, J)"; return t; }
        D.i0 = l.i[0];
        D.i1 = l.i[1];
        D.w = float(std::sqrt(10.0 * 1e-4 * double(l.weight))); // kLimitWeight kLimitPositionWeight
        D.data = int32_t(t.ellipsoidData.size());
        t.ellipsoidData.insert(t.ellipsoidData.end(), l.f, l.f + 27);
        byJoint.push_back({double(D.i1), double(2 * l32), 0.0});
        byJoint.push_back({double(D.i0), double(2 * l32 + 1), 0.0});
        t.ellipsoid = true;
        break;
      default: t = HostLimitTables{}; t.rejected = name + ": unknown limit type"; return t;
    }
    t.numRows += l.type == kLimitEllipsoid ? 3 : 1;
    t.limits.push_back(D);
  }
  limitCsr(J, byJoint, t.jointStart, t.jointEntry, nullptr);
  limitCsr(rows, byRow, t.rowStart, t.rowLimit, &t.rowCoef);
  limitCsr(n, byParam, t.paramStart, t.paramLimit, &t.paramCoef);
  return t;
}

LimitTables hostLimitTables(const HostLimitTables& t) {
  return LimitTables{int32_t(t.limits.size()), t.numRows, t.ellipsoid ? 1 : 0, t.limits.data(), t.ellipsoidData.data(), t.jointStart.data(),
                     t.jointEntry.data(), t.rowStart.data(), t.rowLimit.data(), t.rowCoef.data(), t.paramStart.data(), t.paramLimit.data(),
                     t.paramCoef.data()};
}

namespace {
// Eigen QuaternionBase::_transformVector in double
void rotateDouble(const double* q, const double* v, double* r) {
  const double uv[3] = {2.0 * (q[1] * v[2] - q[2] * v[1]), 2.0 * (q[2] * v[0] - q[0] * v[2]), 2.0 * (q[0] * v[1] - q[1] * v[0])};
  const double c[3] = {q[1] * uv[2] - q[2] * uv[1], q[2] * uv[0] - q[0] * uv[2], q[0] * uv[1] - q[1] * uv[0]};
  for (int i = 0; i < 3; ++i) r[i] = v[i] + q[3] * uv[i] + c[i];
}
// JointStateT::set of every joint at model parameters zero (joint parameters = the ParameterTransform's offsets), in double:
// t [J][3], q [J][4] (x, y, z, w), s [J]
void restPoseDouble(const HostCharacter& ch, std::vector<double>& t, std::vector<double>& q, std::vector<double>& s) {
  const int J = ch.numJoints;
  t.assign(size_t(J) * 3, 0.0);
  q.assign(size_t(J) * 4, 0.0);
  s.assign(size_t(J), 0.0);
  auto mul = [](const double* a, const double* b, double* r) {
    const double x = a[3] * b[0] + a[0] * b[3] + a[1] * b[2] - a[2] * b[1], y = a[3] * b[1] + a[1] * b[3] + a[2] * b[0] - a[0] * b[2];
    const double z = a[3] * b[2] + a[2] * b[3] + a[0] * b[1] - a[1] * b[0], w = a[3] * b[3] - a[0] * b[0] - a[1] * b[1] - a[2] * b[2];
    r[0] = x; r[1] = y; r[2] = z; r[3] = w;
  };
  for (int j = 0; j < J; ++j) {
    const float* p = ch.ptOffsets.data() + size_t(j) * kParametersPerJoint;
    double ql[4] = {ch.prerot[4 * j], ch.prerot[4 * j + 1], ch.prerot[4 * j + 2], ch.prerot[4 * j + 3]};
    for (int k = 2; k >= 0; --k) { // preRot Rz Ry Rx (joint_state.cpp:44-62)
      double r[4] = {0.0, 0.0, 0.0, std::cos(0.5 * double(p[3 + k]))};
      r[k] = std::sin(0.5 * double(p[3 + k]));
      mul(ql, r, ql);
    }
    const double tl[3] = {double(ch.offset[3 * j]) + p[0], double(ch.offset[3 * j + 1]) + p[1], double(ch.offset[3 * j + 2]) + p[2]};
    const double sl = std::exp2(double(p[6]));
    const int par = ch.parent[j];
    if (par < 0) {
      for (int i = 0; i < 3; ++i) t[3 * j + i] = tl[i];
      for (int i = 0; i < 4; ++i) q[4 * j + i] = ql[i];
      s[j] = sl;
      continue;
    }
    const double* qp = &q[4 * par];
    const double v[3] = {s[par] * tl[0], s[par] * tl[1], s[par] * tl[2]};
    double rv[3];
    rotateDouble(qp, v, rv);
    for (int i = 0; i < 3; ++i) t[3 * j + i] = t[3 * par + i] + rv[i];
    mul(qp, ql, &q[4 * j]);
    s[j] = s[par] * sl;
  }
}
} // namespace

std::string makeCollision(const HostCharacter& ch, int32_t count, const mb2_tapered_capsule* capsules, HostCollision& out) {
  if (count < 0 || (count > 0 && capsules == nullptr)) return "collision geometry: count must not be negative and capsules must not be null";
  const int J = ch.numJoints;
  HostCollision h;
  h.capsules.resize(size_t(count));
  std::vector<double> local(size_t(count) * 8); // origin, dir, r0, r1 in double
  for (int k = 0; k < count; ++k) {
    const mb2_tapered_capsule& c = capsules[k];
    const std::string name = "collision geometry: capsule " + std::to_string(k);
    if (c.parent < -1 || c.parent >= J) return name + ": parent " + std::to_string(c.parent) + " is outside [-1, J)";
    const float* values[] = {c.translation, c.translation + 1, c.translation + 2, c.rotation, c.rotation + 1, c.rotation + 2, c.rotation + 3,
                             &c.scale, c.radius, c.radius + 1, &c.length};
    for (const float* v : values)
      if (!std::isfinite(*v)) return name + ": every value must be finite";
    if (c.radius[0] < 0.f || c.radius[1] < 0.f) return name + ": a radius is negative";
    if (c.length < 0.f) return name + ": the length is negative";
    double qn = 0.0;
    for (int i = 0; i < 4; ++i) qn += double(c.rotation[i]) * c.rotation[i];
    if (!(qn > 0.0)) return name + ": the rotation is zero";
    qn = std::sqrt(qn);
    const double q[4] = {c.rotation[0] / qn, c.rotation[1] / qn, c.rotation[2] / qn, c.rotation[3] / qn};
    const double ex[3] = {double(c.scale) * c.length, 0.0, 0.0};
    double* L = &local[size_t(k) * 8];
    rotateDouble(q, ex, L + 3);
    for (int i = 0; i < 3; ++i) L[i] = c.translation[i];
    L[6] = c.radius[0];
    L[7] = c.radius[1];
    CapsuleDesc& d = h.capsules[k];
    d.parent = c.parent;
    for (int i = 0; i < 3; ++i) { d.origin[i] = float(L[i]); d.dir[i] = float(L[3 + i]); }
    for (int i = 0; i < 3; ++i) // scale times length can overflow float although both are finite
      if (!std::isfinite(d.dir[i])) return name + ": its direction (scale times length) overflows float";
    d.r0 = c.radius[0];
    d.r1 = c.radius[1];
  }
  // the rest pose's world capsules (updatePrimitive), in double
  std::vector<double> t, q, s, world(size_t(count) * 8);
  restPoseDouble(ch, t, q, s);
  for (int k = 0; k < count; ++k) {
    const double* L = &local[size_t(k) * 8];
    double* W = &world[size_t(k) * 8];
    const int p = h.capsules[k].parent;
    if (p < 0) { std::copy(L, L + 8, W); continue; }
    const double so[3] = {s[p] * L[0], s[p] * L[1], s[p] * L[2]}, sd[3] = {s[p] * L[3], s[p] * L[4], s[p] * L[5]};
    rotateDouble(&q[4 * p], so, W);
    for (int i = 0; i < 3; ++i) W[i] += t[3 * p + i];
    rotateDouble(&q[4 * p], sd, W + 3);
    W[6] = L[6] * s[p];
    W[7] = L[7] * s[p];
  }
  // updateCollisionPairs / isValidCollisionPair (collision_geometry_state.h:526-557), i < j ascending
  for (int i = 0; i < count; ++i)
    for (int j = i + 1; j < count; ++j) {
      const int p0 = h.capsules[i].parent, p1 = h.capsules[j].parent;
      bool valid;
      if (p0 < 0 || p1 < 0) valid = p0 != p1;
      else if (p0 == p1 || ch.parent[p0] == p1 || ch.parent[p1] == p0) valid = false;
      else valid = !capsuleContact<double>(&world[size_t(i) * 8], &world[size_t(j) * 8]).hit;
      if (valid) { h.pairs.push_back(i); h.pairs.push_back(j); }
    }
  const int P = h.numPairs();
  h.capsuleStart.assign(size_t(count) + 1, 0);
  for (int k = 0; k < 2 * P; ++k) ++h.capsuleStart[size_t(h.pairs[k]) + 1];
  for (int k = 0; k < count; ++k) h.capsuleStart[k + 1] += h.capsuleStart[k];
  h.capsulePair.assign(size_t(2) * P, 0);
  std::vector<int32_t> fill(h.capsuleStart.begin(), h.capsuleStart.end() - 1);
  for (int p = 0; p < P; ++p) // pairs ascending within a capsule
    for (int side = 0; side < 2; ++side) h.capsulePair[fill[size_t(h.pairs[2 * p + side])]++] = p;
  h.jointStart.assign(size_t(J) + 1, 0);
  for (const CapsuleDesc& c : h.capsules)
    if (c.parent >= 0) ++h.jointStart[size_t(c.parent) + 1];
  for (int j = 0; j < J; ++j) h.jointStart[j + 1] += h.jointStart[j];
  h.jointCapsule.assign(size_t(h.jointStart[J]), 0);
  fill.assign(h.jointStart.begin(), h.jointStart.end() - 1);
  for (int k = 0; k < count; ++k)
    if (h.capsules[k].parent >= 0) h.jointCapsule[fill[size_t(h.capsules[k].parent)]++] = k;
  out = std::move(h);
  return "";
}

CollisionTables hostCollisionTables(const HostCollision& c) {
  return CollisionTables{int32_t(c.capsules.size()), c.numPairs(), c.capsules.data(), c.pairs.data(), c.capsuleStart.data(),
                         c.capsulePair.data(), c.jointStart.data(), c.jointCapsule.data()};
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
