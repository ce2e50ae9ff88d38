// Per-lane building blocks of the FK / residual / Jacobian sweep. Every function is
// __host__ __device__ so the same code is exercised by the CPU lane-emulation test
// (tests/emu) before it runs in the sm_90a kernels of ik_kernels.cu.
//
// Reference math (file:line relative to the momentum/ directory of the momentum repository):
//   character/joint_state.cpp:22-82, character/skeleton_state.cpp:87-121,
//   character/parameter_transform.cpp:110-123, math/transform.h:124-129,165-167,193-195,
//   character_solver/joint_error_function-inl.h:179-297, position_/orientation_/state_/limit_error_function.cpp,
//   math/generalized_loss.cpp:24-160, math/utility.cpp:72-180.
#pragma once

#include <cmath>
#include <cfloat>

#include "ik_types.h"

namespace mb2 {

struct F3 {
  float x, y, z;
};
struct Q4 {
  float x, y, z, w;
};

MB2_HD F3 f3(float x, float y, float z) { F3 r; r.x = x; r.y = y; r.z = z; return r; }
MB2_HD F3 operator+(F3 a, F3 b) { return f3(a.x + b.x, a.y + b.y, a.z + b.z); }
MB2_HD F3 operator-(F3 a, F3 b) { return f3(a.x - b.x, a.y - b.y, a.z - b.z); }
MB2_HD F3 operator*(F3 a, float s) { return f3(a.x * s, a.y * s, a.z * s); }
MB2_HD F3 operator*(float s, F3 a) { return f3(a.x * s, a.y * s, a.z * s); }
MB2_HD float dot(F3 a, F3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
MB2_HD F3 cross(F3 a, F3 b) { return f3(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x); }
MB2_HD float comp(F3 a, int i) { return i == 0 ? a.x : (i == 1 ? a.y : a.z); }

MB2_HD Q4 q4(float x, float y, float z, float w) { Q4 r; r.x = x; r.y = y; r.z = z; r.w = w; return r; }
// Eigen quaternion product
MB2_HD Q4 qmul(Q4 a, Q4 b) {
  return q4(a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y, a.w * b.y + a.y * b.w + a.z * b.x - a.x * b.z,
            a.w * b.z + a.z * b.w + a.x * b.y - a.y * b.x, a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z);
}
// Eigen QuaternionBase::_transformVector
MB2_HD F3 qrot(Q4 q, F3 v) {
  F3 u = f3(q.x, q.y, q.z);
  F3 uv = cross(u, v);
  uv = uv + uv;
  return v + q.w * uv + cross(u, uv);
}
MB2_HD Q4 qconj(Q4 q) { return q4(-q.x, -q.y, -q.z, q.w); }
MB2_HD Q4 qnormalized(Q4 q) {
  const float n = sqrtf(q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w);
  return q4(q.x / n, q.y / n, q.z / n, q.w / n);
}
// Eigen QuaternionBase::toRotationMatrix; m[3*col + row]
MB2_HD void qmat(Q4 q, float* m) {
  const float tx = 2.f * q.x, ty = 2.f * q.y, tz = 2.f * q.z;
  const float twx = tx * q.w, twy = ty * q.w, twz = tz * q.w;
  const float txx = tx * q.x, txy = ty * q.x, txz = tz * q.x;
  const float tyy = ty * q.y, tyz = tz * q.y, tzz = tz * q.z;
  m[0] = 1.f - (tyy + tzz); m[3] = txy - twz; m[6] = txz + twy;
  m[1] = txy + twz; m[4] = 1.f - (txx + tzz); m[7] = tyz - twx;
  m[2] = txz - twy; m[5] = tyz + twx; m[8] = 1.f - (txx + tyy);
}
MB2_HD F3 qmatcol(Q4 q, int c) { // column c of toRotationMatrix(q)
  float m[9];
  qmat(q, m);
  return f3(m[3 * c], m[3 * c + 1], m[3 * c + 2]);
}

MB2_HD F3 ld3(const float* p) { return f3(p[0], p[1], p[2]); }
MB2_HD Q4 ld4(const float* p) { return q4(p[0], p[1], p[2], p[3]); }

// ---- GeneralizedLossT (math/generalized_loss.cpp:104-155) ----
MB2_HD float lossValue(const EfDesc& e, float s) {
  switch (e.lossType) {
    case kLossL2: return s * e.invC2;
    case kLossL1: return sqrtf(s * e.invC2 + 1.f) - 1.f;
    case kLossCauchy: return logf(0.5f * (s * e.invC2) + 1.f);
    case kLossWelsch: return 1.f - expf(-0.5f * (s * e.invC2));
    default: return (powf(s * e.invC2 / fabsf(e.alpha - 2.f) + 1.f, 0.5f * e.alpha) - 1.f) * fabsf(e.alpha - 2.f) / e.alpha;
  }
}
MB2_HD float lossDeriv(const EfDesc& e, float s) {
  switch (e.lossType) {
    case kLossL2: return e.invC2;
    case kLossL1: return 0.5f * e.invC2 / sqrtf(s * e.invC2 + 1.f);
    case kLossCauchy: return e.invC2 / (e.invC2 * s + 2.f);
    case kLossWelsch: return 0.5f * e.invC2 * expf(-0.5f * (s * e.invC2));
    default: return 0.5f * e.invC2 * powf(s * e.invC2 / fabsf(e.alpha - 2.f) + 1.f, 0.5f * e.alpha - 1.f);
  }
}

// ---- ParameterTransformT::apply, one row (parameter_transform.cpp:122) ----
MB2_HD float jointParameterRow(const CharacterTables& T, int row, const float* theta) {
  float s = 0.f;
  for (int k = T.ptOuter[row]; k < T.ptOuter[row + 1]; ++k) s += T.ptVals[k] * theta[T.ptInner[k]];
  return s + T.ptOffsets[row];
}

// ---- JointStateT::set for joint j (joint_state.cpp:22-65). js: kJointStateStride floats per joint ----
template <bool kDeriv>
MB2_HD void fkJoint(const CharacterTables& T, int j, const float* jp, float* js) {
  const float* p = jp + j * kParametersPerJoint;
  const int par = T.parent[j];
  F3 tp = f3(0.f, 0.f, 0.f);
  Q4 qp = q4(0.f, 0.f, 0.f, 1.f);
  float sp = 1.f;
  if (par >= 0) {
    const float* ps = js + par * kJointStateStride;
    tp = ld3(ps); qp = ld4(ps + 3); sp = ps[7];
  }
  Q4 ql = ld4(T.prerot + 4 * j);
  float* out = js + j * kJointStateStride;
  for (int index = 2; index >= 0; --index) { // :51-58
    if (kDeriv) {
      const F3 axis = f3(index == 0 ? 1.f : 0.f, index == 1 ? 1.f : 0.f, index == 2 ? 1.f : 0.f);
      const F3 a = qrot(qmul(qp, ql), axis);
      out[8 + 3 * index] = a.x; out[9 + 3 * index] = a.y; out[10 + 3 * index] = a.z;
    }
    const float ha = 0.5f * p[3 + index];
    float sn, cs;
#if defined(__CUDA_ARCH__)
    sincosf(ha, &sn, &cs);
#else
    sn = sinf(ha); cs = cosf(ha);
#endif
    ql = qmul(ql, q4(index == 0 ? sn : 0.f, index == 1 ? sn : 0.f, index == 2 ? sn : 0.f, cs));
  }
  const F3 tl = f3(T.offset[3 * j] + p[0], T.offset[3 * j + 1] + p[1], T.offset[3 * j + 2] + p[2]); // :44
  const float sl = exp2f(p[6]); // :62
  const F3 t = tp + qrot(qp, sp * tl); // transform.h:125
  const Q4 q = qmul(qp, ql);
  out[0] = t.x; out[1] = t.y; out[2] = t.z;
  out[3] = q.x; out[4] = q.y; out[5] = q.z; out[6] = q.w;
  out[7] = sp * sl;
}

// ---- The same joint state in three data-parallel passes (what the kernels run) -----------------------------------------------
// JointStateT::set mixes work that needs the parent (two compositions) with work that does not (three sin/cos pairs, the local
// rotation chain, exp2). Splitting it lets every joint of the skeleton do the expensive part at once, leaves ~50 dependent
// flops per tree level, and turns the derivative axes into one more flat pass:
//   fkLocal   (all joints)         t_l, q_l = preRot Rz Ry Rx, s_l, and the DOF axes in the PARENT frame: a_2 = preRot z, a_1 = (preRot Rz) y,
//                                  a_0 = (preRot Rz Ry) x                                                   (joint_state.cpp:44-62)
//   fkCompose (level by level)     t = t_p + q_p (s_p t_l), q = q_p q_l, s = s_p s_l                          (transform.h:124-129)
//   fkAxis    (all joints x 3)     rotationAxis.col(i) = q_p a_i   [= (q_p preRot ...) e_i of joint_state.cpp:51-55: one rotation of a
//                                  rotated vector instead of a rotation by a quaternion product; equal up to rounding]
// fkJoint above stays the statement-by-statement form (CPU emulation of the oracle order, tests).
// out: the joint's own slot (8 floats, or kJointStateStride with kDeriv)
template <bool kDeriv>
MB2_HD void fkLocalFromParameters(const CharacterTables& T, int j, const float* p, float* out);
template <bool kDeriv>
MB2_HD void fkLocal(const CharacterTables& T, int j, const float* jp, float* js) {
  fkLocalFromParameters<kDeriv>(T, j, jp + j * kParametersPerJoint, js + j * kJointStateStride);
}
// the joint's seven parameters straight from theta (ParameterTransform rows 7 j .. 7 j + 6): no [7 J] array in shared memory, and the
// transform is spread over lanes = joints (three rounds for 72 joints) instead of lanes = rows (sixteen rounds of dependent loads)
template <bool kDeriv>
MB2_HD void fkLocalFromTheta(const CharacterTables& T, int j, const float* theta, float* js) {
  float p[kParametersPerJoint];
#pragma unroll
  for (int r = 0; r < kParametersPerJoint; ++r) p[r] = jointParameterRow(T, j * kParametersPerJoint + r, theta);
  fkLocalFromParameters<kDeriv>(T, j, p, js + j * kJointStateStride);
}
// jp == nullptr: the caller keeps no joint-parameter array (same value, recomputed from theta)
MB2_HD float jointParameterAt(const CharacterTables& T, const float* jp, const float* theta, int row) { return jp != nullptr ? jp[row] : jointParameterRow(T, row, theta); }
template <bool kDeriv>
MB2_HD void fkLocalFromParameters(const CharacterTables& T, int j, const float* p, float* out) {
  Q4 ql = ld4(T.prerot + 4 * j);
#pragma unroll
  for (int index = 2; index >= 0; --index) {
    if (kDeriv) {
      const F3 a = qrot(ql, f3(index == 0 ? 1.f : 0.f, index == 1 ? 1.f : 0.f, index == 2 ? 1.f : 0.f));
      out[8 + 3 * index] = a.x; out[9 + 3 * index] = a.y; out[10 + 3 * index] = a.z;
    }
    const float ha = 0.5f * p[3 + index];
    float sn, cs;
#if defined(__CUDA_ARCH__)
    sincosf(ha, &sn, &cs);
#else
    sn = sinf(ha); cs = cosf(ha);
#endif
    ql = qmul(ql, q4(index == 0 ? sn : 0.f, index == 1 ? sn : 0.f, index == 2 ? sn : 0.f, cs));
  }
  out[0] = T.offset[3 * j] + p[0]; out[1] = T.offset[3 * j + 1] + p[1]; out[2] = T.offset[3 * j + 2] + p[2];
  out[3] = ql.x; out[4] = ql.y; out[5] = ql.z; out[6] = ql.w;
  out[7] = exp2f(p[6]);
}
// the parent (if any) already holds its world transform
MB2_HD void fkCompose(const CharacterTables& T, int j, float* js) {
  const int par = T.parent[j];
  if (par < 0) return; // identity parent: world = local, bit for bit
  const float* ps = js + par * kJointStateStride;
  float* out = js + j * kJointStateStride;
  const F3 tp = ld3(ps);
  const Q4 qp = ld4(ps + 3);
  const float sp = ps[7];
  const F3 t = tp + qrot(qp, sp * ld3(out));
  const Q4 q = qmul(qp, ld4(out + 3));
  out[0] = t.x; out[1] = t.y; out[2] = t.z;
  out[3] = q.x; out[4] = q.y; out[5] = q.z; out[6] = q.w;
  out[7] = sp * out[7];
}
// after every joint is composed: world direction of DOF axis `index` of joint j
MB2_HD void fkAxis(const CharacterTables& T, int j, int index, float* js) {
  const int par = T.parent[j];
  if (par < 0) return;
  float* a = js + j * kJointStateStride + 8 + 3 * index;
  const F3 w = qrot(ld4(js + par * kJointStateStride + 3), ld3(a));
  a[0] = w.x; a[1] = w.y; a[2] = w.z;
}

// translationAxis of joint a = parent.toLinear() (joint_state.cpp:36-42), column d
MB2_HD F3 translationAxisCol(const CharacterTables& T, const float* js, int a, int d) {
  const int par = T.parent[a];
  if (par < 0) return f3(d == 0 ? 1.f : 0.f, d == 1 ? 1.f : 0.f, d == 2 ? 1.f : 0.f);
  const float* ps = js + par * kJointStateStride;
  return qmatcol(ld4(ps + 3), d) * ps[7];
}
MB2_HD F3 rotationAxisCol(const float* js, int a, int d) { return ld3(js + a * kJointStateStride + 8 + 3 * d); }

// derivative of a world point v attached below joint a w.r.t. joint-parameter dof d
// (joint_state.cpp:68-82 + joint_error_function-inl.h:240-291)
MB2_HD F3 pointDerivative(const CharacterTables& T, const float* js, int a, int d, F3 v) {
  if (d < 3) return translationAxisCol(T, js, a, d);
  const F3 off = v - ld3(js + a * kJointStateStride);
  if (d < 6) return cross(rotationAxisCol(js, a, d - 3), off);
  return off * kLn2;
}

// ---- Backward of the skeleton state (t, q = (v, w), s) of every joint with respect to the model parameters ----
// Each joint-parameter DOF of joint a moves the joints of its subtree sub(a) rigidly (the same derivatives pointDerivative uses):
//   translation k:  dt_i = B_a e_k                      (B_a = translationAxisCol)
//   rotation k:     dt_i = w x (t_i - t_a), dq_i = 1/2 (w, 0) (x) q_i   (w = rotationAxisCol k)
//   scale:          dt_i = ln2 (t_i - t_a), ds_i = ln2 s_i
// so with the upstream gradient G_i = (g_t, g_v, g_w, g_s) every joint needs 11 subtree sums, accumulated once from the leaves up
// (O(J) instead of one ancestor walk per joint and DOF):
//   [0..2] S_g = sum g_t    [3..5] R = sum (t_i - t_a) x g_t    [6] D = sum (t_i - t_a) . g_t
//   [7..9] S_c = sum 1/2 (w_i g_v + v_i x g_v - g_w v_i)        [10] S_s = sum s_i g_s
// R and D are kept relative to the joint's own origin and shifted once per child edge: the form sum t_i x g - t_a x sum g cancels
// catastrophically for a rig far from the origin.
// (kSkelAccStride, ik_types.h: the 11 floats above per joint)

// the joint's own term (its subtree before any child is folded in); g: the joint's 8 upstream gradient floats
MB2_HD void skelGradSeed(const float* js, int i, const float* g, float* acc) {
  const float* ps = js + i * kJointStateStride;
  const F3 v = ld3(ps + 3), gv = ld3(g + 3);
  const float w = ps[6], gw = g[6];
  const F3 sc = 0.5f * (w * gv + cross(v, gv) - gw * v);
  float* a = acc + i * kSkelAccStride;
  a[0] = g[0]; a[1] = g[1]; a[2] = g[2];
  a[3] = 0.f; a[4] = 0.f; a[5] = 0.f; a[6] = 0.f;
  a[7] = sc.x; a[8] = sc.y; a[9] = sc.z;
  a[10] = ps[7] * g[7];
}
// adds the children's finished subtree sums to joint a, children in ascending index order (deterministic)
MB2_HD void skelGradFold(const SkeletonTables& S, const float* js, int a, float* acc) {
  float* A = acc + a * kSkelAccStride;
  const F3 ta = ld3(js + a * kJointStateStride);
  F3 sg = ld3(A), r = ld3(A + 3), sc = ld3(A + 7);
  float d = A[6], ss = A[10];
  for (int k = S.childStart[a]; k < S.childStart[a + 1]; ++k) {
    const int c = S.children[k];
    const float* C = acc + c * kSkelAccStride;
    const F3 off = ld3(js + c * kJointStateStride) - ta, sgc = ld3(C);
    r = r + (ld3(C + 3) + cross(off, sgc));
    d = d + (C[6] + dot(off, sgc));
    sg = sg + sgc;
    sc = sc + ld3(C + 7);
    ss = ss + C[10];
  }
  A[0] = sg.x; A[1] = sg.y; A[2] = sg.z;
  A[3] = r.x; A[4] = r.y; A[5] = r.z; A[6] = d;
  A[7] = sc.x; A[8] = sc.y; A[9] = sc.z; A[10] = ss;
}
// dLoss / d joint parameter `row` (= 7 a + k) from the finished sums of joint a; js holds the world state and DOF axes (fkAxis)
MB2_HD float skelGradJointParameter(const CharacterTables& T, const float* js, const float* acc, int row) {
  const int a = row / kParametersPerJoint, k = row - a * kParametersPerJoint;
  const float* A = acc + a * kSkelAccStride;
  if (k < 3) return dot(translationAxisCol(T, js, a, k), ld3(A));
  if (k < 6) return dot(rotationAxisCol(js, a, k - 3), ld3(A + 3) + ld3(A + 7));
  return kLn2 * (A[6] + A[10]);
}
// dLoss / d model parameter p = column p of the ParameterTransform against the joint-parameter gradient, rows ascending
MB2_HD float skelGradModelParameter(const SkeletonTables& S, const float* gjp, int p) {
  float s = 0.f;
  for (int k = S.ptColStart[p]; k < S.ptColStart[p + 1]; ++k) s += S.ptColVals[k] * gjp[S.ptColRows[k]];
  return s;
}

// ---- Points fixed in joints' frames (pymomentum jointParametersToPositions, tensor_joint_parameters_to_positions.cpp:33-119) ----------
// Point i on joint a (ps: a's world state): p_i = t_a + d_i with d_i = rot(q_a, s_a off_i), the position constraint's point
// (transform.h:193-195). A point moves rigidly with its joint, so its backward is the skeleton-state backward seeded from the points
// instead of a state gradient: joint a's own term is S_g = sum g_i, R = sum d_i x g_i, D = sum d_i . g_i, S_c = S_s = 0. d_i is the
// rotated and scaled offset, never p_i - t_a, which cancels catastrophically for a rig far from the origin.
MB2_HD F3 pointRelative(const float* ps, F3 off) { return qrot(ld4(ps + 3), ps[7] * off); }
// dLoss / d off_i = s_a R_a^T g_i
MB2_HD F3 pointOffsetGradient(const float* ps, F3 g) { return ps[7] * qrot(qconj(ld4(ps + 3)), g); }
// joint a's seed in skelGradSeed's layout from its own points, in the order of P.pointIndex; off [N][3], g [N][3] dLoss / d p
MB2_HD void pointGradSeed(const PointTables& P, const float* js, int a, const float* off, const float* g, float* acc) {
  const float* ps = js + a * kJointStateStride;
  F3 sg = f3(0.f, 0.f, 0.f), r = sg;
  float d = 0.f;
#pragma unroll 1
  for (int k = P.pointStart[a]; k < P.pointStart[a + 1]; ++k) {
    const int i = P.pointIndex[k];
    const F3 di = pointRelative(ps, ld3(off + 3 * i)), gi = ld3(g + 3 * i);
    sg = sg + gi;
    r = r + cross(di, gi);
    d = d + dot(di, gi);
  }
  float* A = acc + a * kSkelAccStride;
  A[0] = sg.x; A[1] = sg.y; A[2] = sg.z;
  A[3] = r.x; A[4] = r.y; A[5] = r.z; A[6] = d;
  A[7] = 0.f; A[8] = 0.f; A[9] = 0.f; A[10] = 0.f;
}
// A gradient of an input shared by the batch (skin_points' rest points, the positions' offsets) is the batch sum of per-instance terms:
// summed in instance order within chunks of this many instances, at most kBatchSumChunks of them, then chunk by chunk in order. The
// chunking depends on the batch size only.
constexpr int kBatchSumChunks = 128;
MB2_HD int batchSumChunk(int batch) {
  const int c = batch / kBatchSumChunks + (batch % kBatchSumChunks != 0);
  return c > 8 ? c : 8;
}

// ---- Joint parameters <-> local and world skeleton states, one joint at a time (pymomentum tensor_skeleton_state.cpp:139-185, :346-498,
// :589-668, tensor_transforms.cpp:86-164, tensor_quaternion.cpp:179-230) ----------------------------------------------------------------
// The local state of joint j from its seven parameters is fkLocalFromParameters. Its backward, from the kDeriv local state ls (the DOF
// axes a_k in the parent frame after t, q, s): g_p[0..2] = g_t; g_p[3+k] = a_k . 1/2 (w g_v + v x g_v - g_w v), since
// dq/dp[3+k] = 1/2 (a_k, 0) (x) q for a unit pre-rotation (the S_c term of skelGradSeed); g_p[6] = ln2 s g_s.
MB2_HD void localStateGradient(const float* ls, const float* g, float* gp) {
  const F3 v = ld3(ls + 3), gv = ld3(g + 3);
  const float w = ls[6], gw = g[6];
  const F3 sc = 0.5f * (w * gv + cross(v, gv) - gw * v);
  gp[0] = g[0]; gp[1] = g[1]; gp[2] = g[2];
  for (int k = 0; k < 3; ++k) gp[3 + k] = dot(ld3(ls + 8 + 3 * k), sc);
  gp[6] = kLn2 * (ls[7] * g[7]);
}

// pymomentum's quaternion inverse conj(q) / |q|^2 and rotation v + 2 (w (u x v) + u x (u x v)), as written: neither normalises q
MB2_HD Q4 qinverse(Q4 q) {
  const float n2 = q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w;
  return q4(-q.x / n2, -q.y / n2, -q.z / n2, q.w / n2);
}
MB2_HD F3 qrotWritten(Q4 q, F3 v) {
  const F3 u = f3(q.x, q.y, q.z);
  const F3 av = cross(u, v), aav = cross(u, av);
  return v + 2.f * (av * q.w + aav);
}
// the asin argument clamped to [-1, 1]; a NaN passes through (fminf / fmaxf would replace it)
MB2_HD float clampUnit(float a) { return a > 1.f ? 1.f : (a < -1.f ? -1.f : a); }

// joint parameters p [7] of joint j from its local state ls [8] (localSkeletonStateToJointParameters, :611-648): t - offset_j, the XYZ
// Euler angles of r = inv(preRot_j) (x) q (quaternionToXYZEuler, on r as it is, unit or not), log2 s
MB2_HD void jointParametersFromLocal(const CharacterTables& T, int j, const float* ls, float* p) {
  p[0] = ls[0] - T.offset[3 * j]; p[1] = ls[1] - T.offset[3 * j + 1]; p[2] = ls[2] - T.offset[3 * j + 2];
  const Q4 r = qmul(qinverse(ld4(T.prerot + 4 * j)), ld4(ls + 3));
  p[3] = atan2f(2.f * (r.w * r.x + r.y * r.z), 1.f - 2.f * (r.x * r.x + r.y * r.y));
  p[4] = asinf(clampUnit(2.f * (r.w * r.y - r.z * r.x)));
  p[5] = atan2f(2.f * (r.w * r.z + r.x * r.y), 1.f - 2.f * (r.y * r.y + r.z * r.z));
  p[6] = log2f(ls[7]);
}
// its backward: g [8] = (dp / d ls)^T gp. d atan2(Y, X) = (X dY - Y dX) / (X^2 + Y^2), skipped for a zero upstream angle gradient (at
// gimbal lock X = Y = 0 can hold exactly, and 0 / 0 would turn the other angles' gradient into NaN); d asin(A) = dA / sqrt(1 - A^2), 0
// where the clamp holds (|A| >= 1); r is linear in q, so g_q = conj(inv(preRot)) (x) g_r; d log2 s = ds / (s ln2)
MB2_HD void jointParametersFromLocalGradient(const CharacterTables& T, int j, const float* ls, const float* gp, float* g) {
  g[0] = gp[0]; g[1] = gp[1]; g[2] = gp[2];
  const Q4 pinv = qinverse(ld4(T.prerot + 4 * j));
  const Q4 r = qmul(pinv, ld4(ls + 3));
  float gx, gy, gz, gw;
  { // rx = atan2(Y, X), Y = 2 (w x + y z), X = 1 - 2 (x^2 + y^2)
    const float Y = 2.f * (r.w * r.x + r.y * r.z), X = 1.f - 2.f * (r.x * r.x + r.y * r.y);
    const float c = gp[3] == 0.f ? 0.f : gp[3] / (X * X + Y * Y), cY = c * X, cX = -c * Y;
    gx = 2.f * cY * r.w - 4.f * cX * r.x; gy = 2.f * cY * r.z - 4.f * cX * r.y; gz = 2.f * cY * r.y; gw = 2.f * cY * r.x;
  }
  { // ry = asin(A), A = 2 (w y - z x)
    const float A = 2.f * (r.w * r.y - r.z * r.x);
    const float cA = (A >= 1.f || A <= -1.f) ? 0.f : gp[4] / sqrtf(1.f - A * A);
    gx -= 2.f * cA * r.z; gy += 2.f * cA * r.w; gz -= 2.f * cA * r.x; gw += 2.f * cA * r.y;
  }
  { // rz = atan2(Z, W), Z = 2 (w z + x y), W = 1 - 2 (y^2 + z^2)
    const float Z = 2.f * (r.w * r.z + r.x * r.y), W = 1.f - 2.f * (r.y * r.y + r.z * r.z);
    const float c = gp[5] == 0.f ? 0.f : gp[5] / (W * W + Z * Z), cZ = c * W, cW = -c * Z;
    gx += 2.f * cZ * r.y; gy += 2.f * cZ * r.x - 4.f * cW * r.y; gz += 2.f * cZ * r.w - 4.f * cW * r.z; gw += 2.f * cZ * r.z;
  }
  const Q4 gq = qmul(qconj(pinv), q4(gx, gy, gz, gw));
  g[3] = gq.x; g[4] = gq.y; g[5] = gq.z; g[6] = gq.w;
  g[7] = gp[6] / (ls[7] * kLn2);
}

// local state ls [8] of joint j from the world states X [J][8] of its instance (skeletonStateToJointParameters, :650-668):
// inv(X_parent) o X_j, with inv(t, q, s) = (-s^-1 rot(q^-1, t), q^-1, s^-1) and (t1, q1, s1) o (t2, q2, s2) = (t1 + rot(q1, s1 t2),
// q1 (x) q2, s1 s2) as written; above a root is the identity, so a root's local state is its world state
MB2_HD void localFromWorld(const CharacterTables& T, int j, const float* X, float* ls) {
  const float* c = X + 8 * j;
  const int par = T.parent[j];
  if (par < 0) {
    for (int k = 0; k < 8; ++k) ls[k] = c[k];
    return;
  }
  const float* P = X + 8 * par;
  const Q4 qi = qinverse(ld4(P + 3));
  const float si = 1.f / P[7];
  const F3 t = (-si) * qrotWritten(qi, ld3(P)) + qrotWritten(qi, si * ld3(c));
  const Q4 q = qmul(qi, ld4(c + 3));
  ls[0] = t.x; ls[1] = t.y; ls[2] = t.z;
  ls[3] = q.x; ls[4] = q.y; ls[5] = q.z; ls[6] = q.w;
  ls[7] = si * c[7];
}
// The backward of local = inv(P) o C for the local state's gradient gl [8], with qi = q_P^-1, si = 1 / s_P, d = t_C - t_P and
// M = rot(qi, .), so that t = si M d, q = qi q_C, s = si s_C (M^T h = rot(conj(qi), h)):
//   to C (written): g_tC = si M^T g_t, g_qC = conj(qi) (x) g_q, g_sC = si g_s
MB2_HD void localFromWorldChildGradient(const float* P, const float* gl, float* gc) {
  const Q4 qi = qinverse(ld4(P + 3));
  const float si = 1.f / P[7];
  const F3 gt = qrotWritten(qconj(qi), si * ld3(gl));
  const Q4 gq = qmul(qconj(qi), ld4(gl + 3));
  gc[0] = gt.x; gc[1] = gt.y; gc[2] = gt.z;
  gc[3] = gq.x; gc[4] = gq.y; gc[5] = gq.z; gc[6] = gq.w;
  gc[7] = si * gl[7];
}
//   to P (added to gp): g_tP = -si M^T g_t, g_sP = -si (g_t . t + g_s s), and through qi: g_qi = g_q (x) conj(q_C) + d/dqi [h . rot(qi, d)]
//   (h = si g_t: 2 h . (u x d) for w; 2 w (d x h) + 2 (u . d) h + 2 (h . u) d - 4 (h . d) u for u), g_qP = (conj(g_qi) - 2 (qi . g_qi) q_P) / |q_P|^2
MB2_HD void localFromWorldParentGradient(const float* P, const float* C, const float* ls, const float* gl, float* gp) {
  const Q4 qp = ld4(P + 3);
  const Q4 qi = qinverse(qp);
  const float si = 1.f / P[7];
  const F3 h = si * ld3(gl), d = ld3(C) - ld3(P), u = f3(qi.x, qi.y, qi.z);
  const F3 gt = qrotWritten(qconj(qi), h);
  const Q4 gqc = qmul(ld4(gl + 3), qconj(ld4(C + 3)));
  const F3 gu = 2.f * (qi.w * cross(d, h) + dot(u, d) * h + dot(h, u) * d) - 4.f * dot(h, d) * u;
  const Q4 gqi = q4(gqc.x + gu.x, gqc.y + gu.y, gqc.z + gu.z, gqc.w + 2.f * dot(h, cross(u, d)));
  const float n2 = qp.x * qp.x + qp.y * qp.y + qp.z * qp.z + qp.w * qp.w;
  const float dq = 2.f * (qi.x * gqi.x + qi.y * gqi.y + qi.z * gqi.z + qi.w * gqi.w);
  gp[0] -= gt.x; gp[1] -= gt.y; gp[2] -= gt.z;
  gp[3] += (-gqi.x - dq * qp.x) / n2; gp[4] += (-gqi.y - dq * qp.y) / n2; gp[5] += (-gqi.z - dq * qp.z) / n2;
  gp[6] += (gqi.w - dq * qp.w) / n2;
  gp[7] -= si * (dot(ld3(gl), ld3(ls)) + gl[7] * ls[7]);
}
// dLoss / d X_j [8] from the joint-parameter gradient gjp [J][7] of the instance: the own local's term, then for each child in ascending
// index order the term of its local with respect to its parent (no atomics: every output is gathered by one thread)
MB2_HD void worldStateGradient(const CharacterTables& T, const SkeletonTables& S, int j, const float* X, const float* gjp, float* gX) {
  float ls[8], gl[8];
  localFromWorld(T, j, X, ls);
  jointParametersFromLocalGradient(T, j, ls, gjp + kParametersPerJoint * j, gl);
  if (T.parent[j] < 0)
    for (int k = 0; k < 8; ++k) gX[k] = gl[k];
  else
    localFromWorldChildGradient(X + 8 * T.parent[j], gl, gX);
  for (int k = S.childStart[j]; k < S.childStart[j + 1]; ++k) {
    const int c = S.children[k];
    localFromWorld(T, c, X, ls);
    jointParametersFromLocalGradient(T, c, ls, gjp + kParametersPerJoint * c, gl);
    localFromWorldParentGradient(X + 8 * j, X + 8 * c, ls, gl, gX);
  }
}

// Model parameter p of the joint parameters jp [7 J] of one instance (InverseParameterTransform::apply,
// inverse_parameter_transform.cpp:30-38): theta_p = sum_k W_pk (jp_k - o_k) over W's entries in table order, the offsets subtracted
// before the product
MB2_HD float inverseParameterRow(const CharacterTables& T, const SkeletonTables& S, int p, const float* jp) {
  float s = 0.f;
  for (int k = S.invStart[p]; k < S.invStart[p + 1]; ++k) {
    const int r = S.invRows[k];
    s += S.invVals[k] * (jp[r] - T.ptOffsets[r]);
  }
  return s;
}
// its backward for joint-parameter row r from dLoss / d theta [n]: (W^T g)_r over the row's entries, parameters ascending
MB2_HD float inverseParameterGradient(const SkeletonTables& S, int r, const float* gTheta) {
  float s = 0.f;
  for (int k = S.invRowStart[r]; k < S.invRowStart[r + 1]; ++k) s += S.invRowVals[k] * gTheta[S.invParams[k]];
  return s;
}

// The flat operations of a batch (JointOp), one element per thread: kOp's per-instance item count (rows, parameters or joints) and
// element i of the batch, for input `in`, upstream gradient `grad` (backward) and output `out`, every array [B][...] dense.
template <int kOp, bool kBackward>
MB2_HD int jointOpItems(const CharacterTables& T) {
  if constexpr (kOp == kJointOpParameterTransform) return kBackward ? T.numParams : T.numJoints * kParametersPerJoint;
  else if constexpr (kOp == kJointOpInverseParameterTransform) return kBackward ? T.numJoints * kParametersPerJoint : T.numParams;
  else if constexpr (kOp == kJointOpClampParameters) return T.numParams;
  else return T.numJoints;
}
template <int kOp, bool kBackward>
MB2_HD void jointOpElement(const CharacterTables& T, const SkeletonTables& S, long i, const float* in, const float* grad, float* out) {
  const int per = jointOpItems<kOp, kBackward>(T);
  const long b = i / per;
  const int k = int(i - b * per), J = T.numJoints, n = T.numParams;
  if constexpr (kOp == kJointOpParameterTransform) {
    if constexpr (kBackward) out[i] = skelGradModelParameter(S, grad + b * (7L * J), k);
    else out[i] = jointParameterRow(T, k, in + b * n);
  } else if constexpr (kOp == kJointOpInverseParameterTransform) {
    if constexpr (kBackward) out[i] = inverseParameterGradient(S, k, grad + b * n);
    else out[i] = inverseParameterRow(T, S, k, in + b * (7L * J));
  } else if constexpr (kOp == kJointOpClampParameters) {
    // pymomentum apply_model_param_limits (tensor_parameter_transform.cpp:638-697): torch.clamp of the limited parameters, which keeps
    // NaN and passes the gradient where min <= theta <= max
    const float* c = S.paramClamp + 3 * k;
    const float x = in[i];
    if constexpr (kBackward) out[i] = c[2] == 0.f || (x >= c[0] && x <= c[1]) ? grad[i] : 0.f;
    else out[i] = c[2] == 0.f || x != x ? x : fminf(fmaxf(x, c[0]), c[1]);
  } else if constexpr (kOp == kJointOpLocalState) {
    if constexpr (kBackward) {
      float ls[kJointStateStride];
      fkLocalFromParameters<true>(T, k, in + 7 * i, ls);
      localStateGradient(ls, grad + 8 * i, out + 7 * i);
    } else {
      fkLocalFromParameters<false>(T, k, in + 7 * i, out + 8 * i);
    }
  } else if constexpr (kOp == kJointOpFromLocal) {
    if constexpr (kBackward) jointParametersFromLocalGradient(T, k, in + 8 * i, grad + 7 * i, out + 8 * i);
    else jointParametersFromLocal(T, k, in + 8 * i, out + 7 * i);
  } else {
    const float* X = in + b * (8L * J);
    if constexpr (kBackward) {
      worldStateGradient(T, S, k, X, grad + b * (7L * J), out + 8 * i);
    } else {
      float ls[8];
      localFromWorld(T, k, X, ls);
      jointParametersFromLocal(T, k, ls, out + 7 * i);
    }
  }
}

// ---- Input contractions of the implicit-function backward of solve_ik: d/d input [grad_theta E_c . v] ----
// Under the parameter direction v every joint moves rigidly: angular velocity w, log-scale rate sigma, origin velocity tdot. With the
// joint-parameter velocity u = P v (linear part of the ParameterTransform; its offsets do not move) and pi = parent(j):
//   w_j = w_pi + sum_k u[7j+3+k] A_jk,   sigma_j = sigma_pi + ln2 u[7j+6],
//   tdot_j = tdot_pi + w_pi x (t_j - t_pi) + sigma_pi (t_j - t_pi) + sum_k u[7j+k] B_jk
// (A = rotationAxisCol, B = translationAxisCol; zero motion above a root). A point p attached to j moves at
// pdot = tdot_j + w_j x (p - t_j) + sigma_j (p - t_j) = J_c v. t_j - t_pi stays relative (no cancellation for a rig far from the origin).
// (kTangentStride, ik_types.h: w(3) sigma tdot(3) per joint)

// u[row] = (P v)[row] without ptOffsets (jointParameterRow adds them)
MB2_HD float tangentJointParameter(const CharacterTables& T, int row, const float* v) {
  float s = 0.f;
  for (int k = T.ptOuter[row]; k < T.ptOuter[row + 1]; ++k) s += T.ptVals[k] * v[T.ptInner[k]];
  return s;
}
// the joint's own share of its motion (all joints at once; js holds the world state and DOF axes, fkAxis)
MB2_HD void tangentLocal(const CharacterTables& T, const float* js, int j, const float* v, float* tan) {
  const int r0 = j * kParametersPerJoint;
  F3 w = f3(0.f, 0.f, 0.f), td = f3(0.f, 0.f, 0.f);
  for (int k = 0; k < 3; ++k) {
    td = td + translationAxisCol(T, js, j, k) * tangentJointParameter(T, r0 + k, v);
    w = w + rotationAxisCol(js, j, k) * tangentJointParameter(T, r0 + 3 + k, v);
  }
  float* o = tan + j * kTangentStride;
  o[0] = w.x; o[1] = w.y; o[2] = w.z;
  o[3] = kLn2 * tangentJointParameter(T, r0 + 6, v);
  o[4] = td.x; o[5] = td.y; o[6] = td.z;
}
// level by level from the roots: adds the (finished) parent's motion to the joint's own share
MB2_HD void tangentCompose(const CharacterTables& T, const float* js, int j, float* tan) {
  const int par = T.parent[j];
  if (par < 0) return;
  const float* P = tan + par * kTangentStride;
  float* o = tan + j * kTangentStride;
  const F3 wp = ld3(P), off = ld3(js + j * kJointStateStride) - ld3(js + par * kJointStateStride);
  const float sp = P[3];
  const F3 w = wp + ld3(o);
  const F3 td = ld3(P + 4) + cross(wp, off) + sp * off + ld3(o + 4);
  o[0] = w.x; o[1] = w.y; o[2] = w.z;
  o[3] = sp + o[3];
  o[4] = td.x; o[5] = td.y; o[6] = td.z;
}

// ---- Lane groups and the per-instance pass sequences -------------------------------------------------------------------------
// A lane group is the set of lanes that work on one instance: `lane` in [0, size) and sync(), the barrier between two passes. The pass
// functions below state each pass sequence with its barriers once, for the kernels and for the CPU emulators (tests/emu), which run
// them with HostLanes. Only reduction-free passes are shared: within a pass no lane reads what another lane of the pass writes, so one
// lane running every index in order computes the same bits.
struct HostLanes {
  static constexpr int size = 1, lane = 0;
  MB2_HD void sync() const {}
};
#if defined(__CUDACC__)
// W warps of a CTA per instance; group = warp / W waits on named barrier 1 + group (0 is __syncthreads), a single warp on __syncwarp
template <int W>
struct WarpLanes {
  static constexpr int size = 32 * W;
  int group, lane;
  __device__ static WarpLanes of(int warp, int lane) { return {warp / W, (warp % W) * 32 + lane}; } // warp, lane of the CTA
  MB2_HD void sync() const {
#if defined(__CUDA_ARCH__)
    if (W == 1) __syncwarp();
    else asm volatile("bar.sync %0, %1;" ::"r"(1 + group), "r"(size) : "memory");
#endif
  }
};
// the whole CTA of kThreads threads on one instance
template <int kThreads>
struct CtaLanes {
  static constexpr int size = kThreads;
  int lane;
  MB2_HD void sync() const {
#if defined(__CUDA_ARCH__)
    __syncthreads();
#endif
  }
};
#endif

// SkeletonState::set of one instance in the three data-parallel passes above: the local part of every joint, its joint parameters
// computed from theta or (kFromJointParameters) read from a staged [7 J] array, then the composition level by level from the roots, then
// (kAxes) the DOF axes in world space. The axes pass ends without a barrier, so that the caller's next pass can share it.
template <bool kAxes, bool kFromJointParameters, class Lanes>
MB2_HD void fkPasses(const Lanes& g, const CharacterTables& C, const float* src, float* js) {
  for (int j = g.lane; j < C.numJoints; j += g.size) {
    if constexpr (kFromJointParameters) fkLocal<kAxes>(C, j, src, js);
    else fkLocalFromTheta<kAxes>(C, j, src, js);
  }
  g.sync();
  for (int lvl = 1; lvl < C.numLevels; ++lvl) { // level 0 = roots: world = local
    const int end = C.levelStart[lvl + 1];
    for (int k = C.levelStart[lvl] + g.lane; k < end; k += g.size) fkCompose(C, C.levelJoints[k], js);
    g.sync();
  }
  if constexpr (kAxes)
    for (int i = g.lane; i < 3 * C.numJoints; i += g.size) fkAxis(C, i / 3, i % 3, js);
}

// The tail of the skeleton-state backward of one instance, once every joint's seed is in acc and a barrier has passed: the levels from
// the deepest up fold in their children, lanes = joint-parameter rows into gjp [7 J], lanes = model parameters into out [n]
// (out == nullptr: stops after gjp). Ends without a barrier.
template <class Lanes>
MB2_HD void skelGradTail(const Lanes& g, const CharacterTables& C, const SkeletonTables& S, const float* js, float* acc, float* gjp, float* out) {
  for (int lvl = C.numLevels - 2; lvl >= 0; --lvl) { // the deepest level has no children
    const int end = C.levelStart[lvl + 1];
    for (int k = C.levelStart[lvl] + g.lane; k < end; k += g.size) skelGradFold(S, js, C.levelJoints[k], acc);
    g.sync();
  }
  for (int row = g.lane; row < C.numJoints * kParametersPerJoint; row += g.size) gjp[row] = skelGradJointParameter(C, js, acc, row);
  if (out == nullptr) return; // the joint-parameter gradient is the result (joint_parameters_to_skeleton_state)
  g.sync();
  for (int p = g.lane; p < C.numParams; p += g.size) out[p] = skelGradModelParameter(S, gjp, p);
}

// The skeleton-state backward of one instance, right after fkPasses<true> (fkAxis writes only the axes and the seed reads only t, q, s:
// the seed shares the axes' barrier): every joint seeds its subtree sums from the upstream gradient grad [J][8], then skelGradTail.
template <class Lanes>
MB2_HD void skelGradPasses(const Lanes& g, const CharacterTables& C, const SkeletonTables& S, const float* js, const float* grad, float* acc,
                           float* gjp, float* out) {
  for (int i = g.lane; i < C.numJoints; i += g.size) skelGradSeed(js, i, grad + 8 * i, acc);
  g.sync();
  skelGradTail(g, C, S, js, acc, gjp, out);
}

// The positions [N][3] of one instance's points with offsets off [N][3], lanes = points, once fkPasses<false> has ended (with its
// barrier). Ends without a barrier.
template <class Lanes>
MB2_HD void positionPasses(const Lanes& g, const PointTables& P, const float* js, const float* off, float* out) {
  for (int i = g.lane; i < P.numPoints; i += g.size) {
    const float* ps = js + P.parent[i] * kJointStateStride;
    const F3 p = ld3(ps) + pointRelative(ps, ld3(off + 3 * i));
    out[3 * i] = p.x; out[3 * i + 1] = p.y; out[3 * i + 2] = p.z;
  }
}

// Their backward from grad [N][3], right after fkPasses<true>: lanes = points write dLoss / d off into gOff [N][3] (when set), and every
// joint seeds its subtree sums from its points (when gjp is set), both reading only t, q, s, so they share the axes' barrier; then
// skelGradTail into gjp and out. Ends without a barrier.
template <class Lanes>
MB2_HD void positionGradPasses(const Lanes& g, const CharacterTables& C, const SkeletonTables& S, const PointTables& P, const float* js,
                               const float* off, const float* grad, float* acc, float* gjp, float* out, float* gOff) {
  if (gOff != nullptr)
#pragma unroll 1
    for (int i = g.lane; i < P.numPoints; i += g.size) {
      const F3 r = pointOffsetGradient(js + P.parent[i] * kJointStateStride, ld3(grad + 3 * i));
      gOff[3 * i] = r.x; gOff[3 * i + 1] = r.y; gOff[3 * i + 2] = r.z;
    }
  if (gjp == nullptr) return;
  for (int j = g.lane; j < C.numJoints; j += g.size) pointGradSeed(P, js, j, off, grad, acc);
  g.sync();
  skelGradTail(g, C, S, js, acc, gjp, out);
}

// The joint motions of one instance under the parameter direction v (js: world state and DOF axes, complete): every joint's own share,
// then the parent's motion added level by level from the roots. Ends with a barrier.
template <class Lanes>
MB2_HD void tangentPasses(const Lanes& g, const CharacterTables& C, const float* js, const float* v, float* tan) {
  for (int j = g.lane; j < C.numJoints; j += g.size) tangentLocal(C, js, j, v, tan);
  g.sync();
  for (int lvl = 1; lvl < C.numLevels; ++lvl) {
    const int end = C.levelStart[lvl + 1];
    for (int k = C.levelStart[lvl] + g.lane; k < end; k += g.size) tangentCompose(C, js, C.levelJoints[k], tan);
    g.sync();
  }
}

// Position constraint (L2), p = t_j + s_j R_j o, d = p - t, W = e.weight w_c / c^2, g = 2 W d . pdot:
//   dg/dw_c = 2 e.weight / c^2 d . pdot,   dg/dt = -2 W pdot,   dg/do = 2 W s_j R_j^T (pdot - w_j x d + sigma_j d)
// tg: the constraint's target record (xyz, then the offset for an instanced block). Null outputs are skipped.
MB2_HD void positionInputGradient(const UnitDesc& u, const EfDesc& e, const float* js, const float* tan, const float* tg, float cw, float* gW,
                                  float* gO, float* gT) {
  const float* ps = js + u.joint * kJointStateStride;
  const float* tj = tan + u.joint * kTangentStride;
  const Q4 q = ld4(ps + 3);
  const float s = ps[7];
  const F3 off = u.pad[2] != 0 ? f3(tg[3], tg[4], tg[5]) : f3(u.f[0], u.f[1], u.f[2]);
  const F3 rel = qrot(q, s * off); // p - t_j
  const F3 d = ld3(ps) + rel - ld3(tg);
  const F3 w = ld3(tj);
  const float sg = tj[3];
  const F3 pdot = ld3(tj + 4) + cross(w, rel) + sg * rel;
  const float ew = e.weight * e.invC2, W = ew * cw;
  if (gW) gW[0] = 2.f * ew * dot(d, pdot);
  if (gT) { const F3 g = pdot * (-2.f * W); gT[0] = g.x; gT[1] = g.y; gT[2] = g.z; }
  if (gO) {
    const F3 g = qrot(qconj(q), pdot - cross(w, d) + sg * d) * (2.f * W * s);
    gO[0] = g.x; gO[1] = g.y; gO[2] = g.z;
  }
}

// <dR(q)/dq_k, X> for k = x, y, z, w (qmat's quadratic form, X column-major m[3*col + row])
MB2_HD void qmatDerivativeDot(Q4 q, const float* X, float* out) {
  const float x01 = X[3] + X[1], x02 = X[6] + X[2], x12 = X[7] + X[5];
  const float a01 = X[1] - X[3], a02 = X[6] - X[2], a21 = X[5] - X[7]; // X10 - X01, X02 - X20, X21 - X12
  out[0] = 2.f * (q.y * x01 + q.z * x02 + q.w * a21) - 4.f * q.x * (X[4] + X[8]);
  out[1] = 2.f * (q.x * x01 + q.w * a02 + q.z * x12) - 4.f * q.y * (X[0] + X[8]);
  out[2] = 2.f * (q.w * a01 + q.x * x02 + q.y * x12) - 4.f * q.z * (X[0] + X[4]);
  out[3] = 2.f * (q.z * a01 + q.y * a02 + q.x * a21);
}

// Orientation constraint (matrix difference, L2), R_c = R_j R(q_o), F = R_c - R(q_t), dR_c = [w_j]x R_c, g = 2 W <F, [w_j]x R_c>:
//   dg/dw_c = 2 e.weight / c^2 <F, [w_j]x R_c>,   dg/dq_t,k = -2 W <dR/dq_k(q_t), [w_j]x R_c>,
//   dg/dq_o,k = 2 W <R_j dR/dq_k(q_o), [w_j]x R(q_t)>   (R_c - F = R(q_t))
// at the normalised quaternions the record holds (target xyzw, then the offset for an instanced block).
MB2_HD void orientationInputGradient(const UnitDesc& u, const EfDesc& e, const float* js, const float* tan, const float* tg, float cw, float* gW,
                                     float* gO, float* gT) {
  const Q4 q = ld4(js + u.joint * kJointStateStride + 3);
  const F3 w = ld3(tan + u.joint * kTangentStride);
  const Q4 qo = u.pad[2] != 0 ? ld4(tg + 4) : q4(u.f[0], u.f[1], u.f[2], u.f[3]);
  const Q4 qt = ld4(tg);
  float ro[9], rt[9], xt[9], xo[9];
  qmat(qo, ro);
  qmat(qt, rt);
  float fx = 0.f;
  for (int k = 0; k < 3; ++k) {
    const F3 rc = qrot(q, f3(ro[3 * k], ro[3 * k + 1], ro[3 * k + 2])); // column k of R_c, as evalUnit forms it
    const F3 rtk = f3(rt[3 * k], rt[3 * k + 1], rt[3 * k + 2]);
    const F3 a = cross(w, rc), b = qrot(qconj(q), cross(w, rtk)); // [w]x R_c and R_j^T [w]x R_t, column k
    fx += dot(rc - rtk, a);
    xt[3 * k] = a.x; xt[3 * k + 1] = a.y; xt[3 * k + 2] = a.z;
    xo[3 * k] = b.x; xo[3 * k + 1] = b.y; xo[3 * k + 2] = b.z;
  }
  const float ew = e.weight * e.invC2, W = ew * cw;
  if (gW) gW[0] = 2.f * ew * fx;
  float d[4];
  if (gT) { qmatDerivativeDot(qt, xt, d); for (int k = 0; k < 4; ++k) gT[k] = -2.f * W * d[k]; }
  if (gO) { qmatDerivativeDot(qo, xo, d); for (int k = 0; k < 4; ++k) gO[k] = 2.f * W * d[k]; }
}

// ---- quaternion log map (math/utility.cpp:72-180) ----
MB2_HD F3 quaternionLogMap(Q4 q) {
  const Q4 qn = qnormalized(q);
  const F3 vec = f3(qn.x, qn.y, qn.z);
  const float vn = sqrtf(dot(vec, vec));
  if (vn < 3.5e-4f) {
    if (qn.w > 0.f) return vec * (2.f * (1.f + dot(vec, vec) / 6.f));
    return f3(kPi, 0.f, 0.f);
  }
  const float theta = 2.f * atan2f(vn, qn.w);
  return vec * (theta / vn);
}
MB2_HD void quaternionLogMapDerivative(Q4 q, float* jac /* [row*4 + col], cols x,y,z,w */) {
  const Q4 qn = qnormalized(q);
  const float v[3] = {qn.x, qn.y, qn.z};
  const float w = qn.w;
  const float vn2 = v[0] * v[0] + v[1] * v[1] + v[2] * v[2];
  const float vn = sqrtf(vn2);
  if (vn < 3.5e-4f) {
    const float scale = 2.f * (1.f + vn2 / 6.f);
    for (int i = 0; i < 3; ++i) {
      for (int j = 0; j < 3; ++j) jac[4 * i + j] = (i == j ? scale : 0.f) + 2.f * v[i] * v[j] / 3.f;
      jac[4 * i + 3] = 0.f;
    }
    return;
  }
  const float theta = 2.f * atan2f(vn, w);
  const float scale = theta / vn;
  const float denom = w * w + vn * vn;
  const float dthetaDw = -2.f * vn / denom;
  for (int j = 0; j < 3; ++j) {
    const float dthetaDvj = 2.f * w * v[j] / (vn * denom);
    const float dScale = dthetaDvj / vn - theta * v[j] / (vn * vn * vn);
    for (int i = 0; i < 3; ++i) jac[4 * i + j] = dScale * v[i] + (i == j ? scale : 0.f);
  }
  for (int i = 0; i < 3; ++i) jac[4 * i + 3] = dthetaDw / vn * v[i];
}
// state_error_function.cpp:33-66
MB2_HD F3 logMapRelativeDerivativeQ1(Q4 q1, Q4 q2, F3 dir, const float* dLogDq) {
  const F3 vHalf = dir * 0.5f;
  const F3 q1v = f3(q1.x, q1.y, q1.z);
  const float dq1w = -dot(vHalf, q1v);
  const F3 dq1v = vHalf * q1.w + cross(vHalf, q1v);
  const F3 mq2v = f3(-q2.x, -q2.y, -q2.z);
  const float dqRelW = q2.w * dq1w - dot(mq2v, dq1v);
  const F3 dqRelV = q2.w * dq1v + dq1w * mq2v + cross(mq2v, dq1v);
  return f3(dLogDq[0] * dqRelV.x + dLogDq[1] * dqRelV.y + dLogDq[2] * dqRelV.z + dLogDq[3] * dqRelW,
            dLogDq[4] * dqRelV.x + dLogDq[5] * dqRelV.y + dLogDq[6] * dqRelV.z + dLogDq[7] * dqRelW,
            dLogDq[8] * dqRelV.x + dLogDq[9] * dqRelV.y + dLogDq[10] * dqRelV.z + dLogDq[11] * dqRelW);
}

MB2_HD bool limitInRange(float rangeMin, float rangeMax, float v) { // parameter_limits.cpp:105-123
  if (rangeMin == 0.f && rangeMax == 0.f) return true;
  return v >= rangeMin && v < rangeMax;
}

// Ellipsoid limit geometry (limit_error_function.cpp:713-722) from the parent's state ps, the ellipsoid parent's state es and the limit's
// 27 floats d (ellipsoid 3x4, ellipsoidInv 3x4, offset): the constrained point, its difference to its projection onto the ellipsoid, and
// what the backward reuses (the normalised ellipsoid-space point, 1 / its norm before, the projection relative to the ellipsoid parent)
struct EllipsoidPoint {
  F3 position, diff, ep, projected;
  float inv;
};
MB2_HD void ellipsoidGeometry(const float* ps, const float* es, const float* d, EllipsoidPoint& e) {
  F3& position = e.position;
  position = ld3(ps) + qrot(ld4(ps + 3), ps[7] * f3(d[24], d[25], d[26]));
  const F3 et = ld3(es);
  const Q4 eq = ld4(es + 3);
  const float esc = es[7];
  // TransformT::inverse (math/transform.cpp:93-101), Eigen quaternion inverse = conj / squaredNorm
  const float n2 = eq.x * eq.x + eq.y * eq.y + eq.z * eq.z + eq.w * eq.w;
  const Q4 iq = q4(-eq.x / n2, -eq.y / n2, -eq.z / n2, eq.w / n2);
  const float is = 1.f / esc;
  const F3 it = (qrot(iq, et) * is) * -1.f;
  const F3 local = it + qrot(iq, is * position);
  F3 ep = f3(d[12] * local.x + d[13] * local.y + d[14] * local.z + d[15], d[16] * local.x + d[17] * local.y + d[18] * local.z + d[19],
             d[20] * local.x + d[21] * local.y + d[22] * local.z + d[23]);
  const float inv = 1.f / sqrtf(dot(ep, ep));
  ep = ep * inv;
  const F3 proj = f3(d[0] * ep.x + d[1] * ep.y + d[2] * ep.z + d[3], d[4] * ep.x + d[5] * ep.y + d[6] * ep.z + d[7],
                     d[8] * ep.x + d[9] * ep.y + d[10] * ep.z + d[11]);
  e.projected = qrot(eq, esc * proj);
  e.diff = position - (et + e.projected);
  e.ep = ep;
  e.inv = inv;
}
// the solver's unit: returns position, diff
MB2_HD void evalEllipsoid(const FunctionTables& T, const UnitDesc& u, const float* js, F3& position, F3& diff) {
  EllipsoidPoint e;
  ellipsoidGeometry(js + u.joint * kJointStateStride, js + u.i[0] * kJointStateStride, T.limitData + u.extra, e); // parent, ellipsoidParent
  position = e.position;
  diff = e.diff;
}

constexpr float kLimitWeight = 10.f;        // limit_error_function.h:91
constexpr float kLimitPositionWeight = 1e-4f; // limit_error_function.cpp:21
constexpr float kStatePositionWeight = 1e-3f; // state_error_function.h:115
constexpr float kStateOrientationWeight = 1.f; // state_error_function.h:116

// ---- Parameter limits as a character operation (parameter_limits_residual): the rows of evalUnit's limit cases at weight 1, L2 loss --
// The residual of a joint-space or parameter-space limit before its row scale, in evalUnit's operation order; `active` false: a zero row.
// th: theta [n], jp: P theta + o [7 J].
MB2_HD float limitResidual(const LimitDesc& D, const float* th, const float* jp, bool& active) {
  active = true;
  switch (D.type) {
    case kLimitMinMax:
    case kLimitMinMaxJoint: {
      const float p = D.type == kLimitMinMax ? th[D.i0] : jp[D.i0];
      if (p < D.f[0]) return p - D.f[0];
      if (p > D.f[1]) return p - D.f[1];
      break;
    }
    case kLimitLinear:
    case kLimitLinearJoint: {
      const float* x = D.type == kLimitLinear ? th : jp;
      if (limitInRange(D.f[2], D.f[3], x[D.i1])) return x[D.i1] * D.f[0] - D.f[1] - x[D.i0];
      break;
    }
    case kLimitHalfPlane: {
      const float res = th[D.i0] * D.f[0] + th[D.i1] * D.f[1] - D.f[2];
      if (res < 0.f) return res;
      break;
    }
    default: break;
  }
  active = false;
  return 0.f;
}

// limit l's rows in out [R] (js: the world states, read by an Ellipsoid only)
template <bool kEllipsoid>
MB2_HD void limitRows(const LimitTables& L, int l, const float* th, const float* jp, const float* js, float* out) {
  const LimitDesc& D = L.limits[l];
  if (kEllipsoid && D.type == kLimitEllipsoid) {
    EllipsoidPoint e;
    ellipsoidGeometry(js + D.i1 * kJointStateStride, js + D.i0 * kJointStateStride, L.ellipsoidData + D.data, e);
    out[D.row] = e.diff.x * D.w; out[D.row + 1] = e.diff.y * D.w; out[D.row + 2] = e.diff.z * D.w;
    return;
  }
  bool active;
  const float res = limitResidual(D, th, jp, active);
  out[D.row] = active ? res * D.w : 0.f;
}

// The backward of an Ellipsoid's rows w diff from their upstream gradient g (gd = w g), the exact derivative of ellipsoidGeometry,
// projection included, as rigid-motion seeds in skelGradSeed's layout (S_g, R, D; S_c = S_s = 0). With y = t_e + s_e R_e proj the
// projected point and h = (1 / s_e) R_e A_inv^T (I - ep ep^T) A^T (-s_e R_e^T gd) / |u| the gradient reaching the point through its
// ellipsoid-space coordinates, the loss gd . diff moves
//   role 0, the parent joint, with the point x = t_p + d:   S_g = gx, R = d x gx, D = d . gx,   gx = gd + h
//   role 1, the ellipsoid parent (x held):                  S_g = -gx, R = -(y - t_e) x gd - (x - t_e) x h, D likewise with dots
// (unit quaternions assumed, R_e^T = rot(conj q_e)). Added to sg, r, dd.
MB2_HD void ellipsoidSeed(const float* ps, const float* es, const float* d, F3 gd, int role, F3& sg, F3& r, float& dd) {
  EllipsoidPoint e;
  ellipsoidGeometry(ps, es, d, e);
  const Q4 eq = ld4(es + 3);
  const float esc = es[7];
  const F3 gp = esc * qrot(qconj(eq), gd * -1.f); // dLoss / d proj
  const F3 gep = f3(d[0] * gp.x + d[4] * gp.y + d[8] * gp.z, d[1] * gp.x + d[5] * gp.y + d[9] * gp.z, d[2] * gp.x + d[6] * gp.y + d[10] * gp.z);
  const F3 gu = (gep - e.ep * dot(e.ep, gep)) * e.inv;
  const F3 gl = f3(d[12] * gu.x + d[16] * gu.y + d[20] * gu.z, d[13] * gu.x + d[17] * gu.y + d[21] * gu.z, d[14] * gu.x + d[18] * gu.y + d[22] * gu.z);
  const F3 h = qrot(eq, gl) * (1.f / esc);
  const F3 gx = gd + h;
  if (role == 0) {
    const F3 dp = pointRelative(ps, f3(d[24], d[25], d[26]));
    sg = sg + gx;
    r = r + cross(dp, gx);
    dd = dd + dot(dp, gx);
  } else {
    const F3 rx = e.position - ld3(es);
    sg = sg - gx;
    r = r - (cross(e.projected, gd) + cross(rx, h));
    dd = dd - (dot(e.projected, gd) + dot(rx, h));
  }
}
// joint j's seed from the Ellipsoids that name it, in the order of L.jointEntry; g: the instance's upstream gradient [R]
MB2_HD void limitJointSeed(const LimitTables& L, const float* js, int j, const float* g, float* acc) {
  F3 sg = f3(0.f, 0.f, 0.f), r = sg;
  float d = 0.f;
#pragma unroll 1
  for (int k = L.jointStart[j]; k < L.jointStart[j + 1]; ++k) {
    const int e = L.jointEntry[k];
    const LimitDesc& D = L.limits[e >> 1];
    const F3 gd = f3(g[D.row], g[D.row + 1], g[D.row + 2]) * D.w;
    ellipsoidSeed(js + D.i1 * kJointStateStride, js + D.i0 * kJointStateStride, L.ellipsoidData + D.data, gd, e & 1, sg, r, d);
  }
  float* A = acc + j * kSkelAccStride;
  A[0] = sg.x; A[1] = sg.y; A[2] = sg.z;
  A[3] = r.x; A[4] = r.y; A[5] = r.z; A[6] = d;
  A[7] = 0.f; A[8] = 0.f; A[9] = 0.f; A[10] = 0.f;
}
// the sum over one group of a CSR (start, limit, coef) of coef g[row] for each active limit, in entry order
MB2_HD float limitTermSum(const LimitTables& L, const int32_t* start, const int32_t* limit, const float* coef, int k, const float* th, const float* jp,
                          const float* g) {
  float s = 0.f;
#pragma unroll 1
  for (int e = start[k]; e < start[k + 1]; ++e) {
    const LimitDesc& D = L.limits[limit[e]];
    bool active;
    limitResidual(D, th, jp, active);
    if (active) s += coef[e] * g[D.row];
  }
  return s;
}

// jp [7 J] = P theta + o of the staged theta th, lanes = rows, then (kFk) the FK passes from jp: kAxes ends without a barrier, else
// with one
template <bool kFk, bool kAxes, class Lanes>
MB2_HD void limitStatePasses(const Lanes& g, const CharacterTables& C, const float* th, float* jp, float* js) {
  for (int r = g.lane; r < C.numJoints * kParametersPerJoint; r += g.size) jp[r] = jointParameterRow(C, r, th);
  g.sync();
  if constexpr (kFk) fkPasses<kAxes, true>(g, C, jp, js);
}

// The residual rows out [R] of one instance, lanes = limits (kEllipsoid: the character has an Ellipsoid, so the FK runs). Ends without a
// barrier.
template <bool kEllipsoid, class Lanes>
MB2_HD void limitPasses(const Lanes& g, const CharacterTables& C, const LimitTables& L, const float* th, float* jp, float* js, float* out) {
  limitStatePasses<kEllipsoid, false>(g, C, th, jp, js);
  for (int l = g.lane; l < L.numLimits; l += g.size) limitRows<kEllipsoid>(L, l, th, jp, js, out);
}

// Its backward from grad [R] into out [n]: (kEllipsoid) lanes = joints seed their subtree sums from the Ellipsoids, sharing the axes'
// barrier, and skelGradTail gives the joint-parameter gradient gjp [7 J]; lanes = rows add the joint-space terms to gjp (the lanes that
// wrote those rows in skelGradTail, so no barrier); lanes = model parameters: P^T gjp plus the parameter-space terms. Ends without a
// barrier.
template <bool kEllipsoid, class Lanes>
MB2_HD void limitGradPasses(const Lanes& g, const CharacterTables& C, const SkeletonTables& S, const LimitTables& L, const float* th, float* jp,
                            float* js, float* acc, float* gjp, const float* grad, float* out) {
  limitStatePasses<kEllipsoid, true>(g, C, th, jp, js);
  const int rows = C.numJoints * kParametersPerJoint;
  if constexpr (kEllipsoid) {
    for (int j = g.lane; j < C.numJoints; j += g.size) limitJointSeed(L, js, j, grad, acc);
    g.sync();
    skelGradTail(g, C, S, js, acc, gjp, nullptr);
    for (int r = g.lane; r < rows; r += g.size) gjp[r] = gjp[r] + limitTermSum(L, L.rowStart, L.rowLimit, L.rowCoef, r, th, jp, grad);
  } else {
    for (int r = g.lane; r < rows; r += g.size) gjp[r] = limitTermSum(L, L.rowStart, L.rowLimit, L.rowCoef, r, th, jp, grad);
  }
  g.sync();
  for (int p = g.lane; p < C.numParams; p += g.size)
    out[p] = skelGradModelParameter(S, gjp, p) + limitTermSum(L, L.paramStart, L.paramLimit, L.paramCoef, p, th, jp, grad);
}

// ---- Self-collision of tapered capsules as a character operation (collision_residual) ---------------------------------------------
// The world capsule (CollisionGeometryStateT::updatePrimitive, collision_geometry_state.cpp:28-48), the narrow phase of overlaps
// (collision_geometry_state.h:120-157) over closestPointsOnSegments (math/utility.cpp:443-552), branch for branch in the reference's
// operation order, and the exact derivative of the overlap. A capsule's world geometry is 8 values: origin, direction (its length is the
// segment's), r0, r1; delta = r1 - r0 (kCapsuleFloats, ik_types.h).
MB2_HD void skinStateGradient(const float* acc, const float* state, float* out); // below, with the skinning
// sqrt(kCollisionWeight) at weight 1 (collision_error_function.h:139, collision_error_function.cpp getJacobian's wgt), in float
MB2_HD float collisionRowWeight() { return sqrtf(5e-3f); }

// capsule c's world geometry out [8] from its parent's skeleton state ps [8] (t, q, s; q normalised), nullptr for a world-fixed capsule:
// origin t + rot(q^, s o), direction rot(q^, s d), radii s r
MB2_HD void capsuleWorld(const CapsuleDesc& c, const float* ps, float* out) {
  F3 o = ld3(c.origin), d = ld3(c.dir);
  float r0 = c.r0, r1 = c.r1;
  if (ps != nullptr) {
    const Q4 u = qnormalized(ld4(ps + 3));
    const float s = ps[7];
    o = ld3(ps) + qrot(u, s * o);
    d = qrot(u, s * d);
    r0 = r0 * s;
    r1 = r1 * s;
  }
  out[0] = o.x; out[1] = o.y; out[2] = o.z;
  out[3] = d.x; out[4] = d.y; out[5] = d.z;
  out[6] = r0; out[7] = r1;
}

// Which closed form a segment parameter of a contact came from: a constant (a clamp, or the 1e-7 snap), the interior solution
// s = (b e - c d) / D, t = (a e - b d) / D, or the projection onto an edge of the other segment.
enum SegmentForm : int {
  kSegConst = 0,
  kSegInterior = 1,
  kSegEdge0 = 2, // s on the t = 0 edge: -d / a;        t on the s = 0 edge (and the parallel branch): e / c
  kSegEdge1 = 3, // s on the t = 1 edge: (b - d) / a;   t on the s = 1 edge: (e + b) / c
};
template <class T>
struct CapsuleContact {
  bool hit;     // overlaps(): overlap > 0 and dist >= Eps
  T s, t;       // the closest-point parameters
  T dist, overlap;
  int sForm, tForm;
};
template <class T>
MB2_HD T segDot(const T* a, const T* b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }

// overlaps(A, B) of two world capsules A, B [8] (T = float: the reference's float build; the planner's rest pose runs it in double, with
// double's Eps as the reference's double build has it). A non-finite input fails every comparison that would report a contact.
template <class T>
MB2_HD CapsuleContact<T> capsuleContact(const T* A, const T* B) {
  CapsuleContact<T> r;
  r.hit = false;
  r.s = r.t = r.dist = r.overlap = T(0);
  r.sForm = r.tForm = kSegConst;
  const T maxA = A[6] < A[7] ? A[7] : A[6], maxB = B[6] < B[7] ? B[7] : B[6]; // Vector2::maxCoeff
  const T maxDist = maxA + maxB;
  const T maxSq = maxDist * maxDist;
  const T* d1 = A + 3;
  const T* d2 = B + 3;
  const T w[3] = {A[0] - B[0], A[1] - B[1], A[2] - B[2]};
  const T a = segDot(d1, d1), b = segDot(d1, d2), c = segDot(d2, d2), d = segDot(d1, w), e = segDot(d2, w);
  const T D = a * c - b * b;
  T sN, sD = D, tN, tD = D;
  int sF, tF;
  if (D < T(1e-7)) { // parallel: s = 0, t along d2; too far when the origins are (the reference's early-out)
    sN = T(0); sD = T(1); tN = e; tD = c;
    sF = kSegConst; tF = kSegEdge0;
    if (segDot(w, w) > maxSq) return r;
  } else {
    sN = b * e - c * d;
    tN = a * e - b * d;
    sF = tF = kSegInterior;
    const T q[3] = {w[0] + d1[0] * sN / D - d2[0] * tN / D, w[1] + d1[1] * sN / D - d2[1] * tN / D, w[2] + d1[2] * sN / D - d2[2] * tN / D};
    if (segDot(q, q) > maxSq) return r; // the infinite lines are too far
    if (sN < T(0)) { sN = T(0); tN = e; tD = c; sF = kSegConst; tF = kSegEdge0; }
    else if (sN > sD) { sN = sD; tN = e + b; tD = c; sF = kSegConst; tF = kSegEdge1; }
  }
  if (tN < T(0)) {
    tN = T(0); tF = kSegConst;
    if (-d < T(0)) { sN = T(0); sF = kSegConst; }
    else if (-d > a) { sN = sD; sF = kSegConst; }
    else { sN = -d; sD = a; sF = kSegEdge0; }
  } else if (tN > tD) {
    tN = tD; tF = kSegConst;
    if ((-d + b) < T(0)) { sN = T(0); sF = kSegConst; }
    else if ((-d + b) > a) { sN = sD; sF = kSegConst; }
    else { sN = (-d + b); sD = a; sF = kSegEdge1; }
  }
  using std::fabs;
  using std::sqrt;
  const bool sSnap = fabs(sN) < T(1e-7) || fabs(sD) < T(1e-7), tSnap = fabs(tN) < T(1e-7) || fabs(tD) < T(1e-7);
  const T s = sSnap ? T(0) : sN / sD, t = tSnap ? T(0) : tN / tD;
  const T dP[3] = {w[0] + d1[0] * s - d2[0] * t, w[1] + d1[1] * s - d2[1] * t, w[2] + d1[2] * s - d2[2] * t};
  const T distSq = segDot(dP, dP);
  if (distSq > maxSq) return r;
  const T dist = sqrt(distSq);
  const T overlap = A[6] + s * (A[7] - A[6]) + B[6] + t * (B[7] - B[6]) - dist;
  r.s = s; r.t = t; r.dist = dist; r.overlap = overlap;
  r.sForm = sSnap ? int(kSegConst) : sF;
  r.tForm = tSnap ? int(kSegConst) : tF;
  r.hit = overlap > T(0) && dist >= (sizeof(T) == 4 ? T(1e-8) : T(1e-17));
  return r;
}

// The exact derivative of a contact's overlap with respect to A [8] and B [8], times gw, added to gA and gB (either may be nullptr):
// at fixed (s, t), d overlap = -n . d(dP) + ds (r1 - r0)_A ... with n = dP / dist; s and t move through the closed form of their branch
// (sForm, tForm) with g_s = delta_A - n . dA, g_t = delta_B + n . dB, by way of a = dA.dA, b = dA.dB, c = dB.dB, d = dA.w, e = dB.w.
// Constants (clamps, snaps) do not move. Unlike CollisionErrorFunction::getJacobian, which holds (s, t) fixed, this keeps delta ds.
template <class T>
MB2_HD void capsuleContactGrad(const T* A, const T* B, const CapsuleContact<T>& k, T gw, T* gA, T* gB) {
  const T* d1 = A + 3;
  const T* d2 = B + 3;
  const T w[3] = {A[0] - B[0], A[1] - B[1], A[2] - B[2]};
  const T a = segDot(d1, d1), b = segDot(d1, d2), c = segDot(d2, d2), d = segDot(d1, w), e = segDot(d2, w);
  const T D = a * c - b * b;
  const T s = k.s, t = k.t;
  const T n[3] = {(w[0] + d1[0] * s - d2[0] * t) / k.dist, (w[1] + d1[1] * s - d2[1] * t) / k.dist, (w[2] + d1[2] * s - d2[2] * t) / k.dist};
  const T gs = (A[7] - A[6]) - segDot(n, d1), gt = (B[7] - B[6]) + segDot(n, d2);
  T ga = T(0), gb = T(0), gc = T(0), gd = T(0), ge = T(0);
  if (k.sForm == kSegInterior) {
    ga += gs * (-s * c) / D; gb += gs * (e + T(2) * b * s) / D; gc += gs * (-d - s * a) / D; gd += gs * (-c) / D; ge += gs * b / D;
  } else if (k.sForm == kSegEdge0) {
    gd += -gs / a; ga += -gs * s / a;
  } else if (k.sForm == kSegEdge1) {
    gb += gs / a; gd += -gs / a; ga += -gs * s / a;
  }
  if (k.tForm == kSegInterior) {
    ga += gt * (e - t * c) / D; gb += gt * (-d + T(2) * b * t) / D; gc += gt * (-t * a) / D; gd += gt * (-b) / D; ge += gt * a / D;
  } else if (k.tForm == kSegEdge0) {
    ge += gt / c; gc += -gt * t / c;
  } else if (k.tForm == kSegEdge1) {
    ge += gt / c; gb += gt / c; gc += -gt * t / c;
  }
  for (int i = 0; i < 3; ++i) {
    const T gW = -n[i] + gd * d1[i] + ge * d2[i];
    if (gA != nullptr) {
      gA[i] += gw * gW;
      gA[3 + i] += gw * (-s * n[i] + T(2) * ga * d1[i] + gb * d2[i] + gd * w[i]);
    }
    if (gB != nullptr) {
      gB[i] += gw * -gW;
      gB[3 + i] += gw * (t * n[i] + gb * d1[i] + T(2) * gc * d2[i] + ge * w[i]);
    }
  }
  if (gA != nullptr) { gA[6] += gw * (T(1) - s); gA[7] += gw * s; }
  if (gB != nullptr) { gB[6] += gw * (T(1) - t); gB[7] += gw * t; }
}

// lanes = capsules: the world geometry geo [C][8] of one instance's states st [J][8]. Ends with a barrier.
template <class Lanes>
MB2_HD void collisionGeometryPasses(const Lanes& g, const CollisionTables& L, const float* st, float* geo) {
  for (int k = g.lane; k < L.numCapsules; k += g.size) {
    const CapsuleDesc& c = L.capsules[k];
    capsuleWorld(c, c.parent >= 0 ? st + size_t(c.parent) * 8 : nullptr, geo + size_t(k) * kCapsuleFloats);
  }
  g.sync();
}

// The rows out [P] of one instance, lanes = pairs: sqrt(kCollisionWeight) overlap at a contact, else 0. Ends without a barrier.
template <class Lanes>
MB2_HD void collisionPasses(const Lanes& g, const CollisionTables& L, const float* st, float* geo, float* out) {
  collisionGeometryPasses(g, L, st, geo);
  const float wgt = collisionRowWeight();
  for (int k = g.lane; k < L.numPairs; k += g.size) {
    const CapsuleContact<float> c = capsuleContact(geo + size_t(L.pairs[2 * k]) * kCapsuleFloats, geo + size_t(L.pairs[2 * k + 1]) * kCapsuleFloats);
    out[k] = c.hit ? wgt * c.overlap : 0.f;
  }
}

// Its backward from grad [P] into out [J][8]: lanes = capsules walk their own pairs in ascending order, recompute each contact and sum
// their own side's gradient into cg [C][8]; lanes = joints then take their capsules in order: the origin and the end point are fixed in the
// parent's frame (a = sum g_o, E = sum g_o o^T + g_d d^T, skinStateGradient's (a, E) with q normalised) and the radii scale with s, so
// ds gains sum (r0 g_r0 + r1 g_r1). Joints without a capsule get 0. Ends without a barrier.
template <class Lanes>
MB2_HD void collisionGradPasses(const Lanes& g, const CollisionTables& L, int numJoints, const float* st, float* geo, float* cg, const float* grad,
                                float* out) {
  collisionGeometryPasses(g, L, st, geo);
  const float wgt = collisionRowWeight();
  for (int k = g.lane; k < L.numCapsules; k += g.size) {
    float acc[kCapsuleFloats] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (int e = L.capsuleStart[k]; e < L.capsuleStart[k + 1]; ++e) {
      const int p = L.capsulePair[e], i = L.pairs[2 * p], j = L.pairs[2 * p + 1];
      const float* A = geo + size_t(i) * kCapsuleFloats;
      const float* B = geo + size_t(j) * kCapsuleFloats;
      const CapsuleContact<float> c = capsuleContact(A, B);
      if (c.hit) capsuleContactGrad(A, B, c, wgt * grad[p], i == k ? acc : nullptr, i == k ? nullptr : acc);
    }
    for (int i = 0; i < kCapsuleFloats; ++i) cg[size_t(k) * kCapsuleFloats + i] = acc[i];
  }
  g.sync();
  for (int j = g.lane; j < numJoints; j += g.size) {
    float* o = out + size_t(j) * 8;
    if (L.jointStart[j] == L.jointStart[j + 1]) {
      for (int i = 0; i < 8; ++i) o[i] = 0.f;
      continue;
    }
    float acc[12] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f}; // skinAccumulate's (a, E)
    float dsr = 0.f;
    for (int e = L.jointStart[j]; e < L.jointStart[j + 1]; ++e) {
      const int k = L.jointCapsule[e];
      const CapsuleDesc& c = L.capsules[k];
      const float* gk = cg + size_t(k) * kCapsuleFloats;
      for (int r = 0; r < 3; ++r) {
        acc[r] += gk[r];
        for (int col = 0; col < 3; ++col) acc[3 + 3 * r + col] += gk[r] * c.origin[col] + gk[3 + r] * c.dir[col];
      }
      dsr += c.r0 * gk[6] + c.r1 * gk[7];
    }
    skinStateGradient(acc, st + size_t(j) * 8, o);
    o[7] += dsr;
  }
}

// ------------------------------------------------------------------------------------------------
// Evaluate one unit: residual rows, error contribution, and the evaluation record consumed by its
// Jacobian cells. kJacobian=false is the getError() path (joint_error_function-inl.h:35-54 etc.):
// same value, no residual/record stores.
// Returns the unit's error contribution (float, summed in double by the caller like the reference).
// ------------------------------------------------------------------------------------------------
template <bool kJacobian>
MB2_HD float evalUnit(const FunctionTables& T, int ui, const float* theta, const float* jp, const float* js, const float* targets,
                      const float* cweights, float* rec, float* residual) {
  const UnitDesc& u = T.units[ui];
  const EfDesc& e = T.efs[u.ef];
  float* r = kJacobian ? residual + u.row0 : nullptr;
  float* rc = kJacobian ? rec + u.recOff : nullptr;
  if (u.pad[0] != 0) { // limit gated off by enabledParameters_/activeJointParams_: zero row(s), no error
    if (kJacobian) { for (int k = 0; k < u.numRows; ++k) r[k] = 0.f; rc[0] = 0.f; }
    return 0.f;
  }
  switch (u.kind) {
    case kUnitPosition: {
      const float cw = cweights[u.weightIdx];
      if (cw == 0.f) { // joint_error_function-inl.h:197-199
        if (kJacobian) { r[0] = r[1] = r[2] = 0.f; rc[0] = rc[1] = rc[2] = rc[3] = 0.f; }
        return 0.f;
      }
      const float* ps = js + u.joint * kJointStateStride;
      const float* tg = targets + u.targetOff;
      // the constraint offset is shared by the batch (u.f) or, for an "instanced" block, follows the target in the instance's record
      const F3 off = u.pad[2] != 0 ? f3(tg[3], tg[4], tg[5]) : f3(u.f[0], u.f[1], u.f[2]);
      const F3 v = ld3(ps) + qrot(ld4(ps + 3), ps[7] * off); // transform.h:193-195
      const F3 f = f3(v.x - tg[0], v.y - tg[1], v.z - tg[2]);
      const float sq = dot(f, f);
      if (!kJacobian) return cw * lossValue(e, sq) * e.weight;
      const float w = cw * e.weight;
      float ds = sqrtf(w * lossDeriv(e, sq));
      r[0] = ds * f.x; r[1] = ds * f.y; r[2] = ds * f.z;
      if (fabsf(ds) < 1e-9f) ds = 0.f; // :216-218 rows stay zero
      rc[0] = v.x; rc[1] = v.y; rc[2] = v.z; rc[3] = ds;
      return w * lossValue(e, sq);
    }
    case kUnitOrientation:
    case kUnitOrientationRotDiff: {
      const float cw = cweights[u.weightIdx];
      if (cw == 0.f) {
        if (kJacobian) { for (int k = 0; k < 9; ++k) r[k] = 0.f; for (int k = 0; k < 10; ++k) rc[k] = 0.f; }
        return 0.f;
      }
      const Q4 q = ld4(js + u.joint * kJointStateStride + 3);
      float ro[9], rt[9], f[9], v[9];
      // the offset is shared by the batch (u.f) or, for an instanced block, follows the target quaternion in the instance's record
      Q4 qo = q4(u.f[0], u.f[1], u.f[2], u.f[3]);
      if (u.pad[2] != 0) qo = ld4(targets + u.targetOff + 4);
      qmat(qo, ro);
      qmat(ld4(targets + u.targetOff), rt);
      for (int k = 0; k < 3; ++k) {
        const F3 vk = qrot(q, f3(ro[3 * k], ro[3 * k + 1], ro[3 * k + 2]));
        v[3 * k] = vk.x; v[3 * k + 1] = vk.y; v[3 * k + 2] = vk.z;
      }
      if (u.kind == kUnitOrientation) {
        for (int k = 0; k < 9; ++k) f[k] = v[k] - rt[k];
      } else {
        // NB: the reference forms vec = R(q) * R(offset) as a matrix product; v_k = vec.col(k) (orientation_error_function.cpp:52-60)
        float rq[9];
        qmat(q, rq);
        for (int k = 0; k < 3; ++k)
          for (int rr = 0; rr < 3; ++rr) v[3 * k + rr] = rq[rr] * ro[3 * k] + rq[3 + rr] * ro[3 * k + 1] + rq[6 + rr] * ro[3 * k + 2];
        for (int k = 0; k < 3; ++k)
          for (int rr = 0; rr < 3; ++rr) // (R_t^T vec)(rr,k) - I
            f[3 * k + rr] = rt[3 * rr] * v[3 * k] + rt[3 * rr + 1] * v[3 * k + 1] + rt[3 * rr + 2] * v[3 * k + 2] - (rr == k ? 1.f : 0.f);
      }
      float sq = 0.f;
      for (int k = 0; k < 9; ++k) sq += f[k] * f[k];
      if (!kJacobian) return cw * lossValue(e, sq) * e.weight;
      const float w = cw * e.weight;
      float ds = sqrtf(w * lossDeriv(e, sq));
      for (int k = 0; k < 9; ++k) r[k] = ds * f[k];
      if (fabsf(ds) < 1e-9f) ds = 0.f;
      for (int k = 0; k < 9; ++k) rc[k] = v[k];
      rc[9] = ds;
      return w * lossValue(e, sq);
    }
    case kUnitStateMatrix:
    case kUnitStateLogMap: {
      const float* ps = js + u.joint * kJointStateStride;
      const float* tg = targets + u.targetOff; // t(3) q(4) s
      const F3 td = f3(ps[0] - tg[0], ps[1] - tg[1], ps[2] - tg[2]);
      const Q4 target = qnormalized(ld4(tg + 3));
      const Q4 rot = ld4(ps + 3);
      const float posW = u.f[0], rotW = u.f[1];
      float rotationError = 0.f;
      F3 lv = f3(0, 0, 0);
      float rd[9];
      if (u.kind == kUnitStateLogMap) {
        lv = quaternionLogMap(qmul(qconj(target), rot));
        rotationError = dot(lv, lv);
      } else {
        float a[9], b[9];
        qmat(rot, a); qmat(target, b);
        for (int k = 0; k < 9; ++k) { rd[k] = a[k] - b[k]; rotationError += rd[k] * rd[k]; }
      }
      if (!kJacobian) { // state_error_function.cpp:251-255
        float err = rotationError * kStateOrientationWeight * e.rotWgt * rotW;
        err += dot(td, td) * kStatePositionWeight * e.posWgt * posW;
        return err * e.weight;
      }
      const float pwgt = kStatePositionWeight * e.posWgt * e.weight * posW; // :440-441
      const float rwgt = kStateOrientationWeight * e.rotWgt * e.weight * rotW;
      const float wgt = sqrtf(pwgt), awgt = sqrtf(rwgt);
      r[0] = td.x * wgt; r[1] = td.y * wgt; r[2] = td.z * wgt;
      rc[0] = wgt; rc[1] = awgt;
      if (u.kind == kUnitStateLogMap) {
        r[3] = lv.x * awgt; r[4] = lv.y * awgt; r[5] = lv.z * awgt;
        quaternionLogMapDerivative(qmul(qconj(target), rot), rc + 2);
      } else {
        for (int k = 0; k < 9; ++k) r[3 + k] = rd[k] * awgt;
      }
      return dot(td, td) * pwgt + rotationError * rwgt;
    }
    case kUnitPlane: { // plane_error_function.cpp:49-70 through joint_error_function-inl.h (FuncDim = 1)
      const float cw = cweights[u.weightIdx];
      if (cw == 0.f) {
        if (kJacobian) { r[0] = 0.f; for (int k = 0; k < 6; ++k) rc[k] = 0.f; }
        return 0.f;
      }
      const float* ps = js + u.joint * kJointStateStride;
      const F3 v = ld3(ps) + qrot(ld4(ps + 3), ps[7] * f3(u.f[0], u.f[1], u.f[2]));
      const float* tg = targets + u.targetOff; // normal (not necessarily unit: PlaneDataT's ctor normalises), d
      const float nlen = sqrtf(tg[0] * tg[0] + tg[1] * tg[1] + tg[2] * tg[2]);
      const F3 nrm = f3(tg[0] / nlen, tg[1] / nlen, tg[2] / nlen);
      float val = dot(v, nrm) - tg[3];
      if (e.halfPlane && val > 0.f) val = 0.f;
      const bool on = !e.halfPlane || val < 0.f;
      const float sq = val * val;
      if (!kJacobian) return cw * lossValue(e, sq) * e.weight;
      const float w = cw * e.weight;
      float ds = sqrtf(w * lossDeriv(e, sq));
      r[0] = ds * val;
      if (fabsf(ds) < 1e-9f || !on) ds = 0.f; // :216-223 tiny scale or all-zero dfdv: the row stays zero
      rc[0] = v.x; rc[1] = v.y; rc[2] = v.z;
      rc[3] = ds * nrm.x; rc[4] = ds * nrm.y; rc[5] = ds * nrm.z;
      return w * lossValue(e, sq);
    }
    case kUnitModelParameter: { // model_parameters_error_function.cpp:38-58, 90-133; kMotionWeight = 1e-1 (.h:61)
      const float pdiff = u.f[0] * (theta[u.i[0]] - targets[u.targetOff]);
      const float scale = e.weight * 1e-1f;
      if (u.pad[1] != 0) return kJacobian ? 0.f : pdiff * pdiff * scale; // negative target weight: counted by getError only (:56-59 vs :113)
      if (kJacobian) { const float sw = sqrtf(scale); r[0] = pdiff * sw; rc[0] = sw; }
      return pdiff * pdiff * scale;
    }
    default: break;
  }
  // ---- limits (limit_error_function.cpp) ----
  const bool L2 = e.lossType == kLossL2;
  const float lw = u.f[7]; // limit.weight
  if (!kJacobian) {
    // getErrorImpl (:818-867): per-limit term, then * kLimitWeight * weight (* invC2 for L2)
    const float post = kLimitWeight * e.weight * (L2 ? e.invC2 : 1.f);
    float sq = -1.f;
    float pre = lw;
    switch (u.kind) {
      case kUnitLimitMinMax: {
        const float p = theta[u.i[0]];
        if (p < u.f[0]) sq = (u.f[0] - p) * (u.f[0] - p);
        if (p > u.f[1]) sq = (u.f[1] - p) * (u.f[1] - p);
        break;
      }
      case kUnitLimitMinMaxJoint: {
        const float p = jointParameterAt(T, jp, theta, u.i[0]);
        if (p < u.f[0]) sq = (u.f[0] - p) * (u.f[0] - p);
        if (p > u.f[1]) sq = (u.f[1] - p) * (u.f[1] - p);
        break;
      }
      case kUnitLimitLinear: {
        if (limitInRange(u.f[2], u.f[3], theta[u.i[1]])) { const float res = theta[u.i[1]] * u.f[0] - u.f[1] - theta[u.i[0]]; sq = res * res; }
        break;
      }
      case kUnitLimitLinearJoint: {
        const float p1 = jointParameterAt(T, jp, theta, u.i[1]);
        if (limitInRange(u.f[2], u.f[3], p1)) { const float res = p1 * u.f[0] - u.f[1] - jointParameterAt(T, jp, theta, u.i[0]); sq = res * res; }
        break;
      }
      case kUnitLimitHalfPlane: {
        const float res = theta[u.i[0]] * u.f[0] + theta[u.i[1]] * u.f[1] - u.f[2];
        if (res < 0.f) sq = res * res;
        break;
      }
      case kUnitLimitEllipsoid: {
        F3 pos, diff;
        evalEllipsoid(T, u, js, pos, diff);
        sq = dot(diff, diff);
        pre = kLimitPositionWeight * lw;
        break;
      }
      default: break;
    }
    if (sq < 0.f) return 0.f;
    return pre * (L2 ? sq : lossValue(e, sq)) * post;
  }
  // Jacobian path (:992-1121): tWeight folds invC2 for L2
  const float tWeight = kLimitWeight * e.weight * (L2 ? e.invC2 : 1.f);
  float res = 0.f;
  bool active = false;
  switch (u.kind) {
    case kUnitLimitMinMax: {
      const float p = theta[u.i[0]];
      if (p < u.f[0]) { res = p - u.f[0]; active = true; }
      else if (p > u.f[1]) { res = p - u.f[1]; active = true; }
      break;
    }
    case kUnitLimitMinMaxJoint: {
      const float p = jointParameterAt(T, jp, theta, u.i[0]);
      if (p < u.f[0]) { res = p - u.f[0]; active = true; }
      else if (p > u.f[1]) { res = p - u.f[1]; active = true; }
      break;
    }
    case kUnitLimitLinear:
      if (limitInRange(u.f[2], u.f[3], theta[u.i[1]])) { res = theta[u.i[1]] * u.f[0] - u.f[1] - theta[u.i[0]]; active = true; }
      break;
    case kUnitLimitLinearJoint:
      { const float p1 = jointParameterAt(T, jp, theta, u.i[1]);
        if (limitInRange(u.f[2], u.f[3], p1)) { res = p1 * u.f[0] - u.f[1] - jointParameterAt(T, jp, theta, u.i[0]); active = true; } }
      break;
    case kUnitLimitHalfPlane:
      res = theta[u.i[0]] * u.f[0] + theta[u.i[1]] * u.f[1] - u.f[2];
      active = res < 0.f;
      break;
    case kUnitLimitEllipsoid: {
      F3 pos, diff;
      evalEllipsoid(T, u, js, pos, diff);
      const float sq = dot(diff, diff);
      const float jwgt = L2 ? sqrtf(tWeight * kLimitPositionWeight * lw) : sqrtf(tWeight * kLimitPositionWeight * lw * lossDeriv(e, sq));
      r[0] = diff.x * jwgt; r[1] = diff.y * jwgt; r[2] = diff.z * jwgt;
      rc[0] = pos.x; rc[1] = pos.y; rc[2] = pos.z; rc[3] = jwgt;
      return L2 ? tWeight * kLimitPositionWeight * lw * sq : tWeight * kLimitPositionWeight * lw * lossValue(e, sq);
    }
    default: break;
  }
  if (!active) { r[0] = 0.f; rc[0] = 0.f; return 0.f; }
  const float sq = res * res;
  const float wl = L2 ? sqrtf(tWeight * lw) : sqrtf(tWeight * lw * lossDeriv(e, sq));
  r[0] = res * wl;
  rc[0] = wl;
  return L2 ? tWeight * lw * sq : tWeight * lw * lossValue(e, sq);
}

// ------------------------------------------------------------------------------------------------
// Fill one Jacobian cell: rows [row0, row0+numRows) of column cell.col. Jcol points at the start
// of that column (row stride 1). Contributions are summed in the reference's walk order.
// ------------------------------------------------------------------------------------------------
MB2_HD void jacobianCell(const FunctionTables& T, int ci, const float* js, const float* rec, const float* targets, float* Jbase) {
  const CellDesc& c = T.cells[ci];
  const UnitDesc& u = T.units[c.unit];
  const float* rc = rec + u.recOff;
  // row k of the unit lands at out[MB2_ROW(k)]: contiguous in the K-major matrix; in the strip layout four rows of one quad are
  // contiguous and consecutive quads are quadStride strips apart
  float* out = T.stripMode ? Jbase + c.stripOff : Jbase + (size_t)c.col * T.ldJ + u.row0;
  const int rowShift = T.stripMode ? (u.row0 & 3) : 0, quadFloats = T.stripMode ? int(c.quadStride) * 64 : 4;
#define MB2_ROW(k) ((((k) + rowShift) >> 2) * quadFloats + (((k) + rowShift) & 3))
  const ContribDesc* cb = T.contribs + c.contribBegin;
  switch (u.kind) {
    case kUnitPosition:
    case kUnitLimitEllipsoid: {
      const F3 v = ld3(rc);
      const float ds = rc[3];
      F3 acc = f3(0.f, 0.f, 0.f);
      for (int k = 0; k < c.contribCount; ++k) acc = acc + (pointDerivative(T, js, cb[k].joint, cb[k].dof, v) * ds) * cb[k].coef;
#if defined(__CUDA_ARCH__)
      // strip layout, unit on a quad boundary (every multi-row unit owns whole quads: its fourth row is a structural zero): the three
      // rows of this column are ONE 16-byte store instead of three scattered 4-byte ones (the global stores were a third of the sweep's
      // LSU wavefronts, its busiest pipe)
      if (T.stripMode && rowShift == 0) { *reinterpret_cast<float4*>(out) = make_float4(acc.x, acc.y, acc.z, 0.f); break; }
#endif
      out[MB2_ROW(0)] = acc.x; out[MB2_ROW(1)] = acc.y; out[MB2_ROW(2)] = acc.z;
      break;
    }
    case kUnitPlane: {
      const F3 v = ld3(rc);
      F3 acc = f3(0.f, 0.f, 0.f);
      for (int k = 0; k < c.contribCount; ++k) acc = acc + pointDerivative(T, js, cb[k].joint, cb[k].dof, v) * cb[k].coef;
      out[MB2_ROW(0)] = dot(ld3(rc + 3), acc); // (sqrt(w loss') n)^T dv/dp
      break;
    }
    case kUnitOrientation:
    case kUnitOrientationRotDiff: {
      const float ds = rc[9];
      float acc[9];
      for (int k = 0; k < 9; ++k) acc[k] = 0.f;
      float it[9]; // R_target (RotDiff: rows 3k.. = R_t^T * d)
      if (u.kind == kUnitOrientationRotDiff) qmat(ld4(targets + u.targetOff), it);
      for (int k = 0; k < c.contribCount; ++k) {
        const F3 axis = rotationAxisCol(js, cb[k].joint, cb[k].dof - 3);
        for (int jv = 0; jv < 3; ++jv) {
          F3 d = cross(axis, ld3(rc + 3 * jv));
          if (u.kind == kUnitOrientationRotDiff) d = f3(it[0] * d.x + it[1] * d.y + it[2] * d.z, it[3] * d.x + it[4] * d.y + it[5] * d.z, it[6] * d.x + it[7] * d.y + it[8] * d.z);
          acc[3 * jv] += (ds * d.x) * cb[k].coef; acc[3 * jv + 1] += (ds * d.y) * cb[k].coef; acc[3 * jv + 2] += (ds * d.z) * cb[k].coef;
        }
      }
#if defined(__CUDA_ARCH__)
      if (T.stripMode && rowShift == 0) { // nine rows = three quads of this column (the last one holds row 8 and three structural zeros)
        *reinterpret_cast<float4*>(out) = make_float4(acc[0], acc[1], acc[2], acc[3]);
        *reinterpret_cast<float4*>(out + quadFloats) = make_float4(acc[4], acc[5], acc[6], acc[7]);
        *reinterpret_cast<float4*>(out + 2 * quadFloats) = make_float4(acc[8], 0.f, 0.f, 0.f);
        break;
      }
#endif
      for (int k = 0; k < 9; ++k) out[MB2_ROW(k)] = acc[k];
      break;
    }
    case kUnitStateMatrix:
    case kUnitStateLogMap: {
      const float wgt = rc[0], awgt = rc[1];
      const float* ps = js + u.joint * kJointStateStride;
      const F3 ti = ld3(ps);
      const Q4 rot = ld4(ps + 3);
      const bool lm = u.kind == kUnitStateLogMap;
      float acc[12];
      for (int k = 0; k < 12; ++k) acc[k] = 0.f;
      float rm[9];
      Q4 target = q4(0, 0, 0, 1);
      if (lm) target = qnormalized(ld4(targets + u.targetOff + 3)); else qmat(rot, rm);
      for (int k = 0; k < c.contribCount; ++k) {
        const int a = cb[k].joint, d = cb[k].dof;
        const float coef = cb[k].coef;
        const F3 jc = pointDerivative(T, js, a, d, ti) * wgt; // state_error_function.cpp:498-510,546-550
        acc[0] += jc.x * coef; acc[1] += jc.y * coef; acc[2] += jc.z * coef;
        if (d >= 3 && d < 6) {
          const F3 axis = rotationAxisCol(js, a, d - 3);
          if (lm) {
            const F3 jr = logMapRelativeDerivativeQ1(rot, target, axis, rc + 2) * awgt;
            acc[3] += jr.x * coef; acc[4] += jr.y * coef; acc[5] += jr.z * coef;
          } else { // vec([axis]x R) * awgt (state_error_function.cpp:116-121)
            for (int cc = 0; cc < 3; ++cc) {
              const F3 col = cross(axis, f3(rm[3 * cc], rm[3 * cc + 1], rm[3 * cc + 2]));
              acc[3 + 3 * cc] += (col.x * awgt) * coef; acc[4 + 3 * cc] += (col.y * awgt) * coef; acc[5 + 3 * cc] += (col.z * awgt) * coef;
            }
          }
        }
      }
      const int nr = lm ? 6 : 12;
      for (int k = 0; k < nr; ++k) out[MB2_ROW(k)] = acc[k];
      break;
    }
    default: // simple limits: value = wgtLoss * static coefficient
      out[MB2_ROW(0)] = rc[0] * c.coef;
      break;
  }
#undef MB2_ROW
}

// ---- Linear-blend skinning (linear_skinning.cpp:22-102) and its backward -------------------------------------------------------------
// M_j = T_j o IBP_j with T_j(y) = t + s R(q^) y (q^ = q / |q|, as pymomentum's skel-state backend normalises) and IBP_j = [N | c];
// p_i = sum_k w_ik M_{j_ik}(x_i). m: row-major 3x4, m[4 r + 3] the translation.
MB2_HD void skinTransform(const float* state, const float* ibp, float* m) {
  const Q4 q = qnormalized(ld4(state + 3));
  const float s = state[7];
  float R[9];
  qmat(q, R);
  for (int r = 0; r < 3; ++r) {
    const F3 sr = f3(s * R[r], s * R[3 + r], s * R[6 + r]); // row r of s R
    m[4 * r + 0] = dot(sr, f3(ibp[0], ibp[4], ibp[8]));
    m[4 * r + 1] = dot(sr, f3(ibp[1], ibp[5], ibp[9]));
    m[4 * r + 2] = dot(sr, f3(ibp[2], ibp[6], ibp[10]));
    m[4 * r + 3] = dot(sr, f3(ibp[3], ibp[7], ibp[11])) + state[r];
  }
}
// one vertex: sum over its active slots of w (t + L x), slots in order (linear_skinning.cpp:84-90); M: [J][12]
MB2_HD F3 skinBlend(const SkinTables& S, const float* M, int v, F3 x) {
  F3 p = f3(0.f, 0.f, 0.f);
  for (int k = S.vertStart[v]; k < S.vertStart[v + 1]; ++k) {
    const float* m = M + S.vertJoint[k] * kSkinIbpStride;
    const F3 temp = f3(m[3] + dot(ld3(m), x), m[7] + dot(ld3(m + 4), x), m[11] + dot(ld3(m + 8), x));
    p = p + temp * S.vertWeight[k];
  }
  return p;
}
// Backward, with g_i = dL/dp_i and the bone-local point y_ij = N_j x_i + c_j, per joint: a_j = sum w g_i (12 floats: a, then
// E_j = sum w g_i y_ij^T row-major). E is summed from the bone-local y: the expanded form (sum w g x^T) N^T + a c^T cancels
// catastrophically for a mesh far from the origin.
constexpr int kSkinAccFloats = 12;
MB2_HD void skinAccumulate(const float* ibp, F3 x, F3 g, float w, float* acc) {
  const F3 y = f3(dot(ld3(ibp), x) + ibp[3], dot(ld3(ibp + 4), x) + ibp[7], dot(ld3(ibp + 8), x) + ibp[11]);
  const F3 wg = g * w;
  acc[0] += wg.x; acc[1] += wg.y; acc[2] += wg.z;
  acc[3] += wg.x * y.x; acc[4] += wg.x * y.y; acc[5] += wg.x * y.z;
  acc[6] += wg.y * y.x; acc[7] += wg.y * y.y; acc[8] += wg.y * y.z;
  acc[9] += wg.z * y.x; acc[10] += wg.z * y.y; acc[11] += wg.z * y.z;
}
// (a_j, E_j) and the joint's state -> dL/d(t, q xyzw, s): dt = a, ds = <E, R(q^)>, dq^ = s d<E, R(q^)>/dq^ through the
// normalisation Jacobian (I - q^ q^T) / |q|
MB2_HD void skinStateGradient(const float* acc, const float* state, float* out) {
  const Q4 q = ld4(state + 3);
  const float nq = sqrtf(q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w);
  const Q4 u = q4(q.x / nq, q.y / nq, q.z / nq, q.w / nq);
  const float s = state[7];
  const float* E = acc + 3; // E[3 r + c]
  float R[9];
  qmat(u, R); // R[3 c + r]
  float ds = 0.f;
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) ds += E[3 * r + c] * R[3 * c + r];
  // d<E, R(u)>/du for Eigen's toRotationMatrix polynomial
  const float s01 = E[1] + E[3], s02 = E[2] + E[6], s12 = E[5] + E[7];
  const float d21 = E[7] - E[5], d02 = E[2] - E[6], d10 = E[3] - E[1];
  const float gx = 2.f * (u.y * s01 + u.z * s02 + u.w * d21 - 2.f * u.x * (E[4] + E[8]));
  const float gy = 2.f * (u.x * s01 + u.z * s12 + u.w * d02 - 2.f * u.y * (E[0] + E[8]));
  const float gz = 2.f * (u.x * s02 + u.y * s12 + u.w * d10 - 2.f * u.z * (E[0] + E[4]));
  const float gw = 2.f * (u.x * d21 + u.y * d02 + u.z * d10);
  const Q4 gu = q4(s * gx, s * gy, s * gz, s * gw);
  const float along = u.x * gu.x + u.y * gu.y + u.z * gu.z + u.w * gu.w;
  out[0] = acc[0]; out[1] = acc[1]; out[2] = acc[2];
  out[3] = (gu.x - u.x * along) / nq; out[4] = (gu.y - u.y * along) / nq;
  out[5] = (gu.z - u.z * along) / nq; out[6] = (gu.w - u.w * along) / nq;
  out[7] = ds;
}
// dL/dx_i = sum over the vertex's slots of w L_j^T g_i, slots in order
MB2_HD F3 skinRestGradient(const SkinTables& S, const float* M, int v, F3 g) {
  F3 r = f3(0.f, 0.f, 0.f);
  for (int k = S.vertStart[v]; k < S.vertStart[v + 1]; ++k) {
    const float* m = M + S.vertJoint[k] * kSkinIbpStride;
    const F3 lt = f3(m[0] * g.x + m[4] * g.y + m[8] * g.z, m[1] * g.x + m[5] * g.y + m[9] * g.z, m[2] * g.x + m[6] * g.y + m[10] * g.z);
    r = r + lt * S.vertWeight[k];
  }
  return r;
}

// ---- Blend-shape skinning (skinWithBlendShapes, blend_shape_skinning.cpp:50-140) ----------------------------------------------------
// The rest point of vertex v for T instances at once, x_t = base_v + sum_{k < K'} S_kv w_tk with k in order: each S_kv is read once
// for all T. w: [K'][T], instance fastest. The sum of an instance does not depend on T or on the other instances.
template <int T>
MB2_HD void blendShapeRest(const BlendShapeTables& Bs, int V, int v, const float* w, int numWeights, F3 (&x)[T]) {
  const F3 b = ld3(Bs.baseShape + 3 * size_t(v));
#pragma unroll
  for (int t = 0; t < T; ++t) x[t] = b;
  for (int k = 0; k < numWeights; ++k) {
    const F3 s = ld3(Bs.shapeVectors + (size_t(k) * V + v) * 3);
#pragma unroll
    for (int t = 0; t < T; ++t) x[t] = x[t] + s * w[k * T + t];
  }
}
// Backward: dL/dw_k = sum_v <S_kv, r_v> with r_v = dL/dx_v (skinRestGradient). One vertex's contribution, component by component.
MB2_HD float blendWeightAccumulate(float acc, F3 s, F3 r) {
  acc += s.x * r.x;
  acc += s.y * r.y;
  acc += s.z * r.z;
  return acc;
}

// ---- Vertex normals (pymomentum compute_vertex_normals, tensor_skinning.cpp:354-383; the sum of MeshT::updateNormals, mesh.cpp:17-51) --
// n_v = sum over the corners of the faces that are v of the face's (x1 - x0) x (x2 - x0), faces ascending, corners in order; the normal
// is n_v / max(|n_v|, 1e-12) (torch.nn.functional.normalize). Non-finite positions propagate (updateNormals' NaN-face skip is not copied).
constexpr float kNormalEps = 1e-12f;

MB2_HD F3 faceNormal(F3 x0, F3 x1, F3 x2) { return cross(x1 - x0, x2 - x0); }
MB2_HD F3 normalizeClamped(F3 n) {
  const float d = fmaxf(sqrtf(dot(n, n)), kNormalEps);
  return f3(n.x / d, n.y / d, n.z / d);
}
// Backward of normalizeClamped at n for the upstream g: h = (g - u (u . g)) / |n| with u = n / |n|, or g / 1e-12 on the clamp branch
// (|n| < 1e-12, an isolated vertex or one whose faces have zero area included).
MB2_HD F3 normalGradient(F3 n, F3 g) {
  const float len = sqrtf(dot(n, n));
  if (len < kNormalEps) return f3(g.x / kNormalEps, g.y / kNormalEps, g.z / kNormalEps);
  const F3 u = f3(n.x / len, n.y / len, n.z / len);
  const F3 p = g - u * dot(u, g);
  return f3(p.x / len, p.y / len, p.z / len);
}
// The gradient that corner k of a face adds to its vertex, with G the sum of h over the face's corners in order:
// d/dx_k [G . (x1 - x0) x (x2 - x0)] = (x_{k+1} - x_{k+2}) x G, corners mod 3.
MB2_HD F3 cornerGradient(F3 xNext, F3 xPrev, F3 G) { return cross(xNext - xPrev, G); }

// ---- Closest point on a triangle mesh (pymomentum find_closest_points_on_mesh over axel::TriBvh) ----------------------------------
// The closest point q of triangle (a, b, c) to p and its barycentrics (Ericson, Real-Time Collision Detection, 5.1.5; the region tests of
// axel::projectOnTriangle in the same order): the three vertex regions, the three edge regions, then the interior. A zero-area face whose
// point falls through to the interior gives NaN there.
MB2_HD void closestPointOnTriangle(F3 p, F3 a, F3 b, F3 c, F3& q, F3& bary) {
  const F3 ab = b - a, ac = c - a, ap = p - a;
  const float d1 = dot(ab, ap), d2 = dot(ac, ap);
  if (d1 <= 0.f && d2 <= 0.f) { q = a; bary = f3(1.f, 0.f, 0.f); return; }
  const F3 bp = p - b;
  const float d3 = dot(ab, bp), d4 = dot(ac, bp);
  if (d3 >= 0.f && d4 <= d3) { q = b; bary = f3(0.f, 1.f, 0.f); return; }
  const float vc = d1 * d4 - d3 * d2;
  if (vc <= 0.f && d1 >= 0.f && d3 <= 0.f) {
    const float v = d1 / (d1 - d3);
    q = a + v * ab; bary = f3(1.f - v, v, 0.f); return;
  }
  const F3 cp = p - c;
  const float d5 = dot(ab, cp), d6 = dot(ac, cp);
  if (d6 >= 0.f && d5 <= d6) { q = c; bary = f3(0.f, 0.f, 1.f); return; }
  const float vb = d5 * d2 - d1 * d6;
  if (vb <= 0.f && d2 >= 0.f && d6 <= 0.f) {
    const float w = d2 / (d2 - d6);
    q = a + w * ac; bary = f3(1.f - w, 0.f, w); return;
  }
  const float va = d3 * d6 - d5 * d4;
  if (va <= 0.f && (d4 - d3) >= 0.f && (d5 - d6) >= 0.f) {
    const float w = (d4 - d3) / ((d4 - d3) + (d5 - d6));
    q = b + w * (c - b); bary = f3(0.f, 1.f - w, w); return;
  }
  const float denom = 1.f / (va + vb + vc);
  const float v = vb * denom, w = vc * denom;
  q = a + ab * v + ac * w;
  bary = f3(1.f - v - w, v, w);
}

MB2_HD bool finite3(F3 a) { return fabsf(a.x) <= FLT_MAX && fabsf(a.y) <= FLT_MAX && fabsf(a.z) <= FLT_MAX; }

// d^2 = |q - p|^2 of face (a, b, c) with its q and barycentrics; NaN when a vertex is not finite, so that such a face is never a candidate
MB2_HD float faceDistance2(F3 p, F3 a, F3 b, F3 c, F3& q, F3& bary) {
  closestPointOnTriangle(p, a, b, c, q, bary);
  const F3 e = q - p;
  const float d2 = dot(e, e);
  return finite3(a) && finite3(b) && finite3(c) ? d2 : NAN;
}

// Face f with d2 is a candidate when d2 is finite and d2 <= maxDist2; the result is the candidate with the smallest (d2, f). With
// (best, bestFace) initialised to (maxDist2, INT_MAX), a candidate beats it exactly when closerFace holds.
MB2_HD bool closerFace(float d2, int f, float best, int bestFace) {
  return fabsf(d2) <= FLT_MAX && (d2 < best || (d2 == best && f < bestFace));
}

// A lower bound, in float, of the d2 that any face whose vertices lie in the box [lo, hi] can give at p (p finite). Per axis the gap
// g = max(lo - p, p - hi) is reduced by 2^-18 (M + |p|), M = max(|lo|, |hi|): that covers q of a face leaving the box by its rounding
// (at most 26 u M) and g's own rounding (u (M + |p|)), u = 2^-24; the sum of squares is then scaled by 1 - 2^-20 against the rounding of
// this sum (4 u) and of d2 (6 u). A non-finite box gives 0. DESIGN §4 has the argument. A subtree is pruned only when this is > best.
MB2_HD float boxLowerBound(const float* box, F3 p) { // box: lo xyz, hi xyz
  float s = 0.f;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const float pk = comp(p, k), lo = box[k], hi = box[3 + k];
    const float g = fmaxf(lo - pk, pk - hi);
    const float tau = 0x1p-18f * (fmaxf(fabsf(lo), fabsf(hi)) + fabsf(pk));
    const float h = fmaxf(g - tau, 0.f); // NaN (a non-finite box) gives 0
    s += h * h;
  }
  return s * (1.f - 0x1p-20f);
}
MB2_HD bool pruneBox(float lowerBound, float best) { return lowerBound > best; } // never on >=: an equal bound may hold a lower face index

// Refit: the box of a leaf is the exact min / max of its faces' vertices, the box of an internal node that of its two children's boxes.
// fminf / fmaxf skip NaN coordinates; a face with one is never a candidate (faceDistance2).
MB2_HD void boxEmpty(float* box) {
  box[0] = box[1] = box[2] = INFINITY;
  box[3] = box[4] = box[5] = -INFINITY;
}
MB2_HD void boxGrow(float* box, F3 x) {
  box[0] = fminf(box[0], x.x); box[1] = fminf(box[1], x.y); box[2] = fminf(box[2], x.z);
  box[3] = fmaxf(box[3], x.x); box[4] = fmaxf(box[4], x.y); box[5] = fmaxf(box[5], x.z);
}
MB2_HD void boxUnion(float* box, const float* l, const float* r) {
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    box[k] = fminf(l[k], r[k]);
    box[3 + k] = fmaxf(l[3 + k], r[3 + k]);
  }
}

// ---- Closest point of a point cloud (pymomentum find_closest_points over axel::SimdKdTree) ---------------------------------------
// d^2 = |t - p|^2 as an explicit fmaf chain, so that the device and the CPU emulator give the same bits with or without contraction;
// NaN when t is not finite, so that such a target is never a candidate (closerFace).
MB2_HD float pointDistance2(F3 p, F3 t) {
  const float dx = t.x - p.x, dy = t.y - p.y, dz = t.z - p.z;
  const float d2 = fmaf(dx, dx, fmaf(dy, dy, dz * dz));
  return finite3(t) ? d2 : NAN;
}
// The normal variant's filter: dot(n_p, n_t) >= maxNormalDot, the dot an explicit fmaf chain; a NaN dot never passes.
MB2_HD bool normalCompatible(F3 np, F3 nt, float maxNormalDot) { return fmaf(np.x, nt.x, fmaf(np.y, nt.y, np.z * nt.z)) >= maxNormalDot; }

// A box with no point on some axis (lo > hi: a padding leaf, or a leaf whose points all have a NaN there) holds no finite point.
MB2_HD bool boxVoid(const float* box) { return !(box[0] <= box[3] && box[1] <= box[4] && box[2] <= box[5]); }

// 10 bits of v spread to every third bit
MB2_HD uint32_t mortonSpread(uint32_t v) {
  v = (v | (v << 16)) & 0x030000FFu;
  v = (v | (v << 8)) & 0x0300F00Fu;
  v = (v | (v << 4)) & 0x030C30C3u;
  v = (v | (v << 2)) & 0x09249249u;
  return v;
}
// The 30-bit Morton code of x quantised to 1024 cells per axis of its instance's bounds [lo xyz, hi xyz] over the finite points: an
// axis of zero (or non-finite) extent gives 0 there; a point with a non-finite coordinate gets kMortonNonFinite, which sorts last.
MB2_HD uint32_t mortonCode(F3 x, const float* bounds) {
  if (!finite3(x)) return kMortonNonFinite;
  uint32_t c = 0;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const float lo = bounds[k], ext = bounds[3 + k] - lo;
    const float s = (comp(x, k) - lo) / ext * 1024.f; // NaN or not >= 1 when ext is 0 or not finite
    const uint32_t q = ext > 0.f && s >= 1.f ? uint32_t(fminf(s, 1023.f)) : 0u;
    c |= mortonSpread(q) << (2 - k);
  }
  return c;
}
// The implicit tree over m sorted points: the number of real leaves and P, the leaves padded to a power of two (P = 1 for m <= kLeafPoints)
MB2_HD int cloudLeaves(int m) { return (m + kLeafPoints - 1) / kLeafPoints; }
MB2_HD int cloudPadded(int m) {
  int P = 1;
  while (P < cloudLeaves(m)) P *= 2;
  return P;
}

} // namespace mb2
