// ORACLE — TEST INFRASTRUCTURE ONLY.
//
// CPU restatement (float and double) of facebookresearch/momentum's Gauss-Newton IK hot path.
// It is the checker for the CUDA product in momentum_b200/: only tests/, __graft_entry__.smoke()
// and bench.py's cpu_baseline / --impl reference legs may build, load or call anything here.
// The product never links or falls back to this code.
//
// Parity status: PINNED by the reference's own known-answer tests (SURVEY.md §8c, KA-1..KA-5) and
// the derivative property suites, see tests/test_oracle_known_answers.py. The reference itself cannot
// be compiled in this image (Eigen 5, ms-gsl, fmt, spdlog, dispenso absent), so Eigen's small-matrix
// and quaternion formulas are restated below (each tagged "Eigen:").
//
// Every function cites the reference file:line it follows (paths relative to the momentum/ directory of the momentum repository).
#pragma once

#include <algorithm>
#include <array>
#include <cfloat>
#include <cmath>
#include <cstddef>
#include <cstdint>
#include <limits>
#include <stdexcept>
#include <string>
#include <type_traits>
#include <vector>

namespace oracle {

constexpr int kParametersPerJoint = 7; // character/types.h:21
constexpr int kInvalid = -1; // kInvalidIndex (size_t max in the reference)

// math/constants.h:29-36
template <class T>
constexpr T Eps(double f, double d) {
  return std::is_same<T, float>::value ? T(f) : T(d);
}
template <class T>
constexpr T ln2() {
  return T(0.69314718055994530942); // math/constants.h:40
}
template <class T>
constexpr T pi() {
  return T(3.14159265358979323846);
}

// ----------------------------------------------------------------------------------------------
// Small fixed-size algebra (Eigen: Vector3 / Quaternion / Matrix3 formulas)
// ----------------------------------------------------------------------------------------------
template <class T>
struct V3 {
  T x{0}, y{0}, z{0};
  T& operator[](int i) { return i == 0 ? x : (i == 1 ? y : z); }
  const T& operator[](int i) const { return i == 0 ? x : (i == 1 ? y : z); }
};
template <class T> V3<T> operator+(V3<T> a, V3<T> b) { return {a.x + b.x, a.y + b.y, a.z + b.z}; }
template <class T> V3<T> operator-(V3<T> a, V3<T> b) { return {a.x - b.x, a.y - b.y, a.z - b.z}; }
template <class T> V3<T> operator-(V3<T> a) { return {-a.x, -a.y, -a.z}; }
template <class T> V3<T> operator*(V3<T> a, T s) { return {a.x * s, a.y * s, a.z * s}; }
template <class T> V3<T> operator*(T s, V3<T> a) { return {a.x * s, a.y * s, a.z * s}; }
template <class T> V3<T> operator/(V3<T> a, T s) { return {a.x / s, a.y / s, a.z / s}; }
template <class T> T dot(V3<T> a, V3<T> b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
template <class T> V3<T> cross(V3<T> a, V3<T> b) {
  return {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x};
}
template <class T> T sqnorm(V3<T> a) { return dot(a, a); }
template <class T> T norm(V3<T> a) { return std::sqrt(dot(a, a)); }

template <class T>
struct Quat { // coefficient order follows Eigen storage (x, y, z, w)
  T x{0}, y{0}, z{0}, w{1};
  V3<T> vec() const { return {x, y, z}; }
};
// Eigen: Quaternion product (Geometry/Quaternion.h, quat_product)
template <class T>
Quat<T> operator*(const Quat<T>& a, const Quat<T>& b) {
  Quat<T> r;
  r.w = a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z;
  r.x = a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y;
  r.y = a.w * b.y + a.y * b.w + a.z * b.x - a.x * b.z;
  r.z = a.w * b.z + a.z * b.w + a.x * b.y - a.y * b.x;
  return r;
}
// Eigen: QuaternionBase::_transformVector:  v + 2w(u x v) + 2 u x (u x v)
template <class T>
V3<T> rotate(const Quat<T>& q, V3<T> v) {
  V3<T> uv = cross(q.vec(), v);
  uv = uv + uv;
  return v + q.w * uv + cross(q.vec(), uv);
}
template <class T> Quat<T> conjugate(const Quat<T>& q) { return {-q.x, -q.y, -q.z, q.w}; }
template <class T> T sqnorm(const Quat<T>& q) { return q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w; }
template <class T> Quat<T> normalized(const Quat<T>& q) {
  const T n = std::sqrt(sqnorm(q));
  return {q.x / n, q.y / n, q.z / n, q.w / n};
}
// Eigen: QuaternionBase::inverse = conjugate / squaredNorm
template <class T> Quat<T> inverse(const Quat<T>& q) {
  const T n2 = sqnorm(q);
  return {-q.x / n2, -q.y / n2, -q.z / n2, q.w / n2};
}
// Eigen: Quaternion(AngleAxis(angle, unit axis k))
template <class T> Quat<T> axisAngle(int k, T angle) {
  const T ha = T(0.5) * angle;
  const T s = std::sin(ha);
  Quat<T> q;
  q.w = std::cos(ha);
  q.x = k == 0 ? s : T(0);
  q.y = k == 1 ? s : T(0);
  q.z = k == 2 ? s : T(0);
  return q;
}

template <class T>
struct M3 { // column access m.c[col][row]
  T c[3][3];
  V3<T> col(int j) const { return {c[j][0], c[j][1], c[j][2]}; }
  void setCol(int j, V3<T> v) { c[j][0] = v.x; c[j][1] = v.y; c[j][2] = v.z; }
  T operator()(int r, int cc) const { return c[cc][r]; }
  T& operator()(int r, int cc) { return c[cc][r]; }
  static M3 identity() {
    M3 m;
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) m.c[i][j] = (i == j) ? T(1) : T(0);
    return m;
  }
};
// Eigen: QuaternionBase::toRotationMatrix
template <class T>
M3<T> toRotationMatrix(const Quat<T>& q) {
  M3<T> R;
  const T tx = T(2) * q.x, ty = T(2) * q.y, tz = T(2) * q.z;
  const T twx = tx * q.w, twy = ty * q.w, twz = tz * q.w;
  const T txx = tx * q.x, txy = ty * q.x, txz = tz * q.x;
  const T tyy = ty * q.y, tyz = tz * q.y, tzz = tz * q.z;
  R(0, 0) = T(1) - (tyy + tzz); R(0, 1) = txy - twz; R(0, 2) = txz + twy;
  R(1, 0) = txy + twz; R(1, 1) = T(1) - (txx + tzz); R(1, 2) = tyz - twx;
  R(2, 0) = txz - twy; R(2, 1) = tyz + twx; R(2, 2) = T(1) - (txx + tyy);
  return R;
}
template <class T> V3<T> mul(const M3<T>& m, V3<T> v) {
  return {m(0, 0) * v.x + m(0, 1) * v.y + m(0, 2) * v.z, m(1, 0) * v.x + m(1, 1) * v.y + m(1, 2) * v.z,
          m(2, 0) * v.x + m(2, 1) * v.y + m(2, 2) * v.z};
}
template <class T> M3<T> mul(const M3<T>& a, const M3<T>& b) {
  M3<T> r;
  for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) {
    T s = 0;
    for (int k = 0; k < 3; ++k) s += a(i, k) * b(k, j);
    r(i, j) = s;
  }
  return r;
}
template <class T> M3<T> transpose(const M3<T>& a) {
  M3<T> r;
  for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) r(i, j) = a(j, i);
  return r;
}
// math/utility.h:340-344
template <class T> M3<T> crossProductMatrix(V3<T> v) {
  M3<T> r;
  r(0, 0) = 0; r(0, 1) = -v.z; r(0, 2) = v.y;
  r(1, 0) = v.z; r(1, 1) = 0; r(1, 2) = -v.x;
  r(2, 0) = -v.y; r(2, 1) = v.x; r(2, 2) = 0;
  return r;
}

// ----------------------------------------------------------------------------------------------
// math/transform.h:36-42 TransformT (translation, rotation, uniform scale)
// ----------------------------------------------------------------------------------------------
template <class T>
struct Transform {
  V3<T> t;
  Quat<T> q;
  T s{1};
  // math/transform.h:124-129
  Transform operator*(const Transform& o) const {
    Transform r;
    r.t = t + rotate(q, s * o.t);
    r.q = q * o.q;
    r.s = s * o.s;
    return r;
  }
  // math/transform.h:193-195
  V3<T> transformPoint(V3<T> p) const { return t + rotate(q, s * p); }
  // math/transform.h:165-167  toLinear = R * scale
  M3<T> toLinear() const {
    M3<T> R = toRotationMatrix(q);
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) R.c[i][j] *= s;
    return R;
  }
  // math/transform.cpp:93-101
  Transform inverse() const {
    Transform r;
    r.q = oracle::inverse(q);
    r.s = T(1) / s;
    r.t = -(r.s * rotate(r.q, t));
    return r;
  }
};

// ----------------------------------------------------------------------------------------------
// math/generalized_loss.h:46-110, generalized_loss.cpp:24-160
// ----------------------------------------------------------------------------------------------
template <class T>
struct GeneralizedLoss {
  enum Type { L1, L2, Cauchy, Welsch, General };
  T alpha, invC2;
  Type type;
  static constexpr T kWelsch() { return std::numeric_limits<T>::lowest(); }
  explicit GeneralizedLoss(T a = T(2), T c = T(1)) : alpha(a), invC2(T(1) / (c * c)) {
    if (!(c > 0)) throw std::runtime_error("Parameter c should be positive");
    const T kEps = T(1e-9);
    if (alpha >= T(2) - kEps && alpha <= T(2) + kEps) type = L2;
    else if (alpha >= T(1) - kEps && alpha <= T(1) + kEps) type = L1;
    else if (alpha >= T(0) - kEps && alpha <= T(0) + kEps) type = Cauchy;
    else if (alpha == kWelsch()) type = Welsch;
    else type = General;
  }
  bool isL2() const { return type == L2; }
  T value(T s) const { // generalized_loss.cpp:104-128
    switch (type) {
      case L2: return s * invC2;
      case L1: return std::sqrt(s * invC2 + T(1)) - T(1);
      case Cauchy: return std::log(T(0.5) * (s * invC2) + T(1));
      case Welsch: return T(1) - std::exp(T(-0.5) * (s * invC2));
      default:
        return (std::pow(s * invC2 / std::abs(alpha - T(2)) + T(1), T(0.5) * alpha) - T(1)) *
            std::abs(alpha - T(2)) / alpha;
    }
  }
  T deriv(T s) const { // generalized_loss.cpp:131-155
    switch (type) {
      case L2: return invC2;
      case L1: return T(0.5) * invC2 / std::sqrt(s * invC2 + T(1));
      case Cauchy: return invC2 / (invC2 * s + T(2));
      case Welsch: return T(0.5) * invC2 * std::exp(T(-0.5) * (s * invC2));
      default:
        return T(0.5) * invC2 * std::pow(s * invC2 / std::abs(alpha - T(2)) + T(1), T(0.5) * alpha - T(1));
    }
  }
};

// ----------------------------------------------------------------------------------------------
// math/utility.cpp:72-180 quaternion log map and its derivative
// ----------------------------------------------------------------------------------------------
template <class T>
V3<T> quaternionLogMap(const Quat<T>& q) {
  const Quat<T> qn = normalized(q);
  const T w = qn.w;
  const V3<T> vec = qn.vec();
  const T vecNorm = norm(vec);
  const T kSmall = Eps<T>(3.5e-4, 1.5e-8);
  if (vecNorm < kSmall) {
    if (w > T(0)) {
      const T scale = T(2) * (T(1) + sqnorm(vec) / T(6));
      return scale * vec;
    }
    return {pi<T>(), T(0), T(0)};
  }
  const T theta = T(2) * std::atan2(vecNorm, w);
  return (theta / vecNorm) * vec;
}
template <class T>
void quaternionLogMapDerivative(const Quat<T>& q, T jac[3][4]) { // jac[row][col], cols = x,y,z,w
  const Quat<T> qn = normalized(q);
  const T w = qn.w;
  const V3<T> vec = qn.vec();
  const T vecNorm = norm(vec);
  const T kSmall = Eps<T>(3.5e-4, 1.5e-8);
  if (vecNorm < kSmall) {
    const T scale = T(2) * (T(1) + sqnorm(vec) / T(6));
    for (int i = 0; i < 3; ++i) {
      for (int j = 0; j < 3; ++j) jac[i][j] = (i == j ? scale : T(0)) + T(2) * vec[i] * vec[j] / T(3);
      jac[i][3] = T(0);
    }
    return;
  }
  const T theta = T(2) * std::atan2(vecNorm, w);
  const T scale = theta / vecNorm;
  const T denom = w * w + vecNorm * vecNorm;
  const T dthetaDw = -T(2) * vecNorm / denom;
  for (int j = 0; j < 3; ++j) {
    const T dthetaDvecj = T(2) * w * vec[j] / (vecNorm * denom);
    const T dScale = dthetaDvecj / vecNorm - theta * vec[j] / (vecNorm * vecNorm * vecNorm);
    for (int i = 0; i < 3; ++i) jac[i][j] = dScale * vec[i] + (i == j ? scale : T(0));
  }
  for (int i = 0; i < 3; ++i) jac[i][3] = dthetaDw / vecNorm * vec[i];
}

// ----------------------------------------------------------------------------------------------
// character/parameter_limits.h:20-138
// ----------------------------------------------------------------------------------------------
enum LimitType { MinMax = 0, MinMaxJoint, MinMaxJointPassive, Linear, LinearJoint, Ellipsoid, HalfPlane };
struct Limit { // all limit data is float in the reference
  int type{MinMax};
  float weight{1.f};
  // MinMax: i0=parameterIndex, f0,f1 = limits.  MinMaxJoint: i0=jointIndex, i1=jointParameter.
  // Linear: i0=referenceIndex, i1=targetIndex, f0=scale, f1=offset, f2=rangeMin, f3=rangeMax.
  // LinearJoint: i0=refJoint, i1=refJointParam, i2=tgtJoint, i3=tgtJointParam, f0..f3 as Linear.
  // HalfPlane: i0=param1, i1=param2, f0,f1=normal, f2=offset.
  // Ellipsoid: i0=ellipsoidParent, i1=parent, f[0..11]=ellipsoid 3x4 (row-major linear|translation),
  //            f[12..23]=ellipsoidInv 3x4, f[24..26]=offset.
  int i[4]{0, 0, 0, 0};
  float f[27]{};
};
// character/parameter_limits.cpp:105-123
inline bool isInRange(float rangeMin, float rangeMax, float value) {
  if (rangeMin == 0 && rangeMax == 0) return true;
  return value >= rangeMin && value < rangeMax;
}

// ----------------------------------------------------------------------------------------------
// character/joint.h:18-76, skeleton.h:22-77, parameter_transform.h:62-184 (rig data is float)
// ----------------------------------------------------------------------------------------------
struct Rig {
  int numJoints{0};
  std::vector<int> parent; // -1 for root; parents precede children (skeleton.h:23-24)
  std::vector<float> offset; // 3 per joint (translationOffset)
  std::vector<float> prerot; // 4 per joint (x,y,z,w) (preRotation)
  int numParams{0};
  std::vector<int> outer, inner; // CSR of the 7J x n parameter transform (SparseRowMatrix)
  std::vector<float> vals;
  std::vector<float> ptOffsets; // 7J
  std::vector<Limit> limits;
  std::vector<uint8_t> activeJointParamsDefault; // ParameterTransform::activeJointParams

  // character/parameter_transform.cpp:97-107
  std::vector<uint8_t> computeActiveJointParams(const std::vector<uint8_t>& enabled) const {
    std::vector<uint8_t> r(numJoints * kParametersPerJoint, 0);
    for (int row = 0; row < numJoints * kParametersPerJoint; ++row)
      for (int k = outer[row]; k < outer[row + 1]; ++k)
        if (enabled[inner[k]]) r[row] = 1;
    return r;
  }
};

// character/joint_state.h:50-74
template <class T>
struct JointState {
  Transform<T> local, world;
  M3<T> translationAxis, rotationAxis;
  V3<T> translation() const { return world.t; }
  const Quat<T>& rotation() const { return world.q; }
  V3<T> getRotationDerivative(int d, V3<T> ref) const { return cross(rotationAxis.col(d), ref); } // joint_state.cpp:68-71
  V3<T> getTranslationDerivative(int d) const { return translationAxis.col(d); } // :74-77
  V3<T> getScaleDerivative(V3<T> ref) const { return ref * ln2<T>(); } // :80-82
};

template <class T>
struct SkeletonState {
  std::vector<T> jointParameters; // 7J
  std::vector<JointState<T>> jointState;
};

// character/parameter_transform.cpp:110-123  apply = transform * params + offsets
template <class T>
void applyParameterTransform(const Rig& rig, const T* params, std::vector<T>& jp) {
  const int rows = rig.numJoints * kParametersPerJoint;
  jp.assign(rows, T(0));
  for (int r = 0; r < rows; ++r) {
    T s = 0;
    for (int k = rig.outer[r]; k < rig.outer[r + 1]; ++k) s += T(rig.vals[k]) * params[rig.inner[k]];
    jp[r] = s + T(rig.ptOffsets[r]);
  }
}

// character/joint_state.cpp:22-65
template <class T>
void setJointState(const Rig& rig, int j, const T* p, const JointState<T>* parentState, JointState<T>& js) {
  Transform<T> parent;
  if (parentState != nullptr) parent = parentState->world;
  if (parentState != nullptr) js.translationAxis = parentState->world.toLinear(); // :36-42
  else js.translationAxis = M3<T>::identity();
  js.local.t = V3<T>{T(rig.offset[3 * j]) + p[0], T(rig.offset[3 * j + 1]) + p[1], T(rig.offset[3 * j + 2]) + p[2]}; // :44
  js.local.q = Quat<T>{T(rig.prerot[4 * j]), T(rig.prerot[4 * j + 1]), T(rig.prerot[4 * j + 2]), T(rig.prerot[4 * j + 3])}; // :46
  for (int index = 2; index >= 0; --index) { // :51-58
    V3<T> axis{T(index == 0), T(index == 1), T(index == 2)};
    js.rotationAxis.setCol(index, rotate(parent.q * js.local.q, axis));
    js.local.q = js.local.q * axisAngle<T>(index, p[3 + index]);
  }
  js.local.s = std::exp2(p[6]); // :62
  js.world = parent * js.local; // :64
}

// character/skeleton_state.cpp:87-121
template <class T>
void setSkeletonState(const Rig& rig, const std::vector<T>& jp, SkeletonState<T>& st) {
  st.jointParameters = jp;
  st.jointState.resize(rig.numJoints);
  for (int j = 0; j < rig.numJoints; ++j) {
    const int par = rig.parent[j];
    setJointState<T>(rig, j, &st.jointParameters[j * kParametersPerJoint], par < 0 ? nullptr : &st.jointState[par], st.jointState[j]);
  }
}

// ----------------------------------------------------------------------------------------------
// Dense column-major matrix helper (math/resizeable_matrix.h:40-117 semantics: zero-filled scratch)
// ----------------------------------------------------------------------------------------------
template <class T>
struct Mat {
  int rows{0}, cols{0};
  std::vector<T> a;
  void resizeAndSetZero(int r, int c) { rows = r; cols = c; a.assign(size_t(r) * c, T(0)); }
  T& operator()(int r, int c) { return a[size_t(c) * rows + r]; }
  T operator()(int r, int c) const { return a[size_t(c) * rows + r]; }
};

// ----------------------------------------------------------------------------------------------
// Error functions (character_solver/skeleton_error_function.h:19-150 base contract)
// ----------------------------------------------------------------------------------------------
enum Kind { kPosition = 0, kOrientation = 1, kOrientationRotDiff = 2, kState = 3, kLimit = 4, kPlane = 5, kModelParameters = 6 };
inline int funcDimOf(int kind) { return kind == kPosition ? 3 : kind == kPlane ? 1 : 9; } // JointErrorFunctionT<T, Data, FuncDim, NumVec, NumPos>
inline int numVecOf(int kind) { return (kind == kPosition || kind == kPlane) ? 1 : 3; }
inline int numPosOf(int kind) { return (kind == kPosition || kind == kPlane) ? 1 : 0; }
enum RotationErrorType { RotationMatrixDifference = 0, QuaternionLogMap = 1 }; // state_error_function.h:17-32

template <class T>
struct ErrorFunction {
  int kind{kPosition};
  T weight{1};
  T lossAlpha{2}, lossC{1};
  // joint-type constraints (error_function_types.h:34-44 ConstraintData: parent, float weight)
  std::vector<int> cparent;
  std::vector<float> cweight;
  std::vector<T> coffset; // 3 (position, plane) or 4 xyzw (orientation; normalised like OrientationDataT ctor)
  std::vector<T> ctarget; // 3 (position), 4 xyzw (orientation), or plane: unit normal xyz + d (PlaneDataT ctor normalises, plane_error_function.h:28-36)
  bool halfPlane{false};  // PlaneErrorFunctionT(above): plane_error_function.h:54-61
  // model parameters (model_parameters_error_function.h): per-parameter target and weight
  std::vector<T> targetParameters, targetWeights;
  // state
  int rotErrType{RotationMatrixDifference};
  T posWgt{1}, rotWgt{1};
  std::vector<T> targetPosW, targetRotW; // per joint
  std::vector<T> targetState; // 8 per joint: t(3), q(xyzw), s
  // set by SkeletonSolverFunction::setEnabledParameters (skeleton_solver_function.cpp:56-60)
  std::vector<uint8_t> activeJointParams;
  std::vector<uint8_t> enabledParameters;

  int numConstraints() const { return int(cparent.size()); }

  // getJacobianSize(): joint_error_function-inl.h:300-302, state_error_function.cpp:394-404,
  // limit_error_function.cpp:1138-1161
  int jacobianSize(const Rig& rig) const {
    switch (kind) {
      case kPosition: return 3 * numConstraints();
      case kOrientation:
      case kOrientationRotDiff: return 9 * numConstraints();
      case kState: {
        int n = 0;
        for (size_t i = 0; i < targetPosW.size(); ++i) n += (targetPosW[i] != 0 || targetRotW[i] != 0) ? 1 : 0;
        return n * (rotErrType == QuaternionLogMap ? 6 : 12);
      }
      case kPlane: return numConstraints();
      case kModelParameters: { // model_parameters_error_function.cpp:93-95
        int n = 0;
        for (T w : targetWeights) n += w > 0 ? 1 : 0;
        return n;
      }
      case kLimit: {
        int n = 0;
        for (const auto& l : rig.limits) {
          if (l.type == MinMaxJointPassive) continue;
          n += (l.type == Ellipsoid) ? 3 : 1;
        }
        return n;
      }
    }
    return 0;
  }
};

// --- joint-type evalFunction: position_error_function.cpp:15-27, orientation_error_function.cpp:15-65
template <class T>
void evalJointFunction(const ErrorFunction<T>& ef, int c, const JointState<T>& st, T* f, V3<T>* v, T dfdv[3][9][3]) {
  if (ef.kind == kPosition) {
    const V3<T> off{ef.coffset[3 * c], ef.coffset[3 * c + 1], ef.coffset[3 * c + 2]};
    v[0] = st.world.transformPoint(off);
    f[0] = v[0].x - ef.ctarget[3 * c];
    f[1] = v[0].y - ef.ctarget[3 * c + 1];
    f[2] = v[0].z - ef.ctarget[3 * c + 2];
    for (int r = 0; r < 3; ++r) for (int k = 0; k < 3; ++k) dfdv[0][r][k] = (r == k) ? T(1) : T(0);
    return;
  }
  if (ef.kind == kPlane) { // plane_error_function.cpp:49-70
    const V3<T> off{ef.coffset[3 * c], ef.coffset[3 * c + 1], ef.coffset[3 * c + 2]};
    const V3<T> nrm{ef.ctarget[4 * c], ef.ctarget[4 * c + 1], ef.ctarget[4 * c + 2]};
    v[0] = st.world.transformPoint(off);
    T val = dot(v[0], nrm) - ef.ctarget[4 * c + 3];
    if (ef.halfPlane && val > T(0)) val = T(0);
    f[0] = val;
    const bool on = !ef.halfPlane || val < T(0);
    for (int k = 0; k < 3; ++k) dfdv[0][0][k] = on ? nrm[k] : T(0);
    return;
  }
  const Quat<T> off{ef.coffset[4 * c], ef.coffset[4 * c + 1], ef.coffset[4 * c + 2], ef.coffset[4 * c + 3]};
  const Quat<T> tgt{ef.ctarget[4 * c], ef.ctarget[4 * c + 1], ef.ctarget[4 * c + 2], ef.ctarget[4 * c + 3]};
  const M3<T> rotMat = toRotationMatrix(off);
  const M3<T> tgtMat = toRotationMatrix(tgt);
  if (ef.kind == kOrientation) {
    for (int k = 0; k < 3; ++k) v[k] = rotate(st.rotation(), rotMat.col(k));
    for (int k = 0; k < 3; ++k) for (int r = 0; r < 3; ++r) f[3 * k + r] = v[k][r] - tgtMat(r, k);
    for (int iv = 0; iv < 3; ++iv)
      for (int r = 0; r < 9; ++r) for (int k = 0; k < 3; ++k) dfdv[iv][r][k] = (r == 3 * iv + k) ? T(1) : T(0);
  } else { // RotDiff: orientation_error_function.cpp:43-65
    const M3<T> vec = mul(toRotationMatrix(st.rotation()), rotMat);
    const M3<T> invTarget = transpose(tgtMat);
    const M3<T> prod = mul(invTarget, vec);
    for (int k = 0; k < 3; ++k) for (int r = 0; r < 3; ++r) f[3 * k + r] = prod(r, k) - (r == k ? T(1) : T(0));
    for (int k = 0; k < 3; ++k) v[k] = vec.col(k);
    for (int iv = 0; iv < 3; ++iv)
      for (int r = 0; r < 9; ++r) for (int k = 0; k < 3; ++k)
        dfdv[iv][r][k] = (r >= 3 * iv && r < 3 * iv + 3) ? invTarget(r - 3 * iv, k) : T(0);
  }
}

// joint_error_function-inl.h:35-54 getError
template <class T>
double jointGetError(const Rig&, const ErrorFunction<T>& ef, const SkeletonState<T>& state) {
  const int FuncDim = funcDimOf(ef.kind);
  const GeneralizedLoss<T> loss(ef.lossAlpha, ef.lossC);
  T f[9];
  V3<T> v[3];
  static thread_local T dfdv[3][9][3];
  double error = 0.0;
  for (int c = 0; c < ef.numConstraints(); ++c) {
    if (ef.cweight[c] == 0) continue;
    evalJointFunction(ef, c, state.jointState[ef.cparent[c]], f, v, dfdv);
    T sq = 0;
    for (int r = 0; r < FuncDim; ++r) sq += f[r] * f[r];
    error += ef.cweight[c] * loss.value(sq);
  }
  return ef.weight * error;
}

// joint_error_function-inl.h:179-297 getJacobian
template <class T>
double jointGetJacobian(const Rig& rig, const ErrorFunction<T>& ef, const SkeletonState<T>& state, Mat<T>& jac, int row0, T* residual, int& usedRows) {
  const int FuncDim = funcDimOf(ef.kind), NumVec = numVecOf(ef.kind), NumPos = numPosOf(ef.kind);
  const GeneralizedLoss<T> loss(ef.lossAlpha, ef.lossC);
  usedRows = FuncDim * ef.numConstraints();
  T f[9];
  V3<T> v[3];
  static thread_local T dfdv[3][9][3];
  double error = 0.0;
  for (int c = 0; c < ef.numConstraints(); ++c) {
    if (ef.cweight[c] == 0) continue; // :197-199
    evalJointFunction(ef, c, state.jointState[ef.cparent[c]], f, v, dfdv);
    T sq = 0;
    for (int r = 0; r < FuncDim; ++r) sq += f[r] * f[r];
    const T w = ef.cweight[c] * ef.weight;
    error += w * loss.value(sq);
    const T derivScale = std::sqrt(w * loss.deriv(sq));
    const int rowIndex = row0 + FuncDim * c;
    for (int r = 0; r < FuncDim; ++r) residual[rowIndex + r] = derivScale * f[r];
    if (std::abs(derivScale - T(0)) < Eps<T>(1e-9, 1e-16)) continue; // :216-218
    { // :219-223 all-zero dfdv (the clamped half plane): rows stay zero
      bool any = false;
      for (int jv = 0; jv < NumVec; ++jv) for (int r = 0; r < FuncDim; ++r) for (int k = 0; k < 3; ++k) any = any || dfdv[jv][r][k] != T(0);
      if (!any) continue;
    }
    int jnt = ef.cparent[c];
    while (jnt != kInvalid) { // :229-294
      const JointState<T>& js = state.jointState[jnt];
      const int pbase = jnt * kParametersPerJoint;
      for (int jv = 0; jv < NumVec; ++jv) {
        V3<T> offset = (jv < NumPos) ? (v[jv] - js.translation()) : v[jv];
        auto scatter = [&](int jointParam, V3<T> d) {
          T jc[9];
          for (int r = 0; r < FuncDim; ++r)
            jc[r] = derivScale * (dfdv[jv][r][0] * d.x + dfdv[jv][r][1] * d.y + dfdv[jv][r][2] * d.z);
          for (int k = rig.outer[jointParam]; k < rig.outer[jointParam + 1]; ++k) {
            const int col = rig.inner[k];
            if (ef.enabledParameters[col])
              for (int r = 0; r < FuncDim; ++r) jac(rowIndex + r, col) += jc[r] * T(rig.vals[k]);
          }
        };
        if (jv < NumPos)
          for (int d = 0; d < 3; ++d)
            if (ef.activeJointParams[pbase + d]) scatter(pbase + d, js.getTranslationDerivative(d));
        for (int d = 0; d < 3; ++d)
          if (ef.activeJointParams[pbase + 3 + d]) scatter(pbase + 3 + d, js.getRotationDerivative(d, offset));
        if (jv < NumPos)
          if (ef.activeJointParams[pbase + 6]) scatter(pbase + 6, js.getScaleDerivative(offset));
      }
      jnt = rig.parent[jnt];
    }
  }
  return error;
}

// --- State: state_error_function.cpp:199-262 (error), :407-558 (Jacobian), helpers :33-121
template <class T>
Transform<T> stateTarget(const ErrorFunction<T>& ef, int i) {
  Transform<T> t;
  const T* p = &ef.targetState[8 * i];
  t.t = {p[0], p[1], p[2]};
  t.q = {p[3], p[4], p[5], p[6]};
  t.s = p[7];
  return t;
}
template <class T>
double stateGetError(const Rig& rig, const ErrorFunction<T>& ef, const SkeletonState<T>& state) {
  const T kPositionWeight = T(1e-3), kOrientationWeight = T(1); // state_error_function.h:115-116
  double error = 0.0;
  if (int(ef.targetState.size()) != 8 * rig.numJoints) return error;
  for (int i = 0; i < rig.numJoints; ++i) {
    T rotationError = 0;
    const Quat<T> target = normalized(stateTarget(ef, i).q);
    const Quat<T>& rot = state.jointState[i].rotation();
    if (ef.rotErrType == QuaternionLogMap) {
      rotationError = sqnorm(quaternionLogMap(conjugate(target) * rot));
    } else {
      const M3<T> a = toRotationMatrix(rot), b = toRotationMatrix(target);
      for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) rotationError += (a(r, c) - b(r, c)) * (a(r, c) - b(r, c));
    }
    error += rotationError * kOrientationWeight * ef.rotWgt * ef.targetRotW[i];
    const V3<T> diff = state.jointState[i].translation() - stateTarget(ef, i).t;
    error += sqnorm(diff) * kPositionWeight * ef.posWgt * ef.targetPosW[i];
  }
  return error * ef.weight;
}
// state_error_function.cpp:33-66
template <class T>
V3<T> quaternionLogMapRelativeDerivativeQ1(const Quat<T>& q1, const Quat<T>& q2, V3<T> dir, const T dLogDq[3][4]) {
  const V3<T> vHalf = dir / T(2);
  const V3<T> q1v = q1.vec();
  const T dq1w = -dot(vHalf, q1v);
  const V3<T> dq1v = vHalf * q1.w + cross(vHalf, q1v);
  const V3<T> mq2v = -q2.vec();
  const T dqRelW = q2.w * dq1w - dot(mq2v, dq1v);
  const V3<T> dqRelV = q2.w * dq1v + dq1w * mq2v + cross(mq2v, dq1v);
  V3<T> r;
  for (int i = 0; i < 3; ++i) r[i] = dLogDq[i][0] * dqRelV.x + dLogDq[i][1] * dqRelV.y + dLogDq[i][2] * dqRelV.z + dLogDq[i][3] * dqRelW;
  return r;
}
template <class T>
double stateGetJacobian(const Rig& rig, const ErrorFunction<T>& ef, const SkeletonState<T>& state, Mat<T>& jac, int row0, T* residual, int& usedRows) {
  const T kPositionWeight = T(1e-3), kOrientationWeight = T(1);
  double error = 0.0;
  usedRows = 0;
  if (int(ef.targetState.size()) != 8 * rig.numJoints) return error;
  int offset = row0;
  const int rotSize = (ef.rotErrType == QuaternionLogMap) ? 3 : 9;
  // error_function_utils.h:33-45 — no enabledParameters gating
  auto toModel = [&](const T* jc, int nr, int jointParam, int rowStart) {
    for (int k = rig.outer[jointParam]; k < rig.outer[jointParam + 1]; ++k)
      for (int r = 0; r < nr; ++r) jac(rowStart + r, rig.inner[k]) += jc[r] * T(rig.vals[k]);
  };
  for (int i = 0; i < rig.numJoints; ++i) {
    if (ef.targetRotW[i] == 0 && ef.targetPosW[i] == 0) continue;
    const Transform<T> tgt = stateTarget(ef, i);
    const V3<T> transDiff = state.jointState[i].translation() - tgt.t;
    const Quat<T> target = normalized(tgt.q);
    const Quat<T>& rot = state.jointState[i].rotation();
    const T pwgt = kPositionWeight * ef.posWgt * ef.weight * ef.targetPosW[i];
    const T rwgt = kOrientationWeight * ef.rotWgt * ef.weight * ef.targetRotW[i];
    const T wgt = std::sqrt(pwgt), awgt = std::sqrt(rwgt);
    error += sqnorm(transDiff) * pwgt;
    for (int r = 0; r < 3; ++r) residual[offset + r] = transDiff[r] * wgt;
    T dLogDq[3][4];
    const M3<T> rotM = toRotationMatrix(rot);
    if (ef.rotErrType == QuaternionLogMap) {
      const Quat<T> qRel = conjugate(target) * rot;
      quaternionLogMapDerivative(qRel, dLogDq);
      const V3<T> lv = quaternionLogMap(qRel);
      error += sqnorm(lv) * rwgt;
      for (int r = 0; r < 3; ++r) residual[offset + 3 + r] = lv[r] * awgt;
    } else {
      const M3<T> b = toRotationMatrix(target);
      T sq = 0;
      for (int c = 0; c < 3; ++c) for (int r = 0; r < 3; ++r) {
        const T d = rotM(r, c) - b(r, c);
        sq += d * d;
        residual[offset + 3 + 3 * c + r] = d * awgt;
      }
      error += sq * rwgt;
    }
    int jnt = i;
    while (jnt != kInvalid) {
      const JointState<T>& js = state.jointState[jnt];
      const int pbase = jnt * kParametersPerJoint;
      const V3<T> posd = state.jointState[i].translation() - js.translation();
      for (int d = 0; d < 3; ++d) {
        if (ef.activeJointParams[pbase + d]) {
          const V3<T> jc = js.getTranslationDerivative(d) * wgt;
          const T a[3] = {jc.x, jc.y, jc.z};
          toModel(a, 3, pbase + d, offset);
        }
        if (ef.activeJointParams[pbase + 3 + d]) {
          const V3<T> jc = js.getRotationDerivative(d, posd) * wgt;
          const T a[3] = {jc.x, jc.y, jc.z};
          toModel(a, 3, pbase + 3 + d, offset);
          const V3<T> axis = js.rotationAxis.col(d);
          if (ef.rotErrType == QuaternionLogMap) {
            const V3<T> jr = awgt * quaternionLogMapRelativeDerivativeQ1(rot, target, axis, dLogDq);
            const T b[3] = {jr.x, jr.y, jr.z};
            toModel(b, 3, pbase + 3 + d, offset + 3);
          } else {
            const M3<T> rotD = mul(crossProductMatrix(axis), rotM); // state_error_function.cpp:116-121
            T b[9];
            for (int c = 0; c < 3; ++c) for (int r = 0; r < 3; ++r) b[3 * c + r] = rotD(r, c) * awgt;
            toModel(b, 9, pbase + 3 + d, offset + 3);
          }
        }
      }
      if (ef.activeJointParams[pbase + 6]) {
        const V3<T> jc = js.getScaleDerivative(posd) * wgt;
        const T a[3] = {jc.x, jc.y, jc.z};
        toModel(a, 3, pbase + 6, offset);
      }
      jnt = rig.parent[jnt];
    }
    offset += 3 + rotSize;
  }
  usedRows = offset - row0;
  return error;
}

// --- Limit: limit_error_function.cpp:31-193 (error), :459-785 (Jacobians), :818-867, :992-1161
constexpr float kLimitWeight = 10.f; // limit_error_function.h:91
constexpr float kLimitPositionWeight = 1e-4f; // limit_error_function.cpp:21

template <class T>
struct EllipsoidEval {
  V3<T> position, diff;
};
template <class T>
EllipsoidEval<T> evalEllipsoid(const Limit& l, const SkeletonState<T>& state) {
  // limit_error_function.cpp:176-187 / :713-722
  auto affine = [&](const float* a, V3<T> p) {
    V3<T> r;
    for (int i = 0; i < 3; ++i) r[i] = T(a[4 * i]) * p.x + T(a[4 * i + 1]) * p.y + T(a[4 * i + 2]) * p.z + T(a[4 * i + 3]);
    return r;
  };
  EllipsoidEval<T> e;
  const V3<T> off{T(l.f[24]), T(l.f[25]), T(l.f[26])};
  e.position = state.jointState[l.i[1]].world.transformPoint(off);
  const V3<T> localPosition = state.jointState[l.i[0]].world.inverse().transformPoint(e.position);
  const V3<T> ellipsoidPosition = affine(&l.f[12], localPosition);
  const V3<T> normalizedPosition = ellipsoidPosition / norm(ellipsoidPosition);
  const V3<T> projected = affine(&l.f[0], normalizedPosition);
  e.diff = e.position - state.jointState[l.i[0]].world.transformPoint(projected);
  return e;
}

template <class T>
double limitGetError(const Rig& rig, const ErrorFunction<T>& ef, const T* params, const SkeletonState<T>& state) {
  const GeneralizedLoss<T> loss(ef.lossAlpha, ef.lossC);
  const bool L2 = loss.isL2();
  auto lv = [&](T s) { return L2 ? s : loss.value(s); };
  double error = 0.0;
  for (const Limit& l : rig.limits) {
    const T lw = T(l.weight);
    switch (l.type) {
      case MinMax: {
        if (!ef.enabledParameters[l.i[0]]) break;
        T e = 0;
        if (params[l.i[0]] < l.f[0]) { const T v = l.f[0] - params[l.i[0]]; e = lw * lv(v * v); }
        if (params[l.i[0]] > l.f[1]) { const T v = l.f[1] - params[l.i[0]]; e = lw * lv(v * v); }
        error += e;
        break;
      }
      case MinMaxJoint: {
        const int pi = l.i[0] * kParametersPerJoint + l.i[1];
        if (!ef.activeJointParams[pi]) break;
        T e = 0;
        if (state.jointParameters[pi] < l.f[0]) { const T v = l.f[0] - state.jointParameters[pi]; e = lw * lv(v * v); }
        if (state.jointParameters[pi] > l.f[1]) { const T v = l.f[1] - state.jointParameters[pi]; e = lw * lv(v * v); }
        error += e;
        break;
      }
      case MinMaxJointPassive: break;
      case Linear: {
        if ((!ef.enabledParameters[l.i[1]] && !ef.enabledParameters[l.i[0]]) || !isInRange(l.f[2], l.f[3], float(params[l.i[1]]))) break;
        const T res = params[l.i[1]] * l.f[0] - l.f[1] - params[l.i[0]];
        error += lw * lv(res * res);
        break;
      }
      case LinearJoint: {
        const int ri = l.i[0] * kParametersPerJoint + l.i[1];
        const int ti = l.i[2] * kParametersPerJoint + l.i[3];
        if ((!ef.activeJointParams[ri] && !ef.activeJointParams[ti]) || !isInRange(l.f[2], l.f[3], float(state.jointParameters[ti]))) break;
        const T res = state.jointParameters[ti] * l.f[0] - l.f[1] - state.jointParameters[ri];
        error += lw * lv(res * res);
        break;
      }
      case HalfPlane: {
        if (!ef.enabledParameters[l.i[0]] && !ef.enabledParameters[l.i[1]]) break;
        const T res = params[l.i[0]] * T(l.f[0]) + params[l.i[1]] * T(l.f[1]) - l.f[2];
        if (res < 0) error += lw * lv(res * res);
        break;
      }
      case Ellipsoid: {
        const EllipsoidEval<T> e = evalEllipsoid(l, state);
        error += T(kLimitPositionWeight) * lw * lv(sqnorm(e.diff));
        break;
      }
      default: throw std::runtime_error("Unknown parameter type for joint limit");
    }
  }
  // limit_error_function.cpp:859-865
  if (L2) return error * kLimitWeight * ef.weight * loss.invC2;
  return error * kLimitWeight * ef.weight;
}

template <class T>
double limitGetJacobian(const Rig& rig, const ErrorFunction<T>& ef, const T* params, const SkeletonState<T>& state, Mat<T>& jac, int row0, T* residual, int& usedRows) {
  const GeneralizedLoss<T> loss(ef.lossAlpha, ef.lossC);
  const bool L2 = loss.isL2();
  double error = 0.0;
  T tWeight = kLimitWeight * ef.weight; // :1006-1009
  if (L2) tWeight *= loss.invC2;
  int count = row0;
  auto rowToModel = [&](T val, int jointParam, int row) { // error_function_utils.h:77-91
    for (int k = rig.outer[jointParam]; k < rig.outer[jointParam + 1]; ++k) jac(row, rig.inner[k]) += val * T(rig.vals[k]);
  };
  for (const Limit& l : rig.limits) {
    const T lw = T(l.weight);
    const T wgtL2 = L2 ? std::sqrt(tWeight * lw) : T(0);
    auto wl = [&](T sq) { return L2 ? wgtL2 : std::sqrt(tWeight * lw * loss.deriv(sq)); };
    auto ev = [&](T sq) { return L2 ? tWeight * lw * sq : tWeight * lw * loss.value(sq); };
    switch (l.type) {
      case MinMax: { // :459-503
        const int p = l.i[0];
        if (ef.enabledParameters[p]) {
          if (params[p] < l.f[0]) {
            const T val = params[p] - l.f[0];
            const T w = wl(val * val);
            jac(count, p) = w; residual[count] = val * w; error += ev(val * val);
          } else if (params[p] > l.f[1]) {
            const T val = params[p] - l.f[1];
            const T w = wl(val * val);
            jac(count, p) = w; residual[count] = val * w; error += ev(val * val);
          }
        }
        count++;
        break;
      }
      case MinMaxJoint: { // :505-558
        const int pi = l.i[0] * kParametersPerJoint + l.i[1];
        if (ef.activeJointParams[pi]) {
          if (state.jointParameters[pi] < l.f[0]) {
            const T val = state.jointParameters[pi] - l.f[0];
            const T w = wl(val * val);
            rowToModel(w, pi, count); residual[count] = val * w; error += ev(val * val);
          } else if (state.jointParameters[pi] > l.f[1]) {
            const T val = state.jointParameters[pi] - l.f[1];
            const T w = wl(val * val);
            rowToModel(w, pi, count); residual[count] = val * w; error += ev(val * val);
          }
        }
        count++;
        break;
      }
      case MinMaxJointPassive: break;
      case Linear: { // :560-598
        const int ref = l.i[0], tgt = l.i[1];
        if (!((!ef.enabledParameters[tgt] && !ef.enabledParameters[ref]) || !isInRange(l.f[2], l.f[3], float(params[tgt])))) {
          const T res = params[tgt] * l.f[0] - l.f[1] - params[ref];
          const T w = wl(res * res);
          residual[count] = res * w;
          if (ef.enabledParameters[tgt]) jac(count, tgt) = T(l.f[0]) * w;
          if (ef.enabledParameters[ref]) jac(count, ref) = -w;
          error += ev(res * res);
        }
        count++;
        break;
      }
      case LinearJoint: { // :600-656
        const int ri = l.i[0] * kParametersPerJoint + l.i[1];
        const int ti = l.i[2] * kParametersPerJoint + l.i[3];
        if (!((!ef.activeJointParams[ri] && !ef.activeJointParams[ti]) || !isInRange(l.f[2], l.f[3], float(state.jointParameters[ti])))) {
          const T res = state.jointParameters[ti] * l.f[0] - l.f[1] - state.jointParameters[ri];
          const T w = wl(res * res);
          residual[count] = res * w;
          if (ef.activeJointParams[ti]) rowToModel(T(l.f[0]) * w, ti, count);
          if (ef.activeJointParams[ri]) rowToModel(-w, ri, count);
          error += ev(res * res);
        }
        count++;
        break;
      }
      case HalfPlane: { // :658-699
        const int p1 = l.i[0], p2 = l.i[1];
        if (ef.enabledParameters[p1] || ef.enabledParameters[p2]) {
          const T res = params[p1] * T(l.f[0]) + params[p2] * T(l.f[1]) - l.f[2];
          if (res < T(0)) {
            const T w = wl(res * res);
            residual[count] = res * w;
            if (ef.enabledParameters[p1]) jac(count, p1) = T(l.f[0]) * w;
            if (ef.enabledParameters[p2]) jac(count, p2) = T(l.f[1]) * w;
            error += ev(res * res);
          }
        }
        count++;
        break;
      }
      case Ellipsoid: { // :701-785
        const EllipsoidEval<T> e = evalEllipsoid(l, state);
        const T sq = sqnorm(e.diff);
        const T jwgt = L2 ? std::sqrt(tWeight * T(kLimitPositionWeight) * lw)
                          : std::sqrt(tWeight * T(kLimitPositionWeight) * lw * loss.deriv(sq));
        int jnt = l.i[1];
        while (jnt != l.i[0] && jnt != kInvalid) {
          const JointState<T>& js = state.jointState[jnt];
          const int pbase = jnt * kParametersPerJoint;
          const V3<T> posd = e.position - js.translation();
          auto col3 = [&](V3<T> jc, int jointParam) {
            for (int k = rig.outer[jointParam]; k < rig.outer[jointParam + 1]; ++k)
              for (int r = 0; r < 3; ++r) jac(count + r, rig.inner[k]) += jc[r] * T(rig.vals[k]);
          };
          for (int d = 0; d < 3; ++d) {
            if (ef.activeJointParams[pbase + d]) col3(js.getTranslationDerivative(d) * jwgt, pbase + d);
            if (ef.activeJointParams[pbase + 3 + d]) col3(js.getRotationDerivative(d, posd) * jwgt, pbase + 3 + d);
          }
          if (ef.activeJointParams[pbase + 6]) col3(js.getScaleDerivative(posd) * jwgt, pbase + 6);
          jnt = rig.parent[jnt];
        }
        for (int r = 0; r < 3; ++r) residual[count + r] = e.diff[r] * jwgt;
        error += L2 ? tWeight * T(kLimitPositionWeight) * lw * sq : tWeight * T(kLimitPositionWeight) * lw * loss.value(sq);
        count += 3;
        break;
      }
      default: throw std::runtime_error("Unknown parameter type for joint limit");
    }
  }
  usedRows = count - row0;
  return error;
}

// --- ModelParametersErrorFunctionT: model_parameters_error_function.cpp:38-58 (error), :90-133 (Jacobian); kMotionWeight = 1e-1 (.h:61)
template <class T>
double modelParametersGetError(const ErrorFunction<T>& ef, const T* params, int n) {
  if (int(ef.targetParameters.size()) != n || int(ef.targetWeights.size()) != n) return 0.0;
  const T kMotionWeight = T(1e-1);
  double error = 0;
  for (int i = 0; i < n; ++i)
    if (ef.enabledParameters[i]) {
      const T pdiff = ef.targetWeights[i] * (params[i] - ef.targetParameters[i]);
      error += pdiff * pdiff;
    }
  return error * ef.weight * kMotionWeight;
}
template <class T>
double modelParametersGetJacobian(const ErrorFunction<T>& ef, const T* params, int n, Mat<T>& jac, int row0, T* residual, int& usedRows) {
  usedRows = 0;
  if (int(ef.targetParameters.size()) != n || int(ef.targetWeights.size()) != n) return 0.0;
  const T kMotionWeight = T(1e-1);
  const float sWeight = std::sqrt(float(ef.weight * kMotionWeight)); // `const float sWeight` in the reference (:108)
  int out = 0;
  double error = 0;
  for (int i = 0; i < n; ++i)
    if (ef.enabledParameters[i] && ef.targetWeights[i] > 0) {
      const T pdiff = ef.targetWeights[i] * (params[i] - ef.targetParameters[i]);
      error += pdiff * pdiff;
      residual[row0 + out] = pdiff * T(sWeight);
      jac(row0 + out, i) = T(sWeight) * ef.targetWeights[i];
      ++out;
    }
  usedRows = out;
  return error * ef.weight * kMotionWeight;
}

// ----------------------------------------------------------------------------------------------
// character_solver/skeleton_solver_function.{h,cpp} + solver/solver_function.{h,cpp}
// ----------------------------------------------------------------------------------------------
inline int padToSimdAlignment(int n) { return (n + 7) & ~7; } // solver_function.h:27-29

template <class T>
struct SkeletonSolverFunction {
  const Rig* rig{nullptr};
  std::vector<ErrorFunction<T>> errorFunctions;
  int numParameters{0}, actualParameters{0};
  std::vector<uint8_t> activeJointParams;
  SkeletonState<T> state;
  std::vector<T> jpScratch;
  Mat<T> tJacobian;
  std::vector<T> tResidual, jt_;

  explicit SkeletonSolverFunction(const Rig* r) : rig(r) { // skeleton_solver_function.cpp:25-39
    numParameters = actualParameters = r->numParams;
    activeJointParams = r->activeJointParamsDefault;
  }
  void addErrorFunction(ErrorFunction<T> ef) { // skeleton_error_function.h:22-29 defaults
    ef.activeJointParams = rig->activeJointParamsDefault;
    ef.enabledParameters.assign(rig->numParams, 1);
    errorFunctions.push_back(std::move(ef));
  }
  // skeleton_solver_function.cpp:45-61
  void setEnabledParameters(const std::vector<uint8_t>& ps) {
    actualParameters = 0;
    for (int i = 0; i < numParameters; ++i) if (ps[i]) actualParameters = i + 1;
    activeJointParams = rig->computeActiveJointParams(ps);
    for (auto& ef : errorFunctions) { ef.activeJointParams = activeJointParams; ef.enabledParameters = ps; }
  }
  void updateState(const T* params) { // :200-214
    applyParameterTransform<T>(*rig, params, jpScratch);
    setSkeletonState<T>(*rig, jpScratch, state);
  }
  // skeleton_solver_function.cpp:64-83 (note the float cast at :82)
  double getError(const T* params) {
    updateState(params);
    double error = 0.0;
    for (auto& ef : errorFunctions) {
      if (!(ef.weight > 0)) continue;
      double e = 0;
      if (ef.kind == kState) e = stateGetError(*rig, ef, state);
      else if (ef.kind == kLimit) e = limitGetError(*rig, ef, params, state);
      else if (ef.kind == kModelParameters) e = modelParametersGetError(ef, params, numParameters);
      else e = jointGetError(*rig, ef, state);
      error += e;
    }
    return (float)error;
  }
  size_t getJacobianBlockCount() const { return errorFunctions.size(); }
  int getJacobianBlockSize(size_t i) const { // :222-233
    if (!(errorFunctions[i].weight > 0)) return 0;
    return errorFunctions[i].jacobianSize(*rig);
  }
  // :235-261
  double computeJacobianBlock(const T* params, size_t i, Mat<T>& jac, int row0, T* residual, int& actualRows) {
    const auto& ef = errorFunctions[i];
    actualRows = 0;
    if (!(ef.weight > 0)) return 0.0;
    if (ef.kind == kState) return stateGetJacobian(*rig, ef, state, jac, row0, residual, actualRows);
    if (ef.kind == kLimit) return limitGetJacobian(*rig, ef, params, state, jac, row0, residual, actualRows);
    if (ef.kind == kModelParameters) return modelParametersGetJacobian(ef, params, numParameters, jac, row0, residual, actualRows);
    return jointGetJacobian(*rig, ef, state, jac, row0, residual, actualRows);
  }
  // solver_function.cpp:22-71 default getJacobian (rows padded to 8)
  double getJacobian(const T* params, Mat<T>& jac, std::vector<T>& residual, int& actualRows) {
    updateState(params);
    int total = 0;
    for (size_t i = 0; i < errorFunctions.size(); ++i) total += getJacobianBlockSize(i);
    total = padToSimdAlignment(total);
    jac.resizeAndSetZero(total, numParameters);
    residual.assign(total, T(0));
    double error = 0.0;
    int position = 0;
    actualRows = total;
    for (size_t i = 0; i < errorFunctions.size(); ++i) {
      const int bs = getJacobianBlockSize(i);
      if (bs == 0) continue;
      int rows = 0;
      error += computeJacobianBlock(params, i, jac, position, residual.data(), rows);
      position += bs;
    }
    return error;
  }
  // solver_function.cpp:74-121 default getJtJR: per block, lower-triangular rankUpdate + GEMV
  double getJtJR(const T* params, Mat<T>& jtj, std::vector<T>& jtr) {
    updateState(params);
    const int ap = actualParameters;
    jtj.resizeAndSetZero(ap, ap);
    jtr.assign(ap, T(0));
    double error = 0.0;
    for (size_t b = 0; b < errorFunctions.size(); ++b) {
      const int bs = padToSimdAlignment(getJacobianBlockSize(b));
      if (bs == 0) continue;
      tJacobian.resizeAndSetZero(bs, numParameters);
      tResidual.assign(bs, T(0));
      int rows = 0;
      error += computeJacobianBlock(params, b, tJacobian, 0, tResidual.data(), rows);
      if (rows == 0) continue;
      // lower triangle (selfadjointView<Lower>().rankUpdate) as a sequence of rank-1 updates over a
      // transposed copy of the block: every (i,j) still sums its products in row order k = 0..rows-1,
      // but the inner loop runs over contiguous memory like Eigen's kernels do (SIMD-friendly baseline).
      jt_.assign(size_t(rows) * ap, T(0));
      for (int c = 0; c < ap; ++c) for (int k = 0; k < rows; ++k) jt_[size_t(k) * ap + c] = tJacobian(k, c);
      for (int k = 0; k < rows; ++k) {
        const T* row = &jt_[size_t(k) * ap];
        const T rk = tResidual[k];
        for (int j = 0; j < ap; ++j) {
          const T t = row[j];
          if (t == T(0)) { continue; }
          T* hcol = &jtj.a[size_t(j) * ap];
          for (int i = j; i < ap; ++i) hcol[i] += row[i] * t;
          jtr[j] += t * rk;
        }
      }
    }
    return error;
  }
  // skeleton_solver_function.cpp:153-159
  void updateParameters(std::vector<T>& params, const std::vector<T>& delta) const {
    for (int i = 0; i < numParameters; ++i) params[i] -= delta[i];
  }
};

// Eigen: LLT<MatrixX<T>, Lower>::compute + solve, restated with Eigen's own structure
// (Eigen/src/Cholesky/LLT.h llt_inplace<Lower>::unblocked / ::blocked): left-looking unblocked
// factorisation for n < 32, otherwise right-looking at block granularity with
// blockSize = clamp((n/8)/16*16, 8, 128). A non-positive pivot makes Eigen return early
// (info = NumericalIssue) with the remaining columns left as they are; GaussNewtonSolverT ignores
// info() (gauss_newton_solver.cpp:251) and still runs the two triangular solves on the lower
// triangle — restated here because the reference's float IK tests rely on it (e.g. a zero Jacobian
// column with regularization 1e-7, inverse_kinematics_test.cpp:115-122).
template <class T>
int lltUnblocked(Mat<T>& A, int o, int size) { // block A[o:o+size, o:o+size]
  for (int k = 0; k < size; ++k) {
    T x = A(o + k, o + k);
    for (int j = 0; j < k; ++j) x -= A(o + k, o + j) * A(o + k, o + j);
    if (!(x > T(0))) return k;
    x = std::sqrt(x);
    A(o + k, o + k) = x;
    for (int i = k + 1; i < size; ++i) {
      T s = A(o + i, o + k);
      for (int j = 0; j < k; ++j) s -= A(o + i, o + j) * A(o + k, o + j);
      A(o + i, o + k) = s / x;
    }
  }
  return -1;
}
template <class T>
int lltBlocked(Mat<T>& A, int n) {
  if (n < 32) return lltUnblocked(A, 0, n);
  int blockSize = n / 8;
  blockSize = (blockSize / 16) * 16;
  blockSize = std::min(std::max(blockSize, 8), 128);
  for (int k = 0; k < n; k += blockSize) {
    const int bs = std::min(blockSize, n - k);
    const int rs = n - k - bs;
    const int ret = lltUnblocked(A, k, bs);
    if (ret >= 0) return k + ret;
    // A21 = A21 * L11^-T
    for (int i = k + bs; i < n; ++i)
      for (int c = 0; c < bs; ++c) {
        T s = A(i, k + c);
        for (int j = 0; j < c; ++j) s -= A(i, k + j) * A(k + c, k + j);
        A(i, k + c) = s / A(k + c, k + c);
      }
    // A22 -= A21 A21^T (lower)
    for (int j = k + bs; j < n; ++j)
      for (int i = j; i < n; ++i) {
        T s = 0;
        for (int c = 0; c < bs; ++c) s += A(i, k + c) * A(j, k + c);
        A(i, j) -= s;
      }
    (void)rs;
  }
  return -1;
}
#ifdef ORACLE_FAST
// TIMING BUILD ONLY (liboracle_native.so, bench.py's CPU arm): the same blocked LLT on a row-major copy of the lower triangle, so
// that every inner loop is a contiguous dot product / axpy the compiler vectorises (built with -march=native and reassociation
// allowed, like Eigen's vectorised kernels). The checker build keeps the strictly ordered column-major restatement above.
template <class T>
bool choleskySolveLowerFast(Mat<T>& A, int n, std::vector<T>& b) {
  std::vector<T> R(size_t(n) * n);
  for (int i = 0; i < n; ++i) for (int j = 0; j <= i; ++j) R[size_t(i) * n + j] = A(i, j);
  auto row = [&](int i) { return R.data() + size_t(i) * n; };
  int blockSize = n < 32 ? n : std::min(std::max((n / 8 / 16) * 16, 8), 128);
  bool ok = true;
  for (int k = 0; k < n && ok; k += blockSize) {
    const int bs = std::min(blockSize, n - k);
    for (int c = k; c < k + bs; ++c) { // diagonal block + panel, left-looking inside the block (columns k..c-1)
      T* rc = row(c);
      T x = rc[c];
      for (int j = k; j < c; ++j) x -= rc[j] * rc[j];
      if (!(x > T(0))) { ok = false; break; }
      x = std::sqrt(x);
      rc[c] = x;
      const T inv = T(1) / x;
      for (int i = c + 1; i < n; ++i) {
        T* ri = row(i);
        T s = ri[c];
        for (int j = k; j < c; ++j) s -= ri[j] * rc[j];
        ri[c] = s * inv;
      }
    }
    if (!ok) break;
    for (int i = k + bs; i < n; ++i) { // trailing update, lower part
      T* ri = row(i);
      for (int j = k + bs; j <= i; ++j) {
        const T* rj = row(j);
        T s = 0;
        for (int c = k; c < k + bs; ++c) s += ri[c] * rj[c];
        ri[j] -= s;
      }
    }
  }
  for (int i = 0; i < n; ++i) { // L y = b
    const T* ri = row(i);
    T s = b[i];
    for (int k = 0; k < i; ++k) s -= ri[k] * b[k];
    b[i] = s / ri[i];
  }
  for (int i = n - 1; i >= 0; --i) { // L^T x = y, column-oriented: row i of L is contiguous
    const T* ri = row(i);
    const T x = b[i] / ri[i];
    b[i] = x;
    for (int k = 0; k < i; ++k) b[k] -= ri[k] * x;
  }
  for (int i = 0; i < n; ++i) for (int j = 0; j <= i; ++j) A(i, j) = R[size_t(i) * n + j];
  return ok;
}
#endif
template <class T>
bool choleskySolveLower(Mat<T>& A, int n, std::vector<T>& b) { // A overwritten by L (lower), b by solution
#ifdef ORACLE_FAST
  return choleskySolveLowerFast(A, n, b);
#endif
  const bool ok = lltBlocked(A, n) < 0;
  for (int i = 0; i < n; ++i) { // L y = b
    T s = b[i];
    for (int k = 0; k < i; ++k) s -= A(i, k) * b[k];
    b[i] = s / A(i, i);
  }
  for (int i = n - 1; i >= 0; --i) { // L^T x = y
    T s = b[i];
    for (int k = i + 1; k < n; ++k) s -= A(k, i) * b[k];
    b[i] = s / A(i, i);
  }
  return ok;
}

// ----------------------------------------------------------------------------------------------
// solver/solver.h:19-34 + gauss_newton_solver.h:17-59 options
// ----------------------------------------------------------------------------------------------
struct GaussNewtonOptions {
  size_t minIterations{1}, maxIterations{2};
  float threshold{1.0f};
  float regularization{0.05f};
  bool doLineSearch{false};
  bool useBlockJtJ{false};
  bool subsetSolver{false}; // SubsetGaussNewtonSolverT semantics (line search c1=1e-4 w/ gradient)
  bool qrSolver{false};     // GaussNewtonSolverQRT: the step from an online Householder QR of [sqrt(lambda) I; J] (gauss_newton_solver_qr.cpp:50-150)
  bool trustRegionQr{false}; // TrustRegionQRT (trust_region_qr.cpp:52-270): QR of J, Newton search for the damping that keeps the step inside the radius
  float trustRegionRadius{1.0f}; // TrustRegionQROptions::trustRegionRadius_ (trust_region_qr.h:23)
};

// math/online_householder_qr.cpp:20-243 — OnlineHouseholderQR<T>: R starts as lambda * I (the caller passes sqrt of the damping), every
// add() sweeps one Householder reflector per column over the stacked [R; A], leaving R upper triangular with R^T R = lambda^2 I + sum A^T A
// and y = Q^T b. v_1 = 1 is implicit, the reflector tail overwrites A's column (computeHouseholderVec, Golub & van Loan alg. 5.1.1).
template <class T>
struct OnlineHouseholderQR {
  int n{0};
  std::vector<T> R; // n x n, R(i, j) at R[i * n + j]
  std::vector<T> y;
  void reset(int n_, T lambda) { // :133-144
    n = n_;
    R.assign(size_t(n) * n, T(0));
    if (lambda != T(0)) for (int i = 0; i < n; ++i) R[size_t(i) * n + i] = lambda;
    y.assign(n, T(0));
  }
  // A: rows x n, column c at A + c * lda (rows contiguous); b: rows. Both are overwritten (addMutating :171-221).
  void addMutating(T* A, int lda, int rows, T* b) {
    for (int iCol = 0; iCol < n; ++iCol) {
      T* col = A + size_t(iCol) * lda;
      T sigma = 0; // computeHouseholderVec :97-118
      for (int k = 0; k < rows; ++k) sigma += col[k] * col[k];
      if (sigma == T(0)) continue; // beta == 0: nothing below R(iCol, iCol)
      const T x1 = R[size_t(iCol) * n + iCol];
      const T mu = std::sqrt(x1 * x1 + sigma);
      const T v1 = (x1 <= T(0)) ? (x1 - mu) : (-sigma / (x1 + mu));
      const T beta = T(2) * v1 * v1 / (sigma + v1 * v1);
      for (int k = 0; k < rows; ++k) col[k] /= v1;
      R[size_t(iCol) * n + iCol] = mu;
      for (int jCol = iCol + 1; jCol <= n; ++jCol) { // applyHouseholderTransformation :30-46 on the remaining columns, then on (y, b)
        T* y2 = jCol < n ? A + size_t(jCol) * lda : b;
        T& y1 = jCol < n ? R[size_t(iCol) * n + jCol] : y[iCol];
        T dot = 0;
        for (int k = 0; k < rows; ++k) dot += col[k] * y2[k];
        const T scalar = (y1 + dot) * beta;
        y1 -= scalar;
        for (int k = 0; k < rows; ++k) y2[k] -= scalar * col[k];
      }
    }
  }
  std::vector<T> result() const { // R.triangularView<Upper>().solve(y); a zero pivot with a zero right-hand side gives 0 (:235-243)
    std::vector<T> x(y);
    for (int i = n - 1; i >= 0; --i) {
      T s = x[i];
      for (int k = i + 1; k < n; ++k) s -= R[size_t(i) * n + k] * x[k];
      const T d = R[size_t(i) * n + i];
      x[i] = (d == T(0) && s == T(0)) ? T(0) : s / d;
    }
    return x;
  }
  std::vector<T> AtTimesB() const { // R^T y (:224-232)
    std::vector<T> g(n, T(0));
    for (int i = 0; i < n; ++i)
      for (int j = i; j < n; ++j) g[j] += R[size_t(i) * n + j] * y[i];
    return g;
  }
};

// solver/solver.cpp:50-128 + gauss_newton_solver.cpp:49-313 (+ subset_gauss_newton_solver.cpp:72-145)
template <class T>
struct GaussNewtonSolver {
  GaussNewtonOptions opt;
  SkeletonSolverFunction<T>* fn;
  std::vector<uint8_t> activeParameters;
  std::vector<int> enabled;
  std::vector<T> parameters;
  std::vector<double> errorHistory;
  double error{0}, lastError{0};
  size_t iteration{0};
  Mat<T> hessian, jacobian;
  std::vector<T> jtr, residual, jt_;

  GaussNewtonSolver(const GaussNewtonOptions& o, SkeletonSolverFunction<T>* f) : opt(o), fn(f) {
    activeParameters.assign(f->numParameters, 1); // solver.cpp:27 activeParameters_.flip()
  }
  void setEnabledParameters(const std::vector<uint8_t>& ps) { // solver.cpp:41-48
    activeParameters = ps;
    fn->setEnabledParameters(ps);
  }
  // character_solver/gauss_newton_solver_qr.cpp:50-150
  void doIterationQR() {
    const int n = fn->numParameters;
    const int ns = int(enabled.size());
    if (ns == 0) return;
    fn->updateState(parameters.data()); // initializeJacobianComputation
    OnlineHouseholderQR<T> qr;
    qr.reset(ns, std::sqrt(T(opt.regularization))); // "the QR solver wants the square root of that lambda" (:74-76)
    double errorOrig = 0.0;
    Mat<T> jac;
    std::vector<T> res;
    for (size_t b = 0; b < fn->getJacobianBlockCount(); ++b) {
      const int bs = fn->getJacobianBlockSize(b);
      if (bs == 0) continue;
      const int rows = padToSimdAlignment(bs);
      jac.resizeAndSetZero(rows, n);
      res.assign(rows, T(0));
      int used = 0;
      errorOrig += fn->computeJacobianBlock(parameters.data(), b, jac, 0, res.data(), used);
      if (used == 0) continue;
      std::vector<T> A(size_t(used) * ns); // ColumnIndexedMatrix(jacobian.topRows(used), enabledParameters)
      for (int a = 0; a < ns; ++a) for (int k = 0; k < used; ++k) A[size_t(a) * used + k] = jac(k, enabled[a]);
      qr.addMutating(A.data(), used, used, res.data());
    }
    error = errorOrig;
    const std::vector<T> sub = qr.result();
    std::vector<T> dir(n, T(0));
    for (int a = 0; a < ns; ++a) dir[enabled[a]] = sub[a];
    if (!opt.doLineSearch) { fn->updateParameters(parameters, dir); return; }
    const std::vector<T> atb = qr.AtTimesB();
    T dotp = 0;
    for (int a = 0; a < ns; ++a) dotp += atb[a] * sub[a];
    const double innerProd = -double(dotp);
    const std::vector<T> orig = parameters;
    float alpha = 1.0f;
    for (size_t k = 0; k < 10 && std::fpclassify(alpha) == FP_NORMAL; ++k) { // :124-143
      parameters = orig;
      std::vector<T> d(n);
      for (int q = 0; q < n; ++q) d[q] = alpha * dir[q];
      fn->updateParameters(parameters, d);
      const double errorNew = fn->getError(parameters.data());
      if ((errorOrig - errorNew) >= 1e-4f * alpha * -innerProd) break;
      alpha *= 0.5f;
    }
  }
  // character_solver/trust_region_qr.cpp:52-270. Arithmetic in T except where the reference mixes in the double error_.
  T curTrustRegionRadius{1}, maxTrustRegionRadius{10}; // trust_region_qr.h:73-74; initializeSolver (:38-40) resets the current radius
  void doIterationTrustRegionQR() {
    const int n = fn->numParameters;
    const int ns = int(enabled.size());
    fn->updateState(parameters.data()); // :57-60 skeletonState_.set(...)
    T lambda = T(1e-10); // :81-82 "a tiny lambda just to make sure we don't divide by zero"
    OnlineHouseholderQR<T> qr;
    qr.reset(ns, lambda);
    double errorOrig = 0.0;
    Mat<T> jac;
    std::vector<T> res;
    for (size_t b = 0; b < fn->getJacobianBlockCount(); ++b) { // :86-110, one block per error function with weight > 0
      const int bs = fn->getJacobianBlockSize(b);
      if (bs == 0) continue;
      const int rows = padToSimdAlignment(bs);
      jac.resizeAndSetZero(rows, n);
      res.assign(rows, T(0));
      int used = 0;
      errorOrig += fn->computeJacobianBlock(parameters.data(), b, jac, 0, res.data(), used);
      if (used == 0) continue;
      std::vector<T> A(size_t(used) * ns);
      for (int a = 0; a < ns; ++a) for (int k = 0; k < used; ++k) A[size_t(a) * used + k] = jac(k, enabled[a]);
      qr.addMutating(A.data(), used, used, res.data());
    }
    error = errorOrig;
    std::vector<T> grad = qr.AtTimesB(); // :116 gradientSub_ = 2 * At_times_b()
    for (T& v : grad) v *= T(2);
    const std::vector<T> Rsaved = qr.R; // :119
    auto dotT = [&](const std::vector<T>& a, const std::vector<T>& b) { T s = 0; for (int i = 0; i < ns; ++i) s += a[i] * b[i]; return s; };
    auto evalQuadraticModel = [&](const std::vector<T>& p) { // :133-140
      T result = T(error);
      result -= dotT(grad, p);
      T sq = 0;
      for (int i = 0; i < ns; ++i) { T r = 0; for (int j = i; j < ns; ++j) r += Rsaved[size_t(i) * ns + j] * p[j]; sq += r * r; }
      result += sq;
      return result;
    };
    auto solveUpper = [&](const std::vector<T>& R, std::vector<T> b) { // R x = b
      for (int i = ns - 1; i >= 0; --i) { T s = b[i]; for (int k = i + 1; k < ns; ++k) s -= R[size_t(i) * ns + k] * b[k]; b[i] = s / R[size_t(i) * ns + i]; }
      return b;
    };
    auto solveUpperTransposed = [&](const std::vector<T>& R, std::vector<T> b) { // R^T x = b
      for (int i = 0; i < ns; ++i) { T s = b[i]; for (int k = 0; k < i; ++k) s -= R[size_t(k) * ns + i] * b[k]; b[i] = s / R[size_t(i) * ns + i]; }
      return b;
    };
    const T nu = 0; // :153
    for (size_t iTrustStep = 0; iTrustStep < 10; ++iTrustStep) {
      std::vector<T> dir = qr.result();
      if (double(dotT(dir, grad)) < double(std::numeric_limits<float>::epsilon() * (T(1.0) + error))) break; // :162-164 (FLT_EPSILON * (T(1) + double error_))
      for (size_t iIter = 0; iIter < 3; ++iIter) { // :180-236 Newton iteration on lambda (Nocedal & Wright 4.3), lambda only grows
        if (std::sqrt(dotT(dir, dir)) < T(1.05) * curTrustRegionRadius) break;
        std::vector<T> mhg(ns);
        for (int i = 0; i < ns; ++i) mhg[i] = -T(0.5) * grad[i];
        const std::vector<T> pl = solveUpper(qr.R, solveUpperTransposed(qr.R, mhg));
        const std::vector<T> ql = solveUpperTransposed(qr.R, pl);
        const T pl2 = dotT(pl, pl), ql2 = dotT(ql, ql);
        if (ql2 < std::numeric_limits<float>::epsilon()) break;
        const T plNorm = std::sqrt(pl2);
        const T deltaLambda = (pl2 / ql2) * ((plNorm - curTrustRegionRadius) / curTrustRegionRadius);
        if (deltaLambda <= 0) break;
        const T lambdaNew = lambda + deltaLambda;
        const T yv = std::sqrt(lambdaNew - lambda);
        std::vector<T> D(size_t(ns) * ns, T(0)), zero(ns, T(0)); // :214-222 lambdaDiag_ = y I as ns extra rows, right-hand side 0
        for (int i = 0; i < ns; ++i) D[size_t(i) * ns + i] = yv;
        qr.addMutating(D.data(), ns, ns, zero.data());
        lambda = lambdaNew;
        dir = qr.result();
      }
      const std::vector<T> orig = parameters;
      std::vector<T> full(n, T(0)); // subsetToFullVector :142-150
      for (int a = 0; a < ns; ++a) full[enabled[a]] = dir[a];
      fn->updateParameters(parameters, full);
      const double errorNew = fn->getError(parameters.data());
      const T model = evalQuadraticModel(dir);
      const T rho = T((error - errorNew) / (error - double(model))); // :249 (double - double) / (double - T)
      if (rho < T(0.25)) curTrustRegionRadius = T(0.25) * curTrustRegionRadius;
      else if (rho > T(0.75) && lambda > 0) curTrustRegionRadius = std::min(T(2) * curTrustRegionRadius, maxTrustRegionRadius);
      if (rho > nu) break;
      parameters = orig; // reject the step, the radius has shrunk: try again
    }
  }
  void doIteration() { // gauss_newton_solver.cpp:224-280
    if (opt.trustRegionQr) { doIterationTrustRegionQR(); return; }
    if (opt.qrSolver) { doIterationQR(); return; }
    const int n = fn->numParameters;
    const int ns = int(enabled.size());
    if (opt.useBlockJtJ && !opt.subsetSolver) { // :69-107
      error = fn->getJtJR(parameters.data(), hessian, jtr);
      Mat<T> h2;
      h2.resizeAndSetZero(ns, ns);
      std::vector<T> g2(ns);
      for (int a = 0; a < ns; ++a) {
        g2[a] = jtr[enabled[a]];
        for (int b = 0; b <= a; ++b) h2(a, b) = hessian(enabled[a], enabled[b]);
      }
      hessian = h2;
      jtr = g2;
    } else { // :110-221 (single chunk) / subset_gauss_newton_solver.cpp:76-105
      int rows = 0;
      error = fn->getJacobian(parameters.data(), jacobian, residual, rows);
      hessian.resizeAndSetZero(ns, ns);
      jtr.assign(ns, T(0));
      jt_.assign(size_t(rows) * ns, T(0)); // transposed, column-compacted copy (see getJtJR)
      for (int a = 0; a < ns; ++a) for (int k = 0; k < rows; ++k) jt_[size_t(k) * ns + a] = jacobian(k, enabled[a]);
      for (int k = 0; k < rows; ++k) {
        const T* row = &jt_[size_t(k) * ns];
        const T rk = residual[k];
        for (int b = 0; b < ns; ++b) {
          const T t = row[b];
          if (t == T(0)) { continue; }
          T* hcol = &hessian.a[size_t(b) * ns];
          for (int a = b; a < ns; ++a) hcol[a] += row[a] * t;
          jtr[b] += t * rk;
        }
      }
    }
    const std::vector<T> gradSubset = jtr;
    for (int a = 0; a < ns; ++a) hessian(a, a) += T(opt.regularization); // :248
    choleskySolveLower(hessian, ns, jtr); // :251
    std::vector<T> delta(n, T(0));
    for (int a = 0; a < ns; ++a) delta[enabled[a]] = jtr[a]; // :254-257
    if (!opt.doLineSearch) { fn->updateParameters(parameters, delta); return; }
    const std::vector<T> orig = parameters;
    if (!opt.subsetSolver) { // gauss_newton_solver.cpp:292-312
      const T scaledError = T(1e-3) * T(error);
      T scale = 1;
      for (size_t i = 0; i < 10 && std::isnormal(scale); ++i) {
        parameters = orig;
        std::vector<T> d(n);
        for (int k = 0; k < n; ++k) d[k] = scale * delta[k];
        fn->updateParameters(parameters, d);
        const double errorNew = fn->getError(parameters.data());
        if ((error - errorNew) >= scale * scaledError) break;
        scale *= T(0.5);
      }
    } else { // subset_gauss_newton_solver.cpp:119-141
      double innerProd = 0;
      for (int a = 0; a < ns; ++a) innerProd -= double(gradSubset[a] * jtr[a]);
      float alpha = 1.0f;
      for (size_t k = 0; k < 10 && std::fpclassify(alpha) == FP_NORMAL; ++k) {
        parameters = orig;
        std::vector<T> d(n);
        for (int q = 0; q < n; ++q) d[q] = alpha * delta[q];
        fn->updateParameters(parameters, d);
        const double errorNew = fn->getError(parameters.data());
        if ((error - errorNew) >= 1e-4f * alpha * -innerProd) break;
        alpha *= 0.5f;
      }
    }
  }
  double solve(std::vector<T>& params) { // solver.cpp:50-128
    if (int(params.size()) != fn->numParameters) throw std::runtime_error("params size mismatch");
    errorHistory.clear();
    parameters = params;
    error = lastError = std::numeric_limits<double>::max();
    curTrustRegionRadius = T(opt.trustRegionRadius); // TrustRegionQRT::initializeSolver (trust_region_qr.cpp:38-40)
    enabled.clear(); // gauss_newton_solver.cpp:57-66
    for (int i = 0; i < fn->numParameters; ++i) if (activeParameters[i]) enabled.push_back(i);
    for (iteration = 0; iteration < opt.maxIterations; ++iteration) {
      doIteration();
      errorHistory.push_back(error);
      bool converged = false;
      if (std::fabs(lastError - error) / (std::fabs(error) + std::numeric_limits<float>::min()) <=
          opt.threshold * std::numeric_limits<float>::epsilon())
        converged = true;
      if (iteration >= opt.minIterations && converged) break;
      lastError = error;
    }
    params = parameters;
    return error;
  }
};

} // namespace oracle
