// Building blocks of the implicit-function direction of solve_ik's backward (implicitDirectionKernel, ik_kernels.cu): the reference's
// hessianInverseTimes (diff_ik/fully_differentiable_body_ik.cpp:74-109),
//   v = (2 J_E^T J_E)^+ g = 1/2 V diag(s^-2 if s^2 >= tau, else 0) V^T g,   J_E = U S V^T,  tau = 1e-5,
// through the eigen-decomposition of the Gram matrix on the smaller side of J_E (rows x n_E), k = min(rows, n_E):
//   rows <= n_E:  K = J_E J_E^T (k = rows), y = J_E g,  v_E = 1/2 J_E^T Q Lambda^-2 Q^T y
//   otherwise:    K = J_E^T J_E (k = n_E),  y = g,      v_E = 1/2 Q Lambda^-1 Q^T y
// with K = Q Lambda Q^T (Lambda = the s^2) and every lambda < tau truncated to 0. K is float64: a product of two float32 Jacobian
// entries is exact there, the sums run in a fixed order.
//
// The eigen-solve is the cyclic parallel Jacobi method with round-robin ordering: a step applies k/2 disjoint rotations (a dummy index
// pads an odd k), a sweep is k - 1 steps and visits every pair once. Once a step's rotations are known, every 2 x 2 block of K transforms
// independently as R_i^T B_ij R_j, so a step is two barrier-separated phases: the rotations (and the diagonal blocks), then the
// off-diagonal blocks of the packed upper triangle. Q is never formed: Q^T y is rotated as the rotations are made, and each step's
// rotations go to a log that is replayed backwards once to apply Q. Every function here is __host__ __device__ so that the CPU
// emulator (tests/emu/emu_implicit_direction.cu) runs the same arithmetic lane by lane.
#pragma once

#include <cmath>
#include <cstddef>
#include <cstdint>

#include "ik_types.h"

namespace mb2 {

constexpr double kJacobiTau = 1e-5;                   // s^2 below this is truncated (fully_differentiable_body_ik.cpp:95)
constexpr double kJacobiEps = 2.220446049250313e-16;  // float64 machine epsilon (jacobiRotation's skip test)
constexpr int kJacobiMaxSweeps = 32;                  // the rotation log is sized for this many sweeps (the test fixtures take 5 to 17)

// index slots of the round-robin ordering (k rounded up to even), rotations per step, steps per sweep
MB2_HD int jacobiSlots(int k) { return k + (k & 1); }
MB2_HD int jacobiPairs(int k) { return jacobiSlots(k) / 2; }
MB2_HD int jacobiSteps(int k) { return k > 0 ? jacobiSlots(k) - 1 : 0; }
// doubles of one rotation log: (c, s) for every pair slot of every step of every sweep up to the cap
MB2_HD size_t jacobiLogDoubles(int k) { return size_t(kJacobiMaxSweeps) * size_t(jacobiSteps(k)) * size_t(jacobiPairs(k)) * 2; }
// entries of the packed upper triangle, and the position of (a, b), a <= b (row-major)
MB2_HD size_t jacobiPackedSize(int k) { return size_t(k) * size_t(k + 1) / 2; }
MB2_HD size_t jacobiPacked(int a, int b, int k) { return size_t(a) * size_t(2 * k - a + 1) / 2 + size_t(b - a); }

// pair t of round-robin step `step`: slot 0 stays, slots 1 .. m-1 rotate by one per step; slot t meets slot m-1-t. p < q; q = -1 when
// the partner is the dummy index of an odd k.
MB2_HD void jacobiPair(int k, int step, int t, int& p, int& q) {
  const int m = jacobiSlots(k);
  const int a = t == 0 ? 0 : 1 + (t - 1 + step) % (m - 1);
  const int b = 1 + (m - 2 - t + step) % (m - 1); // slot m-1-t >= 1
  p = a < b ? a : b;
  q = a < b ? b : a;
  if (q >= k) q = -1;
}

// off-diagonal block L (0 <= L < h (h - 1) / 2) of the h pair slots: pair slots i < j, column by column (L = j (j - 1) / 2 + i)
MB2_HD void jacobiBlock(int L, int& i, int& j) {
  int c = int((1.0 + sqrt(1.0 + 8.0 * double(L))) * 0.5);
  while (c * (c - 1) / 2 > L) --c;
  while ((c + 1) * c / 2 <= L) ++c;
  j = c;
  i = L - c * (c - 1) / 2;
}

// The Jacobian J is K-major: column c (model parameter c) at J + c * ld, rows 0 .. rows - 1. E = the enabled parameters.
// K_ab of the smaller side: rows side sum_i J[a][E_i] J[b][E_i], parameter side sum_r J[r][E_a] J[r][E_b]
MB2_HD double jacobiGram(const float* J, int ld, const int32_t* E, int nE, int rows, bool rowsSide, int a, int b) {
  double s = 0.0;
  if (rowsSide) {
    for (int i = 0; i < nE; ++i) {
      const float* col = J + size_t(E[i]) * ld;
      s += double(col[a]) * double(col[b]);
    }
  } else {
    const float* ca = J + size_t(E[a]) * ld;
    const float* cb = J + size_t(E[b]) * ld;
    for (int r = 0; r < rows; ++r) s += double(ca[r]) * double(cb[r]);
  }
  return s;
}
// y_a: rows side (J_E g)_a, parameter side g_a (g over E)
MB2_HD double jacobiRhs(const float* J, int ld, const int32_t* E, int nE, bool rowsSide, const double* g, int a) {
  if (!rowsSide) return g[a];
  double s = 0.0;
  for (int i = 0; i < nE; ++i) s += double(J[size_t(E[i]) * ld + a]) * g[i];
  return s;
}
// (2 J_E^T r)_i, r = the residual column
MB2_HD double jacobiGradient(const float* J, int ld, const int32_t* E, int rows, const float* residual, int i) {
  const float* col = J + size_t(E[i]) * ld;
  double s = 0.0;
  for (int r = 0; r < rows; ++r) s += double(col[r]) * double(residual[r]);
  return 2.0 * s;
}

// The rotation that zeroes K_pq (K' = R^T K R, R_pp = R_qq = c, R_pq = s, R_qp = -s), t = s / c. False (c = 1, s = 0): skipped, K_pq is
// already negligible against the diagonal (all-zero blocks included) or below `floor` = eps max_i K_ii of the Gram matrix as formed, the
// rounding level of its entries: the pairs of (numerically) zero eigenvalues a rank-deficient J_E gives would otherwise trade rounding
// noise forever, and a rotation at that level moves no eigenvalue by more than about eps ||K||, far below tau.
MB2_HD double jacobiFloor(double maxDiagonal) { return kJacobiEps * maxDiagonal; }
MB2_HD bool jacobiRotation(double app, double aqq, double apq, double floor, double& c, double& s, double& t) {
  const double small = kJacobiEps * sqrt(fabs(app * aqq));
  if (!(fabs(apq) > (small > floor ? small : floor))) {
    c = 1.0; s = 0.0; t = 0.0;
    return false;
  }
  const double theta = (aqq - app) / (2.0 * apq);
  const double at = fabs(theta);
  t = at > 1e150 ? 0.5 / theta : (theta >= 0.0 ? 1.0 : -1.0) / (at + sqrt(1.0 + theta * theta));
  c = 1.0 / sqrt(1.0 + t * t);
  s = t * c;
  return true;
}
// the diagonal block of a rotated pair: K_pp -= t K_pq, K_qq += t K_pq, K_pq = 0
MB2_HD void jacobiRotateDiagonal(double* K, int k, int p, int q, double t) {
  double& apq = K[jacobiPacked(p, q, k)];
  K[jacobiPacked(p, p, k)] -= t * apq;
  K[jacobiPacked(q, q, k)] += t * apq;
  apq = 0.0;
}
// the off-diagonal block of pair slots i != j (four distinct indices; an index -1 is the dummy: it reads 0 and is not written):
// B = K[(p_i, q_i), (p_j, q_j)] becomes R_i^T B R_j
MB2_HD void jacobiRotateBlock(double* K, int k, int pi, int qi, double ci, double si, int pj, int qj, double cj, double sj) {
  const int r[2] = {pi, qi}, cidx[2] = {pj, qj};
  double* e[4];
  double b[4];
  for (int u = 0; u < 2; ++u)
    for (int w = 0; w < 2; ++w) {
      const int x = r[u], y = cidx[w];
      e[2 * u + w] = (x < 0 || y < 0) ? nullptr : K + (x <= y ? jacobiPacked(x, y, k) : jacobiPacked(y, x, k));
      b[2 * u + w] = e[2 * u + w] ? *e[2 * u + w] : 0.0;
    }
  // C = B R_j, then R_i^T C
  const double c00 = cj * b[0] - sj * b[1], c01 = sj * b[0] + cj * b[1];
  const double c10 = cj * b[2] - sj * b[3], c11 = sj * b[2] + cj * b[3];
  const double n[4] = {ci * c00 - si * c10, ci * c01 - si * c11, si * c00 + ci * c10, si * c01 + ci * c11};
  for (int u = 0; u < 4; ++u)
    if (e[u]) *e[u] = n[u];
}
// Q^T y as the rotations are made: (y_p, y_q) <- R^T (y_p, y_q); and the replay, (z_p, z_q) <- R (z_p, z_q)
MB2_HD void jacobiRotateTransposed(double* y, int p, int q, double c, double s) {
  const double yp = y[p], yq = y[q];
  y[p] = c * yp - s * yq;
  y[q] = s * yp + c * yq;
}
MB2_HD void jacobiRotateForward(double* z, int p, int q, double c, double s) {
  const double zp = z[p], zq = z[q];
  z[p] = c * zp + s * zq;
  z[q] = -s * zp + c * zq;
}

// (Q^T y)_a scaled by the truncated inverse eigenvalue: Lambda^-2 on the rows side, Lambda^-1 on the parameter side
MB2_HD double jacobiScale(double lambda, double y, bool rowsSide) {
  if (!(lambda >= kJacobiTau)) return 0.0;
  return rowsSide ? y / (lambda * lambda) : y / lambda;
}
// v_i (i over E) from z = Q Lambda^-p Q^T y: rows side 1/2 (J_E^T z)_i, parameter side 1/2 z_i
MB2_HD double jacobiDirection(const float* J, int ld, const int32_t* E, int rows, bool rowsSide, const double* z, int i) {
  if (!rowsSide) return 0.5 * z[i];
  const float* col = J + size_t(E[i]) * ld;
  double s = 0.0;
  for (int r = 0; r < rows; ++r) s += double(col[r]) * z[r];
  return 0.5 * s;
}
// (J_E v_E)_r
MB2_HD double jacobiJv(const float* J, int ld, const int32_t* E, int nE, const double* vE, int r) {
  double s = 0.0;
  for (int i = 0; i < nE; ++i) s += double(J[size_t(E[i]) * ld + r]) * vE[i];
  return s;
}

} // namespace mb2
