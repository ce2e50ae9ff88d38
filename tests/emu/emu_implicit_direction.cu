// TEST HARNESS ONLY — CPU lane-emulation of implicitDirectionKernel (mb2_solver_function_implicit_direction_device), part of
// tests/emu/libmb2_emu.so.
//
// The __host__ __device__ building blocks of ik_jacobi.cuh run pass by pass in the kernel's order, the lanes of each pass in sequence,
// on any rows x n_E float32 matrix. It also reports the sweeps the Jacobi iteration used. It is not part of the product library and
// nothing in momentum_b200/ loads it.
#include <cmath>
#include <cstdint>
#include <vector>

#include "../../momentum_b200/csrc/ik_jacobi.cuh"

using namespace mb2;

// jt: the matrix K-major, column i (enabled parameter i) at jt + i * rows; residual [rows]; g [nE] ->
// v [nE], jv [rows], *rms, *sweeps (host memory). Returns 0.
extern "C" int emu_implicit_direction(int32_t rows, int32_t nE, const float* jt, const float* residual, const float* gIn, double* v, double* jv,
                                      double* rms, int32_t* sweepsOut) {
  const int ld = rows;
  std::vector<int32_t> E(static_cast<size_t>(nE));
  for (int i = 0; i < nE; ++i) E[i] = i;
  const bool rowsSide = rows <= nE;
  const int k = rowsSide ? rows : nE, h = jacobiPairs(k), steps = jacobiSteps(k);
  std::vector<double> K(jacobiPackedSize(k)), y(static_cast<size_t>(k)), g(static_cast<size_t>(nE)), vE(static_cast<size_t>(nE));
  std::vector<double> rc(static_cast<size_t>(h)), rs(static_cast<size_t>(h));
  std::vector<int> rp(static_cast<size_t>(h)), rq(static_cast<size_t>(h));
  std::vector<double> rlog(jacobiLogDoubles(k));
  const int32_t* Ep = E.data();
  for (int i = 0; i < nE; ++i) g[i] = double(gIn[i]);
  for (int i = 0; i < nE; ++i) {
    const double gi = jacobiGradient(jt, ld, Ep, rows, residual, i);
    vE[i] = gi * gi;
  }
  for (int r = 0; r < k; ++r)
    for (int c = r; c < k; ++c) K[jacobiPacked(r, c, k)] = jacobiGram(jt, ld, Ep, nE, rows, rowsSide, r, c);
  for (int i = 0; i < k; ++i) y[i] = jacobiRhs(jt, ld, Ep, nE, rowsSide, g.data(), i);
  double s2 = 0.0;
  for (int i = 0; i < nE; ++i) s2 += vE[i];
  *rms = nE > 0 ? double(float(std::sqrt(s2 / nE))) : 0.0;
  double d = 0.0;
  for (int i = 0; i < k; ++i) d = std::fmax(d, K[jacobiPacked(i, i, k)]);
  const double floor = jacobiFloor(d);
  int sweeps = 0;
  while (k > 1 && sweeps < kJacobiMaxSweeps) {
    bool rotated = false;
    for (int st = 0; st < steps; ++st) {
      double* lg = rlog.data() + (size_t(sweeps) * steps + st) * h * 2;
      for (int t = 0; t < h; ++t) {
        int p, q;
        jacobiPair(k, st, t, p, q);
        double c = 1.0, s = 0.0, tt = 0.0;
        if (q >= 0 && jacobiRotation(K[jacobiPacked(p, p, k)], K[jacobiPacked(q, q, k)], K[jacobiPacked(p, q, k)], floor, c, s, tt)) {
          jacobiRotateDiagonal(K.data(), k, p, q, tt);
          jacobiRotateTransposed(y.data(), p, q, c, s);
          rotated = true;
        }
        rp[t] = p; rq[t] = q; rc[t] = c; rs[t] = s;
        lg[2 * t] = c; lg[2 * t + 1] = s;
      }
      const int blocks = h * (h - 1) / 2;
      for (int L = 0; L < blocks; ++L) {
        int i, j;
        jacobiBlock(L, i, j);
        if (rs[i] == 0.0 && rs[j] == 0.0) continue;
        jacobiRotateBlock(K.data(), k, rp[i], rq[i], rc[i], rs[i], rp[j], rq[j], rc[j], rs[j]);
      }
    }
    if (!rotated) break;
    ++sweeps;
  }
  for (int i = 0; i < k; ++i) y[i] = jacobiScale(K[jacobiPacked(i, i, k)], y[i], rowsSide);
  for (int st = sweeps * steps - 1; st >= 0; --st) {
    const double* lg = rlog.data() + size_t(st) * h * 2;
    for (int t = 0; t < h; ++t) {
      if (lg[2 * t + 1] == 0.0) continue;
      int p, q;
      jacobiPair(k, st % steps, t, p, q);
      jacobiRotateForward(y.data(), p, q, lg[2 * t], lg[2 * t + 1]);
    }
  }
  for (int i = 0; i < nE; ++i) vE[i] = jacobiDirection(jt, ld, Ep, rows, rowsSide, y.data(), i);
  for (int i = 0; i < nE; ++i) v[i] = double(float(vE[i]));
  for (int r = 0; r < rows; ++r) jv[r] = double(float(jacobiJv(jt, ld, Ep, nE, vE.data(), r)));
  *sweepsOut = sweeps;
  return 0;
}
