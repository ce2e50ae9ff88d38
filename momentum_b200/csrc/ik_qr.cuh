// Alternative linear step: the QR-accurate Gauss-Newton step of GaussNewtonSolverQRT (character_solver/gauss_newton_solver_qr.cpp:50-150,
// the default solver of pymomentum's solve_ik and of the marker tracker) on the device.
//
// One CTA per instance keeps the upper-triangular R (packed, fp32) and y in shared memory, seeded with sqrt(lambda) I, and folds the
// Jacobian in row chunks — one chunk per error-function block like the reference's addMutating per block (:80-106), split further only
// when a block does not fit beside R — by Householder reflectors, column by column (math/online_householder_qr.cpp:171-221):
//     [beta, mu] from (R(i,i), A(:,i));  every remaining column j (and the right-hand side): s = beta (R(i,j) + v . A(:,j)),
//     R(i,j) -= s, A(:,j) -= s v      with v = A(:,i) / v1, v_1 = 1 implicit.
// At step i, thread t takes the columns i + 1 + t, i + 1 + t + 256, ... (and the right-hand side when it falls on one of them): their
// dot products, updates and the squared norms of the updated columns (the next reflectors' sigma). Which thread holds a column moves by
// one at every step, so nothing carries over in a thread: what step i + 1 reads (the norms and the updated chunk columns) was written
// by other threads at step i and is ordered by the ONE block barrier that ends each step. A column that is still structurally
// zero in this chunk with R(i,j) = 0 is skipped (the reference's beta == 0 / exact-zero cases). Then R x = y by one warp, g = R^T y
// (= J^T r, for the line search), theta -= delta and the SolverT bookkeeping through the same tail as the Cholesky kernels.
// R^T R = J^T J + lambda I, so the step equals the Cholesky path's up to rounding — without squaring the condition number.
// (included by ik_kernels.cu: the kernel shares cholFinish, the tail of every linear-step kernel, with the Cholesky kernels)
#pragma once

namespace mb2 {

constexpr int kQrThreads = 256;

__device__ __forceinline__ int qrRowOffset(int i, int n) { return i * n - (i * (i - 1)) / 2 - i; } // R(i, j), j >= i, at offset + j

// R = diag0 I, y = 0, then every row chunk of instance b's Jacobian folded in by Householder reflectors (see the file header). Block-wide.
__device__ void qrFoldJacobian(const QrArgs& a, int b, float* R, float* y, float* norms, float* As, int n, float diag0) {
  const int tid = threadIdx.x;
  for (int idx = tid; idx < n * (n + 1) / 2; idx += kQrThreads) R[idx] = 0.f;
  for (int i = tid; i < n; i += kQrThreads) y[i] = 0.f;
  __syncthreads();
  for (int i = tid; i < n; i += kQrThreads) R[qrRowOffset(i, n) + i] = diag0;
  const float* Jg = a.jacobian + size_t(b) * size_t(a.numCols + 1) * a.ldJ;
  for (int ch = 0; ch < a.numChunks; ++ch) {
    const int r0 = a.chunkStart[ch], p = a.chunkStart[ch + 1] - r0, ps = p | 1;
    __syncthreads();
    // the chunk: columns of the enabled parameters (the compact device columns) + the residual column
    for (int idx = tid; idx < (n + 1) * p; idx += kQrThreads) {
      const int j = idx / p, k = idx - j * p;
      As[j * ps + k] = Jg[size_t(j < n ? j : a.numCols) * a.ldJ + r0 + k];
    }
    __syncthreads();
    for (int j = tid; j <= n; j += kQrThreads) {
      float s = 0.f;
      for (int k = 0; k < p; ++k) s = fmaf(As[j * ps + k], As[j * ps + k], s);
      norms[j] = s;
    }
    __syncthreads();
    for (int i = 0; i < n; ++i) {
      const float sigma = norms[i];
      if (sigma == 0.f) continue; // (uniform) nothing below R(i, i): the reflector is the identity
      const int ro = qrRowOffset(i, n);
      const float x1 = R[ro + i];
      const float mu = sqrtf(x1 * x1 + sigma);
      const float v1 = (x1 <= 0.f) ? (x1 - mu) : (-sigma / (x1 + mu)); // Golub & van Loan 5.1.1, cancellation-free branch
      const float beta = 2.f * v1 * v1 / (sigma + v1 * v1);
      const float inv = 1.f / v1;
      const float* u = As + i * ps; // v = u / v1
      for (int j = i + 1 + tid; j <= n; j += kQrThreads) {
        float* col = As + j * ps;
        float* y1 = j < n ? R + ro + j : y + i;
        const float r = *y1;
        if (norms[j] == 0.f && r == 0.f) continue; // column untouched by this chunk so far and no fill from R
        float dot = 0.f;
        for (int k = 0; k < p; ++k) dot = fmaf(u[k], col[k], dot);
        const float s = (r + dot * inv) * beta;
        *y1 = r - s;
        const float si = s * inv;
        float nn = 0.f;
        for (int k = 0; k < p; ++k) { const float v = fmaf(-si, u[k], col[k]); col[k] = v; nn = fmaf(v, v, nn); }
        norms[j] = nn;
      }
      __syncthreads(); // R(i, i) is read by every thread before thread 0 may replace it below
      if (tid == 0) R[ro + i] = mu;
    }
  }
}
// R x = rhs by one warp (lanes over the row's dot product); a zero pivot with a zero numerator gives 0 like Eigen's triangular solve
// (online_householder_qr.cpp:235-243). x may alias rhs. Call from warp 0 only.
__device__ void qrSolveUpperWarp(const float* R, const float* rhs, float* x, int n, int lane) {
  for (int i = n - 1; i >= 0; --i) {
    const int ro = qrRowOffset(i, n);
    float s = 0.f;
    for (int k = i + 1 + lane; k < n; k += 32) s = fmaf(R[ro + k], x[k], s);
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) { const float num = rhs[i] - s, d = R[ro + i]; x[i] = (d == 0.f && num == 0.f) ? 0.f : num / d; }
    __syncwarp();
  }
}
// R^T x = rhs by one warp. x may alias rhs.
__device__ void qrSolveUpperTransposedWarp(const float* R, const float* rhs, float* x, int n, int lane) {
  for (int i = 0; i < n; ++i) {
    float s = 0.f;
    for (int k = lane; k < i; k += 32) s = fmaf(R[qrRowOffset(k, n) + i], x[k], s);
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) x[i] = (rhs[i] - s) / R[qrRowOffset(i, n) + i];
    __syncwarp();
  }
}

template <bool kUnused>
__global__ void __launch_bounds__(kQrThreads, 1) qrSolveKernel(const QrArgs a) {
  extern __shared__ __align__(16) float qrSmem[];
  const CholArgs& c = a.c;
  const int b = blockIdx.x;
  if (c.state.active[b] == 0) return;
  const int n = c.ns, tid = threadIdx.x, lane = tid & 31;
  float* R = qrSmem;                                  // packed upper triangle, row-major
  float* y = R + (size_t(n) * (n + 1) / 2 + 3 & ~size_t(3));
  float* x = y + ((n + 3) & ~3);
  float* g = x + ((n + 3) & ~3);
  float* norms = g + ((n + 3) & ~3);                  // [n + 1] squared norms of the chunk's columns (column n = right-hand side)
  float* As = norms + ((n + 4) & ~3);                 // [n + 1][ps] the chunk, column-major, odd stride
  const float sqrtLambda = sqrtf(c.regularization);   // "the QR solver wants the square root of that lambda" (:74-76)
  qrFoldJacobian(a, b, R, y, norms, As, n, sqrtLambda);
  __syncthreads();
  if (tid < 32) qrSolveUpperWarp(R, y, x, n, lane); // R x = y
  // g = R^T y = J^T r (At_times_b, :224-232)
  for (int j = tid; j < n; j += kQrThreads) {
    float s = 0.f;
    for (int i = 0; i <= j; ++i) s = fmaf(R[qrRowOffset(i, n) + j], y[i], s);
    g[j] = s;
  }
  __syncthreads();
  cholFinish(c, b, n, x, g, false);
}

cudaError_t launchQrSolve(const QrArgs& a, int maxChunkRows, cudaStream_t stream) {
  const size_t smem = qrSmemFloats(a.c.ns, maxChunkRows) * sizeof(float);
  cudaError_t e = cudaFuncSetAttribute(qrSolveKernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem));
  if (e != cudaSuccess) return e;
  qrSolveKernel<false><<<a.c.batch, kQrThreads, smem, stream>>>(a);
  return cudaGetLastError();
}

} // namespace mb2
