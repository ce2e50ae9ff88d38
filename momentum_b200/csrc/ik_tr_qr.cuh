// TrustRegionQRT on the device (character_solver/trust_region_qr.cpp:52-270; selectable in pymomentum's solve_ik,
// tensor_ik.cpp:149-152): one CTA per instance runs a whole doIteration().
//
//   1. Householder QR of the Jacobian with a 1e-10 diagonal (:81-110) - qrFoldJacobian of ik_qr.cuh -, g = 2 R^T y (:116), R saved (:119)
//   2. up to ten trust steps (:155-267): x = R^-1 y; stop when g.x is below FLT_EPSILON (1 + error); up to three Newton iterations on the
//      damping (Nocedal & Wright 4.3, :180-236): p = R^-1 R^-T (-g / 2), q = R^-T p, dlambda = |p|^2 / |q|^2 (|p| - radius) / radius, then
//      sqrt(dlambda) I is folded into R as n extra rows (addMutating of a diagonal matrix, :214-222) and x recomputed
//   3. the trial parameters theta - x, their error by the FK sweep + residuals INSIDE the kernel (getError rounds through float like
//      skeleton_solver_function.cpp:82), the quadratic model error - g.x + |R_saved x|^2 (:133-140), rho (:249), the radius update
//      (:258-264); rho > 0 accepts the step, otherwise the parameters are kept and the next trust step runs with the smaller radius
// The current radius is per-instance solver state (initializeSolver :38-40 resets it at the start of a solve).
//
// Shared memory: R and D (the rows being folded in), both packed upper triangles; D shares its storage with the Jacobian chunk of step 1.
// n = 220 (humanoid72) needs 208 KB; larger systems are refused by the launcher.
// (included by ik_kernels.cu after ik_qr.cuh)
#pragma once

namespace mb2 {

__device__ __forceinline__ float trBlockSum(float v, float* red) { // every thread gets the total, summed in a fixed order
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads(); // (red may still be read from the previous call)
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float s = 0.f;
  for (int w = 0; w < kQrThreads / 32; ++w) s += red[w];
  return s;
}
__device__ __forceinline__ float trDot(const float* a, const float* b, int n, float* red) {
  float s = 0.f;
  for (int i = threadIdx.x; i < n; i += kQrThreads) s = fmaf(a[i], b[i], s);
  return trBlockSum(s, red);
}

// [R; D] -> R with D = diag I (n extra rows, right-hand side 0): OnlineHouseholderQR::addMutating on a diagonal matrix. Column i of D is
// non-zero in rows 0..i only (fill from the earlier reflectors), so D stays upper triangular and is stored packed like R. Thread j owns
// column j; the reflector of a step is read by everyone from column i of D (a broadcast read).
__device__ void trFoldDiagonal(float* R, float* y, float* D, float* dvec, float* scal, int n, float diag) {
  const int tid = threadIdx.x;
  for (int idx = tid; idx < n * (n + 1) / 2; idx += kQrThreads) D[idx] = 0.f;
  for (int i = tid; i < n; i += kQrThreads) dvec[i] = 0.f;
  __syncthreads();
  for (int i = tid; i < n; i += kQrThreads) D[qrRowOffset(i, n) + i] = diag;
  __syncthreads();
  for (int i = 0; i < n; ++i) {
    if (tid == (i % kQrThreads)) { // the owner of column i: sigma and the reflector scalars (computeHouseholderVec, online_householder_qr.cpp:97-118)
      float sigma = 0.f;
      for (int k = 0; k <= i; ++k) { const float v = D[qrRowOffset(k, n) + i]; sigma = fmaf(v, v, sigma); }
      const float x1 = R[qrRowOffset(i, n) + i];
      const float mu = sqrtf(x1 * x1 + sigma);
      const float v1 = (x1 <= 0.f) ? (x1 - mu) : (-sigma / (x1 + mu));
      scal[0] = sigma;
      scal[1] = sigma == 0.f ? 0.f : 2.f * v1 * v1 / (sigma + v1 * v1);
      scal[2] = sigma == 0.f ? 0.f : 1.f / v1;
      scal[3] = mu;
    }
    __syncthreads();
    const float sigma = scal[0], beta = scal[1], inv = scal[2];
    if (sigma != 0.f) {
      const int ro = qrRowOffset(i, n);
      for (int j = i + 1 + tid; j <= n; j += kQrThreads) {
        float* y1 = j < n ? R + ro + j : y + i;
        float dot = 0.f;
        if (j < n) { for (int k = 0; k <= i; ++k) dot = fmaf(D[qrRowOffset(k, n) + i], D[qrRowOffset(k, n) + j], dot); }
        else { for (int k = 0; k <= i; ++k) dot = fmaf(D[qrRowOffset(k, n) + i], dvec[k], dot); }
        const float r = *y1;
        const float s = (r + dot * inv) * beta;
        *y1 = r - s;
        const float si = s * inv;
        if (j < n) { for (int k = 0; k <= i; ++k) D[qrRowOffset(k, n) + j] = fmaf(-si, D[qrRowOffset(k, n) + i], D[qrRowOffset(k, n) + j]); }
        else { for (int k = 0; k <= i; ++k) dvec[k] = fmaf(-si, D[qrRowOffset(k, n) + i], dvec[k]); }
      }
    }
    __syncthreads();
    if (tid == 0 && sigma != 0.f) R[qrRowOffset(i, n) + i] = scal[3];
    __syncthreads();
  }
}

// getError(theta) for one instance by the whole CTA: FK (three passes) + the units' error contributions, summed in double, rounded
// through float (skeleton_solver_function.cpp:64-83). js: [J][kJointStateStride] scratch.
__device__ double trGetError(const FunctionTables& T, const float* th, float* js, const float* targets, const float* cw, double* dred) {
  const int tid = threadIdx.x;
  fkPasses<false, false>(CtaLanes<kQrThreads>{tid}, T, th, js);
  double err = 0.0;
  for (int u = tid; u < T.numUnits; u += kQrThreads) err += (double)evalUnit<false>(T, u, th, nullptr, js, targets, cw, nullptr, nullptr);
  for (int o = 16; o > 0; o >>= 1) err += __shfl_xor_sync(0xffffffffu, err, o);
  if ((tid & 31) == 0) dred[tid >> 5] = err;
  __syncthreads();
  double e = 0.0;
  for (int w = 0; w < kQrThreads / 32; ++w) e += dred[w];
  __syncthreads();
  return (double)(float)e;
}

__global__ void __launch_bounds__(kQrThreads, 1) trustRegionQrKernel(const TrQrArgs a) {
  extern __shared__ __align__(16) float trSmem[];
  const CholArgs& c = a.q.c;
  const int b = blockIdx.x;
  if (c.state.active[b] == 0) return;
  const FunctionTables& T = a.T;
  const int n = c.ns, tid = threadIdx.x, lane = tid & 31;
  const size_t packed = (size_t(n) * (n + 1) / 2 + 3) & ~size_t(3);
  const size_t n4 = size_t((n + 3) & ~3), np4 = size_t((T.numParams + 3) & ~3);
  const size_t chunk = (size_t(n + 1) * size_t(a.maxChunkRows | 1) + 3) & ~size_t(3); // (every region starts on a multiple of four floats)
  float* R = trSmem;
  float* D = R + packed;                         // step 1: the Jacobian chunk; step 2: the diagonal rows being folded in
  float* y = D + (packed > chunk ? packed : chunk);
  float* x = y + n4;
  float* g = x + n4;
  float* pl = g + n4;
  float* ql = pl + n4;
  float* dvec = ql + n4;
  float* step = dvec + n4;                       // the accepted step (zero when every trust step was rejected)
  float* norms = step + n4;                      // [n + 1]
  float* th = norms + ((n + 4) & ~3);            // current parameters (all numParams of them)
  float* trial = th + np4;
  float* js = trial + np4;
  float* red = js + ((T.numJoints * kJointStateStride + 3) & ~3); // [8] float partials | [4] reflector scalars | doubles
  float* scal = red + 8;
  double* dred = reinterpret_cast<double*>(red + 16); // [8] (64-byte offset from a 16-byte aligned base: 8-byte aligned)

  float* theta = c.theta + size_t(b) * c.ldTheta;
  for (int i = tid; i < T.numParams; i += kQrThreads) th[i] = theta[i];
  for (int i = tid; i < n; i += kQrThreads) step[i] = 0.f;
  qrFoldJacobian(a.q, b, R, y, norms, D, n, 1e-10f); // (:81-110; ends with a barrier-free tail: synchronise before reading R)
  __syncthreads();
  for (int j = tid; j < n; j += kQrThreads) { // gradientSub_ = 2 R^T y (:116)
    float s = 0.f;
    for (int i = 0; i <= j; ++i) s = fmaf(R[qrRowOffset(i, n) + j], y[i], s);
    g[j] = 2.f * s;
  }
  float* Rsaved = a.rSaved + size_t(b) * packed; // Rmatrix_ (:119)
  for (size_t idx = tid; idx < size_t(n) * (n + 1) / 2; idx += kQrThreads) Rsaved[idx] = R[idx];
  __syncthreads();
  const double error = c.state.errors[b];
  const float* targets = a.targets + size_t(b) * T.targetStride;
  const float* cw = a.cweights + (T.weightsPerInstance ? size_t(b) * T.numWeights : 0);
  float radius = a.radius[b], lambda = 1e-10f;
  bool accepted = false;
  for (int iTrustStep = 0; iTrustStep < 10; ++iTrustStep) {
    if (tid < 32) qrSolveUpperWarp(R, y, x, n, lane); // searchDir_sub = qrSolver_.result()
    __syncthreads();
    const float xg = trDot(x, g, n, red);
    if ((double)xg < (double)FLT_EPSILON * (1.0 + error)) break; // (:162-164) block-uniform
    for (int iIter = 0; iIter < 3; ++iIter) {
      const float xn = sqrtf(trDot(x, x, n, red));
      if (xn < 1.05f * radius) break;
      for (int i = tid; i < n; i += kQrThreads) ql[i] = -0.5f * g[i];
      __syncthreads();
      if (tid < 32) { qrSolveUpperTransposedWarp(R, ql, ql, n, lane); qrSolveUpperWarp(R, ql, pl, n, lane); qrSolveUpperTransposedWarp(R, pl, ql, n, lane); }
      __syncthreads();
      const float pl2 = trDot(pl, pl, n, red), ql2 = trDot(ql, ql, n, red);
      if (ql2 < FLT_EPSILON) break;
      const float plNorm = sqrtf(pl2);
      const float deltaLambda = (pl2 / ql2) * ((plNorm - radius) / radius); // Nocedal & Wright (4.44)
      if (deltaLambda <= 0.f) break; // lambda may only grow
      const float lambdaNew = lambda + deltaLambda;
      trFoldDiagonal(R, y, D, dvec, scal, n, sqrtf(lambdaNew - lambda));
      lambda = lambdaNew;
      if (tid < 32) qrSolveUpperWarp(R, y, x, n, lane);
      __syncthreads();
    }
    // trial parameters (subsetToFullVector + updateParameters: theta -= delta) and their error
    for (int i = tid; i < T.numParams; i += kQrThreads) trial[i] = th[i];
    __syncthreads();
    for (int i = tid; i < n; i += kQrThreads) { const int col = c.cols[i]; if (col >= 0) trial[col] = th[col] - x[i]; }
    __syncthreads();
    const double errorNew = trGetError(T, trial, js, targets, cw, dred);
    // quadratic model (:133-140): error - g.x + |R_saved x|^2, in float
    float sq = 0.f;
    for (int i = tid; i < n; i += kQrThreads) {
      const float* row = Rsaved + qrRowOffset(i, n);
      float r = 0.f;
      for (int j = i; j < n; ++j) r = fmaf(row[j], x[j], r);
      sq = fmaf(r, r, sq);
    }
    sq = trBlockSum(sq, red);
    const float gx = trDot(g, x, n, red); // (the damping search may have changed x since the test above)
    const float model = ((float)error - gx) + sq;
    const float rho = (float)((error - errorNew) / (error - (double)model)); // (:249)
    if (rho < 0.25f) radius = 0.25f * radius;
    else if (rho > 0.75f && lambda > 0.f) radius = fminf(2.f * radius, a.maxRadius);
    if (rho > 0.f) { accepted = true; break; }
    // rejected: parameters stay, the radius has shrunk (R keeps the damping added so far, as in the reference)
  }
  if (accepted) {
    for (int i = tid; i < n; i += kQrThreads) step[i] = x[i];
    __syncthreads();
    for (int i = tid; i < n; i += kQrThreads) { const int col = c.cols[i]; if (col >= 0) theta[col] = th[col] - x[i]; }
  }
  if (tid == 0) a.radius[b] = radius;
  for (int i = tid; i < n; i += kQrThreads) g[i] = 0.5f * g[i]; // J^T r, the convention of the other kernels' tail
  __syncthreads();
  CholArgs tail = c;
  tail.applyUpdate = 0; // the parameters were written above
  cholFinish(tail, b, n, step, g, false);
}

cudaError_t launchTrustRegionQr(const TrQrArgs& a, cudaStream_t stream) {
  const size_t smem = trQrSmemFloats(a.q.c.ns, a.T.numParams, a.T.numJoints, a.maxChunkRows) * sizeof(float);
  cudaError_t e = cudaFuncSetAttribute(trustRegionQrKernel, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem));
  if (e != cudaSuccess) return e;
  trustRegionQrKernel<<<a.q.c.batch, kQrThreads, smem, stream>>>(a);
  return cudaGetLastError();
}

} // namespace mb2
