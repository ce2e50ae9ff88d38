// Latency / throughput probes of the instructions the per-instance kernels are built from (one CTA, clock64 around unrolled loops).
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -I momentum_b200/csrc -o scratch/microbench scripts/microbench.cu
#include <cstdio>
#include <cuda_runtime.h>
#include "ik_chol_sched.cuh"
using namespace mb2;

__global__ void probe(float* out, long long* cyc, int warpsActive) {
#if defined(__CUDA_ARCH__)
  __shared__ __align__(16) float tiles[8 * 256 * 2];
  __shared__ float y[16 * 16];
  __shared__ int flag;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int i = tid; i < 8 * 256 * 2; i += blockDim.x) tiles[i] = 0.001f * float((i * 37) % 101);
  for (int i = tid; i < 256; i += blockDim.x) y[i] = 1.f;
  // make diagonal tiles SPD
  for (int t = 0; t < 16; ++t) for (int i = tid; i < 16; i += blockDim.x) tiles[t * 256 + tileIdx(i, i)] += 4.f;
  __syncthreads();
  float acc = 0.f;
  long long t0, t1;
  // 1. dependent HMMA chain
  {
    float d[4] = {0.f, 0.f, 0.f, 0.f};
    const float a = 1.0f + lane, b = 0.5f;
    __syncthreads();
    t0 = clock64();
    if (warp < warpsActive) {
#pragma unroll
      for (int i = 0; i < 64; ++i) mmaTf32K8(d, a, a, a, a, b, b);
    }
    t1 = clock64();
    acc += d[0] + d[1] + d[2] + d[3];
    if (tid == 0) cyc[0] = (t1 - t0) / 64;
  }
  // 2. independent HMMA (4 accumulators)
  {
    float d0[4] = {0, 0, 0, 0}, d1[4] = {0, 0, 0, 0}, d2[4] = {0, 0, 0, 0}, d3[4] = {0, 0, 0, 0};
    const float a = 1.0f + lane, b = 0.5f;
    __syncthreads();
    t0 = clock64();
    if (warp < warpsActive) {
#pragma unroll
      for (int i = 0; i < 32; ++i) { mmaTf32K8(d0, a, a, a, a, b, b); mmaTf32K8(d1, a, a, a, a, b, b); mmaTf32K8(d2, a, a, a, a, b, b); mmaTf32K8(d3, a, a, a, a, b, b); }
    }
    t1 = clock64();
    acc += d0[0] + d1[1] + d2[2] + d3[3];
    if (tid == 0) cyc[1] = (t1 - t0) / 128;
  }
  // 3. dependent SHFL chain
  {
    float v = acc + lane;
    __syncthreads();
    t0 = clock64();
    if (warp < warpsActive) {
#pragma unroll
      for (int i = 0; i < 64; ++i) v = __shfl_sync(0xffffffffu, v, (lane + 1) & 31);
    }
    t1 = clock64();
    acc += v;
    if (tid == 0) cyc[2] = (t1 - t0) / 64;
  }
  // 4. independent SHFLs (16 per group)
  {
    float v[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) v[j] = acc + lane + j;
    __syncthreads();
    t0 = clock64();
    if (warp < warpsActive) {
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 16; ++j) v[j] = __shfl_sync(0xffffffffu, v[j], (lane + j) & 31);
    }
    t1 = clock64();
#pragma unroll
    for (int j = 0; j < 16; ++j) acc += v[j];
    if (tid == 0) cyc[3] = (t1 - t0) / 128;
  }
  // 5. one diagonal tile per half-warp
  {
    __syncthreads();
    t0 = clock64();
    if (warp < warpsActive) cholDiagTile(tiles + warp * 256, y + 16 * warp, lane, 0.05f, &flag);
    __syncthreads();
    t1 = clock64();
    if (tid == 0) cyc[4] = t1 - t0;
  }
  // 6. update-task-like chain: 8 tile products into one accumulator pair
  {
    float d[2][4] = {{0, 0, 0, 0}, {0, 0, 0, 0}}, s[2][4] = {{0, 0, 0, 0}, {0, 0, 0, 0}};
    __syncthreads();
    t0 = clock64();
    if (warp < warpsActive) {
      for (int p = 0; p < 8; ++p) tileProduct(tiles + ((p + warp) & 7) * 256, tiles + ((p + warp + 3) & 7) * 256 + 2048, lane, d, s);
    }
    t1 = clock64();
    acc += d[0][0] + d[1][3] + s[0][1] + s[1][2];
    if (tid == 0) cyc[5] = (t1 - t0) / 8;
  }
  // 7. dependent LDS chain (pointer chasing) and STS->LDS round trip
  {
    __shared__ int chain[64];
    if (tid < 64) chain[tid] = (tid + 7) & 63;
    __syncthreads();
    int p = lane;
    t0 = clock64();
#pragma unroll
    for (int i = 0; i < 64; ++i) p = chain[p];
    t1 = clock64();
    acc += p;
    if (tid == 0) cyc[6] = (t1 - t0) / 64;
  }
  // 8. block-wide barrier cost with all warps arriving together
  {
    __syncthreads();
    t0 = clock64();
#pragma unroll
    for (int i = 0; i < 16; ++i) __syncthreads();
    t1 = clock64();
    if (tid == 0) cyc[7] = (t1 - t0) / 16;
  }
  // 9. MUFU rcp + rsqrt dependent chain
  {
    float v = 1.5f + acc * 1e-30f;
    t0 = clock64();
#pragma unroll
    for (int i = 0; i < 32; ++i) { float r; asm volatile("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(v)); v = r + 1.f; }
    t1 = clock64();
    acc += v;
    if (tid == 0) cyc[8] = (t1 - t0) / 32;
  }
  out[tid] = acc;
#endif
}

// SM-level throughput of the Gram inner loop and of bare HMMA issue: every warp of one CTA runs `steps` mma3x steps over strips in shared
// memory (the gramTileAccumulate loop), then `steps` x 6 independent HMMAs; cycles for the whole CTA, so cycles / (steps * warps) is the
// SM's cost per step (per 6 HMMAs) at that occupancy.
__global__ void gramProbe(float* out, long long* cyc) {
#if defined(__CUDA_ARCH__)
  extern __shared__ __align__(16) float strips[]; // 116 strips of 64 floats
  __shared__ __align__(16) int quads[4 * 32];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int i = tid; i < 116 * 64; i += blockDim.x) strips[i] = 0.01f * float((i * 37) % 101) - 0.5f;
  for (int i = tid; i < 128; i += blockDim.x) quads[i] = 64 * ((i * 29 + 5) % 116);
  __syncthreads();
  float d[2][4] = {{0, 0, 0, 0}, {0, 0, 0, 0}};
  long long t0 = clock64();
  for (int rep = 0; rep < 4; ++rep) gramTileAccumulate(strips, quads, (warp & 15), (warp & 15) + 16, lane, d);
  __syncthreads();
  long long t1 = clock64();
  if (tid == 0) cyc[0] = (t1 - t0) / 64;
  float e0[4] = {0, 0, 0, 0}, e1[4] = {0, 0, 0, 0}, e2[4] = {0, 0, 0, 0}, e3[4] = {0, 0, 0, 0}, e4[4] = {0, 0, 0, 0}, e5[4] = {0, 0, 0, 0};
  const float a = 1.0f + lane, b = 0.5f;
  __syncthreads();
  t0 = clock64();
#pragma unroll 4
  for (int i = 0; i < 64; ++i) { mmaTf32K8(e0, a, a, a, a, b, b); mmaTf32K8(e1, a, a, a, a, b, b); mmaTf32K8(e2, a, a, a, a, b, b); mmaTf32K8(e3, a, a, a, a, b, b); mmaTf32K8(e4, a, a, a, a, b, b); mmaTf32K8(e5, a, a, a, a, b, b); }
  __syncthreads();
  t1 = clock64();
  if (tid == 0) cyc[1] = (t1 - t0) / 64;
  out[tid] = d[0][0] + d[1][3] + e0[0] + e1[1] + e2[2] + e3[3] + e4[0] + e5[1];
#endif
}

int main() {
  float* out; long long* cyc;
  cudaMalloc(&out, 1024 * 4); cudaMalloc(&cyc, 16 * 8);
  const char* names[9] = {"HMMA tf32 m16n8k8 dependent (cycles each)", "HMMA independent x4 (cycles each)", "SHFL dependent", "SHFL independent", "cholDiagTile (whole phase incl. barrier)",
                          "tileProduct per pair (chained accumulators)", "LDS dependent", "__syncthreads", "rcp + add dependent"};
  for (int threads : {32, 64, 256}) {
    for (int wa : {1, threads / 32}) {
      if (wa == 1 && threads == 32) continue;
      probe<<<1, threads>>>(out, cyc, wa);
      probe<<<1, threads>>>(out, cyc, wa);
      cudaDeviceSynchronize();
      long long h[16];
      cudaMemcpy(h, cyc, sizeof(h), cudaMemcpyDeviceToHost);
      printf("== %d threads, %d active warp(s): %s\n", threads, wa, cudaGetErrorString(cudaGetLastError()));
      for (int i = 0; i < 9; ++i) printf("  %-50s %lld\n", names[i], h[i]);
    }
  }
  cudaFuncSetAttribute(gramProbe, cudaFuncAttributeMaxDynamicSharedMemorySize, 116 * 64 * 4);
  for (int threads : {32, 128, 256, 512, 1024}) {
    gramProbe<<<1, threads, 116 * 64 * 4>>>(out, cyc);
    gramProbe<<<1, threads, 116 * 64 * 4>>>(out, cyc);
    cudaDeviceSynchronize();
    long long h[2];
    cudaMemcpy(h, cyc, sizeof(h), cudaMemcpyDeviceToHost);
    printf("== gramProbe %d warps on one SM: %lld cycles per mma3x step-round (all warps one step each) = %.1f cycles per step per SM; 6 independent HMMA round: %lld cycles = %.1f per HMMA per SM  (%s)\n",
           threads / 32, h[0], double(h[0]) / (threads / 32), h[1], double(h[1]) / (6.0 * threads / 32), cudaGetErrorString(cudaGetLastError()));
  }
  return 0;
}
