// PTX wrappers shared by the sm_90a kernels: mbarrier, TMA (tensor and 1-D bulk copies into shared memory).
#pragma once

#include <cuda.h>

#include <cstdint>
#include <cstdio>

namespace mb2 {

constexpr unsigned long long kSpinLimit = 4000000000ull; // ~2 s of SM cycles: a barrier that never completes traps instead of hanging the GPU

__device__ __forceinline__ uint32_t smemAddr(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

__device__ __forceinline__ void mbarInit(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbarExpectTx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbarArrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbarWait(uint32_t bar, uint32_t parity) {
  uint32_t done = 0;
  const long long t0 = clock64();
  while (true) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(bar), "r"(parity)
        : "memory");
    if (done) break;
    if ((uint64_t)(clock64() - t0) > kSpinLimit) {
      printf("momentum_b200: mbarrier timeout (block %d thread %d bar %u parity %u)\n", blockIdx.x, threadIdx.x, bar, parity);
      __trap();
    }
  }
}
// same, without the diagnostic print: for kernels that issue wgmma, where any function call (printf) makes the compiler serialise
// the wgmma pipeline. kSleep: sleep between polls (waiters with slack)
template <bool kSleep>
__device__ __forceinline__ void mbarWaitSilent(uint32_t bar, uint32_t parity) {
  uint32_t done = 0;
  const long long t0 = clock64();
  while (true) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(bar), "r"(parity)
        : "memory");
    if (done) break;
    if constexpr (kSleep) __nanosleep(32);
    if ((uint64_t)(clock64() - t0) > kSpinLimit) __trap();
  }
}
// same, for waiters with slack (producer / converter / epilogue roles): sleeps between polls so that the spinning warp does not
// take issue slots from the warps doing the work
__device__ __forceinline__ void mbarWaitRelaxed(uint32_t bar, uint32_t parity) {
  uint32_t done = 0;
  const long long t0 = clock64();
  while (true) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(bar), "r"(parity)
        : "memory");
    if (done) break;
    __nanosleep(32);
    if ((uint64_t)(clock64() - t0) > kSpinLimit) {
      printf("momentum_b200: mbarrier timeout (block %d thread %d bar %u parity %u)\n", blockIdx.x, threadIdx.x, bar, parity);
      __trap();
    }
  }
}
__device__ __forceinline__ void tmaLoad3d(uint32_t dst, const CUtensorMap* map, int c0, int c1, int c2, uint32_t bar) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];" ::"r"(dst),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(c2), "r"(bar)
      : "memory");
}
// 1-D bulk copy global -> shared (bytes % 16 == 0, both addresses 16-byte aligned), completion on an mbarrier
__device__ __forceinline__ void bulkLoad(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}
// makes mbarrier.init visible to the async proxy before the first TMA completes on it
__device__ __forceinline__ void fenceBarrierInit() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fenceProxyAsync() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

} // namespace mb2
