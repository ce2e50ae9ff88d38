// K2 on the Hopper tensor cores: per-instance [J r]^T [J r] (upper triangle) with wgmma (tf32 inputs, fp32 accumulators in
// registers), operands staged global -> shared by TMA.
//
//   reference computation: jtj.selfadjointView<Lower>().rankUpdate(J^T); jtr += J^T r
//   (momentum/solver/solver_function.cpp:113-116, gauss_newton_solver.cpp:215-216)
//
// Data layout. The device Jacobian of an instance is R = numCols + 1 "column vectors" of ldJ floats
// (column c of J at J + c*ldJ, the residual r as vector numCols): a K-major [R x K] operand, which is
// exactly what both wgmma operands want for D = X X^T with X = [J r]^T (tf32 wgmma takes K-major operands only). D's last row is
// J^T r, so Jtr costs nothing extra. One TMA box (boxRows x 32 floats, SWIZZLE_128B) per 32-row K block lands the whole K slab of
// an instance; out-of-range rows are zero-filled by TMA.
//
// Precision. tf32 keeps 10 mantissa bits, so a single pass gives ~1e-3 relative error, which would change the Gauss-Newton path
// of the under-determined IK problems (m < n). The default is the 3xTF32 split: x = hi + lo with hi = tf32(x), lo = tf32(x - hi);
// D += hi*hi + hi*lo + lo*hi. The consumer threads derive hi (in place) and lo (second buffer, same swizzled positions) from the
// raw fp32 slab that TMA delivered.
//
// Work items. The result is cut into row tiles of 128 (two warpgroups of M = 64); row tile t needs the columns 128 t .. only (the
// upper triangle). An item is (row tile t, a chunk of at most 256 of those columns) = one register accumulator of N = 128 or 256
// columns per warpgroup:
//   * diagonal item: columns 128 t .. 128 t + 255 - ONE box of up to 256 operand rows, whose first 128 rows are also the A operand;
//   * far item (only when numCols + 1 > 128 t + 256): the remaining columns - a B box of those rows plus a separate 128-row A box.
// Up to numCols + 1 = 512 (bodyhands300: 425) there are at most four row tiles and at most one far item per tile. Columns of an
// accumulator beyond the item's width multiply rows that TMA zero-filled and are not stored.
//
// Roles in one persistent CTA (1 CTA / SM, 288 threads):
//   warps 0..7  two consumer warpgroups: hi/lo conversion of a landed stage (all 256 threads), then each warpgroup issues the
//               wgmmas of its 64 rows; the conversion of stage s + 1 overlaps the wgmmas of stage s. After an item's last K
//               block the accumulators go straight from registers to the rows (upper triangle) of the symmetric matrix.
//   warp 8      TMA producer (one elected lane)
// Pipeline: smem ring full (TMA) -> empty (both warpgroups' wgmmas of the stage have completed).
#include "ik_jtj_tc.cuh"
#include "ik_ptx.cuh"

#include <cuda.h>

#include <cstdint>
#include <cstdio>
#include <cstdlib>

namespace mb2 {

namespace {

constexpr int kConsumerThreads = 256; // two warpgroups
constexpr int kTcThreads = kConsumerThreads + 32;
constexpr int kKBlock = kJtjKBlock; // floats per K block = one 128-byte swizzle row
constexpr int kRowBytes = 128;
constexpr int kWgmmaK = 8;          // tf32: 32 bytes of K per instruction

constexpr int kMaxItems = 8;
struct TcItem {
  int aRow0;    // first operand row of the A box = first row of the row tile (128 t)
  int bRow0;    // first operand row of the B box = first column of the chunk
  int n;        // columns of the chunk, a multiple of 16, <= 256
  int bBoxRows; // 256 or 128: which tensor map loads the B box (also the wgmma N)
  int sepA;     // far item: the A rows are not in the B box, a second (128-row) box is loaded behind the B region
};
struct TcParams {
  int batch;
  int ns, numCols, ldJ, kBlocks;
  float* H;
  int ldH;
  const int32_t* active;
  int passes;     // 3 or 1
  int numItems;
  TcItem items[kMaxItems];
  int bRegionRows; // operand rows reserved for the B box in a stage (256, or 128 when every item fits a 128-row box)
  int planeRows;   // bRegionRows (+ 128 when some item needs a separate A box): rows of one hi (or lo) plane of a stage
  int stages;
  size_t hStride;
  float* G;       // optional [batch][ldG]: J^T r as a contiguous vector (the scheduled Cholesky bulk-copies it)
  int ldG;
};

__device__ __forceinline__ void wgmmaTf32N128(float (&d)[64], uint64_t descA, uint64_t descB, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(descA), "l"(descB), "r"(accumulate)
      : "memory");
}
__device__ __forceinline__ void wgmmaTf32N256(float (&d)[128], uint64_t descA, uint64_t descB, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n256k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(descA), "l"(descB), "r"(accumulate)
      : "memory");
}

__device__ __forceinline__ uint32_t toTf32(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return r;
}

// K-major, SWIZZLE_128B shared-memory matrix descriptor of wgmma (the stage buffers are 1024-byte aligned, base offset 0):
// start>>4 [0,14) | LBO>>4 [16,30) (=1, unused for swizzled K-major) | SBO>>4 [32,46) (8 rows * 128 B) | layout 1 = SWIZZLE_128B [62,64)
__device__ __forceinline__ uint64_t makeSmemDesc(uint32_t addr) {
  return (uint64_t)((addr & 0x3FFFF) >> 4) | (1ull << 16) | ((uint64_t)(1024 >> 4) << 32) | (1ull << 62);
}

struct TcSmem {
  uint32_t base;      // shared-window address of the 1024-aligned stage ring
  uint8_t* gen;       // generic pointer to the same byte
  uint32_t slabBytes, stageBytes, aRegionOff, barBase;
  int stages;
  __device__ uint32_t fullBar(int s) const { return barBase + 8u * s; }
  __device__ uint32_t emptyBar(int s) const { return barBase + 8u * (stages + s); }
};

// One work item of instance b for both consumer warpgroups: the K loop (convert, wgmma) and the store of the accumulators.
// N = the item's B box rows = the wgmma N.
template <int N>
__device__ __forceinline__ void consumeItem(const TcParams& p, const TcSmem& m, const TcItem& I, int b, int& s, uint32_t& ph) {
  constexpr int kRegs = N / 2;
  float d[kRegs];
#pragma unroll
  for (int i = 0; i < kRegs; ++i) d[i] = 0.f;
  const int ct = threadIdx.x, wg = ct >> 7, t = ct & 127;
  // two segments of a plane: the B box, and (far items) the A box behind the B region
  const int vecsB = I.bBoxRows * kRowBytes / 16, vecsA = I.sepA ? 128 * kRowBytes / 16 : 0, offA = int(m.aRegionOff / 16u);
  const uint32_t aOff = (I.sepA ? m.aRegionOff : 0u) + uint32_t(wg * 64 * kRowBytes); // this warpgroup's 64 rows of the A operand
  int prev = -1;
  for (int kb = 0; kb < p.kBlocks; ++kb) {
    mbarWaitSilent<false>(m.fullBar(s), ph);
    float4* hi = reinterpret_cast<float4*>(m.gen + m.stageBytes * s);
    float4* lo = reinterpret_cast<float4*>(m.gen + m.stageBytes * s + m.slabBytes);
#pragma unroll 4
    for (int j = ct; j < vecsB + vecsA; j += kConsumerThreads) {
      const int i = j < vecsB ? j : offA + (j - vecsB);
      const float4 x = hi[i];
      uint4 h;
      h.x = toTf32(x.x); h.y = toTf32(x.y); h.z = toTf32(x.z); h.w = toTf32(x.w);
      reinterpret_cast<uint4*>(hi)[i] = h;
      if (p.passes == 3) {
        uint4 l;
        l.x = toTf32(x.x - __uint_as_float(h.x)); l.y = toTf32(x.y - __uint_as_float(h.y));
        l.z = toTf32(x.z - __uint_as_float(h.z)); l.w = toTf32(x.w - __uint_as_float(h.w));
        reinterpret_cast<uint4*>(lo)[i] = l;
      }
    }
    fenceProxyAsync(); // generic-proxy stores -> visible to the tensor core (async proxy)
    asm volatile("bar.sync 1, %0;" ::"n"(kConsumerThreads) : "memory");
    asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
    const uint32_t hiA = m.base + m.stageBytes * s, loA = hiA + m.slabBytes;
    for (int pass = 0; pass < p.passes; ++pass) {
      const uint32_t aBase = (pass == 2 ? loA : hiA) + aOff; // hi*hi, hi*lo, lo*hi
      const uint32_t bBase = pass == 1 ? loA : hiA;
#pragma unroll
      for (int k4 = 0; k4 < kKBlock / kWgmmaK; ++k4) {
        const uint32_t acc = (kb == 0 && pass == 0 && k4 == 0) ? 0u : 1u;
        if constexpr (N == 256) wgmmaTf32N256(d, makeSmemDesc(aBase + k4 * 32u), makeSmemDesc(bBase + k4 * 32u), acc);
        else wgmmaTf32N128(d, makeSmemDesc(aBase + k4 * 32u), makeSmemDesc(bBase + k4 * 32u), acc);
      }
    }
    asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
    asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory"); // the previous stage's wgmmas are done: release it
    if (prev >= 0 && t == 0) mbarArrive(m.emptyBar(prev));
    prev = s;
    if (++s == p.stages) { s = 0; ph ^= 1u; }
  }
  asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
  if (t == 0) mbarArrive(m.emptyBar(prev));

  // accumulator fragment: d[4j + 2h + e] = D(16 warp + lane / 4 + 8 h, 8 j + 2 (lane % 4) + e) of this warpgroup's 64 rows
  float* H = p.H + (size_t)b * p.hStride;
  const int warp = t >> 5, lane = t & 31;
  const int colEnd = I.bRow0 + I.n;
  const bool solverPath = p.ns == p.numCols;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int row = I.aRow0 + wg * 64 + warp * 16 + (lane >> 2) + 8 * h;
    const int i = row < p.ns ? row : (row == p.numCols ? p.ns : -1); // row of the (ns+1) system; -1: not wanted
    if (i < 0) continue;
    float* Hrow = H + (size_t)i * p.ldH;
#pragma unroll
    for (int j = 0; j < N / 8; ++j) {
      const int c = I.bRow0 + 8 * j + 2 * (lane & 3);
      const float v0 = d[4 * j + 2 * h], v1 = d[4 * j + 2 * h + 1];
      if (solverPath) {
        // full rows, upper triangle (col >= row) only: everything downstream reads H(min, max)
        if (c + 1 < colEnd && c + 1 < p.ldH && c >= i) *reinterpret_cast<float2*>(Hrow + c) = make_float2(v0, v1);
        else {
          if (c < colEnd && c < p.ldH && c >= i) Hrow[c] = v0;
          if (c + 1 < colEnd && c + 1 < p.ldH && c + 1 >= i) Hrow[c + 1] = v1;
        }
        if (p.G != nullptr && i < p.ns) { // column numCols = J^T r
          if (c == p.numCols) p.G[(size_t)b * p.ldG + i] = v0;
          if (c + 1 == p.numCols) p.G[(size_t)b * p.ldG + i] = v1;
        }
      } else {
        // leading-block request (ns < numCols, getJtJR parity entry): columns ns.. are skipped except the residual column
        if (c < p.ns) Hrow[c] = v0; else if (c == p.numCols) Hrow[p.ns] = v0;
        if (c + 1 < p.ns) Hrow[c + 1] = v1; else if (c + 1 == p.numCols) Hrow[p.ns] = v1;
      }
    }
  }
}

__global__ void __launch_bounds__(kTcThreads, 1) jtjTensorKernel(const __grid_constant__ CUtensorMap tmap, const __grid_constant__ CUtensorMap tmapHalf, const TcParams p) {
  extern __shared__ __align__(1024) uint8_t smemRaw[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  TcSmem m;
  m.base = (smemAddr(smemRaw) + 1023u) & ~1023u;
  m.gen = smemRaw + (m.base - smemAddr(smemRaw));
  m.slabBytes = (uint32_t)p.planeRows * kRowBytes;                // one K block of every operand row of an item: [B box | A box of far items]
  m.stageBytes = m.slabBytes * (p.passes == 3 ? 2u : 1u);          // hi [+ lo]
  m.aRegionOff = (uint32_t)p.bRegionRows * kRowBytes;              // where a far item's A box sits inside a plane
  m.barBase = m.base + m.stageBytes * p.stages;
  m.stages = p.stages;

  if (threadIdx.x == 0) {
    for (int s = 0; s < p.stages; ++s) { mbarInit(m.fullBar(s), 1); mbarInit(m.emptyBar(s), 2); } // empty: one arrival per consumer warpgroup
    fenceBarrierInit();
  }
  __syncthreads();

  int s = 0;
  uint32_t ph = 0;
  if (warp == kConsumerThreads / 32) {
    // ---------------- TMA producer ----------------
    if (lane == 0) {
      for (int b = blockIdx.x; b < p.batch; b += gridDim.x) {
        if (p.active != nullptr && p.active[b] == 0) continue;
        for (int it = 0; it < p.numItems; ++it) {
          const TcItem I = p.items[it];
          const uint32_t bBytes = (uint32_t)I.bBoxRows * kRowBytes;
          for (int kb = 0; kb < p.kBlocks; ++kb) {
            mbarWaitSilent<true>(m.emptyBar(s), ph ^ 1u);
            mbarExpectTx(m.fullBar(s), bBytes + (I.sepA ? 128u * kRowBytes : 0u));
            tmaLoad3d(m.base + m.stageBytes * s, I.bBoxRows == 128 ? &tmapHalf : &tmap, kb * kKBlock, I.bRow0, b, m.fullBar(s));
            if (I.sepA) tmaLoad3d(m.base + m.stageBytes * s + m.aRegionOff, &tmapHalf, kb * kKBlock, I.aRow0, b, m.fullBar(s));
            if (++s == p.stages) { s = 0; ph ^= 1u; }
          }
        }
      }
    }
  } else {
    // ---------------- consumer warpgroups ----------------
    for (int b = blockIdx.x; b < p.batch; b += gridDim.x) {
      if (p.active != nullptr && p.active[b] == 0) continue;
      for (int it = 0; it < p.numItems; ++it) {
        const TcItem I = p.items[it];
        if (I.bBoxRows == 128) consumeItem<128>(p, m, I, b, s, ph);
        else consumeItem<256>(p, m, I, b, s, ph);
      }
    }
  }
}

using EncodeTiledFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                   const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn encodeTiled() {
  static EncodeTiledFn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

int roundUpI(int v, int m) { return (v + m - 1) / m * m; }

struct Shape {
  int rows, r16, numItems, bRegionRows, planeRows;
  bool anySepA;
  TcItem items[kMaxItems];
};
Shape shapeFor(int numCols) {
  Shape s{};
  s.rows = numCols + 1;
  s.r16 = roundUpI(s.rows, 16);
  const int tiles = (s.rows + 127) / 128;
  for (int t = tiles - 1; t >= 0; --t) { // last row tile first, as the kernel's roles walk them
    const int c0 = 128 * t, left = s.r16 - c0;
    TcItem d{};
    d.aRow0 = c0; d.bRow0 = c0; d.n = left < 256 ? left : 256; d.bBoxRows = d.n <= 128 ? 128 : 256; d.sepA = 0;
    s.items[s.numItems++] = d;
    if (left > 256) { // the columns beyond the diagonal box: a far item with its own A box
      TcItem f{};
      f.aRow0 = c0; f.bRow0 = c0 + 256; f.n = left - 256; f.bBoxRows = f.n <= 128 ? 128 : 256; f.sepA = 1;
      s.items[s.numItems++] = f;
      s.anySepA = true;
    }
  }
  for (int i = 0; i < s.numItems; ++i) s.bRegionRows = s.bRegionRows > s.items[i].bBoxRows ? s.bRegionRows : s.items[i].bBoxRows;
  s.planeRows = s.bRegionRows + (s.anySepA ? 128 : 0);
  return s;
}

} // namespace

cudaError_t makeTensorMap3d(CUtensorMap* map, const float* base, const uint64_t dims[3], const uint64_t strideBytes[2], const uint32_t box[3], int swizzleBytes) {
  if (encodeTiled() == nullptr) return cudaErrorNotSupported;
  const cuuint64_t d[3] = {dims[0], dims[1], dims[2]};
  const cuuint64_t st[2] = {strideBytes[0], strideBytes[1]};
  const cuuint32_t bx[3] = {box[0], box[1], box[2]};
  const cuuint32_t estr[3] = {1u, 1u, 1u};
  const CUtensorMapSwizzle sw = swizzleBytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : swizzleBytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B
                              : swizzleBytes == 32 ? CU_TENSOR_MAP_SWIZZLE_32B : CU_TENSOR_MAP_SWIZZLE_NONE;
  const CUresult r = encodeTiled()(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float*>(base), d, st, bx, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, sw,
                                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? cudaSuccess : cudaErrorInvalidValue;
}

bool jtjTensorSupported(int ns, int numCols, int ldJ) {
  return encodeTiled() != nullptr && jtjTensorShape(ns, numCols, ldJ);
}

cudaError_t launchJtJTensor(const JtJArgs& a, int passes, cudaStream_t stream) {
  if (!jtjTensorSupported(a.ns, a.numCols, a.ldJ)) return cudaErrorNotSupported;
  const Shape sh = shapeFor(a.numCols);
  // TMA descriptors over the device Jacobian [batch][numCols + 1][ldJ] (innermost first): 256-row and 128-row boxes of one 32-float K block
  CUtensorMap map;
  const uint64_t dims[3] = {(uint64_t)a.ldJ, (uint64_t)(a.numCols + 1), (uint64_t)a.batch};
  const uint64_t strides[2] = {(uint64_t)a.ldJ * sizeof(float), (uint64_t)(a.numCols + 1) * a.ldJ * sizeof(float)};
  const uint32_t box[3] = {(uint32_t)kKBlock, 256u, 1u};
  cudaError_t me = makeTensorMap3d(&map, a.jacobian, dims, strides, box, 128);
  if (me != cudaSuccess) return me;
  CUtensorMap mapHalf;
  const uint32_t boxHalf[3] = {(uint32_t)kKBlock, 128u, 1u};
  me = makeTensorMap3d(&mapHalf, a.jacobian, dims, strides, boxHalf, 128);
  if (me != cudaSuccess) return me;
  TcParams p{};
  p.batch = a.batch;
  p.ns = a.ns;
  p.numCols = a.numCols;
  p.ldJ = a.ldJ;
  p.kBlocks = (a.kRows + kKBlock - 1) / kKBlock;
  p.H = a.H;
  p.ldH = a.ldH;
  p.active = a.active;
  p.passes = passes == 3 ? 3 : 1;
  p.numItems = sh.numItems;
  for (int i = 0; i < sh.numItems; ++i) p.items[i] = sh.items[i];
  p.bRegionRows = sh.bRegionRows;
  p.planeRows = sh.planeRows;
  p.hStride = a.hStride;
  p.G = a.g;
  p.ldG = a.ldG;
  // stage ring within 196 KB of the 227 KB a block may have: 3 stages of the humanoid's 3xTF32 slab (2 x 32 KB), 2 of bodyhands' (2 x 48 KB)
  const size_t stageBytes = size_t(sh.planeRows) * kRowBytes * (p.passes == 3 ? 2 : 1);
  int stages = int((196 * 1024) / stageBytes);
  if (stages > 6) stages = 6;
  if (stages < 2) return cudaErrorInvalidConfiguration;
  p.stages = stages;
  const size_t smem = stageBytes * stages + 1024 /*alignment slack*/ + 8 * 2 * stages;
  cudaError_t e = cudaFuncSetAttribute(jtjTensorKernel, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem));
  if (e != cudaSuccess) return e;
  int dev = 0, sms = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const int grid = a.batch < sms ? a.batch : sms;
  jtjTensorKernel<<<grid, kTcThreads, smem, stream>>>(map, mapHalf, p);
  return cudaGetLastError();
}

} // namespace mb2
