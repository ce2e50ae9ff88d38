// Tensor-core JtJ (wgmma tf32, accumulators in registers, operands staged by TMA).
#pragma once

#include <cuda.h>
#include <cuda_runtime.h>

#include "ik_kernels.cuh"

namespace mb2 {

// true when the wgmma kernel handles this (subset size, Jacobian row stride)
bool jtjTensorSupported(int ns, int numCols, int ldJ);
// passes: 3 = 3xTF32 split (fp32-class accuracy), 1 = single TF32 pass
cudaError_t launchJtJTensor(const JtJArgs& a, int passes, cudaStream_t stream);

// 3-D fp32 tensor map (innermost dimension first); swizzleBytes in {0, 32, 64, 128}
cudaError_t makeTensorMap3d(CUtensorMap* map, const float* base, const uint64_t dims[3], const uint64_t strideBytes[2], const uint32_t box[3], int swizzleBytes);

} // namespace mb2
