// Fused Gauss-Newton solve: ONE persistent kernel runs SolverT::solve (solver.cpp:50-128) for the whole batch.
//
// A CTA holds up to three *instance groups* of 256 threads. Every table the iteration walks (character, plan, Gram plan, Cholesky
// schedule) is staged once per CTA by bulk copies; a group then takes instances off a device-side work counter and keeps each one
// in shared memory for ALL of its iterations:
//
//   theta --ParameterTransform / FK sweep--> joint frames --units/cells--> Jacobian strips (shared memory)
//         --tile-sparse Gram (mma.sync 3xTF32)--> 16x16 tiles of J^T J + lambda I; a tile that would overwrite strips still being
//           read is parked in thread-local memory and written over them once they are dead
//         --level-scheduled Cholesky + both substitutions--> delta --> theta -= delta, convergence test (solver.cpp:98-113)
//
// so per solve an instance moves theta, its targets and three result words through HBM and nothing else: no Jacobian, no normal
// matrix, no per-iteration launch, no host round trip for the stopping rule (an instance that converges frees its group at once).
// The device functions are the ones the multi-kernel path uses (ik_device.cuh, ik_chol_sched.cuh): same arithmetic, same order.
#pragma once

#include <cuda_runtime.h>

#include "ik_chol_sched.cuh"
#include "ik_solve_path.h"
#include "ik_types.h"

namespace mb2 {

constexpr int kFusedGroupThreads = 256;

struct FusedArgs {
  int32_t batch;
  FunctionTables T;            // sizes; the table pointers are replaced by shared-memory addresses inside the kernel
  const int32_t* blob;         // the plan blob in global memory
  FusedBlobLayout L;
  CholSchedDev S;              // table pointers relative to `schedGlobal` (rebased onto the staged copy)
  const int32_t* schedGlobal;  // = S.blob
  int32_t gramOff[8];          // makeGramBlob offsets
  int32_t numStrips, stripStride, residOff, numOrder; // GramPlan (numOrder: entries of the tile-order table)
  float regularization;
  float* theta;                // [B][ldTheta] in/out
  int32_t ldTheta;
  const float* targets;        // [B][T.targetStride]
  const float* cweights;       // [numWeights] or [B][numWeights]
  SolveState state;            // errors (what SolverT::solve returns), iterations, status, history, options; the rest is in shared memory
  int32_t* workCounter;        // zeroed before the launch
  unsigned long long* phaseCycles; // optional [16]: per-phase cycles of the first group of CTA 0 (profiling instantiation)
  int32_t groups;              // instance groups per CTA (1..3)
  int32_t groupFloats;         // shared-memory floats per group
  int32_t unionFloats;         // ... of which the strips / tiles union region
};

// cfg: SolvePath::fused (ik_solve_path.h)
cudaError_t launchFusedSolve(const FusedArgs& a, const FusedConfig& cfg, int numSms, bool profile, cudaStream_t stream);

} // namespace mb2
