// The loop-control kernel of the device-driven conflict loop (lossless engine, mp_octree_run_fused_async).  It sits apart
// from octree_kernels.cuh because it calls the device runtime's cudaGraphSetConditional: a CPU model of the kernels declares
// its own cudaGraphSetConditional before including this header, and the rest of the engine's kernels need none.
#pragma once
#include "octree_kernels.cuh"

namespace octree_k {

// one thread: conflict_loop_continue's decision, handed to the WHILE node's condition `cond` (a
// cudaGraphConditionalHandle)
__global__ void loop_control_kernel(const int32_t* count, int32_t* passes, int32_t* truncated, int level, int cap,
                                    unsigned long long cond) {
  if (threadIdx.x == 0) cudaGraphSetConditional(cond, conflict_loop_continue(count, passes, truncated, level, cap));
}

}  // namespace octree_k
