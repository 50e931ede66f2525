// vampnet_b200 — the fixed-order block reduction of the audio kernels (onset.cu, beat.cu, mel.cu): a xor tree in each
// warp, then the warps' results added or compared in warp order, so a result depends on the block's values alone.
#pragma once
#include <cuda_runtime.h>

namespace vnb {

enum class Reduce { SUM, MAX, MIN };

template <Reduce OP, class T>
__device__ __forceinline__ T reduce_op(T a, T b) {
  if (OP == Reduce::SUM) return a + b;
  if (OP == Reduce::MAX) return fmax(a, b);
  return fmin(a, b);
}

// Every thread of a WARPS-warp block must call it; each gets the result.  red: WARPS values in shared memory, which the
// leading barrier lets a previous reduction finish reading.
template <Reduce OP, int WARPS, class T>
__device__ __forceinline__ T block_reduce(T v, T* red) {
  for (int o = 16; o; o >>= 1) v = reduce_op<OP>(v, __shfl_xor_sync(0xffffffffu, v, o));
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  v = red[0];
  for (int w = 1; w < WARPS; ++w) v = reduce_op<OP>(v, red[w]);
  return v;
}

}  // namespace vnb
