// vampnet_b200 — LoRA down-projection of per-request adapters (DESIGN.md §1):
//
//   u[m, j] = sum_k y[m, k] * A'[k, j]      for every adapted row m, j < R (R = 16 for QKV: [q | v], else 8)
//
// y is the bf16 A operand the consuming GEMM reads (y for QKV and FFN-up, att for the attention output projection, h for
// FFN-down).  The adapted GEMM epilogue then adds u[m] . B'[n] to the accumulators (gemm_wgmma.cu, lora_update).
//
// Four threads per row (k split into interleaved 8-element groups: thread s of a row takes groups s, s + 4, ...), 64
// rows per block.  A' of one adapter is staged in shared memory 256 k at a time (k-major, a 16-byte pad per 8 k so that
// the four splits' float4 reads hit disjoint banks; the lanes of a split read the same address, a broadcast); rows of
// other adapters wait while it is staged, so a block runs one pass per distinct adapter among its rows.  Each u[m, j] is
// four fma chains in fp32 over a fixed k order, added as (s0 + s1) + (s2 + s3): the result of a row does not depend on
// which rows share its block.  CUDA cores; M * R * K fma per launch.
#include "common.cuh"
#include "kernels.h"

namespace vnb {

constexpr int LORA_ROWS = 64, LORA_SPLIT = 4, LORA_THREADS = LORA_ROWS * LORA_SPLIT, LORA_KC = 256;

// float index in the staged chunk of element (k, j): k-major with 4 floats of padding after every 8 k
template <int R> __device__ __forceinline__ int lora_sidx(int k, int j) { return k * R + (k >> 3) * 4 + j; }

template <int R>
__global__ void __launch_bounds__(LORA_THREADS) lora_down_kernel(const __nv_bfloat16* __restrict__ y, int M, int K,
                                                                  const AdapterRefs r) {
  __shared__ __align__(16) float sA[LORA_KC * R + (LORA_KC / 8) * 4];
  const int split = static_cast<int>(threadIdx.x) & (LORA_SPLIT - 1);
  const int m = blockIdx.x * LORA_ROWS + (static_cast<int>(threadIdx.x) >> 2);
  const int id = m < M ? r.grp_adapter[r.rowgrp[m / r.rows_per_grp].group] : -1;
  for (int a = 0; a < VNB_MAX_ADAPTERS; ++a) {
    if (!__syncthreads_or(id == a)) continue;
    const float* A = r.table[a].a[r.slot] + static_cast<size_t>(r.layer) * K * R;
    float acc[R];
#pragma unroll
    for (int j = 0; j < R; ++j) acc[j] = 0.f;
    const __nv_bfloat16* yr = y + static_cast<size_t>(id == a ? m : 0) * K;
    for (int k0 = 0; k0 < K; k0 += LORA_KC) {
      __syncthreads();  // the previous chunk has been read by every thread
      for (int i = threadIdx.x; i < LORA_KC * R / 4; i += LORA_THREADS) {
        const int k = (4 * i) / R;
        *reinterpret_cast<float4*>(sA + 4 * i + (k >> 3) * 4) =
            __ldg(reinterpret_cast<const float4*>(A + static_cast<size_t>(k0) * R) + i);
      }
      __syncthreads();
      if (id == a) {
#pragma unroll 1
        for (int kk = split * 8; kk < LORA_KC; kk += 8 * LORA_SPLIT) {
          const uint4 raw = __ldg(reinterpret_cast<const uint4*>(yr + k0 + kk));
          const __nv_bfloat16* yb = reinterpret_cast<const __nv_bfloat16*>(&raw);
#pragma unroll
          for (int e = 0; e < 8; ++e) {
            const float x = __bfloat162float(yb[e]);
            const float* ak = sA + lora_sidx<R>(kk + e, 0);
#pragma unroll
            for (int j4 = 0; j4 < R / 4; ++j4) {
              const float4 w = *reinterpret_cast<const float4*>(ak + 4 * j4);
              acc[4 * j4 + 0] = __fmaf_rn(x, w.x, acc[4 * j4 + 0]);
              acc[4 * j4 + 1] = __fmaf_rn(x, w.y, acc[4 * j4 + 1]);
              acc[4 * j4 + 2] = __fmaf_rn(x, w.z, acc[4 * j4 + 2]);
              acc[4 * j4 + 3] = __fmaf_rn(x, w.w, acc[4 * j4 + 3]);
            }
          }
        }
      }
    }
    // the four splits of a row are lanes 4q .. 4q+3 of one warp: (s0 + s1) + (s2 + s3), every lane of the warp takes part
#pragma unroll
    for (int j = 0; j < R; ++j) {
      acc[j] = __fadd_rn(acc[j], __shfl_xor_sync(0xffffffffu, acc[j], 1));
      acc[j] = __fadd_rn(acc[j], __shfl_xor_sync(0xffffffffu, acc[j], 2));
    }
    if (id == a && split == 0) {
      float4* out = reinterpret_cast<float4*>(r.u + static_cast<size_t>(m) * R);
#pragma unroll
      for (int j4 = 0; j4 < R / 4; ++j4) out[j4] = make_float4(acc[4 * j4], acc[4 * j4 + 1], acc[4 * j4 + 2], acc[4 * j4 + 3]);
    }
  }
}

cudaError_t launch_lora_down(const void* y, int M, int K, const AdapterRefs& r, cudaStream_t st) {
  if (K % LORA_KC != 0 || M < 1 || !r.table || !r.grp_adapter || !r.rowgrp || !r.u || r.rows_per_grp < 1)
    return cudaErrorInvalidValue;
  const int blocks = (M + LORA_ROWS - 1) / LORA_ROWS;
  const auto* yb = reinterpret_cast<const __nv_bfloat16*>(y);
  if (r.slot == LORA_QKV) lora_down_kernel<16><<<blocks, LORA_THREADS, 0, st>>>(yb, M, K, r);
  else lora_down_kernel<8><<<blocks, LORA_THREADS, 0, st>>>(yb, M, K, r);
  return cudaGetLastError();
}

}  // namespace vnb
