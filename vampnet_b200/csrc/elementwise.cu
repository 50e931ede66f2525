// vampnet_b200 — HBM-bound helper kernels of the forward pass: the codebook-embedding gather (A operand of the
// out_proj contraction) and the (B,C,T) int64 <-> (B,T,C) int32 state conversions of generate().
#include "common.cuh"
#include "kernels.h"

namespace vnb {

// ------------------------------------------------------------------------------------------------
// CodebookEmbedding.from_codes (reference vampnet/modules/layers.py:134-156) as the A operand of the out_proj
// contraction (:162), which runs on the tensor cores (gemm_wgmma_kernel<BIAS_F32>, api.cu):
//   latent[m, c*8 + j] = table[c][code[m, c]][j]        (code == V selects the learned MASK row)
//   A[m, :] = [ hi(latent) | hi(latent) | lo(latent) ]   bf16, each third zero-padded to Kp columns
// so that A . [w_hi | w_lo | w_hi]^T = latent . w to fp32 accuracy (split-bf16: hi = bf16(v), lo = bf16(v - hi)).
// HBM-bound: reads M*C codes + table rows (L2-resident), writes M * 3*Kp bf16.  Also zeroes the row-sum-of-squares
// partials [zero_from, ss_parts) that the GEMM epilogue (which writes d/256 of them) does not cover.
template <bool FROM_CODES>
__global__ void __launch_bounds__(256) embed_gather_kernel(const int32_t* __restrict__ codes, const float* __restrict__ lat_in,
                                                           const float* __restrict__ table, __nv_bfloat16* __restrict__ A,
                                                           int M, int T, int C, int V1, int K, int Kp,
                                                           float* __restrict__ ss, int zero_from, int ss_parts,
                                                           const int32_t* __restrict__ live) {
  // rows at or past live[0] * T belong to idle calls (a launch of calls with different step counts): not touched
  const int m_live = live != nullptr ? min(M, __ldg(live) * T) : M;
  const long long total = static_cast<long long>(m_live) * Kp;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int m = static_cast<int>(i / Kp), k = static_cast<int>(i - static_cast<long long>(m) * Kp);
    float v = 0.f;
    if (k < K) {
      if constexpr (FROM_CODES) {
        const int c = k >> 3, j = k & 7;
        const int code = codes[static_cast<size_t>(m) * C + c];
        v = __ldg(table + (static_cast<size_t>(c) * V1 + code) * 8 + j);
      } else {
        const int b = m / T, t = m - b * T;  // latents (B, K, T)
        v = lat_in[(static_cast<size_t>(b) * K + k) * T + t];
      }
    }
    const __nv_bfloat16 hi = __float2bfloat16_rn(v);
    const __nv_bfloat16 lo = __float2bfloat16_rn(v - __bfloat162float(hi));
    __nv_bfloat16* row = A + static_cast<size_t>(m) * 3 * Kp;
    row[k] = hi;
    row[Kp + k] = hi;
    row[2 * Kp + k] = lo;
    if (ss != nullptr && k < ss_parts - zero_from) ss[static_cast<size_t>(zero_from + k) * M + m] = 0.f;
  }
}

cudaError_t launch_embed_gather(const int32_t* codes_btc, const float* latents, const float* table, void* A, int M, int T,
                                int C, int V1, int K, int Kp, float* ss, int zero_from, int ss_parts,
                                const int32_t* live, cudaStream_t st) {
  if (K > Kp || ss_parts - zero_from > Kp) return cudaErrorInvalidValue;
  const long long total = static_cast<long long>(M) * Kp;
  long long blocks = (total + 255) / 256;
  const long long cap = 16LL * device_sm_count();
  if (blocks > cap) blocks = cap;
  if (codes_btc != nullptr)
    embed_gather_kernel<true><<<static_cast<unsigned>(blocks), 256, 0, st>>>(codes_btc, nullptr, table,
                                                                             reinterpret_cast<__nv_bfloat16*>(A), M, T, C, V1, K,
                                                                             Kp, ss, zero_from, ss_parts, live);
  else
    embed_gather_kernel<false><<<static_cast<unsigned>(blocks), 256, 0, st>>>(nullptr, latents, nullptr,
                                                                              reinterpret_cast<__nv_bfloat16*>(A), M, T, C, V1,
                                                                              K, Kp, ss, zero_from, ss_parts, live);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// generate() set-up (reference transformer.py:749-766): z_masked = z.masked_fill(mask, MASK);
// N0 = count(z_masked == MASK) over the WHOLE batch of one generate() call, i.e. per row group of a launch.  State is
// kept as (B, T, C) int32 so that the codes of one frame are contiguous for the embedding gather and "b (t c)"
// flattening (util.py:39) of the predicted codebooks is a plain stride.  blockIdx.y is the batch row, so each block's
// count belongs to one group.
__global__ void gen_init_kernel(const int64_t* __restrict__ z, const int32_t* __restrict__ mask,
                                int32_t* __restrict__ zcur, int32_t* __restrict__ zorig, int32_t* __restrict__ n0,
                                const RowGroup* __restrict__ rowgrp, int C, int T, int ncc, int mask_token) {
  const int b = blockIdx.y;
  const int per_row = C * T;
  const size_t base = static_cast<size_t>(b) * per_row;
  int local = 0;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < per_row; i += gridDim.x * blockDim.x) {
    const int t = i % T;
    const int c = i / T;
    const int v = static_cast<int>(z[base + i]);
    const int mk = mask ? mask[base + i] : (c >= ncc ? 1 : 0);  // default mask, transformer.py:749-751
    const int vm = mk ? mask_token : v;
    const size_t o = (static_cast<size_t>(b) * T + t) * C + c;
    zorig[o] = v;
    zcur[o] = vm;
    local += (vm == mask_token);
  }
  // block reduce then one atomic
  __shared__ int sh[32];
  for (int o = 16; o > 0; o >>= 1) local += __shfl_xor_sync(0xffffffffu, local, o);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = local;
  __syncthreads();
  if (threadIdx.x < 32) {
    int v = threadIdx.x < (blockDim.x >> 5) ? sh[threadIdx.x] : 0;
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (threadIdx.x == 0 && v) atomicAdd(n0 + (rowgrp ? rowgrp[b].group : 0), v);
  }
}

cudaError_t launch_gen_init(const int64_t* z, const int32_t* mask, int32_t* zcur, int32_t* zorig, int32_t* n0,
                            const RowGroup* rowgrp, int n_groups, int B, int C, int T, int ncc, int mask_token,
                            cudaStream_t st) {
  if (B > 65535) return cudaErrorInvalidValue;  // grid y
  cudaError_t e = cudaMemsetAsync(n0, 0, sizeof(int32_t) * n_groups, st);
  if (e != cudaSuccess) return e;
  int gx = (C * T + 255) / 256;
  const int cap = (1184 + B - 1) / B;  // about as many blocks in all as a grid-stride launch of 1184
  if (gx > cap) gx = cap;
  gen_init_kernel<<<dim3(gx, B), 256, 0, st>>>(z, mask, zcur, zorig, n0, rowgrp, C, T, ncc, mask_token);
  return cudaGetLastError();
}

// sampled_z (B, T, Cp) + conditioning codebooks of the ORIGINAL z -> (B, C, T) int64 (transformer.py:935-938)
__global__ void gen_finish_kernel(const int32_t* __restrict__ tokens, const int32_t* __restrict__ zorig,
                                  int64_t* __restrict__ out, int B, int C, int T, int ncc) {
  const int total = B * C * T;
  const int Cp = C - ncc;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int t = i % T;
    const int c = (i / T) % C;
    const int b = i / (T * C);
    const size_t bt = static_cast<size_t>(b) * T + t;
    out[i] = c < ncc ? zorig[bt * C + c] : tokens[bt * Cp + (c - ncc)];
  }
}
cudaError_t launch_gen_finish(const int32_t* tokens, const int32_t* zorig, int64_t* out, int B, int C, int T, int ncc,
                              cudaStream_t st) {
  const int total = B * C * T;
  int grid = (total + 255) / 256;
  if (grid > 1184) grid = 1184;
  gen_finish_kernel<<<grid, 256, 0, st>>>(tokens, zorig, out, B, C, T, ncc);
  return cudaGetLastError();
}

}  // namespace vnb
