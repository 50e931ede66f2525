// vampnet_b200 — fused bidirectional self-attention with T5-style relative-position bias on the sm_90a tensor cores.
//
// Replaces MultiHeadRelativeAttention.forward between the projections (reference vampnet/modules/transformer.py:234-254):
// scores = q.k^T / sqrt(64) + bias[h, k - q]; softmax over keys; out = P.v; heads merged as "b l (head v)".  The
// reference materialises (H,B,T,T) scores in HBM three times per layer; here they live only in registers.  The
// position bias (compute_bias, :183-209) is Toeplitz in (k - q) and saturates beyond |k - q| >= sat, so it is a
// (2*sat+1)-entry table per head held in shared memory.
//
// One CTA = (batch, head, 128 queries), 64-key blocks, two CTAs per SM:
//   warp 8      TMA producer: Q once; K_j and V^T_j through a 3-stage ring
//   warps 0..7  two consumer warpgroups, 64 query rows each.  Per key block: S = Q.K_j^T (wgmma, both operands in shared
//               memory, 32 fp32 scores per thread) -> bias: one table value for a block wholly beyond +-sat from
//               the warp's rows, else an unclamped lookup in an edge-padded table; the key < len mask only in a ragged
//               last block -> online softmax in registers (exp2 domain; a row's four threads
//               exchange maxima and sums by shuffles) -> P packed to bf16 in registers, which is exactly the A-operand
//               fragment of the next wgmma -> O += P.V_j (wgmma with A from registers, B = V^T_j in shared memory).
//               O (64 x 64 fp32) stays in registers for the whole key loop.
#include <stdlib.h>

#include "common.cuh"
#include "kernels.h"
#include "wgmma.cuh"

namespace vnb {
namespace att {

constexpr int AQ = 128, AK = 64, DH = 64, KV_STAGES = 3;
constexpr int Q_BYTES = AQ * DH * 2;        // 16 KiB
constexpr int K_BYTES = AK * DH * 2;        // 8 KiB
constexpr int V_BYTES = DH * AK * 2;        // 8 KiB
constexpr int MAX_SAT = 128;
constexpr int PAD = 80;                     // edge copies on each side of the table: >= one key block + a warp's rows
constexpr int TAB = 2 * MAX_SAT + 1 + 2 * PAD;
constexpr int THREADS = 256 + 32;
constexpr float LOG2E = 1.4426950408889634f;

// shared-memory map, byte offsets from the base aligned up to 1024 bytes inside the allocation
constexpr uint32_t OFF_Q = 0;
constexpr uint32_t OFF_K = OFF_Q + Q_BYTES;
constexpr uint32_t OFF_V = OFF_K + KV_STAGES * K_BYTES;
constexpr uint32_t OFF_BIAS = OFF_V + KV_STAGES * V_BYTES;
constexpr uint32_t OFF_BAR = (OFF_BIAS + TAB * 4 + 7) & ~7u;
constexpr uint32_t BAR_Q_FULL = OFF_BAR;
constexpr uint32_t BAR_KV_FULL = OFF_BAR + 8;                      // [KV_STAGES]
constexpr uint32_t BAR_KV_EMPTY = BAR_KV_FULL + 8 * KV_STAGES;     // [KV_STAGES]
constexpr int SMEM = BAR_KV_EMPTY + 8 * KV_STAGES + 1024;  // + slack for aligning the base to 1024

struct Args {
  __nv_bfloat16* out;
  const float* rel;
  const int32_t* frames;  // (B) key length of every batch row, null: every row has T
  const int32_t* live;    // (1) batch rows b >= live[0] are idle this iteration, null: every row is live
  int sat, B, T, H, d;
};

__global__ void __launch_bounds__(THREADS, 2)
attention_wgmma_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                       const __grid_constant__ CUtensorMap tmVT, const Args a) {
  extern __shared__ uint8_t smem[];
  const uint32_t sb = (smem_u32(smem) + 1023u) & ~1023u;   // 128B-swizzled tiles need the 1024-byte alignment

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * AQ;
  const int h = blockIdx.y;
  const int b = blockIdx.z;
  if (a.live != nullptr && b >= __ldg(a.live)) return;  // an idle row: the whole CTA, before any barrier or TMA work
  // this batch row's own length: keys, queries and stores stop there (rows of a shorter call in a longer launch)
  const int len = a.frames != nullptr ? __ldg(a.frames + b) : a.T;
  if (q0 >= len) return;  // the whole CTA, before any barrier or TMA work
  const int nblk = (len + AK - 1) / AK;
  const int sat = a.sat;

  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmK);
    tma_prefetch_desc(&tmVT);
    mbar_init_a(sb + BAR_Q_FULL, 1);
    for (int s = 0; s < KV_STAGES; ++s) {
      mbar_init_a(sb + BAR_KV_FULL + 8 * s, 1);
      mbar_init_a(sb + BAR_KV_EMPTY + 8 * s, 8);  // lane 0 of every consumer warp
    }
    mbar_fence_init();
  }
  // bias table of this head, times log2(e): entry [rel + sat + PAD] for rel in [-sat - PAD, sat + PAD], clamped
  for (int i = threadIdx.x; i <= 2 * (sat + PAD); i += THREADS) {
    const int e = min(max(i - PAD, 0), 2 * sat);
    sts_f32(sb + OFF_BIAS + 4u * i, a.rel[e * a.H + h] * LOG2E);
  }
  __syncthreads();

  if (warp == 8) {
    // ===================== TMA producer =====================
    if (lane == 0) {
      mbar_expect_tx_a(sb + BAR_Q_FULL, Q_BYTES);
      tma_load_3d_a(sb + OFF_Q, &tmQ, sb + BAR_Q_FULL, h * DH, q0, b);
      for (int j = 0; j < nblk; ++j) {
        const int st = j % KV_STAGES;
        const uint32_t ph = (j / KV_STAGES) & 1;
        mbar_wait_a(sb + BAR_KV_EMPTY + 8 * st, ph ^ 1);
        mbar_expect_tx_a(sb + BAR_KV_FULL + 8 * st, K_BYTES + V_BYTES);
        tma_load_3d_a(sb + OFF_K + st * K_BYTES, &tmK, sb + BAR_KV_FULL + 8 * st, a.d + h * DH, j * AK, b);
        tma_load_3d_a(sb + OFF_V + st * V_BYTES, &tmVT, sb + BAR_KV_FULL + 8 * st, j * AK, h * DH, b);
      }
    }
    return;
  }

  // ===================== consumers =====================
  // Accumulator fragment of m64nNk16: thread (warp w of the warpgroup, lane l) holds rows 16 w + l/4 (regs 4i, 4i+1)
  // and 16 w + l/4 + 8 (regs 4i+2, 4i+3), columns 8 i + 2 (l % 4) + {0, 1}.
  const int wg = warp >> 2;
  const int qw = q0 + wg * 64 + (warp & 3) * 16;                // first query row of this warp
  const int qr = qw + (lane >> 2);                               // query of this thread's first row (second: qr + 8)
  const int kc = 2 * (lane & 3);                                 // first key column of this thread inside an n8 block
  const uint32_t sQ = sb + OFF_Q + wg * (64 * 128);
  const float c = 0.125f * LOG2E;                                // 1/sqrt(64) folded with log2(e)
  const bool ragged = (len % AK) != 0;
  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};        // running max / this thread's share of the row sum

  mbar_wait_a(sb + BAR_Q_FULL, 0);
  for (int j = 0; j < nblk; ++j) {
    const int st = j % KV_STAGES;
    mbar_wait_a(sb + BAR_KV_FULL + 8 * st, (j / KV_STAGES) & 1);
    const uint32_t sK = sb + OFF_K + st * K_BYTES, sV = sb + OFF_V + st * V_BYTES;
    float s[32];
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < DH / 16; ++k)
      wgmma_ss_n64(s, wgmma_desc_sw128(sQ + k * 32), wgmma_desc_sw128(sK + k * 32), k != 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(s);

    // t = score * c + bias[clamp(k - q)] (log2 domain); keys beyond T -> -inf.  A warp's 16 rows against a 64-key
    // block span k - q in [lo, lo + 78]: wholly at or beyond -sat or +sat the bias is one table entry; otherwise the
    // index k - q + sat + PAD stays inside the edge-padded table and needs no clamp.
    const int lo = j * AK - qw - 15;
    if (ragged && j == nblk - 1) {
#pragma unroll
      for (int i = 0; i < 8; ++i) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int key = j * AK + 8 * i + kc + e;
#pragma unroll
          for (int r = 0; r < 2; ++r) {
            int rel = key - (qr + 8 * r);
            rel = rel < -sat ? -sat : (rel > sat ? sat : rel);
            float t = __fmaf_rn(s[4 * i + 2 * r + e], c, lds_f32(sb + OFF_BIAS + 4u * (rel + sat + PAD)));
            if (key >= len) t = -INFINITY;
            s[4 * i + 2 * r + e] = t;
          }
        }
      }
    } else if (lo + 78 <= -sat || lo >= sat) {
      const float bc = lds_f32(sb + OFF_BIAS + 4u * (lo >= sat ? 2 * sat + PAD : PAD));  // bias[+-sat]
#pragma unroll
      for (int i = 0; i < 32; ++i) s[i] = __fmaf_rn(s[i], c, bc);
    } else {
      const uint32_t tb = sb + OFF_BIAS + 4u * (j * AK + kc - qr + sat + PAD);
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int e = 0; e < 2; ++e)
#pragma unroll
          for (int r = 0; r < 2; ++r)
            s[4 * i + 2 * r + e] = __fmaf_rn(s[4 * i + 2 * r + e], c, lds_f32(tb + 4 * (8 * i + e - 8 * r)));
    }
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      mx[0] = fmaxf(mx[0], fmaxf(s[4 * i], s[4 * i + 1]));
      mx[1] = fmaxf(mx[1], fmaxf(s[4 * i + 2], s[4 * i + 3]));
    }
    float alpha[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
      const float m_new = fmaxf(m[r], mx[r]);      // finite: every block has a key < len
      alpha[r] = fast_exp2(m[r] - m_new);          // 0 on the first block
      m[r] = m_new;
      l[r] *= alpha[r];
    }
    // P = exp2(t - m), in place
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      s[4 * i] = fast_exp2(s[4 * i] - m[0]); s[4 * i + 1] = fast_exp2(s[4 * i + 1] - m[0]);
      s[4 * i + 2] = fast_exp2(s[4 * i + 2] - m[1]); s[4 * i + 3] = fast_exp2(s[4 * i + 3] - m[1]);
      l[0] += s[4 * i] + s[4 * i + 1];
      l[1] += s[4 * i + 2] + s[4 * i + 3];
    }
    // P packed as bf16 pairs: key chunk kk (16 keys) = n8 blocks 2kk, 2kk+1 = the A fragment of k-step kk
    uint32_t p[4][4];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      p[i >> 1][(i & 1) * 2] = pack_bf16x2(s[4 * i], s[4 * i + 1]);
      p[i >> 1][(i & 1) * 2 + 1] = pack_bf16x2(s[4 * i + 2], s[4 * i + 3]);
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      o[4 * i] *= alpha[0]; o[4 * i + 1] *= alpha[0];
      o[4 * i + 2] *= alpha[1]; o[4 * i + 3] *= alpha[1];
    }
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < AK / 16; ++kk) wgmma_rs_n64(o, p[kk], wgmma_desc_sw128(sV + kk * 32), 1u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(o);
    __syncwarp();
    if (lane == 0) mbar_arrive_a(sb + BAR_KV_EMPTY + 8 * st);
  }

  // ---- finalize: O / l -> bf16 -> (B, T, d) at [b, q, h*64 + col]
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    l[r] += __shfl_xor_sync(0xffffffffu, l[r], 1);
    l[r] += __shfl_xor_sync(0xffffffffu, l[r], 2);
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int q = qr + 8 * r;
    if (q < len) {
      const float inv_l = 1.0f / l[r];
      uint32_t* orow = reinterpret_cast<uint32_t*>(a.out + (static_cast<size_t>(b) * a.T + q) * a.d + h * DH + kc);
#pragma unroll
      for (int i = 0; i < 8; ++i) orow[4 * i] = pack_bf16x2(o[4 * i + 2 * r] * inv_l, o[4 * i + 2 * r + 1] * inv_l);
    }
  }
}

}  // namespace att

cudaError_t launch_attention(const AttnPlan& p, cudaStream_t st) {
  static PerDeviceOnce once;
  int dev;
  if (once.need(&dev)) {
    cudaError_t e = cudaFuncSetAttribute(att::attention_wgmma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, att::SMEM);
    if (e != cudaSuccess) return e;
    once.mark(dev);
  }
  if (p.sat > att::MAX_SAT || p.sat < 1) return cudaErrorInvalidValue;
  att::Args a;
  a.out = reinterpret_cast<__nv_bfloat16*>(p.out);
  a.rel = p.rel;
  a.frames = p.frames;
  a.live = p.live;
  a.sat = p.sat; a.B = p.B; a.T = p.T; a.H = p.H; a.d = p.H * att::DH;
  dim3 grid((p.T + att::AQ - 1) / att::AQ, p.H, p.B);
  att::attention_wgmma_kernel<<<grid, att::THREADS, att::SMEM, st>>>(p.tmQ, p.tmK, p.tmVT, a);
  return cudaGetLastError();
}

}  // namespace vnb
