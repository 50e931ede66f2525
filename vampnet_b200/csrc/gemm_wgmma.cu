// vampnet_b200 — bf16 GEMM on the sm_90a tensor cores (wgmma, register accumulators, TMA operands).
//
//   out = epilogue( A (M,K) row-major bf16  x  W (N,K)^T row-major bf16 ),  fp32 accumulation
//
// One kernel family covers every dense contraction of VampNet.forward (reference
// vampnet/modules/transformer.py): QKV projection (:229-231), attention output projection (:255),
// FFN up-projection with the GatedGELU fused (:81-83, activations.py:16-35), FFN down-projection
// with the residual add fused (:84, :367), the classifier (:632) and, in the generate loop, the classifier with
// sample_from_logits (:952-1034) fused into its epilogue (EPI_SAMPLE), and the embedding out_proj (layers.py:162).
//
// Structure (one 128 x 256 output tile per CTA; option: clusters of two CTAs on vertically adjacent tiles that share
// the W tile, see the note above the kernel):
//   warp 8       TMA producer   : 4-stage ring of {A 128x64, W 256x64} bf16 tiles, 128B-swizzled
//   warps 0..7   two consumer warpgroups: wgmma m64n256k16, rows [64 wg, 64 wg + 64) of the tile, 128 fp32
//                accumulators per thread; then the epilogue: the accumulators go to a padded fp32 tile that overlays the
//                drained ring, and each epilogue warp reads 32 x 32 chunks of it in store order -> fused op -> global
//                (4 warps; 8 for the residual and the sampling epilogues)
//
// Roofline: tensor-bound.  Algorithmic work = 2*M*N*K flop per launch; bytes (A+W+out) are a few
// MB against > 10 GFLOP, far right of the ridge.
#include <stdlib.h>

#include "common.cuh"
#include "kernels.h"
#include "wgmma.cuh"

#ifndef VNB_GEMM_PAIR_DEFAULT
#define VNB_GEMM_PAIR_DEFAULT false
#endif

namespace vnb {

constexpr int BM = 128, BN = 256, BK = 64, STAGES = 4;
constexpr int A_BYTES = BM * BK * 2;  // 16 KiB
constexpr int B_BYTES = BN * BK * 2;  // 32 KiB
constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
constexpr int SBIAS_BYTES = BN * 4;                // EPI_SAMPLE: the tile's bias in shared memory
constexpr int RING_BYTES = STAGES * STAGE_BYTES;  // 192 KiB
constexpr int ACC_PITCH = BN + 1;                 // fp32 accumulator tile: odd pitch, every epilogue read is conflict-free
static_assert(BM * ACC_PITCH * 4 <= RING_BYTES, "the accumulator tile overlays the ring");
static_assert(BM * ACC_PITCH * 4 + 4 * BM + 16 + 32 * BM <= RING_BYTES, "the adapted epilogue's row table follows it");
constexpr int GEMM_SMEM = RING_BYTES + SBIAS_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;
static_assert(GEMM_SMEM <= 227 * 1024, "H100: at most 227 KiB of shared memory per block");
constexpr int GEMM_THREADS = 256 + 32;            // two consumer warpgroups + the producer warp
// The residual epilogue is bound by memory-level parallelism (residual rows must be fetched before they can be
// updated): it gets 8 epilogue warps, two per 32-row quadrant of the tile, splitting the 32-column chunks even / odd.
template <int EPI> constexpr int gemm_epi_warps() { return (EPI == VNB_EPI_RESID || EPI == VNB_EPI_SAMPLE) ? 8 : 4; }

struct GemmArgs {
  int M, N, K;
  int epi;
  void* out;          // see VNB_EPI_*
  void* out2;         // vT for EPI_QKV
  const float* bias;  // EPI_BIAS_F32
  int T, Tpad;        // EPI_QKV: rows m = b*T + t
  int d2;             // EPI_QKV: 2*d_model (column where V starts)
  // ---- fused RMSNorm (reference transformer.py:43-58), see DESIGN.md §4 ----
  __nv_bfloat16* out_bf16;  // EPI_RESID / EPI_BIAS_F32: bf16 copy of the fp32 output (A operand of the next GEMM)
  float* ss_out;            // partial row sums of squares of the fp32 output, part p at [p * M + row]: EPI_RESID
                            // (N/128, M), parts 2j / 2j+1 = even / odd 32-column chunks of n-tile j; EPI_BIAS_F32
                            // (N/256, M), one part per n-tile
  const float* ss_in;       // consumers: partial row sums of squares of THEIR A operand; null = no row scaling
  int ss_parts;             // number of partials to add (fixed order: deterministic)
  float inv_d, eps;         // row scale = rsqrt(sum * inv_d + eps)
  // ---- EPI_SAMPLE (see the epilogue) ----
  const int32_t* zcur;
  const SampleDyn* dyn;     // this step's row of the (step, group) table
  const RowGroup* rowgrp;   // (B) group of every batch row
  float4* partials;
  int C, ncc, V, mask_token;
  // ---- adapted variants (ADAPT): per-row LoRA update of the accumulators, see lora_update() ----
  AdapterRefs lora;
};

__device__ __forceinline__ float gelu_tanh(float x) {
  // 0.5*x*(1+tanh(sqrt(2/pi)*(x+0.044715*x^3)))   (activations.py:16-26); tanh(y) = 1 - 2/(1+exp(2y))
  const float y = 0.7978845608028654f * (x + 0.044715f * x * x * x);
  const float e = __expf(2.0f * y);
  const float t = 1.0f - __fdividef(2.0f, 1.0f + e);
  return 0.5f * x * (1.0f + t);
}

// ---- epilogue ---------------------------------------------------------------------------------
// The epilogue reads the fp32 accumulator tile in the order of its global stores, so that a warp instruction covers
// whole rows: 128 contiguous bytes per 8 lanes for fp32 outputs, 64 for bf16 (the odd tile pitch keeps these reads
// bank-conflict free).  `quad` is the shared-space byte address of column 0 of the warp's first row (32-row quadrant);
// `rs` is the row scale (fused RMSNorm of the A operand) of quadrant row `lane`, handed by a shuffle to the lane that
// stores that row.

// Sum of squares of four consecutive outputs, in a fixed operation order (the fused RMSNorm statistics are
// deterministic).
__device__ __forceinline__ float sumsq4(float x, float y, float z, float w) {
  return __fmaf_rn(w, w, __fmaf_rn(z, z, __fmaf_rn(y, y, __fmul_rn(x, x))));
}

// fp32 destinations: lane -> (row = it*4 + lane/8, 4 columns at (lane%8)*4).
// The addend (residual rows or bias) of a chunk is fetched by prefetch_addend() one chunk ahead, so its global-load
// latency overlaps the previous chunk, and all eight loads are in flight before the first store.
template <int EPI>
__device__ __forceinline__ void prefetch_addend(const GemmArgs& g, int lane, int row_base, int col0, float4 (&add)[8]) {
  const int c4 = (lane & 7) * 4;
  const int r0 = row_base + (lane >> 3);
  if constexpr (EPI == VNB_EPI_RESID) {
    const float* base = reinterpret_cast<const float*>(g.out) + static_cast<size_t>(r0) * g.N + col0 + c4;
    const size_t step = static_cast<size_t>(4) * g.N;
#pragma unroll
    for (int it = 0; it < 8; ++it)
      add[it] = (r0 + it * 4 < g.M) ? __ldcg(reinterpret_cast<const float4*>(base + it * step))
                                    : make_float4(0.f, 0.f, 0.f, 0.f);
  } else {
    const float4 b4 = __ldg(reinterpret_cast<const float4*>(g.bias + col0 + c4));
#pragma unroll
    for (int it = 0; it < 8; ++it) add[it] = b4;
  }
}
template <bool FUSED>
__device__ __forceinline__ void drain_f32(const GemmArgs& g, uint32_t quad, float rs, int lane, int row_base, int n0,
                                          int c, const float4 (&add)[8], float (&ssacc)[8]) {
  const int c4 = (lane & 7) * 4;
  const int r0 = row_base + (lane >> 3);
  const int col0 = n0 + c * 32;
  float* const base = reinterpret_cast<float*>(g.out) + static_cast<size_t>(r0) * g.N + col0 + c4;
  const size_t step = static_cast<size_t>(4) * g.N;
#pragma unroll
  for (int it = 0; it < 8; ++it) {
    const int r = it * 4 + (lane >> 3);
    const float rsr = __shfl_sync(0xffffffffu, rs, r);  // rs == 1 unless a norm is fused in
    const uint32_t sp = quad + 4u * (r * ACC_PITCH + c * 32 + c4);
    float4 a = make_float4(__fmul_rn(lds_f32(sp), rsr), __fmul_rn(lds_f32(sp + 4), rsr), __fmul_rn(lds_f32(sp + 8), rsr),
                           __fmul_rn(lds_f32(sp + 12), rsr));
    a.x = __fadd_rn(a.x, add[it].x); a.y = __fadd_rn(a.y, add[it].y);
    a.z = __fadd_rn(a.z, add[it].z); a.w = __fadd_rn(a.w, add[it].w);
    if (r0 + it * 4 < g.M) {
      *reinterpret_cast<float4*>(base + it * step) = a;
      if constexpr (FUSED) {
        uint2 w;
        w.x = pack_bf16x2(a.x, a.y);
        w.y = pack_bf16x2(a.z, a.w);
        *reinterpret_cast<uint2*>(g.out_bf16 + static_cast<size_t>(r0 + it * 4) * g.N + col0 + c4) = w;
        ssacc[it] = __fadd_rn(ssacc[it], sumsq4(a.x, a.y, a.z, a.w));
      }
    }
  }
}

// bf16 destinations: lane -> (row = it*8 + lane/4, 8 columns at (lane%4)*8) of tile columns [tc, tc + 32), stored at
// output columns [oc, oc + 32) with output row pitch `pitch`.  GEGLU: value * gelu_tanh(gate), the gate 128 tile
// columns to the right of its value.
template <bool GEGLU>
__device__ __forceinline__ void drain_bf16(__nv_bfloat16* out, int pitch, int M, uint32_t quad, float rs, int lane,
                                           int row_base, int tc, int oc) {
  const int c8 = (lane & 3) * 8;
#pragma unroll
  for (int it = 0; it < 4; ++it) {
    const int r = it * 8 + (lane >> 2);
    const float rsr = __shfl_sync(0xffffffffu, rs, r);
    const uint32_t sp = quad + 4u * (r * ACC_PITCH + tc + c8);
    float x[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      x[k] = lds_f32(sp + 4u * k) * rsr;
      if constexpr (GEGLU) x[k] = x[k] * gelu_tanh(lds_f32(sp + 4u * (128 + k)) * rsr);
    }
    const int row = row_base + r;
    if (row < M) {
      uint4 w;
      w.x = pack_bf16x2(x[0], x[1]);
      w.y = pack_bf16x2(x[2], x[3]);
      w.z = pack_bf16x2(x[4], x[5]);
      w.w = pack_bf16x2(x[6], x[7]);
      *reinterpret_cast<uint4*>(out + static_cast<size_t>(row) * pitch + oc + c8) = w;
    }
  }
}

// 32 consecutive fp32 columns of one accumulator-tile row (byte address `addr` of the first)
__device__ __forceinline__ void acc_ld_x32(uint32_t addr, uint32_t (&v)[32]) {
#pragma unroll
  for (int j = 0; j < 32; ++j) v[j] = __float_as_uint(lds_f32(addr + 4u * j));
}

// LoRA update of the accumulator tile (adapted variants only; DESIGN.md §1): for every adapted row m of the tile and
// every column n, acc[m][n] += sum_k u[m][k] * B'[n][k], k = 0..7 in a fixed fma chain, added before anything the
// epilogue does (row scale, rounding, GEGLU, residual).  Base rows (adapter -1) are skipped, not updated by zero.  The
// arithmetic of a row depends only on its own u and its adapter's B', never on which rows share its tile.
// The adapter and the u of every tile row are staged once in `scratch` (free shared memory past the accumulator tile).
// Then, per adapter present in the tile, thread t keeps B' of its four columns (t % 64) + 64 j in registers and updates
// them in the rows (t / 64) + 4 i of that adapter: a warp covers 32 consecutive columns of one row (conflict-free), and
// the row's u is a broadcast shared-memory read.
template <int EPI>
__device__ __forceinline__ void lora_update(const GemmArgs& g, uint8_t* scratch, uint32_t acc_tile, int m0, int n0) {
  int uoff = 0, brow0 = n0;
  if constexpr (EPI == VNB_EPI_QKV) {
    // columns [0, d) q, [d, 2d) k (w_ks has no LoRA: no update), [2d, 3d) v; a 256-column tile lies in one of them
    const int d = g.N / 3;
    if (n0 >= d && n0 < 2 * d) return;
    if (n0 >= 2 * d) { uoff = 8; brow0 = n0 - d; }
  }
  const AdapterRefs& L = g.lora;
  const int t = static_cast<int>(threadIdx.x);
  int32_t* sid = reinterpret_cast<int32_t*>(scratch);               // adapter of tile row r (-1: base, or past M)
  uint32_t* smask = reinterpret_cast<uint32_t*>(scratch + 4 * BM);  // adapters present among the rows of warps 0..3
  float4* su = reinterpret_cast<float4*>(scratch + 4 * BM + 16);     // u of tile row r: su[2 r], su[2 r + 1]
  constexpr int R = EPI == VNB_EPI_QKV ? 16 : 8;
  if (t < BM) {
    const int m = m0 + t;
    const int id = m < g.M ? L.grp_adapter[L.rowgrp[m / L.rows_per_grp].group] : -1;
    sid[t] = id;
    if (id >= 0) {
      su[2 * t] = __ldg(reinterpret_cast<const float4*>(L.u + static_cast<size_t>(m) * R + uoff));
      su[2 * t + 1] = __ldg(reinterpret_cast<const float4*>(L.u + static_cast<size_t>(m) * R + uoff + 4));
    }
    uint32_t bits = 0;
    for (int a = 0; a < VNB_MAX_ADAPTERS; ++a) bits |= __ballot_sync(0xffffffffu, id == a) ? (1u << a) : 0u;
    if ((t & 31) == 0) smask[t >> 5] = bits;
  }
  asm volatile("bar.sync 1, 256;" ::: "memory");
  const uint32_t present = smask[0] | smask[1] | smask[2] | smask[3];
  const int nb = EPI == VNB_EPI_QKV ? 2 * (g.N / 3) : g.N;  // rows of B' per layer
  const int c0 = t & 63, rq = t >> 6;
  for (int a = 0; a < VNB_MAX_ADAPTERS; ++a) {
    if (!((present >> a) & 1u)) continue;
    const float* bp = L.table[a].b[L.slot] + (static_cast<size_t>(L.layer) * nb + brow0 + c0) * 8;
    float4 b0[4], b1[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      b0[j] = __ldg(reinterpret_cast<const float4*>(bp + 64 * 8 * j));
      b1[j] = __ldg(reinterpret_cast<const float4*>(bp + 64 * 8 * j + 4));
    }
#pragma unroll 4
    for (int i = 0; i < BM / 4; ++i) {
      const int r = rq + 4 * i;
      if (sid[r] != a) continue;
      const float4 ua = su[2 * r], ub = su[2 * r + 1];
      const uint32_t row_addr = acc_tile + 4u * (r * ACC_PITCH + c0);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float s = __fmul_rn(ua.x, b0[j].x);
        s = __fmaf_rn(ua.y, b0[j].y, s); s = __fmaf_rn(ua.z, b0[j].z, s); s = __fmaf_rn(ua.w, b0[j].w, s);
        s = __fmaf_rn(ub.x, b1[j].x, s); s = __fmaf_rn(ub.y, b1[j].y, s); s = __fmaf_rn(ub.z, b1[j].z, s);
        s = __fmaf_rn(ub.w, b1[j].w, s);
        const uint32_t addr = row_addr + 4u * (64 * j);
        sts_f32(addr, __fadd_rn(lds_f32(addr), s));
      }
    }
  }
}

// PAIR = true: clusters of two CTAs on vertically adjacent 128 x 256 tiles (the same 256 W rows).  Each CTA fetches
// half of the W tile (128 rows) and the TMA multicasts it into both CTAs' shared memory, so per CTA the W bytes pulled
// from L2 are halved; a stage is refilled only when the consumer warps of both CTAs have released it.  Every output
// element sees the same operands in the same K order as in the single-CTA variant: the two are bit-identical.  On an
// H100 the single-CTA kernel is faster (the pair couples the two CTAs' progress and constrains their placement; same-
// box A/B at the default bench workload: 403 vs 333 TFLOP/s for the GEMM family), so it is the default.
template <int EPI, bool PAIR, bool ADAPT = false>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                  const GemmArgs g) {
  extern __shared__ uint8_t smem_raw[];
  // 128B swizzle atoms are 1024 B: align the tile ring to 1024.
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  float* sbias_all = reinterpret_cast<float*>(smem + RING_BYTES);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + RING_BYTES + SBIAS_BYTES);
  uint64_t* empty_bar = full_bar + STAGES;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const uint32_t rank = PAIR ? cluster_ctarank() : 0u;
  const int tile = PAIR ? static_cast<int>(blockIdx.x >> 1) : static_cast<int>(blockIdx.x);
  constexpr int TM = PAIR ? 2 * BM : BM;  // output rows per cluster (per CTA: always BM)
  const int num_n = g.N / BN;
  const int num_kb = g.K / BK;
  // n-fastest rasterisation: the N/256 tiles that share an A row-block run concurrently, so A is fetched from HBM once
  // (the weights, <= 13 MB, stay L2-resident)
  const int m0 = (tile / num_n) * TM + static_cast<int>(rank) * BM;
  const int n0 = (tile % num_n) * BN;

  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 8 * (PAIR ? 2 : 1));  // lane 0 of every consumer warp (of both CTAs in a pair)
    }
    mbar_fence_init();
  }
  if constexpr (PAIR) cluster_sync_all();  // the peer's barriers must be initialised before anything signals them
  else __syncthreads();

  if (warp == 8) {
    // ===================== TMA producer =====================
    if (lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int kb = 0; kb < num_kb; ++kb) {
        if constexpr (PAIR) mbar_wait_cluster(&empty_bar[stage], phase ^ 1);
        else mbar_wait(&empty_bar[stage], phase ^ 1);
        uint8_t* sa = smem + stage * STAGE_BYTES;
        uint8_t* sb = sa + A_BYTES;
        mbar_expect_tx(&full_bar[stage], STAGE_BYTES);  // A + the whole W tile (pair: one half from each CTA)
        tma_load_2d(sa, &tmA, &full_bar[stage], kb * BK, m0);
        if constexpr (PAIR)
          tma_load_2d_mc(sb + rank * (B_BYTES / 2), &tmB, &full_bar[stage], kb * BK, n0 + static_cast<int>(rank) * (BN / 2),
                         uint16_t(3));
        else
          tma_load_2d(sb, &tmB, &full_bar[stage], kb * BK, n0);
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
    }
    __syncwarp();
  } else {
    // ===================== consumers: mainloop =====================
    const int wg = warp >> 2;
    {
      float acc[128];
#pragma unroll
      for (int i = 0; i < 128; ++i) acc[i] = 0.f;
      const uint32_t peer_empty = PAIR ? mapa_u32(smem_u32(empty_bar), rank ^ 1u) : 0u;
      auto release = [&](int s) {
        if (lane == 0) {
          mbar_arrive(&empty_bar[s]);
          if constexpr (PAIR) mbar_arrive_cluster(peer_empty + 8u * s);
        }
      };
      int stage = 0;
      uint32_t phase = 0;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t sa = smem_u32(smem + stage * STAGE_BYTES) + wg * (64 * 128);
        const uint32_t sb = smem_u32(smem + stage * STAGE_BYTES + A_BYTES);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / 16; ++k)  // advance 16 bf16 = 32 B along K inside the 128B swizzle span
          wgmma_ss_n256(acc, wgmma_desc_sw128(sa + k * 32), wgmma_desc_sw128(sb + k * 32), 1u);
        wgmma_commit();
        wgmma_wait<1>();  // the previous k-block's MMAs have retired: its stage can be refilled
        wgmma_fence_regs(acc);
        if (kb > 0) release(stage == 0 ? STAGES - 1 : stage - 1);
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      wgmma_fence_regs(acc);
      if (num_kb > 0) release(stage == 0 ? STAGES - 1 : stage - 1);
      // both warpgroups are done reading the ring (every TMA write into it has landed: all full barriers were waited
      // on); the accumulators go to the fp32 tile that overlays it.  Fragment of m64nNk16: thread (warp w, lane l)
      // holds rows 16 w + l/4 and + 8, columns 8 i + 2 (l % 4) + {0, 1}.
      asm volatile("bar.sync 1, 256;" ::: "memory");
      const uint32_t acc_tile = smem_u32(smem);
      const int r = wg * 64 + (warp & 3) * 16 + (lane >> 2);
      const uint32_t p0 = acc_tile + 4u * (r * ACC_PITCH + 2 * (lane & 3));
#pragma unroll
      for (int i = 0; i < 32; ++i) {
        sts_f32(p0 + 32u * i, acc[4 * i]);
        sts_f32(p0 + 32u * i + 4, acc[4 * i + 1]);
        sts_f32(p0 + 4u * (8 * ACC_PITCH) + 32u * i, acc[4 * i + 2]);
        sts_f32(p0 + 4u * (8 * ACC_PITCH) + 32u * i + 4, acc[4 * i + 3]);
      }
      asm volatile("bar.sync 1, 256;" ::: "memory");
      if constexpr (ADAPT) {
        lora_update<EPI>(g, smem + BM * ACC_PITCH * 4, acc_tile, m0, n0);
        asm volatile("bar.sync 1, 256;" ::: "memory");
      }
    }
    // ===================== epilogue =====================
    constexpr bool kWide = gemm_epi_warps<EPI>() == 8;
    if (kWide || warp < 4) {
      const int quad = warp & 3;  // 32-row quadrant of the tile this warp drains
      const int row = m0 + quad * 32 + lane;
      const bool row_ok = row < g.M;
      int b_idx = 0, t_idx = 0;
      if constexpr (EPI == VNB_EPI_QKV || EPI == VNB_EPI_SAMPLE) {
        b_idx = row / g.T;
        t_idx = row - b_idx * g.T;
      }
      const int half = kWide ? (warp >> 2) : 0;  // 8-warp epilogue: this warp takes chunks with (c & 1) == half
      const int row_base = m0 + quad * 32;
      float rs = 1.0f;  // fused RMSNorm of the A operand: rsqrt(mean(x^2) + eps) of this thread's row
      if (g.ss_in != nullptr && row_ok) {
        float t = 0.f;
        for (int p = 0; p < g.ss_parts; ++p) t += __ldg(g.ss_in + static_cast<size_t>(p) * g.M + row);
        rs = rsqrtf(t * g.inv_d + g.eps);
      }
      // this warp's quadrant of the accumulator tile, and this thread's row in it (column c at t_addr + 4 c)
      const uint32_t qaddr = smem_u32(smem) + 4u * (quad * 32 * ACC_PITCH);
      const uint32_t t_addr = qaddr + 4u * (lane * ACC_PITCH);
      if constexpr (EPI == VNB_EPI_GEGLU) {
#pragma unroll 1
        for (int c = 0; c < 4; ++c)
          drain_bf16<true>(reinterpret_cast<__nv_bfloat16*>(g.out), g.N / 2, g.M, qaddr, rs, lane, row_base, c * 32,
                           (n0 >> 1) + c * 32);
      } else if constexpr (EPI == VNB_EPI_SAMPLE) {
        // The classifier of the generate loop (transformer.py:632-634 followed by sample_from_logits, :952-1034): the
        // logits of a still-masked position are consumed where they are produced.  A thread owns one row and one
        // 128-column strip = one 128-entry tile of one codebook's vocabulary; three sweeps over the strip in the
        // accumulator tile: max / arg-max, sum of exp((x - max) / temperature), and the inverse-CDF draw inside the strip
        // with this row's second uniform.  What leaves the SM is 16 bytes per (row, strip); sample_combine_kernel picks
        // the strip with the first uniform.  Same arithmetic for the logit as the materialising epilogue (acc * row
        // scale, + bias), so vnb_forward_* shows exactly what was sampled from.
        constexpr float LOG2E_F = 1.4426950408889634f;
        const int et = static_cast<int>(threadIdx.x);                    // 0..255 over the eight epilogue warps
        const uint32_t sbias = smem_u32(sbias_all);
        sts_f32(sbias + 4u * et, __ldg(g.bias + n0 + et));
        asm volatile("bar.sync 2, 256;" ::: "memory");
        const int strip = warp >> 2;                                     // columns [128 strip, 128 strip + 128) of the tile
        const int col0 = n0 + strip * 128;
        const int cp = col0 / g.V, v0 = col0 - cp * g.V;
        const int Cp = g.C - g.ncc;
        const bool active = row_ok && __ldg(g.zcur + static_cast<size_t>(row) * g.C + g.ncc + cp) == g.mask_token;
        if (__any_sync(0xffffffffu, active)) {
          const uint32_t t_strip = t_addr + 4u * (strip * 128);
          const uint32_t sb4 = sbias + 4u * (strip * 128);
          // this row's generate() call: its temperature, greedy / sampling step and key, and the row's index in it
          const RowGroup rg = g.rowgrp[row_ok ? b_idx : 0];
          const SampleDyn& dyn = g.dyn[rg.group];
          const float inv_temp = dyn.inv_temp;
          const int do_sample = dyn.do_sample;
          // sweep 1: maximum and arg-max (lowest index on ties) of the logits
          float mx = -INFINITY;
          int am = 0;
#pragma unroll 1
          for (int c = 0; c < 4; ++c) {
            uint32_t v[32];
            acc_ld_x32(t_strip + 4u * (c * 32), v);
#pragma unroll
            for (int j4 = 0; j4 < 8; ++j4) {
              const float4 b4 = lds_f4(sb4 + 16u * (c * 8 + j4));
              const float bj[4] = {b4.x, b4.y, b4.z, b4.w};
#pragma unroll
              for (int j = 0; j < 4; ++j) {
                const float x = __fadd_rn(__fmul_rn(__uint_as_float(v[j4 * 4 + j]), rs), bj[j]);
                if (x > mx) { mx = x; am = c * 32 + j4 * 4 + j; }
              }
            }
          }
          // sweep 2: s = sum over the strip of e = 2^((x - mx) * c1), c1 = log2(e) / temperature, in column order
          const float c1 = __fmul_rn(inv_temp, LOG2E_F);
          const float c0 = -__fmul_rn(mx, c1);
          float ssum = 0.f;
#pragma unroll 1
          for (int c = 0; c < 4; ++c) {
            uint32_t v[32];
            acc_ld_x32(t_strip + 4u * (c * 32), v);
#pragma unroll
            for (int j4 = 0; j4 < 8; ++j4) {
              const float4 b4 = lds_f4(sb4 + 16u * (c * 8 + j4));
              const float bj[4] = {b4.x, b4.y, b4.z, b4.w};
#pragma unroll
              for (int j = 0; j < 4; ++j) {
                const float x = __fadd_rn(__fmul_rn(__uint_as_float(v[j4 * 4 + j]), rs), bj[j]);
                ssum += fast_exp2(__fmaf_rn(x, c1, c0));
              }
            }
          }
          // sweep 3 (sampling steps only): first column whose running sum exceeds u2 * s; the arg-max if rounding
          // leaves none.  Greedy steps take the arg-max.
          int cand = am;
          float xc = mx;
          if (do_sample) {
            uint32_t r4[4];
            philox4x32_10(static_cast<uint32_t>(t_idx * Cp + cp), static_cast<uint32_t>(b_idx - rg.first),
                          static_cast<uint32_t>(dyn.step), 0u, dyn.seed_lo, dyn.seed_hi, r4);
            const float target = u01(r4[1]) * ssum;
            float run = 0.f;
            int found = -1;
#pragma unroll 1
            for (int c = 0; c < 4; ++c) {
              uint32_t v[32];
              acc_ld_x32(t_strip + 4u * (c * 32), v);
#pragma unroll
              for (int j4 = 0; j4 < 8; ++j4) {
                const float4 b4 = lds_f4(sb4 + 16u * (c * 8 + j4));
                const float bj[4] = {b4.x, b4.y, b4.z, b4.w};
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                  const float x = __fadd_rn(__fmul_rn(__uint_as_float(v[j4 * 4 + j]), rs), bj[j]);
                  run += fast_exp2(__fmaf_rn(x, c1, c0));
                  if (run > target && found < 0) { found = c * 32 + j4 * 4 + j; xc = x; }
                }
              }
            }
            if (found >= 0) cand = found;
            else xc = mx;
          }
          if (active)
            g.partials[(static_cast<size_t>(row) * Cp + cp) * (g.V >> 7) + (v0 >> 7)] =
                make_float4(mx, ssum, xc, __uint_as_float(static_cast<uint32_t>(v0 + cand) |
                                                          (static_cast<uint32_t>(v0 + am) << 16)));
        }
      } else if constexpr (EPI == VNB_EPI_RESID || EPI == VNB_EPI_BIAS_F32) {
        // software-pipelined: the residual rows of chunk c+1 are in flight while chunk c is read from the accumulator
        // tile and stored (the global-load latency would otherwise be paid 8 times per tile, serially)
        const bool fused_out = g.out_bf16 != nullptr;  // residual GEMMs, and the embedding projection (BIAS_F32)
        constexpr int CSTEP = kWide ? 2 : 1;  // chunks owned by this warp: half, half + CSTEP, ...
        float ssacc[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) ssacc[i] = 0.f;
        auto process = [&](int c, const float4 (&add)[8]) {
          if (fused_out) drain_f32<true>(g, qaddr, rs, lane, row_base, n0, c, add, ssacc);
          else drain_f32<false>(g, qaddr, rs, lane, row_base, n0, c, add, ssacc);
        };
        float4 addA[8], addB[8];
        prefetch_addend<EPI>(g, lane, row_base, n0 + half * 32, addA);
#pragma unroll 1
        for (int c = half; c < BN / 32; c += 2 * CSTEP) {
          prefetch_addend<EPI>(g, lane, row_base, n0 + (c + CSTEP) * 32, addB);
          process(c, addA);
          if (c + 2 * CSTEP < BN / 32) prefetch_addend<EPI>(g, lane, row_base, n0 + (c + 2 * CSTEP) * 32, addA);
          process(c + CSTEP, addB);
        }
        if (fused_out) {
          // per-row sum of squares over this warp's columns of the tile: 8 lanes share a row; fixed reduction order
#pragma unroll
          for (int it = 0; it < 8; ++it) {
            float v = ssacc[it];
            v += __shfl_xor_sync(0xffffffffu, v, 1);
            v += __shfl_xor_sync(0xffffffffu, v, 2);
            v += __shfl_xor_sync(0xffffffffu, v, 4);
            const int rr = row_base + it * 4 + (lane >> 3);
            const int part = (n0 / BN) * (kWide ? 2 : 1) + half;
            if ((lane & 7) == 0 && rr < g.M) g.ss_out[static_cast<size_t>(part) * g.M + rr] = v;
          }
        }
      } else {
#pragma unroll 1
        for (int c = 0; c < BN / 32; ++c) {
          const int col0 = n0 + c * 32;
          if constexpr (EPI == VNB_EPI_QKV) {
            if (col0 >= g.d2) {
              uint32_t v[32];
              acc_ld_x32(t_addr + 4u * (c * 32), v);
              // v : transposed (B, d, Tpad) so that attention's P.V B-operand is K-major over keys.
              // lane == row == consecutive t: each of the 32 stores is one contiguous 64-byte segment.
              if (row_ok) {
                const int d = g.N - g.d2;
                __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(g.out2) +
                                   (static_cast<size_t>(b_idx) * d + (col0 - g.d2)) * g.Tpad + t_idx;
#pragma unroll
                for (int j = 0; j < 32; ++j)
                  o[static_cast<size_t>(j) * g.Tpad] = __float2bfloat16_rn(__uint_as_float(v[j]) * rs);
              }
              continue;
            }
          }
          drain_bf16<false>(reinterpret_cast<__nv_bfloat16*>(g.out), EPI == VNB_EPI_BF16 ? g.N : g.d2, g.M, qaddr, rs, lane,
                            row_base, c * 32, col0);
        }
      }
    }
  }
  // a CTA of a pair may not exit while its peer can still arrive on its barriers
  if constexpr (PAIR) cluster_sync_all();
}

// ------------------------------------------------------------------------------------------------
// Single-CTA tiles or clusters of two CTAs sharing the W tile: vnb_set_option("gemm_pair", 0|1), else the environment
// variable VNB_GEMM_PAIR, else the compiled default.
static int g_gemm_pair = -1;
void set_gemm_pair(int on) { g_gemm_pair = on ? 1 : 0; }
static bool gemm_pair_enabled() {
  if (g_gemm_pair < 0) {
    const char* e = getenv("VNB_GEMM_PAIR");
    g_gemm_pair = e != nullptr ? (e[0] == '1') : (VNB_GEMM_PAIR_DEFAULT ? 1 : 0);
  }
  return g_gemm_pair == 1;
}
int get_gemm_pair() { return gemm_pair_enabled() ? 1 : 0; }

// Once per device and epilogue: opt in to the large dynamic shared memory for both tile variants and ask how many
// clusters of two can be co-resident.  Called eagerly by prepare_gemm() (model creation), so that none of this runs
// inside a stream capture.
static int g_max_clusters[6][64];
template <int EPI>
static cudaError_t init_epi() {
  static PerDeviceOnce once;
  int dev;
  if (!once.need(&dev)) return cudaSuccess;
  cudaError_t e = cudaFuncSetAttribute(gemm_wgmma_kernel<EPI, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, GEMM_SMEM);
  if (e != cudaSuccess) return e;
  e = cudaFuncSetAttribute(gemm_wgmma_kernel<EPI, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, GEMM_SMEM);
  if (e != cudaSuccess) return e;
  if constexpr (EPI == VNB_EPI_QKV || EPI == VNB_EPI_RESID || EPI == VNB_EPI_GEGLU) {
    e = cudaFuncSetAttribute(gemm_wgmma_kernel<EPI, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, GEMM_SMEM);
    if (e != cudaSuccess) return e;
    e = cudaFuncSetAttribute(gemm_wgmma_kernel<EPI, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, GEMM_SMEM);
    if (e != cudaSuccess) return e;
  }
  cudaLaunchConfig_t q = {};
  q.gridDim = dim3(2 * device_sm_count());
  q.blockDim = dim3(GEMM_THREADS);
  q.dynamicSmemBytes = GEMM_SMEM;
  cudaLaunchAttribute qa[1];
  qa[0].id = cudaLaunchAttributeClusterDimension;
  qa[0].val.clusterDim.x = 2; qa[0].val.clusterDim.y = 1; qa[0].val.clusterDim.z = 1;
  q.attrs = qa; q.numAttrs = 1;
  int n = 0;
  e = cudaOccupancyMaxActiveClusters(&n, gemm_wgmma_kernel<EPI, true>, &q);
  if (e != cudaSuccess || n <= 0) { (void)cudaGetLastError(); n = device_sm_count() / 2; }
  if (dev >= 0 && dev < 64) g_max_clusters[EPI][dev] = n;
  once.mark(dev);
  return cudaSuccess;
}
cudaError_t prepare_gemm() {
  cudaError_t e;
  if ((e = init_epi<VNB_EPI_BF16>()) != cudaSuccess) return e;
  if ((e = init_epi<VNB_EPI_QKV>()) != cudaSuccess) return e;
  if ((e = init_epi<VNB_EPI_RESID>()) != cudaSuccess) return e;
  if ((e = init_epi<VNB_EPI_GEGLU>()) != cudaSuccess) return e;
  if ((e = init_epi<VNB_EPI_BIAS_F32>()) != cudaSuccess) return e;
  return init_epi<VNB_EPI_SAMPLE>();
}

int get_gemm_max_clusters() {
  int dev = 0;
  cudaGetDevice(&dev);
  if (prepare_gemm() != cudaSuccess || dev < 0 || dev >= 64) return 0;
  return g_max_clusters[VNB_EPI_RESID][dev];
}

// One CTA per output tile (the accumulator tile overlays the operand ring, so a CTA does not start a second tile).
template <int EPI, bool ADAPT = false>
static cudaError_t launch_epi(const GemmPlan& p, const GemmArgs& g, cudaStream_t st) {
  cudaError_t e = init_epi<EPI>();
  if (e != cudaSuccess) return e;
  if (gemm_pair_enabled()) {
    const int clusters = ((g.M + 2 * BM - 1) / (2 * BM)) * (g.N / BN);
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(2 * clusters);
    cfg.blockDim = dim3(GEMM_THREADS);
    cfg.dynamicSmemBytes = GEMM_SMEM;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = 2; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr; cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, gemm_wgmma_kernel<EPI, true, ADAPT>, p.tmA, p.tmBh, g);
  }
  const int tiles = ((g.M + BM - 1) / BM) * (g.N / BN);
  gemm_wgmma_kernel<EPI, false, ADAPT><<<tiles, GEMM_THREADS, GEMM_SMEM, st>>>(p.tmA, p.tmB, g);
  return cudaGetLastError();
}

cudaError_t launch_gemm(const GemmPlan& p, cudaStream_t st) {
  GemmArgs g;
  g.M = p.M; g.N = p.N; g.K = p.K; g.epi = p.epi; g.out = p.out; g.out2 = p.out2; g.bias = p.bias;
  g.T = p.T; g.Tpad = p.Tpad; g.d2 = p.d2;
  g.out_bf16 = reinterpret_cast<__nv_bfloat16*>(p.out_bf16); g.ss_out = p.ss_out; g.ss_in = p.ss_in;
  g.ss_parts = p.ss_parts; g.inv_d = p.inv_d; g.eps = p.eps;
  g.zcur = p.zcur; g.dyn = p.dyn; g.rowgrp = p.rowgrp; g.partials = reinterpret_cast<float4*>(p.partials);
  g.C = p.C; g.ncc = p.ncc; g.V = p.V; g.mask_token = p.mask_token;
  g.lora = p.lora;
  if (p.lora.table != nullptr) {
    if (!p.lora.grp_adapter || !p.lora.rowgrp || !p.lora.u || p.lora.rows_per_grp < 1) return cudaErrorInvalidValue;
    switch (p.epi) {
      case VNB_EPI_QKV: return launch_epi<VNB_EPI_QKV, true>(p, g, st);
      case VNB_EPI_RESID: return launch_epi<VNB_EPI_RESID, true>(p, g, st);
      case VNB_EPI_GEGLU: return launch_epi<VNB_EPI_GEGLU, true>(p, g, st);
      default: return cudaErrorInvalidValue;  // the embedding and the classifier carry no LoRA
    }
  }
  switch (p.epi) {
    case VNB_EPI_BF16: return launch_epi<VNB_EPI_BF16>(p, g, st);
    case VNB_EPI_QKV: return launch_epi<VNB_EPI_QKV>(p, g, st);
    case VNB_EPI_RESID: return launch_epi<VNB_EPI_RESID>(p, g, st);
    case VNB_EPI_GEGLU: return launch_epi<VNB_EPI_GEGLU>(p, g, st);
    case VNB_EPI_BIAS_F32: return launch_epi<VNB_EPI_BIAS_F32>(p, g, st);
    case VNB_EPI_SAMPLE:
      if (!p.zcur || !p.dyn || !p.rowgrp || !p.partials || !p.bias || p.V % 128 != 0 || p.V > 1024) return cudaErrorInvalidValue;
      return launch_epi<VNB_EPI_SAMPLE>(p, g, st);
    default: return cudaErrorInvalidValue;
  }
}

// ------------------------------------------------------------------------------------------------
// Naive SIMT GEMM (test-only bisecting aid; never on the product path).
__global__ void gemm_ref_kernel(const __nv_bfloat16* A, const __nv_bfloat16* W, int M, int N, int K, float* out) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  const int m = blockIdx.y;
  if (n >= N || m >= M) return;
  float acc = 0.f;
  for (int k = 0; k < K; ++k)
    acc += __bfloat162float(A[static_cast<size_t>(m) * K + k]) * __bfloat162float(W[static_cast<size_t>(n) * K + k]);
  out[static_cast<size_t>(m) * N + n] = acc;
}
cudaError_t launch_gemm_ref(const void* A, const void* W, int M, int N, int K, float* out, cudaStream_t st) {
  dim3 grid((N + 127) / 128, M);
  gemm_ref_kernel<<<grid, 128, 0, st>>>(reinterpret_cast<const __nv_bfloat16*>(A),
                                        reinterpret_cast<const __nv_bfloat16*>(W), M, N, K, out);
  return cudaGetLastError();
}

}  // namespace vnb
