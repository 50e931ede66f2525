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
// The FFN-up and QKV GEMMs without adapters run gemm_persistent_kernel instead: the same mainloop in one CTA per SM,
// with each tile's stores overlapping the next tile's MMAs.
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

// Rows [0, live_rows) of the launch are live: M without a live bound.
__device__ __forceinline__ int live_rows(const GemmArgs& g) {
  if (g.live == nullptr) return g.M;
  const int r = __ldg(g.live) * g.T;
  return r < g.M ? r : g.M;
}

__device__ __forceinline__ float gelu_tanh(float x) {
  // 0.5*x*(1+tanh(sqrt(2/pi)*(x+0.044715*x^3)))   (activations.py:16-26); tanh(y) = 1 - 2/(1+exp(2y))
  const float y = 0.7978845608028654f * (x + 0.044715f * x * x * x);
  const float e = __expf(2.0f * y);
  const float t = 1.0f - __fdividef(2.0f, 1.0f + e);
  return 0.5f * x * (1.0f + t);
}

// Row scale of the fused RMSNorm of the A operand: rsqrt(mean(x^2) + eps) of output row `row`, from the partial sums of
// squares in a fixed order; 1 without a fused norm and past M.
__device__ __forceinline__ float row_scale(const GemmArgs& g, int row) {
  float rs = 1.0f;
  if (g.ss_in != nullptr && row < g.M) {
    float t = 0.f;
    for (int p = 0; p < g.ss_parts; ++p) t += __ldg(g.ss_in + static_cast<size_t>(p) * g.M + row);
    rs = rsqrtf(t * g.inv_d + g.eps);
  }
  return rs;
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

// The k-block loop of one tile (consumer warpgroup `wg`, rows [64 wg, 64 wg + 64)): acc += A W^T over every k-block in
// order, 4 x k16 per 64-wide k-block, from a ring of NS stages.  `stage` / `phase` are the ring position of the first
// k-block and are left at the one after the last, so a persistent CTA continues the ring from tile to tile.  release(s)
// hands stage s back to the producer once the MMAs reading it have retired.
template <int NS, typename Release>
__device__ __forceinline__ void gemm_mainloop(float (&acc)[128], uint8_t* ring, uint64_t* full_bar, int num_kb, int wg,
                                              int& stage, uint32_t& phase, Release&& release) {
#pragma unroll
  for (int i = 0; i < 128; ++i) acc[i] = 0.f;
  for (int kb = 0; kb < num_kb; ++kb) {
    mbar_wait(&full_bar[stage], phase);
    const uint32_t sa = smem_u32(ring + stage * STAGE_BYTES) + wg * (64 * 128);
    const uint32_t sb = smem_u32(ring + stage * STAGE_BYTES + A_BYTES);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < BK / 16; ++k)  // advance 16 bf16 = 32 B along K inside the 128B swizzle span
      wgmma_ss_n256(acc, wgmma_desc_sw128(sa + k * 32), wgmma_desc_sw128(sb + k * 32), 1u);
    wgmma_commit();
    wgmma_wait<1>();  // the previous k-block's MMAs have retired: its stage can be refilled
    wgmma_fence_regs(acc);
    if (kb > 0) release(stage == 0 ? NS - 1 : stage - 1);
    if (++stage == NS) { stage = 0; phase ^= 1; }
  }
  wgmma_wait<0>();
  wgmma_fence_regs(acc);
  if (num_kb > 0) release(stage == 0 ? NS - 1 : stage - 1);
}

// PAIR = true: clusters of two CTAs on vertically adjacent 128 x 256 tiles (the same 256 W rows).  Each CTA fetches
// half of the W tile (128 rows) and the TMA multicasts it into both CTAs' shared memory, so per CTA the W bytes pulled
// from L2 are halved; a stage is refilled only when the consumer warps of both CTAs have released it.  Every output
// element sees the same operands in the same K order as in the single-CTA variant: the two are bit-identical.  On an
// H100 the single-CTA kernel is faster (the pair couples the two CTAs' progress and constrains their placement; same-
// box A/B at the default bench workload: 403 vs 333 TFLOP/s for the GEMM family), so it is the default.
// SPLIT (EPI_SAMPLE only): a launch that mixes nucleus (top-p) and plain groups; see the sampling epilogue.
template <int EPI, bool PAIR, bool ADAPT = false, bool SPLIT = false>
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
  // a tile (pair: the cluster's first row, so both CTAs decide alike) past the live rows exits before any barrier or TMA
  if (g.live != nullptr && (tile / num_n) * TM >= live_rows(g)) return;

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
      const uint32_t peer_empty = PAIR ? mapa_u32(smem_u32(empty_bar), rank ^ 1u) : 0u;
      int stage = 0;
      uint32_t phase = 0;
      gemm_mainloop<STAGES>(acc, smem, full_bar, num_kb, wg, stage, phase, [&](int s) {
        if (lane == 0) {
          mbar_arrive(&empty_bar[s]);
          if constexpr (PAIR) mbar_arrive_cluster(peer_empty + 8u * s);
        }
      });
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
      const float rs = row_scale(g, row);  // fused RMSNorm of the A operand, this thread's row
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
        bool active = row_ok && __ldg(g.zcur + static_cast<size_t>(row) * g.C + g.ncc + cp) == g.mask_token;
        if constexpr (SPLIT) {
          // A launch of nucleus (top-p) and plain groups: a still-masked position of a nucleus group gets no record.
          // Its strip of logits goes to g.out instead, at the index and with the arithmetic of the materialising
          // epilogue (drain_f32: acc * row scale, + bias), for sample_rows_kernel.  The warp stores one such row at a
          // time, each lane four columns 32 apart: every store instruction is one contiguous 128-byte segment.
          if (__any_sync(0xffffffffu, active)) {
            const SampleDyn& dyn = g.dyn[g.rowgrp[row_ok ? b_idx : 0].group];
            const bool nucleus = dyn.top_p > 0.f && dyn.top_p < 1.f;
            uint32_t pend = __ballot_sync(0xffffffffu, active && nucleus);
            float* const strip_out = reinterpret_cast<float*>(g.out) + static_cast<size_t>(row_base) * g.N + col0 + lane;
            const uint32_t src = qaddr + 4u * (strip * 128 + lane);
            const uint32_t bsrc = sbias + 4u * (strip * 128 + lane);
            while (pend != 0u) {
              const int r = __ffs(pend) - 1;
              pend &= pend - 1u;
              const float rsr = __shfl_sync(0xffffffffu, rs, r);
              float* const dst = strip_out + static_cast<size_t>(r) * g.N;
#pragma unroll
              for (int k = 0; k < 4; ++k)
                dst[32 * k] = __fadd_rn(__fmul_rn(lds_f32(src + 4u * (r * ACC_PITCH + 32 * k)), rsr),
                                        lds_f32(bsrc + 128u * k));
            }
            active = active && !nucleus;
          }
        }
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
                // a frame past its call's own length is a zero key column, as in the call's own launch (zeroed
                // padding, TMA out-of-bounds fill); a select, so whatever the padded row holds cannot leak in
                const bool pad = g.frames != nullptr && t_idx >= __ldg(g.frames + b_idx);
#pragma unroll
                for (int j = 0; j < 32; ++j)
                  o[static_cast<size_t>(j) * g.Tpad] =
                      pad ? __float2bfloat16_rn(0.f) : __float2bfloat16_rn(__uint_as_float(v[j]) * rs);
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

// Persistent layer GEMMs without adapters, FFN-up (GEGLU) and QKV: one CTA per SM walks the tiles blockIdx.x,
// blockIdx.x + gridDim.x, ... in the same n-fastest order, and a tile's stores run on dedicated warps while the
// consumers compute the next tile.
//   warp 11      TMA producer: a ring of {A 128x64, W 256x64} stages as in gemm_wgmma_kernel, continued across tile
//                boundaries (GEGLU: 4 stages; QKV: 3, its staging tile is twice as large)
//   warps 0..7   consumers: the same mainloop; then the row scale (and GEGLU) in registers, rounded to bf16 into the
//                staging tile
//   warps 8..10  epilogue: copy the staging tile to global memory, then compute the row scales of the CTA's next tile
//                into shared memory
// GEGLU: value * gelu_tanh(gate) (value column c and gate column c + 128 are fragments i and i + 16 of the same thread),
// a 128 x 128 result stored in whole rows.  QKV: every 256-column tile is wholly q / k or wholly v (N = 3 d and
// N % 256 == 0, so d2 = 2 d is a multiple of 512); q / k tiles are staged row-major and stored in whole rows at pitch
// d2, v tiles are staged transposed and stored as runs of t into v^T (B, d, Tpad).
// Per output element the operands, the k order, the accumulator and the arithmetic (row scale, GEGLU, rounding, the
// frames select) are those of gemm_wgmma_kernel's epilogue: bit-identical.
constexpr int PERS_EPI_WARPS = 3;
constexpr int PERS_THREADS = 256 + 32 * PERS_EPI_WARPS + 32;  // 384: ptxas sizes registers per SM sub-partition, a
                                                              // 13th warp would cap every thread at 128
template <int EPI> constexpr int pers_stages() { return EPI == VNB_EPI_QKV ? 3 : STAGES; }
// bf16 result tile: GEGLU 128 x 128 (rows of 256 B), QKV 128 x 256 (q / k: rows of 512 B; v: 256 d-rows of 256 B)
template <int EPI> constexpr int pers_out_bytes() { return EPI == VNB_EPI_QKV ? BM * BN * 2 : BM * (BN / 2) * 2; }
template <int EPI>
constexpr int pers_smem() {
  return pers_stages<EPI>() * STAGE_BYTES + pers_out_bytes<EPI>() + 4 * BM /*row scales*/ + 1024 /*align slack*/ +
         128 /*barriers*/;
}
static_assert(pers_smem<VNB_EPI_GEGLU>() <= 227 * 1024, "H100: at most 227 KiB of shared memory per block");
static_assert(pers_smem<VNB_EPI_QKV>() <= 227 * 1024, "H100: at most 227 KiB of shared memory per block");
static_assert((2 * STAGES + 2) * 8 <= 128, "the barriers fit their slot");

// byte offset of the 4-byte word w of row r in a staging tile of PITCH-byte rows: the 16-byte unit w / 4 is XORed with
// r % 8, so the consumers' fragment stores (8 rows x 4 words) and the epilogue's row reads (consecutive units of one
// row) are both bank-conflict free.  The transposed v tile is the PITCH = 256 case with one row per d-row, word w
// holding tile rows 2 w and 2 w + 1.
template <int PITCH>
__device__ __forceinline__ uint32_t stage_off(int r, int w) {
  return static_cast<uint32_t>(r * PITCH + (((w >> 2) ^ (r & 7)) << 4) + ((w & 3) << 2));
}

template <int EPI>
__global__ void __launch_bounds__(PERS_THREADS, 1)
gemm_persistent_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                       const GemmArgs g) {
  constexpr int NS = pers_stages<EPI>();
  constexpr int RING = NS * STAGE_BYTES;
  constexpr int OUT_BYTES = pers_out_bytes<EPI>();
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const uint32_t stage_tile = smem_u32(smem + RING);
  float* srs = reinterpret_cast<float*>(smem + RING + OUT_BYTES);  // row scales of the tile being computed
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + RING + OUT_BYTES + 4 * BM);
  uint64_t* empty_bar = full_bar + NS;
  uint64_t* out_full = empty_bar + NS;  // the staging tile holds a result tile (256 consumer threads)
  uint64_t* out_free = out_full + 1;    // the staging tile is free and srs holds the next tile's row scales

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int num_n = g.N / BN;
  const int num_kb = g.K / BK;
  // m-major tile order: the tiles of the live rows are a prefix; every warp role reads the same bound
  const int tiles = ((live_rows(g) + BM - 1) / BM) * num_n;
  constexpr int kProducer = 8 + PERS_EPI_WARPS;

  if (warp == kProducer && lane == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int s = 0; s < NS; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 8);  // lane 0 of every consumer warp
    }
    mbar_init(out_full, 256);
    mbar_init(out_free, 32 * PERS_EPI_WARPS);
    mbar_fence_init();
  }
  __syncthreads();

  if (warp == kProducer) {
    // ===================== TMA producer =====================
    if (lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
        const int m0 = (tile / num_n) * BM, n0 = (tile % num_n) * BN;
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* sa = smem + stage * STAGE_BYTES;
          mbar_expect_tx(&full_bar[stage], STAGE_BYTES);
          tma_load_2d(sa, &tmA, &full_bar[stage], kb * BK, m0);
          tma_load_2d(sa + A_BYTES, &tmB, &full_bar[stage], kb * BK, n0);
          if (++stage == NS) { stage = 0; phase ^= 1; }
        }
      }
    }
    __syncwarp();
  } else if (warp < 8) {
    // ===================== consumers =====================
    int stage = 0;
    uint32_t phase = 0;
    uint32_t it = 0;
    // fragment of m64nNk16: thread (warp w, lane l) holds rows 16 w + l/4 and + 8, columns 8 i + 2 (l % 4) + {0, 1}
    const int r = (warp >> 2) * 64 + (warp & 3) * 16 + (lane >> 2);
    for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x, ++it) {
      float acc[128];
      gemm_mainloop<NS>(acc, smem, full_bar, num_kb, warp >> 2, stage, phase, [&](int s) {
        if (lane == 0) mbar_arrive(&empty_bar[s]);
      });
      mbar_wait(out_free, it & 1u);  // the previous result tile is stored, srs holds this tile's row scales
      const float rs0 = srs[r], rs1 = srs[r + 8];
      if constexpr (EPI == VNB_EPI_GEGLU) {
#pragma unroll
        for (int i = 0; i < 16; ++i) {
          float x[4];
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const float rsr = k < 2 ? rs0 : rs1;
            x[k] = acc[4 * i + k] * rsr;
            x[k] = x[k] * gelu_tanh(acc[4 * (i + 16) + k] * rsr);
          }
          const int w = 4 * i + (lane & 3);
          sts_u32(stage_tile + stage_off<256>(r, w), pack_bf16x2(x[0], x[1]));
          sts_u32(stage_tile + stage_off<256>(r + 8, w), pack_bf16x2(x[2], x[3]));
        }
      } else if ((tile % num_n) * BN < g.d2) {  // q / k
#pragma unroll
        for (int i = 0; i < 32; ++i) {
          const int w = 4 * i + (lane & 3);
          sts_u32(stage_tile + stage_off<512>(r, w), pack_bf16x2(acc[4 * i] * rs0, acc[4 * i + 1] * rs0));
          sts_u32(stage_tile + stage_off<512>(r + 8, w), pack_bf16x2(acc[4 * i + 2] * rs1, acc[4 * i + 3] * rs1));
        }
      } else {
        // v, transposed: tile column c is d-row c of v^T.  The lanes 4 apart hold tile rows r and r + 1 (r even) of
        // the same two columns; they swap their packed pairs, and each stores one column's two rows as one word: the
        // even row's lane column 8 i + 2 (l % 4), the odd row's lane the column after it.
        const bool odd = (lane >> 2) & 1;
#pragma unroll
        for (int i = 0; i < 32; ++i) {
          const int c = 8 * i + 2 * (lane & 3) + (odd ? 1 : 0);
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const float rsr = h ? rs1 : rs0;
            const uint32_t own = pack_bf16x2(acc[4 * i + 2 * h] * rsr, acc[4 * i + 2 * h + 1] * rsr);
            const uint32_t peer = __shfl_xor_sync(0xffffffffu, own, 4);
            sts_u32(stage_tile + stage_off<256>(c, (r + 8 * h) >> 1),
                    odd ? __byte_perm(peer, own, 0x7632) : __byte_perm(own, peer, 0x5410));
          }
        }
      }
      mbar_arrive(out_full);
    }
  } else {
    // ===================== epilogue =====================
    const int e = warp - 8;
    __nv_bfloat16* const out = reinterpret_cast<__nv_bfloat16*>(g.out);
    const int pitch = EPI == VNB_EPI_GEGLU ? g.N / 2 : g.d2;
    auto row_scales = [&](int tile) {  // row scales of `tile` into srs, then hand the staging tile to the consumers
      if (tile < tiles) {
        const int m0 = (tile / num_n) * BM;
        for (int j = e * 32 + lane; j < BM; j += 32 * PERS_EPI_WARPS) srs[j] = row_scale(g, m0 + j);
      }
      mbar_arrive(out_free);
    };
    row_scales(blockIdx.x);
    uint32_t it = 0;
    for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x, ++it) {
      const int m0 = (tile / num_n) * BM, n0 = (tile % num_n) * BN;
      mbar_wait(out_full, it & 1u);
      if constexpr (EPI == VNB_EPI_GEGLU) {
        // two tile rows per warp instruction: lane -> (row 2 u + lane / 16, 16-byte unit lane % 16)
#pragma unroll 4
        for (int u = e; u < BM / 2; u += PERS_EPI_WARPS) {
          const int rr = 2 * u + (lane >> 4);
          const float4 v = lds_f4(stage_tile + stage_off<256>(rr, 4 * (lane & 15)));
          if (m0 + rr < g.M)
            *reinterpret_cast<float4*>(out + static_cast<size_t>(m0 + rr) * pitch + (n0 >> 1) + 8 * (lane & 15)) = v;
        }
      } else if (n0 < g.d2) {
        // q / k: one 512-byte tile row per warp instruction
#pragma unroll 4
        for (int rr = e; rr < BM; rr += PERS_EPI_WARPS) {
          const float4 v = lds_f4(stage_tile + stage_off<512>(rr, 4 * lane));
          if (m0 + rr < g.M)
            *reinterpret_cast<float4*>(out + static_cast<size_t>(m0 + rr) * pitch + n0 + 8 * lane) = v;
        }
      } else {
        // v^T: lane -> tile rows 4 lane .. 4 lane + 3 of every d-row, so a warp instruction stores a d-row's run of t.
        // Their (b, t), bounds and frames select do not depend on the d-row.  Four rows of one batch row whose first
        // t is a multiple of 4 go as one 8-byte store; any other group (a batch-row boundary, an odd T) element by
        // element.  A frame past its call's own length is stored as 0 (a select, as in the one-tile epilogue).
        const int d = g.N - g.d2;
        uint16_t* const vt = reinterpret_cast<uint16_t*>(g.out2) + static_cast<size_t>(n0 - g.d2) * g.Tpad;
        size_t off[4];
        bool ok[4];
        int bk[4];
        uint32_t keep[2] = {0xffffffffu, 0xffffffffu};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const int m = m0 + 4 * lane + k;
          bk[k] = m / g.T;
          const int t = m - bk[k] * g.T;
          ok[k] = m < g.M;
          off[k] = static_cast<size_t>(bk[k]) * d * g.Tpad + t;
          if (ok[k] && g.frames != nullptr && t >= __ldg(g.frames + bk[k])) keep[k >> 1] &= (k & 1) ? 0xffffu : 0xffff0000u;
        }
        const bool wide = ok[3] && bk[3] == bk[0] && (off[0] & 3) == 0 && (g.Tpad & 3) == 0 &&
                          (reinterpret_cast<uintptr_t>(g.out2) & 7) == 0;
#pragma unroll 2
        for (int c = e; c < BN; c += PERS_EPI_WARPS) {
          uint2 v = lds_u2(stage_tile + stage_off<256>(c, 2 * lane));
          v.x &= keep[0];
          v.y &= keep[1];
          uint16_t* const o = vt + static_cast<size_t>(c) * g.Tpad;
          if (wide) {
            *reinterpret_cast<uint2*>(o + off[0]) = v;
          } else {
#pragma unroll
            for (int k = 0; k < 4; ++k) {
              const uint32_t w = k < 2 ? v.x : v.y;
              if (ok[k]) o[off[k]] = static_cast<uint16_t>((k & 1) ? (w >> 16) : w);
            }
          }
        }
      }
      row_scales(tile + gridDim.x);
    }
  }
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
  if constexpr (EPI == VNB_EPI_GEGLU || EPI == VNB_EPI_QKV) {
    e = cudaFuncSetAttribute(gemm_persistent_kernel<EPI>, cudaFuncAttributeMaxDynamicSharedMemorySize, pers_smem<EPI>());
    if (e != cudaSuccess) return e;
  }
  if constexpr (EPI == VNB_EPI_SAMPLE) {
    e = cudaFuncSetAttribute(gemm_wgmma_kernel<EPI, false, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                             GEMM_SMEM);
    if (e != cudaSuccess) return e;
    e = cudaFuncSetAttribute(gemm_wgmma_kernel<EPI, true, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                             GEMM_SMEM);
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

// One CTA per output tile (the accumulator tile overlays the operand ring, so a CTA does not start a second tile), except
// for the FFN-up and QKV GEMMs without adapters: the persistent kernel, one CTA per SM (the SM count is cached by
// prepare_gemm(), so none is queried inside a capture).
template <int EPI, bool ADAPT = false, bool SPLIT = false>
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
    return cudaLaunchKernelEx(&cfg, gemm_wgmma_kernel<EPI, true, ADAPT, SPLIT>, p.tmA, p.tmBh, g);
  }
  const int tiles = ((g.M + BM - 1) / BM) * (g.N / BN);
  if constexpr ((EPI == VNB_EPI_GEGLU || EPI == VNB_EPI_QKV) && !ADAPT) {
    const int grid = tiles < device_sm_count() ? tiles : device_sm_count();
    gemm_persistent_kernel<EPI><<<grid, PERS_THREADS, pers_smem<EPI>(), st>>>(p.tmA, p.tmB, g);
    return cudaGetLastError();
  }
  gemm_wgmma_kernel<EPI, false, ADAPT, SPLIT><<<tiles, GEMM_THREADS, GEMM_SMEM, st>>>(p.tmA, p.tmB, g);
  return cudaGetLastError();
}

cudaError_t launch_gemm(const GemmPlan& p, cudaStream_t st) {
  GemmArgs g = p.args;
  if (g.epi != VNB_EPI_QKV) g.frames = nullptr;  // only the QKV epilogue writes per-row padding
  if (g.lora.table != nullptr) {
    if (!g.lora.grp_adapter || !g.lora.rowgrp || !g.lora.u || g.lora.rows_per_grp < 1) return cudaErrorInvalidValue;
    switch (g.epi) {
      case VNB_EPI_QKV: return launch_epi<VNB_EPI_QKV, true>(p, g, st);
      case VNB_EPI_RESID: return launch_epi<VNB_EPI_RESID, true>(p, g, st);
      case VNB_EPI_GEGLU: return launch_epi<VNB_EPI_GEGLU, true>(p, g, st);
      default: return cudaErrorInvalidValue;  // the embedding and the classifier carry no LoRA
    }
  }
  switch (g.epi) {
    case VNB_EPI_BF16: return launch_epi<VNB_EPI_BF16>(p, g, st);
    case VNB_EPI_QKV: return launch_epi<VNB_EPI_QKV>(p, g, st);
    case VNB_EPI_RESID: return launch_epi<VNB_EPI_RESID>(p, g, st);
    case VNB_EPI_GEGLU: return launch_epi<VNB_EPI_GEGLU>(p, g, st);
    case VNB_EPI_BIAS_F32: return launch_epi<VNB_EPI_BIAS_F32>(p, g, st);
    case VNB_EPI_SAMPLE:
      if (!g.zcur || !g.dyn || !g.rowgrp || !g.partials || !g.bias || g.V % 128 != 0 || g.V > 1024) return cudaErrorInvalidValue;
      if (p.sample_split) {
        if (!g.out) return cudaErrorInvalidValue;
        return launch_epi<VNB_EPI_SAMPLE, false, true>(p, g, st);
      }
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
