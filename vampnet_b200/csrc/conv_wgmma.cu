// vampnet_b200 — codec convolutions on the sm_90a tensor cores (SURVEY.md §8f row f-1).
//
// A 1-D convolution is a GEMM over (tap, input-channel) with the A operand read at a time shift per tap:
//   y[b, q, n] = bias[n] + sum_tap sum_ci W[n, tap, ci] * a[b, q*s + tap*dil - pad, ci]
// Activations are channels-last (B, T, C), so the A tile of k-block (tap, channel block) is a plain TMA box at row
// q0 + shift; rows outside [0, T) are zero-filled by TMA, which IS the convolution's zero padding.  Strided
// convolutions view the input as (B, T/s, s*C): x[q*s + e] = view[q + floor(e/s), (e mod s)*C + ci].  A transposed
// convolution (kernel 2s, stride s) is ONE GEMM with N = s*Cout columns (phase-major) and two taps (x[q], x[q-1]);
// its (T+1, s*Cout) result is the (T*s, Cout) output shifted by `pad` rows, so the store is row-major plus an
// offset and a validity mask.  (Architecture: transformers/models/dac/modeling_dac.py:173-268, 405-473; reference
// call sites vampnet/interface.py:223, vampnet/modules/transformer.py:671-675.)
//
// Precision: the codec must stay within 1e-3 of the fp32 reference waveform, which bf16 operands cannot give
// over ~30 layers.  Operands are therefore SPLIT bf16 pairs (x = hi + lo, 16 mantissa bits together) and every
// k-step issues three wgmma (hi*hi + hi*lo + lo*hi) into the same fp32 register accumulators: fp32-grade
// products at 1/3 of the bf16 tensor rate, still >20x the fp32 CUDA-core rate.
//
// Epilogue (fused): + bias, + fp32 skip (residual units), store the fp32 stream, and/or apply the NEXT layer's
// Snake activation (x + sin^2(alpha x)/alpha) and store it split as hi/lo bf16 = the next conv's A operand.
//
// VGGish (fad.cu) runs its 3x3 convolutions and fully connected layers through the same kernel.  A 2-D convolution
// (g.W > 0) reads NHWC images (Bn, H, W, Cin): a 128-row tile is 128 / W whole image rows, and the A box of tap (dh, dw)
// is a 4-D TMA box at (h0 + dh - 1, w0 + dw - 1) whose out-of-bounds zero fill is the padding on both axes.  Its
// epilogue adds the bias and applies ReLU, and with the 2 x 2 max-pool (an even number of image rows per tile) stores
// the pooled (H/2, W/2) image, split hi/lo.
//
// Same warp-specialised structure as gemm_wgmma.cu: TMA producer warp, two consumer warpgroups (64 rows x NW columns
// of wgmma accumulators each), one CTA per tile of 128 rows x BN columns (BN <= 128, runtime).  The MMA width NW is
// the narrowest of 32 / 64 / 128 that covers BN, so the narrow audio-rate layers issue no MMAs for columns they do not
// have (only BN = 96 computes 32 columns it drops); the 8-warp epilogue reads the accumulators from a shared-memory
// tile that overlays the drained ring.
#include "common.cuh"
#include "kernels.h"
#include "wgmma.cuh"

namespace vnb {

constexpr int CT_BM = 128, CT_BK = 64, CT_STAGES = 3, CT_MAXBN = 128;
constexpr int CT_A_BYTES = CT_BM * CT_BK * 2;        // 16 KiB (one of hi / lo)
constexpr int CT_B_BYTES = CT_MAXBN * CT_BK * 2;     // 16 KiB (one of hi / lo)
constexpr int CT_STAGE_BYTES = 2 * CT_A_BYTES + 2 * CT_B_BYTES;  // 64 KiB
constexpr int CT_EPI_WARPS = 8;                       // two warps per 32-row quadrant (even / odd 32-column chunks)
constexpr int CT_SMEM = CT_STAGES * CT_STAGE_BYTES + 1024 + 256;
constexpr int CT_THREADS = 32 * CT_EPI_WARPS + 32;  // the epilogue warps are the two consumer warpgroups; + producer
constexpr int CT_ACC_PITCH = CT_MAXBN + 1;           // fp32 accumulator tile, odd pitch: row reads are conflict-free
static_assert(CT_BM * CT_ACC_PITCH * 4 <= CT_STAGES * CT_STAGE_BYTES, "the accumulator tile overlays the ring");
static_assert(CT_SMEM <= 227 * 1024, "H100: at most 227 KiB of shared memory per block");

struct ConvTcArgs {
  int Bn, Tq, N, BN;            // batch, output rows per batch item, output columns, column tile
  int cblocks, taps, dil, pad, s, Cin;
  const float* bias; int bias_mod;
  const float* alpha; int alpha_mod;
  const float* resid;           // fp32, same indexing as out
  float* out_f32;
  __nv_bfloat16* out_hi; __nv_bfloat16* out_lo;
  long long out_batch_stride;   // elements
  long long out_offset;         // elements added to q*N + n (negative for transposed convs)
  long long out_limit;          // valid flat range per batch item: [0, out_limit)
  int do_tanh;
  // Clips of different lengths in one launch (vnb_codec_conv_tc_ragged): DEVICE [Bn] valid output rows of each item,
  // in rows of row_elems elements (N for a plain convolution, Cout for a transposed one).  NULL: every item is Tq rows.
  const int* lens; int row_elems;
  // CT_RELU / CT_RELU_POOL: image height and width of a 2-D convolution (Tq = H * W), W = 0 for 1-D addressing
  int H, W;
};

// Halo of a ragged launch: rows [len_b, len_b + CT_HALO) of every output hold +0, so that the next layer's valid rows
// read exactly the zeros that TMA's out-of-bounds fill gives a clip coded alone.  The reach past an item's last valid
// row of each codec layer, in its input rows: k = 7 residual convs 3 * dil <= 27 (dil 1, 3, 9); 1 x 1 convs 0;
// encoder.conv2 (k 3) 1; decoder.conv1 (k 7) 3; the strided convs (k = 2s, pad ceil(s/2)) one view row, i.e. at most s
// <= 12 samples; the transposed convs one input row; decoder.conv2 (k 7, codec_out_kernel) 3.
constexpr int CT_HALO = 128;
static_assert(CT_HALO >= 27 && CT_HALO >= 12, "the halo covers the largest reach of any codec layer");

// Snake: v + sin^2(a v) / (a + 1e-9).  sin via two-constant Cody-Waite reduction to [-pi, pi] + MUFU.SIN
// (abs error < 1e-6 for |a v| < 1e4, far below the split-bf16 product error); 1/(a+1e-9) is passed in.
__device__ __forceinline__ float snake_act(float v, float a, float inv_a) {
  const float t = a * v;
  const float k = rintf(t * 0.15915494309189535f);
  float r = fmaf(k, -6.2831854820251465f, t);   // 2*pi rounded to fp32
  r = fmaf(k, 1.7484555e-7f, r);                 // minus the remainder of 2*pi
  const float s = __sinf(r);
  return fmaf(s * s, inv_a, v);
}

// MODE selects the fused epilogue at compile time (the epilogue is the critical path of the narrow layers, and every
// run-time switch in it costs issue slots on the eight warps that execute it):
//   CT_GENERIC      everything decided at run time from ConvTcArgs (any combination; encoder.conv2, tests)
//   CT_SPLIT        y -> snake_next(y) -> hi/lo                                  (k = 7 convolution of a residual unit)
//   CT_SPLIT_SKIP   y + skip -> fp32 stream (in place) and snake_next -> hi/lo   (1 x 1 convolution closing the unit)
//   CT_SPLIT_F32    y -> fp32 stream and snake_next -> hi/lo                     (strided / transposed convolutions)
//   CT_RELU         relu(y + bias) -> hi/lo                         (VGGish: 3x3 convolutions without a pool, FC 1-2)
//   CT_RELU_POOL    2x2 max-pool of relu(y + bias) -> hi/lo         (VGGish: 3x3 convolutions followed by a pool)
enum : int { CT_GENERIC = 0, CT_SPLIT = 1, CT_SPLIT_SKIP = 2, CT_SPLIT_F32 = 3, CT_RELU = 4, CT_RELU_POOL = 5 };

template <int MODE, int NW>
__global__ void __launch_bounds__(CT_THREADS, 1)
conv_wgmma_kernel(const __grid_constant__ CUtensorMap tmAh, const __grid_constant__ CUtensorMap tmAl,
                  const __grid_constant__ CUtensorMap tmWh, const __grid_constant__ CUtensorMap tmWl,
                  const ConvTcArgs g) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + CT_STAGES * CT_STAGE_BYTES);
  uint64_t* empty_bar = full_bar + CT_STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m_tiles = (g.Tq + CT_BM - 1) / CT_BM;
  const int n_tiles = (g.N + g.BN - 1) / g.BN;
  const int num_kb = g.taps * g.cblocks;
  const uint32_t stage_tx = 2 * CT_A_BYTES + 2 * g.BN * CT_BK * 2;
  // tile -> (batch, q0, n0): n fastest so that consecutive CTAs share the same A rows (L2 reuse of activations)
  const int tile = blockIdx.x;
  const int n0 = (tile % n_tiles) * g.BN;
  const int q0 = ((tile / n_tiles) % m_tiles) * CT_BM;
  const int b = tile / n_tiles / m_tiles;
  // stores are kept to flat indices [0, store_limit); values to [0, value_limit), the rest of that range gets +0
  long long value_limit = g.out_limit, store_limit = g.out_limit;
  if (g.lens != nullptr) {
    const long long len = g.lens[b];
    const long long halo_end = (len + CT_HALO) * g.row_elems;
    // no output row of this tile lies below the halo's end (block-uniform): nothing to load, compute or store
    if (static_cast<long long>(q0) * g.N + g.out_offset >= halo_end) return;
    value_limit = min(len * g.row_elems, g.out_limit);
    store_limit = min(halo_end, g.out_limit);
  }

  if (warp == CT_EPI_WARPS && lane == 0) {
    tma_prefetch_desc(&tmAh); tma_prefetch_desc(&tmAl); tma_prefetch_desc(&tmWh); tma_prefetch_desc(&tmWl);
    for (int s = 0; s < CT_STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], CT_EPI_WARPS); }
    mbar_fence_init();
  }
  __syncthreads();

  if (warp == CT_EPI_WARPS) {
    if (lane == 0) {
      int stage = 0; uint32_t phase = 0;
      for (int kb = 0; kb < num_kb; ++kb) {
        const int tap = kb / g.cblocks, cblk = kb - tap * g.cblocks;
        const int e = tap * g.dil - g.pad;                     // time shift in input samples
        const int qs = (e >= 0) ? e / g.s : -((-e + g.s - 1) / g.s);  // floor(e / s)
        const int r = e - qs * g.s;                            // 0 <= r < s
        const int col = r * g.Cin + cblk * CT_BK;
        mbar_wait(&empty_bar[stage], phase ^ 1);
        uint8_t* sa = smem + stage * CT_STAGE_BYTES;
        mbar_expect_tx(&full_bar[stage], stage_tx);
        if (MODE >= CT_RELU && g.W > 0) {  // 2-D 3x3 convolution: tap = 3 dh + dw
          const int h = q0 / g.W + tap / 3 - 1, w = tap % 3 - 1;
          tma_load_4d(sa, &tmAh, &full_bar[stage], cblk * CT_BK, w, h, b);
          tma_load_4d(sa + CT_A_BYTES, &tmAl, &full_bar[stage], cblk * CT_BK, w, h, b);
        } else {
          tma_load_3d(sa, &tmAh, &full_bar[stage], col, q0 + qs, b);
          tma_load_3d(sa + CT_A_BYTES, &tmAl, &full_bar[stage], col, q0 + qs, b);
        }
        tma_load_2d(sa + 2 * CT_A_BYTES, &tmWh, &full_bar[stage], kb * CT_BK, n0);
        tma_load_2d(sa + 2 * CT_A_BYTES + CT_B_BYTES, &tmWl, &full_bar[stage], kb * CT_BK, n0);
        if (++stage == CT_STAGES) { stage = 0; phase ^= 1; }
      }
    }
    return;
  }

  const int quad = warp & 3;
  const int half = warp >> 2;  // this warp takes the 32-column chunks with (c & 1) == half
  const int c4 = (lane & 7) * 4;
  const int nchunks = g.BN / 32;
  const bool has_skip = MODE == CT_GENERIC ? g.resid != nullptr : MODE == CT_SPLIT_SKIP;
  const long long row_step = 4LL * g.N;   // this lane's rows are (lane >> 3) + 4 * itr
  // The layers that carry a skip connection (the 1x1 convolutions closing a residual unit) have almost no MMA work per
  // tile, so the epilogue IS the kernel and the fp32 skip rows are its only synchronous global read: they are fetched
  // one chunk ahead, so eight 512-byte row segments per warp are in flight while the previous chunk is activated,
  // split and stored.
  auto fetch_skip = [&](int c, float4 (&pre)[8]) {
    const int n = n0 + c * 32 + c4;
    const int q = q0 + quad * 32 + (lane >> 3);
    const long long flat0 = static_cast<long long>(q) * g.N + n + g.out_offset;
    const float* base = g.resid + static_cast<long long>(b) * g.out_batch_stride + flat0;
#pragma unroll
    for (int itr = 0; itr < 8; ++itr) {
      const long long flat = flat0 + itr * row_step;
      const bool ok = n < g.N && q + 4 * itr < g.Tq && flat >= 0 && flat < g.out_limit;
      pre[itr] = ok ? __ldcg(reinterpret_cast<const float4*>(base + itr * row_step)) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  };
  float4 skip[8], skip_next[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) skip[i] = skip_next[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  if (has_skip && half < nchunks) fetch_skip(half, skip);

  {
    // ===================== consumers: mainloop =====================
    const int wg = warp >> 2;
    static_assert(NW == 32 || NW == 64 || NW == 128, "wgmma width");
    float acc[NW / 2];
#pragma unroll
    for (int i = 0; i < NW / 2; ++i) acc[i] = 0.f;
    int stage = 0; uint32_t phase = 0;
    auto release = [&](int s) { if (lane == 0) mbar_arrive(&empty_bar[s]); };
    for (int kb = 0; kb < num_kb; ++kb) {
      mbar_wait(&full_bar[stage], phase);
      const uint32_t ah = smem_u32(smem + stage * CT_STAGE_BYTES) + wg * (64 * 128);
      const uint32_t al = ah + CT_A_BYTES;
      const uint32_t wh = smem_u32(smem + stage * CT_STAGE_BYTES + 2 * CT_A_BYTES), wl = wh + CT_B_BYTES;
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < CT_BK / 16; ++k) {
        const uint64_t dAh = wgmma_desc_sw128(ah + k * 32), dAl = wgmma_desc_sw128(al + k * 32);
        const uint64_t dWh = wgmma_desc_sw128(wh + k * 32), dWl = wgmma_desc_sw128(wl + k * 32);
        if constexpr (NW == 128) {
          wgmma_ss_n128(acc, dAh, dWh, 1u);  // hi*hi
          wgmma_ss_n128(acc, dAh, dWl, 1u);  // hi*lo
          wgmma_ss_n128(acc, dAl, dWh, 1u);  // lo*hi
        } else if constexpr (NW == 64) {
          wgmma_ss_n64(acc, dAh, dWh, 1u);
          wgmma_ss_n64(acc, dAh, dWl, 1u);
          wgmma_ss_n64(acc, dAl, dWh, 1u);
        } else {
          wgmma_ss_n32(acc, dAh, dWh, 1u);
          wgmma_ss_n32(acc, dAh, dWl, 1u);
          wgmma_ss_n32(acc, dAl, dWh, 1u);
        }
      }
      wgmma_commit();
      wgmma_wait<1>();  // the previous k-block's MMAs have retired: its stage can be refilled
      wgmma_fence_regs(acc);
      if (kb > 0) release(stage == 0 ? CT_STAGES - 1 : stage - 1);
      if (++stage == CT_STAGES) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    wgmma_fence_regs(acc);
    // (no release of the last stage: nothing is loaded after it)
    // both warpgroups are done with the ring; accumulators -> fp32 tile (fragment layout as in gemm_wgmma.cu)
    asm volatile("bar.sync 1, 256;" ::: "memory");
    const int r = wg * 64 + (warp & 3) * 16 + (lane >> 2);
    const uint32_t p0 = smem_u32(smem) + 4u * (r * CT_ACC_PITCH + 2 * (lane & 3));
#pragma unroll
    for (int i = 0; i < NW / 8; ++i) {
      sts_f32(p0 + 32u * i, acc[4 * i]);
      sts_f32(p0 + 32u * i + 4, acc[4 * i + 1]);
      sts_f32(p0 + 4u * (8 * CT_ACC_PITCH) + 32u * i, acc[4 * i + 2]);
      sts_f32(p0 + 4u * (8 * CT_ACC_PITCH) + 32u * i + 4, acc[4 * i + 3]);
    }
    asm volatile("bar.sync 1, 256;" ::: "memory");
  }

  // ===================== epilogue =====================
  const uint32_t acc_tile = smem_u32(smem);
  if constexpr (MODE == CT_RELU_POOL) {
    // pooled pixel p of this tile's (128 / W / 2) x (W / 2), four columns per thread; relu(max(.) + bias) equals the
    // max of relu(. + bias)
    const int W2 = g.W / 2, H2 = g.H / 2, nq = g.BN / 4;
    const int ph0 = q0 / g.W / 2;
    for (int i = threadIdx.x; i < (CT_BM / 4) * nq; i += 32 * CT_EPI_WARPS) {
      const int p = i / nq, cq = (i - p * nq) * 4, n = n0 + cq;
      const int ph = p / W2, pw = p - ph * W2;
      if (ph0 + ph >= H2 || n >= g.N) continue;
      const int r = 2 * ph * g.W + 2 * pw;
      const float4 bv = __ldg(reinterpret_cast<const float4*>(g.bias + n));
      float v[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const uint32_t sp = acc_tile + 4u * (r * CT_ACC_PITCH + cq + j);
        const float m = fmaxf(fmaxf(lds_f32(sp), lds_f32(sp + 4u * CT_ACC_PITCH)),
                              fmaxf(lds_f32(sp + 4u * (g.W * CT_ACC_PITCH)), lds_f32(sp + 4u * ((g.W + 1) * CT_ACC_PITCH))));
        v[j] = fmaxf(m + (&bv.x)[j], 0.f);
      }
      const __nv_bfloat162 h01 = __floats2bfloat162_rn(v[0], v[1]), h23 = __floats2bfloat162_rn(v[2], v[3]);
      const float2 f01 = __bfloat1622float2(h01), f23 = __bfloat1622float2(h23);
      uint2 hi, lo;
      hi.x = *reinterpret_cast<const uint32_t*>(&h01);
      hi.y = *reinterpret_cast<const uint32_t*>(&h23);
      lo.x = pack_bf16x2(v[0] - f01.x, v[1] - f01.y);
      lo.y = pack_bf16x2(v[2] - f23.x, v[3] - f23.y);
      const long long o = static_cast<long long>(b) * g.out_batch_stride +
                          (static_cast<long long>(ph0 + ph) * W2 + pw) * g.N + n;
      *reinterpret_cast<uint2*>(g.out_hi + o) = hi;
      *reinterpret_cast<uint2*>(g.out_lo + o) = lo;
    }
    return;
  }
  const bool out_f32 = MODE == CT_GENERIC || MODE == CT_RELU ? g.out_f32 != nullptr : MODE != CT_SPLIT;
  const bool out_split = MODE == CT_GENERIC || MODE == CT_RELU ? g.out_hi != nullptr : true;
  const bool snake = MODE == CT_GENERIC ? g.alpha != nullptr : MODE != CT_RELU;
  const bool do_tanh = MODE == CT_GENERIC ? g.do_tanh != 0 : false;
  const bool has_bias = MODE == CT_GENERIC ? g.bias != nullptr : true;
  const long long bbase = static_cast<long long>(b) * g.out_batch_stride;
  for (int c = half; c < nchunks; c += 2) {
    if (has_skip && c + 2 < nchunks) fetch_skip(c + 2, skip_next);
    const int n = n0 + c * 32 + c4;  // first of this lane's 4 columns
    const bool n_ok = n < g.N;
    // per-channel constants first: their (L1/L2) latency hides behind the accumulator-tile reads
    float4 bv = make_float4(0.f, 0.f, 0.f, 0.f), al4 = make_float4(1.f, 1.f, 1.f, 1.f);
    if (n_ok) {
      if (has_bias) bv = __ldg(reinterpret_cast<const float4*>(g.bias + (g.bias_mod == g.N ? n : n % g.bias_mod)));
      if (snake) al4 = __ldg(reinterpret_cast<const float4*>(g.alpha + (g.alpha_mod == g.N ? n : n % g.alpha_mod)));
    }
    if (n_ok) {
      const float4 ia4 = make_float4(1.0f / (al4.x + 1e-9f), 1.0f / (al4.y + 1e-9f), 1.0f / (al4.z + 1e-9f),
                                     1.0f / (al4.w + 1e-9f));
      const int q = q0 + quad * 32 + (lane >> 3);
      const long long flat0 = static_cast<long long>(q) * g.N + n + g.out_offset;
      const long long o0 = bbase + flat0;
      // 8 lanes per accumulator-tile row, 4 columns each (odd pitch: conflict-free)
      const uint32_t sp0 = acc_tile + 4u * ((quad * 32 + (lane >> 3)) * CT_ACC_PITCH + c * 32 + c4);
#pragma unroll
      for (int itr = 0; itr < 8; ++itr) {
        const long long flat = flat0 + itr * row_step;
        if (q + 4 * itr < g.Tq && flat >= 0 && flat < store_limit) {
          // halo rows of a ragged launch: +0 by a select (padded rows may have accumulated NaN), never a product
          const bool halo = flat >= value_limit;
          const uint32_t sp = sp0 + 4u * (itr * 4 * CT_ACC_PITCH);
          float4 a = make_float4(lds_f32(sp) + bv.x, lds_f32(sp + 4) + bv.y, lds_f32(sp + 8) + bv.z,
                                 lds_f32(sp + 12) + bv.w);
          const long long o = o0 + itr * row_step;
          if (has_skip) {
            const float4 x = skip[itr];
            a.x += x.x; a.y += x.y; a.z += x.z; a.w += x.w;
          }
          if (do_tanh) { a.x = tanhf(a.x); a.y = tanhf(a.y); a.z = tanhf(a.z); a.w = tanhf(a.w); }
          if (MODE == CT_RELU) { a.x = fmaxf(a.x, 0.f); a.y = fmaxf(a.y, 0.f); a.z = fmaxf(a.z, 0.f); a.w = fmaxf(a.w, 0.f); }
          if (halo) a = make_float4(0.f, 0.f, 0.f, 0.f);
          if (out_f32) *reinterpret_cast<float4*>(g.out_f32 + o) = a;
          if (out_split) {
            if (snake) {
              a.x = snake_act(a.x, al4.x, ia4.x); a.y = snake_act(a.y, al4.y, ia4.y);
              a.z = snake_act(a.z, al4.z, ia4.z); a.w = snake_act(a.w, al4.w, ia4.w);
            }
            const __nv_bfloat162 h01 = __floats2bfloat162_rn(a.x, a.y), h23 = __floats2bfloat162_rn(a.z, a.w);
            const float2 f01 = __bfloat1622float2(h01), f23 = __bfloat1622float2(h23);
            uint2 hi, lo;
            hi.x = *reinterpret_cast<const uint32_t*>(&h01);
            hi.y = *reinterpret_cast<const uint32_t*>(&h23);
            lo.x = pack_bf16x2(a.x - f01.x, a.y - f01.y);
            lo.y = pack_bf16x2(a.z - f23.x, a.w - f23.y);
            if (halo) { hi = make_uint2(0u, 0u); lo = make_uint2(0u, 0u); }
            *reinterpret_cast<uint2*>(g.out_hi + o) = hi;
            *reinterpret_cast<uint2*>(g.out_lo + o) = lo;
          }
        }
      }
    }
    __syncwarp();
    if (has_skip) {
#pragma unroll
      for (int i = 0; i < 8; ++i) skip[i] = skip_next[i];
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Edge layers on CUDA cores (Cin = 1 / Cout = 1: not GEMM shaped, < 0.1 % of the codec's FLOPs, HBM-bound).
// encoder.conv1: x (B, 1, T) fp32 -> y (B, T, C) channels-last; stores the fp32 stream and snake_next(y) split hi/lo.
// One thread = four consecutive channels of one frame: 16-byte fp32 store + two 8-byte bf16 stores; the K input samples
// are shared by the whole row of threads (L1 broadcast).  Algorithmic bytes: 8 per output element.
__global__ void __launch_bounds__(256) codec_in_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                                       const float* __restrict__ bias, const float* __restrict__ alpha,
                                                       float* __restrict__ out_f32, __nv_bfloat16* __restrict__ out_hi,
                                                       __nv_bfloat16* __restrict__ out_lo, int B, int T, int C, int K,
                                                       int pad, const int* __restrict__ lens) {
  const int C4 = C >> 2;                                  // threads per frame
  const int per_block = blockDim.x / C4;                  // frames per block (host guarantees divisibility)
  const int t = blockIdx.x * per_block + static_cast<int>(threadIdx.x) / C4, b = blockIdx.y;
  if (t >= T) return;
  const int Tb = lens != nullptr ? lens[b] : T;           // this item's samples (ragged launch) or the launch's
  if (t >= Tb + CT_HALO) return;
  const int c = (static_cast<int>(threadIdx.x) % C4) * 4;
  const long long bt = static_cast<long long>(b) * T + t;
  if (t >= Tb) {                                          // halo of a ragged launch: +0 in all three outputs
    const long long o = bt * C + c;
    *reinterpret_cast<float4*>(out_f32 + o) = make_float4(0.f, 0.f, 0.f, 0.f);
    *reinterpret_cast<uint2*>(out_hi + o) = make_uint2(0u, 0u);
    *reinterpret_cast<uint2*>(out_lo + o) = make_uint2(0u, 0u);
    return;
  }
  const float4 b4 = __ldg(reinterpret_cast<const float4*>(bias + c));
  float acc[4] = {b4.x, b4.y, b4.z, b4.w};
  for (int k = 0; k < K; ++k) {
    const int xi = t + k - pad;
    if (xi >= 0 && xi < Tb) {
      const float xv = __ldg(x + static_cast<long long>(b) * T + xi);
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[j] = fmaf(__ldg(w + (c + j) * K + k), xv, acc[j]);
    }
  }
  const long long o = bt * C + c;
  *reinterpret_cast<float4*>(out_f32 + o) = make_float4(acc[0], acc[1], acc[2], acc[3]);
  const float4 al = __ldg(reinterpret_cast<const float4*>(alpha + c));
  const float a0 = snake_act(acc[0], al.x, 1.0f / (al.x + 1e-9f)), a1 = snake_act(acc[1], al.y, 1.0f / (al.y + 1e-9f));
  const float a2 = snake_act(acc[2], al.z, 1.0f / (al.z + 1e-9f)), a3 = snake_act(acc[3], al.w, 1.0f / (al.w + 1e-9f));
  const __nv_bfloat162 h01 = __floats2bfloat162_rn(a0, a1), h23 = __floats2bfloat162_rn(a2, a3);
  const float2 f01 = __bfloat1622float2(h01), f23 = __bfloat1622float2(h23);
  uint2 hi, lo;
  hi.x = *reinterpret_cast<const uint32_t*>(&h01);
  hi.y = *reinterpret_cast<const uint32_t*>(&h23);
  lo.x = pack_bf16x2(a0 - f01.x, a1 - f01.y);
  lo.y = pack_bf16x2(a2 - f23.x, a3 - f23.y);
  *reinterpret_cast<uint2*>(out_hi + o) = hi;
  *reinterpret_cast<uint2*>(out_lo + o) = lo;
}

// decoder.conv2: activated input (B, T, C) as hi/lo -> audio (B, 1, T) = tanh(bias + sum_k sum_c w[c, k] * a[t+k-pad, c]).
// One warp = 32 consecutive output samples.  Lanes own four channels each (C <= 128) and walk the 32 + K - 1 input frames
// once, every frame one coalesced row read (8 bytes of hi and of lo per lane); a frame feeds the K outputs it overlaps,
// so each lane carries 32 partial sums which a 5-step butterfly then reduces across lanes so that lane o ends up with
// output o.  All loads are independent of the arithmetic (38 x 2 in flight per lane).  Algorithmic bytes: 4*C per sample
// (+ 6/32 halo); the previous shared-memory version spent its time in 2-byte loads with an integer division each.
constexpr int CO_K = 7;
__global__ void __launch_bounds__(256) codec_out_kernel(const __nv_bfloat16* __restrict__ ah,
                                                        const __nv_bfloat16* __restrict__ al, const float* __restrict__ w,
                                                        const float* __restrict__ bias, float* __restrict__ audio, int B,
                                                        int T, int C, int pad, const int* __restrict__ lens) {
  const int lane = threadIdx.x & 31;
  const int t0 = (blockIdx.x * 8 + (threadIdx.x >> 5)) * 32;
  const int b = blockIdx.y;
  const int Tb = lens != nullptr ? lens[b] : T;   // this item's samples (ragged launch: input frames past it are not read)
  if (t0 >= Tb) return;
  const int c = lane * 4;
  const bool lane_on = c < C;
  float wr[4][CO_K];  // weight (1, C, K) -> this lane's [channel][tap]
#pragma unroll
  for (int j = 0; j < 4; ++j)
#pragma unroll
    for (int k = 0; k < CO_K; ++k) wr[j][k] = lane_on ? __ldg(w + (c + j) * CO_K + k) : 0.f;
  float acc[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) acc[i] = 0.f;
  const int c_safe = lane_on ? c : 0;
  const __nv_bfloat16* ph = ah + static_cast<long long>(b) * T * C + c_safe;
  const __nv_bfloat16* pl = al + static_cast<long long>(b) * T * C + c_safe;
#pragma unroll
  for (int r = 0; r < 32 + CO_K - 1; ++r) {
    const int t = t0 - pad + r;   // input frame; it is tap k of output r - k
    // unconditional loads from a clamped address (no branch between the loads: they are issued back to back and
    // their latency overlaps); frames outside the clip and idle lanes contribute zeros
    const bool ok = lane_on && t >= 0 && t < Tb;
    const long long off = static_cast<long long>(ok ? t : 0) * C;
    const uint2 h = __ldg(reinterpret_cast<const uint2*>(ph + off));
    const uint2 l = __ldg(reinterpret_cast<const uint2*>(pl + off));
    const float2 h01 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&h.x));
    const float2 h23 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&h.y));
    const float2 l01 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&l.x));
    const float2 l23 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&l.y));
    float v[4];
    v[0] = ok ? h01.x + l01.x : 0.f; v[1] = ok ? h01.y + l01.y : 0.f;
    v[2] = ok ? h23.x + l23.x : 0.f; v[3] = ok ? h23.y + l23.y : 0.f;
#pragma unroll
    for (int k = 0; k < CO_K; ++k) {
      const int o = r - k;
      if (o >= 0 && o < 32) {
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[o] = fmaf(wr[j][k], v[j], acc[o]);
      }
    }
  }
  // butterfly: after the step with distance s a lane keeps the half of its partial sums whose output index has bit s
  // equal to the lane's bit s, and adds the partner's partial sums for that half
#pragma unroll
  for (int s = 16; s >= 1; s >>= 1) {
    const bool up = (lane & s) != 0;
#pragma unroll
    for (int i = 0; i < s; ++i) {
      const float keep = up ? acc[i + s] : acc[i];
      const float send = up ? acc[i] : acc[i + s];
      acc[i] = keep + __shfl_xor_sync(0xffffffffu, send, s);
    }
  }
  const int t = t0 + lane;
  if (t < Tb) audio[static_cast<long long>(b) * T + t] = tanhf(bias[0] + acc[0]);
}

// Opts the four epilogue variants of width NW in to the large shared memory (once per device) and launches the one
// this layer needs: one CTA per tile.
template <int NW>
static cudaError_t launch_conv(const CUtensorMap& tAh, const CUtensorMap& tAl, const CUtensorMap& tWh,
                               const CUtensorMap& tWl, const ConvTcArgs& g, const float* bias, const float* alpha,
                               const float* resid, const float* out_f32, const void* out_hi, const void* out_lo,
                               int do_tanh, void* stream) {
  static PerDeviceOnce once;
  int dev;
  if (once.need(&dev)) {
    cudaError_t e = cudaFuncSetAttribute(conv_wgmma_kernel<CT_GENERIC, NW>, cudaFuncAttributeMaxDynamicSharedMemorySize, CT_SMEM);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(conv_wgmma_kernel<CT_SPLIT, NW>, cudaFuncAttributeMaxDynamicSharedMemorySize, CT_SMEM);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(conv_wgmma_kernel<CT_SPLIT_SKIP, NW>, cudaFuncAttributeMaxDynamicSharedMemorySize, CT_SMEM);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(conv_wgmma_kernel<CT_SPLIT_F32, NW>, cudaFuncAttributeMaxDynamicSharedMemorySize, CT_SMEM);
    if (e != cudaSuccess) return e;
    once.mark(dev);
  }
  const int tiles = g.Bn * ((g.Tq + CT_BM - 1) / CT_BM) * ((g.N + g.BN - 1) / g.BN);
  const dim3 grid(tiles);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  // the common layer shapes get a compile-time epilogue; anything else runs the run-time one
  const bool fast = bias && alpha && out_hi && out_lo && !do_tanh;
  if (fast && resid && out_f32 == resid) conv_wgmma_kernel<CT_SPLIT_SKIP, NW><<<grid, CT_THREADS, CT_SMEM, st>>>(tAh, tAl, tWh, tWl, g);
  else if (fast && !resid && out_f32) conv_wgmma_kernel<CT_SPLIT_F32, NW><<<grid, CT_THREADS, CT_SMEM, st>>>(tAh, tAl, tWh, tWl, g);
  else if (fast && !resid && !out_f32) conv_wgmma_kernel<CT_SPLIT, NW><<<grid, CT_THREADS, CT_SMEM, st>>>(tAh, tAl, tWh, tWl, g);
  else conv_wgmma_kernel<CT_GENERIC, NW><<<grid, CT_THREADS, CT_SMEM, st>>>(tAh, tAl, tWh, tWl, g);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------
// VGGish's first layer on CUDA cores (Cin = 1, K = 9: 0.4 % of the network's FLOPs): examples (Bn, 96, 64) fp32 ->
// relu(3x3 conv, pad 1, + bias) -> 2x2 max-pool -> (Bn, 48, 32, 64) NHWC, split hi/lo.  One thread = four channels of
// one pooled pixel: its 4x4 input patch, the four conv outputs under the pool, in fp32 with the taps in (dh, dw) order.
__global__ void __launch_bounds__(256) vggish_in_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                                        const float* __restrict__ bias, __nv_bfloat16* __restrict__ out_hi,
                                                        __nv_bfloat16* __restrict__ out_lo, int Bn) {
  constexpr int H = 96, W = 64, C = 64, H2 = H / 2, W2 = W / 2, C4 = C / 4;
  const long long pix = static_cast<long long>(blockIdx.x) * (256 / C4) + threadIdx.x / C4;  // (b, ph, pw)
  if (pix >= static_cast<long long>(Bn) * H2 * W2) return;
  const int c = (threadIdx.x % C4) * 4;
  const int b = static_cast<int>(pix / (H2 * W2)), rem = static_cast<int>(pix % (H2 * W2));
  const int h0 = (rem / W2) * 2 - 1, w0 = (rem % W2) * 2 - 1;
  const float* xb = x + static_cast<long long>(b) * H * W;
  float patch[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int h = h0 + i, ww = w0 + j;
      patch[i][j] = (h >= 0 && h < H && ww >= 0 && ww < W) ? __ldg(xb + h * W + ww) : 0.f;
    }
  float v[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const float bk = __ldg(bias + c + k);
    float m = -INFINITY;
#pragma unroll
    for (int oy = 0; oy < 2; ++oy)
#pragma unroll
      for (int ox = 0; ox < 2; ++ox) {
        float acc = bk;
#pragma unroll
        for (int t = 0; t < 9; ++t) acc = fmaf(__ldg(w + (c + k) * 9 + t), patch[oy + t / 3][ox + t % 3], acc);
        m = fmaxf(m, acc);
      }
    v[k] = fmaxf(m, 0.f);
  }
  const __nv_bfloat162 h01 = __floats2bfloat162_rn(v[0], v[1]), h23 = __floats2bfloat162_rn(v[2], v[3]);
  const float2 f01 = __bfloat1622float2(h01), f23 = __bfloat1622float2(h23);
  uint2 hi, lo;
  hi.x = *reinterpret_cast<const uint32_t*>(&h01);
  hi.y = *reinterpret_cast<const uint32_t*>(&h23);
  lo.x = pack_bf16x2(v[0] - f01.x, v[1] - f01.y);
  lo.y = pack_bf16x2(v[2] - f23.x, v[3] - f23.y);
  const long long o = pix * C + c;
  *reinterpret_cast<uint2*>(out_hi + o) = hi;
  *reinterpret_cast<uint2*>(out_lo + o) = lo;
}

cudaError_t launch_vggish_in(const float* x, const float* w, const float* bias, int Bn, void* out_hi, void* out_lo,
                             cudaStream_t st) {
  const long long pix = static_cast<long long>(Bn) * 48 * 32;
  vggish_in_kernel<<<static_cast<unsigned>((pix + 15) / 16), 256, 0, st>>>(
      x, w, bias, reinterpret_cast<__nv_bfloat16*>(out_hi), reinterpret_cast<__nv_bfloat16*>(out_lo), Bn);
  count_launch();
  return cudaGetLastError();
}

// One VGGish layer on the tensor cores at 128-column tiles (every N is a multiple of 128): a 3x3 convolution (W > 0:
// A = (Bn, H, W, Cin) NHWC, pool selects CT_RELU_POOL) or a fully connected layer (W = 0: A = (M, K) = (Bn, Cin), relu
// selects CT_RELU with hi/lo output, else fp32 output without activation).  TMA maps that cannot be encoded return
// cudaErrorInvalidValue with tmap_error() set.
cudaError_t launch_vggish_tc(const void* a_hi, const void* a_lo, int Bn, int H, int W, int Cin, const void* w_hi,
                             const void* w_lo, int N, const float* bias, bool relu, bool pool, void* out_hi,
                             void* out_lo, float* out_f32, cudaStream_t st) {
  static PerDeviceOnce once;
  int dev;
  if (once.need(&dev)) {
    cudaError_t e = cudaFuncSetAttribute(conv_wgmma_kernel<CT_RELU, 128>, cudaFuncAttributeMaxDynamicSharedMemorySize, CT_SMEM);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(conv_wgmma_kernel<CT_RELU_POOL, 128>, cudaFuncAttributeMaxDynamicSharedMemorySize, CT_SMEM);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(conv_wgmma_kernel<CT_GENERIC, 128>, cudaFuncAttributeMaxDynamicSharedMemorySize, CT_SMEM);
    if (e != cudaSuccess) return e;
    once.mark(dev);
  }
  ConvTcArgs g{};
  const bool conv = W > 0;
  g.Bn = conv ? Bn : 1; g.Tq = conv ? H * W : Bn; g.N = N; g.BN = 128;
  g.cblocks = (Cin + CT_BK - 1) / CT_BK; g.taps = conv ? 9 : 1; g.dil = 1; g.pad = 0; g.s = 1; g.Cin = Cin;
  g.bias = bias; g.bias_mod = N;
  g.out_hi = relu ? reinterpret_cast<__nv_bfloat16*>(out_hi) : nullptr;
  g.out_lo = relu ? reinterpret_cast<__nv_bfloat16*>(out_lo) : nullptr;
  g.out_f32 = relu ? nullptr : out_f32;
  g.out_batch_stride = static_cast<long long>(pool ? (H / 2) * (W / 2) : g.Tq) * N;
  g.out_limit = static_cast<long long>(g.Tq) * N;
  g.H = conv ? H : 0; g.W = conv ? W : 0;
  CUtensorMap tAh, tAl, tWh, tWl;
  const int Ktot = g.taps * g.cblocks * CT_BK;
  const bool ok = conv ? make_tmap_4d(&tAh, a_hi, Bn, H, W, Cin, CT_BM / W, CT_BK) &&
                             make_tmap_4d(&tAl, a_lo, Bn, H, W, Cin, CT_BM / W, CT_BK)
                       : make_tmap_3d(&tAh, a_hi, 1, Bn, Cin, Cin, CT_BM, CT_BK) &&
                             make_tmap_3d(&tAl, a_lo, 1, Bn, Cin, Cin, CT_BM, CT_BK);
  if (!ok || !make_tmap_2d(&tWh, w_hi, N, Ktot, g.BN, CT_BK) || !make_tmap_2d(&tWl, w_lo, N, Ktot, g.BN, CT_BK))
    return cudaErrorInvalidValue;
  const dim3 grid(g.Bn * ((g.Tq + CT_BM - 1) / CT_BM) * (N / g.BN));
  if (pool) conv_wgmma_kernel<CT_RELU_POOL, 128><<<grid, CT_THREADS, CT_SMEM, st>>>(tAh, tAl, tWh, tWl, g);
  else if (relu) conv_wgmma_kernel<CT_RELU, 128><<<grid, CT_THREADS, CT_SMEM, st>>>(tAh, tAl, tWh, tWl, g);
  else conv_wgmma_kernel<CT_GENERIC, 128><<<grid, CT_THREADS, CT_SMEM, st>>>(tAh, tAl, tWh, tWl, g);
  count_launch();
  return cudaGetLastError();
}

}  // namespace vnb

using namespace vnb;

static int32_t conv_tc(const void* a_hi, const void* a_lo, int32_t B, int32_t Tin, int32_t Cin, int32_t s,
                       const void* w_hi, const void* w_lo, int32_t N, int32_t taps, int32_t dil, int32_t pad, int32_t Tq,
                       const float* bias, int32_t bias_mod, const float* alpha, int32_t alpha_mod, const float* resid,
                       float* out_f32, void* out_hi, void* out_lo, int64_t out_batch_stride, int64_t out_offset,
                       int64_t out_limit, int32_t do_tanh, const int32_t* lens, int32_t row_elems, void* stream) {
  if (Tin % s != 0) return vnb_set_error_cuda("vnb_codec_conv_tc: Tin must be a multiple of the stride", 1);
  if (N % 32 != 0 || Cin % 4 != 0) return vnb_set_error_cuda("vnb_codec_conv_tc: N % 32 and Cin % 4 required", 1);
  ConvTcArgs g;
  g.Bn = B; g.Tq = Tq; g.N = N;
  g.BN = N >= 128 ? 128 : N;         // N in {64, 96, 128, ...}: multiples of 32 up to 128
  if (N > 128 && N % 128 != 0) g.BN = (N % 96 == 0) ? 96 : 64;
  g.cblocks = (Cin + CT_BK - 1) / CT_BK; g.taps = taps; g.dil = dil; g.pad = pad; g.s = s; g.Cin = Cin;
  g.bias = bias; g.bias_mod = bias_mod; g.alpha = alpha; g.alpha_mod = alpha_mod; g.resid = resid; g.out_f32 = out_f32;
  g.out_hi = reinterpret_cast<__nv_bfloat16*>(out_hi); g.out_lo = reinterpret_cast<__nv_bfloat16*>(out_lo);
  g.out_batch_stride = out_batch_stride; g.out_offset = out_offset; g.out_limit = out_limit; g.do_tanh = do_tanh;
  g.lens = lens; g.row_elems = row_elems;
  const int Ktot = taps * g.cblocks * CT_BK;
  CUtensorMap tAh, tAl, tWh, tWl;
  const uint64_t rows = static_cast<uint64_t>(Tin / s), cols = static_cast<uint64_t>(s) * Cin;
  if (!make_tmap_3d(&tAh, a_hi, B, rows, cols, cols, CT_BM, CT_BK) || !make_tmap_3d(&tAl, a_lo, B, rows, cols, cols, CT_BM, CT_BK) ||
      !make_tmap_2d(&tWh, w_hi, N, Ktot, g.BN, CT_BK) || !make_tmap_2d(&tWl, w_lo, N, Ktot, g.BN, CT_BK))
    return vnb_set_error_cuda(tmap_error(), 1);
  cudaError_t e = g.BN <= 32 ? launch_conv<32>(tAh, tAl, tWh, tWl, g, bias, alpha, resid, out_f32, out_hi, out_lo, do_tanh, stream)
                  : g.BN <= 64 ? launch_conv<64>(tAh, tAl, tWh, tWl, g, bias, alpha, resid, out_f32, out_hi, out_lo, do_tanh, stream)
                               : launch_conv<128>(tAh, tAl, tWh, tWl, g, bias, alpha, resid, out_f32, out_hi, out_lo, do_tanh, stream);
  if (e != cudaSuccess) return vnb_set_error_cuda("conv_wgmma_kernel launch", static_cast<int>(e));
  count_launch();
  return 0;
}

static int32_t conv_in(const float* x, const float* w, const float* bias, const float* alpha, float* out_f32,
                       void* out_hi, void* out_lo, int32_t B, int32_t T, int32_t C, int32_t K, int32_t pad,
                       const int32_t* lens, void* stream) {
  if (C % 4 != 0 || 256 % (C / 4) != 0) return vnb_set_error_cuda("vnb_codec_conv_in: C/4 must divide 256", 1);
  const int per_block = 256 / (C / 4);
  dim3 grid((T + per_block - 1) / per_block, B);
  codec_in_kernel<<<grid, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      x, w, bias, alpha, out_f32, reinterpret_cast<__nv_bfloat16*>(out_hi), reinterpret_cast<__nv_bfloat16*>(out_lo), B, T,
      C, K, pad, lens);
  cudaError_t e = cudaGetLastError();
  if (e == cudaSuccess) count_launch();
  return e == cudaSuccess ? 0 : vnb_set_error_cuda("codec_in_kernel", static_cast<int>(e));
}

static int32_t conv_out(const void* a_hi, const void* a_lo, const float* w, const float* bias, float* audio, int32_t B,
                        int32_t T, int32_t C, int32_t K, int32_t pad, const int32_t* lens, void* stream) {
  if (K != CO_K || C % 4 != 0 || C > 128)
    return vnb_set_error_cuda("vnb_codec_conv_out: kernel size 7 and C % 4 == 0, C <= 128 required", 1);
  dim3 grid((T + 255) / 256, B);
  codec_out_kernel<<<grid, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const __nv_bfloat16*>(a_hi), reinterpret_cast<const __nv_bfloat16*>(a_lo), w, bias, audio, B, T, C,
      pad, lens);
  cudaError_t e = cudaGetLastError();
  if (e == cudaSuccess) count_launch();
  return e == cudaSuccess ? 0 : vnb_set_error_cuda("codec_out_kernel", static_cast<int>(e));
}

extern "C" {

int32_t vnb_codec_conv_tc(const void* a_hi, const void* a_lo, int32_t B, int32_t Tin, int32_t Cin, int32_t s,
                          const void* w_hi, const void* w_lo, int32_t N, int32_t taps, int32_t dil, int32_t pad,
                          int32_t Tq, const float* bias, int32_t bias_mod, const float* alpha, int32_t alpha_mod,
                          const float* resid, float* out_f32, void* out_hi, void* out_lo, int64_t out_batch_stride,
                          int64_t out_offset, int64_t out_limit, int32_t do_tanh, void* stream) {
  return conv_tc(a_hi, a_lo, B, Tin, Cin, s, w_hi, w_lo, N, taps, dil, pad, Tq, bias, bias_mod, alpha, alpha_mod, resid,
                 out_f32, out_hi, out_lo, out_batch_stride, out_offset, out_limit, do_tanh, nullptr, 0, stream);
}

int32_t vnb_codec_conv_tc_ragged(const void* a_hi, const void* a_lo, int32_t B, int32_t Tin, int32_t Cin, int32_t s,
                                 const void* w_hi, const void* w_lo, int32_t N, int32_t taps, int32_t dil, int32_t pad,
                                 int32_t Tq, const float* bias, int32_t bias_mod, const float* alpha, int32_t alpha_mod,
                                 const float* resid, float* out_f32, void* out_hi, void* out_lo,
                                 int64_t out_batch_stride, int64_t out_offset, int64_t out_limit, int32_t do_tanh,
                                 const int32_t* lens, int32_t row_elems, void* stream) {
  if (lens == nullptr || row_elems < 1)
    return vnb_set_error_cuda("vnb_codec_conv_tc_ragged: a length table and row_elems >= 1 required", 1);
  return conv_tc(a_hi, a_lo, B, Tin, Cin, s, w_hi, w_lo, N, taps, dil, pad, Tq, bias, bias_mod, alpha, alpha_mod, resid,
                 out_f32, out_hi, out_lo, out_batch_stride, out_offset, out_limit, do_tanh, lens, row_elems, stream);
}

int32_t vnb_codec_conv_in(const float* x, const float* w, const float* bias, const float* alpha, float* out_f32,
                          void* out_hi, void* out_lo, int32_t B, int32_t T, int32_t C, int32_t K, int32_t pad,
                          void* stream) {
  return conv_in(x, w, bias, alpha, out_f32, out_hi, out_lo, B, T, C, K, pad, nullptr, stream);
}

int32_t vnb_codec_conv_in_ragged(const float* x, const float* w, const float* bias, const float* alpha, float* out_f32,
                                 void* out_hi, void* out_lo, int32_t B, int32_t T, int32_t C, int32_t K, int32_t pad,
                                 const int32_t* lens, void* stream) {
  if (lens == nullptr) return vnb_set_error_cuda("vnb_codec_conv_in_ragged: a length table is required", 1);
  return conv_in(x, w, bias, alpha, out_f32, out_hi, out_lo, B, T, C, K, pad, lens, stream);
}

int32_t vnb_codec_conv_out(const void* a_hi, const void* a_lo, const float* w, const float* bias, float* audio, int32_t B,
                           int32_t T, int32_t C, int32_t K, int32_t pad, void* stream) {
  return conv_out(a_hi, a_lo, w, bias, audio, B, T, C, K, pad, nullptr, stream);
}

int32_t vnb_codec_conv_out_ragged(const void* a_hi, const void* a_lo, const float* w, const float* bias, float* audio,
                                  int32_t B, int32_t T, int32_t C, int32_t K, int32_t pad, const int32_t* lens,
                                  void* stream) {
  if (lens == nullptr) return vnb_set_error_cuda("vnb_codec_conv_out_ragged: a length table is required", 1);
  return conv_out(a_hi, a_lo, w, bias, audio, B, T, C, K, pad, lens, stream);
}
}
