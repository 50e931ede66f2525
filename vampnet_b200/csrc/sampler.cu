// vampnet_b200 — one sampling iteration of VampNet.generate, after the logits exist
// (reference vampnet/modules/transformer.py:849-932): sample_from_logits (:952-1034; typical_filter's
// result is discarded by the reference and so is absent here), the where()s that keep known tokens,
// the cosine-schedule count (:903-913, mask.py:8-9) and mask_by_random_topk (:1038-1074).
//
// In the generate loop the draw itself happens inside the classifier GEMM's epilogue (gemm_wgmma.cu, EPI_SAMPLE: the
// logits never reach HBM); what runs here afterwards:
//   sample_combine_kernel  one thread per (batch, position): picks the 128-entry vocabulary tile from the per-tile
//                          records the epilogue left (uniform 1), takes that tile's candidate, writes token + confidence.
//   remask_kernel          one CTA per batch row: exact k-th order statistic of the S confidences by a 4-pass radix
//                          select (what sort()[k] yields in the reference), then z <- where(conf < cut, MASK, token).
// With nucleus (top-p) sampling, with vnb_set_option("fused_sampler", 0) and through vnb_sample_step the logits are a
// tensor and the draw is
//   sample_rows_kernel     one warp per (batch, position): reads the 1024 logits of a STILL-MASKED position once (32 per
//                          lane, float4), warp-shuffle max / sum-exp, the same two-level inverse-CDF draw with two
//                          counter-based Philox uniforms per row, writes token + confidence.  Known positions cost
//                          4 bytes.  Algorithmic bytes: V*4 per masked position.
// A fused launch that mixes nucleus and plain groups runs both draws after the split classifier epilogue, each kernel
// on its own groups' rows only: sample_combine_kernel<true> from the records, sample_rows_kernel<true, true> from the
// logits the epilogue stored for the nucleus rows; then remask_kernel.
#include "common.cuh"
#include "kernels.h"

namespace vnb {

__device__ __forceinline__ float gumbel(float u) { return -logf(-logf(u)); }

using SampleDynDev = SampleDyn;

__device__ __forceinline__ uint32_t f2key(float f) {  // order-preserving float -> uint
  const uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

struct SampleStatic {
  const float* logits;
  int32_t* zcur;
  const int32_t* zorig;
  int32_t* tokens;
  float* conf;
  const int32_t* n0;
  const RowGroup* rowgrp;
  int B, T, C, ncc, V, mask_token;
  const int32_t* live;  // (1) batch rows b >= live[0] are idle this iteration and left untouched; null: all live
};

// TOPP = false compiles the nucleus filter out (its 32 extra live registers cost occupancy on the common path).
// SPLIT (with TOPP): a launch of nucleus and plain groups; this kernel serves the rows of nucleus groups only and leaves
// the others to sample_combine_kernel<true>.
template <bool TOPP, bool SPLIT = false>
__global__ void __launch_bounds__(256, TOPP ? 2 : 3) sample_rows_kernel(const SampleStatic a, const SampleDynDev* __restrict__ dynp) {
  const int Cp = a.C - a.ncc;
  const int S = a.T * Cp;
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= a.B * S) return;
  const int lane = threadIdx.x & 31;
  const int b = row / S, s = row - b * S;
  if (a.live != nullptr && b >= __ldg(a.live)) return;  // an idle call's row: its state is not touched
  const RowGroup rg = a.rowgrp[b];
  const SampleDynDev dyn = dynp[rg.group];
  if constexpr (SPLIT) {
    if (!(dyn.top_p > 0.f && dyn.top_p < 1.f)) return;  // a plain group's row: not touched
  }
  const uint32_t bg = static_cast<uint32_t>(b - rg.first);  // Philox counter word: the row within its own call
  const int t = s / Cp, cp = s - t * Cp;
  const int zi = a.zcur[(static_cast<size_t>(b) * a.T + t) * a.C + a.ncc + cp];
  if (zi != a.mask_token) {  // known token: kept, never re-masked (transformer.py:893-900)
    if (lane == 0) {
      a.tokens[row] = zi;
      a.conf[row] = INFINITY;
    }
    return;
  }
  const int V = a.V;  // 1024 -> 8 float4 per lane
  const float4* lr = reinterpret_cast<const float4*>(a.logits + static_cast<size_t>(row) * V);
  constexpr int MAXV4 = 8;
  float4 x[MAXV4];
  const int n4 = V >> 7;  // float4s per lane
  float mx = -INFINITY;
#pragma unroll
  for (int i = 0; i < MAXV4; ++i) {
    if (i < n4) {
      float4 v = lr[i * 32 + lane];
      x[i] = v;
      mx = fmaxf(mx, fmaxf(fmaxf(v.x, v.y), fmaxf(v.z, v.w)));
    }
  }
  // nucleus (top-p) filtering on the RAW logits (reference transformer.py:1001-1016): sorted descending, a token is
  // removed when the softmax mass of the tokens strictly before it exceeds top_p ("shift right by one" keeps the
  // first token over the threshold).  Equivalent per-token rule: keep v iff sum_{u: x_u > x_v} p_u <= top_p.
  // The smallest kept key is found by bisection over the order-preserving uint image of the floats.
  if (TOPP && dyn.top_p > 0.f && dyn.top_p < 1.f) {
    // +0 and -0 are one logit value (a tie, kept or dropped whole) but have different keys: make every zero +0.  No
    // other use of x can tell the two apart.
#pragma unroll
    for (int i = 0; i < MAXV4; ++i) {
      if (i < n4) { x[i].x += 0.f; x[i].y += 0.f; x[i].z += 0.f; x[i].w += 0.f; }
    }
    const float gm = warp_max(mx);
    float pr[MAXV4 * 4];
    float ps = 0.f;
#pragma unroll
    for (int i = 0; i < MAXV4; ++i) {
      if (i < n4) {
        const float xs[4] = {x[i].x, x[i].y, x[i].z, x[i].w};
#pragma unroll
        for (int j = 0; j < 4; ++j) { pr[i * 4 + j] = expf(xs[j] - gm); ps += pr[i * 4 + j]; }
      }
    }
    ps = warp_sum(ps);
    const float budget = dyn.top_p * ps;  // compare un-normalised masses
    uint32_t lo = 0u, hi = 0xFFFFFFFFu;
    for (int it = 0; it < 32; ++it) {
      const uint32_t mid = lo + ((hi - lo) >> 1);
      float above = 0.f;
#pragma unroll
      for (int i = 0; i < MAXV4; ++i) {
        if (i < n4) {
          const float xs[4] = {x[i].x, x[i].y, x[i].z, x[i].w};
#pragma unroll
          for (int j = 0; j < 4; ++j) above += f2key(xs[j]) > mid ? pr[i * 4 + j] : 0.f;
        }
      }
      above = warp_sum(above);
      if (above <= budget) hi = mid; else lo = mid + 1u;
    }
    mx = -INFINITY;
#pragma unroll
    for (int i = 0; i < MAXV4; ++i) {
      if (i < n4) {
        if (f2key(x[i].x) < lo) x[i].x = -INFINITY;
        if (f2key(x[i].y) < lo) x[i].y = -INFINITY;
        if (f2key(x[i].z) < lo) x[i].z = -INFINITY;
        if (f2key(x[i].w) < lo) x[i].w = -INFINITY;
        mx = fmaxf(mx, fmaxf(fmaxf(x[i].x, x[i].y), fmaxf(x[i].z, x[i].w)));
      }
    }
  }
  // arg-max of the raw logits (greedy) or of logits*inv_t + Gumbel (sampling), lowest index on ties
  // greedy arg-max of the raw logits, lowest index on ties (torch.argmax) -- also the fallback of the sampler
  float best = -INFINITY;
  int best_i = 0x7fffffff;
#pragma unroll
  for (int i = 0; i < MAXV4; ++i) {
    if (i < n4) {
      const int i4 = i * 32 + lane;
      const float xs[4] = {x[i].x, x[i].y, x[i].z, x[i].w};
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (xs[j] > best) { best = xs[j]; best_i = i4 * 4 + j; }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ob = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, best_i, o);
    if (ob > best || (ob == best && oi < best_i)) { best = ob; best_i = oi; }
  }
  mx = warp_max(mx);
  const float m = __fmul_rn(mx, dyn.inv_temp);  // inv_t > 0 so the max commutes
  // un-normalised probabilities e_v = exp(x_v * inv_t - m); lane `l` holds v = i*128 + l*4 + j: consecutive
  // vocabulary entries, so a categorical draw by inverse CDF in natural vocabulary order needs only one prefix
  // scan per 128-entry chunk.  torch.multinomial (transformer.py:1025) draws from the same distribution.
  float e[MAXV4][4], csum[MAXV4];
  float se = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV4; ++i) {
    csum[i] = 0.f;
    if (i < n4) {
      const float xs[4] = {x[i].x, x[i].y, x[i].z, x[i].w};
      float ls = 0.f;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        e[i][j] = expf(__fmul_rn(xs[j], dyn.inv_temp) - m);
        ls += e[i][j];
      }
      csum[i] = ls;                 // this lane's 4 entries of chunk i
      se += warp_sum(ls);           // chunk totals added in chunk order
    }
  }
  if (dyn.do_sample) {
    uint32_t r[4];
    philox4x32_10(static_cast<uint32_t>(s), bg, static_cast<uint32_t>(dyn.step), 0u, dyn.seed_lo, dyn.seed_hi, r);
    // Two-level inverse CDF (oracle/vampnet_oracle.py sample_from_logits, rng="philox"): uniform 1 picks the
    // 128-entry tile (= chunk i of this layout) by its mass, uniform 2 the entry inside it.  The classifier GEMM's
    // sampling epilogue (gemm_wgmma.cu, EPI_SAMPLE) draws the same way from its own 128-column strips.
    const float target = u01(r[0]) * se;  // tile = first i with cumsum(tile mass)[i] > target
    const float u2 = u01(r[1]);
    float base = 0.f;
    int pick = -1;
#pragma unroll
    for (int i = 0; i < MAXV4; ++i) {
      if (i < n4 && pick < 0) {
        const float tot = warp_sum(csum[i]);
        if (base + tot > target) {
          const float target_in = u2 * tot;  // token = first v of the tile with cumsum(e)[v] > target_in
          // inclusive scan of the lane sums of this chunk (Hillis-Steele)
          float inc = csum[i];
#pragma unroll
          for (int o = 1; o < 32; o <<= 1) {
            const float t = __shfl_up_sync(0xffffffffu, inc, o);
            if (lane >= o) inc += t;
          }
          const float before = inc - csum[i];
          int cand = 0x7fffffff;
          if (inc > target_in) {  // the crossing is at or before this lane's last entry
            float run = before;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              run += e[i][j];
              if (run > target_in && cand == 0x7fffffff) cand = (i * 32 + lane) * 4 + j;
            }
          }
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) cand = min(cand, __shfl_xor_sync(0xffffffffu, cand, o));
          if (cand == 0x7fffffff) {
            // rounding left target_in >= the tile's mass: the tile's largest entry (lowest index on ties)
            float tb = -INFINITY;
            int ti = 0x7fffffff;
            const float xs[4] = {x[i].x, x[i].y, x[i].z, x[i].w};
#pragma unroll
            for (int j = 0; j < 4; ++j)
              if (xs[j] > tb) { tb = xs[j]; ti = (i * 32 + lane) * 4 + j; }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
              const float ob = __shfl_xor_sync(0xffffffffu, tb, o);
              const int oi = __shfl_xor_sync(0xffffffffu, ti, o);
              if (ob > tb || (ob == tb && oi < ti)) { tb = ob; ti = oi; }
            }
            cand = ti;
          }
          pick = cand;
        }
        base += tot;
      }
    }
    if (pick >= 0 && pick < V) best_i = pick;  // else (rounding left target >= total): keep the arg-max
  }
  // softmax probability of the chosen token: probs = softmax(logits * inv_t) (transformer.py:1019-1023)
  float xt = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV4; ++i) {
    if (i < n4) {
      const int i4 = i * 32 + lane;
      const float xs[4] = {x[i].x, x[i].y, x[i].z, x[i].w};
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (i4 * 4 + j == best_i) xt = __fmul_rn(xs[j], dyn.inv_temp);
    }
  }
  xt = warp_sum(xt);  // exactly one lane contributed
  if (lane == 0) {
    const float p = expf(xt - m) / se;
    uint32_t r[4];
    philox4x32_10(static_cast<uint32_t>(s), bg, static_cast<uint32_t>(dyn.step), 1u, dyn.seed_lo, dyn.seed_hi, r);
    // confidence = log p + temperature * Gumbel (transformer.py:1055-1057)
    const float cf = __fadd_rn(logf(p), __fmul_rn(dyn.temp_eff, gumbel(u01(r[0]))));
    a.tokens[row] = best_i;
    a.conf[row] = cf;
  }
}

__global__ void __launch_bounds__(1024) remask_kernel(const SampleStatic a, const SampleDynDev* __restrict__ dynp) {
  const int Cp = a.C - a.ncc;
  const int S = a.T * Cp;
  const int b = blockIdx.x;
  if (a.live != nullptr && b >= __ldg(a.live)) return;  // an idle call's row: zcur is not touched
  const int grp = a.rowgrp[b].group;
  const SampleDynDev dyn = dynp[grp];
  const float* conf = a.conf + static_cast<size_t>(b) * S;
  const int32_t* tok = a.tokens + static_cast<size_t>(b) * S;
  int32_t* zrow = a.zcur + static_cast<size_t>(b) * a.T * a.C;
  __shared__ unsigned hist[256];
  __shared__ unsigned s_prefix, s_maskbits;
  __shared__ int s_rank, s_cnt;

  if (threadIdx.x == 0) s_cnt = 0;
  __syncthreads();
  // masked positions in this row before the update (mask.sum(dim=-1), transformer.py:906-913)
  int local = 0;
  for (int s = threadIdx.x; s < S; s += blockDim.x) {
    const int t = s / Cp, cp = s - t * Cp;
    local += (zrow[t * a.C + a.ncc + cp] == a.mask_token);
  }
  for (int o = 16; o > 0; o >>= 1) local += __shfl_xor_sync(0xffffffffu, local, o);
  if ((threadIdx.x & 31) == 0 && local) atomicAdd(&s_cnt, local);
  __syncthreads();
  if (threadIdx.x == 0) {
    // num_to_mask = floor(gamma(r) * N0) in fp32 (transformer.py:903), N0 of this row's call, clamped unless last step
    int n = static_cast<int>(floorf(__fmul_rn(dyn.gamma, static_cast<float>(a.n0[grp]))));
    if (!dyn.is_last) {
      int up = s_cnt - 1;
      if (n > up) n = up;
      if (n < 1) n = 1;
    }
    if (n > S - 1) n = S - 1;
    if (n < 0) n = 0;
    s_rank = n;
    s_prefix = 0;
    s_maskbits = 0;
  }
  __syncthreads();
  // radix select: key of the element at sorted position n (ascending)
  for (int pass = 3; pass >= 0; --pass) {
    for (int i = threadIdx.x; i < 256; i += blockDim.x) hist[i] = 0;
    __syncthreads();
    const unsigned prefix = s_prefix, mb = s_maskbits;
    for (int s = threadIdx.x; s < S; s += blockDim.x) {
      const uint32_t k = f2key(conf[s]);
      if ((k & mb) == prefix) atomicAdd(&hist[(k >> (8 * pass)) & 255u], 1u);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      int rank = s_rank;
      unsigned cum = 0;
      int bkt = 0;
      for (; bkt < 255; ++bkt) {
        if (cum + hist[bkt] > static_cast<unsigned>(rank)) break;
        cum += hist[bkt];
      }
      s_rank = rank - static_cast<int>(cum);
      s_prefix = prefix | (static_cast<unsigned>(bkt) << (8 * pass));
      s_maskbits = mb | (0xFFu << (8 * pass));
    }
    __syncthreads();
  }
  const uint32_t cut = s_prefix;
  // z_masked = where(conf < cut, MASK, sampled_z) (transformer.py:922-924); conditioning codebooks are
  // re-attached from the ORIGINAL z (transformer.py:930-932)
  for (int s = threadIdx.x; s < S; s += blockDim.x) {
    const int t = s / Cp, cp = s - t * Cp;
    const bool rm = f2key(conf[s]) < cut;
    zrow[t * a.C + a.ncc + cp] = rm ? a.mask_token : tok[s];
  }
  if (a.zorig != nullptr && a.ncc > 0) {
    const int32_t* zo = a.zorig + static_cast<size_t>(b) * a.T * a.C;
    for (int i = threadIdx.x; i < a.T * a.ncc; i += blockDim.x) {
      const int t = i / a.ncc, c = i - t * a.ncc;
      zrow[t * a.C + c] = zo[t * a.C + c];
    }
  }
}

// Second half of the fused path.  The classifier GEMM's sampling epilogue (gemm_wgmma.cu, EPI_SAMPLE) left one
// 16-byte record per (row, 128-entry vocabulary tile): {tile max of the logits, sum of exp((x - max) / temperature),
// logit of the tile's candidate, candidate | arg-max << 16 (vocabulary indices)}; the candidate was drawn inside the tile
// with uniform 2.  One thread per row: pick the tile with uniform 1 by mass, take its candidate, and compute
// confidence = log softmax(token) + temperature * Gumbel exactly as sample_rows_kernel does.  The logits themselves
// never reach HBM.  Algorithmic bytes: 16 * V/128 per masked row.
// SPLIT: a launch of nucleus and plain groups; the rows of nucleus groups are left to sample_rows_kernel<true, true>.
template <bool SPLIT>
__global__ void __launch_bounds__(256) sample_combine_kernel(const SampleStatic a, const float4* __restrict__ partials,
                                                             const SampleDynDev* __restrict__ dynp) {
  const int Cp = a.C - a.ncc;
  const int S = a.T * Cp;
  const int row = blockIdx.x * blockDim.x + threadIdx.x;
  if (row >= a.B * S) return;
  const int b = row / S, s = row - b * S;
  if (a.live != nullptr && b >= __ldg(a.live)) return;  // an idle call's row: tokens and confidences are not touched
  const RowGroup rg = a.rowgrp[b];
  const SampleDynDev dyn = dynp[rg.group];
  if constexpr (SPLIT) {
    if (dyn.top_p > 0.f && dyn.top_p < 1.f) return;  // a nucleus group's row: not touched
  }
  const uint32_t bg = static_cast<uint32_t>(b - rg.first);
  const int t = s / Cp, cp = s - t * Cp;
  const int zi = a.zcur[(static_cast<size_t>(b) * a.T + t) * a.C + a.ncc + cp];
  if (zi != a.mask_token) {  // known token: kept, never re-masked (transformer.py:893-900)
    a.tokens[row] = zi;
    a.conf[row] = INFINITY;
    return;
  }
  constexpr int MAXT = 8;
  const int nt = a.V >> 7;
  float4 rec[MAXT];
  float M = -INFINITY;
  int kmax = 0;
#pragma unroll
  for (int k = 0; k < MAXT; ++k) {
    if (k < nt) {
      rec[k] = __ldg(partials + static_cast<size_t>(row) * nt + k);
      if (rec[k].x > M) { M = rec[k].x; kmax = k; }
    }
  }
  const float c1 = __fmul_rn(dyn.inv_temp, 1.4426950408889634f);
  float mass[MAXT], total = 0.f;
#pragma unroll
  for (int k = 0; k < MAXT; ++k) {
    mass[k] = 0.f;
    if (k < nt) {
      mass[k] = rec[k].y * fast_exp2(__fmul_rn(rec[k].x - M, c1));
      total += mass[k];
    }
  }
  int kk = kmax;
  if (dyn.do_sample) {
    uint32_t r[4];
    philox4x32_10(static_cast<uint32_t>(s), bg, static_cast<uint32_t>(dyn.step), 0u, dyn.seed_lo, dyn.seed_hi, r);
    const float target = u01(r[0]) * total;
    float run = 0.f;
    int pick = -1;
#pragma unroll
    for (int k = 0; k < MAXT; ++k) {
      if (k < nt) {
        run += mass[k];
        if (run > target && pick < 0) pick = k;
      }
    }
    if (pick >= 0) kk = pick;
  }
  float xc = 0.f;
  uint32_t bits = 0;
#pragma unroll
  for (int k = 0; k < MAXT; ++k)
    if (k == kk) { xc = rec[k].z; bits = __float_as_uint(rec[k].w); }
  const int token = dyn.do_sample ? static_cast<int>(bits & 0xffffu) : static_cast<int>(bits >> 16);
  const float p = fast_exp2(__fmul_rn(xc - M, c1)) / total;
  uint32_t r[4];
  philox4x32_10(static_cast<uint32_t>(s), bg, static_cast<uint32_t>(dyn.step), 1u, dyn.seed_lo, dyn.seed_hi, r);
  a.tokens[row] = token;
  a.conf[row] = __fadd_rn(logf(p), __fmul_rn(dyn.temp_eff, gumbel(u01(r[0]))));
}

static SampleStatic make_static(const SampleArgs& s) {
  SampleStatic a;
  a.logits = s.logits; a.zcur = s.zcur; a.zorig = s.zorig; a.tokens = s.tokens; a.conf = s.conf; a.n0 = s.n0;
  a.rowgrp = s.rowgrp;
  a.B = s.B; a.T = s.T; a.C = s.C; a.ncc = s.ncc; a.V = s.V; a.mask_token = s.mask_token;
  a.live = s.live;
  return a;
}

cudaError_t launch_remask_dev(const SampleArgs& s, const SampleDyn* dyn_dev, cudaStream_t st) {
  remask_kernel<<<s.B, 1024, 0, st>>>(make_static(s), dyn_dev);
  return cudaGetLastError();
}

cudaError_t launch_sample_step_dev(const SampleArgs& s, const SampleDyn* dyn_dev, cudaStream_t st, bool use_top_p) {
  const SampleStatic a = make_static(s);
  if (s.V % 128 != 0 || s.V > 1024) return cudaErrorInvalidValue;
  const int rows = s.B * s.T * (s.C - s.ncc);
  if (use_top_p) sample_rows_kernel<true><<<(rows + 7) / 8, 256, 0, st>>>(a, dyn_dev);
  else sample_rows_kernel<false><<<(rows + 7) / 8, 256, 0, st>>>(a, dyn_dev);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  return launch_remask_dev(s, dyn_dev, st);
}

cudaError_t launch_sample_combine_dev(const SampleArgs& s, const void* partials, const SampleDyn* dyn_dev, cudaStream_t st) {
  const SampleStatic a = make_static(s);
  if (s.V % 128 != 0 || s.V > 1024) return cudaErrorInvalidValue;
  const int rows = s.B * s.T * (s.C - s.ncc);
  sample_combine_kernel<false><<<(rows + 255) / 256, 256, 0, st>>>(a, reinterpret_cast<const float4*>(partials), dyn_dev);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  return launch_remask_dev(s, dyn_dev, st);
}

cudaError_t launch_sample_split_dev(const SampleArgs& s, const void* partials, const SampleDyn* dyn_dev, cudaStream_t st) {
  const SampleStatic a = make_static(s);
  if (s.V % 128 != 0 || s.V > 1024) return cudaErrorInvalidValue;
  const int rows = s.B * s.T * (s.C - s.ncc);
  sample_combine_kernel<true><<<(rows + 255) / 256, 256, 0, st>>>(a, reinterpret_cast<const float4*>(partials), dyn_dev);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  sample_rows_kernel<true, true><<<(rows + 7) / 8, 256, 0, st>>>(a, dyn_dev);
  e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  return launch_remask_dev(s, dyn_dev, st);
}

}  // namespace vnb
