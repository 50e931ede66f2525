// vampnet_b200 — onset detection for the onset-prompt mask (reference vampnet/mask.py:203-226, which calls librosa
// 0.10's onset.onset_detect(y, sr, hop_length=H, backtrack=True)), all on one stream with no host round trip:
//   mel_spec_kernel     (mel.cu, ONSET_DB mode) one CTA per (frame, row): Hann-windowed zero-padded frame -> fp32
//                       2048-point real FFT -> |X|^2 -> 128 Slaney mel bands -> 10 log10(max(1e-10, S))
//   onset_pick_kernel   one CTA per row: the clip's dB maximum (top_db = 80 clamp), the clamped spectral flux
//                       averaged over the bands, shifted and trimmed, normalised to [0, 1]; every frame's peak and
//                       minimum tests in parallel, then one warp walks them 32 frames at a time for peak_pick's
//                       wait rule and onset_backtrack
//   onset_mask_kernel   the reference's mask[:, :, idx - w:idx + w] = 0 loop, with Python slice semantics
// DESIGN.md §9 has the numerics; oracle/onset_oracle.py restates the algorithm in float64.  The peak-pick geometry is
// host arithmetic here; the FFT tables and the mel bank are mel.cu's, cached by device_table.
#include <algorithm>
#include <cmath>

#include "kernels.h"
#include "reduce.cuh"

namespace vnb {

namespace {
constexpr int NMELS = ONSET_NMELS, THREADS = 256, WARPS = THREADS / 32;

__global__ void __launch_bounds__(THREADS) onset_pick_kernel(float* db, int F, int pad, OnsetTables t, int backtrack,
                                                             float* __restrict__ env_out, int32_t* __restrict__ onsets,
                                                             int32_t* __restrict__ counts) {
  __shared__ float red[WARPS];
  const int b = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const float* d = db + (size_t)b * F * NMELS;
  float* env = env_out + (size_t)b * F;
  // power_to_db's top_db clamp: the maximum over the whole clip
  float mx = -INFINITY;
  for (size_t i = threadIdx.x; i < (size_t)F * NMELS; i += THREADS) mx = fmaxf(mx, d[i]);
  const float floor_db = block_reduce<Reduce::MAX, WARPS>(mx, red) - 80.f;
  // flux S[t] - S[t-1] clamped at 0, mean over bands, left-padded by `pad` frames and trimmed to F (a warp per frame)
  float lo = INFINITY;
  for (int i = warp; i < F; i += WARPS) {
    float s = 0.f;
    if (i >= pad) {
      const float* cur = d + (size_t)(i - pad + 1) * NMELS;
      const float* prev = cur - NMELS;
      for (int m = lane; m < NMELS; m += 32) s += fmaxf(0.f, fmaxf(cur[m], floor_db) - fmaxf(prev[m], floor_db));
      for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    }
    const float e = s / (float)NMELS;
    if (lane == 0) env[i] = e;
    lo = fminf(lo, e);
  }
  lo = block_reduce<Reduce::MIN, WARPS>(lo, red);
  float hi = -INFINITY;
  for (int i = threadIdx.x; i < F; i += THREADS) hi = fmaxf(hi, env[i] - lo);
  const float denom = block_reduce<Reduce::MAX, WARPS>(hi, red) + 1.17549435e-38f;  // + tiny(float32)
  int any = 0, finite = 1;
  for (int i = threadIdx.x; i < F; i += THREADS) {
    const float e = (env[i] - lo) / denom;
    env[i] = e;
    any |= e != 0.f;
    finite &= isfinite(e);
  }
  any = __syncthreads_or(any);  // also orders the normalised writes before the reads below
  finite = __syncthreads_and(finite);
  if (!(any && finite)) {
    if (threadIdx.x == 0) counts[b] = 0;
    return;
  }
  // per-frame decisions, one byte each (bit 0: peak_pick keeps it, bit 1: a local minimum for onset_backtrack), over
  // the row's dB workspace, which is no longer read
  uint8_t* flags = reinterpret_cast<uint8_t*>(db + (size_t)b * F * NMELS);
  for (int i = threadIdx.x; i < F; i += THREADS) {
    const float x = env[i];
    float mmax = x;
    for (int j = max(0, i - t.g.pre_max); j < min(F, i + t.g.post_max); ++j) mmax = fmaxf(mmax, env[j]);
    const int a0 = max(0, i - t.g.pre_avg), a1 = min(F, i + t.g.post_avg);
    float s = 0.f;
    for (int j = a0; j < a1; ++j) s += env[j];
    const bool keep = x == mmax && x >= s / (float)(a1 - a0) + t.delta && x != 0.f;
    const bool is_min = i == 0 || (i + 1 < F && x <= env[i - 1] && x < env[i + 1]);
    flags[i] = (uint8_t)(keep | (is_min << 1));
  }
  __syncthreads();
  if (warp != 0) return;
  // the greedy walk of peak_pick (i > last + wait) and the backtrack, 32 frames per step
  int count = 0, last = 0, last_min = 0;
  for (int base = 0; base < F; base += 32) {
    const int f = base + lane < F ? flags[base + lane] : 0;
    const unsigned km = __ballot_sync(0xffffffffu, f & 1), mm = __ballot_sync(0xffffffffu, f & 2);
    if (lane == 0) {
      for (unsigned bits = km | mm; bits; bits &= bits - 1) {
        const int bit = __ffs(bits) - 1, fr = base + bit;
        if ((mm >> bit) & 1u) last_min = fr;
        if (((km >> bit) & 1u) && (count == 0 || fr > last + t.g.wait)) {
          onsets[(size_t)b * F + count++] = backtrack ? last_min : fr;
          last = fr;
        }
      }
    }
  }
  if (lane == 0) counts[b] = count;
}

// Python's slice bound normalisation for a sequence of length T
__device__ __forceinline__ long long slice_bound(long long s, int T) {
  if (s < 0) return s + T < 0 ? 0 : s + T;
  return s > T ? T : s;
}

__global__ void __launch_bounds__(THREADS) onset_mask_kernel(const int32_t* __restrict__ onsets,
                                                             const int32_t* __restrict__ counts, int onset_rows, int F,
                                                             int width, int64_t* __restrict__ mask, int B, int C, int T) {
  const size_t n = (size_t)B * C * T;
  for (size_t idx = (size_t)blockIdx.x * THREADS + threadIdx.x; idx < n; idx += (size_t)gridDim.x * THREADS) {
    const int t = (int)(idx % T), b = (int)(idx / ((size_t)C * T));
    const int r = onset_rows == 1 ? 0 : b;
    const int32_t* on = onsets + (size_t)r * F;
    int64_t v = 1;
    for (int k = 0, cnt = counts[r]; k < cnt; ++k) {
      const long long start = slice_bound((long long)on[k] - width, T), stop = slice_bound((long long)on[k] + width, T);
      if (t >= start && t < stop) { v = 0; break; }
    }
    mask[idx] = v;
  }
}

double py_floordiv(double a, double b) {  // CPython's float // (floatobject.c: float_floor_div)
  double mod = std::fmod(a, b);
  double div = (a - mod) / b;
  if (mod != 0 && ((b < 0) != (mod < 0))) div -= 1.0;
  if (div == 0) return std::copysign(0.0, a / b);
  double fl = std::floor(div);
  if (div - fl > 0.5) fl += 1.0;
  return fl;
}
}  // namespace

OnsetGeometry onset_geometry(int sr, int hop) {
  OnsetGeometry g;
  const double dsr = sr;
  g.pre_max = (int)std::ceil(py_floordiv(0.03 * dsr, hop));
  g.post_max = (int)std::ceil(py_floordiv(0.00 * dsr, hop) + 1);
  g.pre_avg = (int)std::ceil(py_floordiv(0.10 * dsr, hop));
  g.post_avg = (int)std::ceil(py_floordiv(0.10 * dsr, hop) + 1);
  g.wait = (int)std::ceil(py_floordiv(0.03 * dsr, hop));
  g.pad = 1 + ONSET_NFFT / (2 * hop);
  return g;
}

cudaError_t onset_tables(int sr, int hop, OnsetTables* out) {
  cudaError_t e = fft_tables(ONSET_NFFT, &out->fft);
  if (e != cudaSuccess) return e;
  if ((e = mel_filterbank(sr, ONSET_NFFT, NMELS, 0.0, 0.5 * sr, &out->bank)) != cudaSuccess) return e;
  out->g = onset_geometry(sr, hop);
  out->delta = 0.07f;
  return cudaSuccess;
}

size_t onset_workspace_bytes(int B, int F) { return (size_t)B * F * NMELS * sizeof(float); }

cudaError_t launch_onset_detect(const float* samples, int B, int N, int hop, const OnsetTables& t, float* db_ws,
                                float* env, int32_t* onsets, int32_t* counts, int backtrack, cudaStream_t st) {
  cudaError_t e =
      launch_spectrogram(SpecMode::ONSET_DB, samples, B, N, hop, ONSET_NFFT, t.fft, t.bank, NMELS, db_ws, st);
  if (e != cudaSuccess) return e;
  onset_pick_kernel<<<B, THREADS, 0, st>>>(db_ws, 1 + N / hop, t.g.pad, t, backtrack, env, onsets, counts);
  count_launch();
  return cudaGetLastError();
}

cudaError_t launch_onset_mask(const int32_t* onsets, const int32_t* counts, int onset_rows, int F, int width,
                              int64_t* mask, int B, int C, int T, cudaStream_t st) {
  const size_t n = (size_t)B * C * T;
  const int blocks = (int)std::min<size_t>((n + THREADS - 1) / THREADS, 4096);
  onset_mask_kernel<<<blocks, THREADS, 0, st>>>(onsets, counts, onset_rows, F, width, mask, B, C, T);
  count_launch();
  return cudaGetLastError();
}

}  // namespace vnb
