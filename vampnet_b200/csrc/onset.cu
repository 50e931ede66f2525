// vampnet_b200 — onset detection for the onset-prompt mask (reference vampnet/mask.py:203-226, which calls librosa
// 0.10's onset.onset_detect(y, sr, hop_length=H, backtrack=True)), all on one stream with no host round trip:
//   onset_spec_kernel   one CTA per (frame, row): Hann-windowed frame -> fp32 2048-point real FFT in shared memory
//                       (a 1024-point complex FFT of the even/odd sample pairs, then the real split) -> |X|^2 ->
//                       128 Slaney mel bands, each read over its nonzero bin range only -> 10 log10(max(1e-10, S))
//   onset_pick_kernel   one CTA per row: the clip's dB maximum (top_db = 80 clamp), the clamped spectral flux
//                       averaged over the bands, shifted and trimmed, normalised to [0, 1]; every frame's peak and
//                       minimum tests in parallel, then one warp walks them 32 frames at a time for peak_pick's
//                       wait rule and onset_backtrack
//   onset_mask_kernel   the reference's mask[:, :, idx - w:idx + w] = 0 loop, with Python slice semantics
// DESIGN.md §9 has the numerics; oracle/onset_oracle.py restates the algorithm in float64.  The FFT (fft.cuh) and
// the host tables built here (fft_tables, mel_filterbank) are shared with mel.cu.
#include <algorithm>
#include <initializer_list>
#include <cmath>
#include <cstring>
#include <map>
#include <mutex>
#include <tuple>
#include <utility>
#include <vector>

#include "fft.cuh"
#include "kernels.h"

namespace vnb {

namespace {
constexpr int NFFT = 2048, NH = NFFT / 2, NBINS = NH + 1, NMELS = 128, THREADS = 256;

__global__ void __launch_bounds__(THREADS) onset_spec_kernel(const float* __restrict__ samples, int N, int F, int hop,
                                                             OnsetTables t, float* __restrict__ db) {
  __shared__ float2 z[NH];
  __shared__ float P[NBINS];
  const int f = blockIdx.x, b = blockIdx.y;
  const float* x = samples + (size_t)b * N;
  const long long s0 = (long long)f * hop - NFFT / 2;  // center=True, zero padding (pad_mode="constant")
  for (int m = threadIdx.x; m < NH; m += THREADS) {
    const long long s = s0 + 2 * m;
    const float a = (s >= 0 && s < N) ? x[s] : 0.f;
    const float c = (s + 1 >= 0 && s + 1 < N) ? x[s + 1] : 0.f;
    z[__brev(m) >> 22] = make_float2(a * t.window[2 * m], c * t.window[2 * m + 1]);  // bit-reversed 10-bit index
  }
  __syncthreads();
  fft_radix2<NFFT>(z, t.twiddle, threadIdx.x, THREADS);
  for (int k = threadIdx.x; k < NBINS; k += THREADS) {
    const float2 X = rfft_bin<NFFT>(z, t.twiddle, k);
    P[k] = X.x * X.x + X.y * X.y;
  }
  __syncthreads();
  if (threadIdx.x < NMELS) {
    const int m = threadIdx.x, o0 = t.mel_off[m], o1 = t.mel_off[m + 1];
    const float* p = P + t.mel_lo[m] - o0;
    float s = 0.f;
    for (int o = o0; o < o1; ++o) s = fmaf(t.mel_w[o], p[o], s);
    db[((size_t)b * F + f) * NMELS + m] = 10.f * log10f(fmaxf(1e-10f, s));
  }
}

template <bool MAX>
__device__ float block_reduce(float v, float* red) {
  for (int o = 16; o; o >>= 1) {
    const float w = __shfl_xor_sync(0xffffffffu, v, o);
    v = MAX ? fmaxf(v, w) : fminf(v, w);
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __syncthreads();  // red[] may still be read by a previous reduction
  if (lane == 0) red[warp] = v;
  __syncthreads();
  v = red[0];
  for (int w = 1; w < THREADS / 32; ++w) v = MAX ? fmaxf(v, red[w]) : fminf(v, red[w]);
  return v;
}

__global__ void __launch_bounds__(THREADS) onset_pick_kernel(float* db, int F, int pad, OnsetTables t, int backtrack,
                                                             float* __restrict__ env_out, int32_t* __restrict__ onsets,
                                                             int32_t* __restrict__ counts) {
  __shared__ float red[THREADS / 32];
  const int b = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const float* d = db + (size_t)b * F * NMELS;
  float* env = env_out + (size_t)b * F;
  // power_to_db's top_db clamp: the maximum over the whole clip
  float mx = -INFINITY;
  for (size_t i = threadIdx.x; i < (size_t)F * NMELS; i += THREADS) mx = fmaxf(mx, d[i]);
  const float floor_db = block_reduce<true>(mx, red) - 80.f;
  // flux S[t] - S[t-1] clamped at 0, mean over bands, left-padded by `pad` frames and trimmed to F (a warp per frame)
  float lo = INFINITY;
  for (int i = warp; i < F; i += THREADS / 32) {
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
  lo = block_reduce<false>(lo, red);
  float hi = -INFINITY;
  for (int i = threadIdx.x; i < F; i += THREADS) hi = fmaxf(hi, env[i] - lo);
  const float denom = block_reduce<true>(hi, red) + 1.17549435e-38f;  // + tiny(float32)
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
    for (int j = max(0, i - t.pre_max); j < min(F, i + t.post_max); ++j) mmax = fmaxf(mmax, env[j]);
    const int a0 = max(0, i - t.pre_avg), a1 = min(F, i + t.post_avg);
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
        if (((km >> bit) & 1u) && (count == 0 || fr > last + t.wait)) {
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

// ---------------------------------------------------------------------------------------------- host tables
double py_floordiv(double a, double b) {  // CPython's float // (floatobject.c: float_floor_div)
  double mod = std::fmod(a, b);
  double div = (a - mod) / b;
  if (mod != 0 && ((b < 0) != (mod < 0))) div -= 1.0;
  if (div == 0) return std::copysign(0.0, a / b);
  double fl = std::floor(div);
  if (div - fl > 0.5) fl += 1.0;
  return fl;
}
double hz_to_mel(double f) {
  const double f_sp = 200.0 / 3, min_log_hz = 1000.0, min_log_mel = min_log_hz / f_sp, logstep = std::log(6.4) / 27.0;
  return f >= min_log_hz ? min_log_mel + std::log(f / min_log_hz) / logstep : f / f_sp;
}
double mel_to_hz(double m) {
  const double f_sp = 200.0 / 3, min_log_hz = 1000.0, min_log_mel = min_log_hz / f_sp, logstep = std::log(6.4) / 27.0;
  return m >= min_log_mel ? min_log_hz * std::exp(logstep * (m - min_log_mel)) : f_sp * m;
}

// one device allocation holding the given host blocks back to back; *dev points at the first
cudaError_t upload_blocks(std::initializer_list<std::pair<const void*, size_t>> blocks, char** dev) {
  size_t total = 0;
  for (const auto& b : blocks) total += b.second;
  std::vector<char> host(total);
  size_t at = 0;
  for (const auto& b : blocks) { if (b.second) memcpy(host.data() + at, b.first, b.second); at += b.second; }
  cudaError_t e = cudaMalloc(dev, total);
  if (e != cudaSuccess) return e;
  e = cudaMemcpy(*dev, host.data(), total, cudaMemcpyHostToDevice);
  if (e != cudaSuccess) { cudaFree(*dev); *dev = nullptr; }
  return e;
}

std::mutex g_onset_mu;  // guards the three caches below
std::map<std::tuple<int, int, int>, OnsetTables> g_onset_tables;  // (device, sr, hop)
std::map<std::pair<int, int>, FftTables> g_fft_tables;           // (device, n_fft)
std::map<std::tuple<int, int, int, int, double, double>, MelBank> g_mel_banks;  // (device, sr, n_fft, n_mels, fmin, fmax)

cudaError_t fft_tables_locked(int dev, int n_fft, FftTables* out) {
  auto it = g_fft_tables.find({dev, n_fft});
  if (it != g_fft_tables.end()) { *out = it->second; return cudaSuccess; }
  // twiddles exp(-2 pi i k / n_fft), k = 0..n_fft/2, and the periodic Hann window, both computed in float64
  const int nbins = n_fft / 2 + 1;
  std::vector<float2> tw(nbins);
  for (int k = 0; k < nbins; ++k) {
    const double a = 2.0 * M_PI * k / n_fft;
    tw[k] = make_float2((float)std::cos(a), (float)-std::sin(a));
  }
  std::vector<float> win(n_fft);
  for (int k = 0; k < n_fft; ++k) win[k] = (float)(0.5 - 0.5 * std::cos(2.0 * M_PI * k / n_fft));
  char* p = nullptr;
  const size_t b_tw = sizeof(float2) * nbins;
  cudaError_t e = upload_blocks({{tw.data(), b_tw}, {win.data(), sizeof(float) * n_fft}}, &p);
  if (e != cudaSuccess) return e;
  FftTables t;
  t.twiddle = reinterpret_cast<const float2*>(p);
  t.window = reinterpret_cast<const float*>(p + b_tw);
  g_fft_tables[{dev, n_fft}] = t;
  *out = t;
  return cudaSuccess;
}

cudaError_t mel_filterbank_locked(int dev, int sr, int n_fft, int n_mels, double fmin, double fmax, MelBank* out) {
  const auto key = std::make_tuple(dev, sr, n_fft, n_mels, fmin, fmax);
  auto it = g_mel_banks.find(key);
  if (it != g_mel_banks.end()) { *out = it->second; return cudaSuccess; }
  // librosa.filters.mel(sr, n_fft, n_mels, fmin, fmax, htk=False, norm="slaney", dtype=float32)
  const int nbins = n_fft / 2 + 1;
  std::vector<double> mel_f(n_mels + 2), fft_f(nbins);
  const double m0 = hz_to_mel(fmin), m1 = hz_to_mel(fmax), mstep = (m1 - m0) / (n_mels + 1);
  for (int i = 0; i < n_mels + 2; ++i) mel_f[i] = mel_to_hz(i == n_mels + 1 ? m1 : m0 + i * mstep);  // np.linspace
  for (int k = 0; k < nbins; ++k) fft_f[k] = k / (n_fft * (1.0 / sr));                             // np.fft.rfftfreq
  std::vector<float> wpack, row(nbins);
  std::vector<int32_t> off(n_mels + 1), lo(n_mels);
  for (int m = 0; m < n_mels; ++m) {
    const double enorm = 2.0 / (mel_f[m + 2] - mel_f[m]);
    int first = -1, last = -1;
    for (int k = 0; k < nbins; ++k) {
      const double lower = -(mel_f[m] - fft_f[k]) / (mel_f[m + 1] - mel_f[m]);
      const double upper = (mel_f[m + 2] - fft_f[k]) / (mel_f[m + 2] - mel_f[m + 1]);
      const float w = (float)std::max(0.0, std::min(lower, upper));
      row[k] = (float)((double)w * enorm);
      if (row[k] != 0.f) { if (first < 0) first = k; last = k; }
    }
    off[m] = (int32_t)wpack.size();
    lo[m] = first < 0 ? 0 : first;
    if (first >= 0) wpack.insert(wpack.end(), row.begin() + first, row.begin() + last + 1);
  }
  off[n_mels] = (int32_t)wpack.size();
  const size_t b_w = sizeof(float) * wpack.size(), b_off = sizeof(int32_t) * (n_mels + 1);
  char* p = nullptr;
  cudaError_t e = upload_blocks({{wpack.data(), b_w}, {off.data(), b_off}, {lo.data(), sizeof(int32_t) * n_mels}}, &p);
  if (e != cudaSuccess) return e;
  MelBank b;
  b.w = reinterpret_cast<const float*>(p);
  b.off = reinterpret_cast<const int32_t*>(p + b_w);
  b.lo = reinterpret_cast<const int32_t*>(p + b_w + b_off);
  g_mel_banks[key] = b;
  *out = b;
  return cudaSuccess;
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
  g.pad = 1 + NFFT / (2 * hop);
  return g;
}

cudaError_t fft_tables(int n_fft, FftTables* out) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  std::lock_guard<std::mutex> lock(g_onset_mu);
  return fft_tables_locked(dev, n_fft, out);
}

cudaError_t mel_filterbank(int sr, int n_fft, int n_mels, double fmin, double fmax, MelBank* out) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  std::lock_guard<std::mutex> lock(g_onset_mu);
  return mel_filterbank_locked(dev, sr, n_fft, n_mels, fmin, fmax, out);
}

cudaError_t onset_tables(int sr, int hop, OnsetTables* out) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  std::lock_guard<std::mutex> lock(g_onset_mu);
  auto key = std::make_tuple(dev, sr, hop);
  auto it = g_onset_tables.find(key);
  if (it != g_onset_tables.end()) { *out = it->second; return cudaSuccess; }
  FftTables f;
  MelBank m;
  if ((e = fft_tables_locked(dev, NFFT, &f)) != cudaSuccess) return e;
  if ((e = mel_filterbank_locked(dev, sr, NFFT, NMELS, 0.0, 0.5 * sr, &m)) != cudaSuccess) return e;
  OnsetTables t;
  t.twiddle = f.twiddle;
  t.window = f.window;
  t.mel_w = m.w;
  t.mel_off = m.off;
  t.mel_lo = m.lo;
  const OnsetGeometry g = onset_geometry(sr, hop);
  t.pre_max = g.pre_max; t.post_max = g.post_max; t.pre_avg = g.pre_avg; t.post_avg = g.post_avg;
  t.wait = g.wait; t.pad = g.pad;
  t.delta = 0.07f;
  g_onset_tables[key] = t;
  *out = t;
  return cudaSuccess;
}

cudaError_t launch_onset_detect(const float* samples, int B, int N, int hop, const OnsetTables& t, float* db_ws,
                                float* env, int32_t* onsets, int32_t* counts, int backtrack, cudaStream_t st) {
  const int F = 1 + N / hop;
  onset_spec_kernel<<<dim3(F, B), THREADS, 0, st>>>(samples, N, F, hop, t, db_ws);
  count_launch();
  onset_pick_kernel<<<B, THREADS, 0, st>>>(db_ws, F, t.pad, t, backtrack, env, onsets, counts);
  count_launch();
  return cudaGetLastError();
}

cudaError_t launch_onset_spec(const float* samples, int B, int N, int hop, const OnsetTables& t, float* db,
                              cudaStream_t st) {
  const int F = 1 + N / hop;
  onset_spec_kernel<<<dim3(F, B), THREADS, 0, st>>>(samples, N, F, hop, t, db);
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
