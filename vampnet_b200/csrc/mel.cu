// vampnet_b200 — the spectrogram kernel that onset detection, the beat tracker and the mel distance share, and the
// multi-scale mel distance of audiotools' MelSpectrogramLoss (the reference's scripts/exp/eval.py scores generated
// audio with it), all on one stream with no host round trip:
//   mel_spec_kernel<NFFT, MODE>  one CTA per (FPC frames, row): Hann-windowed frame -> fp32 NFFT-point real FFT in
//                                shared memory (fft.cuh) -> each Slaney mel band summed over its nonzero bin range.
//                                ONSET_DB (NFFT 2048; onset.cu, beat.cu): zero padding, |X|^2 on 128 bands, then
//                                10 log10(max(1e-10, S)); (rows, F, 128).  MEL_MAG: reflect padding, |X|;
//                                (rows, n_mels, F)
//   mel_diff_kernel              one CTA per (chunk of MEL_CHUNK elements, item) of one scale: |d log10| and |d| in
//                                float64
//   mel_final_kernel             one CTA: each item's chunk sums in order -> item losses, then the items in order ->
//                                loss
// The FFT tables and Slaney filterbanks are built here on the host in float64 and cached by device_table.  DESIGN.md
// §9 and §13 have the numerics; oracle/onset_oracle.py and oracle/mel_oracle.py restate them in float64.
#include <algorithm>
#include <cmath>
#include <cstring>

#include "fft.cuh"
#include "kernels.h"
#include "reduce.cuh"

namespace vnb {

namespace {
constexpr int THREADS = 256, MEL_CHUNK = 4096;

// threads per frame and frames per CTA: one frame per CTA from 2048 points, down to a warp per frame
template <int NFFT>
struct MelGeom {
  static constexpr int TPF = NFFT >= 2048 ? THREADS : (NFFT / 8 > 32 ? NFFT / 8 : 32);
  static constexpr int FPC = THREADS / TPF;
};

constexpr int ilog2(int n) { return n <= 1 ? 0 : 1 + ilog2(n / 2); }

struct MelSpecArgs {
  FftTables fft;
  MelBank bank;
  int n_mels;
};

template <int NFFT, SpecMode MODE>
__global__ void __launch_bounds__(THREADS) mel_spec_kernel(const float* __restrict__ samples, int N, int F, int hop,
                                                           MelSpecArgs t, float* __restrict__ out) {
  constexpr bool DB = MODE == SpecMode::ONSET_DB;
  constexpr int NH = NFFT / 2, NBINS = NH + 1, TPF = MelGeom<NFFT>::TPF, FPC = MelGeom<NFFT>::FPC;
  __shared__ float2 zs[FPC * NH];
  __shared__ float Ps[FPC * NBINS];
  const int g = threadIdx.x / TPF, lt = threadIdx.x % TPF;
  const int f = blockIdx.x * FPC + g, row = blockIdx.y;
  const bool live = FPC == 1 || f < F;  // the last CTA's spare groups still take part in the block-wide barriers
  float2* z = zs + g * NH;
  float* P = Ps + g * NBINS;
  const float* x = samples + (size_t)row * N;
  const long long s0 = (long long)f * hop - NFFT / 2;  // center=True
  for (int m = lt; m < NH; m += TPF) {
    float a = 0.f, c = 0.f;
    if (live) {
      long long s = s0 + 2 * m, s1 = s0 + 2 * m + 1;
      if (DB) {  // zero padding (pad_mode="constant"), any N
        a = (s >= 0 && s < N) ? x[s] : 0.f;
        c = (s1 >= 0 && s1 < N) ? x[s1] : 0.f;
      } else {  // reflect padding: N > NFFT / 2, so one reflection reaches
        s = s < 0 ? -s : s >= N ? 2 * (long long)(N - 1) - s : s;
        s1 = s1 < 0 ? -s1 : s1 >= N ? 2 * (long long)(N - 1) - s1 : s1;
        a = x[s];
        c = x[s1];
      }
      a *= t.fft.window[2 * m];
      c *= t.fft.window[2 * m + 1];
    }
    z[__brev(m) >> (32 - ilog2(NH))] = make_float2(a, c);
  }
  __syncthreads();
  fft_radix2<NFFT>(z, t.fft.twiddle, lt, TPF);
  for (int k = lt; k < NBINS; k += TPF) {
    const float2 X = rfft_bin<NFFT>(z, t.fft.twiddle, k);
    const float p = X.x * X.x + X.y * X.y;
    P[k] = DB ? p : sqrtf(p);
  }
  __syncthreads();
  if (!live) return;
  const int n_mels = DB ? ONSET_NMELS : t.n_mels;
  for (int m = lt; m < n_mels; m += TPF) {
    const int o0 = t.bank.off[m], o1 = t.bank.off[m + 1];
    const float* p = P + t.bank.lo[m] - o0;
    float s = 0.f;
    for (int o = o0; o < o1; ++o) s = fmaf(t.bank.w[o], p[o], s);
    if (DB)
      out[((size_t)row * F + f) * ONSET_NMELS + m] = 10.f * log10f(fmaxf(1e-10f, s));
    else
      out[((size_t)row * n_mels + m) * F + f] = s;
  }
}

// X and Y (B items of `elems` values each) -> partial[b * chunks + c] = (sum |d log10|, sum |d|) over chunk c
__global__ void __launch_bounds__(THREADS) mel_diff_kernel(const float* __restrict__ X, const float* __restrict__ Y,
                                                           long long elems, int chunks, double eps, double pw,
                                                           double2* __restrict__ partial) {
  __shared__ double red[THREADS / 32];
  const int c = blockIdx.x, b = blockIdx.y;
  const long long first = (long long)c * MEL_CHUNK, n = std::min<long long>(MEL_CHUNK, elems - first);
  const float* xp = X + (size_t)b * elems + first;
  const float* yp = Y + (size_t)b * elems + first;
  double sl = 0.0, sm = 0.0;
  for (int i = threadIdx.x; i < n; i += THREADS) {
    const double xv = xp[i], yv = yp[i];
    // log10(max(v, eps)^pow) as pow * log10(max(v, eps)): equal up to float64 rounding, and it cannot overflow
    sl += fabs(pw * log10(fmax(xv, eps)) - pw * log10(fmax(yv, eps)));
    sm += fabs(xv - yv);
  }
  sl = block_reduce<Reduce::SUM, THREADS / 32>(sl, red);
  sm = block_reduce<Reduce::SUM, THREADS / 32>(sm, red);
  if (threadIdx.x == 0) partial[(size_t)b * chunks + c] = make_double2(sl, sm);
}

struct MelFinalArgs {
  int B, n_scales;
  double log_weight, mag_weight;
  int chunks[MEL_MAX_SCALES];
  size_t partial[MEL_MAX_SCALES];
  double count[MEL_MAX_SCALES];  // C * n_mels * F
};

__global__ void __launch_bounds__(THREADS) mel_final_kernel(const double2* __restrict__ partial, MelFinalArgs a,
                                                            double2* __restrict__ items, float* __restrict__ loss,
                                                            float* __restrict__ item_loss) {
  for (int b = threadIdx.x; b < a.B; b += THREADS) {
    double l = 0.0;
    for (int s = 0; s < a.n_scales; ++s) {
      const double2* p = partial + a.partial[s] + (size_t)b * a.chunks[s];
      double sl = 0.0, sm = 0.0;
      for (int c = 0; c < a.chunks[s]; ++c) { sl += p[c].x; sm += p[c].y; }
      items[(size_t)b * a.n_scales + s] = make_double2(sl, sm);
      l += a.log_weight * (sl / a.count[s]);
      l += a.mag_weight * (sm / a.count[s]);
    }
    if (item_loss) item_loss[b] = (float)l;
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
  double l = 0.0;
  for (int s = 0; s < a.n_scales; ++s) {
    double sl = 0.0, sm = 0.0;
    for (int b = 0; b < a.B; ++b) { sl += items[(size_t)b * a.n_scales + s].x; sm += items[(size_t)b * a.n_scales + s].y; }
    const double n = a.count[s] * a.B;
    l += a.log_weight * (sl / n);
    l += a.mag_weight * (sm / n);
  }
  loss[0] = (float)l;
}

double hz_to_mel(double f) {
  const double f_sp = 200.0 / 3, min_log_hz = 1000.0, min_log_mel = min_log_hz / f_sp, logstep = std::log(6.4) / 27.0;
  return f >= min_log_hz ? min_log_mel + std::log(f / min_log_hz) / logstep : f / f_sp;
}
double mel_to_hz(double m) {
  const double f_sp = 200.0 / 3, min_log_hz = 1000.0, min_log_mel = min_log_hz / f_sp, logstep = std::log(6.4) / 27.0;
  return m >= min_log_mel ? min_log_hz * std::exp(logstep * (m - min_log_mel)) : f_sp * m;
}

cudaError_t spec_args(int sr, const vnb_mel_scale& s, MelSpecArgs* t) {
  cudaError_t e = fft_tables(s.n_fft, &t->fft);
  if (e != cudaSuccess) return e;
  t->n_mels = s.n_mels;
  return mel_filterbank(sr, s.n_fft, s.n_mels, s.fmin, s.fmax, &t->bank);
}
}  // namespace

// one table: the twiddles, then the window
cudaError_t fft_tables(int n_fft, FftTables* out) {
  const int nbins = n_fft / 2 + 1;
  const size_t b_tw = sizeof(float2) * nbins;
  const char* p = nullptr;
  cudaError_t e = device_table({TABLE_FFT, (double)n_fft}, [&] {
    // twiddles exp(-2 pi i k / n_fft), k = 0..n_fft/2, and the periodic Hann window, both computed in float64
    std::vector<char> img(b_tw + sizeof(float) * n_fft);
    float2* tw = reinterpret_cast<float2*>(img.data());
    float* win = reinterpret_cast<float*>(img.data() + b_tw);
    for (int k = 0; k < nbins; ++k) {
      const double a = 2.0 * M_PI * k / n_fft;
      tw[k] = make_float2((float)std::cos(a), (float)-std::sin(a));
    }
    for (int k = 0; k < n_fft; ++k) win[k] = (float)(0.5 - 0.5 * std::cos(2.0 * M_PI * k / n_fft));
    return img;
  }, &p);
  if (e != cudaSuccess) return e;
  out->twiddle = reinterpret_cast<const float2*>(p);
  out->window = reinterpret_cast<const float*>(p + b_tw);
  return cudaSuccess;
}

// one table: off, then lo, then the packed weights
cudaError_t mel_filterbank(int sr, int n_fft, int n_mels, double fmin, double fmax, MelBank* out) {
  const size_t b_off = sizeof(int32_t) * (n_mels + 1), b_lo = sizeof(int32_t) * n_mels;
  const char* p = nullptr;
  cudaError_t e = device_table({TABLE_MEL_BANK, (double)sr, (double)n_fft, (double)n_mels, fmin, fmax}, [&] {
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
    std::vector<char> img(b_off + b_lo + sizeof(float) * wpack.size());
    memcpy(img.data(), off.data(), b_off);
    memcpy(img.data() + b_off, lo.data(), b_lo);
    if (!wpack.empty()) memcpy(img.data() + b_off + b_lo, wpack.data(), sizeof(float) * wpack.size());
    return img;
  }, &p);
  if (e != cudaSuccess) return e;
  out->off = reinterpret_cast<const int32_t*>(p);
  out->lo = reinterpret_cast<const int32_t*>(p + b_off);
  out->w = reinterpret_cast<const float*>(p + b_off + b_lo);
  return cudaSuccess;
}

cudaError_t launch_spectrogram(SpecMode mode, const float* samples, int rows, int N, int hop, int n_fft,
                               const FftTables& fft, const MelBank& bank, int n_mels, float* out, cudaStream_t st) {
  const int F = 1 + N / hop;
  const MelSpecArgs t{fft, bank, n_mels};
#define SPEC_LAUNCH(NF, MODE)                                                                                    \
  mel_spec_kernel<NF, MODE><<<dim3((F + MelGeom<NF>::FPC - 1) / MelGeom<NF>::FPC, rows), THREADS, 0, st>>>(      \
      samples, N, F, hop, t, out)
  if (mode == SpecMode::ONSET_DB) {
    if (n_fft != ONSET_NFFT || n_mels != ONSET_NMELS) return cudaErrorInvalidValue;
    SPEC_LAUNCH(ONSET_NFFT, SpecMode::ONSET_DB);
  } else {
    switch (n_fft) {
#define MEL_CASE(NF) case NF: SPEC_LAUNCH(NF, SpecMode::MEL_MAG); break;
      MEL_CASE(32) MEL_CASE(64) MEL_CASE(128) MEL_CASE(256) MEL_CASE(512) MEL_CASE(1024) MEL_CASE(2048) MEL_CASE(4096)
#undef MEL_CASE
      default: return cudaErrorInvalidValue;
    }
  }
#undef SPEC_LAUNCH
  count_launch();
  return cudaGetLastError();
}

MelLossPlan mel_loss_plan(int B, int C, int N, int sr, const vnb_mel_scale* scales, int n_scales) {
  MelLossPlan p;
  p.B = B; p.C = C; p.N = N; p.sr = sr; p.n_scales = n_scales;
  size_t spec = 0, partials = 0;
  for (int i = 0; i < n_scales; ++i) {
    MelScalePlan& s = p.s[i];
    s.n_fft = scales[i].n_fft; s.hop = scales[i].hop; s.n_mels = scales[i].n_mels;
    s.fmin = scales[i].fmin; s.fmax = scales[i].fmax;
    s.F = 1 + N / s.hop;
    s.elems = (long long)C * s.n_mels * s.F;
    s.chunks = (int)((s.elems + MEL_CHUNK - 1) / MEL_CHUNK);
    s.partial = partials;
    partials += (size_t)B * s.chunks;
    spec = std::max(spec, (size_t)B * (size_t)s.elems * sizeof(float));
  }
  // one X and one Y buffer, reused scale after scale (the stream orders the reuse)
  size_t o = 0;
  p.x_spec = carve(o, spec);
  p.y_spec = carve(o, spec);
  p.partials = carve(o, partials * sizeof(double2));
  p.items = carve(o, (size_t)B * n_scales * sizeof(double2));
  p.total = o;
  return p;
}

cudaError_t launch_mel_spectrogram(const float* samples, int rows, int N, int sr, const vnb_mel_scale& s, float* out,
                                   cudaStream_t st) {
  MelSpecArgs t;
  cudaError_t e = spec_args(sr, s, &t);
  if (e != cudaSuccess) return e;
  return launch_spectrogram(SpecMode::MEL_MAG, samples, rows, N, s.hop, s.n_fft, t.fft, t.bank, t.n_mels, out, st);
}

cudaError_t launch_mel_loss(const float* x, const float* y, const MelLossPlan& p, double clamp_eps, double pow,
                            double log_weight, double mag_weight, void* workspace, float* loss, float* item_loss,
                            cudaStream_t st) {
  char* ws = static_cast<char*>(workspace);
  float* X = reinterpret_cast<float*>(ws + p.x_spec);
  float* Y = reinterpret_cast<float*>(ws + p.y_spec);
  double2* partial = reinterpret_cast<double2*>(ws + p.partials);
  MelFinalArgs a{};
  a.B = p.B; a.n_scales = p.n_scales; a.log_weight = log_weight; a.mag_weight = mag_weight;
  const int rows = p.B * p.C;
  for (int i = 0; i < p.n_scales; ++i) {
    const MelScalePlan& s = p.s[i];
    const vnb_mel_scale sc{s.n_fft, s.hop, s.n_mels, s.fmin, s.fmax};
    MelSpecArgs t;
    cudaError_t e = spec_args(p.sr, sc, &t);
    if (e != cudaSuccess) return e;
    if ((e = launch_spectrogram(SpecMode::MEL_MAG, x, rows, p.N, s.hop, s.n_fft, t.fft, t.bank, t.n_mels, X, st)))
      return e;
    if ((e = launch_spectrogram(SpecMode::MEL_MAG, y, rows, p.N, s.hop, s.n_fft, t.fft, t.bank, t.n_mels, Y, st)))
      return e;
    mel_diff_kernel<<<dim3(s.chunks, p.B), THREADS, 0, st>>>(X, Y, s.elems, s.chunks, clamp_eps, pow, partial + s.partial);
    count_launch();
    a.chunks[i] = s.chunks;
    a.partial[i] = s.partial;
    a.count[i] = (double)s.elems;
  }
  mel_final_kernel<<<1, THREADS, 0, st>>>(partial, a, reinterpret_cast<double2*>(ws + p.items), loss, item_loss);
  count_launch();
  return cudaGetLastError();
}

}  // namespace vnb
