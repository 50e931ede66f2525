// vampnet_b200 — mel spectrogram and the multi-scale mel distance of audiotools' MelSpectrogramLoss (the reference's
// scripts/exp/eval.py scores generated audio with it), all on one stream with no host round trip:
//   mel_spec_kernel<NFFT>   one CTA per (FPC frames, row): reflect-indexed frame times the periodic Hann window ->
//                           fp32 NFFT-point real FFT in shared memory (fft.cuh) -> |X| -> each Slaney mel band summed
//                           over its nonzero bin range; (rows, n_mels, F) fp32
//   mel_diff_kernel         one CTA per (chunk of MEL_CHUNK elements, item) of one scale: |d log10| and |d| in float64
//   mel_final_kernel        one CTA: each item's chunk sums in order -> item losses, then the items in order -> loss
// DESIGN.md §13 has the definition and the numerics; oracle/mel_oracle.py restates it in float64.
#include <algorithm>
#include <cmath>

#include "fft.cuh"
#include "kernels.h"

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

template <int NFFT>
__global__ void __launch_bounds__(THREADS) mel_spec_kernel(const float* __restrict__ samples, int N, int F, int hop,
                                                           MelSpecArgs t, float* __restrict__ out) {
  constexpr int NH = NFFT / 2, NBINS = NH + 1, TPF = MelGeom<NFFT>::TPF, FPC = MelGeom<NFFT>::FPC;
  __shared__ float2 zs[FPC * NH];
  __shared__ float Ps[FPC * NBINS];
  const int g = threadIdx.x / TPF, lt = threadIdx.x % TPF;
  const int f = blockIdx.x * FPC + g, row = blockIdx.y;
  const bool live = f < F;  // the last CTA's spare groups still take part in the block-wide barriers
  float2* z = zs + g * NH;
  float* P = Ps + g * NBINS;
  const float* x = samples + (size_t)row * N;
  const long long s0 = (long long)f * hop - NFFT / 2;  // center=True; N > NFFT / 2, so one reflection reaches
  for (int m = lt; m < NH; m += TPF) {
    float a = 0.f, c = 0.f;
    if (live) {
      long long s = s0 + 2 * m;
      s = s < 0 ? -s : s >= N ? 2 * (long long)(N - 1) - s : s;
      long long s1 = s0 + 2 * m + 1;
      s1 = s1 < 0 ? -s1 : s1 >= N ? 2 * (long long)(N - 1) - s1 : s1;
      a = x[s] * t.fft.window[2 * m];
      c = x[s1] * t.fft.window[2 * m + 1];
    }
    z[__brev(m) >> (32 - ilog2(NH))] = make_float2(a, c);
  }
  __syncthreads();
  fft_radix2<NFFT>(z, t.fft.twiddle, lt, TPF);
  for (int k = lt; k < NBINS; k += TPF) {
    const float2 X = rfft_bin<NFFT>(z, t.fft.twiddle, k);
    P[k] = sqrtf(X.x * X.x + X.y * X.y);
  }
  __syncthreads();
  if (!live) return;
  for (int m = lt; m < t.n_mels; m += TPF) {
    const int o0 = t.bank.off[m], o1 = t.bank.off[m + 1];
    const float* p = P + t.bank.lo[m] - o0;
    float s = 0.f;
    for (int o = o0; o < o1; ++o) s = fmaf(t.bank.w[o], p[o], s);
    out[((size_t)row * t.n_mels + m) * F + f] = s;
  }
}

// fixed-order block sum: a xor tree in each warp, then the warps in order
__device__ double block_sum(double v, double* red) {
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  double s = red[0];
  for (int w = 1; w < THREADS / 32; ++w) s += red[w];
  __syncthreads();
  return s;
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
  sl = block_sum(sl, red);
  sm = block_sum(sm, red);
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

size_t align256(size_t n) { return (n + 255) & ~(size_t)255; }

cudaError_t spec_launch(const float* samples, int rows, int N, int F, int hop, const MelSpecArgs& t, float* out,
                        int n_fft, cudaStream_t st) {
  switch (n_fft) {
#define MEL_CASE(NF)                                                                                             \
  case NF:                                                                                                       \
    mel_spec_kernel<NF><<<dim3((F + MelGeom<NF>::FPC - 1) / MelGeom<NF>::FPC, rows), THREADS, 0, st>>>(         \
        samples, N, F, hop, t, out);                                                                             \
    break;
    MEL_CASE(32) MEL_CASE(64) MEL_CASE(128) MEL_CASE(256) MEL_CASE(512) MEL_CASE(1024) MEL_CASE(2048) MEL_CASE(4096)
#undef MEL_CASE
    default: return cudaErrorInvalidValue;
  }
  count_launch();
  return cudaGetLastError();
}

cudaError_t spec_args(int sr, const vnb_mel_scale& s, MelSpecArgs* t) {
  cudaError_t e = fft_tables(s.n_fft, &t->fft);
  if (e != cudaSuccess) return e;
  t->n_mels = s.n_mels;
  return mel_filterbank(sr, s.n_fft, s.n_mels, s.fmin, s.fmax, &t->bank);
}
}  // namespace

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
  p.x_spec = 0;
  p.y_spec = align256(spec);
  p.partials = p.y_spec + align256(spec);
  p.items = p.partials + align256(partials * sizeof(double2));
  p.total = p.items + align256((size_t)B * n_scales * sizeof(double2));
  return p;
}

cudaError_t launch_mel_spectrogram(const float* samples, int rows, int N, int sr, const vnb_mel_scale& s, float* out,
                                   cudaStream_t st) {
  MelSpecArgs t;
  cudaError_t e = spec_args(sr, s, &t);
  if (e != cudaSuccess) return e;
  return spec_launch(samples, rows, N, 1 + N / s.hop, s.hop, t, out, s.n_fft, st);
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
    if ((e = spec_launch(x, rows, p.N, s.F, s.hop, t, X, s.n_fft, st)) != cudaSuccess) return e;
    if ((e = spec_launch(y, rows, p.N, s.F, s.hop, t, Y, s.n_fft, st)) != cudaSuccess) return e;
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
