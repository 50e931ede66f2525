// vampnet_b200 — pitch shift (torch_pitch_shift 1.2's pitch_shift: torch.stft -> torchaudio's phase vocoder ->
// torch.istft -> torchaudio's sinc resampler, restated on the device; DESIGN.md §11).  Input and output are fp32;
// everything in between is float64, because the vocoder's running phase sum keeps every rounding of a quiet bin's
// angle for the rest of the clip.  One stream, no host round trip, every reduction in a fixed order:
//   dft_gemm_kernel<true>    frames (F x n_fft, read from the signal with reflect padding) x cos/sin basis -> spectrum
//                            (F x n_bins complex), fp64 tensor cores (mma.m16n8k16 .f64, sm_90)
//   to_polar_kernel          spectrum -> (|X|, angle X) in place
//   vocoder_step_kernel      per (chunk of 32 output frames, row): gathers frames floor(ts) and floor(ts) + 1,
//                            interpolated magnitude, wrapped phase increment, and the chunk's sum of increments
//   chunk_offsets_kernel     per (bin, row): exclusive sum over the chunk sums, in chunk order
//   vocoder_polar_kernel     per (chunk, row): running phase from the chunk's offset, polar(mag, phase) in place
//   dft_gemm_kernel<false>   stretched spectrum x inverse basis (1/n_fft and the one-sided x2 folded in) -> frames
//   overlap_add_kernel       each output sample sums its frames in frame order and divides by their count
//   resample_kernel          each output sample evaluates its own sinc taps (|t| < 6) in float64, cut or padded to N
// oracle/pitch_oracle.py restates the same steps in float64 numpy.
#include <algorithm>
#include <cmath>
#include <numeric>

#include "kernels.h"

namespace vnb {

namespace {
constexpr int BM = 64, BN = 64, BK = 16, GT = 128;  // DFT GEMM tile and threads (4 warps, 32 x 32 each)
constexpr int VT = 128, CH = 32;                    // vocoder threads and frames per scan chunk
constexpr double TWO_PI = 6.283185307179586;        // 2 * math.pi

__device__ __forceinline__ void dmma(double (&d)[4], const double (&a)[8], const double (&b)[4]) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, "
      "{%12,%13,%14,%15}, {%0,%1,%2,%3};"
      : "+d"(d[0]), "+d"(d[1]), "+d"(d[2]), "+d"(d[3])
      : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]), "d"(b[0]), "d"(b[1]),
        "d"(b[2]), "d"(b[3]));
}

// The A operand of a DFT GEMM, (M x K) per row.  FRAMES: frame f, tap n is the fp32 signal at f * hop + n - n_fft / 2,
// reflected at both ends (torch.stft, center=True, pad_mode="reflect").  Otherwise a dense float64 matrix.
struct GemmA {
  const float* x;   // FRAMES: (rows, N)
  const double* a;  // dense: (rows, M, lda)
  long long row_stride;
  int M, K, lda, N, hop, pad;
};

template <bool FRAMES>
__device__ __forceinline__ double load_a(const GemmA& A, long long row_off, int r, int c) {
  if (r >= A.M || c >= A.K) return 0.0;
  if (FRAMES) {
    long long s = (long long)r * A.hop + c - A.pad;
    if (s < 0) s = -s;
    if (s >= A.N) s = 2LL * (A.N - 1) - s;
    return (double)A.x[row_off + s];
  }
  return A.a[row_off + (long long)r * A.lda + c];
}

// out (rows, M, ldc) = A (M x K) x basis (Kp x Np, zero padded, row-major), columns < n_out stored.  Every output is
// summed over K in the same order whatever the batch, so a row's result equals that row computed alone.
template <bool FRAMES>
__global__ void __launch_bounds__(GT) dft_gemm_kernel(GemmA A, const double* __restrict__ basis, int Kp, int Np,
                                                      double* __restrict__ out, int ldc, int n_out) {
  __shared__ double As[BM][BK + 4];
  __shared__ double Bs[BK][BN + 4];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = lane >> 2, tig = lane & 3;
  const int wm = warp & 1, wn = warp >> 1;
  const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
  const long long row_off = (long long)blockIdx.z * A.row_stride;
  double acc[2][4][4];
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int v = 0; v < 4; ++v) acc[i][j][v] = 0.0;
  double ra[8], rb[8];
  auto fetch = [&](int k0) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int e = tid + GT * i;
      ra[i] = load_a<FRAMES>(A, row_off, m0 + (e >> 4), k0 + (e & 15));
      rb[i] = basis[(size_t)(k0 + (e >> 6)) * Np + n0 + (e & 63)];
    }
  };
  fetch(0);
  for (int k0 = 0; k0 < Kp; k0 += BK) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int e = tid + GT * i;
      As[e >> 4][e & 15] = ra[i];
      Bs[e >> 6][e & 63] = rb[i];
    }
    __syncthreads();
    if (k0 + BK < Kp) fetch(k0 + BK);
    double fa[2][8], fb[4][4];
#pragma unroll
    for (int mi = 0; mi < 2; ++mi)
#pragma unroll
      for (int v = 0; v < 8; ++v) fa[mi][v] = As[32 * wm + 16 * mi + g + 8 * (v & 1)][tig + 4 * (v >> 1)];
#pragma unroll
    for (int ni = 0; ni < 4; ++ni)
#pragma unroll
      for (int v = 0; v < 4; ++v) fb[ni][v] = Bs[tig + 4 * v][32 * wn + 8 * ni + g];
#pragma unroll
    for (int mi = 0; mi < 2; ++mi)
#pragma unroll
      for (int ni = 0; ni < 4; ++ni) dmma(acc[mi][ni], fa[mi], fb[ni]);
    __syncthreads();
  }
  double* o = out + (size_t)blockIdx.z * A.M * ldc;
#pragma unroll
  for (int mi = 0; mi < 2; ++mi)
#pragma unroll
    for (int ni = 0; ni < 4; ++ni)
#pragma unroll
      for (int v = 0; v < 4; ++v) {
        const int r = m0 + 32 * wm + 16 * mi + g + 8 * (v >> 1), c = n0 + 32 * wn + 8 * ni + 2 * tig + (v & 1);
        if (r < A.M && c < n_out) o[(size_t)r * ldc + c] = acc[mi][ni][v];
      }
}

__global__ void to_polar_kernel(double2* __restrict__ s, long long n) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const double2 v = s[i];
    s[i] = make_double2(hypot(v.x, v.y), atan2(v.y, v.x));
  }
}

// torch.arange(0, F, rate, dtype=float32) on CUDA: float(rate) * float(i), rounded once
__device__ __forceinline__ float time_step(float rate, long long i) { return __fmul_rn(rate, (float)i); }

// TimeStretch's phase_advance, torch.linspace(0, pi * hop, n_bins) in float32 (from both ends, as torch computes it)
__device__ __forceinline__ double phase_advance(int k, int nb, float end) {
  const float step = end / (float)(nb - 1);
  return (double)(k < nb / 2 ? __fmul_rn(step, (float)k) : __fsub_rn(end, __fmul_rn(step, (float)(nb - 1 - k))));
}

struct VocoderArgs {
  const double2* pol;  // (rows, F, nb) (|X|, angle X)
  double2* out;        // (rows, F2, nb) (mag, phase increment), then polar(mag, phase_acc)
  double* chunk;       // (rows, nchunks, nb) chunk sums, then exclusive offsets
  int F, F2, nb, nchunks;
  float rate, adv_end;
};

// torchaudio.functional.phase_vocoder for output frames [c * CH, c * CH + CH): magnitudes and the phase entering each
// frame (the first frame's angle at frame 0, else the previous step's wrapped increment)
__global__ void __launch_bounds__(VT) vocoder_step_kernel(VocoderArgs a) {
  const int c = blockIdx.x, b = blockIdx.y;
  const double2* pol = a.pol + (size_t)b * a.F * a.nb;
  double2* out = a.out + (size_t)b * a.F2 * a.nb;
  const int t0 = c * CH, t1 = min(a.F2, t0 + CH);
  for (int k = threadIdx.x; k < a.nb; k += VT) {
    const double adv = phase_advance(k, a.nb, a.adv_end);
    auto frame = [&](long long i) { return i < a.F ? pol[(size_t)i * a.nb + k] : make_double2(0.0, 0.0); };
    // step t: magnitude, and the increment angle1 - angle0 wrapped about adv (entering frame t + 1)
    auto step = [&](int t, double* mag) {
      const float ts = time_step(a.rate, t);
      const float fl = floorf(ts);
      const double alpha = (double)(ts - fl);
      const double2 p0 = frame((long long)fl), p1 = frame((long long)fl + 1);
      *mag = __dadd_rn(__dmul_rn(alpha, p1.x), __dmul_rn(1.0 - alpha, p0.x));
      double d = __dsub_rn(__dsub_rn(p1.y, p0.y), adv);
      d = __dsub_rn(d, __dmul_rn(TWO_PI, rint(d / TWO_PI)));
      return __dadd_rn(d, adv);
    };
    double prev = 0.0, mag, sum = 0.0;
    if (t0 > 0) prev = step(t0 - 1, &mag);
    for (int t = t0; t < t1; ++t) {
      const double ph = t == 0 ? pol[k].y : prev;
      prev = step(t, &mag);
      out[(size_t)t * a.nb + k] = make_double2(mag, ph);
      sum += ph;
    }
    a.chunk[((size_t)b * a.nchunks + c) * a.nb + k] = sum;
  }
}

__global__ void __launch_bounds__(VT) chunk_offsets_kernel(VocoderArgs a) {
  double* ch = a.chunk + (size_t)blockIdx.y * a.nchunks * a.nb;
  for (int k = blockIdx.x * VT + threadIdx.x; k < a.nb; k += gridDim.x * VT) {
    double acc = 0.0;
    for (int c = 0; c < a.nchunks; ++c) {
      const double v = ch[(size_t)c * a.nb + k];
      ch[(size_t)c * a.nb + k] = acc;
      acc += v;
    }
  }
}

__global__ void __launch_bounds__(VT) vocoder_polar_kernel(VocoderArgs a) {
  const int c = blockIdx.x, b = blockIdx.y;
  double2* out = a.out + (size_t)b * a.F2 * a.nb;
  const int t0 = c * CH, t1 = min(a.F2, t0 + CH);
  for (int k = threadIdx.x; k < a.nb; k += VT) {
    double acc = a.chunk[((size_t)b * a.nchunks + c) * a.nb + k];
    for (int t = t0; t < t1; ++t) {
      const double2 v = out[(size_t)t * a.nb + k];
      acc += v.y;
      double s, co;
      sincos(acc, &s, &co);
      out[(size_t)t * a.nb + k] = make_double2(v.x * co, v.x * s);
    }
  }
}

// torch.istft's overlap-add (rectangular window, center=True): output j is padded position j + n_fft / 2
__global__ void overlap_add_kernel(const double* __restrict__ frames, int F2, int n_fft, int hop, long long L,
                                   double* __restrict__ y) {
  const int b = blockIdx.y;
  const double* fr = frames + (size_t)b * F2 * n_fft;
  for (long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x; j < L; j += (long long)gridDim.x * blockDim.x) {
    const long long t = j + n_fft / 2;
    const long long f1 = std::min<long long>(F2 - 1, t / hop), f0 = t >= n_fft ? (t - n_fft) / hop + 1 : 0;
    double s = 0.0;
    for (long long f = f0; f <= f1; ++f) s += fr[f * n_fft + (t - f * hop)];
    y[(size_t)b * L + j] = s / (double)(f1 - f0 + 1);
  }
}

struct ResampleArgs {
  const double* y;  // (rows, L)
  float* out;       // (rows, N)
  long long L, target, orig_g, new_g;
  double base, scale, reach;  // reach: 6 / base in input periods of orig_g
  int N, width, identity;
};

// torchaudio.functional.resample (sinc_interp_hann, lowpass_filter_width 6, rolloff 0.99): output o = c * new_g + j
// is the conv1d of stride orig_g at c with kernel row j, tap m = u + width reading input c * orig_g + u.  Only taps
// with |t| < 6 are evaluated (the clamped ones are ~1e-50), each with torchaudio's expression order.
__global__ void resample_kernel(ResampleArgs a) {
  const int b = blockIdx.y;
  const double* y = a.y + (size_t)b * a.L;
  float* out = a.out + (size_t)b * a.N;
  for (long long o = (long long)blockIdx.x * blockDim.x + threadIdx.x; o < a.N; o += (long long)gridDim.x * blockDim.x) {
    double v = 0.0;
    if (o < a.target) {
      if (a.identity) {
        v = y[o];
      } else {
        const long long c = o / a.new_g, j = o % a.new_g;
        const double tj = (double)(-j) / (double)a.new_g;
        const double centre = (double)a.orig_g * ((double)j / (double)a.new_g);
        const long long u0 = std::max<long long>(-a.width, (long long)floor(centre - a.reach) - 1);
        const long long u1 = std::min<long long>(a.width + a.orig_g - 1, (long long)ceil(centre + a.reach) + 1);
        for (long long u = u0; u <= u1; ++u) {
          const double t = __dmul_rn(__dadd_rn(tj, (double)u / (double)a.orig_g), a.base);
          if (!(fabs(t) < 6.0)) continue;
          const long long p = c * a.orig_g + u;
          if (p < 0 || p >= a.L) continue;
          double w = cos(__dmul_rn(t, M_PI) / 6.0 / 2.0);
          w = __dmul_rn(w, w);
          const double tp = __dmul_rn(t, M_PI);
          const double k = __dmul_rn(tp == 0.0 ? 1.0 : sin(tp) / tp, __dmul_rn(w, a.scale));
          v = fma(y[p], k, v);
        }
      }
    }
    out[o] = (float)v;
  }
}

__global__ void time_steps_kernel(float rate, long long n, float* __restrict__ out) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    out[i] = time_step(rate, i);
}

int round_up(int x, int m) { return (x + m - 1) / m * m; }

int grid_for(long long n, int threads) { return (int)std::min<long long>((n + threads - 1) / threads, 65535); }
}  // namespace

int pitch_plan(int rows, int N, int sr, int new_freq, int n_fft, int hop, double rate, PitchPlan* p) {
  PitchPlan q;
  q.rows = rows; q.N = N; q.sr = sr; q.new_freq = new_freq; q.n_fft = n_fft; q.hop = hop; q.rate = rate;
  q.nb = n_fft / 2 + 1;
  q.F = 1 + (N + 2 * (n_fft / 2) - n_fft) / hop;  // torch.stft's frame count: 1 + (N - 1) / hop for odd n_fft
  q.stretch = rate != 1.0;
  const double F2 = q.stretch ? std::ceil((double)q.F / rate) : (double)q.F;  // torch.arange's length, in double
  if (!(F2 >= 1 && F2 <= (double)(1 << 30))) return 1;
  q.F2 = (int)F2;
  q.nchunks = (q.F2 + CH - 1) / CH;
  q.L = (long long)n_fft - 2LL * (n_fft / 2) + (long long)hop * (q.F2 - 1);  // torch.istft, center=True, length=None
  if (q.L < 1) return 2;  // one stretched frame of even n_fft: torch.istft refuses the empty signal
  q.resample = new_freq != sr;
  if (q.resample) {
    const long long g = std::gcd((long long)sr, (long long)new_freq);
    q.orig_g = sr / g;
    q.new_g = new_freq / g;
    q.base = (double)std::min(q.orig_g, q.new_g) * 0.99;
    q.width = (int)std::ceil(6.0 * (double)q.orig_g / q.base);
    q.scale = q.base / (double)q.orig_g;
    // torch.ceil(torch.as_tensor(new * L / orig)): the Python float quotient, rounded to float32 first
    q.target = (long long)std::ceil((float)((double)(q.new_g * q.L) / (double)q.orig_g));
  } else {
    q.target = q.L;
  }
  *p = q;
  return 0;
}

PitchLayout pitch_layout(const PitchPlan& p) {
  const size_t R = (size_t)p.rows, z = sizeof(double);
  PitchLayout l;
  size_t o = 0;
  l.spec = carve(o, R * p.F * p.nb * 2 * z);                            // spectrum, then (|X|, angle)
  l.stretched = p.stretch ? carve(o, R * p.F2 * p.nb * 2 * z) : l.spec;  // stretched spectrum
  l.chunk = p.stretch ? carve(o, R * p.nchunks * p.nb * z) : 0;          // chunk sums
  l.frames = carve(o, R * p.F2 * p.n_fft * z);                          // inverse DFT frames
  l.y = carve(o, R * p.L * z);                                          // overlap-added signal
  l.total = o;
  return l;
}

size_t pitch_workspace_bytes(const PitchPlan& p) { return pitch_layout(p).total; }

// one table: the forward basis, then the inverse at a 256-byte aligned offset
cudaError_t pitch_basis(int n_fft, const double** fwd, const double** inv) {
  const int nb = n_fft / 2 + 1;
  const int fk = round_up(n_fft, BK), fn = round_up(2 * nb, BN);  // forward: (n_fft x 2 nb), re/im interleaved
  const int ik = round_up(2 * nb, BK), in = round_up(n_fft, BN);  // inverse: (2 nb x n_fft)
  size_t o = 0;
  const size_t f_at = carve(o, (size_t)fk * fn * sizeof(double)), v_at = carve(o, (size_t)ik * in * sizeof(double));
  const char* p = nullptr;
  cudaError_t e = device_table({TABLE_PITCH_BASIS, (double)n_fft}, [&] {
    std::vector<char> img(o);  // zeroed: the tile padding stays 0
    double* f = reinterpret_cast<double*>(img.data() + f_at);
    double* v = reinterpret_cast<double*>(img.data() + v_at);
    for (int n = 0; n < n_fft; ++n)
      for (int k = 0; k < nb; ++k) {
        const double a = 2.0 * M_PI * (double)(((long long)k * n) % n_fft) / n_fft;  // argument reduced exactly
        const double co = std::cos(a), si = std::sin(a);
        f[(size_t)n * fn + 2 * k] = co;
        f[(size_t)n * fn + 2 * k + 1] = -si;
        // irfft: DC and (even n_fft) Nyquist once, the others twice; their imaginary parts are ignored
        const bool edge = k == 0 || 2 * k == n_fft;
        v[(size_t)(2 * k) * in + n] = (edge ? 1.0 : 2.0) * co / n_fft;
        v[(size_t)(2 * k + 1) * in + n] = edge ? 0.0 : -2.0 * si / n_fft;
      }
    return img;
  }, &p);
  if (e != cudaSuccess) return e;
  *fwd = reinterpret_cast<const double*>(p + f_at);
  *inv = reinterpret_cast<const double*>(p + v_at);
  return cudaSuccess;
}

cudaError_t launch_pitch_shift(const float* x, const PitchPlan& p, const double* fwd, const double* inv, void* ws,
                               float* out, cudaStream_t st) {
  char* w = reinterpret_cast<char*>(ws);
  const PitchLayout l = pitch_layout(p);
  double* spec = reinterpret_cast<double*>(w + l.spec);
  double* stretched = reinterpret_cast<double*>(w + l.stretched);
  double* chunk = p.stretch ? reinterpret_cast<double*>(w + l.chunk) : nullptr;
  double* frames = reinterpret_cast<double*>(w + l.frames);
  double* y = reinterpret_cast<double*>(w + l.y);

  const int nb = p.nb;
  GemmA fa{};
  fa.x = x; fa.row_stride = p.N; fa.M = p.F; fa.K = p.n_fft; fa.N = p.N; fa.hop = p.hop; fa.pad = p.n_fft / 2;
  dft_gemm_kernel<true><<<dim3((p.F + BM - 1) / BM, (2 * nb + BN - 1) / BN, p.rows), GT, 0, st>>>(
      fa, fwd, round_up(p.n_fft, BK), round_up(2 * nb, BN), spec, 2 * nb, 2 * nb);
  count_launch();
  if (p.stretch) {
    const long long n = (long long)p.rows * p.F * nb;
    to_polar_kernel<<<grid_for(n, 256), 256, 0, st>>>(reinterpret_cast<double2*>(spec), n);
    count_launch();
    VocoderArgs va;
    va.pol = reinterpret_cast<const double2*>(spec); va.out = reinterpret_cast<double2*>(stretched); va.chunk = chunk;
    va.F = p.F; va.F2 = p.F2; va.nb = nb; va.nchunks = p.nchunks;
    va.rate = (float)p.rate; va.adv_end = (float)(M_PI * p.hop);
    vocoder_step_kernel<<<dim3(p.nchunks, p.rows), VT, 0, st>>>(va);
    count_launch();
    chunk_offsets_kernel<<<dim3((nb + VT - 1) / VT, p.rows), VT, 0, st>>>(va);
    count_launch();
    vocoder_polar_kernel<<<dim3(p.nchunks, p.rows), VT, 0, st>>>(va);
    count_launch();
  }
  GemmA ia{};
  ia.a = stretched; ia.row_stride = (long long)p.F2 * 2 * nb; ia.M = p.F2; ia.K = 2 * nb; ia.lda = 2 * nb;
  dft_gemm_kernel<false><<<dim3((p.F2 + BM - 1) / BM, (p.n_fft + BN - 1) / BN, p.rows), GT, 0, st>>>(
      ia, inv, round_up(2 * nb, BK), round_up(p.n_fft, BN), frames, p.n_fft, p.n_fft);
  count_launch();
  overlap_add_kernel<<<dim3(grid_for(p.L, 256), p.rows), 256, 0, st>>>(frames, p.F2, p.n_fft, p.hop, p.L, y);
  count_launch();
  ResampleArgs ra;
  ra.y = y; ra.out = out; ra.L = p.L; ra.target = p.target; ra.N = p.N; ra.identity = !p.resample;
  ra.orig_g = p.orig_g; ra.new_g = p.new_g; ra.base = p.base; ra.scale = p.scale; ra.width = p.width;
  ra.reach = p.resample ? 6.0 * (double)p.orig_g / p.base : 0.0;
  resample_kernel<<<dim3(grid_for(p.N, 256), p.rows), 256, 0, st>>>(ra);
  count_launch();
  return cudaGetLastError();
}

cudaError_t launch_pitch_time_steps(float rate, long long n, float* out, cudaStream_t st) {
  time_steps_kernel<<<grid_for(n, 256), 256, 0, st>>>(rate, n, out);
  count_launch();
  return cudaGetLastError();
}

}  // namespace vnb
