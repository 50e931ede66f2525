// vampnet_b200 — beat tracking for the beat-synced mask (reference vampnet/interface.py:226-322 takes its beat times
// from WaveBeat; this is librosa 0.10.1's beat.beat_track(y, sr, hop_length=H) restated instead), all on one stream
// with no host round trip:
//   mel_spec_kernel        (mel.cu, ONSET_DB mode, as onset detection runs it) the fp32 mel dB spectrogram
//   beat_floor_kernel      one CTA per row: the clip's dB maximum minus top_db = 80
//   beat_flux_kernel       one warp per (frame, row): the clamped spectral flux of the 128 bands and its median (the
//                          mean of the 64th and 65th smallest), shifted by the envelope's padding: the fp32 envelope
//   beat_tempogram_kernel  one CTA per (chunk of frames, row), float64 from here on: each frame's ramp-padded,
//                          Hann-windowed 8 s window, its autocorrelation over all W lags divided by the largest |value|,
//                          summed over the chunk's frames
//   beat_track_kernel      one CTA per row: the mean tempogram, the prior and the tempo argmax; the envelope over its
//                          standard deviation and the Gaussian local score; the dynamic programme (one warp, the best
//                          of ~1.5 period predecessors per frame); the last beat, the backtrack and the trim
// DESIGN.md §10 has the numerics; oracle/beat_oracle.py restates the algorithm in float64.  The tables (window, tempo
// frequencies) are built here on the host and cached by device_table.
#include <cfloat>
#include <climits>
#include <cmath>

#include "kernels.h"
#include "reduce.cuh"

namespace vnb {

namespace {
constexpr int NMELS = ONSET_NMELS, THREADS = 256, WARPS = THREADS / 32;
constexpr int MAXG = 2 * BEAT_MAX_LAGS;  // Gaussian taps (2 period + 1) and DP candidates, period <= W - 1

// (value, index) with the larger value, the smaller index on a tie: numpy's argmax keeps the first maximum
__device__ __forceinline__ void arg_better(double& v, int& i, double ov, int oi) {
  if (ov > v || (ov == v && oi < i)) { v = ov; i = oi; }
}
__device__ void warp_argmax(double& v, int& i) {
  for (int o = 16; o; o >>= 1) arg_better(v, i, __shfl_xor_sync(0xffffffffu, v, o), __shfl_xor_sync(0xffffffffu, i, o));
}

__global__ void __launch_bounds__(THREADS) beat_floor_kernel(const float* __restrict__ db, int F,
                                                             float* __restrict__ floor_db) {
  __shared__ double red[WARPS];
  const float* d = db + (size_t)blockIdx.x * F * NMELS;
  float mx = -INFINITY;
  for (size_t i = threadIdx.x; i < (size_t)F * NMELS; i += THREADS) mx = fmaxf(mx, d[i]);
  mx = (float)block_reduce<Reduce::MAX, WARPS>((double)mx, red);  // exact: a float's maximum
  if (threadIdx.x == 0) floor_db[blockIdx.x] = mx - 80.f;
}

__global__ void __launch_bounds__(THREADS) beat_flux_kernel(const float* __restrict__ db, int F, int pad,
                                                            const float* __restrict__ floor_db, float* __restrict__ env) {
  const int b = blockIdx.y, lane = threadIdx.x & 31, i = blockIdx.x * WARPS + (threadIdx.x >> 5);
  if (i >= F) return;
  float e = 0.f;
  if (i >= pad) {  // env[i] = median flux between frames i - pad and i - pad + 1 (librosa's lag + n_fft // 2 hop shift)
    const float fl = floor_db[b];
    const float* cur = db + ((size_t)b * F + (i - pad + 1)) * NMELS;
    const float* prev = cur - NMELS;
    float v[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int m = lane + 32 * q;
      v[q] = fmaxf(0.f, fmaxf(cur[m], fl) - fmaxf(prev[m], fl));
    }
    // rank of band m: how many bands are smaller, or equal with a lower index, so every rank 0..127 occurs once
    int rank[4] = {0, 0, 0, 0};
#pragma unroll
    for (int q2 = 0; q2 < 4; ++q2) {
      for (int l = 0; l < 32; ++l) {
        const float w = __shfl_sync(0xffffffffu, v[q2], l);
        const int n = l + 32 * q2;
#pragma unroll
        for (int q = 0; q < 4; ++q) rank[q] += (w < v[q]) || (w == v[q] && n < lane + 32 * q);
      }
    }
    float lo = 0.f, hi = 0.f;  // the flux is >= 0, so a max over the warp picks the one band holding each rank
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      if (rank[q] == NMELS / 2 - 1) lo = v[q];
      if (rank[q] == NMELS / 2) hi = v[q];
    }
    for (int o = 16; o; o >>= 1) {
      lo = fmaxf(lo, __shfl_xor_sync(0xffffffffu, lo, o));
      hi = fmaxf(hi, __shfl_xor_sync(0xffffffffu, hi, o));
    }
    e = (lo + hi) / 2.f;  // np.median of float32: the mean of the two middle values, in float32
  }
  if (lane == 0) env[(size_t)b * F + i] = e;
}

constexpr int LAGS_PER_THREAD = BEAT_MAX_LAGS / THREADS;

__global__ void __launch_bounds__(THREADS) beat_tempogram_kernel(const float* __restrict__ env, int F, BeatTables t,
                                                                 int fpc, double* __restrict__ partial) {
  __shared__ double a[BEAT_MAX_LAGS];
  __shared__ double red[WARPS];
  const int c = blockIdx.x, b = blockIdx.y, W = t.W, half = W / 2;
  const float* e = env + (size_t)b * F;
  // np.pad(mode="linear_ramp", end_values=0): linspace(0, edge, half, endpoint=False) on the left, reversed on the right
  const double step0 = (double)e[0] / half, step1 = (double)e[F - 1] / half;
  double acc[LAGS_PER_THREAD];
#pragma unroll
  for (int r = 0; r < LAGS_PER_THREAD; ++r) acc[r] = 0.0;
  for (int f = c * fpc, f1 = min(F, f + fpc); f < f1; ++f) {
    for (int j = threadIdx.x; j < W; j += THREADS) {
      const int q = f + j;  // index into the padded envelope
      const double p = q < half ? q * step0 : q < half + F ? (double)e[q - half] : (half - 1 - (q - half - F)) * step1;
      a[j] = t.window[j] * p;
    }
    __syncthreads();
    double ac[LAGS_PER_THREAD], mx = 0.0;
#pragma unroll
    for (int r = 0; r < LAGS_PER_THREAD; ++r) {
      const int k = threadIdx.x + r * THREADS;
      double s = 0.0;
      if (k < W)
        for (int j = 0; j + k < W; ++j) s = fma(a[j], a[j + k], s);
      ac[r] = s;
      mx = fmax(mx, fabs(s));
    }
    // also orders this frame's reads of a[] before the next frame's writes
    mx = block_reduce<Reduce::MAX, WARPS>(mx, red);
    if (mx < DBL_MIN) mx = 1.0;  // util.normalize leaves a frame below tiny(float64) as it is
#pragma unroll
    for (int r = 0; r < LAGS_PER_THREAD; ++r) acc[r] += ac[r] / mx;
  }
  double* out = partial + ((size_t)b * gridDim.x + c) * W;
#pragma unroll
  for (int r = 0; r < LAGS_PER_THREAD; ++r) {
    const int k = threadIdx.x + r * THREADS;
    if (k < W) out[k] = acc[r];
  }
}

// per-row float64 / int32 scratch of beat_track_kernel, row b's slice at b * (its length)
struct TrackScratch {
  const double* partial;           // (B, nchunk, W) tempogram sums per chunk of frames
  int nchunk;
  double *x, *ls, *cum, *vals;     // (B, F): scaled envelope, local score, cumulative score, maxima / smoothed score
  double *gauss, *txwt;            // (B, MAXG)
  int32_t *back, *chain;           // (B, F)
};

__global__ void __launch_bounds__(THREADS) beat_track_kernel(const float* __restrict__ env, int F, BeatTables t,
                                                             TrackScratch s, double fps, double log2_start,
                                                             double tightness, int trim, double* __restrict__ tempo,
                                                             int32_t* __restrict__ beats, int32_t* __restrict__ counts) {
  __shared__ double red[WARPS];
  __shared__ int ired[WARPS];
  __shared__ double s_lo, s_hi;
  __shared__ int s_n;
  const int b = blockIdx.x, W = t.W, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const float* e = env + (size_t)b * F;
  double* x = s.x + (size_t)b * F;
  double* ls = s.ls + (size_t)b * F;
  double* cum = s.cum + (size_t)b * F;
  double* vals = s.vals + (size_t)b * F;
  double* gauss = s.gauss + (size_t)b * MAXG;
  double* txwt = s.txwt + (size_t)b * MAXG;
  int32_t* back = s.back + (size_t)b * F;
  int32_t* chain = s.chain + (size_t)b * F;
  int any = 0;
  for (int i = threadIdx.x; i < F; i += THREADS) any |= e[i] != 0.f;
  if (!__syncthreads_or(any)) {  // beat_track: no onsets, tempo 0 and no beats
    if (threadIdx.x == 0) { tempo[b] = 0.0; counts[b] = 0; }
    return;
  }
  // ---- tempo: argmax over lags of log1p(1e6 mean tempogram) + log-normal prior, lags at >= 320 BPM excluded
  const double* part = s.partial + (size_t)b * s.nchunk * W;
  double best = -INFINITY;
  int bk = INT_MAX;
  for (int k = threadIdx.x; k < W; k += THREADS) {
    double sum = 0.0;
    for (int c = 0; c < s.nchunk; ++c) sum += part[(size_t)c * W + k];
    double lp = -INFINITY;
    if (k >= t.max_idx) {
      const double d = t.log2_bpm[k] - log2_start;  // std_bpm = 1
      lp = -0.5 * (d * d);
    }
    arg_better(best, bk, log1p(1e6 * (sum / F)) + lp, k);
  }
  warp_argmax(best, bk);
  __syncthreads();
  if (lane == 0) { red[warp] = best; ired[warp] = bk; }
  __syncthreads();
  best = red[0];
  bk = ired[0];
  for (int w = 1; w < WARPS; ++w) arg_better(best, bk, red[w], ired[w]);
  if (bk == INT_MAX) bk = 0;  // every score -inf: numpy's argmax is 0
  const double bpm = t.bpm[bk];
  if (threadIdx.x == 0) tempo[b] = bpm;
  const double pr = rint(60.0 * fps / bpm);  // Python's round: half to even
  if (!(pr >= 1.0)) {  // a period below one frame (or an infinite tempo): no beats
    if (threadIdx.x == 0) counts[b] = 0;
    return;
  }
  const int period = (int)pr, h = (int)rint(period * 0.5), L = 2 * period - h + 1;
  // ---- local score: the envelope over its standard deviation (ddof = 1), convolved with a Gaussian
  double sum = 0.0;
  for (int i = threadIdx.x; i < F; i += THREADS) sum += e[i];
  const double mean = block_reduce<Reduce::SUM, WARPS>(sum, red) / F;
  double sq = 0.0;
  for (int i = threadIdx.x; i < F; i += THREADS) sq += ((double)e[i] - mean) * ((double)e[i] - mean);
  sq = block_reduce<Reduce::SUM, WARPS>(sq, red);
  const double norm = F > 1 ? sqrt(sq / (F - 1)) : NAN;
  for (int i = threadIdx.x; i < F; i += THREADS) x[i] = norm > 0 ? (double)e[i] / norm : (double)e[i];
  for (int j = threadIdx.x; j <= 2 * period; j += THREADS) {
    const double u = (double)(j - period) * 32.0 / period;
    gauss[j] = exp(-0.5 * (u * u));
  }
  for (int c = threadIdx.x; c < L; c += THREADS) {  // predecessor i - 2 period + c, weight -tightness log(-w / period)^2
    const double l = log((double)(2 * period - c) / period);
    txwt[c] = -tightness * (l * l);
  }
  __syncthreads();
  double lmax = -INFINITY;
  for (int i = threadIdx.x; i < F; i += THREADS) {
    double acc = 0.0;
    for (int j = max(0, period - i), j1 = min(2 * period, F - 1 - i + period); j <= j1; ++j)
      acc += x[i + j - period] * gauss[j];
    ls[i] = acc;
    lmax = fmax(lmax, acc);
  }
  // also orders the ls[] writes before the reads below
  const double thr = 0.01 * block_reduce<Reduce::MAX, WARPS>(lmax, red);
  // ---- dynamic programme: one warp, frame by frame
  if (warp == 0) {
    bool first = true;
    for (int i = 0; i < F; ++i) {
      double bv = -INFINITY;
      int bc = INT_MAX;
      for (int c = lane; c < L; c += 32) {
        const int q = i - 2 * period + c;
        // a predecessor before frame 0 contributes its weight alone; q == i (period 1) reads librosa's zero
        const double v = q >= 0 && q < i ? txwt[c] + cum[q] : txwt[c];
        if (v > bv) { bv = v; bc = c; }
      }
      warp_argmax(bv, bc);
      const double li = ls[i];
      int link;
      if (first && li < thr) {
        link = -1;
      } else {
        link = i - 2 * period + bc;
        first = false;
      }
      if (lane == 0) { cum[i] = li + bv; back[i] = link; }
      __syncwarp();
    }
  }
  if (threadIdx.x == 0) s_n = 0;
  __syncthreads();
  // ---- last beat: local maxima of cum (edge-padded), the median of their values, the last maximum above half of it
  for (int i = threadIdx.x; i < F; i += THREADS) {
    const double v = cum[i];
    if (v > cum[max(i - 1, 0)] && v >= cum[min(i + 1, F - 1)]) vals[atomicAdd(&s_n, 1)] = v;
  }
  __syncthreads();
  const int K = s_n;
  if (K == 0) {
    if (threadIdx.x == 0) counts[b] = 0;
    return;
  }
  for (int m = threadIdx.x; m < K; m += THREADS) {  // order statistics (K - 1) / 2 and K / 2, ties ranked by slot
    const double v = vals[m];
    int r = 0;
    for (int n = 0; n < K; ++n) r += vals[n] < v || (vals[n] == v && n < m);
    if (r == (K - 1) / 2) s_lo = v;
    if (r == K / 2) s_hi = v;
  }
  __syncthreads();
  const double med = (K & 1) ? s_hi : (s_lo + s_hi) / 2;
  int tail = -1;
  for (int i = threadIdx.x; i < F; i += THREADS) {
    const double v = cum[i];
    if (v > cum[max(i - 1, 0)] && v >= cum[min(i + 1, F - 1)] && 2.0 * v > med) tail = max(tail, i);
  }
  for (int o = 16; o; o >>= 1) tail = max(tail, __shfl_xor_sync(0xffffffffu, tail, o));
  __syncthreads();
  if (lane == 0) ired[warp] = tail;
  __syncthreads();
  if (threadIdx.x != 0) return;
  for (int w = 1; w < WARPS; ++w) tail = max(tail, ired[w]);
  tail = max(tail, ired[0]);
  if (tail < 0) { counts[b] = 0; return; }
  // ---- backtrack, then the trim: the local score at the beats smoothed by [0.5, 1, 0.5], kept above 0.5 RMS
  int n = 0;
  for (int i = tail; i >= 0 && n < F; i = back[i]) ++n;
  for (int k = n - 1, i = tail; k >= 0; --k, i = back[i]) chain[k] = i;
  double ssq = 0.0;
  for (int j = 0; j < n; ++j) {
    const double xm = j > 0 ? ls[chain[j - 1]] : 0.0, xn = j + 1 < n ? ls[chain[j + 1]] : 0.0;
    const double sm = (xm * 0.5 + ls[chain[j]]) + xn * 0.5;
    vals[j] = sm;
    ssq += sm * sm;
  }
  const double cut = trim ? 0.5 * sqrt(ssq / n) : 0.0;
  int lo = -1, hi = -1;
  for (int j = 0; j < n; ++j)
    if (vals[j] > cut) { if (lo < 0) lo = j; hi = j; }
  int32_t* out = beats + (size_t)b * F;
  const int cnt = lo < 0 ? 0 : hi - lo;  // beats[valid.min():valid.max()]
  for (int j = 0; j < cnt; ++j) out[j] = chain[lo + j];
  counts[b] = cnt;
}

// the workspace, in order: mel dB (B, F, 128) f32, floors (B) f32, tempogram chunk sums, TrackScratch's arrays
struct BeatLayout {
  size_t db, floor, partial, x, ls, cum, vals, gauss, txwt, back, chain, total;
};
BeatLayout beat_layout(int B, int F) {
  BeatLayout l;
  size_t o = 0;
  const size_t bf = (size_t)B * F;
  l.db = carve(o, bf * NMELS * sizeof(float));
  l.floor = carve(o, (size_t)B * sizeof(float));
  // nchunk * W <= (F / fpc + 1) * W <= 256 F + W with fpc = ceil(W / 256)
  l.partial = carve(o, (size_t)B * (256 * (size_t)F + BEAT_MAX_LAGS) * sizeof(double));
  l.x = carve(o, bf * sizeof(double));
  l.ls = carve(o, bf * sizeof(double));
  l.cum = carve(o, bf * sizeof(double));
  l.vals = carve(o, bf * sizeof(double));
  l.gauss = carve(o, (size_t)B * MAXG * sizeof(double));
  l.txwt = carve(o, (size_t)B * MAXG * sizeof(double));
  l.back = carve(o, bf * sizeof(int32_t));
  l.chain = carve(o, bf * sizeof(int32_t));
  l.total = o;
  return l;
}

cudaError_t launch_decisions(const float* env, int B, int F, int sr, int hop, const BeatTables& t, double start_bpm,
                             double tightness, int trim, char* ws, double* tempo, int32_t* beats, int32_t* counts,
                             cudaStream_t st) {
  const BeatLayout l = beat_layout(B, F);
  const int fpc = (t.W + 255) / 256, nchunk = (F + fpc - 1) / fpc;
  double* partial = reinterpret_cast<double*>(ws + l.partial);
  beat_tempogram_kernel<<<dim3(nchunk, B), THREADS, 0, st>>>(env, F, t, fpc, partial);
  count_launch();
  TrackScratch s;
  s.partial = partial;
  s.nchunk = nchunk;
  s.x = reinterpret_cast<double*>(ws + l.x);
  s.ls = reinterpret_cast<double*>(ws + l.ls);
  s.cum = reinterpret_cast<double*>(ws + l.cum);
  s.vals = reinterpret_cast<double*>(ws + l.vals);
  s.gauss = reinterpret_cast<double*>(ws + l.gauss);
  s.txwt = reinterpret_cast<double*>(ws + l.txwt);
  s.back = reinterpret_cast<int32_t*>(ws + l.back);
  s.chain = reinterpret_cast<int32_t*>(ws + l.chain);
  beat_track_kernel<<<B, THREADS, 0, st>>>(env, F, t, s, (double)sr / hop, std::log2(start_bpm), tightness, trim,
                                           tempo, beats, counts);
  count_launch();
  return cudaGetLastError();
}

// tempo_frequencies: inf, then 60 sr / (hop k)
double tempo_bpm(int sr, int hop, int k) { return k == 0 ? INFINITY : 60.0 * sr / ((double)hop * k); }
}  // namespace

int beat_lags(int sr, int hop) { return (int)std::min<long long>(8LL * sr / hop, INT_MAX); }

size_t beat_workspace_bytes(int B, int F) { return beat_layout(B, F).total; }

// one table: the window, the tempo frequencies, their log2 (W doubles each)
cudaError_t beat_tables(int sr, int hop, BeatTables* out) {
  const int W = beat_lags(sr, hop);
  if (W < 2 || W > BEAT_MAX_LAGS) return cudaErrorInvalidValue;
  const char* p = nullptr;
  cudaError_t e = device_table({TABLE_BEAT, (double)sr, (double)hop}, [&] {
    // scipy's periodic Hann (0.5 + 0.5 cos of linspace(-pi, pi, W + 1)), tempo_frequencies and their log2, in float64
    std::vector<char> img(3 * sizeof(double) * W);
    double *win = reinterpret_cast<double*>(img.data()), *bpm = win + W, *l2 = bpm + W;
    const double step = 2.0 * M_PI / W;
    for (int k = 0; k < W; ++k) {
      win[k] = 0.5 + 0.5 * std::cos(k * step + -M_PI);
      bpm[k] = tempo_bpm(sr, hop, k);
      l2[k] = std::log2(bpm[k]);
    }
    return img;
  }, &p);
  if (e != cudaSuccess) return e;
  out->window = reinterpret_cast<const double*>(p);
  out->bpm = out->window + W;
  out->log2_bpm = out->bpm + W;
  out->W = W;
  out->max_idx = 0;  // np.argmax of all-False
  for (int k = 0; k < W; ++k)
    if (tempo_bpm(sr, hop, k) < 320.0) { out->max_idx = k; break; }
  return cudaSuccess;
}

cudaError_t launch_beat_track(const float* samples, int B, int N, int sr, int hop, const OnsetTables& ot,
                              const BeatTables& bt, double start_bpm, double tightness, int trim, void* workspace,
                              float* env, double* tempo, int32_t* beats, int32_t* counts, cudaStream_t st) {
  const int F = 1 + N / hop;
  char* ws = static_cast<char*>(workspace);
  const BeatLayout l = beat_layout(B, F);
  float* db = reinterpret_cast<float*>(ws + l.db);
  float* floor_db = reinterpret_cast<float*>(ws + l.floor);
  cudaError_t e =
      launch_spectrogram(SpecMode::ONSET_DB, samples, B, N, hop, ONSET_NFFT, ot.fft, ot.bank, NMELS, db, st);
  if (e != cudaSuccess) return e;
  beat_floor_kernel<<<B, THREADS, 0, st>>>(db, F, floor_db);
  count_launch();
  beat_flux_kernel<<<dim3((F + WARPS - 1) / WARPS, B), THREADS, 0, st>>>(db, F, ot.g.pad, floor_db, env);
  count_launch();
  return launch_decisions(env, B, F, sr, hop, bt, start_bpm, tightness, trim, ws, tempo, beats, counts, st);
}

cudaError_t launch_beat_from_envelope(const float* env, int B, int F, int sr, int hop, const BeatTables& bt,
                                      double start_bpm, double tightness, int trim, void* workspace, double* tempo,
                                      int32_t* beats, int32_t* counts, cudaStream_t st) {
  return launch_decisions(env, B, F, sr, hop, bt, start_bpm, tightness, trim, static_cast<char*>(workspace), tempo,
                          beats, counts, st);
}

}  // namespace vnb
