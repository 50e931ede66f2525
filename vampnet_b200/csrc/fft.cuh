// vampnet_b200 — the radix-2 real FFT in shared memory of the spectrogram kernel (mel.cu), in fp32 (float2) or float64
// (double2).  An NFFT-point real transform runs as an NFFT/2-point complex FFT of the even/odd sample pairs, then the
// real split.  Twiddles are twiddle[k] = exp(-2 pi i k / NFFT), k = 0..NFFT/2 (fft_tables()).
#pragma once
#include <cuda_runtime.h>

namespace vnb {

__device__ __forceinline__ float2 cmul(float2 a, float2 b) {
  return make_float2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x);
}
__device__ __forceinline__ double2 cmul(double2 a, double2 b) {
  return make_double2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x);
}

// z[NFFT/2], loaded in bit-reversed order by the caller, is transformed in place by the `nthreads` threads tid of the
// block; every thread of the block must call it (it synchronises the block after each stage).  Radix-2 decimation in
// time; stage `len` uses W_len^k = twiddle[k * NFFT / len].
template <int NFFT, typename C2>
__device__ __forceinline__ void fft_radix2(C2* z, const C2* twiddle, int tid, int nthreads) {
  constexpr int NH = NFFT / 2;
  for (int len = 2; len <= NH; len <<= 1) {
    const int half = len >> 1, step = NFFT / len;
    for (int j = tid; j < NH / 2; j += nthreads) {
      const int k = j & (half - 1);
      const int i0 = (j - k) * 2 + k, i1 = i0 + half;
      const C2 u = z[i0], v = cmul(z[i1], twiddle[k * step]);
      z[i0] = C2{u.x + v.x, u.y + v.y};
      z[i1] = C2{u.x - v.x, u.y - v.y};
    }
    __syncthreads();
  }
}

// bin k (0..NFFT/2) of the real transform from the complex FFT z: E = (Z[k] + conj Z[NH-k]) / 2,
// O = (Z[k] - conj Z[NH-k]) / 2i, X[k] = E + W_NFFT^k O
template <int NFFT, typename C2>
__device__ __forceinline__ C2 rfft_bin(const C2* z, const C2* twiddle, int k) {
  constexpr int NH = NFFT / 2;
  using R = decltype(C2::x);
  const R h = R(0.5);
  const C2 zk = z[k & (NH - 1)], zn = z[(NH - k) & (NH - 1)];
  const C2 e = C2{h * (zk.x + zn.x), h * (zk.y - zn.y)};
  const C2 o = C2{h * (zk.y + zn.y), -h * (zk.x - zn.x)};
  const C2 wo = cmul(o, twiddle[k]);
  return C2{e.x + wo.x, e.y + wo.y};
}

}  // namespace vnb
