// vampnet_b200 — the fp32 radix-2 real FFT in shared memory of the spectrogram kernel (mel.cu).  An NFFT-point real
// transform runs as an NFFT/2-point complex FFT of the even/odd sample pairs, then the real split.  Twiddles are
// twiddle[k] = exp(-2 pi i k / NFFT), k = 0..NFFT/2 (fft_tables()).
#pragma once
#include <cuda_runtime.h>

namespace vnb {

__device__ __forceinline__ float2 cmul(float2 a, float2 b) {
  return make_float2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x);
}

// z[NFFT/2], loaded in bit-reversed order by the caller, is transformed in place by the `nthreads` threads tid of the
// block; every thread of the block must call it (it synchronises the block after each stage).  Radix-2 decimation in
// time; stage `len` uses W_len^k = twiddle[k * NFFT / len].
template <int NFFT>
__device__ __forceinline__ void fft_radix2(float2* z, const float2* twiddle, int tid, int nthreads) {
  constexpr int NH = NFFT / 2;
  for (int len = 2; len <= NH; len <<= 1) {
    const int half = len >> 1, step = NFFT / len;
    for (int j = tid; j < NH / 2; j += nthreads) {
      const int k = j & (half - 1);
      const int i0 = (j - k) * 2 + k, i1 = i0 + half;
      const float2 u = z[i0], v = cmul(z[i1], twiddle[k * step]);
      z[i0] = make_float2(u.x + v.x, u.y + v.y);
      z[i1] = make_float2(u.x - v.x, u.y - v.y);
    }
    __syncthreads();
  }
}

// bin k (0..NFFT/2) of the real transform from the complex FFT z: E = (Z[k] + conj Z[NH-k]) / 2,
// O = (Z[k] - conj Z[NH-k]) / 2i, X[k] = E + W_NFFT^k O
template <int NFFT>
__device__ __forceinline__ float2 rfft_bin(const float2* z, const float2* twiddle, int k) {
  constexpr int NH = NFFT / 2;
  const float2 zk = z[k & (NH - 1)], zn = z[(NH - k) & (NH - 1)];
  const float2 e = make_float2(0.5f * (zk.x + zn.x), 0.5f * (zk.y - zn.y));
  const float2 o = make_float2(0.5f * (zk.y + zn.y), -0.5f * (zk.x - zn.x));
  const float2 wo = cmul(o, twiddle[k]);
  return make_float2(e.x + wo.x, e.y + wo.y);
}

}  // namespace vnb
