// vampnet_b200 — the Fréchet audio distance of the reference's evaluation script (frechet_audio_distance with
// torchvggish's VGGish, use_pca=False, use_activation=False), restated on the device (DESIGN.md §14):
//   examples   launch_vggish_frontend (mel.cu): 16 kHz samples -> float64 log-mel examples rounded to fp32 once
//   embed      vggish_in_kernel (conv_wgmma.cu) for the Cin = 1 layer, then conv_wgmma_kernel for the five 3x3
//              convolutions (2-D addressing, ReLU and the fused 2x2 max-pool) and the three fully connected layers,
//              every layer NHWC, split-bf16 operands into fp32 accumulators
//   moments    fad_mean_kernel, fad_cov_kernel: np.mean and np.cov(rowvar=False) of the embeddings in float64, every
//              sum in row order, so they do not depend on how the embeddings were batched
// The 128 x 128 matrix square root of the distance stays on the host (scipy.linalg.sqrtm, the reference's call).
#include <utility>

#include "kernels.h"

namespace vnb {

namespace {
// the largest activation of one example: layer 1's (48, 32, 64) and layer 3's (24, 16, 256)
constexpr size_t VGG_ACT = 48 * 32 * 64;
static_assert(VGG_ACT == 24 * 16 * 256, "the two largest activations");
constexpr int EMB = 128;

__global__ void __launch_bounds__(EMB) fad_mean_kernel(const float* __restrict__ x, long long M,
                                                       double* __restrict__ mu) {
  const int i = threadIdx.x;
  double s = 0.0;
  for (long long m = 0; m < M; ++m) s += (double)x[m * EMB + i];
  mu[i] = s / (double)M;
}

// one CTA per row i of sigma, thread j: sum over m in order of (x[m, i] - mu[i]) (x[m, j] - mu[j]), times 1 / (M - 1)
// as np.cov scales it
__global__ void __launch_bounds__(EMB) fad_cov_kernel(const float* __restrict__ x, long long M,
                                                      const double* __restrict__ mu, double* __restrict__ sigma) {
  const int i = blockIdx.x, j = threadIdx.x;
  const double mi = mu[i], mj = mu[j];
  double s = 0.0;
  for (long long m = 0; m < M; ++m) s = fma((double)x[m * EMB + i] - mi, (double)x[m * EMB + j] - mj, s);
  sigma[i * EMB + j] = s * (1.0 / (double)(M - 1));
}
}  // namespace

size_t vggish_workspace_bytes(int n_ex) {
  size_t o = 0;
  for (int k = 0; k < 4; ++k) carve(o, (size_t)n_ex * VGG_ACT * sizeof(__nv_bfloat16));  // A hi / lo, B hi / lo
  return o;
}

cudaError_t launch_vggish_embed(const VggishNet& net, const float* examples, int n_ex, void* workspace, float* out,
                                cudaStream_t st) {
  size_t o = 0;
  char* ws = static_cast<char*>(workspace);
  void* buf[4];
  for (int k = 0; k < 4; ++k) buf[k] = ws + carve(o, (size_t)n_ex * VGG_ACT * sizeof(__nv_bfloat16));
  void *ah = buf[0], *al = buf[1], *bh = buf[2], *bl = buf[3];
  cudaError_t e = launch_vggish_in(examples, net.w1, net.b1, n_ex, ah, al, st);
  // features 3..13: (H, W, Cin) -> Cout, pooled or not; the activations alternate between the A and B buffers
  struct Conv { int H, W, Cin, Cout; bool pool; };
  const Conv convs[5] = {{48, 32, 64, 128, true}, {24, 16, 128, 256, false}, {24, 16, 256, 256, true},
                         {12, 8, 256, 512, false}, {12, 8, 512, 512, true}};
  for (int l = 0; l < 5 && e == cudaSuccess; ++l) {
    const Conv& c = convs[l];
    e = launch_vggish_tc(ah, al, n_ex, c.H, c.W, c.Cin, net.conv_hi[l], net.conv_lo[l], c.Cout, net.conv_b[l], true,
                         c.pool, bh, bl, nullptr, st);
    std::swap(ah, bh);
    std::swap(al, bl);
  }
  // embeddings 0, 2, 4: the pooled (6, 4, 512) NHWC image is torchvggish's flatten order
  const int fc_k[3] = {6 * 4 * 512, 4096, 4096}, fc_n[3] = {4096, 4096, EMB};
  for (int l = 0; l < 3 && e == cudaSuccess; ++l) {
    const bool relu = l < 2;
    e = launch_vggish_tc(ah, al, n_ex, 0, 0, fc_k[l], net.fc_hi[l], net.fc_lo[l], fc_n[l], net.fc_b[l], relu, false,
                         bh, bl, relu ? nullptr : out, st);
    std::swap(ah, bh);
    std::swap(al, bl);
  }
  return e;
}

cudaError_t launch_fad_moments(const float* emb, long long M, double* mu, double* sigma, cudaStream_t st) {
  fad_mean_kernel<<<1, EMB, 0, st>>>(emb, M, mu);
  fad_cov_kernel<<<EMB, EMB, 0, st>>>(emb, M, mu, sigma);
  count_launch(2);
  return cudaGetLastError();
}

}  // namespace vnb
