// vampnet_b200 — the validation metrics of the reference's training script (scripts/exp/train.py:155-213, 327-371):
// the label-smoothed cross-entropy over the masked tokens and top-1 / top-25 accuracy split by masked and unmasked
// positions and by mask ratio, from the fp32 logits (B, S, V) a forward wrote.  Three launches on one stream, no host
// round trip, every reduction in a fixed order:
//   xent_rows_kernel   one warp per (b, s) row: the row's V logits read once (16-byte loads), the max by shuffles,
//                      sum exp(x - max) and sum x in float64 (each lane over its columns in a fixed order, then a
//                      fixed shuffle tree), the target's logit from its lane and the ranks gt / eq by ballots; one
//                      XentRow record per row
//   xent_items_kernel  one CTA per batch item: the masked rows' nll / smooth sums and the {unmasked, masked} x
//                      {top-1, top-25} correct / ambiguous / total / bad counts
//   xent_final_kernel  one thread: the loss over all items in float64 (rounded to fp32 once) and the 8 accuracies
//                      over the items of each r range
// A row's record depends on that row's logits alone, so a batched row equals the row run alone, bit for bit.
// DESIGN.md §12 has the semantics; oracle/validate_oracle.py restates them in float64.
#include <cmath>

#include "kernels.h"

namespace vnb {

namespace {
constexpr int ROW_WARPS = 8;                  // rows per CTA of xent_rows_kernel
constexpr int SLOTS = XENT_MAX_V / 128;       // float4s per lane
constexpr int ITEM_THREADS = 256, ITEM_WARPS = ITEM_THREADS / 32;
__host__ __device__ constexpr int topk(int k) { return k ? 25 : 1; }  // k 0 = top-1, 1 = top-25

// per batch item: the masked rows' nll / smooth sums and 12 counts; sel 0 = unmasked rows, 1 = masked rows; k 0 =
// top-1, 1 = top-25
constexpr int ITEM_INTS = 12;
__host__ __device__ constexpr int N_(int sel) { return sel; }                     // rows
__host__ __device__ constexpr int COR(int sel, int k) { return 2 + 2 * sel + k; }  // target in every top-k
__host__ __device__ constexpr int AMB(int sel, int k) { return 6 + 2 * sel + k; }  // a tie at the k-th place decides
__host__ __device__ constexpr int BAD(int sel) { return 10 + sel; }                // out-of-range target
struct XentItem {
  double nll, smooth;
  int32_t cnt[ITEM_INTS];
};

__global__ void __launch_bounds__(ROW_WARPS * 32)
xent_rows_kernel(const float* __restrict__ logits, const int64_t* __restrict__ z, long long rows, long long S, int C,
                 int T, int ncc, int V, XentRow* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const long long row = (long long)blockIdx.x * ROW_WARPS + (threadIdx.x >> 5);
  if (row >= rows) return;  // the whole warp leaves together
  const int Cp = C - ncc, nv = V >> 2;
  const long long b = row / S, s = row - b * S;
  const int64_t tgt = z[(b * C + ncc + s % Cp) * T + s / Cp];
  const float4* x4 = reinterpret_cast<const float4*>(logits + row * V);
  float4 x[SLOTS];
#pragma unroll
  for (int j = 0; j < SLOTS; ++j)
    x[j] = lane + 32 * j < nv ? __ldcs(x4 + lane + 32 * j) : make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
  float m = -INFINITY;
#pragma unroll
  for (int j = 0; j < SLOTS; ++j) m = fmaxf(m, fmaxf(fmaxf(x[j].x, x[j].y), fmaxf(x[j].z, x[j].w)));
  for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  const double md = m;
  double se = 0.0, sx = 0.0;
#pragma unroll
  for (int j = 0; j < SLOTS; ++j) {
    if (lane + 32 * j < nv) {
      const float v[4] = {x[j].x, x[j].y, x[j].z, x[j].w};
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        se += exp((double)v[c] - md);
        sx += (double)v[c];
      }
    }
  }
  // xor pairs add the same two values in either lane, so every lane ends with the same bits
  for (int o = 16; o; o >>= 1) {
    se += __shfl_xor_sync(0xffffffffu, se, o);
    sx += __shfl_xor_sync(0xffffffffu, sx, o);
  }
  XentRow r;
  if (tgt < 0 || tgt >= V) {  // an out-of-range code: the record is NaN, so are the loss and accuracies it enters
    r.nll = r.smooth = __longlong_as_double(0x7ff8000000000000ll);
    r.gt = r.eq = -1;
  } else {
    const int t = (int)tgt, slot = (t >> 2) >> 5, owner = (t >> 2) & 31, comp = t & 3;
    float mine = 0.f;
#pragma unroll
    for (int j = 0; j < SLOTS; ++j)
      if (j == slot) mine = comp == 0 ? x[j].x : comp == 1 ? x[j].y : comp == 2 ? x[j].z : x[j].w;
    const float xt = __shfl_sync(0xffffffffu, mine, owner);
    int gt = 0, eq = 0;
#pragma unroll
    for (int j = 0; j < SLOTS; ++j) {
      const bool ok = lane + 32 * j < nv;
      const float v[4] = {x[j].x, x[j].y, x[j].z, x[j].w};
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const int col = 4 * (lane + 32 * j) + c;
        gt += __popc(__ballot_sync(0xffffffffu, ok && v[c] > xt));
        eq += __popc(__ballot_sync(0xffffffffu, ok && v[c] == xt && col != t));
      }
    }
    const double lse = md + log(se);
    r.nll = lse - (double)xt;
    r.smooth = lse - sx / V;
    r.gt = gt;
    r.eq = eq;
  }
  if (lane == 0) out[row] = r;
}

// SEL a template argument, so that cnt[] stays in registers
template <int SEL>
__device__ __forceinline__ void tally(const XentRow& r, int* cnt) {
  ++cnt[N_(SEL)];
  if (r.gt < 0) {
    ++cnt[BAD(SEL)];
    return;
  }
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    if (r.gt + r.eq < topk(k)) ++cnt[COR(SEL, k)];
    else if (r.gt < topk(k)) ++cnt[AMB(SEL, k)];
  }
}

__global__ void __launch_bounds__(ITEM_THREADS)
xent_items_kernel(const XentRow* __restrict__ rows, const int64_t* __restrict__ mask, long long S, int C, int T,
                  int ncc, XentItem* __restrict__ items) {
  __shared__ double red_d[2][ITEM_WARPS];
  __shared__ int red_i[ITEM_INTS][ITEM_WARPS];
  const int b = blockIdx.x, Cp = C - ncc, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double nll = 0.0, smooth = 0.0;
  int cnt[ITEM_INTS] = {};
  for (long long s = threadIdx.x; s < S; s += ITEM_THREADS) {
    const XentRow r = rows[b * S + s];
    if (mask[((long long)b * C + ncc + s % Cp) * T + s / Cp] != 0) {
      tally<1>(r, cnt);
      nll += r.nll;
      smooth += r.smooth;
    } else {
      tally<0>(r, cnt);
    }
  }
  for (int o = 16; o; o >>= 1) {
    nll += __shfl_xor_sync(0xffffffffu, nll, o);
    smooth += __shfl_xor_sync(0xffffffffu, smooth, o);
  }
#pragma unroll
  for (int i = 0; i < ITEM_INTS; ++i) cnt[i] = __reduce_add_sync(0xffffffffu, cnt[i]);
  if (lane == 0) {
    red_d[0][warp] = nll;
    red_d[1][warp] = smooth;
#pragma unroll
    for (int i = 0; i < ITEM_INTS; ++i) red_i[i][warp] = cnt[i];
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    XentItem it;
    it.nll = red_d[0][0];
    it.smooth = red_d[1][0];
    for (int w = 1; w < ITEM_WARPS; ++w) {
      it.nll += red_d[0][w];
      it.smooth += red_d[1][w];
    }
    for (int i = 0; i < ITEM_INTS; ++i) {
      int v = 0;
      for (int w = 0; w < ITEM_WARPS; ++w) v += red_i[i][w];
      it.cnt[i] = v;
    }
    items[b] = it;
  }
}

// out[0] = loss; out[1 + 4 range + 2 k + sel] = accuracy, range 0 = [0, 0.5), 1 = [0.5, 1.0), the reference's key order
__global__ void xent_final_kernel(const XentItem* __restrict__ items, const double* __restrict__ r, int B, double eps,
                                  float* __restrict__ out, int32_t* __restrict__ ambiguous) {
  if (threadIdx.x != 0) return;
  double nll = 0.0, smooth = 0.0;
  long long n = 0, bad_all = 0;
  long long tot[2][2] = {}, cor[2][2][2] = {}, amb[2][2][2] = {}, bad[2][2] = {};  // [range][sel], [range][sel][k]
  for (int b = 0; b < B; ++b) {
    const XentItem& it = items[b];
    nll += it.nll;
    smooth += it.smooth;
    n += it.cnt[N_(1)];
    bad_all += it.cnt[BAD(0)] + it.cnt[BAD(1)];
    const double rb = r[b];
    const int range = rb >= 0.0 && rb < 0.5 ? 0 : rb >= 0.5 && rb < 1.0 ? 1 : -1;
    if (range < 0) continue;
    for (int sel = 0; sel < 2; ++sel) {
      tot[range][sel] += it.cnt[N_(sel)];
      bad[range][sel] += it.cnt[BAD(sel)];
      for (int k = 0; k < 2; ++k) {
        cor[range][sel][k] += it.cnt[COR(sel, k)];
        amb[range][sel][k] += it.cnt[AMB(sel, k)];
      }
    }
  }
  const float qnan = __int_as_float(0x7fc00000);
  // an out-of-range code anywhere makes the loss NaN, even in an unmasked row (the reference raises there)
  const bool any_bad = bad_all > 0;
  out[0] = n > 0 && !any_bad ? (float)(((1.0 - eps) * nll + eps * smooth) / (double)n) : qnan;
  if (ambiguous) ambiguous[0] = 0;
  for (int range = 0; range < 2; ++range)
    for (int k = 0; k < 2; ++k)
      for (int sel = 0; sel < 2; ++sel) {
        const int i = 1 + 4 * range + 2 * k + sel;
        // torch's mean of 0 / 1 floats: an exact fp32 count over an fp32 count (both below 2^24)
        out[i] = tot[range][sel] > 0 && bad[range][sel] == 0
                     ? (float)cor[range][sel][k] / (float)tot[range][sel] : qnan;
        if (ambiguous) ambiguous[i] = (int32_t)amb[range][sel][k];
      }
}

size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }
}  // namespace

size_t xent_workspace_bytes(long long B, long long S) {
  return align256((size_t)(B * S) * sizeof(XentRow)) + (size_t)B * sizeof(XentItem);
}

cudaError_t launch_xent_rows(const float* logits, const int64_t* z, int B, int C, int T, int ncc, int V, XentRow* rows,
                             cudaStream_t st) {
  const long long S = (long long)T * (C - ncc), n = (long long)B * S;
  xent_rows_kernel<<<(unsigned)((n + ROW_WARPS - 1) / ROW_WARPS), ROW_WARPS * 32, 0, st>>>(logits, z, n, S, C, T, ncc,
                                                                                          V, rows);
  count_launch();
  return cudaGetLastError();
}

cudaError_t launch_xent_metrics(const float* logits, const int64_t* z, const int64_t* mask, const double* r, int B,
                                int C, int T, int ncc, int V, double eps, void* workspace, float* out,
                                int32_t* ambiguous, cudaStream_t st) {
  const long long S = (long long)T * (C - ncc);
  XentRow* rows = static_cast<XentRow*>(workspace);
  XentItem* items = reinterpret_cast<XentItem*>(static_cast<char*>(workspace) + align256((size_t)(B * S) * sizeof(XentRow)));
  cudaError_t e = launch_xent_rows(logits, z, B, C, T, ncc, V, rows, st);
  if (e != cudaSuccess) return e;
  xent_items_kernel<<<B, ITEM_THREADS, 0, st>>>(rows, mask, S, C, T, ncc, items);
  count_launch();
  if ((e = cudaGetLastError()) != cudaSuccess) return e;
  xent_final_kernel<<<1, 32, 0, st>>>(items, r, B, eps, out, ambiguous);
  count_launch();
  return cudaGetLastError();
}

}  // namespace vnb
