// vampnet_b200 — C ABI (include/vampnet_b200.h): model handle, per-(B,T) workspaces with their TMA
// tensor maps, the forward pass, and the graph-captured generate() loop.
#include <cuda_bf16.h>
#include <cudaTypedefs.h>

#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <map>
#include <memory>
#include <string>
#include <tuple>
#include <vector>

#include "kernels.h"

namespace vnb {

static thread_local std::string g_err;
static thread_local std::string g_tmap_err;

static int fail(const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  g_err = buf;
  return 1;
}
#define CK(expr)                                                                                   \
  do {                                                                                             \
    cudaError_t _e = (expr);                                                                       \
    if (_e != cudaSuccess) return fail("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
  } while (0)

// ---------------------------------------------------------------------------------- tensor maps
static PFN_cuTensorMapEncodeTiled_v12000 get_encode() {
  static PFN_cuTensorMapEncodeTiled_v12000 fn = nullptr;
  if (fn) return fn;
  void* p = nullptr;
  cudaDriverEntryPointQueryResult q;
  cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q);
  if (e != cudaSuccess || q != cudaDriverEntryPointSuccess || !p) {
    g_tmap_err = std::string("cudaGetDriverEntryPoint(cuTensorMapEncodeTiled) failed: ") + cudaGetErrorString(e);
    return nullptr;
  }
  fn = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(p);
  return fn;
}
const char* tmap_error() { return g_tmap_err.c_str(); }

bool make_tmap_2d(CUtensorMap* tm, const void* base, uint64_t rows, uint64_t cols, uint32_t box_rows,
                  uint32_t box_cols) {
  auto enc = get_encode();
  if (!enc) return false;
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {cols * 2};
  cuuint32_t box[2] = {box_cols, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    char b[256];
    snprintf(b, sizeof(b), "cuTensorMapEncodeTiled(2d rows=%llu cols=%llu box=%ux%u) -> %d", (unsigned long long)rows,
             (unsigned long long)cols, box_rows, box_cols, (int)r);
    g_tmap_err = b;
    return false;
  }
  return true;
}
bool make_tmap_3d(CUtensorMap* tm, const void* base, uint64_t batch, uint64_t rows, uint64_t cols,
                  uint64_t pitch_elems, uint32_t box_rows, uint32_t box_cols) {
  auto enc = get_encode();
  if (!enc) return false;
  cuuint64_t dims[3] = {cols, rows, batch};
  cuuint64_t strides[2] = {pitch_elems * 2, rows * pitch_elems * 2};
  cuuint32_t box[3] = {box_cols, box_rows, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(base), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    char b[256];
    snprintf(b, sizeof(b), "cuTensorMapEncodeTiled(3d batch=%llu rows=%llu cols=%llu pitch=%llu box=%ux%u) -> %d",
             (unsigned long long)batch, (unsigned long long)rows, (unsigned long long)cols,
             (unsigned long long)pitch_elems, box_rows, box_cols, (int)r);
    g_tmap_err = b;
    return false;
  }
  return true;
}

bool make_tmap_4d(CUtensorMap* tm, const void* base, uint64_t batch, uint64_t H, uint64_t W, uint64_t C,
                  uint32_t box_h, uint32_t box_c) {
  auto enc = get_encode();
  if (!enc) return false;
  cuuint64_t dims[4] = {C, W, H, batch};
  cuuint64_t strides[3] = {C * 2, W * C * 2, H * W * C * 2};
  cuuint32_t box[4] = {box_c, static_cast<cuuint32_t>(W), box_h, 1};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(base), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    char b[256];
    snprintf(b, sizeof(b), "cuTensorMapEncodeTiled(4d batch=%llu H=%llu W=%llu C=%llu box=%ux%llux%u) -> %d",
             (unsigned long long)batch, (unsigned long long)H, (unsigned long long)W, (unsigned long long)C, box_h,
             (unsigned long long)W, box_c, (int)r);
    g_tmap_err = b;
    return false;
  }
  return true;
}

// Fills a plan's tensor maps (A (M,K) bf16, W (N,K) bf16) and arguments, with the fused RMSNorm (DESIGN.md §4) wired as
// in the forward: ss_in (non-null) makes the plan a consumer that scales its rows by rsqrt(mean(A^2) + eps) from ss_parts
// partial row sums of squares; out_bf16 (non-null) a producer that also stores bf16(out) and its row sums of squares
// to ss_out, the next GEMM's operand.
static bool make_gemm_plan(GemmPlan* p, int epi, const void* A, const void* W, int M, int N, int K, void* out,
                           void* out2, const float* bias, int T, int Tpad, const float* ss_in, int ss_parts,
                           float inv_d, float eps, void* out_bf16, float* ss_out) {
  if (N % 256 != 0 || K % 64 != 0 || M < 1) {
    g_tmap_err = "gemm: need N % 256 == 0 and K % 64 == 0";
    return false;
  }
  GemmArgs& a = p->args;
  a.M = M; a.N = N; a.K = K; a.epi = epi; a.out = out; a.out2 = out2; a.bias = bias;
  a.T = T; a.Tpad = Tpad; a.d2 = epi == VNB_EPI_QKV ? (N / 3) * 2 : 0;  // QKV: N = 3 d_model, v starts at 2 d_model
  if (ss_in != nullptr) { a.ss_in = ss_in; a.ss_parts = ss_parts; a.inv_d = inv_d; a.eps = eps; }
  a.out_bf16 = reinterpret_cast<__nv_bfloat16*>(out_bf16); a.ss_out = ss_out;
  return make_tmap_2d(&p->tmA, A, M, K, 128, 64) && make_tmap_2d(&p->tmB, W, N, K, 256, 64) &&
         make_tmap_2d(&p->tmBh, W, N, K, 128, 64);
}

bool make_attn_plan(AttnPlan* p, const void* qk, const void* vT, void* out, const float* rel, int sat, int B, int T,
                    int Tpad, int H) {
  const int d = H * 64;
  p->out = out; p->rel = rel; p->sat = sat; p->B = B; p->T = T; p->Tpad = Tpad; p->H = H;
  return make_tmap_3d(&p->tmQ, qk, B, T, 2 * d, 2 * d, 128, 64) && make_tmap_3d(&p->tmK, qk, B, T, 2 * d, 2 * d, 64, 64) &&
         make_tmap_3d(&p->tmVT, vT, B, d, Tpad, Tpad, 64, 64);
}

// ---------------------------------------------------------------------------------- model
struct DevBuf {
  void* p = nullptr;
  size_t n = 0;
  ~DevBuf() { if (p) cudaFree(p); }
  cudaError_t alloc(size_t bytes, bool zero = false) {
    n = bytes;
    cudaError_t e = cudaMalloc(&p, bytes ? bytes : 1);
    if (e == cudaSuccess && zero) e = cudaMemset(p, 0, bytes);
    return e;
  }
  template <class T> T* as() const { return reinterpret_cast<T*>(p); }
};

// Which kernels a launch runs.  It is also the key of a captured generate graph (graphs bake pointers, so generate()
// stages z/mask/out in workspace-owned buffers); a forward runs the default.
struct Variant {
  int steps = 0;          // generate iterations
  bool has_mask = false;
  bool top_p = false;     // selects the sampler kernel variant
  int gemm_pair = 0;      // GEMM kernel variant baked into the graph (vnb_set_option "gemm_pair")
  bool fused = false;     // sampler fused into the classifier epilogue (vnb_set_option "fused_sampler")
  bool adapted = false;   // LoRA down-projections + adapted GEMM epilogues (some group has an adapter)
  bool ragged = false;    // QKV and attention read the frames table (some group is shorter than T)
  bool mixed_steps = false;  // every kernel of iteration i reads the live table (some group has fewer steps than S)
  bool split = false;        // nucleus and plain groups in one fused launch: split classifier epilogue and sampler
  bool operator<(const Variant& o) const {
    return std::tie(steps, has_mask, top_p, gemm_pair, fused, adapted, ragged, mixed_steps, split) <
           std::tie(o.steps, o.has_mask, o.top_p, o.gemm_pair, o.fused, o.adapted, o.ragged, o.mixed_steps, o.split);
  }
};

struct Workspace {
  int B = 0, T = 0, Tpad = 0, M = 0;
  unsigned long long last_use = 0;
  // generate(): n0 (B) = initial mask count per group, dyn (kMaxSteps, B) = the SampleDyn table [step][group] with row
  // stride B, rowgrp (B) = the group of every batch row; all three are rewritten before every launch or graph replay
  DevBuf x, y, qk, vT, att, h, logits, zcur, zorig, tokens, conf, n0, dyn, rowgrp, z_in, mask_in, z_out, ssA, ssB, embA,
      partials;
  // adapted launches: grp_adapter (B) = the adapter of every group (-1: base), rewritten before every launch or replay;
  // lora_u (M, 16) = the down-projection of the GEMM about to run
  DevBuf grp_adapter, lora_u;
  // launches of calls with different lengths: frames (B) = the length of every batch row's call, rewritten before every
  // launch or replay (read by the QKV epilogue and attention)
  DevBuf frames;
  // launches of calls with different step counts: live (kMaxSteps) = the batch rows live at every iteration (a prefix),
  // rewritten before every launch or replay (read by every kernel of the iteration)
  DevBuf live;
  int embKp = 0;
  int ss_parts = 0;
  std::vector<GemmPlan> qkv, wo, up, down;
  GemmPlan cls, emb;
  GemmPlan cls_sample;  // the classifier with the sampling epilogue (generate loop)
  bool can_fuse = false;
  AttnPlan attn;
  std::map<Variant, cudaGraphExec_t> graphs;
  std::map<Variant, unsigned long long> graph_kernels;
  ~Workspace() { for (auto& kv : graphs) cudaGraphExecDestroy(kv.second); }
};

}  // namespace vnb

namespace vnb {
enum { FAM_EMBED = 0, FAM_RMSNORM, FAM_GEMM_QKV, FAM_ATTN, FAM_GEMM_O, FAM_GEMM_UP, FAM_GEMM_DOWN, FAM_GEMM_CLS,
       FAM_SAMPLE, FAM_STATE, FAM_LORA_DOWN, FAM_COUNT };
static unsigned long long g_captures = 0;  // generate graphs captured + instantiated so far
static unsigned long long g_launches = 0;  // kernels launched by this library (graph replays add their node count)
void count_launch(unsigned long long n) { g_launches += n; }
struct Profiler {
  bool on = false;
  std::vector<cudaEvent_t> pool;
  std::vector<int> fam;  // family of the launch that FOLLOWS event i
  size_t used = 0;
  ~Profiler() { for (auto e : pool) cudaEventDestroy(e); }
  void mark(int family, cudaStream_t st) {
    if (!on) return;
    if (used == pool.size()) {
      cudaEvent_t e;
      if (cudaEventCreate(&e) != cudaSuccess) { on = false; return; }
      pool.push_back(e);
      fam.push_back(-1);
    }
    fam[used] = family;
    cudaEventRecord(pool[used++], st);
  }
};
}  // namespace vnb

struct vnb_model {
  vnb_config cfg;
  vnb_weights w;
  vnb::Profiler prof;
  std::map<std::pair<int, int>, std::unique_ptr<vnb::Workspace>> ws;
  vnb::Workspace* last = nullptr;
  static constexpr int kMaxSteps = 256;
  static constexpr size_t kMaxWorkspaces = 6;
  unsigned long long use_clock = 0;
  // registered adapters: host copy of the table and its device image (rewritten before every adapted launch)
  vnb::AdapterDev adapters[VNB_MAX_ADAPTERS] = {};
  bool adapter_live[VNB_MAX_ADAPTERS] = {};
  vnb::DevBuf adapter_tab;
};

namespace vnb {

static int get_workspace(vnb_model* m, int B, int T, Workspace** out) {
  auto key = std::make_pair(B, T);
  auto it = m->ws.find(key);
  if (it != m->ws.end()) { it->second->last_use = ++m->use_clock; *out = it->second.get(); return 0; }
  // bound the number of live (B, T) workspaces (each holds activations, logits and captured graphs): evict the
  // least recently used one.  cudaFree synchronises the device, so nothing in flight can still touch it.
  while (m->ws.size() >= vnb_model::kMaxWorkspaces) {
    auto lru = m->ws.begin();
    for (auto i = m->ws.begin(); i != m->ws.end(); ++i)
      if (i->second->last_use < lru->second->last_use) lru = i;
    if (m->last == lru->second.get()) m->last = nullptr;
    cudaDeviceSynchronize();
    m->ws.erase(lru);
  }
  const vnb_config& c = m->cfg;
  const int d = c.d_model, L = c.n_layers, Cp = c.n_codebooks - c.n_conditioning_codebooks;
  auto ws = std::make_unique<Workspace>();
  ws->B = B; ws->T = T; ws->M = B * T; ws->Tpad = (T + 7) / 8 * 8;
  const size_t M = ws->M;
  CK(ws->x.alloc(M * d * 4));
  CK(ws->y.alloc(M * d * 2));  // bf16 copy of the residual stream (A operand of QKV / FFN-up / classifier)
  ws->ss_parts = 2 * (d / 256);  // two partial row-sums-of-squares (even / odd chunks) per 256-column tile of the producing GEMM
  CK(ws->ssA.alloc(M * ws->ss_parts * 4, true));
  CK(ws->ssB.alloc(M * ws->ss_parts * 4, true));
  ws->embKp = (c.n_codebooks * 8 + 63) / 64 * 64;                 // gathered latents [hi | hi | lo], each third padded to Kp
  CK(ws->embA.alloc(M * 3 * ws->embKp * 2));
  CK(ws->qk.alloc(M * 2 * d * 2));
  CK(ws->vT.alloc(static_cast<size_t>(B) * d * ws->Tpad * 2, /*zero=*/true));  // padding keys stay 0 forever
  CK(ws->att.alloc(M * d * 2));
  CK(ws->h.alloc(M * 2 * d * 2));
  // ws->logits (M x Cp*V fp32, 0.4-1 GB at the bench shapes) is only needed when generate() samples from a materialised
  // tensor (top-p, fused_sampler = 0): allocated on first use in vnb_generate
  CK(ws->zcur.alloc(M * c.n_codebooks * 4));
  CK(ws->zorig.alloc(M * c.n_codebooks * 4));
  CK(ws->tokens.alloc(M * Cp * 4));
  CK(ws->conf.alloc(M * Cp * 4));
  CK(ws->n0.alloc(4 * static_cast<size_t>(B), true));
  CK(ws->dyn.alloc(sizeof(SampleDyn) * vnb_model::kMaxSteps * B));
  CK(ws->rowgrp.alloc(sizeof(RowGroup) * B));
  CK(ws->grp_adapter.alloc(sizeof(int32_t) * B));
  CK(ws->frames.alloc(sizeof(int32_t) * B));
  CK(ws->live.alloc(sizeof(int32_t) * vnb_model::kMaxSteps));
  CK(ws->lora_u.alloc(M * 16 * 4));
  CK(ws->z_in.alloc(M * c.n_codebooks * 8));
  CK(ws->mask_in.alloc(M * c.n_codebooks * 4));
  CK(ws->z_out.alloc(M * c.n_codebooks * 8));
  const __nv_bfloat16* wqkv = reinterpret_cast<const __nv_bfloat16*>(m->w.wqkv);
  const __nv_bfloat16* wo = reinterpret_cast<const __nv_bfloat16*>(m->w.wo);
  const __nv_bfloat16* w1 = reinterpret_cast<const __nv_bfloat16*>(m->w.w1);
  const __nv_bfloat16* w2 = reinterpret_cast<const __nv_bfloat16*>(m->w.w2);
  ws->qkv.resize(L); ws->wo.resize(L); ws->up.resize(L); ws->down.resize(L);
  const size_t dd = static_cast<size_t>(d) * d;
  const float inv_d = 1.0f / static_cast<float>(d), eps = 1e-6f;
  // ss_in: the row sums of squares a consumer's A operand came with; ss_out: where a producer leaves them, with bf16(x) in y
  auto plan = [&](GemmPlan& p, int epi, const void* A, const void* W, int N, int K, void* out, void* out2,
                  const float* bias, const DevBuf* ss_in, const DevBuf* ss_out) {
    return make_gemm_plan(&p, epi, A, W, ws->M, N, K, out, out2, bias, T, ws->Tpad,
                          ss_in ? ss_in->as<float>() : nullptr, ws->ss_parts, inv_d, eps, ss_out ? ws->y.p : nullptr,
                          ss_out ? ss_out->as<float>() : nullptr);
  };
  for (int l = 0; l < L; ++l) {
    // residual stream x (fp32) + its bf16 copy y + row sums of squares: ssA feeds QKV, ssB feeds FFN-up
    bool ok = plan(ws->qkv[l], VNB_EPI_QKV, ws->y.p, wqkv + l * 3 * dd, 3 * d, d, ws->qk.p, ws->vT.p, nullptr, &ws->ssA,
                   nullptr) &&
              plan(ws->wo[l], VNB_EPI_RESID, ws->att.p, wo + l * dd, d, d, ws->x.p, nullptr, nullptr, nullptr, &ws->ssB) &&
              plan(ws->up[l], VNB_EPI_GEGLU, ws->y.p, w1 + l * 4 * dd, 4 * d, d, ws->h.p, nullptr, nullptr, &ws->ssB,
                   nullptr) &&
              plan(ws->down[l], VNB_EPI_RESID, ws->h.p, w2 + l * 2 * dd, d, 2 * d, ws->x.p, nullptr, nullptr, nullptr,
                   &ws->ssA);
    if (!ok) return fail("plan layer %d: %s", l, tmap_error());
  }
  if (!plan(ws->cls, VNB_EPI_BIAS_F32, ws->y.p, m->w.wcls, Cp * c.vocab_size, d, nullptr, nullptr, m->w.bcls, &ws->ssA,
            nullptr))
    return fail("plan classifier: %s", tmap_error());
  // generate loop: the same GEMM with the sampling epilogue; the logits are consumed in the epilogue and never stored
  ws->can_fuse = c.vocab_size % 128 == 0 && c.vocab_size <= 1024;
  if (ws->can_fuse) {
    CK(ws->partials.alloc(M * static_cast<size_t>(Cp) * (c.vocab_size / 128) * 16));
    ws->cls_sample = ws->cls;
    GemmArgs& s = ws->cls_sample.args;
    s.epi = VNB_EPI_SAMPLE;
    s.out = nullptr;
    s.zcur = ws->zcur.as<int32_t>();
    s.rowgrp = ws->rowgrp.as<RowGroup>();
    s.partials = ws->partials.as<float4>();
    s.C = c.n_codebooks; s.ncc = c.n_conditioning_codebooks; s.V = c.vocab_size; s.mask_token = c.vocab_size;
  }
  // embedding out_proj (layers.py:162) as a split-bf16 tensor-core contraction: x = A . emb_w3^T + bias, which also
  // emits bf16(x) and the row sums of squares the first QKV projection's fused RMSNorm consumes
  if (!plan(ws->emb, VNB_EPI_BIAS_F32, ws->embA.p, m->w.emb_w3, d, 3 * ws->embKp, ws->x.p, nullptr, m->w.emb_b, nullptr,
            &ws->ssA))
    return fail("plan embedding: %s", tmap_error());
  if (!make_attn_plan(&ws->attn, ws->qk.p, ws->vT.p, ws->att.p, m->w.rel_bias, m->w.rel_sat, B, T, ws->Tpad, c.n_heads))
    return fail("plan attention: %s", tmap_error());
  ws->last_use = ++m->use_clock;
  *out = ws.get();
  m->ws[key] = std::move(ws);
  return 0;
}

#define LAUNCH(fam_, expr)        \
  do {                            \
    m->prof.mark((fam_), st);     \
    CK(expr);                     \
    ++g_launches;                 \
  } while (0)

// CodebookEmbedding (layers.py:134-162): gather (+ split) the latents, then the out_proj contraction on the tensor cores.
// live (device, null = every row): batch rows at or past live[0] are not embedded.
static int run_embed(vnb_model* m, Workspace* ws, const int32_t* codes_btc, const float* latents, cudaStream_t st,
                     const int32_t* live = nullptr) {
  const vnb_config& c = m->cfg;
  LAUNCH(FAM_EMBED, launch_embed_gather(codes_btc, latents, m->w.emb_table, ws->embA.p, ws->M, ws->T, c.n_codebooks,
                                        c.vocab_size + 1, c.n_codebooks * 8, ws->embKp, ws->ssA.as<float>(),
                                        c.d_model / 256, ws->ss_parts, live, st));
  GemmPlan emb = ws->emb;
  emb.args.live = live;
  LAUNCH(FAM_EMBED, launch_gemm(emb, st));
  return 0;
}

// One LoRA'd GEMM of layer l: plain, or (adapted) the down-projection of its A operand `a` then the adapted epilogue.
static int run_lora_gemm(vnb_model* m, Workspace* ws, const GemmPlan& plan, int fam, bool adapted, int slot, int l,
                         const void* a, cudaStream_t st) {
  if (!adapted) {
    LAUNCH(fam, launch_gemm(plan, st));
    return 0;
  }
  GemmPlan p = plan;  // carries the live bound of the iteration, which the down-projection shares
  AdapterRefs& r = p.args.lora;
  r.table = m->adapter_tab.as<AdapterDev>();
  r.grp_adapter = ws->grp_adapter.as<int32_t>();
  r.rowgrp = ws->rowgrp.as<RowGroup>();
  r.rows_per_grp = ws->T;
  r.slot = slot;
  r.layer = l;
  r.u = ws->lora_u.as<float>();
  LAUNCH(FAM_LORA_DOWN, launch_lora_down(a, p.args.M, p.args.K, r, p.args.live, p.args.T, st));
  LAUNCH(fam, launch_gemm(p, st));
  return 0;
}

// x already holds the embedded input; runs the L layers + final norm + classifier into `logits`.  v.fused: the
// classifier samples in its epilogue instead, from row `iter` of the ws->dyn table; with v.split as well, the split
// epilogue stores the logits of the rows of nucleus (top-p) groups to `logits`.  v.ragged: batch row b is a call of
// ws->frames[b] frames; its later frames are padding that no earlier frame attends to.  v.mixed_steps: batch rows at or
// past ws->live[iter] are idle; every kernel skips the tiles and CTAs wholly past them.  acts (non-null): the residual
// stream after every layer.
static int run_stack(vnb_model* m, Workspace* ws, const Variant& v, int iter, float* logits, float* acts,
                     cudaStream_t st) {
  const vnb_config& c = m->cfg;
  // RMSNorm (transformer.py:43-58) is fused: norm weights are folded into wqkv / w1 / wcls at pack time, the
  // producers of x (embed, attn-out, ffn-down) also emit bf16(x) and per-row sums of squares, and the consumers
  // scale their accumulator rows by rsqrt(mean(x^2) + eps).
  const int32_t* frames = v.ragged ? ws->frames.as<int32_t>() : nullptr;
  const int32_t* live = v.mixed_steps ? ws->live.as<int32_t>() + iter : nullptr;
  AttnPlan attn = ws->attn;
  attn.frames = frames;
  attn.live = live;
  const auto bounded = [live](const GemmPlan& p) {
    GemmPlan q = p;
    q.args.live = live;
    return q;
  };
  for (int l = 0; l < c.n_layers; ++l) {
    GemmPlan qkv = bounded(ws->qkv[l]);
    qkv.args.frames = frames;
    if (run_lora_gemm(m, ws, qkv, FAM_GEMM_QKV, v.adapted, LORA_QKV, l, ws->y.p, st)) return 1;
    LAUNCH(FAM_ATTN, launch_attention(attn, st));
    if (run_lora_gemm(m, ws, bounded(ws->wo[l]), FAM_GEMM_O, v.adapted, LORA_WO, l, ws->att.p, st) ||
        run_lora_gemm(m, ws, bounded(ws->up[l]), FAM_GEMM_UP, v.adapted, LORA_W1, l, ws->y.p, st) ||
        run_lora_gemm(m, ws, bounded(ws->down[l]), FAM_GEMM_DOWN, v.adapted, LORA_W2, l, ws->h.p, st))
      return 1;
    if (acts)  // return_activations: the residual stream after this layer (transformer.py:455-456)
      CK(cudaMemcpyAsync(acts + static_cast<size_t>(l) * ws->M * c.d_model, ws->x.p, ws->x.n, cudaMemcpyDeviceToDevice, st));
  }
  if (v.fused) {  // generate loop: sample in the classifier's epilogue, no logits tensor
    GemmPlan cls = bounded(ws->cls_sample);
    cls.args.dyn = ws->dyn.as<SampleDyn>() + static_cast<size_t>(iter) * ws->B;
    if (v.split) {
      cls.args.out = logits;
      cls.sample_split = true;
    }
    LAUNCH(FAM_GEMM_CLS, launch_gemm(cls, st));
  } else {
    GemmPlan cls = bounded(ws->cls);
    cls.args.out = logits;
    LAUNCH(FAM_GEMM_CLS, launch_gemm(cls, st));
  }
  m->prof.mark(-1, st);
  return 0;
}

// temperature <= 0: softmax(logits) without scaling (transformer.py:1019-1023)
static float inv_temperature(float temperature) {
  return temperature > 0.f ? static_cast<float>(1.0 / static_cast<double>(temperature)) : 1.0f;
}

// The single-step entry points take their SampleDyn from a per-device ring of 64 device slots (a process-global ring
// would live on whichever device called first); each call stages its scalars into the next slot, stream-ordered.
static int stage_sample_dyn(const SampleDyn& d, cudaStream_t st, const SampleDyn** out) {
  static SampleDyn* scratch_dev[64] = {nullptr};
  static int slot_dev[64] = {0};
  int dev = 0;
  CK(cudaGetDevice(&dev));
  if (dev < 0 || dev >= 64) return fail("device index %d out of range", dev);
  SampleDyn*& scratch = scratch_dev[dev];
  int& slot = slot_dev[dev];
  if (!scratch) CK(cudaMalloc(&scratch, sizeof(SampleDyn) * 64));
  SampleDyn* dd = scratch + (slot++ & 63);
  CK(cudaMemcpyAsync(dd, &d, sizeof(d), cudaMemcpyHostToDevice, st));
  *out = dd;
  return 0;
}

// The row map of a one-call launch of up to `rows` batch rows: all zeros (group 0, starting at row 0).  One buffer per
// device, grown when a larger batch comes; never written after it is zeroed.
static int one_group_rows(int rows, const RowGroup** out) {
  static RowGroup* buf_dev[64] = {nullptr};
  static int cap_dev[64] = {0};
  int dev = 0;
  CK(cudaGetDevice(&dev));
  if (dev < 0 || dev >= 64) return fail("device index %d out of range", dev);
  if (cap_dev[dev] < rows) {
    if (buf_dev[dev]) CK(cudaFree(buf_dev[dev]));
    buf_dev[dev] = nullptr;
    cap_dev[dev] = 0;
    const int cap = rows > 1024 ? rows : 1024;
    CK(cudaMalloc(&buf_dev[dev], sizeof(RowGroup) * cap));
    CK(cudaMemset(buf_dev[dev], 0, sizeof(RowGroup) * cap));
    CK(cudaDeviceSynchronize());  // zeroed before any stream of any caller reads it
    cap_dev[dev] = cap;
  }
  *out = buf_dev[dev];
  return 0;
}

// The sampling scalars of one group at one step, as the sampling kernels read them.
static SampleDyn sample_dyn(const vnb_sample_group& q) {
  return SampleDyn{inv_temperature(q.temperature), q.gamma, q.temp_eff, q.do_sample, q.is_last, q.step, q.seed_lo,
                   q.seed_hi, q.top_p};
}

// The groups of a launch of B batch rows (vnb_gen_group or vnb_sample_group): 1..B groups of >= 1 rows each, B in all.
template <class Group>
static int check_groups(const Group* groups, int n_groups, int B, const char* who) {
  if (n_groups < 1 || n_groups > B) return fail("%s: n_groups %d out of range 1..B (B = %d)", who, n_groups, B);
  long long total = 0;
  for (int g = 0; g < n_groups; ++g) {
    if (groups[g].rows < 1) return fail("%s: group %d has %d rows", who, g, groups[g].rows);
    total += groups[g].rows;
  }
  if (total != B) return fail("%s: group rows sum to %lld, not B = %d", who, total, B);
  return 0;
}

// The row -> group map of checked groups: group g holds the groups[g].rows batch rows that follow group g - 1's.
template <class Group>
static std::vector<RowGroup> row_groups(const Group* groups, int n_groups, int B) {
  std::vector<RowGroup> rowgrp(B);
  for (int g = 0, first = 0; g < n_groups; first += groups[g].rows, ++g)
    for (int b = first; b < first + groups[g].rows; ++b) rowgrp[b] = RowGroup{g, first};
  return rowgrp;
}

static AdapterDev adapter_dev(const vnb_adapter_weights& w) {
  const float* ptrs[2 * LORA_SLOTS] = {w.a_qkv, w.b_qkv, w.a_wo, w.b_wo, w.a_w1, w.b_w1, w.a_w2, w.b_w2};
  AdapterDev a;
  for (int s = 0; s < LORA_SLOTS; ++s) { a.a[s] = ptrs[2 * s]; a.b[s] = ptrs[2 * s + 1]; }
  return a;
}

// Adapter ids of a launch (host, n entries; NULL = none): each -1 or a live id.
static int check_adapter_ids(const vnb_model* m, const int32_t* ids, int n, const char* who) {
  if (!ids) return 0;
  for (int i = 0; i < n; ++i)
    if (ids[i] != -1 && (ids[i] < 0 || ids[i] >= VNB_MAX_ADAPTERS || !m->adapter_live[ids[i]]))
      return fail("%s: entry %d names adapter %d, which is not registered", who, i, ids[i]);
  return 0;
}
static bool any_adapted(const int32_t* ids, int n) {
  for (int i = 0; ids && i < n; ++i)
    if (ids[i] >= 0) return true;
  return false;
}
// Stream-ordered writes of the adapter table and the group -> adapter map of an adapted launch (pageable sources:
// staged before the calls return).
static int stage_adapters(vnb_model* m, Workspace* ws, const int32_t* grp_adapter, int n_groups, cudaStream_t st) {
  CK(cudaMemcpyAsync(m->adapter_tab.p, m->adapters, sizeof(m->adapters), cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(ws->grp_adapter.p, grp_adapter, sizeof(int32_t) * n_groups, cudaMemcpyHostToDevice, st));
  return 0;
}

}  // namespace vnb

using namespace vnb;

extern "C" {

int32_t vnb_abi_version(void) { return VNB_ABI_VERSION; }
int32_t vnb_set_error_cuda(const char* what, int32_t cuda_error) {
  return fail("%s failed: %s", what, cudaGetErrorString(static_cast<cudaError_t>(cuda_error)));
}
const char* vnb_last_error(void) { return g_err.c_str(); }

int32_t vnb_model_create(const vnb_config* cfg, const vnb_weights* w, vnb_model** out) {
  if (!cfg || !w || !out) return fail("null argument");
  if (cfg->d_model != cfg->n_heads * 64) return fail("d_model must be n_heads*64 (got %d, %d)", cfg->d_model, cfg->n_heads);
  if (cfg->d_model % 256 != 0) return fail("d_model must be a multiple of 256");
  if (cfg->latent_dim != 8) return fail("latent_dim must be 8");
  if (cfg->vocab_size % 256 != 0 || cfg->vocab_size > 1024) return fail("vocab_size must be a multiple of 256, <= 1024");
  if (cfg->n_codebooks * 8 > 128) return fail("n_codebooks too large");
  if (w->rel_sat < 1 || w->rel_sat > 128) return fail("rel_sat out of range");
  int dev = 0, major = 0;
  CK(cudaGetDevice(&dev));
  CK(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev));
  if (major != 9) return fail("vampnet_b200 needs an sm_90 (Hopper) device (got compute capability major %d)", major);
  CK(prepare_gemm());
  auto* m = new vnb_model();
  m->cfg = *cfg;
  m->w = *w;
  if (m->adapter_tab.alloc(sizeof(m->adapters), true) != cudaSuccess) {
    delete m;
    return fail("vnb_model_create: cannot allocate the adapter table");
  }
  *out = m;
  return 0;
}

int32_t vnb_adapter_add(vnb_model* m, const vnb_adapter_weights* w, int32_t* id) {
  if (!m || !w || !id) return fail("vnb_adapter_add: null argument");
  const AdapterDev a = adapter_dev(*w);
  static const char* names[2 * LORA_SLOTS] = {"a_qkv", "b_qkv", "a_wo", "b_wo", "a_w1", "b_w1", "a_w2", "b_w2"};
  for (int i = 0; i < 2 * LORA_SLOTS; ++i)
    if (!(i % 2 ? a.b[i / 2] : a.a[i / 2])) return fail("vnb_adapter_add: %s is NULL", names[i]);
  int slot = -1;
  for (int i = 0; i < VNB_MAX_ADAPTERS && slot < 0; ++i)
    if (!m->adapter_live[i]) slot = i;
  if (slot < 0) return fail("vnb_adapter_add: the adapter table is full (%d live adapters)", VNB_MAX_ADAPTERS);
  m->adapters[slot] = a;
  m->adapter_live[slot] = true;
  *id = slot;
  return 0;
}

int32_t vnb_adapter_remove(vnb_model* m, int32_t id) {
  if (!m) return fail("vnb_adapter_remove: null model");
  if (id < 0 || id >= VNB_MAX_ADAPTERS || !m->adapter_live[id])
    return fail("vnb_adapter_remove: adapter %d is not registered", id);
  m->adapter_live[id] = false;
  m->adapters[id] = AdapterDev{};
  return 0;
}

void vnb_model_destroy(vnb_model* m) { delete m; }

int32_t vnb_forward_codes_adapted(vnb_model* m, const int64_t* codes, int32_t B, int32_t T, const int32_t* row_adapter,
                                  float* logits, void* stream) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (B < 1 || T < 1) return fail("vnb_forward_codes: need B >= 1 and T >= 1 (got %d, %d)", B, T);
  if (check_adapter_ids(m, row_adapter, B, "vnb_forward_codes_adapted")) return 1;
  const bool adapted = any_adapted(row_adapter, B);
  Workspace* ws;
  if (get_workspace(m, B, T, &ws)) return 1;
  if (adapted) {  // batch row b is its own group
    std::vector<RowGroup> rowgrp(B);
    for (int b = 0; b < B; ++b) rowgrp[b] = RowGroup{b, b};
    CK(cudaMemcpyAsync(ws->rowgrp.p, rowgrp.data(), sizeof(RowGroup) * B, cudaMemcpyHostToDevice, st));
    if (stage_adapters(m, ws, row_adapter, B, st)) return 1;
  }
  const vnb_config& c = m->cfg;
  // (B,C,T) int64 -> (B,T,C) int32, no masking (mask = zeros)
  LAUNCH(FAM_STATE, launch_gen_init(codes, nullptr, ws->zcur.as<int32_t>(), ws->zorig.as<int32_t>(), ws->n0.as<int32_t>(),
                                    nullptr, 1, B, c.n_codebooks, T, /*ncc=*/c.n_codebooks, c.vocab_size, st));
  if (run_embed(m, ws, ws->zcur.as<int32_t>(), nullptr, st)) return 1;
  m->last = ws;
  Variant v;
  v.adapted = adapted;
  return run_stack(m, ws, v, 0, logits, nullptr, st);
}

int32_t vnb_forward_codes(vnb_model* m, const int64_t* codes, int32_t B, int32_t T, float* logits, void* stream) {
  return vnb_forward_codes_adapted(m, codes, B, T, nullptr, logits, stream);
}

int32_t vnb_forward_latents(vnb_model* m, const float* latents, int32_t B, int32_t T, float* logits, void* stream) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  Workspace* ws;
  if (get_workspace(m, B, T, &ws)) return 1;
  if (run_embed(m, ws, nullptr, latents, st)) return 1;
  m->last = ws;
  return run_stack(m, ws, Variant{}, 0, logits, nullptr, st);
}

int32_t vnb_forward_latents_acts(vnb_model* m, const float* latents, int32_t B, int32_t T, float* logits, float* acts,
                                 void* stream) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  Workspace* ws;
  if (get_workspace(m, B, T, &ws)) return 1;
  if (run_embed(m, ws, nullptr, latents, st)) return 1;
  m->last = ws;
  return run_stack(m, ws, Variant{}, 0, logits, acts, st);
}

int32_t vnb_get_hidden(vnb_model* m, float* out, void* stream) {
  if (!m->last) return fail("no forward has run");
  CK(cudaMemcpyAsync(out, m->last->x.p, m->last->x.n, cudaMemcpyDeviceToDevice, reinterpret_cast<cudaStream_t>(stream)));
  return 0;
}

// vnb_set_option("fused_sampler", 0|1): sample inside the classifier GEMM's epilogue (default) or from a materialised
// logits tensor.  Nucleus (top-p) filtering needs whole sorted rows: its rows always draw from materialised logits (in a
// fused launch of nucleus and plain groups, from those the split classifier epilogue stores).
static int g_fused_sampler = -1;  // -1: not read yet (environment VNB_FUSED_SAMPLER, else on)
static int fused_sampler_enabled() {
  if (g_fused_sampler < 0) {
    const char* e = getenv("VNB_FUSED_SAMPLER");
    g_fused_sampler = e != nullptr ? (e[0] != '0') : 1;
  }
  return g_fused_sampler;
}
}  // extern "C"

// v.mixed_steps: iteration i runs only the batch rows ws->live[i] counts (a prefix); the others are idle and untouched.
// v.split (with v.fused): nucleus and plain groups; the classifier stores the nucleus rows' logits, and the sampler runs
// the combine for the plain rows and the nucleus draw for the others.
static int enqueue_generate(vnb_model* m, Workspace* ws, const int64_t* z, const int32_t* mask, int64_t* out,
                            const Variant& v, cudaStream_t st) {
  const vnb_config& c = m->cfg;
  const int ncc = c.n_conditioning_codebooks;
  // the whole n0 array is zeroed (a captured graph replays with any number of groups up to B)
  LAUNCH(FAM_STATE, launch_gen_init(z, mask, ws->zcur.as<int32_t>(), ws->zorig.as<int32_t>(), ws->n0.as<int32_t>(),
                                    ws->rowgrp.as<RowGroup>(), ws->B, ws->B, c.n_codebooks, ws->T, ncc, c.vocab_size, st));
  SampleArgs sa;
  sa.logits = ws->logits.as<float>();
  sa.zcur = ws->zcur.as<int32_t>();
  sa.zorig = ws->zorig.as<int32_t>();
  sa.tokens = ws->tokens.as<int32_t>();
  sa.conf = ws->conf.as<float>();
  sa.n0 = ws->n0.as<int32_t>();
  sa.rowgrp = ws->rowgrp.as<RowGroup>();
  sa.B = ws->B; sa.T = ws->T; sa.C = c.n_codebooks; sa.ncc = ncc; sa.V = c.vocab_size; sa.mask_token = c.vocab_size;
  for (int i = 0; i < v.steps; ++i) {
    sa.live = v.mixed_steps ? ws->live.as<int32_t>() + i : nullptr;
    if (run_embed(m, ws, ws->zcur.as<int32_t>(), nullptr, st, sa.live)) return 1;
    if (run_stack(m, ws, v, i, ws->logits.as<float>(), nullptr, st)) return 1;
    const SampleDyn* dyn_i = ws->dyn.as<SampleDyn>() + static_cast<size_t>(i) * ws->B;
    if (v.split) {
      LAUNCH(FAM_SAMPLE, launch_sample_split_dev(sa, ws->partials.p, dyn_i, st));
      ++g_launches;  // the split sampler is one kernel more
    } else if (v.fused) {
      LAUNCH(FAM_SAMPLE, launch_sample_combine_dev(sa, ws->partials.p, dyn_i, st));
    } else {
      LAUNCH(FAM_SAMPLE, launch_sample_step_dev(sa, dyn_i, st, v.top_p));
    }
    ++g_launches;  // sample step = two kernels
  }
  LAUNCH(FAM_STATE, launch_gen_finish(ws->tokens.as<int32_t>(), ws->zorig.as<int32_t>(), out, ws->B, c.n_codebooks, ws->T, ncc, st));
  m->prof.mark(-1, st);
  return 0;
}

// One generate launch as a vnb_generate* entry point describes it.  Group g runs steps_g steps with its own gamma
// schedule: group_steps[g] and group_gamma[g] from the entry points that take them (per_group), else every group runs
// `steps` with `gamma`.
struct GenDesc {
  const char* who;  // the entry point called, named in refusals
  const int64_t* z;
  const int32_t* mask;
  int B, T;
  const vnb_gen_group* groups;
  int n_groups, use_graph;
  int64_t* out;
  int steps = 0;
  const float* gamma = nullptr;
  bool per_group = false;
  const int32_t* group_steps = nullptr;
  const float* const* group_gamma = nullptr;
  const int32_t* group_frames = nullptr;   // null: every group has T frames
  const int32_t* group_adapter = nullptr;  // null: no group is adapted
  bool mixed_top_p = false;  // groups may mix nucleus (top-p) and plain sampling
};

// Every refusal of a generate launch, required pointers first.  Fills what the description decides of the launch's
// variant: v->steps = S, the most steps of any group; *top_p_mix: groups mix nucleus and plain sampling.
static int check_generate(const vnb_model* m, const GenDesc& d, Variant* v, bool* top_p_mix) {
  constexpr int kMax = vnb_model::kMaxSteps;
  if (d.per_group ? (!d.group_steps || !d.group_gamma || !d.groups) : (!d.gamma || !d.groups))
    return fail("%s: %s are required", d.who, d.per_group ? "group_steps, group_gamma and groups" : "gamma and groups");
  if (d.B < 1 || d.T < 1) return fail("%s: need B >= 1 and T >= 1 (got %d, %d)", d.who, d.B, d.T);
  if (check_groups(d.groups, d.n_groups, d.B, d.who)) return 1;
  if (!d.per_group && (d.steps < 1 || d.steps > kMax)) return fail("%s: bad sampling_steps %d (1..%d)", d.who, d.steps, kMax);
  const auto top_p_on = [](float tp) { return tp > 0.f && tp < 1.f; };
  v->steps = d.per_group ? d.group_steps[0] : d.steps;
  v->has_mask = d.mask != nullptr;
  v->top_p = top_p_on(d.groups[0].top_p);
  for (int g = 0; g < d.n_groups; ++g) {
    const vnb_gen_group& q = d.groups[g];
    if (d.per_group) {
      const int n = d.group_steps[g];
      if (n < 1 || n > kMax) return fail("%s: group %d has %d sampling steps, outside 1..%d", d.who, g, n, kMax);
      // longest first: the live rows of every iteration are then a prefix of the batch
      if (g > 0 && n > d.group_steps[g - 1])
        return fail("%s: group %d has %d steps, more than group %d's %d (the order must be non-increasing)", d.who, g,
                    n, g - 1, d.group_steps[g - 1]);
      if (!d.group_gamma[g]) return fail("%s: group %d lacks its schedules (gamma)", d.who, g);
      v->mixed_steps |= n != v->steps;
    }
    if (!q.temp_eff || !q.do_sample) return fail("%s: group %d lacks its schedules", d.who, g);
    // outside vnb_generate_mixed_top_p the sampler variant is chosen per launch: a mixed launch would filter
    // differently from the separate calls
    if (top_p_on(q.top_p) != top_p_on(d.groups[0].top_p)) {
      if (!d.mixed_top_p) return fail("%s: groups mix top-p and no top-p sampling", d.who);
      *top_p_mix = true;
      v->top_p = true;
    }
    // a group shorter than T: its rows' later frames are padding (kept frames in z / mask) that attention never reads
    if (d.group_frames && (d.group_frames[g] < 1 || d.group_frames[g] > d.T))
      return fail("%s: group %d has %d frames, outside 1..T (T = %d)", d.who, g, d.group_frames[g], d.T);
    v->ragged |= d.group_frames && d.group_frames[g] < d.T;
  }
  // without a mask every predicted codebook is masked, padding included: it would be sampled and count in N0
  if (v->ragged && !d.mask) return fail("%s: a launch with groups shorter than T needs a mask", d.who);
  if (check_adapter_ids(m, d.group_adapter, d.n_groups, d.who)) return 1;
  v->adapted = any_adapted(d.group_adapter, d.n_groups);
  return 0;
}

// The launch behind every vnb_generate* entry point.  Group g is idle for the first S - steps_g iterations and then runs
// its own step j = i - (S - steps_g) with j's schedule values, Philox step word and last-step flag.  With mixed_top_p,
// each row draws as its group's own launch would.
static int generate(vnb_model* m, const GenDesc& d, void* stream) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  Variant v;
  bool top_p_mix = false;
  if (check_generate(m, d, &v, &top_p_mix)) return 1;
  const int B = d.B, S = v.steps;
  Workspace* ws;
  if (get_workspace(m, B, d.T, &ws)) return 1;
  m->last = ws;
  // the [step][group] table (row stride B), the row map, the frames and the live rows per iteration, pageable sources:
  // the runtime stages them before returning, so the vectors may die at scope exit
  std::vector<SampleDyn> dyn(static_cast<size_t>(S) * B);
  const std::vector<RowGroup> rowgrp = row_groups(d.groups, d.n_groups, B);
  std::vector<int32_t> frames(v.ragged ? B : 0);
  std::vector<int32_t> live(v.mixed_steps ? S : 0, 0);
  for (int g = 0; g < d.n_groups; ++g) {
    const vnb_gen_group& q = d.groups[g];
    const int steps_g = d.per_group ? d.group_steps[g] : S;
    const float* gam = d.per_group ? d.group_gamma[g] : d.gamma;
    const int idle = S - steps_g;  // iterations before the group's first step
    vnb_sample_group s = {};  // an idle group's entry: no kernel reads more than its temperature, seeds and top-p
    s.temperature = q.temperature; s.seed_lo = q.seed_lo; s.seed_hi = q.seed_hi; s.top_p = q.top_p;
    for (int i = 0; i < S; ++i) {
      if (i >= idle) {
        const int j = i - idle;
        s.gamma = gam[j]; s.temp_eff = q.temp_eff[j]; s.do_sample = q.do_sample[j]; s.is_last = j == steps_g - 1;
        s.step = j;
        if (v.mixed_steps) live[i] += q.rows;
      }
      dyn[static_cast<size_t>(i) * B + g] = sample_dyn(s);
    }
  }
  for (int b = 0; v.ragged && b < B; ++b) frames[b] = d.group_frames[rowgrp[b].group];
  CK(cudaMemcpyAsync(ws->dyn.p, dyn.data(), sizeof(SampleDyn) * dyn.size(), cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(ws->rowgrp.p, rowgrp.data(), sizeof(RowGroup) * B, cudaMemcpyHostToDevice, st));
  if (v.ragged) CK(cudaMemcpyAsync(ws->frames.p, frames.data(), sizeof(int32_t) * B, cudaMemcpyHostToDevice, st));
  if (v.mixed_steps) CK(cudaMemcpyAsync(ws->live.p, live.data(), sizeof(int32_t) * S, cudaMemcpyHostToDevice, st));
  if (v.adapted && stage_adapters(m, ws, d.group_adapter, d.n_groups, st)) return 1;
  // a mix of nucleus and plain groups: the split path when the sampler is fused, else the materialising path with the
  // nucleus kernel for every row (a group whose top-p is off draws there as without the filter, bit for bit)
  v.split = top_p_mix && fused_sampler_enabled() != 0 && ws->can_fuse;
  v.fused = fused_sampler_enabled() != 0 && (!v.top_p || v.split) && ws->can_fuse;
  v.gemm_pair = get_gemm_pair();
  if ((!v.fused || v.split) && ws->logits.p == nullptr)  // before any capture: cudaMalloc is not capturable
    CK(ws->logits.alloc(static_cast<size_t>(ws->M) * (m->cfg.n_codebooks - m->cfg.n_conditioning_codebooks) * m->cfg.vocab_size * 4));
  if (!d.use_graph || m->prof.on) return enqueue_generate(m, ws, d.z, d.mask, d.out, v, st);

  const size_t nz = static_cast<size_t>(B) * m->cfg.n_codebooks * d.T;
  CK(cudaMemcpyAsync(ws->z_in.p, d.z, nz * 8, cudaMemcpyDeviceToDevice, st));
  if (d.mask) CK(cudaMemcpyAsync(ws->mask_in.p, d.mask, nz * 4, cudaMemcpyDeviceToDevice, st));
  const int64_t* gz = ws->z_in.as<int64_t>();
  const int32_t* gmask = d.mask ? ws->mask_in.as<int32_t>() : nullptr;
  int64_t* gout = ws->z_out.as<int64_t>();
  auto it = ws->graphs.find(v);
  if (it == ws->graphs.end()) {
    cudaStream_t cap;
    CK(cudaStreamCreateWithFlags(&cap, cudaStreamNonBlocking));
    cudaGraph_t graph = nullptr;
    cudaError_t e = cudaStreamBeginCapture(cap, cudaStreamCaptureModeThreadLocal);
    if (e != cudaSuccess) { cudaStreamDestroy(cap); return fail("begin capture: %s", cudaGetErrorString(e)); }
    const unsigned long long before = g_launches;
    int rc = enqueue_generate(m, ws, gz, gmask, gout, v, cap);
    const unsigned long long in_graph = g_launches - before;
    g_launches = before;
    e = cudaStreamEndCapture(cap, &graph);
    cudaStreamDestroy(cap);
    if (rc) { if (graph) cudaGraphDestroy(graph); return 1; }
    if (e != cudaSuccess) return fail("end capture: %s", cudaGetErrorString(e));
    cudaGraphExec_t exec = nullptr;
    e = cudaGraphInstantiate(&exec, graph, 0);
    cudaGraphDestroy(graph);
    if (e != cudaSuccess) return fail("graph instantiate: %s", cudaGetErrorString(e));
    if (ws->graphs.size() >= 16) {  // bound the cache
      for (auto& kv : ws->graphs) cudaGraphExecDestroy(kv.second);
      ws->graphs.clear();
      ws->graph_kernels.clear();
    }
    it = ws->graphs.emplace(v, exec).first;
    ++g_captures;
    ws->graph_kernels[v] = in_graph;
  }
  CK(cudaGraphLaunch(it->second, st));
  g_launches += ws->graph_kernels[v];
  CK(cudaMemcpyAsync(d.out, ws->z_out.p, nz * 8, cudaMemcpyDeviceToDevice, st));
  return 0;
}

extern "C" {

// One call is the one-group launch.
int32_t vnb_generate(vnb_model* m, const int64_t* z, const int32_t* mask, int32_t B, int32_t T,
                     const vnb_gen_params* p, int64_t* out, void* stream) {
  if (!p) return fail("vnb_generate: the parameters are required");
  vnb_gen_group g;
  g.rows = B; g.temperature = p->temperature; g.temp_eff = p->temp_eff; g.do_sample = p->do_sample;
  g.seed_lo = p->seed_lo; g.seed_hi = p->seed_hi; g.top_p = p->top_p;
  return generate(m, GenDesc{"vnb_generate", z, mask, B, T, &g, 1, p->use_graph, out, p->sampling_steps, p->gamma},
                  stream);
}

int32_t vnb_generate_many(vnb_model* m, const int64_t* z, const int32_t* mask, int32_t B, int32_t T, int32_t steps,
                          const float* gamma, const vnb_gen_group* groups, int32_t n_groups, int32_t use_graph,
                          int64_t* out, void* stream) {
  return generate(m, GenDesc{"vnb_generate_many", z, mask, B, T, groups, n_groups, use_graph, out, steps, gamma},
                  stream);
}

int32_t vnb_generate_many_adapted(vnb_model* m, const int64_t* z, const int32_t* mask, int32_t B, int32_t T,
                                  int32_t steps, const float* gamma, const vnb_gen_group* groups, int32_t n_groups,
                                  const int32_t* group_adapter, int32_t use_graph, int64_t* out, void* stream) {
  GenDesc d{"vnb_generate_many_adapted", z, mask, B, T, groups, n_groups, use_graph, out, steps, gamma};
  d.group_adapter = group_adapter;
  return generate(m, d, stream);
}

int32_t vnb_generate_ragged(vnb_model* m, const int64_t* z, const int32_t* mask, int32_t B, int32_t T, int32_t steps,
                            const float* gamma, const vnb_gen_group* groups, int32_t n_groups,
                            const int32_t* group_frames, const int32_t* group_adapter, int32_t use_graph, int64_t* out,
                            void* stream) {
  GenDesc d{"vnb_generate_ragged", z, mask, B, T, groups, n_groups, use_graph, out, steps, gamma};
  d.group_frames = group_frames; d.group_adapter = group_adapter;
  return generate(m, d, stream);
}

int32_t vnb_generate_steps(vnb_model* m, const int64_t* z, const int32_t* mask, int32_t B, int32_t T,
                           const int32_t* group_steps, const float* const* group_gamma, const vnb_gen_group* groups,
                           int32_t n_groups, const int32_t* group_frames, const int32_t* group_adapter,
                           int32_t use_graph, int64_t* out, void* stream) {
  GenDesc d{"vnb_generate_steps", z, mask, B, T, groups, n_groups, use_graph, out};
  d.per_group = true; d.group_steps = group_steps; d.group_gamma = group_gamma;
  d.group_frames = group_frames; d.group_adapter = group_adapter;
  return generate(m, d, stream);
}

int32_t vnb_generate_mixed_top_p(vnb_model* m, const int64_t* z, const int32_t* mask, int32_t B, int32_t T,
                                 const int32_t* group_steps, const float* const* group_gamma,
                                 const vnb_gen_group* groups, int32_t n_groups, const int32_t* group_frames,
                                 const int32_t* group_adapter, int32_t use_graph, int64_t* out, void* stream) {
  GenDesc d{"vnb_generate_mixed_top_p", z, mask, B, T, groups, n_groups, use_graph, out};
  d.per_group = true; d.group_steps = group_steps; d.group_gamma = group_gamma;
  d.group_frames = group_frames; d.group_adapter = group_adapter;
  d.mixed_top_p = true;
  return generate(m, d, stream);
}

uint64_t vnb_launch_count(void) { return g_launches; }
uint64_t vnb_graph_capture_count(void) { return g_captures; }

int32_t vnb_set_option(const char* name, int32_t value) {
  if (!name) return fail("null option name");
  if (strcmp(name, "gemm_pair") == 0) {
    set_gemm_pair(value);
    return 0;
  }
  if (strcmp(name, "fused_sampler") == 0) {
    g_fused_sampler = value ? 1 : 0;
    return 0;
  }
  return fail("unknown option '%s'", name);
}
int32_t vnb_get_option(const char* name, int32_t* value) {
  if (!name || !value) return fail("null argument");
  if (strcmp(name, "gemm_pair") == 0) {
    *value = get_gemm_pair();
    return 0;
  }
  if (strcmp(name, "fused_sampler") == 0) {
    *value = fused_sampler_enabled();
    return 0;
  }
  if (strcmp(name, "gemm_pair_max_clusters") == 0) {  // read-only: co-resident CTA pairs on the current device
    *value = get_gemm_max_clusters();
    return 0;
  }
  return fail("unknown option '%s'", name);
}

int32_t vnb_profile_begin(vnb_model* m) {
  m->prof.used = 0;
  m->prof.on = true;
  return 0;
}
int32_t vnb_profile_end(vnb_model* m, float* ms_per_family, int32_t* launches_per_family, int32_t n_families) {
  m->prof.on = false;
  for (int i = 0; i < n_families; ++i) { ms_per_family[i] = 0.f; launches_per_family[i] = 0; }
  if (m->prof.used < 2) return 0;
  CK(cudaEventSynchronize(m->prof.pool[m->prof.used - 1]));
  for (size_t i = 0; i + 1 < m->prof.used; ++i) {
    const int f = m->prof.fam[i];
    if (f < 0 || f >= n_families) continue;
    float ms = 0.f;
    CK(cudaEventElapsedTime(&ms, m->prof.pool[i], m->prof.pool[i + 1]));
    ms_per_family[f] += ms;
    launches_per_family[f] += 1;
  }
  return 0;
}

int32_t vnb_sample_step(const float* logits, int32_t* zflat, int32_t* tokens_out, float* conf_out, const int32_t* n0,
                        int32_t B, int32_t S, int32_t V, int32_t mask_token, int32_t step, int32_t is_last,
                        int32_t do_sample, float temperature, float gamma, float temp_eff, uint32_t seed_lo,
                        uint32_t seed_hi, void* stream) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  vnb_sample_group q = {};
  q.temperature = temperature; q.gamma = gamma; q.temp_eff = temp_eff; q.do_sample = do_sample; q.is_last = is_last;
  q.step = step; q.seed_lo = seed_lo; q.seed_hi = seed_hi;
  const SampleDyn* dd = nullptr;
  const RowGroup* rg = nullptr;
  if (stage_sample_dyn(sample_dyn(q), st, &dd) || one_group_rows(B, &rg)) return 1;
  SampleArgs sa;
  sa.logits = logits; sa.zcur = zflat; sa.zorig = nullptr; sa.tokens = tokens_out; sa.conf = conf_out; sa.n0 = n0;
  sa.rowgrp = rg;
  sa.B = B; sa.T = S; sa.C = 1; sa.ncc = 0; sa.V = V; sa.mask_token = mask_token;
  CK(launch_sample_step_dev(sa, dd, st, false));
  return 0;
}

// ------------------------------------------------------------------------------- unit-level ops
// vnb_dbg_set_live: the live bound the unit-level entry points below give their kernels (device, null = none)
static thread_local const int32_t* g_dbg_live = nullptr;
int32_t vnb_dbg_set_live(const int32_t* live) {
  g_dbg_live = live;
  return 0;
}
}  // extern "C"

// The plan of a unit-level GEMM entry point: built by make_gemm_plan as get_workspace() builds the forward's, so the
// tests reach every epilogue branch the forward launches, and bounded by vnb_dbg_set_live.  Refuses what no forward
// plan is: fused-norm operands and QKV shapes the epilogues cannot take.
static int unit_gemm_plan(GemmPlan* p, const char* who, int epi, const void* A, const void* W, int M, int N, int K,
                          void* out, void* out2, const float* bias, int T, int Tpad, const float* ss_in, int ss_parts,
                          float inv_d, float eps, void* out_bf16, float* ss_out) {
  if ((out_bf16 != nullptr || ss_out != nullptr) && epi != VNB_EPI_RESID && epi != VNB_EPI_BIAS_F32)
    return fail("%s: out_bf16 / ss_out need the RESID or BIAS_F32 epilogue", who);
  if ((out_bf16 == nullptr) != (ss_out == nullptr)) return fail("%s: out_bf16 and ss_out go together", who);
  if (ss_in != nullptr && ss_parts < 1) return fail("%s: ss_parts must be >= 1", who);
  if (epi == VNB_EPI_QKV && (out2 == nullptr || N % 96 != 0 || T < 1 || Tpad < T))
    return fail("%s: QKV needs vT, N a multiple of 96 and 1 <= T <= Tpad", who);
  if (!make_gemm_plan(p, epi, A, W, M, N, K, out, out2, bias, T, Tpad, ss_in, ss_parts, inv_d, eps, out_bf16, ss_out))
    return fail("gemm plan: %s", tmap_error());
  p->args.live = g_dbg_live;
  return 0;
}

// vnb_dbg_gemm_adapted, and (frames non-null) the adapted QKV of vnb_dbg_gemm_qkv_frames
static int dbg_gemm_adapted(const char* who, int32_t epi, const void* A, const void* W, int32_t M, int32_t N, int32_t K,
                            void* out, void* out2, int32_t T, int32_t Tpad, const float* ss_in, int32_t ss_parts,
                            float inv_d, float eps, void* out_bf16, float* ss_out, const vnb_adapter_weights* adapters,
                            int32_t n_adapters, int32_t layer, const int32_t* row_adapter, float* u,
                            const int32_t* frames, void* stream) {
  if (epi != VNB_EPI_QKV && epi != VNB_EPI_RESID && epi != VNB_EPI_GEGLU)
    return fail("%s: epilogue %d has no adapted variant", who, epi);
  if (!adapters || n_adapters < 1 || n_adapters > VNB_MAX_ADAPTERS || !row_adapter || !u || layer < 0)
    return fail("%s: need 1..%d adapters, a row map, u and layer >= 0", who, VNB_MAX_ADAPTERS);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  std::vector<AdapterDev> tab(VNB_MAX_ADAPTERS);
  for (int i = 0; i < n_adapters; ++i) tab[i] = adapter_dev(adapters[i]);
  std::vector<RowGroup> rowgrp(M);
  for (int i = 0; i < M; ++i) rowgrp[i] = RowGroup{i, i};  // row m is its own group: grp_adapter = row_adapter
  GemmPlan p;
  if (unit_gemm_plan(&p, who, epi, A, W, M, N, K, out, out2, nullptr, T, Tpad, ss_in, ss_parts, inv_d, eps, out_bf16,
                     ss_out))
    return 1;
  DevBuf tab_dev, grp_dev;
  CK(tab_dev.alloc(sizeof(AdapterDev) * VNB_MAX_ADAPTERS));
  CK(grp_dev.alloc(sizeof(RowGroup) * M));
  CK(cudaMemcpyAsync(tab_dev.p, tab.data(), sizeof(AdapterDev) * VNB_MAX_ADAPTERS, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(grp_dev.p, rowgrp.data(), sizeof(RowGroup) * M, cudaMemcpyHostToDevice, st));
  AdapterRefs& r = p.args.lora;
  r.table = tab_dev.as<AdapterDev>();
  r.grp_adapter = row_adapter;
  r.rowgrp = grp_dev.as<RowGroup>();
  r.rows_per_grp = 1;
  r.slot = epi == VNB_EPI_QKV ? LORA_QKV : epi == VNB_EPI_GEGLU ? LORA_W1 : (K == N ? LORA_WO : LORA_W2);
  r.layer = layer;
  r.u = u;
  p.args.frames = frames;
  CK(launch_lora_down(A, M, K, r, p.args.live, T, st));
  CK(launch_gemm(p, st));
  CK(cudaStreamSynchronize(st));  // the staged table and row map are freed on return
  return 0;
}

// The [group] table of one step's sampling scalars and the row -> group map of B batch rows, built as generate()
// builds them and staged into dyn_dev / grp_dev (stream-ordered).
static int stage_sample_groups(const vnb_sample_group* groups, int32_t n_groups, int32_t B, DevBuf& dyn_dev,
                               DevBuf& grp_dev, cudaStream_t st, const char* who) {
  if (check_groups(groups, n_groups, B, who)) return 1;
  std::vector<SampleDyn> dyn(n_groups);
  for (int g = 0; g < n_groups; ++g) dyn[g] = sample_dyn(groups[g]);
  const std::vector<RowGroup> rowgrp = row_groups(groups, n_groups, B);
  CK(dyn_dev.alloc(sizeof(SampleDyn) * n_groups));
  CK(grp_dev.alloc(sizeof(RowGroup) * B));
  CK(cudaMemcpyAsync(dyn_dev.p, dyn.data(), sizeof(SampleDyn) * n_groups, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(grp_dev.p, rowgrp.data(), sizeof(RowGroup) * B, cudaMemcpyHostToDevice, st));
  return 0;
}

extern "C" {

int32_t vnb_op_gemm(int32_t epi, const void* A, const void* W, int32_t M, int32_t N, int32_t K, void* out, void* out2,
                    const float* bias, int32_t T, int32_t Tpad, void* stream) {
  GemmPlan p;
  if (unit_gemm_plan(&p, "vnb_op_gemm", epi, A, W, M, N, K, out, out2, bias, T, Tpad, nullptr, 0, 0.f, 0.f, nullptr,
                     nullptr))
    return 1;
  CK(launch_gemm(p, reinterpret_cast<cudaStream_t>(stream)));
  return 0;
}
int32_t vnb_op_attention(const void* qk, const void* vT, void* out, const float* rel_bias, int32_t rel_sat, int32_t B,
                         int32_t T, int32_t Tpad, int32_t H, void* stream) {
  if (T < 1 || Tpad < T) return fail("vnb_op_attention: need 1 <= T <= Tpad");
  AttnPlan p;
  if (!make_attn_plan(&p, qk, vT, out, rel_bias, rel_sat, B, T, Tpad, H)) return fail("attn plan: %s", tmap_error());
  p.live = g_dbg_live;
  CK(launch_attention(p, reinterpret_cast<cudaStream_t>(stream)));
  return 0;
}
int32_t vnb_dbg_attention_ragged(const void* qk, const void* vT, void* out, const float* rel_bias, int32_t rel_sat,
                                 int32_t B, int32_t T, int32_t Tpad, int32_t H, const int32_t* frames, void* stream) {
  if (!frames) return fail("vnb_dbg_attention_ragged: frames is required");
  if (T < 1 || Tpad < T) return fail("vnb_dbg_attention_ragged: need 1 <= T <= Tpad");
  AttnPlan p;
  if (!make_attn_plan(&p, qk, vT, out, rel_bias, rel_sat, B, T, Tpad, H)) return fail("attn plan: %s", tmap_error());
  p.frames = frames;
  p.live = g_dbg_live;
  CK(launch_attention(p, reinterpret_cast<cudaStream_t>(stream)));
  return 0;
}
int32_t vnb_dbg_gemm_ref(const void* A, const void* W, int32_t M, int32_t N, int32_t K, float* out, void* stream) {
  CK(launch_gemm_ref(A, W, M, N, K, out, reinterpret_cast<cudaStream_t>(stream)));
  return 0;
}
int32_t vnb_dbg_gemm_fused(int32_t epi, const void* A, const void* W, int32_t M, int32_t N, int32_t K, void* out,
                           void* out2, const float* bias, int32_t T, int32_t Tpad, const float* ss_in,
                           int32_t ss_parts, float inv_d, float eps, void* out_bf16, float* ss_out, void* stream) {
  if (epi < VNB_EPI_BF16 || epi > VNB_EPI_BIAS_F32) return fail("vnb_dbg_gemm_fused: epilogue %d not supported", epi);
  if (epi == VNB_EPI_BIAS_F32 && bias == nullptr) return fail("vnb_dbg_gemm_fused: BIAS_F32 needs a bias");
  GemmPlan p;
  if (unit_gemm_plan(&p, "vnb_dbg_gemm_fused", epi, A, W, M, N, K, out, out2, bias, T, Tpad, ss_in, ss_parts, inv_d, eps,
                     out_bf16, ss_out))
    return 1;
  CK(launch_gemm(p, reinterpret_cast<cudaStream_t>(stream)));
  return 0;
}

int32_t vnb_dbg_gemm_adapted(int32_t epi, const void* A, const void* W, int32_t M, int32_t N, int32_t K, void* out,
                             void* out2, int32_t T, int32_t Tpad, const float* ss_in, int32_t ss_parts, float inv_d,
                             float eps, void* out_bf16, float* ss_out, const vnb_adapter_weights* adapters,
                             int32_t n_adapters, int32_t layer, const int32_t* row_adapter, float* u, void* stream) {
  return dbg_gemm_adapted("vnb_dbg_gemm_adapted", epi, A, W, M, N, K, out, out2, T, Tpad, ss_in, ss_parts, inv_d, eps,
                          out_bf16, ss_out, adapters, n_adapters, layer, row_adapter, u, nullptr, stream);
}
int32_t vnb_dbg_gemm_qkv_frames(const void* A, const void* W, int32_t M, int32_t N, int32_t K, void* out, void* vT,
                                int32_t T, int32_t Tpad, const float* ss_in, int32_t ss_parts, float inv_d, float eps,
                                const int32_t* frames, const vnb_adapter_weights* adapters, int32_t n_adapters,
                                int32_t layer, const int32_t* row_adapter, float* u, void* stream) {
  const char* who = "vnb_dbg_gemm_qkv_frames";
  if (!frames) return fail("%s: frames is required", who);
  if (adapters)
    return dbg_gemm_adapted(who, VNB_EPI_QKV, A, W, M, N, K, out, vT, T, Tpad, ss_in, ss_parts, inv_d, eps, nullptr,
                            nullptr, adapters, n_adapters, layer, row_adapter, u, frames, stream);
  GemmPlan p;
  if (unit_gemm_plan(&p, who, VNB_EPI_QKV, A, W, M, N, K, out, vT, nullptr, T, Tpad, ss_in, ss_parts, inv_d, eps,
                     nullptr, nullptr))
    return 1;
  p.args.frames = frames;
  CK(launch_gemm(p, reinterpret_cast<cudaStream_t>(stream)));
  return 0;
}
int32_t vnb_dbg_gemm_sample(const void* A, const void* W, const float* bias, int32_t M, int32_t N, int32_t K,
                            const float* ss_in, int32_t ss_parts, float inv_d, float eps, const int32_t* zcur,
                            int32_t T, int32_t C, int32_t ncc, int32_t V, int32_t mask_token, float temperature,
                            int32_t do_sample, int32_t step, uint32_t seed_lo, uint32_t seed_hi, void* partials,
                            void* stream) {
  const char* who = "vnb_dbg_gemm_sample";
  if (V % 128 != 0 || V > 1024 || ncc < 0 || C <= ncc || N != (C - ncc) * V || T < 1)
    return fail("%s: need V %% 128 == 0, V <= 1024, 0 <= ncc < C, N == (C - ncc) * V, T >= 1", who);
  if (!bias || !zcur || !partials) return fail("%s: bias, zcur and partials are required", who);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  vnb_sample_group q = {};
  q.temperature = temperature; q.do_sample = do_sample; q.step = step; q.seed_lo = seed_lo; q.seed_hi = seed_hi;
  GemmPlan p;
  if (unit_gemm_plan(&p, who, VNB_EPI_SAMPLE, A, W, M, N, K, nullptr, nullptr, bias, T, T, ss_in, ss_parts, inv_d, eps,
                     nullptr, nullptr))
    return 1;
  GemmArgs& a = p.args;
  a.zcur = zcur; a.partials = reinterpret_cast<float4*>(partials); a.C = C; a.ncc = ncc; a.V = V; a.mask_token = mask_token;
  if (stage_sample_dyn(sample_dyn(q), st, &a.dyn) || one_group_rows((M + T - 1) / T, &a.rowgrp)) return 1;
  CK(launch_gemm(p, st));
  return 0;
}
}  // extern "C"

// vnb_dbg_sample (paths 0..3) and vnb_dbg_sample_split (path 4: the split combine, the split nucleus draw, the re-mask)
static int dbg_sample(int32_t path, const float* logits, const void* partials, int32_t* zcur, const int32_t* zorig,
                      int32_t* tokens, float* conf, const int32_t* n0, int32_t B, int32_t T, int32_t C, int32_t ncc,
                      int32_t V, int32_t mask_token, const vnb_sample_group* groups, int32_t n_groups, void* stream,
                      const char* who) {
  if (B < 1 || T < 1 || ncc < 0 || C <= ncc) return fail("%s: need B >= 1, T >= 1 and 0 <= ncc < C", who);
  if (V % 128 != 0 || V < 128 || V > 1024) return fail("%s: need V %% 128 == 0, 128 <= V <= 1024 (got %d)", who, V);
  if (!zcur || !tokens || !conf || !n0 || !groups) return fail("%s: zcur, tokens, conf, n0 and groups are required", who);
  if ((path <= 1 || path == 4) && !logits) return fail("%s: path %d needs logits", who, path);
  if ((path == 2 || path == 4) && !partials) return fail("%s: path %d needs partials", who, path);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  DevBuf dyn_dev, grp_dev;
  if (stage_sample_groups(groups, n_groups, B, dyn_dev, grp_dev, st, who)) return 1;
  SampleArgs sa;
  sa.logits = logits; sa.zcur = zcur; sa.zorig = zorig; sa.tokens = tokens; sa.conf = conf; sa.n0 = n0;
  sa.rowgrp = grp_dev.as<RowGroup>();
  sa.B = B; sa.T = T; sa.C = C; sa.ncc = ncc; sa.V = V; sa.mask_token = mask_token;
  sa.live = g_dbg_live;
  const SampleDyn* dd = dyn_dev.as<SampleDyn>();
  if (path <= 1) CK(launch_sample_step_dev(sa, dd, st, path == 1));
  else if (path == 2) CK(launch_sample_combine_dev(sa, partials, dd, st));
  else if (path == 3) CK(launch_remask_dev(sa, dd, st));
  else CK(launch_sample_split_dev(sa, partials, dd, st));
  CK(cudaStreamSynchronize(st));  // the staged table and row map are freed on return
  return 0;
}

extern "C" {

int32_t vnb_dbg_sample(int32_t path, const float* logits, const void* partials, int32_t* zcur, const int32_t* zorig,
                       int32_t* tokens, float* conf, const int32_t* n0, int32_t B, int32_t T, int32_t C, int32_t ncc,
                       int32_t V, int32_t mask_token, const vnb_sample_group* groups, int32_t n_groups, void* stream) {
  if (path < 0 || path > 3) return fail("vnb_dbg_sample: path %d outside 0..3", path);
  return dbg_sample(path, logits, partials, zcur, zorig, tokens, conf, n0, B, T, C, ncc, V, mask_token, groups,
                    n_groups, stream, "vnb_dbg_sample");
}

int32_t vnb_dbg_sample_split(const float* logits, const void* partials, int32_t* zcur, const int32_t* zorig,
                             int32_t* tokens, float* conf, const int32_t* n0, int32_t B, int32_t T, int32_t C,
                             int32_t ncc, int32_t V, int32_t mask_token, const vnb_sample_group* groups,
                             int32_t n_groups, void* stream) {
  return dbg_sample(4, logits, partials, zcur, zorig, tokens, conf, n0, B, T, C, ncc, V, mask_token, groups, n_groups,
                    stream, "vnb_dbg_sample_split");
}

int32_t vnb_dbg_gemm_sample_split(const void* A, const void* W, const float* bias, int32_t M, int32_t N, int32_t K,
                                  const float* ss_in, int32_t ss_parts, float inv_d, float eps, const int32_t* zcur,
                                  int32_t T, int32_t C, int32_t ncc, int32_t V, int32_t mask_token,
                                  const vnb_sample_group* groups, int32_t n_groups, void* partials, float* logits,
                                  void* stream) {
  const char* who = "vnb_dbg_gemm_sample_split";
  if (V % 128 != 0 || V > 1024 || ncc < 0 || C <= ncc || N != (C - ncc) * V || T < 1 || M % T != 0)
    return fail("%s: need V %% 128 == 0, V <= 1024, 0 <= ncc < C, N == (C - ncc) * V, T >= 1 and M a multiple of T", who);
  if (!bias || !zcur || !partials || !logits || !groups)
    return fail("%s: bias, zcur, partials, logits and groups are required", who);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  GemmPlan p;
  if (unit_gemm_plan(&p, who, VNB_EPI_SAMPLE, A, W, M, N, K, logits, nullptr, bias, T, T, ss_in, ss_parts, inv_d, eps,
                     nullptr, nullptr))
    return 1;
  DevBuf dyn_dev, grp_dev;
  if (stage_sample_groups(groups, n_groups, M / T, dyn_dev, grp_dev, st, who)) return 1;
  GemmArgs& a = p.args;
  a.zcur = zcur; a.partials = reinterpret_cast<float4*>(partials); a.C = C; a.ncc = ncc; a.V = V; a.mask_token = mask_token;
  a.dyn = dyn_dev.as<SampleDyn>();
  a.rowgrp = grp_dev.as<RowGroup>();
  p.sample_split = true;
  CK(launch_gemm(p, st));
  CK(cudaStreamSynchronize(st));  // the staged table and row map are freed on return
  return 0;
}

// the refusal of a caller's workspace that is too small for the call
static int32_t check_workspace(const char* fn, uint64_t have, uint64_t need) {
  if (have < need)
    return fail("%s: workspace of %llu bytes, %llu needed", fn, (unsigned long long)have, (unsigned long long)need);
  return 0;
}

// ---- onset detection (onset.cu) ----
int32_t vnb_onset_workspace_bytes(int32_t B, int32_t N, int32_t hop, uint64_t* bytes) {
  if (B < 1 || N < 1 || hop < 1 || !bytes) return fail("vnb_onset_workspace_bytes: need B >= 1, N >= 1, hop >= 1 and bytes");
  *bytes = onset_workspace_bytes(B, 1 + N / hop);
  return 0;
}
int32_t vnb_onset_detect(const float* samples, int32_t B, int32_t N, int32_t sr, int32_t hop, int32_t backtrack,
                         void* workspace, uint64_t workspace_bytes, float* envelope, int32_t* onsets, int32_t* counts,
                         void* stream) {
  if (B < 1 || B > 65535 || N < 1) return fail("vnb_onset_detect: need 1 <= B <= 65535 and N >= 1 (got B = %d, N = %d)", B, N);
  if (sr < 1 || hop < 1) return fail("vnb_onset_detect: need sr >= 1 and hop >= 1 (got sr = %d, hop = %d)", sr, hop);
  if (!samples || !workspace || !envelope || !onsets || !counts)
    return fail("vnb_onset_detect: samples, workspace, envelope, onsets and counts are required");
  if (int32_t rc = check_workspace("vnb_onset_detect", workspace_bytes, onset_workspace_bytes(B, 1 + N / hop)))
    return rc;
  OnsetTables t;
  CK(onset_tables(sr, hop, &t));
  CK(launch_onset_detect(samples, B, N, hop, t, reinterpret_cast<float*>(workspace), envelope, onsets, counts,
                         backtrack != 0, reinterpret_cast<cudaStream_t>(stream)));
  return 0;
}
int32_t vnb_onset_mask(const int32_t* onsets, const int32_t* counts, int32_t onset_rows, int32_t F, int32_t width,
                       int64_t* mask, int32_t B, int32_t C, int32_t T, void* stream) {
  if (B < 1 || C < 1 || T < 1 || F < 1) return fail("vnb_onset_mask: need B, C, T and F >= 1");
  if (onset_rows != 1 && onset_rows != B) return fail("vnb_onset_mask: onset_rows must be 1 or B (got %d, B = %d)", onset_rows, B);
  if (!onsets || !counts || !mask) return fail("vnb_onset_mask: onsets, counts and mask are required");
  CK(launch_onset_mask(onsets, counts, onset_rows, F, width, mask, B, C, T, reinterpret_cast<cudaStream_t>(stream)));
  return 0;
}

// ---- beat tracking (beat.cu) ----
int32_t vnb_beat_workspace_bytes(int32_t B, int32_t N, int32_t hop, uint64_t* bytes) {
  if (B < 1 || N < 1 || hop < 1 || !bytes) return fail("vnb_beat_workspace_bytes: need B >= 1, N >= 1, hop >= 1 and bytes");
  *bytes = beat_workspace_bytes(B, 1 + N / hop);
  return 0;
}
static int32_t beat_args(const char* fn, int32_t B, int32_t F, int32_t sr, int32_t hop, double start_bpm,
                         double tightness, const void* in, const void* workspace, uint64_t workspace_bytes,
                         const void* tempo, const void* beats, const void* counts, BeatTables* t) {
  if (B < 1 || B > 65535) return fail("%s: need 1 <= B <= 65535 (got %d)", fn, B);
  if (sr < 1 || hop < 1) return fail("%s: need sr >= 1 and hop >= 1 (got sr = %d, hop = %d)", fn, sr, hop);
  if (!(start_bpm > 0) || !(tightness > 0)) return fail("%s: start_bpm and tightness must be > 0", fn);
  if (!in || !workspace || !tempo || !beats || !counts) return fail("%s: a required buffer is NULL", fn);
  const int W = beat_lags(sr, hop);
  if (W < 2 || W > BEAT_MAX_LAGS)
    return fail("%s: the 8 s tempo window is int(8 sr) // hop = %d frames; 2..%d are supported", fn, W, BEAT_MAX_LAGS);
  if (int32_t rc = check_workspace(fn, workspace_bytes, beat_workspace_bytes(B, F))) return rc;
  CK(beat_tables(sr, hop, t));
  return 0;
}
int32_t vnb_beat_track(const float* samples, int32_t B, int32_t N, int32_t sr, int32_t hop, double start_bpm,
                       double tightness, int32_t trim, void* workspace, uint64_t workspace_bytes, float* envelope,
                       double* tempo, int32_t* beats, int32_t* counts, void* stream) {
  if (N < 1) return fail("vnb_beat_track: need N >= 1 (got %d)", N);
  BeatTables bt;
  if (int32_t rc = beat_args("vnb_beat_track", B, hop >= 1 ? 1 + N / hop : 1, sr, hop, start_bpm, tightness, samples,
                             envelope ? workspace : nullptr, workspace_bytes, tempo, beats, counts, &bt))
    return rc;
  OnsetTables ot;
  CK(onset_tables(sr, hop, &ot));
  CK(launch_beat_track(samples, B, N, sr, hop, ot, bt, start_bpm, tightness, trim != 0, workspace, envelope, tempo,
                       beats, counts, reinterpret_cast<cudaStream_t>(stream)));
  return 0;
}
int32_t vnb_dbg_beat_from_envelope(const float* envelope, int32_t B, int32_t F, int32_t sr, int32_t hop,
                                   double start_bpm, double tightness, int32_t trim, void* workspace,
                                   uint64_t workspace_bytes, double* tempo, int32_t* beats, int32_t* counts,
                                   void* stream) {
  if (F < 1) return fail("vnb_dbg_beat_from_envelope: need F >= 1 (got %d)", F);
  BeatTables bt;
  if (int32_t rc = beat_args("vnb_dbg_beat_from_envelope", B, F, sr, hop, start_bpm, tightness, envelope, workspace,
                             workspace_bytes, tempo, beats, counts, &bt))
    return rc;
  CK(launch_beat_from_envelope(envelope, B, F, sr, hop, bt, start_bpm, tightness, trim != 0, workspace, tempo, beats,
                               counts, reinterpret_cast<cudaStream_t>(stream)));
  return 0;
}

// ---- pitch shift (pitch.cu) ----
static int32_t pitch_args(const char* fn, int32_t rows, int32_t N, int32_t sr, int32_t new_freq, int32_t n_fft,
                          int32_t hop, double rate, PitchPlan* p) {
  if (rows < 1 || rows > 65535) return fail("%s: need 1 <= rows <= 65535 (got %d)", fn, rows);
  if (n_fft < PITCH_MIN_NFFT || n_fft > PITCH_MAX_NFFT)
    return fail("%s: n_fft = %d; %d..%d are supported", fn, n_fft, PITCH_MIN_NFFT, PITCH_MAX_NFFT);
  if (hop < 1 || hop > n_fft) return fail("%s: need 1 <= hop <= n_fft (got hop = %d, n_fft = %d)", fn, hop, n_fft);
  if (N <= n_fft / 2) return fail("%s: need N > n_fft // 2 for the reflect padding (got N = %d, n_fft = %d)", fn, N, n_fft);
  if (sr < 1 || new_freq < 1) return fail("%s: need sample_rate >= 1 and new_freq >= 1 (got %d, %d)", fn, sr, new_freq);
  if (!(rate > 0) || !std::isfinite(rate)) return fail("%s: need a finite rate > 0 (got %g)", fn, rate);
  const int rc = pitch_plan(rows, N, sr, new_freq, n_fft, hop, rate, p);
  if (rc == 1)
    return fail("%s: ceil(F / rate) stretched frames is out of range (N = %d, hop = %d, rate = %g)", fn, N, hop, rate);
  if (rc)
    return fail("%s: one stretched frame of even n_fft = %d leaves an empty istft signal (N = %d, hop = %d, rate = %g)",
                fn, n_fft, N, hop, rate);
  return 0;
}
int32_t vnb_pitch_workspace_bytes(int32_t rows, int32_t N, int32_t sr, int32_t new_freq, int32_t n_fft, int32_t hop,
                                  double rate, uint64_t* bytes) {
  if (!bytes) return fail("vnb_pitch_workspace_bytes: bytes is NULL");
  PitchPlan p;
  if (int32_t rc = pitch_args("vnb_pitch_workspace_bytes", rows, N, sr, new_freq, n_fft, hop, rate, &p)) return rc;
  *bytes = pitch_workspace_bytes(p);
  return 0;
}
int32_t vnb_pitch_shift(const float* samples, int32_t rows, int32_t N, int32_t sr, int32_t new_freq, int32_t n_fft,
                        int32_t hop, double rate, void* workspace, uint64_t workspace_bytes, float* out, void* stream) {
  if (!samples || !workspace || !out) return fail("vnb_pitch_shift: samples, workspace and out are required");
  PitchPlan p;
  if (int32_t rc = pitch_args("vnb_pitch_shift", rows, N, sr, new_freq, n_fft, hop, rate, &p)) return rc;
  if (int32_t rc = check_workspace("vnb_pitch_shift", workspace_bytes, pitch_workspace_bytes(p))) return rc;
  const double *fwd = nullptr, *inv = nullptr;
  CK(pitch_basis(n_fft, &fwd, &inv));
  CK(launch_pitch_shift(samples, p, fwd, inv, workspace, out, reinterpret_cast<cudaStream_t>(stream)));
  return 0;
}
int32_t vnb_dbg_pitch_layout(int32_t rows, int32_t N, int32_t sr, int32_t new_freq, int32_t n_fft, int32_t hop,
                             double rate, int64_t* offsets, int64_t* dims) {
  if (!offsets || !dims) return fail("vnb_dbg_pitch_layout: offsets and dims are required");
  PitchPlan p;
  if (int32_t rc = pitch_args("vnb_dbg_pitch_layout", rows, N, sr, new_freq, n_fft, hop, rate, &p)) return rc;
  const PitchLayout l = pitch_layout(p);
  offsets[0] = (int64_t)l.spec;
  offsets[1] = p.stretch ? (int64_t)l.stretched : -1;
  offsets[2] = (int64_t)l.frames;
  offsets[3] = (int64_t)l.y;
  dims[0] = p.F; dims[1] = p.F2; dims[2] = p.L; dims[3] = p.target;
  return 0;
}
int32_t vnb_dbg_pitch_time_steps(double rate, int32_t n, float* out, void* stream) {
  if (!out || n < 1 || !(rate > 0)) return fail("vnb_dbg_pitch_time_steps: need out, n >= 1 and rate > 0");
  CK(launch_pitch_time_steps((float)rate, n, out, reinterpret_cast<cudaStream_t>(stream)));
  return 0;
}

// ---- validation metrics (validate.cu) ----
static int32_t xent_args(const char* fn, const float* logits, int32_t B, int32_t C, int32_t T, int32_t ncc, int32_t V) {
  if (B < 1 || C < 1 || T < 1) return fail("%s: need B, C, T >= 1 (got %d, %d, %d)", fn, B, C, T);
  if (ncc < 0 || ncc >= C) return fail("%s: need 0 <= ncc < C (got ncc = %d, C = %d)", fn, ncc, C);
  if (V < 1 || V > XENT_MAX_V || V % 4)
    return fail("%s: V = %d; a multiple of 4 in 1..%d is supported", fn, V, XENT_MAX_V);
  if (reinterpret_cast<uintptr_t>(logits) % 16) return fail("%s: logits must be 16-byte aligned", fn);
  return 0;
}
int32_t vnb_xent_metrics_workspace_bytes(int32_t B, int64_t S, uint64_t* bytes) {
  if (!bytes) return fail("vnb_xent_metrics_workspace_bytes: bytes is NULL");
  if (B < 1 || S < 1) return fail("vnb_xent_metrics_workspace_bytes: need B, S >= 1 (got %d, %lld)", B, (long long)S);
  *bytes = xent_workspace_bytes(B, S);
  return 0;
}
int32_t vnb_xent_metrics(const float* logits, const int64_t* z, const int64_t* mask, const double* r, int32_t B,
                         int32_t C, int32_t T, int32_t ncc, int32_t V, double label_smoothing, void* workspace,
                         uint64_t workspace_bytes, float* out9, int32_t* ambiguous, void* stream) {
  if (!logits || !z || !mask || !r || !workspace || !out9)
    return fail("vnb_xent_metrics: logits, z, mask, r, workspace and out9 are required");
  if (int32_t rc = xent_args("vnb_xent_metrics", logits, B, C, T, ncc, V)) return rc;
  if (!(label_smoothing >= 0.0 && label_smoothing <= 1.0))
    return fail("vnb_xent_metrics: need 0 <= label_smoothing <= 1 (got %g)", label_smoothing);
  const uint64_t need = xent_workspace_bytes(B, (long long)T * (C - ncc));
  if (int32_t rc = check_workspace("vnb_xent_metrics", workspace_bytes, need)) return rc;
  CK(launch_xent_metrics(logits, z, mask, r, B, C, T, ncc, V, label_smoothing, workspace, out9, ambiguous,
                         reinterpret_cast<cudaStream_t>(stream)));
  return 0;
}
int32_t vnb_dbg_xent_rows(const float* logits, const int64_t* z, int32_t B, int32_t C, int32_t T, int32_t ncc,
                          int32_t V, vnb_xent_row* rows, void* stream) {
  if (!logits || !z || !rows) return fail("vnb_dbg_xent_rows: logits, z and rows are required");
  if (int32_t rc = xent_args("vnb_dbg_xent_rows", logits, B, C, T, ncc, V)) return rc;
  CK(launch_xent_rows(logits, z, B, C, T, ncc, V, rows, reinterpret_cast<cudaStream_t>(stream)));
  return 0;
}

// ---- mel spectrogram and multi-scale mel distance (mel.cu) ----
static int32_t mel_scale_args(const char* fn, int32_t N, int32_t sr, const vnb_mel_scale& s) {
  if (sr < 1) return fail("%s: need sr >= 1 (got %d)", fn, sr);
  if (s.n_fft < MEL_MIN_NFFT || s.n_fft > MEL_MAX_NFFT || (s.n_fft & (s.n_fft - 1)))
    return fail("%s: n_fft = %d; a power of two in %d..%d is supported", fn, s.n_fft, MEL_MIN_NFFT, MEL_MAX_NFFT);
  if (N <= s.n_fft / 2)
    return fail("%s: need N > n_fft // 2 for the reflect padding (got N = %d, n_fft = %d)", fn, N, s.n_fft);
  if (s.hop < 1) return fail("%s: need hop >= 1 (got %d)", fn, s.hop);
  if (s.n_mels < 1 || s.n_mels > MEL_MAX_MELS) return fail("%s: n_mels = %d; 1..%d are supported", fn, s.n_mels, MEL_MAX_MELS);
  if (!(s.fmin >= 0.0) || !(s.fmax > s.fmin) || !std::isfinite(s.fmax))
    return fail("%s: need 0 <= fmin < fmax, both finite (got fmin = %g, fmax = %g)", fn, s.fmin, s.fmax);
  return 0;
}
int32_t vnb_mel_spectrogram(const float* samples, int32_t rows, int32_t N, int32_t sr, const vnb_mel_scale* scale,
                            float* out, void* stream) {
  if (!samples || !scale || !out) return fail("vnb_mel_spectrogram: samples, scale and out are required");
  if (rows < 1 || rows > 65535) return fail("vnb_mel_spectrogram: need 1 <= rows <= 65535 (got %d)", rows);
  if (int32_t rc = mel_scale_args("vnb_mel_spectrogram", N, sr, *scale)) return rc;
  CK(launch_mel_spectrogram(samples, rows, N, sr, *scale, out, reinterpret_cast<cudaStream_t>(stream)));
  return 0;
}
static int32_t mel_loss_args(const char* fn, int32_t B, int32_t C, int32_t N, int32_t sr, const vnb_mel_scale* scales,
                             int32_t n_scales) {
  if (B < 1 || C < 1 || (int64_t)B * C > 65535)
    return fail("%s: need B, C >= 1 and B * C <= 65535 (got B = %d, C = %d)", fn, B, C);
  if (!scales) return fail("%s: scales is NULL", fn);
  if (n_scales < 1 || n_scales > MEL_MAX_SCALES) return fail("%s: n_scales = %d; 1..%d are supported", fn, n_scales, MEL_MAX_SCALES);
  for (int i = 0; i < n_scales; ++i)
    if (int32_t rc = mel_scale_args(fn, N, sr, scales[i])) return rc;
  return 0;
}
int32_t vnb_mel_workspace_bytes(int32_t B, int32_t C, int32_t N, int32_t sr, const vnb_mel_scale* scales,
                                int32_t n_scales, uint64_t* bytes) {
  if (!bytes) return fail("vnb_mel_workspace_bytes: bytes is NULL");
  if (int32_t rc = mel_loss_args("vnb_mel_workspace_bytes", B, C, N, sr, scales, n_scales)) return rc;
  *bytes = mel_loss_plan(B, C, N, sr, scales, n_scales).total;
  return 0;
}
int32_t vnb_mel_loss(const float* x, const float* y, int32_t B, int32_t C, int32_t N, int32_t sr,
                     const vnb_mel_scale* scales, int32_t n_scales, double clamp_eps, double pow, double log_weight,
                     double mag_weight, void* workspace, uint64_t workspace_bytes, float* loss, float* item_loss,
                     void* stream) {
  if (!x || !y || !workspace || !loss) return fail("vnb_mel_loss: x, y, workspace and loss are required");
  if (int32_t rc = mel_loss_args("vnb_mel_loss", B, C, N, sr, scales, n_scales)) return rc;
  if (!(clamp_eps > 0.0) || !std::isfinite(clamp_eps))
    return fail("vnb_mel_loss: need a finite clamp_eps > 0 (got %g)", clamp_eps);
  if (!std::isfinite(pow) || !std::isfinite(log_weight) || !std::isfinite(mag_weight))
    return fail("vnb_mel_loss: pow, log_weight and mag_weight must be finite");
  const MelLossPlan p = mel_loss_plan(B, C, N, sr, scales, n_scales);
  if (int32_t rc = check_workspace("vnb_mel_loss", workspace_bytes, p.total)) return rc;
  CK(launch_mel_loss(x, y, p, clamp_eps, pow, log_weight, mag_weight, workspace, loss, item_loss,
                     reinterpret_cast<cudaStream_t>(stream)));
  return 0;
}

// ---- Frechet audio distance with VGGish embeddings (fad.cu) ----
int32_t vnb_vggish_create(const vnb_vggish_weights* w, void** handle) {
  if (!w || !handle) return fail("vnb_vggish_create: weights and handle are required");
  std::vector<std::pair<const char*, const void*>> ptrs = {{"w1", w->w1}, {"b1", w->b1}};
  static const char* conv_names[5] = {"conv 0", "conv 1", "conv 2", "conv 3", "conv 4"};
  static const char* fc_names[3] = {"fc 0", "fc 1", "fc 2"};
  for (int l = 0; l < 5; ++l) {
    ptrs.push_back({conv_names[l], w->conv_hi[l]}); ptrs.push_back({conv_names[l], w->conv_lo[l]});
    ptrs.push_back({conv_names[l], w->conv_b[l]});
  }
  for (int l = 0; l < 3; ++l) {
    ptrs.push_back({fc_names[l], w->fc_hi[l]}); ptrs.push_back({fc_names[l], w->fc_lo[l]});
    ptrs.push_back({fc_names[l], w->fc_b[l]});
  }
  for (const auto& p : ptrs) {
    if (!p.second) return fail("vnb_vggish_create: %s: a weight pointer is NULL", p.first);
    if (reinterpret_cast<uintptr_t>(p.second) % 16) return fail("vnb_vggish_create: %s: a weight pointer is not 16-byte aligned", p.first);
  }
  VggishNet* net = new VggishNet;
  net->w1 = w->w1; net->b1 = w->b1;
  for (int l = 0; l < 5; ++l) { net->conv_hi[l] = w->conv_hi[l]; net->conv_lo[l] = w->conv_lo[l]; net->conv_b[l] = w->conv_b[l]; }
  for (int l = 0; l < 3; ++l) { net->fc_hi[l] = w->fc_hi[l]; net->fc_lo[l] = w->fc_lo[l]; net->fc_b[l] = w->fc_b[l]; }
  *handle = net;
  return 0;
}
void vnb_vggish_destroy(void* handle) { delete static_cast<VggishNet*>(handle); }
int32_t vnb_vggish_frontend(const float* samples, int32_t rows, int32_t N, float* examples, void* stream) {
  if (!samples || !examples) return fail("vnb_vggish_frontend: samples and examples are required");
  if (rows < 1 || rows > 65535) return fail("vnb_vggish_frontend: need 1 <= rows <= 65535 (got %d)", rows);
  if (vggish_examples(N) < 1) return fail("vnb_vggish_frontend: N = %d samples at 16 kHz give no example (15600 needed)", N);
  CK(launch_vggish_frontend(samples, rows, N, examples, reinterpret_cast<cudaStream_t>(stream)));
  return 0;
}
int32_t vnb_vggish_workspace_bytes(int32_t n_ex, uint64_t* bytes) {
  if (!bytes) return fail("vnb_vggish_workspace_bytes: bytes is NULL");
  if (n_ex < 1 || n_ex > 65535) return fail("vnb_vggish_workspace_bytes: need 1 <= n_ex <= 65535 (got %d)", n_ex);
  *bytes = vggish_workspace_bytes(n_ex);
  return 0;
}
int32_t vnb_vggish_embed(void* handle, const float* examples, int32_t n_ex, void* workspace, uint64_t workspace_bytes,
                         float* embeddings, void* stream) {
  if (!handle || !examples || !workspace || !embeddings)
    return fail("vnb_vggish_embed: handle, examples, workspace and embeddings are required");
  if (n_ex < 1 || n_ex > 65535) return fail("vnb_vggish_embed: need 1 <= n_ex <= 65535 (got %d)", n_ex);
  if (int32_t rc = check_workspace("vnb_vggish_embed", workspace_bytes, vggish_workspace_bytes(n_ex))) return rc;
  const cudaError_t e = launch_vggish_embed(*static_cast<const VggishNet*>(handle), examples, n_ex, workspace,
                                            embeddings, reinterpret_cast<cudaStream_t>(stream));
  if (e == cudaErrorInvalidValue && tmap_error()[0]) return fail("vnb_vggish_embed: %s", tmap_error());
  CK(e);
  return 0;
}
int32_t vnb_fad_moments(const float* embeddings, int64_t M, double* mu, double* sigma, void* stream) {
  if (!embeddings || !mu || !sigma) return fail("vnb_fad_moments: embeddings, mu and sigma are required");
  if (M < 2) return fail("vnb_fad_moments: need M >= 2 embeddings (got %lld)", (long long)M);
  CK(launch_fad_moments(embeddings, M, mu, sigma, reinterpret_cast<cudaStream_t>(stream)));
  return 0;
}
int32_t vnb_dbg_vggish_layer(const float* x, const float* w, const void* a_hi, const void* a_lo, int32_t Bn, int32_t H,
                             int32_t W, int32_t Cin, const void* w_hi, const void* w_lo, int32_t N, const float* bias,
                             int32_t relu, int32_t pool, void* out_hi, void* out_lo, float* out_f32, void* stream) {
  const cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (Bn < 1 || Bn > 65535 || !bias) return fail("vnb_dbg_vggish_layer: need 1 <= Bn <= 65535 and a bias");
  if (W == 0 && Cin == 1) {
    if (!x || !w || !out_hi || !out_lo) return fail("vnb_dbg_vggish_layer: x, w, out_hi and out_lo are required");
    CK(launch_vggish_in(x, w, bias, Bn, out_hi, out_lo, st));
    return 0;
  }
  if (!a_hi || !a_lo || !w_hi || !w_lo) return fail("vnb_dbg_vggish_layer: a_hi, a_lo, w_hi and w_lo are required");
  if (N < 128 || N % 128 || Cin < 64 || Cin % 64) return fail("vnb_dbg_vggish_layer: need N % 128 == 0 and Cin % 64 == 0");
  if (W > 0) {
    if (W > 128 || 128 % W || (128 / W) % 2 || H < 2 || H % 2 || (H * W > 128 && (H * W) % 128) || !out_hi || !out_lo)
      return fail("vnb_dbg_vggish_layer: unsupported image %d x %d", H, W);
  } else if (relu ? (!out_hi || !out_lo) : !out_f32) {
    return fail("vnb_dbg_vggish_layer: the output is required");
  }
  const cudaError_t e = launch_vggish_tc(a_hi, a_lo, Bn, H, W, Cin, w_hi, w_lo, N, bias, W > 0 || relu, W > 0 && pool,
                                         out_hi, out_lo, out_f32, st);
  if (e == cudaErrorInvalidValue) return fail("vnb_dbg_vggish_layer: %s", tmap_error());
  CK(e);
  return 0;
}

}  // extern "C"
