/* vampnet_b200 — C ABI of the H100-native (sm_90a) VampNet masked-token generation hot path.
 *
 * The reference (hugofloresgarcia/vampnet) is pure Python/PyTorch and has no FFI of its own; its
 * boundary is the Python class surface (SURVEY.md §8b).  These entry points are what a binding
 * for that surface binds (INTEGRATION.md shows the ctypes stub); each cites the reference
 * function it replaces.  Plain pointers and sizes only: device pointers are raw CUDA addresses,
 * `stream` is a cudaStream_t passed as void*.  All functions return 0 on success, non-zero on
 * error; vnb_last_error() returns a thread-local message.  Nothing here aborts the process.
 *
 * Handles are not thread-safe (the reference is called from one worker thread at a time:
 * app.py:730 demo.queue()).
 */
#ifndef VAMPNET_B200_H
#define VAMPNET_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define VNB_ABI_VERSION 2

typedef struct vnb_model vnb_model;

/* Mirrors VampNet.__init__ (reference vampnet/modules/transformer.py:536-552). */
typedef struct vnb_config {
  int32_t n_heads;
  int32_t n_layers;
  int32_t n_codebooks;
  int32_t n_conditioning_codebooks;
  int32_t latent_dim; /* 8 */
  int32_t d_model;    /* embedding_dim */
  int32_t vocab_size; /* 1024; mask token id == vocab_size */
} vnb_config;

/* Packed weights, all DEVICE pointers owned by the caller and kept alive while the model exists.
 * Packing (LoRA fold, weight-norm fold, bf16 rounding, row permutations) is done by the host
 * side (vampnet_b200/modules/transformer.py: pack_weights). */
typedef struct vnb_weights {
  const float* emb_table;  /* (C, V+1, 8)  codec codebooks with the learned MASK row appended (layers.py:145-150) */
  const void* emb_w3;      /* (d, 3*Kp)    bf16, embedding.out_proj.weight (d, 8C) zero-padded to Kp = 8C rounded up to 64
                                           and split w = hi + lo: rows are [hi | lo | hi], the B operand of the
                                           split-bf16 contraction [a_hi | a_hi | a_lo] . [w_hi | w_lo | w_hi]^T
                                           (fp32-grade: the dropped a_lo.w_lo term is 2^-18 relative) (layers.py:132,162) */
  const float* emb_b;      /* (d) */
  const float* norm1;      /* (L, d)       norm_1.weight (informational; the forward uses the folded form) */
  const void* wqkv;        /* (L, 3d, d)   bf16, rows = [w_qs | w_ks | w_vs] (transformer.py:109-114), columns scaled
                                           by norm_1.weight: RMSNorm (transformer.py:43-58) is fused, the kernels
                                           apply rsqrt(mean(x^2)+eps) as a row scale of the GEMM result */
  const void* wo;          /* (L, d, d)    bf16, fc */
  const float* norm3;      /* (L, d)       norm_3.weight */
  const void* w1;          /* (L, 4d, d)   bf16, feed_forward.w_1 (columns scaled by norm_3.weight) with rows interleaved per 256-row tile:
                                           [128 value rows | 128 gate rows] (activations.py:33-35) */
  const void* w2;          /* (L, d, 2d)   bf16, feed_forward.w_2 */
  const float* norm_f;     /* (d)          transformer.norm.weight */
  const void* wcls;        /* (Cp*V, d)    bf16, classifier g*v/|v| (columns scaled by transformer.norm.weight) with rows
                                           permuted to c*V + p (transformer.py:634) */
  const float* bcls;       /* (Cp*V)       permuted the same way */
  const float* rel_bias;   /* (2*rel_sat+1, H) fp32: bias for clamp(key-query, -rel_sat, rel_sat) (transformer.py:123-209) */
  int32_t rel_sat;
} vnb_weights;

/* ---- per-request LoRA adapters ------------------------------------------------------------------------------
 * A fine-tune of the reference is its base model plus rank-8 LoRA on w_qs, w_vs, fc, w_1 and w_2 (transformer.py:22,
 * 109-114, 70-84); nothing else differs.  Registered adapters are applied per group of batch rows on top of the one
 * packed base weight set, so one launch serves requests for different fine-tunes.  In every LoRA'd GEMM an adapted
 * row computes
 *   acc' = acc + sum_{k<8} u[row, k] * B'[col, k],   u[row, :] = y_bf16[row, :] . A'^T (fp32),
 * added in fp32 to the tensor-core accumulator before the epilogue's own operations (row scale, rounding, GEGLU,
 * residual).  Rows of the base (adapter -1) skip the update.  The form is the same for every adapted row wherever it
 * lands, so batched launches equal the calls made one by one.  It is not bit-identical to a model with the same LoRA
 * folded into its weights (the fold happens before the bf16 rounding of W).
 *
 * vnb_adapter_weights: DEVICE pointers to fp32 tensors owned by the caller and kept alive while the adapter is
 * registered.  A' = lora_A with the RMSNorm weight folded in (norm_1 for q/v, norm_3 for w_1), stored k-major;
 * B' = lora_B * alpha / r (alpha = 1, r = 8), rows permuted exactly like the packed weight rows:
 *   a_qkv (L, d, 16)   [A'_q | A'_v] per input column      b_qkv (L, 2d, 8)  [B'_q rows | B'_v rows] (k has no LoRA)
 *   a_wo  (L, d, 8)    fc                                  b_wo  (L, d, 8)
 *   a_w1  (L, d, 8)    w_1 (columns scaled by norm_3)      b_w1  (L, 4d, 8)  rows interleaved like vnb_weights.w1
 *   a_w2  (L, 2d, 8)   w_2                                 b_w2  (L, d, 8) */
#define VNB_LORA_RANK 8
#define VNB_MAX_ADAPTERS 16 /* live adapters per model */
typedef struct vnb_adapter_weights {
  const float* a_qkv;
  const float* b_qkv;
  const float* a_wo;
  const float* b_wo;
  const float* a_w1;
  const float* b_w1;
  const float* a_w2;
  const float* b_w2;
} vnb_adapter_weights;

/* Mirrors the keyword arguments of VampNet.generate that are live on this path
 * (transformer.py:687-710; SURVEY.md §A.6 lists the dead ones).  The per-step schedule arrays
 * are computed by the host with the reference's own fp32 expressions (mask.py:8-9,
 * transformer.py:831-834, 903, 917-919) so that floor(gamma*N0) matches bit for bit. */
typedef struct vnb_gen_params {
  int32_t sampling_steps;
  float temperature;        /* <=0 means softmax(logits) without scaling (transformer.py:1019-1023) */
  const float* gamma;       /* host, [steps]: _gamma((i+1)/steps) as fp32 */
  const float* temp_eff;    /* host, [steps]: mask_temperature * (1 - r_i) as fp32 */
  const int32_t* do_sample; /* host, [steps]: (i/steps) <= sample_cutoff */
  uint32_t seed_lo, seed_hi; /* Philox key */
  int32_t use_graph;        /* 1: capture the whole loop once per shape and replay it as a CUDA graph */
  float top_p;              /* nucleus filtering on the raw logits (transformer.py:1001-1016); <=0 or >=1: off */
} vnb_gen_params;

int32_t vnb_abi_version(void);
const char* vnb_last_error(void);

/* VampNet.__init__ + load (interface.py:27-50): builds tensor maps / workspace lazily per (B, T). */
int32_t vnb_model_create(const vnb_config* cfg, const vnb_weights* w, vnb_model** out);
void vnb_model_destroy(vnb_model* m);

/* embedding.from_codes + VampNet.forward (layers.py:134-162, transformer.py:617-639).
 * codes: (B, C, T) int64 device.  logits: (B, T*Cp, V) fp32 device, i.e. the reference's
 * (B, V, T*Cp) output transposed (the layout generate() permutes to at transformer.py:849). */
int32_t vnb_forward_codes(vnb_model* m, const int64_t* codes, int32_t B, int32_t T, float* logits, void* stream);
/* Register an adapter (errors: a NULL pointer, VNB_MAX_ADAPTERS already live); *id in [0, VNB_MAX_ADAPTERS).  Ids of
 * removed adapters are reused.  Removing an unknown or removed id is an error.  Neither call touches the device. */
int32_t vnb_adapter_add(vnb_model* m, const vnb_adapter_weights* w, int32_t* id);
int32_t vnb_adapter_remove(vnb_model* m, int32_t id);
/* vnb_forward_codes with an adapter per batch row: row_adapter host [B], entries -1 (base) or live ids; NULL = all
 * base (then this is vnb_forward_codes). */
int32_t vnb_forward_codes_adapted(vnb_model* m, const int64_t* codes, int32_t B, int32_t T, const int32_t* row_adapter,
                                  float* logits, void* stream);
/* VampNet.forward on caller-supplied latents (B, 8C, T) fp32 (transformer.py:617). */
int32_t vnb_forward_latents(vnb_model* m, const float* latents, int32_t B, int32_t T, float* logits, void* stream);
/* VampNet.forward(return_activations=True) (transformer.py:617-639, 443-461): as vnb_forward_latents, and the fp32
 * residual stream after EVERY layer is copied to acts (n_layers, B, T, d_model) — the reference's
 * torch.stack(activations). */
int32_t vnb_forward_latents_acts(vnb_model* m, const float* latents, int32_t B, int32_t T, float* logits, float* acts,
                                 void* stream);
/* Debug tap: copy the fp32 residual stream (B*T, d) after the last layer of the last forward. */
int32_t vnb_get_hidden(vnb_model* m, float* out, void* stream);

/* VampNet.generate(return_signal=False) (transformer.py:686-946).
 * z: (B, C, T) int64; mask: (B, C, T) int32 or NULL (default mask, transformer.py:749-751);
 * out: (B, C, T) int64. */
int32_t vnb_generate(vnb_model* m, const int64_t* z, const int32_t* mask, int32_t B, int32_t T,
                     const vnb_gen_params* p, int64_t* out, void* stream);
/* One generate() call of a vnb_generate_many launch: `rows` consecutive batch rows with their own sampling state.
 * The fields mean what the vnb_gen_params fields of the same names mean. */
typedef struct vnb_gen_group {
  int32_t rows;
  float temperature;
  const float* temp_eff;    /* host, [steps] */
  const int32_t* do_sample; /* host, [steps] */
  uint32_t seed_lo, seed_hi; /* Philox key */
  float top_p;
} vnb_gen_group;
/* n_groups independent VampNet.generate(return_signal=False) calls of the same T and sampling_steps in one launch.
 * The B batch rows are split into n_groups contiguous groups in order (groups[g].rows each).  Every group keeps what a
 * call of its own would have: its N0 (the initial mask count over its rows only, transformer.py:766), its temperature,
 * schedules, top_p and key, and its row numbering (the Philox counter uses the row index within the group).  So
 * out equals, bit for bit, the concatenation of vnb_generate over each group's rows; vnb_generate is the one-group
 * case.  gamma: host [steps], shared (it depends on steps only).  z, mask and out as in vnb_generate.
 * Errors: group rows not summing to B, n_groups < 1 or > B, steps outside 1..256, groups that mix top-p with no top-p
 * (the sampler variant is per launch).  Graphs are cached per (B, T) workspace as for vnb_generate: the grouping, the
 * keys and the temperatures are written before every replay and never cause a new capture. */
int32_t vnb_generate_many(vnb_model* m, const int64_t* z, const int32_t* mask, int32_t B, int32_t T, int32_t steps,
                          const float* gamma, const vnb_gen_group* groups, int32_t n_groups, int32_t use_graph,
                          int64_t* out, void* stream);
/* vnb_generate_many with an adapter per group: group_adapter host [n_groups], -1 (base) or a live id; NULL = all base
 * (then this is vnb_generate_many).  Each group equals vnb_generate_many of its rows alone with its adapter, bit for
 * bit.  A launch with no adapted group runs the plain kernels; otherwise the adapted ones (a second graph per
 * workspace key; the group -> adapter table is written before every replay and never causes a capture). */
int32_t vnb_generate_many_adapted(vnb_model* m, const int64_t* z, const int32_t* mask, int32_t B, int32_t T,
                                  int32_t steps, const float* gamma, const vnb_gen_group* groups, int32_t n_groups,
                                  const int32_t* group_adapter, int32_t use_graph, int64_t* out, void* stream);
/* vnb_generate_many_adapted for calls of different lengths: group g is a call of group_frames[g] frames (host
 * [n_groups], each in 1..T), padded to the launch's T.  Its rows' frames t >= group_frames[g] must be kept frames
 * (mask 0) in z / mask; mask is then required.  Attention stops at each row's own length and the padded key columns
 * are zero, so every group's first group_frames[g] frames of out equal, bit for bit, vnb_generate_many_adapted of
 * its rows alone at T = group_frames[g]; its later frames of out are the padding's codes.  group_frames NULL, or every
 * entry T: vnb_generate_many_adapted.  group_adapter may be NULL (all base).  A launch with a shorter group runs the
 * frames-aware QKV and attention (one more graph per workspace key); the per-row frames table is written before
 * every launch or replay and never causes a capture, so one (B, T) graph serves any mix of lengths.
 * Errors: those of vnb_generate_many, a group_frames entry outside 1..T, and a NULL mask with a group shorter than T
 * (the default mask would mask the padding). */
int32_t vnb_generate_ragged(vnb_model* m, const int64_t* z, const int32_t* mask, int32_t B, int32_t T, int32_t steps,
                            const float* gamma, const vnb_gen_group* groups, int32_t n_groups,
                            const int32_t* group_frames, const int32_t* group_adapter, int32_t use_graph, int64_t* out,
                            void* stream);
/* vnb_generate_ragged for calls of different sampling-step counts: group g runs group_steps[g] steps (host [n_groups],
 * each in 1..256, in NON-INCREASING order) with its own gamma schedule group_gamma[g] (host, [group_steps[g]]); its
 * temp_eff and do_sample have group_steps[g] entries.  The launch runs S = group_steps[0] iterations.  Group g is idle
 * for the first S - group_steps[g] of them: its state is not touched and no kernel does work for its rows.  From then
 * on, iteration i is its own step j = i - (S - group_steps[g]), with gamma[j], temp_eff[j], do_sample[j], Philox step
 * word j and the last-step flag on j = group_steps[g] - 1, so every group ends on the launch's last iteration.  Each
 * group's out therefore equals, bit for bit, vnb_generate_ragged of its rows alone with its own steps.  Because of the
 * order, the rows live at an iteration are a prefix of the batch: the GEMMs, attention, the embedding, the LoRA
 * down-projections and the sampler skip the tiles, CTAs and rows wholly past it, so an idle iteration costs close to
 * nothing.  group_frames and group_adapter may be NULL as in vnb_generate_ragged.  Every group with the same count:
 * vnb_generate_ragged's kernels and graph (each group still uses its own gamma).  Otherwise the launch runs the
 * live-bounded kernels (one more graph per workspace key); the per-iteration live-row table is written before every
 * launch or replay, so one (B, T, S) graph serves any assignment of step counts <= S and any grouping.
 * Errors: those of vnb_generate_ragged, NULL group_steps, group_gamma or group_gamma[g], a count outside 1..256 and
 * counts that increase from one group to the next. */
int32_t vnb_generate_steps(vnb_model* m, const int64_t* z, const int32_t* mask, int32_t B, int32_t T,
                           const int32_t* group_steps, const float* const* group_gamma, const vnb_gen_group* groups,
                           int32_t n_groups, const int32_t* group_frames, const int32_t* group_adapter,
                           int32_t use_graph, int64_t* out, void* stream);
/* vnb_generate_steps for groups that may mix nucleus (top-p) and plain sampling: same arguments, same contract, and each
 * group's out equals, bit for bit, vnb_generate_steps of its rows alone.  A group's top-p is on when 0 < top_p < 1.
 *   every group on, or every group off: vnb_generate_steps's kernels and graph;
 *   a mix, "fused_sampler" 1 (and a vocabulary the fused sampler takes): the classifier's split sampling epilogue writes
 *     the records of the plain groups' still-masked positions and stores the fp32 logits of the nucleus groups'
 *     still-masked positions; then the plain rows draw from the records (sample_combine_kernel) and the nucleus rows
 *     from the logits (sample_rows_kernel with the filter), each kernel touching its own rows only; then the re-mask;
 *   a mix, "fused_sampler" 0: the materialising path with the nucleus kernel for every row (a group whose top-p is off
 *     draws there exactly as it does without the filter).
 * The group -> top-p assignment is read from the per-step table written before every launch or replay: one
 * (B, T, S) graph serves any mix.  The logits tensor (M x (C - ncc) x V fp32) is allocated whenever a group's top-p is
 * on.  Errors: those of vnb_generate_steps except the mix. */
int32_t vnb_generate_mixed_top_p(vnb_model* m, const int64_t* z, const int32_t* mask, int32_t B, int32_t T,
                                 const int32_t* group_steps, const float* const* group_gamma,
                                 const vnb_gen_group* groups, int32_t n_groups, const int32_t* group_frames,
                                 const int32_t* group_adapter, int32_t use_graph, int64_t* out, void* stream);
/* One sampling iteration on caller-supplied logits (B, S, V) fp32 — sample_from_logits +
 * mask_by_random_topk + the where()s around them (transformer.py:849-932).  State is explicit:
 * zflat (B, S) int32 in "t c" order (util.py:39) is updated in place; tokens_out (B, S) int32
 * receives sampled_z; conf_out (B, S) fp32 receives the confidences (debug).
 * n0: device pointer to the whole-batch initial mask count (transformer.py:766). */
int32_t vnb_sample_step(const float* logits, int32_t* zflat, int32_t* tokens_out, float* conf_out,
                        const int32_t* n0, int32_t B, int32_t S, int32_t V, int32_t mask_token, int32_t step,
                        int32_t is_last, int32_t do_sample, float temperature, float gamma, float temp_eff,
                        uint32_t seed_lo, uint32_t seed_hi, void* stream);

/* ---- measurement hooks (bench.py) --------------------------------------------------------------
 * vnb_launch_count: kernels launched by this library so far in this process (a graph replay adds the
 * number of kernel nodes it contains).
 * vnb_graph_capture_count: generate graphs captured so far (a weight hot swap or a repeated call must not
 * add to it: graphs are cached per (workspace, steps, mask, top_p, adapted or not, some group shorter than T or
 * not, some group with fewer steps than the launch or not, nucleus and plain groups in one fused launch or not); the
 * grouping of vnb_generate_many, the group -> adapter table, the per-row frames of vnb_generate_ragged, the step counts
 * of vnb_generate_steps and the group -> top-p assignment of vnb_generate_mixed_top_p are not part of that key).
 * vnb_profile_begin/end: between the two calls every launch of forward/generate is bracketed by CUDA
 * events on the launching stream (graph replay is bypassed so that the events can be recorded);
 * end() returns the summed device time and launch count per kernel family:
 *   0 embed, 1 rmsnorm, 2 gemm_qkv, 3 attention, 4 gemm_attn_out, 5 gemm_ffn_up, 6 gemm_ffn_down,
 *   7 gemm_classifier, 8 sample+remask, 9 state init/finish, 10 LoRA down-projection (adapted launches only; the
 *   adapted GEMMs count in their own families). */
#define VNB_NUM_FAMILIES 11
uint64_t vnb_launch_count(void);
uint64_t vnb_graph_capture_count(void);

/* ---- tuning options ----------------------------------------------------------------------------
 * "gemm_pair": 1 = dense contractions run as clusters of two CTAs on vertically adjacent 128 x 256 tiles that share
 *              the weight tile (each CTA fetches half of it, TMA multicast), 0 (default, faster on H100) = one CTA
 *              per 128 x 256 tile.  Results are bit-identical (same
 *              accumulation order per output element).  Initial value: environment VNB_GEMM_PAIR, else the
 *              compiled default.  Generate graphs are cached per value.
 * "fused_sampler": 1 (default) = vnb_generate samples inside the classifier GEMM's epilogue (VNB_EPI_SAMPLE: the logits of
 *   the generate loop never reach HBM), 0 = from a materialised fp32 logits tensor (sample_rows_kernel).  Both draw
 *   with the same two-level inverse CDF and the same Philox stream; nucleus (top-p) sampling always draws from
 *   materialised logits (in a fused vnb_generate_mixed_top_p launch, those the split epilogue stores for its rows).
 * "gemm_pair_max_clusters" (get only): clusters of two that can be co-resident on the current device. */
int32_t vnb_set_option(const char* name, int32_t value);
int32_t vnb_get_option(const char* name, int32_t* value);
int32_t vnb_profile_begin(vnb_model* m);
int32_t vnb_profile_end(vnb_model* m, float* ms_per_family, int32_t* launches_per_family, int32_t n_families);

/* ---- unit-level entry points (parity tests bisect with these) ------------------------------- */
enum {
  VNB_EPI_BF16 = 0,     /* out bf16 (M, N) */
  VNB_EPI_QKV = 1,      /* cols < 2d -> qk bf16 (M, 2d); cols >= 2d -> vT bf16 (B, d, Tpad) */
  VNB_EPI_RESID = 2,    /* out fp32 (M, N) += acc */
  VNB_EPI_GEGLU = 3,    /* out bf16 (M, N/2) = value * gelu_tanh(gate) */
  VNB_EPI_BIAS_F32 = 4, /* out fp32 (M, N) = acc + bias[n] */
  VNB_EPI_SAMPLE = 5    /* internal to vnb_generate: acc + bias[n] sampled per 128-column strip, nothing stored but
                           16 bytes per (row, strip); not accepted by vnb_op_gemm */
};
/* out = A (M,K) bf16 row-major  x  W (N,K)^T bf16 row-major, fp32 accumulation (wgmma).
 * N % 256 == 0, K % 64 == 0.  For VNB_EPI_QKV: out = qk, out2 = vT, T/Tpad describe the batch split. */
int32_t vnb_op_gemm(int32_t epi, const void* A, const void* W, int32_t M, int32_t N, int32_t K, void* out,
                    void* out2, const float* bias, int32_t T, int32_t Tpad, void* stream);
/* Fused self-attention with relative-position bias (transformer.py:234-254).
 * qk (B, T, 2d) bf16 [q | k], vT (B, d, Tpad) bf16, out (B, T, d) bf16, d = H*64; rel_bias (2*rel_sat+1, H) fp32 with
 * entry [clamp(k - q, -rel_sat, rel_sat) + rel_sat, h].  Preconditions: rel_sat in 1..128, Tpad >= T and a multiple of
 * 8 (refused otherwise), every table entry finite, and the v^T padding columns [T, Tpad) finite (the mask gives them
 * weight 0, and 0 * inf would be NaN). */
int32_t vnb_op_attention(const void* qk, const void* vT, void* out, const float* rel_bias, int32_t rel_sat,
                         int32_t B, int32_t T, int32_t Tpad, int32_t H, void* stream);
/* Test-only: vnb_op_attention with a key length per batch row, frames DEVICE [B], entries in 1..T.  Row b attends to
 * keys t < frames[b] only and writes out rows t < frames[b] only; its later rows of qk may hold anything, its later
 * columns of vT must be finite (the QKV epilogue of vnb_dbg_gemm_qkv_frames leaves them zero).  Query tiles wholly past
 * frames[b] do no work. */
int32_t vnb_dbg_attention_ragged(const void* qk, const void* vT, void* out, const float* rel_bias, int32_t rel_sat,
                                 int32_t B, int32_t T, int32_t Tpad, int32_t H, const int32_t* frames, void* stream);
/* Test-only: the live bound that the unit-level entry points of this calling thread (vnb_op_gemm, vnb_op_attention and
 * every vnb_dbg_* op) give their kernels from now on, as vnb_generate_steps gives it at every iteration.  live: DEVICE
 * pointer to one int32 R, or NULL (the default: every row is live).  Batch rows b >= R are idle: GEMM tiles whose
 * first row is at or past R * T (pair: the cluster's first row) and attention CTAs of rows b >= R do no work, the
 * LoRA down-projection and the sampler (vnb_dbg_sample) leave those rows untouched.  Live rows are bit-equal to a
 * launch without a bound; dead rows of a tile that straddles R * T are unspecified. */
int32_t vnb_dbg_set_live(const int32_t* live);
/* Naive SIMT GEMM used only to bisect the tensor-core path in tests: out fp32 (M, N) = A x W^T. */
int32_t vnb_dbg_gemm_ref(const void* A, const void* W, int32_t M, int32_t N, int32_t K, float* out, void* stream);
/* Test-only: vnb_op_gemm plus the fused-RMSNorm plumbing the forward uses, epi in {BF16, QKV, RESID, GEGLU, BIAS_F32}.
 * Consumer side: ss_in (ss_parts, M) fp32 or NULL; every accumulator row m is scaled by
 *   rs = rsqrt(sum_{p < ss_parts} ss_in[p*M + m] * inv_d + eps)   (partials added in order p = 0, 1, ...)
 * before the epilogue's own operation (GEGLU: value and gate; QKV: qk and vT; BIAS_F32: before the bias).
 * Producer side (RESID and BIAS_F32 only, both or neither, error otherwise): out_bf16 (M, N) bf16 = bf16(out) and
 * ss_out fp32 row sums of squares of out, part p at ss_out[p*M + m]:
 *   RESID     2 parts per 256-column tile j: part 2j over its 32-column chunks {0, 2, 4, 6}, part 2j+1 over {1, 3, 5, 7}
 *             (N/128 parts in all);
 *   BIAS_F32  1 part per 256-column tile (N/256 parts); nothing else is written. */
int32_t vnb_dbg_gemm_fused(int32_t epi, const void* A, const void* W, int32_t M, int32_t N, int32_t K, void* out,
                           void* out2, const float* bias, int32_t T, int32_t Tpad, const float* ss_in,
                           int32_t ss_parts, float inv_d, float eps, void* out_bf16, float* ss_out, void* stream);
/* Test-only: one adapted GEMM, epi in {QKV, RESID, GEGLU}, with the arguments of vnb_dbg_gemm_fused.  First the
 * LoRA down-projection u (M, R) fp32 = A . A'^T of every row m with row_adapter[m] >= 0 (R = 16 for QKV, else 8; rows
 * of the base are not written), then the GEMM whose epilogue adds u[m] . B'[n] to the accumulators of those rows.
 * adapters[n_adapters] (n_adapters <= VNB_MAX_ADAPTERS) as in vnb_adapter_weights, layer = the layer they are read
 * at; row_adapter DEVICE [M], entries -1 or < n_adapters. */
int32_t vnb_dbg_gemm_adapted(int32_t epi, const void* A, const void* W, int32_t M, int32_t N, int32_t K, void* out,
                             void* out2, int32_t T, int32_t Tpad, const float* ss_in, int32_t ss_parts, float inv_d,
                             float eps, void* out_bf16, float* ss_out, const vnb_adapter_weights* adapters,
                             int32_t n_adapters, int32_t layer, const int32_t* row_adapter, float* u, void* stream);
/* Test-only: the QKV GEMM of a launch of calls with different lengths: vnb_dbg_gemm_fused(VNB_EPI_QKV, ...) with
 * adapters NULL, else vnb_dbg_gemm_adapted(VNB_EPI_QKV, ...), plus frames DEVICE [ceil(M / T)]: vT column t of batch
 * row b is written as exactly 0 for t >= frames[b].  Everything else is what the call without frames writes. */
int32_t vnb_dbg_gemm_qkv_frames(const void* A, const void* W, int32_t M, int32_t N, int32_t K, void* out, void* vT,
                                int32_t T, int32_t Tpad, const float* ss_in, int32_t ss_parts, float inv_d, float eps,
                                const int32_t* frames, const vnb_adapter_weights* adapters, int32_t n_adapters,
                                int32_t layer, const int32_t* row_adapter, float* u, void* stream);
/* Test-only: the classifier GEMM with the sampling epilogue of the generate loop (VNB_EPI_SAMPLE) alone.
 * N == (C - ncc) * V, V % 128 == 0, V <= 1024; logits x = (A . W^T) * rs + bias with rs as above.
 * zcur (M, C) int32, row m = b*T + t: codebook ncc + cp of row m is sampled iff it holds mask_token.
 * partials (M * (C-ncc) * V/128) float4: for every sampled (row m, codebook cp, 128-entry tile k), record
 * (m*(C-ncc) + cp) * V/128 + k = {max x, sum exp((x - max) / temperature), x of the candidate, candidate | argmax << 16}
 * (vocabulary indices; argmax: lowest index on ties; candidate: first entry whose running sum exceeds u * sum, u the
 * second Philox uniform of counter (t*(C-ncc) + cp, b, step, 0) and key (seed_lo, seed_hi), the argmax when do_sample
 * is 0).  Records of known positions are not written.  temperature <= 0 means 1. */
int32_t vnb_dbg_gemm_sample(const void* A, const void* W, const float* bias, int32_t M, int32_t N, int32_t K,
                            const float* ss_in, int32_t ss_parts, float inv_d, float eps, const int32_t* zcur,
                            int32_t T, int32_t C, int32_t ncc, int32_t V, int32_t mask_token, float temperature,
                            int32_t do_sample, int32_t step, uint32_t seed_lo, uint32_t seed_hi, void* partials,
                            void* stream);
/* Test-only: one sampling step of the generate loop alone, with everything vnb_generate_many gives it made explicit.
 * A group is `rows` consecutive batch rows with the scalars of one generate() call at one step (fields as in
 * vnb_gen_group and vnb_gen_params; gamma = the schedule value of this step, is_last = this is the last step). */
typedef struct vnb_sample_group {
  int32_t rows;
  float temperature; /* <= 0 means 1 */
  float gamma, temp_eff;
  int32_t do_sample, is_last, step;
  uint32_t seed_lo, seed_hi;
  float top_p; /* <= 0 or >= 1: no nucleus filter */
} vnb_sample_group;
/* path 0: sample_rows_kernel (no nucleus filter) on logits, then the re-mask;
 * path 1: sample_rows_kernel with the nucleus filter (groups whose top_p is disabled draw as in path 0), then the
 *         re-mask;
 * path 2: sample_combine_kernel on caller-supplied partials (the records vnb_dbg_gemm_sample writes, row m = b*T + t),
 *         then the re-mask;
 * path 3: the re-mask alone, on caller-supplied tokens and conf.
 * logits (B*S, V) fp32 (paths 0, 1), S = T * (C - ncc); partials (B*S*V/128) float4 (path 2); zcur (B, T, C) int32,
 * updated in place; zorig (B, T, C) int32 or NULL (then the conditioning codebooks of zcur are left as they are);
 * tokens, conf (B, S) written by paths 0-2, read by path 3; n0 DEVICE [n_groups] initial mask count of each group.
 * The [group] table of sampling scalars and the row -> group map are built as vnb_generate_many builds them (the Philox
 * counter of batch row b uses b minus its group's first row).  Refused: path outside 0..3, B or T < 1, ncc outside
 * 0..C-1, V not a multiple of 128 in 128..1024, group rows that do not sum to B (or n_groups outside 1..B), a NULL buffer
 * the path needs.  Synchronises `stream` before returning (the staged table is freed). */
int32_t vnb_dbg_sample(int32_t path, const float* logits, const void* partials, int32_t* zcur, const int32_t* zorig,
                       int32_t* tokens, float* conf, const int32_t* n0, int32_t B, int32_t T, int32_t C, int32_t ncc,
                       int32_t V, int32_t mask_token, const vnb_sample_group* groups, int32_t n_groups, void* stream);
/* Test-only: the classifier GEMM with the split sampling epilogue of a fused vnb_generate_mixed_top_p launch.  The
 * arguments of vnb_dbg_gemm_sample, except that the per-call scalars come from groups[n_groups] over the M / T batch rows
 * (M a multiple of T; temperature, do_sample, step, seeds and top_p are read), plus logits (M, N) fp32.  A still-masked
 * position of a plain group (top_p <= 0 or >= 1) gets the record vnb_dbg_gemm_sample writes; one of a nucleus group gets
 * no record, and its 128-column strip of logits is stored at logits[m*N + (cp*V + v)] with the bits of
 * vnb_dbg_gemm_fused(VNB_EPI_BIAS_F32).  Nothing else is written.  Synchronises `stream` before returning. */
int32_t vnb_dbg_gemm_sample_split(const void* A, const void* W, const float* bias, int32_t M, int32_t N, int32_t K,
                                  const float* ss_in, int32_t ss_parts, float inv_d, float eps, const int32_t* zcur,
                                  int32_t T, int32_t C, int32_t ncc, int32_t V, int32_t mask_token,
                                  const vnb_sample_group* groups, int32_t n_groups, void* partials, float* logits,
                                  void* stream);
/* Test-only: the sampler of a fused vnb_generate_mixed_top_p launch, with vnb_dbg_sample's arguments and rules: the
 * combine (path 2) on the rows of plain groups from partials, the nucleus draw (path 1) on the rows of nucleus groups
 * from logits, each leaving the other kind's tokens and conf untouched, then the re-mask of every row.  Both partials
 * and logits are required. */
int32_t vnb_dbg_sample_split(const float* logits, const void* partials, int32_t* zcur, const int32_t* zorig,
                             int32_t* tokens, float* conf, const int32_t* n0, int32_t B, int32_t T, int32_t C,
                             int32_t ncc, int32_t V, int32_t mask_token, const vnb_sample_group* groups,
                             int32_t n_groups, void* stream);

/* ---- codec (DAC family; reference call sites: interface.py:223 codec.encode, transformer.py:671-675
 *      codec.quantizer.from_latents + codec.decode).  fp32, (B, C, T) channels-first. ------------------------
 * Generic 1-D convolution with the Snake activation fused on the input:
 *   y[b, co, q*out_stride + out_off] = bias[co] + sum_ci sum_j w[co, ci, j] * act(x[b, ci, q*stride + j*dil - pad])
 *                                      (+ residual) (tanh)
 * q in [0, nq).  snake_alpha (Cin) or NULL; residual (same shape as y) or NULL.  A ConvTranspose1d with stride s
 * is s launches of the K=2, dil=-1 form with out_stride = s (one per output phase). */
int32_t vnb_codec_conv1d(const float* x, const float* w, const float* bias, const float* snake_alpha,
                         const float* residual, float* y, int32_t B, int32_t Cin, int32_t Tin, int32_t Cout,
                         int32_t Tout, int32_t K, int32_t stride, int32_t dil, int32_t pad, int32_t out_stride,
                         int32_t out_off, int32_t nq, int32_t do_tanh, void* stream);
/* Residual vector quantiser.  mode 0 encode: in_f = z (B,D,T) -> codes (B,L,T) int64, zq (B,D,T), latents (B,8L,T).
 * mode 1 from_latents: in_f = latents (B,8L,T) -> zq.  mode 2 from_codes: in_codes (B,L,T) -> zq.
 * win (L,8,D), bin (L,8), wout (L,D,8), bout (L,D), cb (L,V,8) raw and cbn (L,V,8) L2-normalised codebooks. */
int32_t vnb_codec_rvq(int32_t mode, const float* in_f, const int64_t* in_codes, const float* win, const float* bin,
                      const float* wout, const float* bout, const float* cb, const float* cbn, int64_t* codes, float* zq,
                      float* latents, int32_t B, int32_t D, int32_t T, int32_t L, int32_t V, int32_t channels_last,
                      void* zq_hi, void* zq_lo, void* stream);
/* Tensor-core codec path (wgmma, split-bf16 operands = fp32-grade products; see csrc/conv_wgmma.cu).
 * Activations are channels-last (B, T, C) and travel as hi/lo bf16 pairs (x = hi + lo).
 *   y[b, q, n] = bias[n % bias_mod] + sum_tap sum_ci W[n, tap, ci] * a[b, q*s + tap*dil - pad, ci]   (+ resid)
 * w_hi/w_lo: (N, taps * ceil(Cin/64) * 64) bf16, tap-major, channel blocks zero-padded to 64.
 * Outputs (each optional): out_f32 = y, out_hi/out_lo = split(snake_alpha(y)) (alpha NULL: identity).
 * Output element (q, n) of batch b lands at b*out_batch_stride + q*N + n + out_offset, and is dropped unless that
 * flat index (without the batch term) is in [0, out_limit): this is how a transposed convolution with N = s*Cout
 * phase-major columns writes its (T*s, Cout) result. */
int32_t vnb_codec_conv_tc(const void* a_hi, const void* a_lo, int32_t B, int32_t Tin, int32_t Cin, int32_t s,
                          const void* w_hi, const void* w_lo, int32_t N, int32_t taps, int32_t dil, int32_t pad,
                          int32_t Tq, const float* bias, int32_t bias_mod, const float* alpha, int32_t alpha_mod,
                          const float* resid, float* out_f32, void* out_hi, void* out_lo, int64_t out_batch_stride,
                          int64_t out_offset, int64_t out_limit, int32_t do_tanh, void* stream);
/* encoder.conv1 (Cin = 1): x (B,1,T) -> fp32 (B,T,C) + split snake_alpha(y);  decoder.conv2 (Cout = 1) + tanh. */
int32_t vnb_codec_conv_in(const float* x, const float* w, const float* bias, const float* alpha, float* out_f32,
                          void* out_hi, void* out_lo, int32_t B, int32_t T, int32_t C, int32_t K, int32_t pad,
                          void* stream);
int32_t vnb_codec_conv_out(const void* a_hi, const void* a_lo, const float* w, const float* bias, float* audio, int32_t B,
                           int32_t T, int32_t C, int32_t K, int32_t pad, void* stream);
/* Clips of different lengths in one launch.  The _ragged forms take the arguments above (B, T, Tq: the launch's, i.e.
 * the longest item's) plus lens, DEVICE int32 [B]: item b's valid OUTPUT rows at this layer's rate (conv_tc: rows of
 * row_elems elements, N for a plain convolution, Cout for a transposed one, where lens[b] * Cout replaces out_limit;
 * conv_in / conv_out: samples).  Halo contract, per item b with len = lens[b] and H = 128 rows:
 *   - rows [0, len) hold the values a launch of that item alone at length len computes, bit for bit, PROVIDED that
 *     the input rows [len_in, len_in + H) hold +0 (hi and lo) and rows [0, len_in) hold the item's input;
 *   - conv_tc and conv_in store +0 (fp32, hi and lo) on the rows [len, len + H) (within the output buffer);
 *   - output rows from len + H on are not written (CTAs whose rows all lie there exit at once), and neither are
 *     conv_out's samples from len on.
 * H covers the reach of every codec layer (at most 27 rows), so a chain of ragged layers keeps the contract.  The
 * edge kernels bound their reads by len, not by zero padding (a tap on +0 could turn a -0 sum into +0).
 * Refused: a NULL lens, row_elems < 1, and whatever the plain forms refuse. */
int32_t vnb_codec_conv_tc_ragged(const void* a_hi, const void* a_lo, int32_t B, int32_t Tin, int32_t Cin, int32_t s,
                                 const void* w_hi, const void* w_lo, int32_t N, int32_t taps, int32_t dil, int32_t pad,
                                 int32_t Tq, const float* bias, int32_t bias_mod, const float* alpha, int32_t alpha_mod,
                                 const float* resid, float* out_f32, void* out_hi, void* out_lo,
                                 int64_t out_batch_stride, int64_t out_offset, int64_t out_limit, int32_t do_tanh,
                                 const int32_t* lens /* DEVICE [B] */, int32_t row_elems, void* stream);
int32_t vnb_codec_conv_in_ragged(const float* x, const float* w, const float* bias, const float* alpha, float* out_f32,
                                 void* out_hi, void* out_lo, int32_t B, int32_t T, int32_t C, int32_t K, int32_t pad,
                                 const int32_t* lens /* DEVICE [B] */, void* stream);
int32_t vnb_codec_conv_out_ragged(const void* a_hi, const void* a_lo, const float* w, const float* bias, float* audio,
                                  int32_t B, int32_t T, int32_t C, int32_t K, int32_t pad,
                                  const int32_t* lens /* DEVICE [B] */, void* stream);
/* ---- onset detection (reference mask.py:203-226: librosa 0.10 onset.onset_detect(y, sr, hop_length=hop,
 *      backtrack=True), restated on the device; DESIGN.md §9).  Nothing here synchronises. --------------------------
 * samples (B, N) fp32 DEVICE, one clip per row; F = 1 + N / hop frames.  Each row is analysed on its own (its own dB
 * maximum and normalisation), so a row's results equal that row run alone, bit for bit.  Outputs (DEVICE):
 * envelope (B, F) the normalised onset strength; onsets (B, F) int32, row b's first counts[b] entries are its onset
 * frames in increasing order (backtrack != 0: moved to the preceding local minimum of the envelope, which may repeat
 * a frame, as librosa does).  workspace: DEVICE, at least vnb_onset_workspace_bytes(B, N, hop) bytes.  The mel
 * filterbank, window and FFT twiddles are built on the host in float64 on the first call for a (device, sr, hop) and
 * cached; that first call allocates and uploads them.  Refused: B outside 1..65535, N < 1, sr < 1, hop < 1, a NULL
 * buffer, a workspace that is too small. */
int32_t vnb_onset_workspace_bytes(int32_t B, int32_t N, int32_t hop, uint64_t* bytes);
int32_t vnb_onset_detect(const float* samples, int32_t B, int32_t N, int32_t sr, int32_t hop, int32_t backtrack,
                         void* workspace, uint64_t workspace_bytes, float* envelope, int32_t* onsets, int32_t* counts,
                         void* stream);
/* mask (B, C, T) int64 DEVICE = the reference's  mask = ones; for idx in onsets: mask[:, :, idx-width:idx+width] = 0
 * with Python slice semantics (a negative start wraps to T + idx - width, so that slice is usually empty).  Batch
 * row b uses onset row 0 when onset_rows == 1 (the reference analyses samples[0][0] only), else onset row b; onsets
 * and counts as written by vnb_onset_detect with F frames per row.  Refused: B, C, T or F < 1, onset_rows not 1 or B,
 * a NULL buffer. */
int32_t vnb_onset_mask(const int32_t* onsets, const int32_t* counts, int32_t onset_rows, int32_t F, int32_t width,
                       int64_t* mask, int32_t B, int32_t C, int32_t T, void* stream);
/* ---- beat tracking (librosa 0.10.1 beat.beat_track(y, sr, hop_length=hop) with start_bpm, tightness and trim as
 *      given, frame units, restated on the device; DESIGN.md §10).  Nothing here synchronises. ----------------------
 * samples (B, N) fp32 DEVICE, one clip per row; F = 1 + N / hop frames.  Each row is analysed on its own, so a row's
 * results equal that row run alone, bit for bit.  Outputs (DEVICE): envelope (B, F) fp32 onset strength (the median
 * over the 128 mel bands of the clamped dB flux); tempo (B) float64 BPM, 0 for an all-zero envelope; beats (B, F)
 * int32, row b's first counts[b] entries are its beat frames in increasing order.  Everything after the envelope is
 * float64.  workspace: DEVICE, at least vnb_beat_workspace_bytes(B, N, hop) bytes.  The float64 tables are built on
 * the host on the first call for a (device, sr, hop) and cached; that first call allocates and uploads them.
 * Refused: B outside 1..65535; N, sr or hop < 1; start_bpm or tightness <= 0; an 8 s tempo window int(8 sr) // hop
 * outside 2..4096 frames; a NULL buffer; a workspace that is too small. */
int32_t vnb_beat_workspace_bytes(int32_t B, int32_t N, int32_t hop, uint64_t* bytes);
int32_t vnb_beat_track(const float* samples, int32_t B, int32_t N, int32_t sr, int32_t hop, double start_bpm,
                       double tightness, int32_t trim, void* workspace, uint64_t workspace_bytes, float* envelope,
                       double* tempo, int32_t* beats, int32_t* counts, void* stream);
/* test hook: the tempo and beat decisions of vnb_beat_track from a caller's fp32 envelope (B, F) DEVICE.  workspace:
 * vnb_beat_workspace_bytes(B, (F - 1) * hop + 1, hop) bytes.  The same refusals, with F < 1 in place of N < 1. */
int32_t vnb_dbg_beat_from_envelope(const float* envelope, int32_t B, int32_t F, int32_t sr, int32_t hop,
                                   double start_bpm, double tightness, int32_t trim, void* workspace,
                                   uint64_t workspace_bytes, double* tempo, int32_t* beats, int32_t* counts,
                                   void* stream);
/* ---- pitch shift (torch_pitch_shift 1.2's pitch_shift: torch.stft -> torchaudio.functional.phase_vocoder ->
 *      torch.istft -> torchaudio.functional.resample, restated on the device; DESIGN.md §11).  Nothing here
 *      synchronises. -------------------------------------------------------------------------------------------------
 * samples and out (rows, N) fp32 DEVICE, each row shifted on its own with fixed-order reductions, so a row's result
 * equals that row run alone, bit for bit.  The caller passes what the Python wrapper derives from the shift:
 * new_freq = int(sample_rate / ratio) and rate = float(1 / ratio); the library derives the frame counts, the istft
 * length and the gcd of the two rates.  Everything between the fp32 ends is float64.  workspace: DEVICE, at least
 * vnb_pitch_workspace_bytes(...) bytes (about 0.6 GB per 10 s row at 44.1 kHz and +12 semitones).  The float64 DFT
 * bases are built on the host on the first call for a (device, n_fft) and cached; that first call allocates and
 * uploads them.  Refused: a NULL buffer, a workspace that is too small, rows outside 1..65535, n_fft outside 16..4096,
 * hop < 1 or hop > n_fft, N <= n_fft / 2, sample_rate or new_freq < 1, rate <= 0 or not finite, and an empty istft
 * signal (even n_fft with one stretched frame, ceil(F / rate) = 1, as torch.istft refuses it). */
int32_t vnb_pitch_workspace_bytes(int32_t rows, int32_t N, int32_t sample_rate, int32_t new_freq, int32_t n_fft,
                                  int32_t hop, double rate, uint64_t* bytes);
int32_t vnb_pitch_shift(const float* samples, int32_t rows, int32_t N, int32_t sample_rate, int32_t new_freq,
                        int32_t n_fft, int32_t hop, double rate, void* workspace, uint64_t workspace_bytes, float* out,
                        void* stream);
/* Test-only: where vnb_pitch_shift with the same arguments keeps its float64 intermediates in the workspace, as
 * byte offsets (-1: not kept for these arguments), and the shapes it derives:
 *   offsets[0] spectrum (rows, F, nb) complex: X as the forward DFT wrote it when rate == 1; (|X|, angle X) when
 *              rate != 1
 *   offsets[1] stretched spectrum (rows, F2, nb) complex, after the vocoder (-1 when rate == 1)
 *   offsets[2] inverse-DFT frames (rows, F2, n_fft)
 *   offsets[3] overlap-added signal (rows, L)
 * with nb = n_fft / 2 + 1 and dims = {F, F2, L, target}.  Same refusals as vnb_pitch_workspace_bytes, and NULL
 * offsets or dims. */
int32_t vnb_dbg_pitch_layout(int32_t rows, int32_t N, int32_t sample_rate, int32_t new_freq, int32_t n_fft,
                             int32_t hop, double rate, int64_t* offsets, int64_t* dims);
/* test hook: the phase vocoder's time steps, out[i] = float(rate) * float(i) for i < n, fp32 DEVICE */
int32_t vnb_dbg_pitch_time_steps(double rate, int32_t n, float* out, void* stream);
/* ---- validation metrics (the reference's scripts/exp/train.py val_loop / _metrics / accuracy, train.py:155-213,
 *      327-371; DESIGN.md §12).  Nothing here synchronises. -----------------------------------------------------------
 * logits (B, S, V) fp32 DEVICE, 16-byte aligned, as vnb_forward_codes writes them, S = T * (C - ncc), row s = t * (C -
 * ncc) + c.  z and mask (B, C, T) int64 DEVICE: row (b, s)'s target is z[b, ncc + s % (C - ncc), s / (C - ncc)], it is
 * masked where mask at the same place is not 0.  r (B) float64 DEVICE, each item's mask ratio.  Writes out9, fp32
 * DEVICE, in the reference's key order:
 *   [0] loss: CrossEntropyLoss(label_smoothing, ignore_index) over the masked rows, ((1 - ls) sum nll + ls sum smooth) /
 *       n with nll = lse - x[target] and smooth = lse - mean(x), summed in float64 and rounded to fp32 once; NaN when
 *       no row is masked;
 *   [1 + 4 range + 2 k + sel] accuracy over the rows of the items whose r lies in range 0 = [0, 0.5) or 1 = [0.5, 1.0)
 *       (r = 1.0 is in neither), k 0 = top-1 or 1 = top-25, sel 0 = unmasked or 1 = masked rows: the share of rows
 *       whose target is in the top k, NaN for an empty selection.  A row with gt = #{x > x[target]} and eq = #{other
 *       x == x[target]} is correct iff gt + eq < k; a row with gt < k <= gt + eq (a tie at the k-th place, which
 *       torch.topk breaks in an implementation-defined way) counts as not correct and, when ambiguous is not NULL, in
 *       ambiguous[i], int32 DEVICE (9; ambiguous[0] = 0).
 * A code outside 0..V-1 cannot be refused without a host read: it makes the loss NaN, and every accuracy whose
 * selection holds its row.  Every reduction has a fixed order: two calls give the same bits, and a row's record
 * (vnb_dbg_xent_rows) equals that row run in a batch of one.  workspace: DEVICE, at least
 * vnb_xent_metrics_workspace_bytes(B, S) bytes.  Refused: a NULL buffer, B, C or T < 1, ncc outside 0..C-1, V outside
 * 1..1024 or not a multiple of 4, label_smoothing outside [0, 1] or NaN, a workspace that is too small, logits not
 * 16-byte aligned. */
typedef struct vnb_xent_row {
  double nll, smooth; /* NaN for an out-of-range code */
  int32_t gt, eq;     /* -1 for an out-of-range code */
} vnb_xent_row;
int32_t vnb_xent_metrics_workspace_bytes(int32_t B, int64_t S, uint64_t* bytes);
int32_t vnb_xent_metrics(const float* logits, const int64_t* z, const int64_t* mask, const double* r, int32_t B,
                         int32_t C, int32_t T, int32_t ncc, int32_t V, double label_smoothing, void* workspace,
                         uint64_t workspace_bytes, float* out9, int32_t* ambiguous, void* stream);
/* test hook: the per-row records (B * S vnb_xent_row, DEVICE) of vnb_xent_metrics; same refusals */
int32_t vnb_dbg_xent_rows(const float* logits, const int64_t* z, int32_t B, int32_t C, int32_t T, int32_t ncc,
                          int32_t V, vnb_xent_row* rows, void* stream);
/* ---- mel spectrogram and multi-scale mel distance (audiotools' AudioSignal.mel_spectrogram and
 *      metrics.spectral.MelSpectrogramLoss, restated on the device; DESIGN.md §13).  Nothing here synchronises. -----
 * One scale: |torch.stft(x, n_fft, hop, window=periodic Hann, center=True, pad_mode="reflect")| in fp32, F = 1 + N / hop
 * frames, projected on librosa.filters.mel(sr, n_fft, n_mels, fmin, fmax) (Slaney scale and norm, float32 weights).
 * fmax is given explicitly (audiotools' None is sr / 2). */
typedef struct vnb_mel_scale {
  int32_t n_fft, hop, n_mels;
  double fmin, fmax;
} vnb_mel_scale;
/* samples (rows, N) fp32 DEVICE -> out (rows, n_mels, F) fp32 DEVICE.  A row's output depends on that row only, so it
 * equals the row run alone, bit for bit.  The window, twiddles and filterbank are built on the host in float64 on the
 * first call for a (device, sr, n_fft, n_mels, fmin, fmax) and cached; that first call allocates and uploads them.
 * Refused: a NULL buffer, rows outside 1..65535, sr < 1, n_fft not a power of two in 32..4096, N <= n_fft / 2 (the
 * reflect padding), hop < 1, n_mels outside 1..4096, fmin < 0, fmax <= fmin. */
int32_t vnb_mel_spectrogram(const float* samples, int32_t rows, int32_t N, int32_t sr, const vnb_mel_scale* scale,
                            float* out, void* stream);
/* x and y (B, C, N) fp32 DEVICE, the same sample rate.  For each scale, with X and Y the (B, C, n_mels, F) spectrograms:
 *   loss += log_weight * mean|log10(max(X, clamp_eps)^pow) - log10(max(Y, clamp_eps)^pow)| + mag_weight * mean|X - Y|
 * over all B C n_mels F elements (item_loss[b]: over item b's C n_mels F), clamp, pow (as pow * log10) and log10 in
 * float64, every sum in float64 in a fixed order, each result rounded to fp32 once.  loss (1) fp32 DEVICE; item_loss
 * (B) fp32 DEVICE or NULL.  An item's loss depends on that item only, so it equals the item run alone, bit for bit.
 * workspace: DEVICE, at least vnb_mel_workspace_bytes(B, C, N, scales, n_scales) bytes.  Refused: a NULL buffer,
 * B * C outside 1..65535, n_scales outside 1..16, any scale refused as by vnb_mel_spectrogram, clamp_eps <= 0 or not
 * finite, pow, log_weight or mag_weight not finite, a workspace that is too small. */
int32_t vnb_mel_workspace_bytes(int32_t B, int32_t C, int32_t N, int32_t sr, const vnb_mel_scale* scales,
                                int32_t n_scales, uint64_t* bytes);
int32_t vnb_mel_loss(const float* x, const float* y, int32_t B, int32_t C, int32_t N, int32_t sr,
                     const vnb_mel_scale* scales, int32_t n_scales, double clamp_eps, double pow, double log_weight,
                     double mag_weight, void* workspace, uint64_t workspace_bytes, float* loss, float* item_loss,
                     void* stream);
/* internal helper exported for the other translation units */
int32_t vnb_set_error_cuda(const char* what, int32_t cuda_error);

#ifdef __cplusplus
}
#endif
#endif /* VAMPNET_B200_H */
