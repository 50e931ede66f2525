// vampnet_b200 — internal launcher declarations shared by the .cu translation units.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/vampnet_b200.h"

namespace vnb {

// Function attributes (max dynamic smem) are per device: remember them per (kernel, device), not per process.
struct PerDeviceOnce {
  unsigned long long done = 0;  // bit d = attribute already set on device d
  bool need(int* dev_out) {
    int dev = 0;
    cudaGetDevice(&dev);
    *dev_out = dev;
    return dev >= 64 || !((done >> dev) & 1ull);
  }
  void mark(int dev) { if (dev < 64) done |= 1ull << dev; }
};
inline int device_sm_count() {
  static int sms[64] = {0};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev >= 64) { int n = 0; cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev); return n; }
  if (!sms[dev]) cudaDeviceGetAttribute(&sms[dev], cudaDevAttrMultiProcessorCount, dev);
  return sms[dev];
}

// kernels launched by this library so far (vnb_launch_count; graph replays add their node count)
void count_launch(unsigned long long n = 1);

// ---- TMA tensor maps (driver entry point fetched at run time; no link-time libcuda dependency) ----
// 2-D bf16 row-major (rows, cols) with a (box_rows x 64) box, 128B swizzle.
bool make_tmap_2d(CUtensorMap* tm, const void* base, uint64_t rows, uint64_t cols, uint32_t box_rows,
                  uint32_t box_cols);
// 3-D bf16 (batch, rows, cols) row-major with row pitch `pitch_elems`; box (1, box_rows, 64), 128B swizzle.
bool make_tmap_3d(CUtensorMap* tm, const void* base, uint64_t batch, uint64_t rows, uint64_t cols,
                  uint64_t pitch_elems, uint32_t box_rows, uint32_t box_cols);
const char* tmap_error();
}  // namespace vnb
// sets the thread-local error string from a CUDA error code; returns 1
extern "C" int32_t vnb_set_error_cuda(const char* what, int32_t cuda_error);
namespace vnb {

struct SampleDyn;
// Batch row b of a generate launch belongs to group `group` (one would-be generate() call) whose rows start at `first`.
struct RowGroup {
  int32_t group, first;
};

// ---- per-request LoRA adapters (DESIGN.md §1) ----
// One registered adapter: the device pointers of vnb_adapter_weights, indexed by LoRA slot (a[s], b[s]).
enum { LORA_QKV = 0, LORA_WO, LORA_W1, LORA_W2, LORA_SLOTS };
struct AdapterDev {
  const float* a[LORA_SLOTS];  // A' (L, K, R_s) fp32, k-major
  const float* b[LORA_SLOTS];  // B' (L, N_s, 8) fp32
};
// How the rows of a launch find their adapter: row m -> batch row m / rows_per_grp -> rowgrp[.].group ->
// grp_adapter[group] (-1: base row, no update) -> table[id].
struct AdapterRefs {
  const AdapterDev* table = nullptr;
  const int32_t* grp_adapter = nullptr;
  const RowGroup* rowgrp = nullptr;
  int rows_per_grp = 1;
  int slot = 0, layer = 0;
  float* u = nullptr;  // (M, R) the down-projection of every adapted row, R = 16 for LORA_QKV ([q | v]), else 8
};
// u = y . A'^T for every adapted row of y (M, K) bf16; base rows are not touched, nor rows at or past live[0] * T
// (live: device, null = every row)
cudaError_t launch_lora_down(const void* y, int M, int K, const AdapterRefs& r, const int32_t* live, int T,
                             cudaStream_t st);

// ---- GEMM ----
struct GemmPlan {
  CUtensorMap tmA, tmB;
  CUtensorMap tmBh;  // W with a 128-row box: the half tile each CTA of a pair fetches and multicasts (gemm_wgmma.cu, PAIR)
  int M = 0, N = 0, K = 0, epi = 0;
  void* out = nullptr;
  void* out2 = nullptr;
  const float* bias = nullptr;
  int T = 1, Tpad = 1, d2 = 0;
  // fused RMSNorm plumbing (see GemmArgs in gemm_wgmma.cu)
  void* out_bf16 = nullptr;
  float* ss_out = nullptr;
  const float* ss_in = nullptr;
  int ss_parts = 0;
  float inv_d = 0.f, eps = 0.f;
  // VNB_EPI_SAMPLE (the classifier of the generate loop): the logits are sampled in the epilogue instead of being stored
  const int32_t* zcur = nullptr;     // (B, T, C) current tokens: only still-masked positions are sampled
  const SampleDyn* dyn = nullptr;    // this step's scalars, one per group (device memory: graph replay safe)
  const RowGroup* rowgrp = nullptr;  // (B) group of every batch row
  void* partials = nullptr;          // (M * Cp * V/128) float4 records, see sample_combine_kernel
  // a launch of nucleus (top-p) and plain groups: the rows of nucleus groups store their logits to `out` (the
  // materialising epilogue's layout, still-masked positions only) and leave no records
  bool sample_split = false;
  int C = 0, ncc = 0, V = 0, mask_token = 0;
  // adapted variant of QKV / RESID / GEGLU (null table: the plain kernel): acc += u[row] . B'[col] for adapted rows
  AdapterRefs lora;
  // VNB_EPI_QKV of a launch whose calls have different lengths: (B) frames of every batch row; v^T column t of batch row
  // b is written as 0 for t >= frames[b] (null: every row has T frames)
  const int32_t* frames = nullptr;
  // launches of calls with different step counts: (1) the number of live batch rows this iteration (device); tiles
  // wholly at or past row live[0] * T exit at once (null: every row is live)
  const int32_t* live = nullptr;
};
// Fills the tensor maps; A (M,K) bf16, W (N,K) bf16.
bool make_gemm_plan(GemmPlan* p, int epi, const void* A, const void* W, int M, int N, int K, void* out, void* out2,
                    const float* bias, int T, int Tpad, int d2);
bool gemm_plan_set_fused_out(GemmPlan* p, void* out_bf16, float* ss_out);
cudaError_t launch_gemm(const GemmPlan& p, cudaStream_t st);
cudaError_t prepare_gemm();  // per-device kernel attributes; call outside stream capture
void set_gemm_pair(int on);  // 1: CTA pairs (clusters of two sharing the W tile), 0: single-CTA tiles
int get_gemm_pair();
int get_gemm_max_clusters();  // co-resident CTA pairs of the pair kernel on the current device
cudaError_t launch_gemm_ref(const void* A, const void* W, int M, int N, int K, float* out, cudaStream_t st);

// ---- attention ----
struct AttnPlan {
  CUtensorMap tmQ;   // (B, T, 2d)  box (1, 128 rows, 64 cols)
  CUtensorMap tmK;   // (B, T, 2d)  box (1, 64 rows, 64 cols)
  CUtensorMap tmVT;  // (B, d, Tpad) box (1, 64 rows, 64 cols)
  void* out = nullptr;         // (B, T, d) bf16
  const float* rel = nullptr;  // (2*sat+1, H)
  const int32_t* frames = nullptr;  // (B) key length of every batch row (device); null: every row has T
  const int32_t* live = nullptr;    // (1) batch rows b >= live[0] do no work (device); null: every row is live
  int sat = 0, B = 0, T = 0, Tpad = 0, H = 0;
};
bool make_attn_plan(AttnPlan* p, const void* qk, const void* vT, void* out, const float* rel, int sat, int B, int T,
                    int Tpad, int H);
cudaError_t launch_attention(const AttnPlan& p, cudaStream_t st);

// ---- elementwise / gather ----
// codes_btc (B*T, C) int32 (or latents (B, K, T) fp32 when codes_btc is null) -> A (M, 3*Kp) bf16 = [hi | hi | lo] of the
// gathered latents, the A operand of the out_proj contraction; zeroes ss partials [zero_from, ss_parts) of every row.
// live (device, null = every row): rows at or past live[0] * T are not touched.
cudaError_t launch_embed_gather(const int32_t* codes_btc, const float* latents, const float* table, void* A, int M, int T,
                                int C, int V1, int K, int Kp, float* ss, int zero_from, int ss_parts,
                                const int32_t* live, cudaStream_t st);

// ---- generate-loop state kernels ----
// z (B,C,T) int64, mask (B,C,T) int32|null -> zcur (B,T,C) int32 (masked), zorig (B,T,C) int32;
// n0[g] = count(MASK) over the rows of group g (rowgrp null: every row is in group 0), n0 zeroed first for g < n_groups
cudaError_t launch_gen_init(const int64_t* z, const int32_t* mask, int32_t* zcur, int32_t* zorig, int32_t* n0,
                            const RowGroup* rowgrp, int n_groups, int B, int C, int T, int ncc, int mask_token,
                            cudaStream_t st);
// tokens (B, T, Cp) int32 + zorig cond -> out (B, C, T) int64
cudaError_t launch_gen_finish(const int32_t* tokens, const int32_t* zorig, int64_t* out, int B, int C, int T, int ncc,
                              cudaStream_t st);

// per-(step, group) dynamic scalars, read from DEVICE memory so that a captured CUDA graph can be replayed with
// new groupings / temperatures / seeds (the schedule values are computed on the host with the reference's fp32
// expressions: mask.py:8-9, transformer.py:831-834, 917-919).  The sampling kernels take a step's row of the table
// and read entry rowgrp[b].group for batch row b.
struct SampleDyn {
  float inv_temp, gamma, temp_eff;
  int do_sample, is_last, step;
  uint32_t seed_lo, seed_hi;
  float top_p;  // <= 0 or >= 1: disabled (reference transformer.py:1001-1016)
};
struct SampleArgs {
  const float* logits;  // (B*S, V)
  int32_t* zcur;        // (B, T, C) int32, predicted codebooks at c >= ncc ; updated in place by the remask kernel
  const int32_t* zorig; // (B, T, C) int32 or null (then conditioning codebooks are left untouched)
  int32_t* tokens;      // (B, T, Cp) sampled_z
  float* conf;          // (B, S)
  const int32_t* n0;    // (groups) initial mask count of each group
  const RowGroup* rowgrp;  // (B)
  int B, T, C, ncc, V, mask_token;
  const int32_t* live = nullptr;  // (1) device: batch rows b >= live[0] are idle and left untouched; null = all live
};
// use_top_p selects the kernel variant at launch time (it is baked into a captured graph: part of the graph key)
cudaError_t launch_sample_step_dev(const SampleArgs& a, const SampleDyn* dyn_dev, cudaStream_t st, bool use_top_p);
// fused path: the classifier's sampling epilogue wrote `partials`; picks the tile, writes tokens + confidences, re-masks
cudaError_t launch_sample_combine_dev(const SampleArgs& a, const void* partials, const SampleDyn* dyn_dev, cudaStream_t st);
// the re-mask alone (the second kernel of the launchers): reads a.tokens and a.conf, updates a.zcur
cudaError_t launch_remask_dev(const SampleArgs& a, const SampleDyn* dyn_dev, cudaStream_t st);
// a launch of nucleus (top-p) and plain groups after the split classifier epilogue: the combine serves the rows of plain
// groups from `partials`, the nucleus draw the rows of top-p groups from a.logits, then the re-mask
cudaError_t launch_sample_split_dev(const SampleArgs& a, const void* partials, const SampleDyn* dyn_dev, cudaStream_t st);

// ---- onset detection (onset.cu; librosa 0.10 onset_detect restated, DESIGN.md §9) ----
// peak_pick windows of onset_detect's defaults at (sr, hop), and the envelope's left padding lag + n_fft // (2 hop)
struct OnsetGeometry {
  int pre_max = 0, post_max = 0, pre_avg = 0, post_avg = 0, wait = 0, pad = 0;
};
OnsetGeometry onset_geometry(int sr, int hop);
// device tables (built on the host in float64 once per (device, sr, hop), then cached) and the peak_pick parameters
struct OnsetTables {
  const float2* twiddle;   // (1025) exp(-2 pi i k / 2048)
  const float* window;     // (2048) periodic Hann
  const float* mel_w;      // nonzero Slaney mel weights, band m at [mel_off[m], mel_off[m + 1])
  const int32_t* mel_off;  // (129)
  const int32_t* mel_lo;   // (128) first nonzero bin of band m
  int pre_max, post_max, pre_avg, post_avg, wait, pad;
  float delta;
};
cudaError_t onset_tables(int sr, int hop, OnsetTables* out);
// samples (B, N) fp32 -> db_ws (B, F, 128) mel dB, env (B, F) normalised envelope, onsets (B, F) + counts (B)
cudaError_t launch_onset_detect(const float* samples, int B, int N, int hop, const OnsetTables& t, float* db_ws,
                                float* env, int32_t* onsets, int32_t* counts, int backtrack, cudaStream_t st);
// mask (B, C, T) int64: 0 on onset row r's slices [idx - width : idx + width] (Python slice semantics), r = 0 when
// onset_rows == 1, else r = b; 1 elsewhere
cudaError_t launch_onset_mask(const int32_t* onsets, const int32_t* counts, int onset_rows, int F, int width,
                              int64_t* mask, int B, int C, int T, cudaStream_t st);
// samples (B, N) fp32 -> db (B, F, 128) mel dB: onset_spec_kernel alone (the first half of launch_onset_detect)
cudaError_t launch_onset_spec(const float* samples, int B, int N, int hop, const OnsetTables& t, float* db,
                              cudaStream_t st);

// ---- beat tracking (beat.cu; librosa 0.10.1 beat_track restated, DESIGN.md §10) ----
// the tempo estimate's autocorrelation window, W = int(8 sr) // hop lags, is supported for 2 <= W <= BEAT_MAX_LAGS
constexpr int BEAT_MAX_LAGS = 4096;
int beat_lags(int sr, int hop);
// device tables (float64, built on the host once per (device, sr, hop), then cached)
struct BeatTables {
  const double* window;    // (W) periodic Hann
  const double* bpm;       // (W) tempo_frequencies: inf, 60 sr / (hop k)
  const double* log2_bpm;  // (W)
  int W, max_idx;          // max_idx: the first lag below 320 BPM
};
cudaError_t beat_tables(int sr, int hop, BeatTables* out);
size_t beat_workspace_bytes(int B, int F);
// samples (B, N) fp32 -> env (B, F) fp32 onset strength (median over bands), tempo (B) BPM, beats (B, F) + counts (B)
cudaError_t launch_beat_track(const float* samples, int B, int N, int sr, int hop, const OnsetTables& ot,
                              const BeatTables& bt, double start_bpm, double tightness, int trim, void* workspace,
                              float* env, double* tempo, int32_t* beats, int32_t* counts, cudaStream_t st);
// the same decisions from a given envelope (B, F)
cudaError_t launch_beat_from_envelope(const float* env, int B, int F, int sr, int hop, const BeatTables& bt,
                                      double start_bpm, double tightness, int trim, void* workspace, double* tempo,
                                      int32_t* beats, int32_t* counts, cudaStream_t st);

// ---- pitch shift (pitch.cu; torch_pitch_shift's stft -> phase vocoder -> istft -> resample restated, DESIGN.md §11) ----
constexpr int PITCH_MIN_NFFT = 16, PITCH_MAX_NFFT = 4096;
// shapes of one call: F = 1 + (N + 2 (n_fft / 2) - n_fft) / hop STFT frames, F2 = ceil(F / rate) stretched frames (F when rate == 1), L the
// istft length, target the resampled length before the cut or pad to N
struct PitchPlan {
  int rows = 0, N = 0, sr = 0, new_freq = 0, n_fft = 0, hop = 0, nb = 0, F = 0, F2 = 0, nchunks = 0, width = 0;
  double rate = 1.0, base = 0.0, scale = 0.0;
  long long L = 0, target = 0, orig_g = 1, new_g = 1;
  bool stretch = false, resample = false;
};
// 0, or 1 when the stretched frame count is out of range
int pitch_plan(int rows, int N, int sr, int new_freq, int n_fft, int hop, double rate, PitchPlan* p);
size_t pitch_workspace_bytes(const PitchPlan& p);
// float64 forward (n_fft x 2 n_bins) and inverse (2 n_bins x n_fft) DFT bases, zero padded to the GEMM tiles; built on
// the host once per (device, n_fft), then cached
cudaError_t pitch_basis(int n_fft, const double** fwd, const double** inv);
// samples (rows, N) fp32 -> out (rows, N) fp32
cudaError_t launch_pitch_shift(const float* x, const PitchPlan& p, const double* fwd, const double* inv, void* ws,
                               float* out, cudaStream_t st);
// the vocoder's time steps: out[i] = float(rate) * float(i), i < n
cudaError_t launch_pitch_time_steps(float rate, long long n, float* out, cudaStream_t st);

// ---- validation metrics (validate.cu; train.py's val_loop loss and _metrics accuracies, DESIGN.md §12) ----
constexpr int XENT_MAX_V = 1024;
using XentRow = vnb_xent_row;
size_t xent_workspace_bytes(long long B, long long S);
// logits (B, S, V) fp32 -> rows (B * S) records
cudaError_t launch_xent_rows(const float* logits, const int64_t* z, int B, int C, int T, int ncc, int V, XentRow* rows,
                             cudaStream_t st);
// the records, then out (9) fp32 and, when not NULL, ambiguous (9) int32
cudaError_t launch_xent_metrics(const float* logits, const int64_t* z, const int64_t* mask, const double* r, int B,
                                int C, int T, int ncc, int V, double eps, void* workspace, float* out,
                                int32_t* ambiguous, cudaStream_t st);

}  // namespace vnb
