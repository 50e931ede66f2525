// vampnet_b200 — internal launcher declarations shared by the .cu translation units.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <functional>
#include <type_traits>
#include <vector>

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

// Workspaces and tables are laid out as 256-byte aligned blocks: carve(o, bytes) returns the block's offset o and moves
// o past it to the next 256-byte boundary, so after the last block o is the total size.
inline size_t align256(size_t n) { return (n + 255) & ~(size_t)255; }
inline size_t carve(size_t& o, size_t bytes) {
  const size_t at = o;
  o = align256(o + bytes);
  return at;
}

// Constant device tables (tables.cu): the table named by `key` (its kind, then the parameters its values depend on) is
// built on the host by `build` once per (current device, key), uploaded, and kept for the life of the process; *dev
// receives its device copy.
enum TableKind { TABLE_FFT, TABLE_MEL_BANK, TABLE_BEAT, TABLE_PITCH_BASIS, TABLE_VGGISH_FFT, TABLE_VGGISH_HTK };
cudaError_t device_table(const std::vector<double>& key, const std::function<std::vector<char>()>& build,
                         const char** dev);

// ---- TMA tensor maps (driver entry point fetched at run time; no link-time libcuda dependency) ----
// 2-D bf16 row-major (rows, cols) with a (box_rows x 64) box, 128B swizzle.
bool make_tmap_2d(CUtensorMap* tm, const void* base, uint64_t rows, uint64_t cols, uint32_t box_rows,
                  uint32_t box_cols);
// 3-D bf16 (batch, rows, cols) row-major with row pitch `pitch_elems`; box (1, box_rows, 64), 128B swizzle.
bool make_tmap_3d(CUtensorMap* tm, const void* base, uint64_t batch, uint64_t rows, uint64_t cols,
                  uint64_t pitch_elems, uint32_t box_rows, uint32_t box_cols);
// 4-D bf16 NHWC images (batch, H, W, C); box (1, box_h, W, box_c) of whole image rows, 128B swizzle.
bool make_tmap_4d(CUtensorMap* tm, const void* base, uint64_t batch, uint64_t H, uint64_t W, uint64_t C,
                  uint32_t box_h, uint32_t box_c);
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
// The arguments every GEMM kernel takes by value (gemm_wgmma.cu).
struct GemmArgs {
  int M, N, K;
  int epi;
  void* out;          // see VNB_EPI_*
  void* out2;         // vT for EPI_QKV
  const float* bias;  // EPI_BIAS_F32
  int T, Tpad;        // EPI_QKV: rows m = b*T + t
  int d2;             // EPI_QKV: 2*d_model (column where V starts)
  // ---- fused RMSNorm (reference transformer.py:43-58), see DESIGN.md §4 ----
  __nv_bfloat16* out_bf16;  // EPI_RESID / EPI_BIAS_F32: bf16 copy of the fp32 output (A operand of the next GEMM)
  float* ss_out;            // partial row sums of squares of the fp32 output, part p at [p * M + row]: EPI_RESID
                            // (N/128, M), parts 2j / 2j+1 = even / odd 32-column chunks of n-tile j; EPI_BIAS_F32
                            // (N/256, M), one part per n-tile
  const float* ss_in;       // consumers: partial row sums of squares of THEIR A operand; null = no row scaling
  int ss_parts;             // number of partials to add (fixed order: deterministic)
  float inv_d, eps;         // row scale = rsqrt(sum * inv_d + eps)
  // ---- EPI_SAMPLE (the classifier of the generate loop): the logits are sampled in the epilogue, not stored ----
  const int32_t* zcur;      // (B, T, C) current tokens: only still-masked positions are sampled
  const SampleDyn* dyn;     // this step's row of the (step, group) table (device memory: graph replay safe)
  const RowGroup* rowgrp;   // (B) group of every batch row
  float4* partials;         // (M * Cp * V/128) records, see sample_combine_kernel
  int C, ncc, V, mask_token;
  // ---- adapted variants of QKV / RESID / GEGLU (null table: the plain kernel): acc += u[row] . B'[col] for adapted
  // rows, see lora_update() ----
  AdapterRefs lora;
  const int32_t* frames;    // EPI_QKV: (B) frames of every batch row, null = T; v^T columns t >= frames[b] get 0
  // ---- launches of calls with different step counts: batch rows >= *live (rows >= *live * T) are idle this iteration;
  // a tile wholly past them does no work, null = every row is live ----
  const int32_t* live;
};
struct GemmPlan {
  CUtensorMap tmA, tmB;  // A (M,K) bf16, W (N,K) bf16
  CUtensorMap tmBh;  // W with a 128-row box: the half tile each CTA of a pair fetches and multicasts (gemm_wgmma.cu, PAIR)
  // EPI_SAMPLE in a launch of nucleus (top-p) and plain groups: the rows of nucleus groups store their logits to `out`
  // (the materialising epilogue's layout, still-masked positions only) and leave no records
  bool sample_split = false;
  GemmArgs args{};
};
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

// ---- spectrogram tables (mel.cu): built in float64, rounded to the kernel's scalar type R once, cached by device_table ----
template <typename R>
using Complex = typename std::conditional<std::is_same<R, double>::value, double2, float2>::type;
template <typename R>
struct FftTablesT {
  const Complex<R>* twiddle;  // (n_fft / 2 + 1) exp(-2 pi i k / n_fft), for fft.cuh
  const R* window;            // (n_fft) periodic Hann (VGGish: of length 400, zero-extended)
};
using FftTables = FftTablesT<float>;
cudaError_t fft_tables(int n_fft, FftTables* out);  // per (device, n_fft)
// a filterbank's nonzero ranges: librosa.filters.mel(sr, n_fft, n_mels, fmin, fmax, htk=False, norm="slaney",
// dtype=float32) for the fp32 modes, VGGish's HTK matrix for VGGISH_LOG
template <typename R>
struct MelBankT {
  const R* w;           // band m's weights at [off[m], off[m + 1]), for bins lo[m], lo[m] + 1, ...
  const int32_t* off;   // (n_mels + 1)
  const int32_t* lo;    // (n_mels) first nonzero bin of band m (0 for an empty band)
};
using MelBank = MelBankT<float>;
cudaError_t mel_filterbank(int sr, int n_fft, int n_mels, double fmin, double fmax, MelBank* out);  // per (device, all)

// The spectrogram kernel's outputs from samples (rows, N) fp32:
//   ONSET_DB    onset detection's: F = 1 + N / hop frames, zero padding (any N >= 1), ONSET_NFFT points, |X|^2 on
//               ONSET_NMELS bands, then 10 log10(max(1e-10, s)); (rows, F, ONSET_NMELS)
//   MEL_MAG     the mel distance's: F = 1 + N / hop frames, reflect padding (N > n_fft / 2), n_fft a power of two in
//               MEL_MIN_NFFT..MEL_MAX_NFFT, |X| on n_mels bands; (rows, n_mels, F)
//   VGGISH_LOG  VGGish's log-mel examples (fad.cu), in float64: no padding, a VGGISH_WIN-point window in a VGGISH_NFFT-point
//               FFT, hop VGGISH_HOP, |X| on the VGGISH_NMELS-band HTK matrix, log(s + 0.01) rounded to fp32 once; the
//               first n_ex(N) * VGGISH_EX_FRAMES frames of each row, (rows * n_ex, VGGISH_EX_FRAMES, VGGISH_NMELS)
enum class SpecMode { ONSET_DB, MEL_MAG, VGGISH_LOG };
constexpr int ONSET_NFFT = 2048, ONSET_NMELS = 128;
constexpr int VGGISH_SR = 16000, VGGISH_WIN = 400, VGGISH_HOP = 160, VGGISH_NFFT = 512, VGGISH_NMELS = 64;
constexpr int VGGISH_EX_FRAMES = 96;
constexpr double VGGISH_FMIN = 125.0, VGGISH_FMAX = 7500.0;
// examples of N samples at 16 kHz: 1 + (F - 96) // 96 with F = 1 + (N - 400) // 160 frames; 0 below 15600 samples
inline int vggish_examples(long long N) {
  if (N < VGGISH_WIN) return 0;
  const long long F = 1 + (N - VGGISH_WIN) / VGGISH_HOP;
  return F < VGGISH_EX_FRAMES ? 0 : (int)(1 + (F - VGGISH_EX_FRAMES) / VGGISH_EX_FRAMES);
}
cudaError_t launch_spectrogram(SpecMode mode, const float* samples, int rows, int N, int hop, int n_fft,
                               const FftTables& fft, const MelBank& bank, int n_mels, float* out, cudaStream_t st);

// ---- onset detection (onset.cu; librosa 0.10 onset_detect restated, DESIGN.md §9) ----
// peak_pick windows of onset_detect's defaults at (sr, hop), and the envelope's left padding lag + n_fft // (2 hop)
struct OnsetGeometry {
  int pre_max = 0, post_max = 0, pre_avg = 0, post_avg = 0, wait = 0, pad = 0;
};
OnsetGeometry onset_geometry(int sr, int hop);
// the cached FFT tables and Slaney bank at (sr, ONSET_NFFT, ONSET_NMELS), and the peak_pick parameters
struct OnsetTables {
  FftTables fft;
  MelBank bank;
  OnsetGeometry g;
  float delta;
};
cudaError_t onset_tables(int sr, int hop, OnsetTables* out);
size_t onset_workspace_bytes(int B, int F);
// samples (B, N) fp32 -> db_ws (B, F, 128) mel dB, env (B, F) normalised envelope, onsets (B, F) + counts (B)
cudaError_t launch_onset_detect(const float* samples, int B, int N, int hop, const OnsetTables& t, float* db_ws,
                                float* env, int32_t* onsets, int32_t* counts, int backtrack, cudaStream_t st);
// mask (B, C, T) int64: 0 on onset row r's slices [idx - width : idx + width] (Python slice semantics), r = 0 when
// onset_rows == 1, else r = b; 1 elsewhere
cudaError_t launch_onset_mask(const int32_t* onsets, const int32_t* counts, int onset_rows, int F, int width,
                              int64_t* mask, int B, int C, int T, cudaStream_t st);

// ---- beat tracking (beat.cu; librosa 0.10.1 beat_track restated, DESIGN.md §10) ----
// the tempo estimate's autocorrelation window, W = int(8 sr) // hop lags, is supported for 2 <= W <= BEAT_MAX_LAGS
constexpr int BEAT_MAX_LAGS = 4096;
int beat_lags(int sr, int hop);
// device tables (float64, built on the host once per (device, sr, hop), then cached by device_table)
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
// 0; 1 when the stretched frame count is out of range, 2 when the istft length L is 0 (even n_fft, F2 = 1)
int pitch_plan(int rows, int N, int sr, int new_freq, int n_fft, int hop, double rate, PitchPlan* p);
// the workspace of one call, as byte offsets: spectrum (then (|X|, angle) in place), the stretched spectrum and the
// vocoder's chunk sums (rate != 1 only; stretched == spec otherwise), the inverse-DFT frames, the overlap-added signal
struct PitchLayout {
  size_t spec = 0, stretched = 0, chunk = 0, frames = 0, y = 0, total = 0;
};
PitchLayout pitch_layout(const PitchPlan& p);
size_t pitch_workspace_bytes(const PitchPlan& p);
// float64 forward (n_fft x 2 n_bins) and inverse (2 n_bins x n_fft) DFT bases, zero padded to the GEMM tiles; built on
// the host once per (device, n_fft), then cached by device_table as one table
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

// ---- mel spectrogram and multi-scale mel distance (mel.cu; audiotools' MelSpectrogramLoss restated, DESIGN.md §13) ----
constexpr int MEL_MIN_NFFT = 32, MEL_MAX_NFFT = 4096, MEL_MAX_MELS = 4096, MEL_MAX_SCALES = 16;
struct MelScalePlan {
  int n_fft = 0, hop = 0, n_mels = 0, F = 0;  // F = 1 + N / hop frames
  double fmin = 0.0, fmax = 0.0;
  long long elems = 0;  // C * n_mels * F: one item's spectrogram
  int chunks = 0;       // reduction CTAs per item
  size_t partial = 0;   // first of this scale's (B, chunks) partial sums in the workspace's partial array
};
struct MelLossPlan {
  int B = 0, C = 0, N = 0, sr = 0, n_scales = 0;
  MelScalePlan s[MEL_MAX_SCALES];
  size_t x_spec = 0, y_spec = 0, partials = 0, items = 0, total = 0;  // workspace byte offsets and size
};
MelLossPlan mel_loss_plan(int B, int C, int N, int sr, const vnb_mel_scale* scales, int n_scales);
// samples (rows, N) fp32 -> out (rows, n_mels, F) fp32 |STFT| projected on the Slaney filterbank
cudaError_t launch_mel_spectrogram(const float* samples, int rows, int N, int sr, const vnb_mel_scale& s, float* out,
                                   cudaStream_t st);
// loss (1) and, when not null, item_loss (B): fp32, formed in float64 and rounded once
cudaError_t launch_mel_loss(const float* x, const float* y, const MelLossPlan& p, double clamp_eps, double pow,
                            double log_weight, double mag_weight, void* workspace, float* loss, float* item_loss,
                            cudaStream_t st);

// ---- Frechet audio distance with VGGish embeddings (fad.cu, conv_wgmma.cu, mel.cu; DESIGN.md §14) ----
// samples (rows, N) fp32 at 16 kHz -> (rows * vggish_examples(N), 96, 64) fp32 log-mel examples (SpecMode::VGGISH_LOG)
cudaError_t launch_vggish_frontend(const float* samples, int rows, int N, float* out, cudaStream_t st);
// layer 1: examples (Bn, 96, 64) fp32, w (64, 9) fp32 -> relu, 2x2 max-pool -> (Bn, 48, 32, 64) hi/lo bf16
cudaError_t launch_vggish_in(const float* x, const float* w, const float* bias, int Bn, void* out_hi, void* out_lo,
                             cudaStream_t st);
// layers 2-9 on the tensor cores (conv_wgmma_kernel's CT_RELU / CT_RELU_POOL / CT_GENERIC modes)
cudaError_t launch_vggish_tc(const void* a_hi, const void* a_lo, int Bn, int H, int W, int Cin, const void* w_hi,
                             const void* w_lo, int N, const float* bias, bool relu, bool pool, void* out_hi,
                             void* out_lo, float* out_f32, cudaStream_t st);
// the embedding network's weights, as vnb_vggish_weights holds them
struct VggishNet {
  const float* w1; const float* b1;
  const void* conv_hi[5]; const void* conv_lo[5]; const float* conv_b[5];
  const void* fc_hi[3]; const void* fc_lo[3]; const float* fc_b[3];
};
size_t vggish_workspace_bytes(int n_ex);
// examples (n_ex, 96, 64) fp32 -> embeddings (n_ex, 128) fp32
cudaError_t launch_vggish_embed(const VggishNet& net, const float* examples, int n_ex, void* workspace, float* out,
                                cudaStream_t st);
// embeddings (M, 128) fp32 -> mu (128) and sigma (128, 128) float64, np.mean and np.cov(rowvar=False)
cudaError_t launch_fad_moments(const float* emb, long long M, double* mu, double* sigma, cudaStream_t st);

}  // namespace vnb
