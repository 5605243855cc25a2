// Engine-internal launcher declarations (host side). Not part of the public C ABI.
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <vector>

namespace wm {

struct DecModel;

struct DecHostInfo {
  int n_sm;
  int H, K, n_layers, has_block;
  int n_head_layers;   // MedusaResBlocks per head
  int n_tree;      // rows of the verify pass (K + 1 for the chain)
  int d;
  size_t smem;
  size_t smem_ring;
  int cluster = 1; // CTAs per cluster of the ring kernel (1 or 2, dec_ring_cluster_size)
  int lp = 0;      // 1: logits processors on for the iterations enqueued next (the ring kernel's variant with them)
  int smp = 0;     // 1: a sampled attempt (wm_set_sampling): the ring kernel's variant with the sampled scans and folds
};

// ---- decode.cu ----
size_t dec_smem_bytes(int d, int ffn);
cudaError_t dec_configure(int d, size_t smem, size_t smem_ring);
size_t dec_ring_smem_bytes(int d);
void dec_build_program(int n_layers, int has_block, int n_head_layers, std::vector<int>& flat, int off[4]);
cudaError_t dec_relayout_cross_kv(const __half* kv, __half* ck, __half* cv, int S, int S_pad, int d, int H, cudaStream_t s,
                                  int64_t* n_launch);
// {b'_n, c_n} of the LayerNorm-fed GEMMs of the ring kernel: float2 count for n_dec decoder layers, and the derivation
// from the bound weights (enqueued on s)
size_t dec_ln_fold_len(int n_dec, int d, int ffn);
cudaError_t dec_fold_layernorms(const DecModel& hm, int n_dec, float2* out, cudaStream_t s);
struct CtaStage;
struct ChunkDesc;
// the ring kernel's stage records [instruction][cta] and per-CTA chunk schedule (chunk_off: 4 per CTA), for a grid of
// ncta CTAs in clusters of `cluster`
void dec_build_ring_tables(const DecModel& hm, const float2* ln_fold, int ncta, int cluster, std::vector<CtaStage>& stab,
                           std::vector<ChunkDesc>& ctab, std::vector<int>& off);
// host replay of the ring protocol over every launch state (wm_ring_schedule_check)
int dec_check_ring_schedule(const DecModel& hm, int ncta, long long l2_budget, int first[4]);   // l2_budget < 0: as built
cudaError_t dec_launch_iteration_ring(const DecModel* dm, const DecHostInfo& hi, bool profile, cudaStream_t s);
int dec_ring_cluster_size(const DecHostInfo& hi, int n_sm);
// phase: 0 = sweep A over T uncached rows, 1 = tail (candidates), 2 = verify sweep + accept
cudaError_t dec_enqueue_phase(const DecModel* dm, const DecHostInfo& hi, int phase, int T, cudaStream_t s, int64_t* n_launch);
cudaError_t dec_launch_iteration(const DecModel* dm, const DecHostInfo& hi, cudaStream_t s);

// ---- scores.cu ----
#define WM_SCORE_NSEG 16       // vocabulary segments per scored row (fixed: the fold order does not depend on the grid)
#define WM_SCORE_THREADS 512
#define WM_SCORE_UNROLL 4      // elements per thread loaded together (one segment of large-v2's vocabulary: 2 steps)
struct DecState;
struct DecTree;
// What the scoring kernel reads and writes; one launch after each speculative iteration while scoring is on.
struct ScoreArgs {
  const float* logits_a;   // [K+1][V] raw rows of the tail (row 0: the base row c0 was chosen from)
  const float* logits_b;   // [n_tree][V] raw verify rows
  const DecState* st;
  const DecTree* tree;     // null for a chain
  const uint8_t* tok_mask;
  const float* pen_tab;
  const float* adj;        // logits-processor term of the iteration (dec_state_adj), null = processors off
  int V;
  int n_prompt;            // first position scored (prefill launches of a long prompt are not scored)
  int want_lp, want_rows;  // option "scores" bit 0 / bit 1
  int* state;              // {iterations scored, cursor = first unscored position, arrivals}; zero at the start of a call
  float* part;             // [WM_MAX_T + 1][WM_SCORE_NSEG]{max, sum of exp(v - max)}, then [WM_MAX_T + 1] token logits
  float* lp;               // [WM_MAX_POS + 32]: log-probability of the token at each position
  float* rows;             // [cap_rows][V]: processed verify row path[accept] of each iteration
  int cap_rows;
  int tau;                 // 1: a sampled attempt with top-k: token rows are restricted to {v >= tau} (DecState tail_tau,
                           // row_tau), as HF's log_softmax of the warped scores at temperature 1
};
int dec_score_grid(int n_cta, int K);
cudaError_t dec_launch_scores(const ScoreArgs& a, int grid, cudaStream_t s);
// Gumbel noise of a sampled attempt (sample_gumbel) at position n for tokens j0 .. j0 + count - 1 (wm_sample_noise)
cudaError_t dec_launch_sample_noise(const unsigned int key[2], unsigned int window, unsigned int attempt, int n, int j0,
                                    int count, float* out, cudaStream_t s);

// ---- logits_proc.cu ----
#define WM_LP_THREADS 256
#define WM_LP_MAX_SEQS 256       // multi-token sequences of sequence_bias + bad_words_ids (wm_set_logits_processors)
#define WM_LP_MAX_TOKENS 4096    // their tokens in all
// What the logits-processor kernel reads and writes; one launch before each speculative iteration while processors are
// on.  adj[j] = base[j] + the values of the multi-token sequences whose prefix ends the sequence (in table order), or
// -inf for a no-repeat-n-gram ban or the EOS ban of min_length / min_new_tokens.
struct LogitsProcArgs {
  const DecState* st;
  float* base;             // [V] single-token biases (sums in table order; -inf for a banned token)
  int* seq_tok;            // multi-token sequences, flattened
  int* seq_off;            // [n_seq + 1]
  float* seq_val;          // [n_seq] bias, or -inf for a bad word
  int n_seq;
  int ngram;               // no_repeat_ngram_size, 0 = off
  int eos_min_len;         // EOS is banned while len(input_ids) < eos_min_len
  int V;
  float* adj;              // [V]
};
int dec_logits_proc_grid(int n_cta);
cudaError_t dec_launch_logits_proc(const LogitsProcArgs& a, int grid, cudaStream_t s);

// ---- no_speech.cu ----
#define WM_NS_NSEG 512         // vocabulary segments of the no-speech row (fixed: the fold order does not depend on the grid)
#define WM_NS_THREADS 512
// The base-head logits of the captured SOT row and their log-sum-exp; launched once after the loop when capture is on.
struct NoSpeechArgs {
  const float* hidden;     // [d] final-LayerNorm row captured by the loop (DecModel::ns_hidden)
  const __half* head_w;    // base_head type: head 0 [d, d] (the row goes through it first); null for medusa_block
  const float* head_b;     // [d]
  int head_layers;         // base_head type: layers of head 0; layer l's weights at head_w + l * head_stride * d and
  size_t head_stride;      // head_b + l * head_stride (head_stride = (K + 1) d rows per layer)
  float* head_out;         // [2][d] base_head type: x + SiLU(W_l . x + b_l) after each layer l, in half l % 2
  const __half* embed;     // [V, d] proj_out (tied)
  int d, V;
  float* logits;           // [V] raw logits
  float* part;             // [WM_NS_NSEG]{max, sum of exp(v - max)}
  float* lse;              // [1] log-sum-exp of the row
  unsigned int* count;     // arrival counter (zero between launches)
};
// grid: CTAs of each launch (<= decode_ctas); enqueues head_layers + 1 kernels for the base_head type (each layer of
// head 0, then the vocabulary product), 1 for medusa_block, and adds them to *n_launch
cudaError_t dec_launch_no_speech(const NoSpeechArgs& a, int grid, cudaStream_t s, int64_t* n_launch);

// ---- timestamps.cu ----
#define WM_TS_MAX_FILTER 31    // widest median filter
#define WM_TS_MAX_N 448        // DTW rows (the trace of 448 x 1500 cells is 168 KB of shared memory)
#define WM_TS_MAX_F 1500       // DTW columns
// Row softmax of captured scores: probs[head][i][0..S) for rows row0 .. row0 + N - 1 of the slot of each listed head.
struct TsSoftmaxArgs {
  const float* scores;     // TsCapture::scores [slots][WM_TS_ROWS][S]
  const int* head_slot;    // [n_heads] device: slot of each listed (layer, head) pair, duplicates allowed
  int n_heads, S, row0, N;
  float* probs;            // [n_heads][N][S]
};
cudaError_t ts_launch_softmax(const TsSoftmaxArgs& a, cudaStream_t s);
// Normalise, median-filter, average over heads, DTW and backtrace (HF _extract_token_timestamps after the crop).
struct TsExtractArgs {
  float* probs;            // [n_heads][N][ldp]: row probabilities; columns < F are normalised in place
  int ldp, n_heads, N, F, filter;
  double time_precision;
  float* matrix;           // [N][F]
  int* jumps;              // [N]: frame of the first DTW cell of each row (-1 when the path enters the row at frame 0)
  float* times;            // [N + 1]: f32(jump * time_precision), then the last one repeated
};
size_t ts_dtw_smem_bytes(int N, int F);
// enqueues 3 kernels (1 when F = 0) and adds them to *n_launch (may be null)
cudaError_t ts_launch_extract(const TsExtractArgs& a, cudaStream_t s, int64_t* n_launch);

// ---- mel.cu ----
// pcm: device f32 [480000] (already zero padded). Outputs: mel_f32 [80][3000], xT fp16 [rows>=3000+?][80]
// time-major with one leading zero row (conv padding); gmax_bits: device scratch (1 int).
cudaError_t mel_forward(const float* pcm, const float* filters /*[201][80]*/, float* mel_f32, __half* x_tm,
                        int* gmax_bits, cudaStream_t s, int64_t* n_launch);
// mel given by the caller: mel_f32 [80][3000] device -> x_tm
cudaError_t mel_to_time_major(const float* mel_f32, __half* x_tm, cudaStream_t s, int64_t* n_launch);

// ---- resample.cu ----
constexpr int kResampleMaxRate = 1 << 20;   // largest rate after dividing both rates by their gcd
// Polyphase table of one rate pair (host side).  taps [nw][max_taps] row-major, phase p uses taps[p][0 .. n[p]) on
// padded input columns lo[p] .. lo[p] + n[p] of its block; [dlo, dhi): input reach of output o relative to
// floor(o * orig / nw).
struct ResampleTable {
  int orig = 0, nw = 0, width = 0, max_taps = 0;
  int64_t dlo = 0, dhi = 0;
  std::vector<float> taps;
  std::vector<int> lo, n;
};
bool resample_build_table(int orig_hz, int new_hz, ResampleTable& t);
int64_t resample_out_len(int64_t n_in, const ResampleTable& t);
// outputs per CTA (0: the input span of 32 outputs does not fit the staging buffer) and its shared-memory bytes
int resample_block_outputs(const ResampleTable& t, size_t* smem_bytes);
// taps_dev [max_taps][nw] (the transpose of ResampleTable::taps); sup_dev [nw] {lo - width, n}
cudaError_t resample_launch(const float* x, int64_t n_in, float* y, int64_t n_out, const float* taps_dev,
                            const int2* sup_dev, const ResampleTable& t, int T, size_t smem, cudaStream_t s);

// ---- enc_gemm.cu ----
enum EncEpi { ENC_EPI_BIAS_F16 = 0, ENC_EPI_BIAS_GELU_F16 = 1, ENC_EPI_BIAS_RES_F32 = 2, ENC_EPI_BIAS_GELU_POS_F32 = 3 };
struct EncGemmArgs {
  const __half* A; int lda;     // [M_pad, K] fp16, row stride lda (elements)
  const __half* W;              // [N, K] fp16
  const float* bias;            // [N]
  int M, N, K;                  // M valid rows; N % 128 == 0; K % 32 == 0
  int epi;
  __half* out16; int ldo16;     // fp16 outputs
  float* out32; int ldo32;      // fp32 residual stream (+=) or plain store
  const float* pos;             // [M, N] added after GELU (conv2)
  __half* vt; int vt_col0, vt_ld;   // wgmma GEMM, ENC_EPI_BIAS_F16 only: columns >= vt_col0 also written transposed
                                    // (vt[col - vt_col0][row], row stride vt_ld): V^T for the wgmma attention
  __half* ck; __half* cv; int kv_spad;   // wgmma GEMM, ENC_EPI_BIAS_F16 only: the output [pos][k | v] (N = 2 d) goes to the
                                         // decode layout cross_k / cross_v [head][kv_spad][72] instead of out16
  int tile;                     // wgmma GEMM: 0 = tile shape picked per GEMM, 1 = 128 x 128 tiles only (cross-check)
  int pdl;                      // wgmma GEMM: launch with programmatic stream serialization (tc_common.cuh)
};
cudaError_t enc_gemm(const EncGemmArgs& a, cudaStream_t s, int64_t* n_launch);
cudaError_t enc_gemm_configure();
// LayerNorm rows of fp32 x [M, d] -> fp16 y [M, d] (and optional fp32 copy)
// (pdl: launched with programmatic stream serialization, see tc_common.cuh)
cudaError_t enc_layernorm(const float* x, const float* g, const float* b, __half* y16, float* y32, int M, int d,
                          cudaStream_t s, int64_t* n_launch, bool pdl = false);

// ---- enc_gemm_tc.cu (wgmma + TMA) ----
cudaError_t enc_gemm_tc(const EncGemmArgs& a, int a_rows, cudaStream_t s, int64_t* n_launch);
cudaError_t enc_gemm_tc_configure();
// tile shape {rows, columns, ring stages} the wgmma GEMM picks for an M x N x K product (host logic only)
void enc_gemm_tc_tile(int M, int N, int K, bool fp16_out, int n_sm, int out[3]);

// ---- enc_attn.cu ----
// qkv: fp16 [S_pad, 3d] (q pre-scaled | k | v); out: fp16 [S_pad, d]; full (non-causal) attention over S keys
cudaError_t enc_attention(const __half* qkv, __half* out, int S, int d, int H, cudaStream_t s, int64_t* n_launch);

// ---- enc_attn_tc.cu (wgmma + TMA) ----
// qkv as above; vt: scratch fp16 [d][S_pad] (V transposed, written here); out: fp16 [S_pad, d]
// vt_ready: the QKV GEMM already wrote V^T (EncGemmArgs::vt); otherwise a transpose kernel runs first
cudaError_t enc_attention_tc(const __half* qkv, __half* vt, __half* out, int S, int S_pad, int d, int H, bool vt_ready,
                             cudaStream_t s, int64_t* n_launch, bool pdl = false);
cudaError_t enc_attention_tc_configure();

}  // namespace wm
