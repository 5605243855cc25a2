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
  int n_tree;      // rows of the verify pass (K + 1 for the chain)
  int d;
  size_t smem;
  size_t smem_ring;
  int cluster = 1; // CTAs per cluster of the ring kernel (1 or 2, dec_ring_cluster_size)
};

// ---- decode.cu ----
size_t dec_smem_bytes(int d, int ffn);
cudaError_t dec_configure(int d, size_t smem, size_t smem_ring);
size_t dec_ring_smem_bytes(int d);
void dec_build_program(int n_layers, int has_block, std::vector<int>& flat, int off[4]);
struct ChunkDesc;
void dec_build_chunk_table(const DecModel& hm, int ncta, std::vector<ChunkDesc>& tab, std::vector<int>& off);
cudaError_t dec_relayout_cross_kv(const __half* kv, __half* ck, __half* cv, int S, int S_pad, int d, int H, cudaStream_t s,
                                  int64_t* n_launch);
// {b'_n, c_n} of the LayerNorm-fed GEMMs of the ring kernel: float2 count for n_dec decoder layers, and the derivation
// from the bound weights (enqueued on s)
size_t dec_ln_fold_len(int n_dec, int d, int ffn);
cudaError_t dec_fold_layernorms(const DecModel& hm, int n_dec, float2* out, cudaStream_t s);
struct CtaStage;
void dec_build_stage_table(const DecModel& hm, const float2* ln_fold, int ncta, int cluster, std::vector<CtaStage>& tab);
cudaError_t dec_launch_iteration_ring(const DecModel* dm, const DecHostInfo& hi, bool profile, cudaStream_t s);
int dec_ring_cluster_size(const DecHostInfo& hi, int n_sm);
// phase: 0 = sweep A over T uncached rows, 1 = tail (candidates), 2 = verify sweep + accept
cudaError_t dec_enqueue_phase(const DecModel* dm, const DecHostInfo& hi, int phase, int T, cudaStream_t s, int64_t* n_launch);
cudaError_t dec_launch_iteration(const DecModel* dm, const DecHostInfo& hi, cudaStream_t s);

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
