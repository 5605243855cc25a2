// Shared device helpers and engine-internal types (sm_90a only).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#define WM_HEAD_DIM 64
#define WM_MAX_T 16          // max query rows of one decode pass (K+1 <= 16)
#define WM_MAX_DEC_LAYERS 40
#define WM_MAX_POS 512       // self-KV rows allocated per layer (448 + tree slack)
#define WM_CROSS_CHUNKS 8    // cross-attention key chunks per head (flash-decoding split)
#define WM_CH_MAX_KEYS 256   // keys per chunk (one ring slot; S = 1500 => at least 6 chunks per head: large-v2's 20 x 6 items are one wave on 132 SMs)
#ifndef WM_DEC_THREADS
#define WM_DEC_THREADS 352   // compute threads per decode CTA (11 warps; the ring kernel adds a producer warp -> 384 => 168 registers)
#endif

namespace wm {

struct StageInstr;

// Candidate tree of a branching `medusa_choices` (reference medusa_utils.py:305-421 generate_medusa_buffers; built by the
// host in wm_set_medusa_choices).  Nodes are numbered level by level; node 0 = the base-head token.  The engine holds at
// most WM_MAX_T nodes, WM_TREE_MAX_CAND root-to-leaf paths and WM_TREE_MAX_TOPK candidates per head.
#define WM_TREE_MAX_CAND 32
#define WM_TREE_MAX_TOPK 4
struct DecTree {
  int n_tree, n_cand;
  int depth[16];        // medusa_position_ids: level of the node
  int rank[16];         // which of its head's top-k tokens the node carries (tree_indices - first index of the level)
  int parent[16];       // parent node, -1 for the root
  int topk[16];         // k of level i (topk[0] = 1)
  unsigned int anc[16]; // bit j set: node j is the node itself or one of its ancestors (true tree attention)
  int retrieve[WM_TREE_MAX_CAND][16];   // retrieve_indices: path c -> node at depth j
};
// one ring chunk: `nrows` (<= 16) rows of `copy_bytes` each, row r read at src + r * row_bytes and written at
// slot + r * (slot row stride).  Weight chunks: rows of W (copy_bytes = d fp16); cross-attention chunks:
// nrows = 1, one contiguous block of K or V rows.
struct ChunkDesc {
  const void* src;
  uint32_t row_bytes;
  uint32_t nrows;
  uint32_t copy_bytes;
  uint32_t pad_;
};

// One stage of the persistent ring kernel, fully resolved for one CTA by the host (built once per
// model, [instruction][cta], 128 B each): the kernel never derives shapes, row ranges or pointers on
// the critical path -- it prefetches the next record into shared memory while the current stage runs.
struct alignas(16) CtaStage {
  int stage, mode, layer;   // StageId, pass mode, decoder layer
  int epi;                  // GEMM stages: epilogue kind
  int ln;                   // 1: the activations go through LayerNorm (gamma arrives via nx_g of the previous record; bias
                            //    points at the {b'_n, c_n} pairs of the folded beta / gamma, dec_fold_layernorms)
  int x_ld;                 // row stride of X in floats
  int x_rows_fixed;         // 0: the pass's T rows
  int n_begin, n_rows;      // W rows of this CTA
  int N, ldo, out_row0;
  int segs, seg, block;     // K split (FC2): segs > 1
  int pf_bias_lines;        // 128-byte lines of pf_bias
  const float* X;           // activation rows (fp32), already offset by x_row0 and the k segment
  const float* bias;        // [N] or null (LayerNorm stages: float2 [N])
  float* out;
  const float* nx_g;        // LayerNorm gamma of the NEXT instruction (null: it has none)
  const float* pf_bias;     // this CTA's bias slice of the next GEMM stage (L2 prefetch)
  int presplit;             // 1: X was written by its producer in the fp16 hi/lo operand format (no split pass;
                            //    LayerNorm stages: X = xg, the statistics come from the fp32 rows of x)
  int out_split;            // 1: the epilogue writes `out` in that format (the consumer is a presplit stage)
  float* out_gx;            // residual epilogues: also write nx_g o out in that format here (the next stage's xg)
  int x_role;               // staging of X in a 2-CTA cluster (XR_*): the host sets issue / receive only where both CTAs
                            //    of the pair stage the same rows (same X, x_ld, T rule, and both n_rows > 0)
  int pad_;
};
enum XRole { XR_OWN = 0, XR_ISSUE = 1, XR_RECEIVE = 2 };   // own copies / multicast to both CTAs / wait for the peer's multicast
static_assert(sizeof(CtaStage) == 128, "CtaStage must be one 128-byte line");

// Barrier over the WM_DEC_THREADS compute threads of a decode CTA.  The persistent ring kernel has
// one extra warp (the weight producer) that never joins it, hence a named barrier instead of
// __syncthreads(); in the 512-thread kernels it is simply "all threads".
__device__ __forceinline__ void cta_sync() { asm volatile("bar.sync 1, %0;" ::"n"(WM_DEC_THREADS) : "memory"); }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

__device__ __forceinline__ float gelu_erf(float x) {
  // HF ACT2FN["gelu"] = exact erf GELU
  return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f));
}
__device__ __forceinline__ float silu(float x) { return x / (1.0f + expf(-x)); }

// D(16x8,f32) += A(16x16,f16,row) * B(16x8,f16,col)
__device__ __forceinline__ void mma_16816(float* c, uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3,
                                          uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

__device__ __forceinline__ uint4 ldg_nc_v4(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}

// ---- cross-CTA data exchange without L1 invalidation -----------------------------------------
// Everything one decode CTA writes for another (activations, new K/V rows, partials, loop state) is
// READ with L2-coherent loads (ld.global.cg == __ldcg), never through L1.  The grid barrier and the
// last-arriver counters then only need RELEASE semantics on the arriving side (MEMBAR + RED/ATOM);
// no acquire fence, so no CCTL.IVALL: weights' LN/bias vectors, tables and local memory stay
// L1-resident across the ~230 barriers of an iteration.
__device__ __forceinline__ float ldcg_f(const float* p) { return __ldcg(p); }
__device__ __forceinline__ int ldcg_i(const int* p) { return __ldcg(p); }
__device__ __forceinline__ float2 ldcg_f2(const float* p) { return __ldcg(reinterpret_cast<const float2*>(p)); }
__device__ __forceinline__ float4 ldcg_f4(const float* p) { return __ldcg(reinterpret_cast<const float4*>(p)); }
__device__ __forceinline__ uint4 ldcg_u4(const void* p) { return __ldcg(reinterpret_cast<const uint4*>(p)); }
// Activation element (row base `row`, column n) in the fp16 hi/lo operand format of the ring kernel's GEMM stages:
// every float pair (k, k+1) occupies its 8 bytes as { half2 hi(k,k+1), half2 lo(k,k+1) } (decode_ring.cuh).
__device__ __forceinline__ void store_split(float* row, int n, float v) {
  __half* p = reinterpret_cast<__half*>(row) + (size_t)(n >> 1) * 4 + (n & 1);
  const __half h = __float2half_rn(v);
  p[0] = h;
  p[2] = __float2half_rn(v - __half2float(h));
}
__device__ __forceinline__ void red_add_release(unsigned int* p, unsigned int v) {
  asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned int atom_add_release(unsigned int* p, unsigned int v) {
  unsigned int old;
  asm volatile("atom.release.gpu.global.add.u32 %0, [%1], %2;" : "=r"(old) : "l"(p), "r"(v) : "memory");
  return old;
}

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem) {
  uint32_t s = (uint32_t)__cvta_generic_to_shared(smem);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(s), "l"(gmem));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;\n" ::"n"(N));
}

__device__ __forceinline__ void ldmatrix_x4(uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3, const void* smem) {
  uint32_t s = (uint32_t)__cvta_generic_to_shared(smem);
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];\n"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
               : "r"(s));
}
__device__ __forceinline__ void ldmatrix_x4_trans(uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3,
                                                  const void* smem) {
  uint32_t s = (uint32_t)__cvta_generic_to_shared(smem);
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];\n"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
               : "r"(s));
}

__device__ __forceinline__ void ldmatrix_x2_trans(uint32_t& r0, uint32_t& r1, const void* smem) {
  uint32_t s = (uint32_t)__cvta_generic_to_shared(smem);
  asm volatile("ldmatrix.sync.aligned.m8n8.x2.trans.shared.b16 {%0,%1}, [%2];\n" : "=r"(r0), "=r"(r1) : "r"(s));
}

__device__ __forceinline__ uint32_t pack_half2(float lo, float hi) {
  __half2 h = __floats2half2_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&h);
}

// ---------------------------------------------------------------------------------------
// decode-side model description (lives in device memory; kernels take a pointer to it)
// ---------------------------------------------------------------------------------------
struct DecLayer {
  const float *ln1_g, *ln1_b;
  const __half* qkv_w;  // [3d, d]   (q | k | v rows)
  const float* qkv_b;   // [3d]      (k part zero)
  const __half* o_w;    // [d, d]
  const float* o_b;
  const float *ln2_g, *ln2_b;
  const __half* cq_w;   // [d, d]
  const float* cq_b;
  const __half* co_w;   // [d, d]
  const float* co_b;
  const float *ln3_g, *ln3_b;
  const __half* fc1_w;  // [ffn, d]
  const float* fc1_b;
  const __half* fc2_w;  // [d, ffn]
  const float* fc2_b;
  __half* self_k;        // [WM_MAX_POS, d]
  __half* self_v;        // [WM_MAX_POS, d]
  const __half* cross_k;   // [H][S_pad][72]: 64 dims + 8 halfs of padding (the shared-memory row of the attention kernels)
  const __half* cross_v;   // [H][S_pad][72]
};

// Loop state of one stream (device memory; the host only reads it back at sync points).
struct DecState {
  int L;            // len(input_ids)
  int kv_len;       // cached self-attention positions before pass A
  int done;         // loop finished (EOS / max_length / max_iters)
  int n_iter;       // iterations executed
  int max_iters;    // 0 = unlimited
  int max_length;
  int eos, pad;
  int begin_index;
  int accept_last;
  int need_a;       // 1 => the newest token is not cached yet: run sweep A before the tail
  int prefill;      // 1 => this launch only runs sweep A over ids[kv_len .. L) (a 16-token chunk of a long prompt) and stops
  float temperature, post_thr, post_alpha;
  int tree_attn;    // tree mode: 1 = rows attend to their ancestors only (true tree attention), 0 = reference behaviour
  int keep_n;       // tree mode: K/V rows of the verify pass that survive (kept at rows L .. L+keep_n-1) ...
  int keep_src[WM_MAX_T];   // ... and the cache rows they come from (keep_src[j] >= L + j)
  int ids[WM_MAX_POS + 32];
  int cand[WM_MAX_T];            // tokens of the candidate tree nodes (chain: c0, head 1..K)
  int accept_hist[WM_MAX_POS];
  // per-row statistics written by the logits scan, consumed by the accept step
  int row_argmax[WM_MAX_T];
  float row_pc[WM_MAX_T];        // [n]: softmax prob of node n's token in the posterior of its parent row (chain: parent = n-1)
  float row_thr[WM_MAX_T];
};

struct alignas(16) DecModel {   // (copied to shared memory in 16-byte pieces by the ring kernel)
  int d, H, ffn, V, S, S_pad;
  int n_layers;      // decoder layers (without the medusa block)
  int has_block;     // 1 => layers[n_layers] is the medusa block
  int K;             // medusa heads
  int n_tree;        // rows of the verify pass: K+1 for the chain, tree nodes for branching medusa_choices
  int has_tree;      // 1 => branching choices: `tree` describes the candidate tree
  const DecTree* tree;
  float* topk_part;  // [WM_MAX_T rows][32 segments][WM_TREE_MAX_TOPK]{value, index}: per-segment top-k of the tail scan
  DecLayer layers[WM_MAX_DEC_LAYERS];
  const __half* embed;   // [V, d] (also proj_out)
  const float* pos;      // [max_target_positions, d]
  const float *lnf_g, *lnf_b;
  const __half* heads_w; // [(K+1) or K][d, d]
  const float* heads_b;
  const uint8_t* tok_mask;  // [V]: bit0 suppress, bit1 begin-suppress
  const float* pen_tab;     // [WM_MAX_POS + 32]: (factor^(L-start) - 1) as f32, 0 when inactive
  // activations (fp32)
  float* x;        // [WM_MAX_T, d] residual stream
  float* xg;       // [WM_MAX_T, d] gamma o x in the MMA operand format, for the LayerNorm GEMM that follows (ring kernel)
  float* q;        // [WM_MAX_T, d]
  float* attn;     // [WM_MAX_T, d]
  float* ffn_h;    // [WM_MAX_T, ffn]
  float* hidden;   // [WM_MAX_T, d]  final-LN output (block type: input of the block)
  float* head_h;   // [WM_MAX_T, d]
  float* carry;    // [d] final-LN hidden state of the newest cached token (input of the heads)
  float* cross_part;  // [H][WM_CROSS_CHUNKS][WM_MAX_T][WM_HEAD_DIM + 2]
  int cross_chunks;   // key chunks per head of the cross-attention stage: clamp(n_sm / H, 1, 8)
  unsigned int* cross_cnt;  // [H] arrival counters of the cross-attention chunks (last arriver combines)
  float* gemm_part;   // [8 k-segments][WM_MAX_T][d] partial sums of K-split GEMM stages (FC2)
  unsigned int* gemm_cnt;  // [n_sm] arrival counters of their row blocks (last arriver folds)
  float* sel_part;    // [WM_MAX_T][32 segments][4] partials of the logits scan
  int sel_nseg;       // vocabulary segments per row of the logits scan: clamp(n_sm / (K+1), 1, 32)
  float* logits_a;    // [WM_MAX_T, V]
  float* logits_b;    // [WM_MAX_T, V]
  // stage program of the persistent ring kernel: {stage, mode, layer} triples; lists [off[i], off[i+1])
  const struct StageInstr* prog;
  int prog_off[4];
  // per-CTA weight-chunk schedule of the ring producer (built by the host once the weights are bound):
  // chunk_tab[chunk_off[cta*4 + list] .. chunk_off[cta*4 + list + 1]) in consumption order
  const struct ChunkDesc* chunk_tab;
  const int* chunk_off;
  const struct CtaStage* stage_tab;   // [prog_off[3]][n_sm] resolved stage records of the ring kernel
  DecState* st;
  unsigned int* bar;  // grid-barrier words for the persistent kernel
  unsigned long long* prof;  // optional stage timeline [2 CTAs][n_instr][3] (ns), null = off
};

}  // namespace wm
