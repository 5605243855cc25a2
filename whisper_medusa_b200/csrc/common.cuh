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

// Candidate tree of a branching `medusa_choices` (reference medusa_utils.py:305-421 generate_medusa_buffers; built by the
// host in wm_set_medusa_choices).  Nodes are numbered level by level; node 0 = the base-head token.  The engine holds at
// most WM_MAX_T nodes, WM_TREE_MAX_CAND root-to-leaf paths and WM_TREE_MAX_TOPK candidates per head.
#define WM_TREE_MAX_CAND 32
#define WM_TREE_MAX_TOPK 4
// largest top_k of a sampled attempt other than 0 (the whole row); HF's default is 50
#define WM_SMP_MAX_TOPK 64
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
// nrows = 0: a self-attention prefix block whose size is known only at launch (sa_prefix_chunk): src = the layer's
// self_k or self_v cache, block sa_block of the keys of the CTA's sa_item-th item in a pass of mode sa_mode.
struct ChunkDesc {
  const void* src;
  uint32_t row_bytes;
  uint32_t nrows;
  uint32_t copy_bytes;
  uint16_t sa_item;
  uint8_t sa_mode, sa_block;
};
// The largest ring slot of any width (RingGeom<1280>::SLOT_BYTES: 16 rows of the 1280 x 2 + 64-byte ring row stride),
// so no chunk is larger.  A nonzero L2 lookahead of the ring producer must hold at least this much.
#define WM_RING_SLOT_MAX (16 * (1280 * 2 + 64))

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

// Self-attention K/V cache of a decoder layer: [H][WM_MAX_POS][72] fp16, head-major like the cross-attention K/V.  The
// keys [0, n) of one head are one contiguous byte range (one bulk copy into a ring slot), and rows 144 B apart keep
// the 16-byte shared-memory reads of the attention's per-thread dot products free of bank conflicts.
#define WM_KV_ROW 72
// element (position p, channel c = head * 64 + dim) of a self-K/V cache
__host__ __device__ __forceinline__ size_t self_kv_index(int p, int c) {
  return ((size_t)(c >> 6) * WM_MAX_POS + p) * WM_KV_ROW + (c & 63);
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
  __half* self_k;        // [H][WM_MAX_POS][72]: head-major, 64 dims + 8 halfs of padding per row (self_kv_index)
  __half* self_v;        // [H][WM_MAX_POS][72]
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
  int path_node;    // tree mode: node path[accept] of the best candidate of the last iteration (read by the scoring kernel)
  // logits processors (wm_set_logits_processors): the address of the iteration's adj[V] (dec_state_adj), written by
  // logits_proc.cu before each iteration; 0 = off for the whole call (the logits scans then run their variant without
  // it).  Kept here rather than in DecModel, whose size the ring kernel's shared-memory copy depends on, and as two
  // 32-bit words so that DecState keeps its 4-byte alignment (with an 8-byte member the loop kernels compile to
  // different register allocations).
  unsigned int adj_lo, adj_hi;
  // sampled attempt of temperature fallback (wm_set_sampling; smp_on = 0: off, the loop chooses argmaxes).  Gumbel-max
  // with counter-based noise (sample_gumbel): the base row of the tail and verify rows 0 .. K-1 choose
  // argmax_j (processed_j / smp_temp + g(position, j)) over their top-k set {j : processed_j >= tau}; smp_topk = 0: the
  // whole row.  The seed is two 32-bit words for the same reason as adj.
  int smp_on, smp_topk;
  float smp_temp;
  unsigned int smp_key[2], smp_window, smp_attempt;
  float tail_tau;                // tau of the tail's base row (-inf: the whole row), read by the scoring kernel
  float row_tau[WM_MAX_T];       // tau of verify row r of the last accept step
};
__host__ __device__ __forceinline__ const float* dec_state_adj(const DecState* st) {
  return reinterpret_cast<const float*>(((unsigned long long)st->adj_hi << 32) | st->adj_lo);
}
__host__ __device__ __forceinline__ void dec_state_set_adj(DecState* st, const float* adj) {
  const unsigned long long a = reinterpret_cast<unsigned long long>(adj);
  st->adj_lo = (unsigned int)a;
  st->adj_hi = (unsigned int)(a >> 32);
}

// Logits processors applied to element j of a raw logits row, with cur_len = L (HF logits_process.py:1893-1901 suppress,
// :1847-1862 begin-suppress when L == begin_index, :1742-1772 EOS exponential decay with pen = pen_tab[L]).  Shared by
// the loop's logits scan and the scoring kernel.  ADJ: the iteration's per-token term adj[V] of the sequence-bias,
// bad-words, no-repeat-n-gram and min-length processors (logits_proc.cu) is added first, as HF's chain adds it before
// the decay.  Callers instantiate both variants and pick one with a uniform flag, so the off path is today's code.
template <bool ADJ = false>
__device__ __forceinline__ float processed_logit(const float* row, int j, const uint8_t* mask, bool begin_on,
                                                 int eos, float pen, const float* adj = nullptr) {
  const uint8_t mk = mask[j];
  if ((mk & 1) || (begin_on && (mk & 2))) return -INFINITY;
  float v = ldcg_f(row + j);
  if (ADJ) v = v + ldcg_f(adj + j);
  // HF rounds the product and then the sum; a contracted FMA would round once and can differ in the last bit
  if (j == eos && pen != 0.f) v = __fadd_rn(v, __fmul_rn(fabsf(v), pen));
  return v;
}

// Philox4x32-10 (Salmon et al., "Parallel random numbers: as easy as 1, 2, 3", SC 2011): counter c, key k.
__host__ __device__ __forceinline__ uint4 philox4x32_10(uint4 c, unsigned int k0, unsigned int k1) {
#pragma unroll
  for (int i = 0; i < 10; ++i) {
    if (i) { k0 += 0x9E3779B9u; k1 += 0xBB67AE85u; }
    const unsigned long long p0 = 0xD2511F53ull * c.x, p1 = 0xCD9E8D57ull * c.z;
    c = make_uint4((unsigned int)(p1 >> 32) ^ c.y ^ k0, (unsigned int)p1, (unsigned int)(p0 >> 32) ^ c.w ^ k1,
                   (unsigned int)p0);
  }
  return c;
}
// Gumbel noise of token j at position n (the index in DecState::ids the chosen token is written to) of a sampled
// attempt: word j % 4 of Philox4x32-10(counter (j / 4, n, window, attempt), key = the seed's words) -> x,
// u = ((x >> 8) + 0.5) 2^-24 in (0, 1), g = -log(-log u).  u and the logarithms are evaluated in double (u is exact
// there; in fp32 the upper half of the range would round), and g is rounded once to fp32.
__host__ __device__ __forceinline__ float sample_gumbel(const unsigned int key[2], unsigned int window,
                                                        unsigned int attempt, int n, int j) {
  const uint4 x = philox4x32_10(make_uint4((unsigned int)j >> 2, (unsigned int)n, window, attempt), key[0], key[1]);
  const int w = j & 3;
  const unsigned int b = w == 0 ? x.x : w == 1 ? x.y : w == 2 ? x.z : x.w;
  const double u = ((double)(b >> 8) + 0.5) * (1.0 / 16777216.0);
  return (float)(-log(-log(u)));
}

struct alignas(16) DecModel {   // (copied to shared memory in 16-byte pieces by the ring kernel)
  int d, H, ffn, V, S, S_pad;
  int n_layers;      // decoder layers (without the medusa block)
  int has_block;     // 1 => layers[n_layers] is the medusa block
  int K;             // medusa heads
  int n_tree;        // rows of the verify pass: K+1 for the chain, tree nodes for branching medusa_choices
  int has_tree;      // 1 => branching choices: `tree` describes the candidate tree
  int n_head_layers; // MedusaResBlocks per head (medusa_num_layers); fills the padding before `tree`, so the size and
                     // every later offset of this struct are those of the single-layer layout
  const DecTree* tree;
  float* topk_part;  // [WM_MAX_T rows][32 segments][WM_TREE_MAX_TOPK]{value, index}: per-segment top-k of the tail scan
                     // (sampled attempts, which never have a tree: [WM_SMP_MAX_TOPK] entries per row and segment)
  DecLayer layers[WM_MAX_DEC_LAYERS];
  const __half* embed;   // [V, d] (also proj_out)
  const float* pos;      // [max_target_positions, d]
  const float *lnf_g, *lnf_b;
  const __half* heads_w; // [n_head_layers][(K+1) or K][d, d], layer-major
  const float* heads_b;  // [n_head_layers][(K+1) or K][d]
  const uint8_t* tok_mask;  // [V]: bit0 suppress, bit1 begin-suppress
  const float* pen_tab;     // [WM_MAX_POS + 32]: (factor^(L-start) - 1) as f32, 0 when inactive
  // activations (fp32)
  float* x;        // [WM_MAX_T, d] residual stream
  float* xg;       // [WM_MAX_T, d] gamma o x in the MMA operand format, for the LayerNorm GEMM that follows (ring kernel)
  float* q;        // [WM_MAX_T, d]
  float* attn;     // [WM_MAX_T, d]
  float* ffn_h;    // [WM_MAX_T, ffn]
  float* hidden;   // [WM_MAX_T, d]  final-LN output (block type: input of the block)
  float* head_h;   // [2][WM_MAX_T, d]: head-layer outputs, ping-ponged between the halves (head_layer_out); the last
                   // layer, and the block type's base row, are in the first half, which the vocabulary stage reads
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
  // instruction lists of the ring kernel's stage program (dec_build_program): sweep A, tail, verify = [off[i], off[i+1])
  int prog_off[4];
  // per-CTA weight-chunk schedule of the ring producer (built by the host once the weights are bound):
  // chunk_tab[chunk_off[cta*4 + list] .. chunk_off[cta*4 + list + 1]) in consumption order
  const struct ChunkDesc* chunk_tab;
  const int* chunk_off;
  const struct CtaStage* stage_tab;   // [prog_off[3]][n_sm] resolved stage records of the ring kernel
  DecState* st;
  unsigned int* bar;  // grid-barrier words for the persistent kernel
  unsigned long long* prof;  // optional stage timeline [2 CTAs][n_instr][16] (ns, and flags), null = off
  // no-speech capture (option "no_speech_row"): the final LayerNorm stores row ns_row of the first real iteration's
  // sweep A (row index within that pass's tile, prefill chunks excluded) into ns_hidden [d]; -1 = off
  float* ns_hidden;
  int ns_row;
  // token-timestamp capture (wm_set_alignment_heads): null = off (it then costs one predicate per cross-attention item)
  const struct TsCapture* ts;
};

// Token-timestamp capture.  The cross-attention stages of the base decoder layers store, for every alignment head, the
// raw scores (q . k / 8, fp32, before the softmax) of each row r < T of passes A and B at the row's position:
// scores[slot][position][S].  A position is written again by every pass that recomputes it, so the last writer is the
// pass that accepted its token (DESIGN.md section 7).
#define WM_TS_ROWS (WM_MAX_POS + WM_MAX_T)
#define WM_TS_MAX_HEADS 32
struct TsCapture {
  float* scores;                                  // [n_slots][WM_TS_ROWS][S]
  int slot[WM_MAX_DEC_LAYERS * WM_TS_MAX_HEADS];  // [layer * H + head]: capture slot, -1 = not captured
};

}  // namespace wm
