// Persistent decode kernel with a weight ring (included from decode.cu, inside namespace wm).
//
// The stage chain of one speculative iteration is latency-bound if every stage first waits for
// the grid barrier and only then starts pulling its weights from HBM: a d x d GEMV stage moves
// 3.3 MB -- far less than the bandwidth-delay product of the chip.  But WHICH weight bytes a CTA
// needs is static: for every GEMM stage it owns a fixed, contiguous range of rows of W.  So each
// CTA streams its rows for the upcoming stages through a shared-memory ring with bulk async
// copies (cp.async.bulk -> mbarrier complete_tx; SASS UBLKCP), independently of the activation
// dependency chain: the copies for stages s+1, s+2, ... are in flight while the compute warps sit
// in the grid barrier of stage s.  When a stage's activations finally arrive, its weights are
// already on-chip and the stage costs: X staging (L2) + a few MMAs out of shared memory + epilogue.
//
// Roles: warps 0..14 = compute (WM_DEC_THREADS threads, named barrier 1), warp 15 = producer.
// The producer walks a per-CTA chunk table that the host builds once per model (no pointer
// chasing on the device), waits on `empty[slot]`, arms `full[slot]` with the byte count and lets
// lanes 0..nrows-1 issue one bulk copy per weight row.
//
// Everything on the critical path of a stage is either resident or asynchronous:
//   * the kernel is a template of the model width D: strides, slice counts and every shared-memory
//     offset are immediates (no integer divisions, few live registers -- with a 227 KB carve-out
//     only ~27 KB of L1 remain, so a register spill is an L2 round trip);
//   * the stage record of this CTA (row range, pointers, epilogue; built by the host) is prefetched
//     into shared memory while the previous stage runs;
//   * activations arrive by bulk copy, written by their producers in the MMA operand format or split
//     in place (see below); the LayerNorm gamma of the next stage is bulk-copied while the stage
//     before it runs; bias vectors are pulled into L2 one stage ahead and read while the MMAs run.  (A plain global load that is still in
//     flight at a bar.sync stalls the barrier: no long-latency ld may precede one.)
//
// Stages with K > d (FC2) are split over CTAs along K as well: CTA = (row block, k segment); the
// segment partials go to a global scratch and the CTA that arrives last for a row block folds
// them in segment order (deterministic) and runs the epilogue.
//
// On the whole GPU the kernel runs as 2-CTA clusters (CTAs 2i, 2i+1; still a cooperative launch:
// the grid barrier needs every CTA resident).  Every CTA of a GEMM stage stages the same activation
// rows, so where both CTAs of a pair have rows, the even one multicasts them into both CTAs' shared
// memory (one L2 read per pair; CtaStage::x_role) and the odd one only waits for them.  The kernel
// reads the cluster size at run time: partial grids launch unclustered and every CTA copies its own
// rows.
//
// Ring geometry: a "chunk" = up to 16 weight rows x d columns (fp16), row stride d*2 + 64 B
// (bank-conflict-free LDS.128 of the B fragments), or the K or V rows of a cross-attention key chunk or of a
// self-attention prefix block; WM_RING_G chunks are resident; chunks are consumed in program order.
#pragma once

#define WM_RING_G 3
#define WM_RING_THREADS (WM_DEC_THREADS + 32)

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_n(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)),
               "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
// the same copy into the same CTA-relative offsets (dst and mbarrier) of every CTA of the cluster in cta_mask
__device__ __forceinline__ void bulk_g2s_multicast(void* dst, const void* src, uint32_t bytes, uint64_t* bar, uint16_t cta_mask) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1], %2, [%3], %4;" ::"r"(
          smem_u32(dst)),
      "l"(src), "r"(bytes), "r"(smem_u32(bar)), "h"(cta_mask)
      : "memory");
}
__device__ __forceinline__ uint32_t cluster_ncta() {
  uint32_t n;
  asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(n));
  return n;
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ unsigned long long global_timer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ void prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }

__host__ __device__ __forceinline__ bool is_gemm_stage(int st) {
  return st == ST_QKV || st == ST_OPROJ || st == ST_CROSS_Q || st == ST_CROSS_O || st == ST_FC1 || st == ST_FC2 ||
         st == ST_HEADS || st == ST_VOCAB;
}

__host__ __device__ __forceinline__ void cta_rows(int N, int part, int nparts, int& n_begin, int& n_rows) {
  const int rows_per = N / nparts, rem = N % nparts;
  n_begin = part * rows_per + (part < rem ? part : rem);
  n_rows = rows_per + (part < rem ? 1 : 0);
}

// Work of one CTA in a GEMM stage: rows [n_begin, n_begin + n_rows) of W, k segment `seg` of `segs`
// (segs > 1 <=> K > d: the stage is split along K over CTAs; `block` = row block shared by `segs` CTAs).
// Consecutive CTAs take consecutive row blocks of ONE segment, so the two CTAs of a cluster read the same k slice of
// the activations and can share one multicast copy of it.
struct GemmWork { int n_begin, n_rows, seg, segs, block; };
__host__ __device__ __forceinline__ GemmWork gemm_work(int N, int K, int d, int cta, int ncta) {
  GemmWork w;
  w.segs = K / d;
  if (w.segs <= 1) {
    w.segs = 1; w.seg = 0; w.block = cta;
    cta_rows(N, cta, ncta, w.n_begin, w.n_rows);
    return w;
  }
  const int nb = ncta / w.segs;   // host guarantees nb >= 1
  if (cta >= nb * w.segs) { w.n_begin = 0; w.n_rows = 0; w.seg = 0; w.block = 0; return w; }
  w.seg = cta / nb;
  w.block = cta - w.seg * nb;
  cta_rows(N, w.block, nb, w.n_begin, w.n_rows);
  return w;
}

// ---------------------------------------------------------------------------------------------
// compile-time geometry of the kernel for model width D
// ---------------------------------------------------------------------------------------------
__host__ __device__ constexpr size_t cmax(size_t a, size_t b) { return a > b ? a : b; }
__host__ __device__ constexpr size_t round128(size_t a) { return (a + 127) / 128 * 128; }
#ifndef WM_RING_NKS_MAX
#define WM_RING_NKS_MAX 4   /* MMA warps per GEMM stage (k-slices); chosen by A/B timing at large-v2 */
#endif
__host__ __device__ constexpr int ring_nks(int d) {
#ifdef WM_RING_NKS_FORCE
  if (d % (WM_RING_NKS_FORCE * 32) == 0) return WM_RING_NKS_FORCE;
#endif
  return (d % 256 == 0 && WM_RING_NKS_MAX >= 8) ? 8 : (d % 128 == 0 && WM_RING_NKS_MAX >= 4) ? 4 : (d % 64 == 0) ? 2 : 1;
}

#define WM_XS_PADB 16   // bytes of X-row padding: stride = 16 (mod 128) => conflict-free LDS.128 / STS.128

// Keys of a self-attention item that the ring does not bring (sa_prefix_chunk): the pass's own rows and those sweep A
// wrote earlier in the launch, at most WM_MAX_T each.  Their K and V rows are staged behind the stage's scratch.
#define WM_SA_NEW (2 * WM_MAX_T)
__host__ __device__ constexpr size_t self_attn_new_rows_bytes() { return (size_t)2 * WM_SA_NEW * WM_KV_ROW * sizeof(__half); }

template <int D>
struct RingGeom {
  static_assert(D % 32 == 0 && D <= 1280, "decoder width must be a multiple of 32, at most 1280");
  static constexpr int ROW_STRIDE = D * 2 + 64;       // ring row stride, bytes
  // a slot holds 16 weight rows or the K (or V) rows of one cross-attention key chunk ([CH_PAD][72] fp16)
  static constexpr int SLOT_BYTES = (int)round128(cmax((size_t)16 * ROW_STRIDE, (size_t)WM_CH_PAD * 72 * sizeof(__half)));
  static_assert(SLOT_BYTES <= WM_RING_SLOT_MAX && (D < 1280 || SLOT_BYTES == WM_RING_SLOT_MAX), "WM_RING_SLOT_MAX");
  static constexpr int XS = D * 4 + WM_XS_PADB;       // activation row stride, bytes
  static constexpr int NKS = ring_nks(D);             // k-slices per chunk (one MMA warp each)
  static constexpr int KS = D / NKS;
  static_assert(KS % 32 == 0, "k-slice must be a multiple of the 32-column MMA step");
  static constexpr int NV4 = D / 4;                   // float4 per activation row
  static constexpr int NV = (D + 127) / 128;          // float4 per lane of a row-per-warp pass
  // shared-memory map
  static constexpr size_t SCRATCH_OFF = (size_t)WM_RING_G * SLOT_BYTES;
  static constexpr size_t SCRATCH =
      round128(cmax(cmax((size_t)16 * XS, cross_scratch_bytes()), self_attn_smem_bytes() + self_attn_new_rows_bytes()));
  static constexpr size_t PARTIAL_OFF = SCRATCH_OFF + SCRATCH;
  static constexpr size_t PARTIAL = round128((size_t)NKS * 256 * sizeof(float));   // k-slice partials of one unit
  static constexpr size_t GAMMA_OFF = PARTIAL_OFF + PARTIAL;
  static constexpr size_t GAMMA = round128((size_t)D * sizeof(float));             // LayerNorm gamma of the running stage
  static constexpr size_t MODEL_OFF = GAMMA_OFF + GAMMA;
  static constexpr size_t MODEL = round128(sizeof(DecModel));
  static constexpr size_t BAR_OFF = MODEL_OFF + MODEL;
  static constexpr size_t TOTAL = BAR_OFF + 128;
};

// ---------------------------------------------------------------------------------------------
// producer warp: stream the chunk table through the ring
// ---------------------------------------------------------------------------------------------
// Bytes per CTA that the producer keeps prefetched into L2 ahead of its ring copies (ring_walk); chosen by A/B timing at
// large-v2 (DESIGN.md section 4), and used on the whole GPU only (the clustered launch): on partial grids
// (decode_ctas, StreamGroup) concurrent engines share HBM and L2, and the prefetch made four streams of 33 CTAs about
// 10 % slower, so those launches run without it.  0 = no prefetch.  A nonzero budget holds at least the largest chunk, so the cursor
// never stalls.  Full weight chunks at d = 1280 are 40,960 B, so 64 KB keeps about one chunk beyond the three slots in L2
// (two when they are small): a fourth slot, in L2.
#ifndef WM_RING_L2_AHEAD
#define WM_RING_L2_AHEAD (64 * 1024)
#endif
static_assert(WM_RING_L2_AHEAD == 0 || WM_RING_L2_AHEAD >= WM_RING_SLOT_MAX, "the L2 lookahead must hold a whole chunk");

// One ring chunk as a launch copies it: `nrows` rows of `copy_bytes`, row r read at src + r * row_bytes; nrows = 0:
// nothing to copy (a self-attention prefix block that does not exist at this launch's (L0, kv0); the consumer skips it
// too).  The producer's copies, its L2 prefetches and the host replay (dec_check_ring_schedule) all resolve chunks here.
struct ChunkCopy { const unsigned char* src; uint32_t row_bytes, nrows, copy_bytes; };
__host__ __device__ __forceinline__ ChunkCopy resolve_chunk(const ChunkDesc& dsc, int H, int n_tree, int cta, int ncta, int L0,
                                                            int kv0) {
  ChunkCopy c{reinterpret_cast<const unsigned char*>(dsc.src), dsc.row_bytes, dsc.nrows, dsc.copy_bytes};
  if (dsc.nrows == 0) {
    // a self-attention prefix block: one contiguous copy of its K or V rows
    const SaChunk s = sa_prefix_chunk(H, ncta, cta, dsc.sa_mode, L0, kv0, n_tree, dsc.sa_item, dsc.sa_block);
    c.nrows = s.nk > 0 ? 1u : 0u;
    c.copy_bytes = (uint32_t)s.nk * WM_KV_ROW * sizeof(__half);
    if (s.nk > 0) c.src += self_kv_index(s.j0, s.h * 64) * sizeof(__half);
  }
  return c;
}

// The producer's walk over chunks [first, last) of the chunk table (L0, kv0: the loop state at launch, which sizes the
// self-attention prefix chunks).  copy(cp) puts a chunk into the next ring slot, waiting for the slot to free.  Before
// each copy an L2 cursor tops up: it prefetches the chunks from the one about to be copied onwards while the bytes
// prefetched but not yet copied stay within `budget`.  So HBM keeps streaming while the ring is full and the grid waits
// at barriers, and a slot that frees is refilled from L2.  Past `last` the cursor goes on into the first weight chunks
// of the tail program [warm_first, warm_last): the next launch starts there when this one's candidates are accepted,
// and its first copies then hit L2 too.  It stops at the first self-attention prefix block there, which only the next
// launch's loop state sizes.  A prefetch is a hint, and L2 is the point of coherence: no copy can read stale bytes.
template <class Prefetch, class Copy>
__host__ __device__ __forceinline__ void ring_walk(const ChunkDesc* tab, int first, int last, int warm_first, int warm_last,
                                                   uint32_t budget, int H, int n_tree, int cta, int ncta, int L0, int kv0,
                                                   Prefetch prefetch, Copy copy) {
  int pf = first, pf_end = last;   // the cursor and the end of the range it walks
  bool warm = false;               // walking the tail program
  uint32_t ahead = 0;              // bytes prefetched, not yet copied
  auto top_up = [&] {
    while (budget > 0) {
      if (pf == pf_end) {
        if (warm) return;
        warm = true; pf = warm_first; pf_end = warm_last;
        continue;
      }
      const ChunkDesc& dsc = tab[pf];
      if (warm && dsc.nrows == 0) { pf = pf_end; return; }
      const ChunkCopy p = resolve_chunk(dsc, H, n_tree, cta, ncta, L0, kv0);
      if (ahead + p.nrows * p.copy_bytes > budget) return;
      if (p.nrows > 0) prefetch(p);
      ahead += p.nrows * p.copy_bytes;
      ++pf;
    }
  };
  ChunkDesc nxt{};
  if (first < last) nxt = tab[first];
  for (int c = first; c < last; ++c) {
    const ChunkDesc dsc = nxt;
    if (c + 1 < last) nxt = tab[c + 1];   // next descriptor is in flight while we wait
    top_up();
    const ChunkCopy cp = resolve_chunk(dsc, H, n_tree, cta, ncta, L0, kv0);
    if (cp.nrows == 0) continue;
    copy(cp);
    if (budget > 0) ahead -= cp.nrows * cp.copy_bytes;
  }
  top_up();
}

__device__ __forceinline__ void bulk_prefetch_l2(const void* src, uint32_t bytes) {
  asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(src), "r"(bytes) : "memory");
}

template <int D>
__device__ __noinline__ void ring_producer(unsigned char* ring, uint64_t* full, uint64_t* empty,
                                           const ChunkDesc* __restrict__ tab, int first, int last, int warm_first,
                                           int warm_last, const DecModel* m, int cta, int ncta, int L0, int kv0) {
  using G = RingGeom<D>;
  const int lane = threadIdx.x & 31;
  int slot = 0;
  unsigned int par = 1;   // parity to wait for on `empty` (fresh barrier: the "previous" phase counts as complete)
  ring_walk(
      tab, first, last, warm_first, warm_last, cluster_ncta() > 1 ? (uint32_t)WM_RING_L2_AHEAD : 0u, m->H, m->n_tree, cta, ncta, L0, kv0,
      [&](const ChunkCopy& p) {
        // one prefetch per contiguous range: the whole chunk, or each row of FC2's k-segment rows (as the copies go)
        if (p.nrows == 1 || p.row_bytes == p.copy_bytes) {
          if (lane == 0) bulk_prefetch_l2(p.src, p.nrows * p.copy_bytes);
        } else if (lane < p.nrows) {
          bulk_prefetch_l2(p.src + (size_t)lane * p.row_bytes, p.copy_bytes);
        }
      },
      [&](const ChunkCopy& cp) {
        if (lane == 0) {
          while (!mbar_try_wait(empty + slot, par)) { }
          asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic reads of the slot vs async writes
          mbar_expect_tx(full + slot, cp.nrows * cp.copy_bytes);
        }
        __syncwarp();
        if (lane < cp.nrows) {
          bulk_g2s(ring + (size_t)slot * G::SLOT_BYTES + (size_t)lane * G::ROW_STRIDE, cp.src + (size_t)lane * cp.row_bytes,
                   cp.copy_bytes, full + slot);
        }
        __syncwarp();
        if (++slot == WM_RING_G) { slot = 0; par ^= 1u; }
      });
}

// ---------------------------------------------------------------------------------------------
// activation staging
//
// The T activation rows of a GEMM stage (fp32, written by other CTAs before the grid barrier)
// are pulled into shared memory by bulk async copies -- one per row, issued by the lanes of
// warp 0 the moment the barrier opens -- instead of 10 dependent ld.global per lane.  They land
// as fp32 rows of stride d*4 + 16 B and are split IN PLACE into the fp16 hi/lo operand format:
// every 8-byte pair of floats (x[k], x[k+1]) becomes { half2 hi(k,k+1), half2 lo(k,k+1) }, so one
// LDS.128 of the MMA loop fetches the hi AND lo A-fragment registers of two k-pairs.
// LayerNorm stages (QKV, cross-Q, FC1) are not normalised before the MMAs.  With mean mu, rstd and
// gamma / beta of the row,
//     LN(x) W^T + b = rstd * ((gamma o x) W^T - mu * c) + b',   c_n = sum_k gamma_k W_nk,  b'_n = b_n + sum_k beta_k W_nk
// ({b', c} per output row are derived once per weight binding, dec_fold_layernorms).  The operand is
// gamma o x, which needs no row statistics: the residual epilogue before a LayerNorm stage (O-proj,
// cross-O, FC2) writes it in the operand format next to x (xg; element-wise, so the same for every
// grid), and the stage stages xg like any presplit stage.  Stages fed otherwise (layer 0, the
// Medusa block) split gamma o x in place.  mu / rstd: the epilogue warps, from the fp32 rows of x
// in L2, while the rows are staged and the MMAs run.
// Rows >= T keep stale bits: MMA rows are independent and rows >= T are never stored.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint4 split_hilo4(float4 y) {
  // packed conversions: hi = rn(x), lo = rn(x - hi)
  const __half2 a = __floats2half2_rn(y.x, y.y), b = __floats2half2_rn(y.z, y.w);
  const float2 fa = __half22float2(a), fb = __half22float2(b);
  const __half2 c = __floats2half2_rn(y.x - fa.x, y.y - fa.y);
  const __half2 e = __floats2half2_rn(y.z - fb.x, y.w - fb.y);
  uint4 o;
  o.x = *reinterpret_cast<const uint32_t*>(&a); o.y = *reinterpret_cast<const uint32_t*>(&c);
  o.z = *reinterpret_cast<const uint32_t*>(&b); o.w = *reinterpret_cast<const uint32_t*>(&e);
  return o;
}
// value of activation (row r, column n) back from the split buffer (hi + lo is exact in fp32)
__device__ __forceinline__ float xbuf_value(const unsigned char* xb, int xs, int r, int n) {
  const __half* p = reinterpret_cast<const __half*>(xb + (size_t)r * xs + (size_t)(n >> 1) * 8) + (n & 1);
  return __half2float(p[0]) + __half2float(p[2]);
}

// LayerNorm statistics {mu, rstd} of the fp32 rows X (row stride ld, L2-coherent loads: the staged rows are gamma o x):
// warp w of nw takes rows w, w + nw, ...; lane l sums float4 columns l, l+32, ... of its row held in registers (two
// passes: mean, then the centred squares).
template <int D>
__device__ __forceinline__ void ring_row_stats(const float* X, int ld, float2* stat, int T, int w, int nw) {
  using G = RingGeom<D>;
  const int lane = threadIdx.x & 31;
  for (int r = w; r < T; r += nw) {
    const float* x = X + (size_t)r * ld + 4 * lane;
    float4 v[G::NV];
#pragma unroll
    for (int i = 0; i < G::NV; ++i)
      if (i * 32 + lane < G::NV4) v[i] = ldcg_f4(x + i * 128);
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < G::NV; ++i)
      if (i * 32 + lane < G::NV4) s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
    const float mean = warp_sum(s) / (float)D;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < G::NV; ++i)
      if (i * 32 + lane < G::NV4) {
        const float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, e = v[i].w - mean;
        q += (a * a + b * b) + (c * c + e * e);
      }
    const float rstd = rsqrtf(warp_sum(q) / (float)D + 1e-5f);
    if (lane == 0) stat[r] = make_float2(mean, rstd);
  }
}

__device__ __forceinline__ float4 mul4(float4 a, float4 b) { return make_float4(a.x * b.x, a.y * b.y, a.z * b.z, a.w * b.w); }

// per-thread state of the compute warps that survives across stages (uniform over the CTA)
struct RingState {
  int slot;            // ring slot of the next chunk to consume
  unsigned int par;    // its `full` parity
  unsigned int xpar;   // parity of the activation-copy barrier
  unsigned int ppar;   // parity of the LayerNorm-gamma barrier
};

// ---------------------------------------------------------------------------------------------
// GEMM stage fed from the ring (compute warps).  `sd` = this CTA's resolved record (shared memory).
// ---------------------------------------------------------------------------------------------
template <int D>
__device__ __forceinline__ void stage_gemm_ring(RingState& rs, unsigned char* smem, const DecModel* m, const CtaStage* sd,
                                                int Tpass, int base, unsigned long long* pr) {
  using G = RingGeom<D>;
  __shared__ int s_last;
  __shared__ float2 s_stat[WM_MAX_T];   // LayerNorm stages: {mu, rstd} of the token rows
  const int n_rows = sd->n_rows;
  unsigned char* const xb = smem + G::SCRATCH_OFF;
  float* const partial = reinterpret_cast<float*>(smem + G::PARTIAL_OFF);
  const float* const gamma = reinterpret_cast<const float*>(smem + G::GAMMA_OFF);
  uint64_t* const full = reinterpret_cast<uint64_t*>(smem + G::BAR_OFF);
  uint64_t* const empty = full + WM_RING_G;
  uint64_t* const xbar = empty + WM_RING_G;
  uint64_t* const pbar = xbar + 1;
  if (n_rows == 0) {
    // no rows for this CTA (narrow models; the chunk table has no entry either) -- but the LayerNorm gamma
    // was sent to every CTA: consume that phase
    if (sd->ln) { while (!mbar_try_wait(pbar, rs.ppar)) { } rs.ppar ^= 1u; }
    return;
  }
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  constexpr int nwarps = WM_DEC_THREADS >> 5;
  const int gq = lane >> 2, tq = lane & 3;
  const int T = sd->x_rows_fixed ? sd->x_rows_fixed : Tpass;
  const bool ln = sd->ln != 0;

  if (pr) {
    pr[7] = global_timer_ns();
    pr[11] = mbar_try_wait(full + rs.slot, rs.par) ? 1000ull : 0ull;   // weights already here?
  }
  // ---- X rows: global (L2) -> shared, one bulk copy per row ----
  // In a 2-CTA cluster whose CTAs stage the same rows, the issuing CTA multicasts each row into the same offsets of both
  // CTAs (one L2 read per pair) and signals both xbars; the receiving CTA only arms its own xbar for the same bytes.  A
  // complete_tx that reaches the receiver's xbar before its arrival cannot finish the phase (the arrival is pending).
  if (warp == 0) {
    const int role = sd->x_role;
    if (lane == 0) {
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // earlier generic accesses of the buffer vs async writes
      mbar_expect_tx(xbar, (uint32_t)(T * D * 4));
    }
    __syncwarp();
    if (lane < T) {
      if (role == XR_OWN) bulk_g2s(xb + (size_t)lane * G::XS, sd->X + (size_t)lane * sd->x_ld, (uint32_t)(D * 4), xbar);
      else if (role == XR_ISSUE)
        bulk_g2s_multicast(xb + (size_t)lane * G::XS, sd->X + (size_t)lane * sd->x_ld, (uint32_t)(D * 4), xbar, 0x3);
    }
  } else if (warp == 1) {
    // this CTA's bias slice of the NEXT GEMM stage -> L2 (biases are cold: 2 GB of weights pass through L2 per iteration)
    if (lane < sd->pf_bias_lines) prefetch_l2(reinterpret_cast<const unsigned char*>(sd->pf_bias) + (size_t)lane * 128);
  }
  // LayerNorm stages: the epilogue warps compute the statistics from the fp32 rows of x in L2 while the rows are staged
  // (published behind named barrier 4, which only the epilogue warps join)
  if (ln && warp >= G::NKS) ring_row_stats<D>(m->x, D, s_stat, T, warp - G::NKS, nwarps - G::NKS);
  while (!mbar_try_wait(xbar, rs.xpar)) { }
  rs.xpar ^= 1u;
  if (pr) pr[8] = global_timer_ns();
  // every thread has seen the rows land; only a split pass makes the CTA wait for one another
  if (ln) {
    // gamma was bulk-copied into its region during the preceding barrier
    while (!mbar_try_wait(pbar, rs.ppar)) { }
    rs.ppar ^= 1u;
    if (pr) pr[9] = global_timer_ns();
  }
  if (ln && !sd->presplit) {
    // gamma o x -> operand format in place: thread per float4 column, the loads of 4 rows in flight together
    static_assert(G::NV4 <= WM_DEC_THREADS, "one thread per float4 column");
    if (tid < G::NV4) {
      const float4 g = reinterpret_cast<const float4*>(gamma)[tid];
      for (int r0 = 0; r0 < T; r0 += 4) {
        unsigned char* const rows = xb + (size_t)r0 * G::XS + (size_t)tid * 16;
        float4 v[4];
#pragma unroll
        for (int r = 0; r < 4; ++r)
          if (r0 + r < T) v[r] = *reinterpret_cast<const float4*>(rows + (size_t)r * G::XS);
#pragma unroll
        for (int r = 0; r < 4; ++r)
          if (r0 + r < T) *reinterpret_cast<uint4*>(rows + (size_t)r * G::XS) = split_hilo4(mul4(g, v[r]));
      }
    }
    if (pr) pr[10] = global_timer_ns();
    cta_sync();
  } else if (!ln && !sd->presplit) {
    // flat over the buffer (the 16-byte row pad is converted along: no index arithmetic)
    uint4* p = reinterpret_cast<uint4*>(xb);
    const int n16 = T * (G::XS >> 4);
    for (int idx = tid; idx < n16; idx += WM_DEC_THREADS) p[idx] = split_hilo4(*reinterpret_cast<const float4*>(p + idx));
    if (pr) pr[10] = global_timer_ns();
    cta_sync();
  }
  if (pr) pr[3] = global_timer_ns();
  const int units = (n_rows + 15) >> 4;
  const bool ksplit = sd->segs > 1;
  const int epi = sd->epi;
  const int n_begin = sd->n_begin;
  // ---- unit loop, warp-specialised: warps 0..NKS-1 run the MMAs of unit u while the remaining warps finish unit
  // u-1 (k-slice reduction, bias, epilogue, global stores).  Named barrier 2 = "partials of unit u written",
  // named barrier 3 = "partials of unit u read" (the partial buffer is single: its rewrite waits for the readers).
  constexpr int NE = WM_DEC_THREADS - G::NKS * 32;   // epilogue threads
  if (warp < G::NKS) {
    for (int u = 0; u < units; ++u) {
      const int nvalid = min(16, n_rows - u * 16);
      if (pr && u == 0) { pr[12] = mbar_try_wait(full + rs.slot, rs.par) ? 1000ull : 0ull; pr[13] = global_timer_ns(); }
      while (!mbar_try_wait(full + rs.slot, rs.par)) { }
      if (pr && u == 0) pr[4] = global_timer_ns();
      const __half* sl = reinterpret_cast<const __half*>(smem + (size_t)rs.slot * G::SLOT_BYTES);
      const bool v0 = gq < nvalid, v1 = (gq + 8) < nvalid;
      const __half* w0p = sl + (size_t)gq * (G::ROW_STRIDE / 2) + warp * G::KS + 8 * tq;
      const __half* w1p = w0p + (size_t)8 * (G::ROW_STRIDE / 2);
      const unsigned char* x0 = xb + (size_t)gq * G::XS + (size_t)(warp * G::KS + 8 * tq) * 4;
      const unsigned char* x1 = x0 + (size_t)8 * G::XS;
      const bool t1 = (gq + 8) < T;   // token rows 8..15 contribute nothing when T <= 8 + gq
      // four independent accumulator chains: (n8 tile 0 / 1) x (hi / lo part of X)
      float c0h[4] = {0.f, 0.f, 0.f, 0.f}, c0l[4] = {0.f, 0.f, 0.f, 0.f};
      float c1h[4] = {0.f, 0.f, 0.f, 0.f}, c1l[4] = {0.f, 0.f, 0.f, 0.f};
      const uint4 z = make_uint4(0, 0, 0, 0);
#pragma unroll
      for (int kk = 0; kk < G::KS; kk += 32) {
        const uint4 wa = v0 ? *reinterpret_cast<const uint4*>(w0p + kk) : z;
        const uint4 wb = v1 ? *reinterpret_cast<const uint4*>(w1p + kk) : z;
        // {hi(k,k+1), lo(k,k+1), hi(k+2,k+3), lo(k+2,k+3)} for k = kk + 8 tq and k + 4
        const uint4 p0 = *reinterpret_cast<const uint4*>(x0 + kk * 4);
        const uint4 p1 = *reinterpret_cast<const uint4*>(x0 + kk * 4 + 16);
        const uint4 q0 = t1 ? *reinterpret_cast<const uint4*>(x1 + kk * 4) : z;
        const uint4 q1 = t1 ? *reinterpret_cast<const uint4*>(x1 + kk * 4 + 16) : z;
        mma_16816(c0h, p0.x, q0.x, p0.z, q0.z, wa.x, wa.y);
        mma_16816(c0l, p0.y, q0.y, p0.w, q0.w, wa.x, wa.y);
        mma_16816(c1h, p0.x, q0.x, p0.z, q0.z, wb.x, wb.y);
        mma_16816(c1l, p0.y, q0.y, p0.w, q0.w, wb.x, wb.y);
        mma_16816(c0h, p1.x, q1.x, p1.z, q1.z, wa.z, wa.w);
        mma_16816(c0l, p1.y, q1.y, p1.w, q1.w, wa.z, wa.w);
        mma_16816(c1h, p1.x, q1.x, p1.z, q1.z, wb.z, wb.w);
        mma_16816(c1l, p1.y, q1.y, p1.w, q1.w, wb.z, wb.w);
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(empty + rs.slot);   // this warp is done with the slot (the barrier counts NKS arrivals)
      if (++rs.slot == WM_RING_G) { rs.slot = 0; rs.par ^= 1u; }
      if (pr && u == 0) pr[5] = global_timer_ns();
      if (u > 0) asm volatile("bar.sync 3, %0;" ::"n"(WM_DEC_THREADS) : "memory");   // partials of unit u-1 have been read
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        partial[warp * 256 + e * 32 + lane] = c0h[e] + c0l[e];
        partial[warp * 256 + (4 + e) * 32 + lane] = c1h[e] + c1l[e];
      }
      asm volatile("bar.arrive 2, %0;" ::"n"(WM_DEC_THREADS) : "memory");
      if (pr && u == 0) pr[6] = global_timer_ns();
    }
  } else {
    const int etid = tid - G::NKS * 32;
    constexpr int NOUT = (256 + NE - 1) / NE;   // outputs per epilogue thread and unit
    // this thread's bias / residual values of a unit are requested before its partials are awaited: the loads are in
    // flight while the MMA warps work.  aux = the residual (EPI_RESID) or, in LayerNorm stages, c_n (sd->bias then
    // points at the {b'_n, c_n} pairs)
    float bias_v[NOUT], aux[NOUT];
    auto fetch = [&](int u, float* bv, float* av) {
      const int nvalid = min(16, n_rows - u * 16);
#pragma unroll
      for (int k = 0; k < NOUT; ++k) {
        const int o = etid + k * NE, token = o >> 4, rloc = o & 15;
        bv[k] = 0.f; av[k] = 0.f;
        if (o < 256 && token < T && rloc < nvalid && !ksplit) {
          const float* bias = sd->bias;
          const int row = n_begin + u * 16 + rloc;
          if (ln) {
            const float2 bc = reinterpret_cast<const float2*>(bias)[row];
            bv[k] = bc.x; av[k] = bc.y;
          } else {
            if (bias) bv[k] = bias[row];
            if (epi == EPI_RESID) av[k] = ldcg_f(&sd->out[(size_t)token * sd->ldo + row]);
          }
        }
      }
    };
    fetch(0, bias_v, aux);
    // residual epilogues before a LayerNorm stage: that stage's gamma is on its way into the gamma region (the copy is
    // issued when this stage begins; its phase is consumed by the LayerNorm stage)
    if (sd->out_gx) while (!mbar_try_wait(pbar, rs.ppar)) { }
    if (ln) asm volatile("bar.sync 4, %0;" ::"n"(NE) : "memory");   // LayerNorm statistics written
    for (int u = 0; u < units; ++u) {
      const int nvalid = min(16, n_rows - u * 16);
      asm volatile("bar.sync 2, %0;" ::"n"(WM_DEC_THREADS) : "memory");   // partials of unit u are written
      float sum[NOUT];
#pragma unroll
      for (int k = 0; k < NOUT; ++k) {
        const int o = etid + k * NE, token = o >> 4, rloc = o & 15;
        sum[k] = 0.f;
        if (o < 256 && token < T && rloc < nvalid) {
          // where the MMA fragment layout put (token, rloc): accumulator (j = n8 tile, i = register) of lane (g, t)
          const int idx = (((rloc >> 3) * 4) + ((token >= 8) ? 2 : 0) + (rloc & 1)) * 32 + (token & 7) * 4 + ((rloc & 7) >> 1);
#pragma unroll
          for (int ks = 0; ks < G::NKS; ++ks) sum[k] += partial[ks * 256 + idx];
        }
      }
      if (u + 1 < units) asm volatile("bar.arrive 3, %0;" ::"n"(WM_DEC_THREADS) : "memory");
      float* out = sd->out;
      const int ldo = sd->ldo;
#pragma unroll
      for (int k = 0; k < NOUT; ++k) {
        const int o = etid + k * NE, token = o >> 4, rloc = o & 15;
        if (!(o < 256 && token < T && rloc < nvalid)) continue;
        const int row = n_begin + u * 16 + rloc;
        const float s = sum[k];
        float y;   // the GEMM output with its bias
        if (ln) {
          const float2 st = s_stat[token];
          y = st.y * (s - st.x * aux[k]) + bias_v[k];
        } else {
          y = s + bias_v[k];
        }
        // common epilogues inline; the Medusa-head ones are rare
        if (ksplit) {
          m->gemm_part[((size_t)sd->seg * 16 + token) * sd->N + row] = s;
        } else if (epi == EPI_RESID) {
          const float v = aux[k] + y;
          out[(size_t)token * ldo + row] = v;
          if (sd->out_gx) store_split(sd->out_gx + (size_t)token * ldo, row, gamma[row] * v);
        } else if (epi == EPI_STORE || epi == EPI_LOGITS) {
          out[(size_t)token * ldo + row] = y;
        } else if (epi == EPI_GELU) {
          const float v = gelu_erf(y);
          if (sd->out_split) store_split(out + (size_t)token * ldo, row, v);
          else out[(size_t)token * ldo + row] = v;
        } else if (epi == EPI_QKV) {
          const float v = y;
          const DecLayer& L = m->layers[sd->layer];
          if (row < D) out[(size_t)token * ldo + row] = v;
          else if (row < 2 * D) L.self_k[self_kv_index(base + token, row - D)] = __float2half_rn(v);
          else L.self_v[self_kv_index(base + token, row - 2 * D)] = __float2half_rn(v);
        } else if (epi == EPI_HEADS_A || epi == EPI_HEADS_D) {
          // head `row / d`: x + SiLU(W x + b)  (medusa ResBlock), on the newest token's hidden state (A: the one staged
          // row) or, in later head layers, on its own row of the previous layer (D: row `head`, the others discarded)
          const int head = row / D, n = row - head * D;
          if (epi == EPI_HEADS_A || token == head)
            out[(size_t)(sd->out_row0 + head) * ldo + n] = xbuf_value(xb, G::XS, token, n) + silu(y);
        } else {   // EPI_HEAD_B
          out[(size_t)token * ldo + row] = xbuf_value(xb, G::XS, token, row) + silu(y);
        }
      }
      if (u + 1 < units) fetch(u + 1, bias_v, aux);   // (fetching TWO units ahead into a second register set timed slower)
    }
    for (int u = 0; u < units; ++u)
      if (++rs.slot == WM_RING_G) { rs.slot = 0; rs.par ^= 1u; }   // keep the (uniform) ring state in step with the MMA warps
  }
  cta_sync();   // every store of the stage issued; partial buffer and X buffer free
  if (pr) pr[14] = global_timer_ns();
  if (ksplit) {
    // the last of the `segs` CTAs of this row block folds the segment partials, always in segment order
    const int segs = sd->segs, block = sd->block, N = sd->N;
    if (tid == 0) {
      const unsigned int prev = atom_add_release(&m->gemm_cnt[block], 1u);   // (the unit loop ended with a cta_sync)
      s_last = (prev == (unsigned int)(segs - 1)) ? 1 : 0;
      if (s_last) m->gemm_cnt[block] = 0u;
    }
    cta_sync();
    if (s_last) {
      if (sd->out_gx) while (!mbar_try_wait(pbar, rs.ppar)) { }   // (see the epilogue above)
      const float* bias = sd->bias;
      float* out = sd->out;
      const int ldo = sd->ldo;
      // warp per token row, lanes over the rows of W; K-split stages are residual GEMMs (FC2)
      for (int t = warp; t < T; t += nwarps) {
        for (int r = lane; r < n_rows; r += 32) {
          const int row = n_begin + r;
          float* o = out + (size_t)t * ldo + row;
          // all loads in flight together (batches of 4 segments), summed in segment order
          const float xo = ldcg_f(o);
          const float bv = bias ? bias[row] : 0.f;
          float s = 0.f;
          for (int s0 = 0; s0 < segs; s0 += 4) {
            float pv[4];
#pragma unroll
            for (int i = 0; i < 4; ++i)
              if (s0 + i < segs) pv[i] = __ldcg(m->gemm_part + ((size_t)(s0 + i) * 16 + t) * N + row);
#pragma unroll
            for (int i = 0; i < 4; ++i)
              if (s0 + i < segs) s += pv[i];
          }
          const float v = xo + (s + bv);
          *o = v;
          if (sd->out_gx) store_split(sd->out_gx + (size_t)t * ldo, row, gamma[row] * v);
        }
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// cross-attention fed from the ring: the K rows and the V rows of this CTA's (head, key chunk) item
// arrive as two ring chunks, prefetched by the producer while the preceding stages run; the MMAs
// read them in place (the cache rows already have the 72-half shared-memory stride).
// ---------------------------------------------------------------------------------------------
template <int D>
__device__ __forceinline__ void stage_cross_attn_ring(RingState& rs, unsigned char* smem, const DecModel* m, const CtaStage* sd,
                                                      int T, int cta, int ncta, unsigned long long* pr) {
  using G = RingGeom<D>;
  uint64_t* const full = reinterpret_cast<uint64_t*>(smem + G::BAR_OFF);
  uint64_t* const empty = full + WM_RING_G;
  const CrossScratch cs = cross_scratch(smem + G::SCRATCH_OFF);
  const int H = m->H, S = m->S, nch = m->cross_chunks;
  const int tid = threadIdx.x;
  for (int item = cta; item < H * nch; item += ncta) {
    const CrossItem it = cross_item(item, S, nch);
    const int h = it.h, c = it.c, nk = it.nk;
    if (nk == 0) continue;   // (no chunks in the table either)
    const int nk_pad = (nk + 15) & ~15;
    const int slot_k = rs.slot;
    const unsigned int par_k = rs.par;
    if (++rs.slot == WM_RING_G) { rs.slot = 0; rs.par ^= 1u; }
    const int slot_v = rs.slot;
    const unsigned int par_v = rs.par;
    if (++rs.slot == WM_RING_G) { rs.slot = 0; rs.par ^= 1u; }
    __half* sK = reinterpret_cast<__half*>(smem + (size_t)slot_k * G::SLOT_BYTES);
    __half* sV = reinterpret_cast<__half*>(smem + (size_t)slot_v * G::SLOT_BYTES);
    while (!mbar_try_wait(full + slot_k, par_k)) { }
    while (!mbar_try_wait(full + slot_v, par_v)) { }
    if (pr) pr[3] = global_timer_ns();
    // rows nk .. nk_pad read as zero (their probabilities are zero, but 0 * stale bits could be NaN)
    for (int idx = tid; idx < (nk_pad - nk) * 9; idx += WM_DEC_THREADS) {
      reinterpret_cast<uint4*>(sK)[nk * 9 + idx] = make_uint4(0, 0, 0, 0);
      reinterpret_cast<uint4*>(sV)[nk * 9 + idx] = make_uint4(0, 0, 0, 0);
    }
    cross_attn_core<true>(
        m, T, h, c, nch, nk, nk_pad, sK, sV, cs,
        [&] { if (tid == 0) mbar_arrive_n(empty + slot_k, G::NKS); },
        [&] { if (tid == 0) mbar_arrive_n(empty + slot_v, G::NKS); },
        [&](const float* s) { ts_capture(m, sd->mode, sd->layer, T, h, c, nch, nk, s); }, pr);
  }
}

// ---------------------------------------------------------------------------------------------
// self-attention fed from the ring: the keys [0, P) of each item, P = min(base, kv0), arrive as K chunks and then V
// chunks of up to WM_SA_BLOCK keys (sa_prefix_chunk), streamed while QKV and its barrier run.  Only the query rows and
// the keys [P, nk_max) (the pass's own rows, and those sweep A wrote in this launch) come from L2, in one round, into
// the staging rows behind the scratch.  Items, the thread of each (row, key) pair and every sum are those of
// stage_self_attn, so the results are the same bits.
// ---------------------------------------------------------------------------------------------
template <int D>
__device__ __forceinline__ void stage_self_attn_ring(RingState& rs, unsigned char* smem, const DecModel* m, int mode, int layer,
                                                     int cta, int ncta, const PassGeom& g, int L0, int kv0,
                                                     unsigned long long* pr) {
  using G = RingGeom<D>;
  uint64_t* const full = reinterpret_cast<uint64_t*>(smem + G::BAR_OFF);
  uint64_t* const empty = full + WM_RING_G;
  float* const s_q = reinterpret_cast<float*>(smem + G::SCRATCH_OFF);
  __half* const sKn = reinterpret_cast<__half*>(smem + G::SCRATCH_OFF + self_attn_smem_bytes());   // [WM_SA_NEW][72]
  __half* const sVn = sKn + WM_SA_NEW * WM_KV_ROW;
  const int H = m->H;
  const DecLayer& L = m->layers[layer];
  const int tid = threadIdx.x;
  const bool tree_mask = (mode == MODE_B) && m->has_tree && m->st->tree_attn;
  const SelfAttnSplit sp = self_attn_split(H, g.T, ncta);
  const int P = min(g.base, kv0);
  int k = 0;
  for (int item = cta; item < H * sp.groups; item += ncta, ++k) {
    const int h = item / sp.groups, t0 = (item - h * sp.groups) * sp.R;
    const int rg = min(sp.R, g.T - t0);
    const int nnew = g.base + t0 + rg - P;
    // ring chunks of the item: nb K blocks, then nb V blocks, in consecutive slots
    int nb = 0;
    for (int b = 0; b < WM_SA_BLOCKS; ++b)
      if (sa_prefix_chunk(H, ncta, cta, mode, L0, kv0, m->n_tree, k, b).nk > 0) nb = b + 1;
    auto slot_of = [&](int i, unsigned int& par) {
      const int s = rs.slot + i;
      par = rs.par ^ (s >= WM_RING_G ? 1u : 0u);
      return s >= WM_RING_G ? s - WM_RING_G : s;
    };
    unsigned int pk0, pk1;
    const __half* const sK0 = reinterpret_cast<const __half*>(smem + (size_t)slot_of(0, pk0) * G::SLOT_BYTES);
    const __half* const sK1 = reinterpret_cast<const __half*>(smem + (size_t)slot_of(1, pk1) * G::SLOT_BYTES);
    unsigned int pv0, pv1;
    const __half* const sV0 = reinterpret_cast<const __half*>(smem + (size_t)slot_of(nb, pv0) * G::SLOT_BYTES);
    const __half* const sV1 = reinterpret_cast<const __half*>(smem + (size_t)slot_of(nb + 1, pv1) * G::SLOT_BYTES);
    if (pr && k == 0) {
      pr[11] = (nb == 0 || mbar_try_wait(full + slot_of(nb - 1, pk1), pk1)) ? 1000ull : 0ull;   // K prefix here at begin?
      pr[12] = (nb == 0 || mbar_try_wait(full + slot_of(nb, pv0), pv0)) ? 1000ull : 0ull;       // first V block?
    }
    cta_sync();   // (the previous item's readers of the scratch are done)
    for (int idx = tid; idx < rg * 64; idx += WM_DEC_THREADS)
      s_q[idx] = ldcg_f(&m->q[(size_t)(t0 + (idx >> 6)) * D + h * 64 + (idx & 63)]);
    // 16 bytes per thread: (row, K | V, 8 dims)
    for (int idx = tid; idx < nnew * 16; idx += WM_DEC_THREADS) {
      const int r = idx >> 4, v = (idx >> 3) & 1, c = (idx & 7) * 8;
      const __half* src = (v ? L.self_v : L.self_k) + self_kv_index(P + r, h * 64 + c);
      *reinterpret_cast<uint4*>((v ? sVn : sKn) + r * WM_KV_ROW + c) = ldcg_u4(src);
    }
    cta_sync();
    if (pr) pr[3] = global_timer_ns();
    for (int i = 0; i < nb; ++i) {
      unsigned int p;
      const int s = slot_of(i, p);
      while (!mbar_try_wait(full + s, p)) { }
    }
    auto row = [&](const __half* s0, const __half* s1, const __half* sn, int j) {
      return j < P ? (j < WM_SA_BLOCK ? s0 + j * WM_KV_ROW : s1 + (j - WM_SA_BLOCK) * WM_KV_ROW) : sn + (j - P) * WM_KV_ROW;
    };
    self_attn_item<true>(
        m, g, tree_mask, h, t0, rg, s_q,
        [&](int j, uint4* a) {
          const uint4* k0 = reinterpret_cast<const uint4*>(row(sK0, sK1, sKn, j));
#pragma unroll
          for (int c = 0; c < 8; ++c) a[c] = k0[c];
        },
        [&](int j, int dg) { return *reinterpret_cast<const uint4*>(row(sV0, sV1, sVn, j) + dg * 8); },
        [&] {
          if (tid == 0)
            for (int i = 0; i < nb; ++i) { unsigned int p; mbar_arrive_n(empty + slot_of(i, p), G::NKS); }
        },
        [&] {
          for (int i = nb; i < 2 * nb; ++i) {
            unsigned int p;
            const int s = slot_of(i, p);
            while (!mbar_try_wait(full + s, p)) { }
          }
        },
        [&] {
          if (tid == 0)
            for (int i = nb; i < 2 * nb; ++i) { unsigned int p; mbar_arrive_n(empty + slot_of(i, p), G::NKS); }
        },
        pr);
    for (int i = 0; i < 2 * nb; ++i)
      if (++rs.slot == WM_RING_G) { rs.slot = 0; rs.par ^= 1u; }
  }
}

// LP: the logits scans with the logits-processor term (dec_state_adj); SMP: a sampled attempt's scans and folds (DecState
// smp_on; processors chosen at run time); the profiling variant chooses processors at run time
template <int D, bool PROF, bool LP, bool SMP = false>
__global__ void __launch_bounds__(WM_RING_THREADS, 1)
dec_iteration_ring_kernel(const DecModel* __restrict__ gm) {
  using G = RingGeom<D>;
  extern __shared__ __align__(128) unsigned char smem[];
  const DecState* st = gm->st;
  if (st->done) return;
  const int need_a = st->need_a;
  const int L0 = st->L, kv0 = st->kv_len;
  const int cta = blockIdx.x, ncta = gridDim.x;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  DecModel* const sm = reinterpret_cast<DecModel*>(smem + G::MODEL_OFF);   // shared-memory copy of the model description
  uint64_t* const full = reinterpret_cast<uint64_t*>(smem + G::BAR_OFF);
  uint64_t* const empty = full + WM_RING_G;
  uint64_t* const xbar = empty + WM_RING_G;
  uint64_t* const pbar = xbar + 1;
  if (threadIdx.x == 0) {
    for (int i = 0; i < WM_RING_G; ++i) { mbar_init(full + i, 1); mbar_init(empty + i, G::NKS); }   // a slot is released by every MMA warp
    mbar_init(xbar, 1);
    mbar_init(pbar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  {
    const int4* src = reinterpret_cast<const int4*>(gm);
    int4* dst = reinterpret_cast<int4*>(sm);
    // (sizeof(DecModel) is a multiple of 16: alignas(16))
    for (int i = threadIdx.x; i < (int)((sizeof(DecModel) + 15) / 16); i += WM_RING_THREADS) dst[i] = src[i];
  }
  __syncthreads();   // the only full-CTA barrier: after it the producer warp goes its own way
  // Clustered launch: the peer multicasts into this CTA's xbar as soon as its first GEMM stage begins, and with
  // need_a = 0 that is the HEADS stage, with no grid barrier before it.  So every thread of both CTAs passes one cluster
  // barrier after the mbarrier initialisation (released to the cluster above) and before any stage runs.
  if (cluster_ncta() > 1) cluster_sync_all();
  const DecModel* m = sm;

  if (warp == WM_DEC_THREADS / 32) {
    // ===== producer warp =====
    const int* off = m->chunk_off + cta * 4;
    ring_producer<D>(smem, full, empty, m->chunk_tab, need_a ? off[0] : off[1], st->prefill ? off[1] : off[3], off[1], off[3],
                     m, cta, ncta, L0, kv0);
    return;
  }

  // ===== compute warps =====
  __shared__ CtaStage s_desc[2];   // resolved record of the running stage / the next one
  unsigned int epoch = *reinterpret_cast<volatile unsigned int*>(&m->bar[2]);
  RingState rs;
  rs.slot = 0; rs.par = 0u; rs.xpar = 0u; rs.ppar = 0u;

  const int ip_first = need_a ? m->prog_off[0] : m->prog_off[1];
  const int ip_last = st->prefill ? m->prog_off[1] : m->prog_off[3];   // prefill: sweep A only (a chunk of a long prompt)
  const CtaStage* tab = m->stage_tab + cta;   // record of instruction ip: tab[ip * ncta]
  if (warp == 0)
    reinterpret_cast<uint32_t*>(&s_desc[ip_first & 1])[lane] = reinterpret_cast<const uint32_t*>(tab + (size_t)ip_first * ncta)[lane];
  cta_sync();
  for (int ip = ip_first; ip < ip_last; ++ip) {
    const CtaStage* sd = &s_desc[ip & 1];
    // the next record is fetched while this stage runs (and the one after it pulled into L2)
    uint32_t nxt_w = 0u;
    const bool fetch = (warp == (WM_DEC_THREADS / 32 - 1)) && (ip + 1 < ip_last);
    if (fetch) {
      nxt_w = reinterpret_cast<const uint32_t*>(tab + (size_t)(ip + 1) * ncta)[lane];
      if (lane == 0 && ip + 2 < ip_last) prefetch_l2(tab + (size_t)(ip + 2) * ncta);
    }
    // optional per-stage timeline (CTA 0 and the last CTA): begin / end of body / end of barrier
    const bool prof = PROF && m->prof != nullptr && threadIdx.x == 0 && (cta == 0 || cta == ncta - 1);
    unsigned long long* pr = prof ? m->prof + ((size_t)(cta == 0 ? 0 : 1) * ip_last + ip) * 16 : nullptr;
    if (prof) pr[0] = global_timer_ns();
    const int stage = sd->stage, mode = sd->mode;
    // the pass geometry derives from (L0, kv0): the loop state only changes in the very last stage
    const PassGeom pgv = pass_geom(mode, L0, kv0, m->n_tree);
    // LayerNorm gamma of the next stage -> its region (last read by an earlier LayerNorm stage; a LayerNorm stage never
    // precedes another), in flight while this stage runs: its residual epilogue (if any) reads it too
    if (threadIdx.x == 0 && sd->nx_g != nullptr) {
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      mbar_expect_tx(pbar, (uint32_t)(D * 4));
      bulk_g2s(smem + G::GAMMA_OFF, sd->nx_g, (uint32_t)(D * 4), pbar);
    }
    if (is_gemm_stage(stage)) {
      stage_gemm_ring<D>(rs, smem, m, sd, pgv.T, pgv.base, pr);
    } else if (stage == ST_CROSS_ATTN) {
      stage_cross_attn_ring<D>(rs, smem, m, sd, pgv.T, cta, ncta, pr);
    } else if (stage == ST_SELF_ATTN) {
      stage_self_attn_ring<D>(rs, smem, m, mode, sd->layer, cta, ncta, pgv, L0, kv0, pr);
    } else {
      run_stage<false, (PROF || SMP) ? -1 : (LP ? 1 : 0), SMP>(m, stage, mode, sd->layer, cta, ncta,
                                                                      smem + G::SCRATCH_OFF, &pgv, pr);
    }
    if (prof) pr[15] = global_timer_ns();
    if (fetch) reinterpret_cast<uint32_t*>(&s_desc[(ip + 1) & 1])[lane] = nxt_w;
    if (prof) pr[1] = global_timer_ns();
    epoch = grid_barrier_step<false>(m->bar, epoch, ncta);
    if (prof) pr[2] = global_timer_ns();
  }
  // Every instruction ends in a grid barrier, and a CTA arrives there only after its xbar phase of the stage completed,
  // i.e. after every multicast byte addressed to it landed.  So past the last barrier no multicast is in flight and
  // nothing targets the peer's shared memory: the CTAs of a cluster may exit independently.
  if (blockIdx.x == 0 && threadIdx.x == 0) m->bar[2] = epoch;
}

// model widths the ring kernel is instantiated for (Whisper tiny ... large, and the synthetic micro preset)
#define WM_RING_WIDTHS(X) X(128) X(384) X(512) X(768) X(1024) X(1280)
