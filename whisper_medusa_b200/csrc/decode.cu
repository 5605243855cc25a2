// Decode-side kernels of the Medusa speculative loop (sm_90a).
//
// One speculative iteration = pass A (the not-yet-cached token(s), all K+1 heads) followed by
// pass B (verify: the K+1 candidate tokens, base head only) -- reference model.py:635-793 and
// SURVEY.md 3.3.  Every pass is a chain of "stages"; a stage is a __device__ function written
// for an arbitrary (cta, n_cta) so that the same code runs either as its own kernel launch
// (mode 0: one CUDA graph per pass) or inside the persistent cooperative kernel (mode 1: one
// launch per iteration, grid barriers between stages).
//
// Numerics: fp16 weights, fp16 self/cross K/V caches, fp32 activations and accumulation.  The
// skinny GEMMs (T <= 16 rows) run on mma.sync m16n8k16 with the fp32 activation split into
// fp16 hi + lo parts (two MMAs), which keeps ~22 mantissa bits of the activation; the path is
// HBM-bound (weights are streamed exactly once per pass), not tensor-bound.
#include <algorithm>
#include <vector>

#include "common.cuh"
#include "engine.h"

namespace wm {

__device__ __forceinline__ unsigned long long wm_timer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// -----------------------------------------------------------------------------------------
// pass geometry (uniform across the grid; read from the loop state)
// -----------------------------------------------------------------------------------------
// MODE_A   : sweep over the tokens that are not cached yet (prompt, or the extra token after an
//            accept-0 iteration): rows ids[kv_len .. L)
// MODE_B   : verify sweep over the K+1 candidate tokens at positions L .. L+K
// MODE_TAIL: block type only -- the medusa block re-run on the carried hidden state of the newest
//            cached token (position L-1) to feed the heads
enum { MODE_A = 0, MODE_B = 1, MODE_TAIL = 2 };
struct PassGeom {
  int T;     // query rows of this pass
  int base;  // position of row 0 (also the self-KV row it writes)
};
// L, kv_len: the loop state's; n_tree: rows of the verify pass
__host__ __device__ __forceinline__ PassGeom pass_geom(int mode, int L, int kv_len, int n_tree) {
  PassGeom g;
  if (mode == MODE_A) {
    g.T = L - kv_len;
    g.base = kv_len;
  } else if (mode == MODE_B) {
    g.T = n_tree;
    g.base = L;
  } else {
    g.T = 1;
    g.base = L - 1;
  }
  return g;
}
__device__ __forceinline__ PassGeom pass_geom(const DecModel* m, int mode) {
  return pass_geom(mode, m->st->L, m->st->kv_len, m->n_tree);
}

// -----------------------------------------------------------------------------------------
// stage: token + position embedding  (HF modeling_whisper.py:737-763)
// -----------------------------------------------------------------------------------------
__device__ __forceinline__ void stage_embed(const DecModel* m, int mode, int cta, int ncta, const PassGeom* gopt) {
  const PassGeom g = gopt ? *gopt : pass_geom(m, mode);
  const DecState* st = m->st;
  const int d = m->d;
  for (int t = cta; t < g.T; t += ncta) {
    int tok = (mode == MODE_A) ? ldcg_i(&st->ids[g.base + t]) : ldcg_i(&st->cand[t]);
    const __half* e = m->embed + (size_t)tok * d;
    // verify rows of a candidate tree sit at position L + depth (medusa_position_ids, medusa_utils.py:494-496)
    const int posn = (mode == MODE_B && m->has_tree) ? g.base + m->tree->depth[t] : g.base + t;
    const float* p = m->pos + (size_t)posn * d;
    float* x = m->x + (size_t)t * d;
    for (int j = threadIdx.x; j < d; j += WM_DEC_THREADS) x[j] = __half2float(e[j]) + p[j];
  }
}

// -----------------------------------------------------------------------------------------
// skinny GEMM  y[t, n] = sum_k X[t, k] * W[n, k]   (t < 16 rows, W fp16 [N, K] row-major)
// -----------------------------------------------------------------------------------------
enum XSrc { XS_LN = 0, XS_PLAIN = 1 };
enum Epi { EPI_QKV = 0, EPI_RESID, EPI_STORE, EPI_GELU, EPI_HEADS_A, EPI_HEAD_B, EPI_LOGITS, EPI_HEADS_D };

struct GemmDesc {
  const __half* W;
  const float* bias;   // may be null
  int N, K;
  // X source
  int xsrc;            // XSrc
  const float* X;      // [rows, K] fp32 (for XS_LN: the residual stream)
  int x_row0;          // first source row
  int x_rows;          // number of valid rows (<= 16)
  const float *ln_g, *ln_b;
  // epilogue
  int epi;
  float* out;          // EPI_STORE/GELU/LOGITS/HEAD*: destination [16, ldo]; EPI_RESID: residual stream
  int ldo;
  int out_row0;        // EPI_HEADS_A / EPI_HEADS_D: destination row of head 0
  __half *kc, *vc;     // EPI_QKV: self K/V cache rows
  int base;            // EPI_QKV: cache row of token 0
  int d;               // model dim (EPI_QKV / EPI_HEADS_A)
};

#define WM_XPAD 32  // halfs of padding per smem activation row => row stride = 64 B (mod 128 B): conflict-free LDS.128
#define WM_MAXR 3   // max (unit, k-slice) items per warp

// K is processed in `nph` phases of KPH columns so the fp16 hi/lo activation slice fits in
// shared memory; KPH must be a multiple of 64 (bank-conflict-free row stride, 32-wide chunks).
__host__ __device__ inline int gemm_nphase(int K) {
  int nph = (K + 2047) / 2048;
  while (K % (nph * 64) != 0) ++nph;
  return nph;
}

// dynamic shared memory layout of a GEMM stage
//   xhi [16][KPH + 32] half | xlo [16][KPH + 32] half | partial [items][256] float
__host__ __device__ inline size_t gemm_smem_bytes(int K) {
  int nph = gemm_nphase(K);
  int kph = K / nph;
  return (size_t)2 * 16 * (kph + WM_XPAD) * sizeof(__half) + (size_t)(2 * 16 + 8) * 256 * sizeof(float);
}

__device__ __forceinline__ void gemm_epilogue(const GemmDesc& g, int token, int row, float v,
                                              const __half* xhi, const __half* xlo, int xstride) {
  if (g.bias) v += g.bias[row];
  switch (g.epi) {
    case EPI_QKV: {
      int d = g.d;
      if (row < d) {
        g.out[(size_t)token * g.ldo + row] = v;
      } else if (row < 2 * d) {
        g.kc[self_kv_index(g.base + token, row - d)] = __float2half_rn(v);
      } else {
        g.vc[self_kv_index(g.base + token, row - 2 * d)] = __float2half_rn(v);
      }
      break;
    }
    case EPI_RESID:
      g.out[(size_t)token * g.ldo + row] += v;
      break;
    case EPI_STORE:
    case EPI_LOGITS:
      g.out[(size_t)token * g.ldo + row] = v;
      break;
    case EPI_GELU:
      g.out[(size_t)token * g.ldo + row] = gelu_erf(v);
      break;
    case EPI_HEADS_A: {
      // stacked heads applied to ONE input row: row = head * d + n  (reference model.py:1274-1280)
      int head = row / g.d, n = row - head * g.d;
      float xv = __half2float(xhi[n]) + __half2float(xlo[n]);
      g.out[(size_t)(g.out_row0 + head) * g.ldo + n] = xv + silu(v);
      break;
    }
    case EPI_HEAD_B: {
      float xv = __half2float(xhi[(size_t)token * xstride + row]) + __half2float(xlo[(size_t)token * xstride + row]);
      g.out[(size_t)token * g.ldo + row] = xv + silu(v);
      break;
    }
    case EPI_HEADS_D: {
      // head layers after the first: head `row / d` on its own row of the previous layer (input row `head`); the
      // other rows' products of its column block are discarded
      int head = row / g.d, n = row - head * g.d;
      if (token == head) {
        float xv = __half2float(xhi[(size_t)token * xstride + n]) + __half2float(xlo[(size_t)token * xstride + n]);
        g.out[(size_t)(g.out_row0 + head) * g.ldo + n] = xv + silu(v);
      }
      break;
    }
  }
}

// Medusa-head epilogues of the ring kernel (rare: twice per iteration).  Out of line and with scalar
// arguments only, so that the GemmDesc of the caller never has to live in local memory.
__device__ __noinline__ void gemm_epilogue_heads(int epi, float* out, int ldo, int out_row0, int dm, float bias, int token,
                                                 int row, float v, const __half* xhi, const __half* xlo, int xstride) {
  v += bias;
  if (epi == EPI_HEADS_A) {
    const int head = row / dm, n = row - head * dm;
    const float xv = __half2float(xhi[n]) + __half2float(xlo[n]);
    out[(size_t)(out_row0 + head) * ldo + n] = xv + silu(v);
  } else {
    const float xv = __half2float(xhi[(size_t)token * xstride + row]) + __half2float(xlo[(size_t)token * xstride + row]);
    out[(size_t)token * ldo + row] = xv + silu(v);
  }
}

__device__ __noinline__ void stage_gemm(const GemmDesc& g, int cta, int ncta, unsigned char* smem_raw) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int nwarps = (WM_DEC_THREADS >> 5);
  const int gq = lane >> 2, tq = lane & 3;
  const int K = g.K, N = g.N;
  const int nph = gemm_nphase(K);
  const int KPH = K / nph;
  const int xstride = KPH + WM_XPAD;
  __half* xhi = reinterpret_cast<__half*>(smem_raw);
  __half* xlo = xhi + 16 * xstride;
  float* partial = reinterpret_cast<float*>(xlo + 16 * xstride);

  // balanced contiguous row range of this CTA
  const int rows_per = N / ncta, rem = N % ncta;
  const int n_begin = cta * rows_per + min(cta, rem);
  const int n_rows = rows_per + (cta < rem ? 1 : 0);
  const int n_end = n_begin + n_rows;
  const int units = (n_rows + 15) >> 4;
  int ksplit = 1;
  while (ksplit < 8 && units * ksplit * 2 <= nwarps && ((KPH / (ksplit * 2)) % 32) == 0) ksplit <<= 1;
  const int items = units * ksplit;   // host guarantees items <= WM_MAXR * nwarps and <= 40
  const int KS = KPH / ksplit;
  const int T = g.x_rows;

  float acc[WM_MAXR][8];
#pragma unroll
  for (int r = 0; r < WM_MAXR; ++r)
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[r][i] = 0.f;

  for (int ph = 0; ph < nph; ++ph) {
    // ---- stage the activation slice as fp16 hi/lo ----
    if (ph > 0) cta_sync();
    if (g.xsrc == XS_LN) {
      // LayerNorm over the full row (nph == 1 for LN stages: K = d <= 2048)
      for (int r = warp; r < 16; r += nwarps) {
        __half* hi = xhi + r * xstride;
        __half* lo = xlo + r * xstride;
        if (r < T) {
          const float* x = g.X + (size_t)(g.x_row0 + r) * K;
          float s = 0.f;
          for (int j = lane; j < K; j += 32) s += x[j];
          float mean = warp_sum(s) / (float)K;
          float v = 0.f;
          for (int j = lane; j < K; j += 32) { float dlt = x[j] - mean; v += dlt * dlt; }
          float rstd = rsqrtf(warp_sum(v) / (float)K + 1e-5f);
          for (int j = lane; j < K; j += 32) {
            float y = (x[j] - mean) * rstd * g.ln_g[j] + g.ln_b[j];
            __half h = __float2half_rn(y);
            hi[j] = h;
            lo[j] = __float2half_rn(y - __half2float(h));
          }
        } else {
          for (int j = lane; j < K; j += 32) { hi[j] = __float2half_rn(0.f); lo[j] = __float2half_rn(0.f); }
        }
      }
    } else {
      for (int idx = tid; idx < 16 * KPH; idx += WM_DEC_THREADS) {
        int r = idx / KPH, j = idx - r * KPH;
        float y = (r < T) ? g.X[(size_t)(g.x_row0 + r) * K + ph * KPH + j] : 0.f;
        __half h = __float2half_rn(y);
        xhi[r * xstride + j] = h;
        xlo[r * xstride + j] = __float2half_rn(y - __half2float(h));
      }
    }
    cta_sync();

    // ---- stream the weights ----
#pragma unroll
    for (int r = 0; r < WM_MAXR; ++r) {
      const int item = warp + r * nwarps;
      if (item < items) {
        const int u = item / ksplit, ks = item - u * ksplit;
        const int row0 = n_begin + u * 16 + gq, row1 = row0 + 8;
        const bool v0 = row0 < n_end, v1 = row1 < n_end;
        const __half* w0p = g.W + (size_t)(v0 ? row0 : n_begin) * K + (size_t)ph * KPH + 8 * tq;
        const __half* w1p = g.W + (size_t)(v1 ? row1 : n_begin) * K + (size_t)ph * KPH + 8 * tq;
        const __half* xh0 = xhi + gq * xstride + 8 * tq;
        const __half* xh1 = xhi + (gq + 8) * xstride + 8 * tq;
        const __half* xl0 = xlo + gq * xstride + 8 * tq;
        const __half* xl1 = xlo + (gq + 8) * xstride + 8 * tq;
        const int k0 = ks * KS, k1 = k0 + KS;
        float* c0 = &acc[r][0];
        float* c1 = &acc[r][4];
        for (int k = k0; k < k1; k += 128) {
          uint4 wa[4], wb[4];
#pragma unroll
          for (int c = 0; c < 4; ++c) {
            const int kk = k + 32 * c;
            wa[c] = make_uint4(0, 0, 0, 0);
            wb[c] = make_uint4(0, 0, 0, 0);
            if (kk < k1) {
              if (v0) wa[c] = ldg_nc_v4(w0p + kk);
              if (v1) wb[c] = ldg_nc_v4(w1p + kk);
            }
          }
#pragma unroll
          for (int c = 0; c < 4; ++c) {
            const int kk = k + 32 * c;
            if (kk < k1) {
              const uint4 ah0 = *reinterpret_cast<const uint4*>(xh0 + kk);
              const uint4 ah1 = *reinterpret_cast<const uint4*>(xh1 + kk);
              const uint4 al0 = *reinterpret_cast<const uint4*>(xl0 + kk);
              const uint4 al1 = *reinterpret_cast<const uint4*>(xl1 + kk);
              mma_16816(c0, ah0.x, ah1.x, ah0.y, ah1.y, wa[c].x, wa[c].y);
              mma_16816(c0, ah0.z, ah1.z, ah0.w, ah1.w, wa[c].z, wa[c].w);
              mma_16816(c0, al0.x, al1.x, al0.y, al1.y, wa[c].x, wa[c].y);
              mma_16816(c0, al0.z, al1.z, al0.w, al1.w, wa[c].z, wa[c].w);
              mma_16816(c1, ah0.x, ah1.x, ah0.y, ah1.y, wb[c].x, wb[c].y);
              mma_16816(c1, ah0.z, ah1.z, ah0.w, ah1.w, wb[c].z, wb[c].w);
              mma_16816(c1, al0.x, al1.x, al0.y, al1.y, wb[c].x, wb[c].y);
              mma_16816(c1, al0.z, al1.z, al0.w, al1.w, wb[c].z, wb[c].w);
            }
          }
        }
      }
    }
  }

  // ---- epilogue ----
  // accumulator element i of n-tile j: token = gq + (i >= 2 ? 8 : 0), weight row = unit*16 + j*8 + 2*tq + (i & 1)
  if (ksplit == 1) {
#pragma unroll
    for (int r = 0; r < WM_MAXR; ++r) {
      const int item = warp + r * nwarps;
      if (item < items) {
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          const int j = e >> 2, i = e & 3;
          const int token = gq + ((i >= 2) ? 8 : 0);
          const int row = n_begin + item * 16 + j * 8 + 2 * tq + (i & 1);
          if (token < T && row < n_end) gemm_epilogue(g, token, row, acc[r][e], xhi, xlo, xstride);
        }
      }
    }
  } else {
#pragma unroll
    for (int r = 0; r < WM_MAXR; ++r) {
      const int item = warp + r * nwarps;
      if (item < items) {
#pragma unroll
        for (int e = 0; e < 8; ++e) partial[(size_t)item * 256 + e * 32 + lane] = acc[r][e];
      }
    }
    cta_sync();
    for (int o = tid; o < units * 256; o += WM_DEC_THREADS) {
      const int u = o >> 8, el = o & 255;
      const int e = el >> 5, ln = el & 31;
      const int j = e >> 2, i = e & 3;
      const int token = (ln >> 2) + ((i >= 2) ? 8 : 0);
      const int row = n_begin + u * 16 + j * 8 + 2 * (ln & 3) + (i & 1);
      if (token < T && row < n_end) {
        float s = 0.f;
        for (int ks = 0; ks < ksplit; ++ks) s += partial[(size_t)(u * ksplit + ks) * 256 + el];
        gemm_epilogue(g, token, row, s, xhi, xlo, xstride);
      }
    }
  }
}

// -----------------------------------------------------------------------------------------
// stage: causal self-attention over the fp16 cache (HF modeling_whisper.py:284-357, T_q <= 16)
// item = (head, group of R query rows); R = ceil(H*T / n_cta) so that all items run in ONE wave.
// Row t sees keys 0 .. base + t.  Stage kernels read the K/V rows straight from L2; the ring kernel takes the cached
// prefix from ring slots (stage_self_attn_ring).
// -----------------------------------------------------------------------------------------
#define WM_SA_MAXR 4
#ifndef WM_SA_PV_UNROLL
#define WM_SA_PV_UNROLL 4   // independent K/V row loads in flight per thread in the P V loop
#endif
#define WM_PRAGMA_(x) _Pragma(#x)
#define WM_PRAGMA(x) WM_PRAGMA_(x)
#define WM_UNROLL(n) WM_PRAGMA(unroll n)
__host__ __device__ constexpr size_t self_attn_smem_bytes() {
  return (size_t)(WM_SA_MAXR * 64 + WM_SA_MAXR * WM_MAX_POS + 2 * WM_SA_MAXR + (WM_DEC_THREADS / 8) * 64) * sizeof(float);
}
__device__ __forceinline__ float dot64_h(const float* q, const uint4* kp) {
  float s = 0.f;
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    const uint4 kv = kp[c];
    const __half2* k2 = reinterpret_cast<const __half2*>(&kv);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float2 f = __half22float2(k2[e]);
      s = fmaf(q[c * 8 + 2 * e], f.x, s);
      s = fmaf(q[c * 8 + 2 * e + 1], f.y, s);
    }
  }
  return s;
}
// Items of the stage: item = (head, group of R query rows), R = ceil(H * T / ncta) within [1, WM_SA_MAXR]; item i is
// head i / groups, rows from (i % groups) * R.
struct SelfAttnSplit { int R, groups; };
__host__ __device__ __forceinline__ SelfAttnSplit self_attn_split(int H, int T, int ncta) {
  SelfAttnSplit s;
  s.R = (H * T + ncta - 1) / ncta;
  if (s.R > WM_SA_MAXR) s.R = WM_SA_MAXR;
  if (s.R < 1) s.R = 1;
  s.groups = (T + s.R - 1) / s.R;
  return s;
}

// Ring kernel: the cached keys of a self-attention item that every row of the pass sees and that were written before
// the launch, [0, min(base, kv0)), stream through the weight ring as blocks of up to WM_SA_BLOCK keys, a K and a V
// chunk per block (at most WM_SA_BLOCKS, since WM_MAX_POS = 512).  Block `b` of the `k`-th item of CTA `cta` in a pass
// of `mode`: head h, keys [j0, j0 + nk); nk = 0 when the item or the block does not exist at this launch's (L0, kv0).
// The producer warp (which chunks it copies) and the compute warps (which slots they take) both decide from here.
#define WM_SA_BLOCK 256
#define WM_SA_BLOCKS (WM_MAX_POS / WM_SA_BLOCK)
static_assert(WM_SA_BLOCK <= WM_CH_MAX_KEYS, "a self-attention prefix block must fit one ring slot, as a cross-attention chunk does");
struct SaChunk { int h, j0, nk; };
__host__ __device__ __forceinline__ SaChunk sa_prefix_chunk(int H, int ncta, int cta, int mode, int L0, int kv0, int n_tree,
                                                            int k, int b) {
  const PassGeom g = pass_geom(mode, L0, kv0, n_tree);
  const SelfAttnSplit s = self_attn_split(H, g.T, ncta);
  const int item = cta + k * ncta;
  SaChunk c;
  c.h = item / s.groups;
  c.j0 = b * WM_SA_BLOCK;
  const int n = min(g.base, kv0) - c.j0;
  c.nk = (item < H * s.groups && n > 0) ? min(n, WM_SA_BLOCK) : 0;
  return c;
}

// One (head, row group) item once its query rows are in s_q (and visible to the CTA).  Key j's row of K is loaded by
// kload(j, a) into a[0..7] (its 64 dims), dims 8 dg .. 8 dg + 7 of V's row j by vload(j, dg).  after_qk runs once no
// thread reads K any more, before_pv before the first read of V, after_pv once no thread reads V any more.
template <bool SPLIT_OUT, class KLoad, class VLoad, class AfterQK, class BeforePV, class AfterPV>
__device__ __forceinline__ void self_attn_item(const DecModel* m, const PassGeom& g, bool tree_mask, int h, int t0, int rg,
                                               float* s_q, KLoad kload, VLoad vload, AfterQK after_qk, BeforePV before_pv,
                                               AfterPV after_pv, unsigned long long* pr) {
  const int d = m->d;
  float* s_p = s_q + WM_SA_MAXR * 64;                              // [R][WM_MAX_POS]
  float* s_st = s_p + WM_SA_MAXR * WM_MAX_POS;                     // [R] sum
  float* s_acc = s_st + 2 * WM_SA_MAXR;                            // [WM_DEC_THREADS / 8 groups][64]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int nk_max = g.base + t0 + rg;           // keys of the last row of the group
  // scores (scaled by head_dim^-0.5; HF scales q, a power of two, so this is identical)
  const int npairs = rg * nk_max;
  for (int i0 = tid; i0 < npairs; i0 += WM_DEC_THREADS) {
    const int r0 = i0 / nk_max, j0 = i0 - r0 * nk_max;
    uint4 a[8];
    kload(j0, a);
    bool ok0 = j0 <= g.base + t0 + r0;           // causal (over cache order: what the reference does for trees too)
    if (tree_mask && j0 >= g.base) ok0 = ok0 && ((m->tree->anc[t0 + r0] >> (j0 - g.base)) & 1u);   // ancestors only
    s_p[r0 * WM_MAX_POS + j0] = ok0 ? dot64_h(s_q + r0 * 64, a) * 0.125f : -INFINITY;
  }
  cta_sync();
  after_qk();
  if (pr) pr[4] = wm_timer_ns();
  // softmax statistics: one warp per row
  for (int r = warp; r < rg; r += (WM_DEC_THREADS >> 5)) {
    const int nk = g.base + t0 + r + 1;
    float* p = s_p + r * WM_MAX_POS;
    float mx = -INFINITY;
    for (int jj = lane; jj < nk; jj += 32) mx = fmaxf(mx, p[jj]);
    mx = warp_max(mx);
    float sum = 0.f;
    for (int jj = lane; jj < nk; jj += 32) { const float e = expf(p[jj] - mx); p[jj] = e; sum += e; }
    sum = warp_sum(sum);
    if (lane == 0) s_st[r] = sum;
  }
  cta_sync();
  if (pr) pr[5] = wm_timer_ns();
  before_pv();
  // P * V : thread = (row r, key group kg, dim group dg of 8 dims)
  {
    const int KG = (WM_DEC_THREADS / 8) / rg;
    const int dg = tid & 7, gI = tid >> 3;       // groups of 8 threads
    const int r = gI / KG, kg = gI - r * KG;
    float a[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) a[e] = 0.f;
    if (r < rg) {
      const int nk = g.base + t0 + r + 1;
      const float* p = s_p + r * WM_MAX_POS;
      WM_UNROLL(WM_SA_PV_UNROLL)
      for (int jj = kg; jj < nk; jj += KG) {
        const uint4 vv = vload(jj, dg);
        const __half2* v2 = reinterpret_cast<const __half2*>(&vv);
        const float pj = p[jj];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float2 f = __half22float2(v2[e]);
          a[2 * e] = fmaf(pj, f.x, a[2 * e]);
          a[2 * e + 1] = fmaf(pj, f.y, a[2 * e + 1]);
        }
      }
    }
#pragma unroll
    for (int e = 0; e < 8; ++e) s_acc[gI * 64 + dg * 8 + e] = a[e];
    cta_sync();
    after_pv();
    if (pr) pr[6] = wm_timer_ns();
    if (tid < rg * 64) {
      const int rr = tid >> 6, c = tid & 63;
      float o = 0.f;
      for (int k2 = 0; k2 < KG; ++k2) o += s_acc[(rr * KG + k2) * 64 + c];
      if (SPLIT_OUT) store_split(m->attn + (size_t)(t0 + rr) * d, h * 64 + c, o / s_st[rr]);   // (ring kernel: operand format of the O-projection)
      else m->attn[(size_t)(t0 + rr) * d + h * 64 + c] = o / s_st[rr];
    }
  }
}

__device__ __forceinline__ void stage_self_attn(const DecModel* m, int mode, int layer, int cta, int ncta, unsigned char* smem_raw,
                                                const PassGeom* gopt, unsigned long long* pr = nullptr) {
  const PassGeom g = gopt ? *gopt : pass_geom(m, mode);
  const int d = m->d, H = m->H;
  const DecLayer& L = m->layers[layer];
  float* s_q = reinterpret_cast<float*>(smem_raw);                 // [R][64], then the rest of self_attn_smem_bytes()
  const int tid = threadIdx.x;
  const bool tree_mask = (mode == MODE_B) && m->has_tree && m->st->tree_attn;   // (tree_attn is constant during a generate call)
  const SelfAttnSplit sp = self_attn_split(H, g.T, ncta);
  const int R = sp.R, groups = sp.groups;
  for (int item = cta; item < H * groups; item += ncta) {
    const int h = item / groups, t0 = (item - h * groups) * R;
    const int rg = min(R, g.T - t0);               // rows in this group
    cta_sync();
    for (int idx = tid; idx < rg * 64; idx += WM_DEC_THREADS)
      s_q[idx] = ldcg_f(&m->q[(size_t)(t0 + (idx >> 6)) * d + h * 64 + (idx & 63)]);
    cta_sync();
    if (pr) pr[3] = wm_timer_ns();
    // K / V rows straight from L2
    self_attn_item<false>(
        m, g, tree_mask, h, t0, rg, s_q,
        [&](int j, uint4* a) {
          const uint4* k0 = reinterpret_cast<const uint4*>(L.self_k + self_kv_index(j, h * 64));
#pragma unroll
          for (int c = 0; c < 8; ++c) a[c] = ldcg_u4(k0 + c);
        },
        [&](int j, int dg) { return ldcg_u4(L.self_v + self_kv_index(j, h * 64 + dg * 8)); },
        [] {}, [] {}, [] {}, pr);
  }
}

// -----------------------------------------------------------------------------------------
// stage: cross-attention over the encoder K/V (flash-decoding split: m->cross_chunks key chunks per head)
// item = (head, chunk); all T query rows at once.  K/V rows: cross_kv[pos][0:d | d:2d] fp16.
// The chunk that arrives last for a head folds the partials (chunk order => deterministic).
// -----------------------------------------------------------------------------------------
#define WM_CH_MAX WM_CH_MAX_KEYS   // keys per chunk (S = 1500 over >= 6 chunks)
#define WM_CH_PAD 256   // rounded up to the MMA k-step (16 keys)
#define WM_SS_STRIDE (WM_CH_PAD + 8)   // score row stride in floats: 32 B (mod 128) => conflict-free 8-byte fragment loads
static_assert(WM_CH_PAD % 16 == 0 && WM_CH_PAD >= WM_CH_MAX, "a padded key chunk must hold WM_CH_MAX keys");
static_assert(WM_SS_STRIDE * 4 % 128 == 32, "score row stride must stay 32 B (mod 128)");
__host__ __device__ constexpr size_t cross_attn_smem_bytes() {
  return (size_t)2 * WM_CH_PAD * 72 * sizeof(__half) + (size_t)WM_MAX_T * WM_SS_STRIDE * sizeof(float) +
         (size_t)2 * 16 * 72 * sizeof(__half) + (size_t)2 * WM_MAX_T * sizeof(float);   // K, V chunk + cross_scratch_bytes()
}
// Item `item` of the stage = key chunk c of head h: encoder positions [j0, j0 + nk) of S (nk = 0: an empty trailing
// chunk).
// The stage kernels, the ring kernel and the ring's chunk schedule all take their items from here.
struct CrossItem { int h, c, j0, nk; };
__host__ __device__ __forceinline__ CrossItem cross_item(int item, int S, int nch) {
  const int CH = (S + nch - 1) / nch;
  CrossItem it;
  it.h = item / nch;
  it.c = item - it.h * nch;
  it.j0 = it.c * CH;
  it.nk = max(0, min(S, it.j0 + CH) - it.j0);
  return it;
}
__device__ __forceinline__ void split_hilo(float a, float b, uint32_t& hi, uint32_t& lo) {
  const __half ha = __float2half_rn(a), hb = __float2half_rn(b);
  __half2 h = __halves2half2(ha, hb);
  __half2 l = __floats2half2_rn(a - __half2float(ha), b - __half2float(hb));
  hi = *reinterpret_cast<uint32_t*>(&h);
  lo = *reinterpret_cast<uint32_t*>(&l);
}
// Both products run on the tensor cores (mma.sync m16n8k16, fp32 accumulate): S = Q K^T with the
// fp32 query split into fp16 hi + lo, O = P V with the fp32 probabilities split the same way.
//
// cross_attn_core: one (head, key chunk) item once its K / V rows [nk_pad][72] (fp16, rows nk..nk_pad
// zero) sit in shared memory -- in the scratch area (stage kernels) or in two ring slots (ring kernel).
// `after_qk` / `after_pv` run once the last read of sK / sV is over (the ring hands the slots back there).
struct CrossScratch {
  float* sS;      // [16][WM_SS_STRIDE] scores, then the probabilities as fp16 {hi2, lo2} key pairs (in place)
  __half* sQh;    // [16][72]
  __half* sQl;
  float* sM;      // [16] max, [16] sum
};
__host__ __device__ constexpr size_t cross_scratch_bytes() {
  return (size_t)WM_MAX_T * WM_SS_STRIDE * sizeof(float) + (size_t)2 * 16 * 72 * sizeof(__half) + (size_t)2 * WM_MAX_T * sizeof(float);
}
__device__ __forceinline__ CrossScratch cross_scratch(unsigned char* p) {
  CrossScratch cs;
  cs.sS = reinterpret_cast<float*>(p);
  cs.sQh = reinterpret_cast<__half*>(cs.sS + WM_MAX_T * WM_SS_STRIDE);
  cs.sQl = cs.sQh + 16 * 72;
  cs.sM = reinterpret_cast<float*>(cs.sQl + 16 * 72);
  return cs;
}
// combine the chunk partials of head h (run by the CTA that arrives last for the head): warp per query row,
// lane = output dims (lane, lane + 32); the chunk statistics sit one per lane and are broadcast by shuffles.
// Every load is in flight before the first use (a loop with a run-time bound would pay one L2 round trip per
// chunk); chunks are combined in chunk order => deterministic.
template <bool SPLIT_OUT>
__device__ __forceinline__ void cross_attn_fold(const DecModel* m, int T, int h, int nch) {
  const int d = m->d;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = (WM_DEC_THREADS >> 5);
  const size_t cstride = (size_t)WM_MAX_T * (WM_HEAD_DIM + 2);
  for (int rr = warp; rr < T; rr += nwarps) {
    const float* base = m->cross_part + ((size_t)h * WM_CROSS_CHUNKS * WM_MAX_T + rr) * (WM_HEAD_DIM + 2);
    float mm = -INFINITY, ll = 0.f;
    if (lane < nch) { mm = __ldcg(base + lane * cstride + 64); ll = __ldcg(base + lane * cstride + 65); }
    float v0[WM_CROSS_CHUNKS], v1[WM_CROSS_CHUNKS];
#pragma unroll
    for (int cc = 0; cc < WM_CROSS_CHUNKS; ++cc)
      if (cc < nch) { v0[cc] = __ldcg(base + cc * cstride + lane); v1[cc] = __ldcg(base + cc * cstride + 32 + lane); }
    const float M = warp_max(mm);
    const float wl = (lane < nch) ? expf(mm - M) : 0.f;
    float num0 = 0.f, num1 = 0.f, den = 0.f;
#pragma unroll
    for (int cc = 0; cc < WM_CROSS_CHUNKS; ++cc)
      if (cc < nch) {
        const float w = __shfl_sync(0xffffffffu, wl, cc);
        const float l = __shfl_sync(0xffffffffu, ll, cc);
        num0 = fmaf(w, v0[cc], num0);
        num1 = fmaf(w, v1[cc], num1);
        den = fmaf(w, l, den);
      }
    if (SPLIT_OUT) {   // ring kernel: operand format of the cross-O projection (common.cuh: store_split)
      store_split(m->attn + (size_t)rr * d, h * 64 + lane, num0 / den);
      store_split(m->attn + (size_t)rr * d, h * 64 + 32 + lane, num1 / den);
    } else {
      float* o = m->attn + (size_t)rr * d + h * 64;
      o[lane] = num0 / den;
      o[32 + lane] = num1 / den;
    }
  }
}

// Token-timestamp capture of one (head, key chunk) item (out of line: the rare branch adds no registers to the stage):
// when `layer` is a base decoder layer, the pass is A or B and head h is an alignment head, warp r copies the nk raw
// scores of row r < T to the row's position (chain: base + r; tree: base + depth).  Ends in a CTA barrier, so the
// softmax that follows may overwrite the scores in place.
__device__ __noinline__ void ts_capture(const DecModel* m, int mode, int layer, int T, int h, int c, int nch, int nk,
                                        const float* sS) {
  if (mode == MODE_TAIL || layer >= m->n_layers) return;
  const TsCapture* ts = m->ts;
  const int slot = ts->slot[layer * m->H + h];
  if (slot < 0) return;
  const int base = (mode == MODE_A) ? ldcg_i(&m->st->kv_len) : ldcg_i(&m->st->L);
  const int j0 = cross_item(h * nch + c, m->S, nch).j0;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int r = warp; r < T; r += (WM_DEC_THREADS >> 5)) {
    const int pos = base + ((mode == MODE_B && m->has_tree) ? m->tree->depth[r] : r);
    if (pos >= WM_TS_ROWS) continue;
    float* dst = ts->scores + ((size_t)slot * WM_TS_ROWS + pos) * m->S + j0;
    for (int j = lane; j < nk; j += 32) dst[j] = sS[r * WM_SS_STRIDE + j];
  }
  cta_sync();
}

// `on_scores(sS)` runs when token-timestamp capture is on (m->ts), after S = Q K^T is complete and before the softmax
// overwrites it: the caller binds the pass mode and layer (ts_capture).
template <bool SPLIT_OUT, class AfterQK, class AfterPV, class OnScores>
__device__ __forceinline__ void cross_attn_core(const DecModel* m, int T, int h, int c, int nch, int nk, int nk_pad,
                                                const __half* sK, const __half* sV, const CrossScratch& cs,
                                                AfterQK&& after_qk, AfterPV&& after_pv, OnScores&& on_scores,
                                                unsigned long long* pr = nullptr) {
  __shared__ int s_last;
  float* sS = cs.sS; __half* sQh = cs.sQh; __half* sQl = cs.sQl; float* sM = cs.sM;
  const int d = m->d;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = (WM_DEC_THREADS >> 5);
  const int gq = lane >> 2, tq = lane & 3;
  // queries (fp32) -> fp16 hi / lo, rows >= T are zero
  for (int idx = tid; idx < 16 * 32; idx += WM_DEC_THREADS) {
    const int r = idx >> 5, c2 = (idx & 31) * 2;
    float a = 0.f, b = 0.f;
    if (r < T) { const float2 v = ldcg_f2(m->q + (size_t)r * d + h * 64 + c2); a = v.x; b = v.y; }
    uint32_t hi, lo;
    split_hilo(a, b, hi, lo);
    *reinterpret_cast<uint32_t*>(sQh + r * 72 + c2) = hi;
    *reinterpret_cast<uint32_t*>(sQl + r * 72 + c2) = lo;
  }
  cta_sync();
  if (pr) pr[4] = wm_timer_ns();
  // ---- S = Q K^T * head_dim^-0.5 : warp w takes key tiles (8 keys) w, w + nwarps, ... ----
  {
    uint32_t qh[4][4], ql[4][4];
    const int arow = (lane & 7) + ((lane >> 3) & 1) * 8;
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      const int ch = kk * 2 + (lane >> 4);
      ldmatrix_x4(qh[kk][0], qh[kk][1], qh[kk][2], qh[kk][3], sQh + arow * 72 + ch * 8);
      ldmatrix_x4(ql[kk][0], ql[kk][1], ql[kk][2], ql[kk][3], sQl + arow * 72 + ch * 8);
    }
    for (int nt = warp; nt < nk_pad / 8; nt += nwarps) {
      float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int k2 = 0; k2 < 2; ++k2) {
        uint32_t b0, b1, b2, b3;   // (keys nt*8.., k-steps 2*k2 and 2*k2+1)
        ldmatrix_x4(b0, b1, b2, b3, sK + (nt * 8 + (lane & 7)) * 72 + (k2 * 4 + (lane >> 3)) * 8);
        mma_16816(acc, qh[2 * k2][0], qh[2 * k2][1], qh[2 * k2][2], qh[2 * k2][3], b0, b1);
        mma_16816(acc, ql[2 * k2][0], ql[2 * k2][1], ql[2 * k2][2], ql[2 * k2][3], b0, b1);
        mma_16816(acc, qh[2 * k2 + 1][0], qh[2 * k2 + 1][1], qh[2 * k2 + 1][2], qh[2 * k2 + 1][3], b2, b3);
        mma_16816(acc, ql[2 * k2 + 1][0], ql[2 * k2 + 1][1], ql[2 * k2 + 1][2], ql[2 * k2 + 1][3], b2, b3);
      }
      float* s0 = sS + gq * WM_SS_STRIDE + nt * 8 + 2 * tq;
      *reinterpret_cast<float2*>(s0) = make_float2(acc[0] * 0.125f, acc[1] * 0.125f);
      *reinterpret_cast<float2*>(s0 + 8 * WM_SS_STRIDE) = make_float2(acc[2] * 0.125f, acc[3] * 0.125f);
    }
  }
  cta_sync();
  if (pr) pr[5] = wm_timer_ns();
  after_qk();
  if (m->ts != nullptr) on_scores(sS);
  // ---- per-row max / exp / sum : warp per row, two keys per lane; rows >= T and keys >= nk become zero
  // probability.  The probabilities replace the scores IN PLACE as the fp16 operand pairs of the P V MMAs:
  // floats (p[2j], p[2j+1]) -> { half2 hi, half2 lo }, so the 8 warps of the next phase do not each redo the split.
  for (int r = warp; r < 16; r += nwarps) {
    float* p = sS + r * WM_SS_STRIDE;
    if (r < T) {
      float mx = -INFINITY;
      for (int pj = lane; 2 * pj < nk; pj += 32) {
        const float2 v = *reinterpret_cast<const float2*>(p + 2 * pj);
        mx = fmaxf(mx, v.x);
        if (2 * pj + 1 < nk) mx = fmaxf(mx, v.y);
      }
      mx = warp_max(mx);
      float sum = 0.f;
      for (int pj = lane; 2 * pj < nk_pad; pj += 32) {
        const float2 v = *reinterpret_cast<const float2*>(p + 2 * pj);
        const float e0 = (2 * pj < nk) ? expf(v.x - mx) : 0.f;
        const float e1 = (2 * pj + 1 < nk) ? expf(v.y - mx) : 0.f;
        uint2 o;
        split_hilo(e0, e1, o.x, o.y);
        *reinterpret_cast<uint2*>(p + 2 * pj) = o;
        sum += e0 + e1;
      }
      sum = warp_sum(sum);
      if (lane == 0) { sM[r] = mx; sM[WM_MAX_T + r] = sum; }
    } else {
      for (int pj = lane; 2 * pj < nk_pad; pj += 32) *reinterpret_cast<uint2*>(p + 2 * pj) = make_uint2(0u, 0u);
    }
  }
  cta_sync();
  if (pr) pr[6] = wm_timer_ns();
  // ---- O = P V : warp w < 8 owns output dims w*8 .. w*8+7, all key steps ----
  if (warp < 8) {
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    float acl[4] = {0.f, 0.f, 0.f, 0.f};
    for (int ks = 0; ks < nk_pad / 16; ++ks) {
      const float* p0 = sS + gq * WM_SS_STRIDE + ks * 16 + 2 * tq;
      const uint2 a00 = *reinterpret_cast<const uint2*>(p0);                          // row g,   keys 2t..2t+1  {hi, lo}
      const uint2 a10 = *reinterpret_cast<const uint2*>(p0 + 8 * WM_SS_STRIDE);      // row g+8
      const uint2 a01 = *reinterpret_cast<const uint2*>(p0 + 8);                      // row g,   keys 2t+8..
      const uint2 a11 = *reinterpret_cast<const uint2*>(p0 + 8 * WM_SS_STRIDE + 8);  // row g+8
      uint32_t b0, b1;
      ldmatrix_x2_trans(b0, b1, sV + (ks * 16 + (lane & 15)) * 72 + warp * 8);
      mma_16816(acc, a00.x, a10.x, a01.x, a11.x, b0, b1);
      mma_16816(acl, a00.y, a10.y, a01.y, a11.y, b0, b1);
    }
#pragma unroll
    for (int e = 0; e < 4; ++e) acc[e] += acl[e];
    float* out0 = m->cross_part + ((size_t)(h * WM_CROSS_CHUNKS + c) * WM_MAX_T + gq) * (WM_HEAD_DIM + 2) + warp * 8 + 2 * tq;
    if (gq < T) { out0[0] = acc[0]; out0[1] = acc[1]; }
    if (gq + 8 < T) { out0[8 * (WM_HEAD_DIM + 2)] = acc[2]; out0[8 * (WM_HEAD_DIM + 2) + 1] = acc[3]; }
  }
  if (tid < T) {
    float* out = m->cross_part + ((size_t)(h * WM_CROSS_CHUNKS + c) * WM_MAX_T + tid) * (WM_HEAD_DIM + 2);
    out[64] = sM[tid];
    out[65] = sM[WM_MAX_T + tid];
  }
  // fold: the chunk that arrives last for this head (always in chunk order => deterministic)
  // (release-only arrival; the partials are read back with L2-coherent loads, see common.cuh)
  cta_sync();
  if (pr) pr[7] = wm_timer_ns();
  after_pv();
  if (tid == 0) {
    const unsigned int prev = atom_add_release(&m->cross_cnt[h], 1u);
    s_last = (prev == (unsigned int)(nch - 1)) ? 1 : 0;
    if (s_last) m->cross_cnt[h] = 0u;   // everybody has arrived: re-arm for the next layer
  }
  cta_sync();
  if (pr) pr[8] = wm_timer_ns();
  if (s_last) {
    cross_attn_fold<SPLIT_OUT>(m, T, h, nch);
  }
  if (pr) { pr[10] = wm_timer_ns(); pr[11] = s_last ? 1000ull : 0ull; }
}

__device__ __forceinline__ void stage_cross_attn(const DecModel* m, int mode, int layer, int cta, int ncta, unsigned char* smem_raw, const PassGeom* gopt) {
  const PassGeom g = gopt ? *gopt : pass_geom(m, mode);
  const int H = m->H, S = m->S;
  const DecLayer& L = m->layers[layer];
  const int nch = m->cross_chunks;
  __half* sK = reinterpret_cast<__half*>(smem_raw);                 // [CH_PAD][72]
  __half* sV = sK + WM_CH_PAD * 72;                                 // [CH_PAD][72]
  const CrossScratch cs = cross_scratch(reinterpret_cast<unsigned char*>(sV + WM_CH_PAD * 72));
  const int tid = threadIdx.x;
  for (int item = cta; item < H * nch; item += ncta) {
    const CrossItem it = cross_item(item, S, nch);
    const int h = it.h, c = it.c, j0 = it.j0, nk = it.nk;
    const int nk_pad = (nk + 15) & ~15;
    cta_sync();
    // K / V chunk -> shared memory (all loads of a batch in flight before the first store); the cache rows are
    // already in the shared-memory layout: cross_k[h][pos][72]
    const uint4* gk = reinterpret_cast<const uint4*>(L.cross_k + ((size_t)h * m->S_pad + j0) * 72);
    const uint4* gv = reinterpret_cast<const uint4*>(L.cross_v + ((size_t)h * m->S_pad + j0) * 72);
    for (int base = 0; base < nk * 9; base += 4 * WM_DEC_THREADS) {
      uint4 kk[4], vv[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int idx = base + i * WM_DEC_THREADS + tid;
        if (idx < nk * 9) { kk[i] = ldg_nc_v4(gk + idx); vv[i] = ldg_nc_v4(gv + idx); }
      }
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int idx = base + i * WM_DEC_THREADS + tid;
        if (idx < nk * 9) {
          reinterpret_cast<uint4*>(sK)[idx] = kk[i];
          reinterpret_cast<uint4*>(sV)[idx] = vv[i];
        }
      }
    }
    // rows nk .. nk_pad of K and V read as zero (their probabilities are zero, but 0 * garbage could be NaN)
    for (int idx = tid; idx < (nk_pad - nk) * 9; idx += WM_DEC_THREADS) {
      reinterpret_cast<uint4*>(sK)[nk * 9 + idx] = make_uint4(0, 0, 0, 0);
      reinterpret_cast<uint4*>(sV)[nk * 9 + idx] = make_uint4(0, 0, 0, 0);
    }
    cross_attn_core<false>(m, g.T, h, c, nch, nk, nk_pad, sK, sV, cs, [] {}, [] {},
                           [&](const float* s) { ts_capture(m, mode, layer, g.T, h, c, nch, nk, s); });
  }
}

// Encoder side: cross K/V of one decoder layer from the GEMM layout [pos][k | v] into the decode layout
// cross_k / cross_v [H][S_pad][72] (64 dims + 8 halfs of padding = the bank-conflict-free shared-memory row).
__global__ void __launch_bounds__(256) relayout_cross_kv_kernel(const __half* __restrict__ kv, __half* __restrict__ ck,
                                                                __half* __restrict__ cv, int S, int S_pad, int d, int H) {
  const size_t total = (size_t)H * S_pad * 9;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int q = (int)(i % 9);
    const size_t row = i / 9;
    const int pos = (int)(row % S_pad), h = (int)(row / S_pad);
    uint4 k = make_uint4(0, 0, 0, 0), v = k;
    if (q < 8 && pos < S) {
      const __half* src = kv + (size_t)pos * 2 * d + h * 64 + q * 8;
      k = *reinterpret_cast<const uint4*>(src);
      v = *reinterpret_cast<const uint4*>(src + d);
    }
    reinterpret_cast<uint4*>(ck)[i] = k;
    reinterpret_cast<uint4*>(cv)[i] = v;
  }
}

// -----------------------------------------------------------------------------------------
// stage: final LayerNorm -> hidden  (HF modeling_whisper.py:791)
//   sweep A: the last row is also the "carry" (hidden state of the newest cached token, the
//            input of the Medusa heads).  sweep B + block type: base logits read the hidden
//            states directly (reference model.py:1287).
//   no-speech capture: row m->ns_row of the first real iteration's sweep A (n_iter == 0, not a
//            prefill launch) is also stored into m->ns_hidden (read after the loop by no_speech.cu).
// -----------------------------------------------------------------------------------------
// no-speech capture (out of line: the rare branch adds no registers to the stage): warp 0 copies back the row it has
// just stored, each lane only the elements it stored itself
__device__ __noinline__ void ns_capture(const DecModel* m, int t) {
  if (ldcg_i(&m->st->n_iter) != 0 || ldcg_i(&m->st->prefill)) return;
  const float4* src = reinterpret_cast<const float4*>(m->hidden + (size_t)t * m->d);
  float4* dst = reinterpret_cast<float4*>(m->ns_hidden);
  for (int i = threadIdx.x & 31; i < (m->d >> 2); i += 32) dst[i] = __ldcg(src + i);
}
__device__ __forceinline__ void stage_final_ln(const DecModel* m, int mode, int cta, int ncta, const PassGeom* gopt) {
  const PassGeom g = gopt ? *gopt : pass_geom(m, mode);
  const int d = m->d;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int nv = d >> 7;   // float4 per lane (d <= 1280)
  // one row per CTA (warp 0): the rows are few, spreading them keeps each on its own SM
  for (int t = cta; t < g.T; t += ncta) {
    if (warp != 0) continue;
    const float4* x4 = reinterpret_cast<const float4*>(m->x + (size_t)t * d);
    float4 v[10];
#pragma unroll
    for (int i = 0; i < 10; ++i)
      if (i < nv) v[i] = __ldcg(x4 + i * 32 + lane);
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < 10; ++i)
      if (i < nv) s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
    const float mean = warp_sum(s) / (float)d;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < 10; ++i)
      if (i < nv) {
        const float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, e = v[i].w - mean;
        q += (a * a + b * b) + (c * c + e * e);
      }
    const float rstd = rsqrtf(warp_sum(q) / (float)d + 1e-5f);
    const float4* g4 = reinterpret_cast<const float4*>(m->lnf_g);
    const float4* b4 = reinterpret_cast<const float4*>(m->lnf_b);
    float4* hid = reinterpret_cast<float4*>(m->hidden + (size_t)t * d);
#pragma unroll
    for (int i = 0; i < 10; ++i)
      if (i < nv) {
        const float4 gg = __ldg(g4 + i * 32 + lane), bb = __ldg(b4 + i * 32 + lane);   // (read-only path: may run ahead of the stores below)
        float4 y;
        y.x = (v[i].x - mean) * rstd * gg.x + bb.x;
        y.y = (v[i].y - mean) * rstd * gg.y + bb.y;
        y.z = (v[i].z - mean) * rstd * gg.z + bb.z;
        y.w = (v[i].w - mean) * rstd * gg.w + bb.w;
        hid[i * 32 + lane] = y;
        if (mode == MODE_A && t == g.T - 1) reinterpret_cast<float4*>(m->carry)[i * 32 + lane] = y;
        if (mode == MODE_B && m->has_block) reinterpret_cast<float4*>(m->head_h + (size_t)t * d)[i * 32 + lane] = y;
      }
    if (mode == MODE_A && t == m->ns_row) ns_capture(m, t);
  }
}
// block type: the extra layer consumes the LayerNorm'ed hidden states (reference model.py:1374-1376)
__device__ void stage_copy_hidden_to_x(const DecModel* m, int mode, int cta, int ncta, const PassGeom* gopt) {
  const PassGeom g = gopt ? *gopt : pass_geom(m, mode);
  const int total = g.T * m->d;
  for (int idx = cta * WM_DEC_THREADS + threadIdx.x; idx < total; idx += ncta * WM_DEC_THREADS) m->x[idx] = ldcg_f(&m->hidden[idx]);
}
// block type, tail: the block runs on the carried hidden state (one row); vocab row 0 = base logits
__device__ void stage_tail_seed(const DecModel* m, int cta, int ncta) {
  for (int idx = cta * WM_DEC_THREADS + threadIdx.x; idx < m->d; idx += ncta * WM_DEC_THREADS) {
    const float y = ldcg_f(&m->carry[idx]);
    m->x[idx] = y;
    m->head_h[idx] = y;
  }
}

// -----------------------------------------------------------------------------------------
// stage: logits scan = logits processors + argmax (+ softmax statistics for typical acceptance)
//   processors: HF logits_process.py:1893-1901 (suppress), :1847-1862 (begin), :1742-1772 (EOS decay)
//   pass A: generate_candidates with top-1 per head (medusa_utils.py:446-457)
//   pass B: evaluate_posterior (medusa_utils.py:547-588)
// -----------------------------------------------------------------------------------------
__device__ void block_argmax(float& v, int& i, float* s_val, int* s_idx) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = (WM_DEC_THREADS >> 5);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    float ov = __shfl_xor_sync(0xffffffffu, v, o);
    int oi = __shfl_xor_sync(0xffffffffu, i, o);
    if (ov > v || (ov == v && oi < i)) { v = ov; i = oi; }
  }
  cta_sync();
  if (lane == 0) { s_val[warp] = v; s_idx[warp] = i; }
  cta_sync();
  v = s_val[0]; i = s_idx[0];
  for (int w = 1; w < nwarps; ++w) {
    float ov = s_val[w]; int oi = s_idx[w];
    if (ov > v || (ov == v && oi < i)) { v = ov; i = oi; }
  }
}
__device__ float block_sum(float v, float* s_val) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = (WM_DEC_THREADS >> 5);
  v = warp_sum(v);
  cta_sync();
  if (lane == 0) s_val[warp] = v;
  cta_sync();
  float s = 0.f;
  for (int w = 0; w < nwarps; ++w) s += s_val[w];
  return s;
}

// The logits scan is spread over the whole grid: every row is cut into `nseg` vocabulary segments.
//   SELECT1: per (row, segment): processed max / first argmax / sum of exp relative to the local max
//   SELECT2 (verify only): with the row max M and normaliser Z folded from the partials, the entropy
//            term sum p log(p + 1e-5) of the segment and the candidate's probability
//   SELECT_FIN (tail) / ACCEPT (verify): fold the partials in segment order (deterministic).
#define WM_SEL_MAXSEG 32
// the segment count is a property of the model/device (set by the host from the SM count), NOT of the
// launch: the fold stages run on one CTA and must agree with the scan stages
__device__ __forceinline__ int select_nseg(const DecModel* m, int /*ncta*/) { return m->sel_nseg; }
// sel_part layout: [row][seg][4] = {max, argmax (int bits), sumexp, entropy term}

// strict "comes after" in the candidate order (value descending, index ascending)
__device__ __forceinline__ bool ranks_after(float v, int i, float pv, int pi) { return v < pv || (v == pv && i > pi); }

template <bool ADJ>
__device__ __noinline__ void stage_select1_rows(const DecModel* m, int mode, int cta, int ncta, unsigned char* smem_raw) {
  const DecState* st = m->st;
  const int V = m->V, K = m->K;
  float* s_val = reinterpret_cast<float*>(smem_raw);
  int* s_idx = reinterpret_cast<int*>(s_val + 32);
  const int L = st->L;
  const bool begin_on = (L == st->begin_index);
  const float pen = m->pen_tab[L];
  const int eos = st->eos;
  const float* adj = ADJ ? dec_state_adj(st) : nullptr;
  const float* logits = (mode == MODE_A) ? m->logits_a : m->logits_b;
  const int nseg = select_nseg(m, ncta);
  const int seglen = (V + nseg - 1) / nseg;
  const float temp = st->temperature;
  const float inv_t = temp > 0.f ? 1.0f / temp : 1.0f;
  const bool tree = m->has_tree != 0;
  const int n_rows = (mode == MODE_A) ? K + 1 : m->n_tree;
  const int n_stat = tree ? n_rows : K;   // verify rows whose posterior is needed (rows that have a child)
  for (int item = cta; item < n_rows * nseg; item += ncta) {
    const int r = item / nseg, sg = item - r * nseg;
    const int j0 = sg * seglen, j1 = min(V, j0 + seglen);
    const float* row = logits + (size_t)r * V;
    float bv = -INFINITY;
    int bi = 0x7fffffff;
    for (int j = j0 + threadIdx.x; j < j1; j += WM_DEC_THREADS) {
      const float v = processed_logit<ADJ>(row, j, m->tok_mask, begin_on, eos, pen, adj);
      if (v > bv) { bv = v; bi = j; }   // ascending j per thread => first maximum kept
    }
    block_argmax(bv, bi, s_val, s_idx);
    float z = 0.f;
    if (mode == MODE_B && r < n_stat && temp > 0.f && bv > -INFINITY) {
      for (int j = j0 + threadIdx.x; j < j1; j += WM_DEC_THREADS)
        z += expf((processed_logit<ADJ>(row, j, m->tok_mask, begin_on, eos, pen, adj) - bv) * inv_t);
      z = block_sum(z, s_val);
    }
    if (threadIdx.x == 0) {
      float* o = m->sel_part + ((size_t)r * WM_SEL_MAXSEG + sg) * 4;
      o[0] = bv; o[1] = __int_as_float(bi); o[2] = z;
    }
    if (mode == MODE_A && tree) {
      // per-head top-k candidates (medusa_utils.py:446-457): the segment's first k entries in (value desc, index asc)
      // order, one block-wide selection round per rank (k <= WM_TREE_MAX_TOPK; tail only)
      const int kk = m->tree->topk[r];
      float* tp = m->topk_part + ((size_t)r * WM_SEL_MAXSEG + sg) * WM_TREE_MAX_TOPK * 2;
      float pv = bv; int pi = bi;
      if (threadIdx.x == 0) { tp[0] = pv; tp[1] = __int_as_float(pi); }
      for (int q = 1; q < kk; ++q) {
        float cv = -INFINITY; int ci = 0x7fffffff;
        for (int j = j0 + threadIdx.x; j < j1; j += WM_DEC_THREADS) {
          const float v = processed_logit<ADJ>(row, j, m->tok_mask, begin_on, eos, pen, adj);
          if (ranks_after(v, j, pv, pi) && (v > cv)) { cv = v; ci = j; }
        }
        block_argmax(cv, ci, s_val, s_idx);
        pv = cv; pi = ci;
        if (threadIdx.x == 0) { tp[2 * q] = pv; tp[2 * q + 1] = __int_as_float(pi); }
      }
    }
  }
}

// fold the segment partials of row r: global max (first index on ties), normaliser and the sum of the entropy
// partials.  Warp-cooperative (call with all 32 lanes): lane sg fetches segment sg with one 16-byte L2 load --
// one round trip instead of one per segment -- and the fold walks the lanes in segment order (shuffles), so the
// summation order is that of a sequential loop.  Results are uniform across the warp.
__device__ __forceinline__ void select_fold(const DecModel* m, int r, int nseg, float inv_t, float& M, int& idx, float& Z,
                                            float& ent) {
  const int lane = threadIdx.x & 31;
  float4 q = make_float4(-INFINITY, 0.f, 0.f, 0.f);
  if (lane < nseg) q = __ldcg(reinterpret_cast<const float4*>(m->sel_part + (size_t)r * WM_SEL_MAXSEG * 4) + lane);
  M = -INFINITY; idx = 0x7fffffff;
  for (int sg = 0; sg < nseg; ++sg) {
    const float v = __shfl_sync(0xffffffffu, q.x, sg);
    const int i = __float_as_int(__shfl_sync(0xffffffffu, q.y, sg));
    if (v > M || (v == M && i < idx)) { M = v; idx = i; }
  }
  Z = 0.f; ent = 0.f;
  const float w = (q.x > -INFINITY) ? q.z * expf((q.x - M) * inv_t) : 0.f;   // this lane's term (uniform M)
  for (int sg = 0; sg < nseg; ++sg) {
    const float v = __shfl_sync(0xffffffffu, q.x, sg);
    const float t = __shfl_sync(0xffffffffu, w, sg);
    if (v > -INFINITY) Z += t;
    ent += __shfl_sync(0xffffffffu, q.w, sg);
  }
}

template <bool ADJ>
__device__ __noinline__ void stage_select2_rows(const DecModel* m, int cta, int ncta, unsigned char* smem_raw) {
  DecState* st = m->st;
  const int V = m->V, K = m->K;
  float* s_val = reinterpret_cast<float*>(smem_raw);
  const float temp = st->temperature;
  if (temp == 0.f) return;   // exact-match acceptance needs only the argmax (uniform across the grid)
  const float inv_t = 1.0f / temp;
  const int L = st->L;
  const bool begin_on = (L == st->begin_index);
  const float pen = m->pen_tab[L];
  const int eos = st->eos;
  const float* adj = ADJ ? dec_state_adj(st) : nullptr;
  const int nseg = select_nseg(m, ncta);
  const int seglen = (V + nseg - 1) / nseg;
  const bool tree = m->has_tree != 0;
  const int n_stat = tree ? m->n_tree : K;                // chain: evaluate_posterior reads logits[:, :-1]
  for (int item = cta; item < n_stat * nseg; item += ncta) {
    const int r = item / nseg, sg = item - r * nseg;
    const int j0 = sg * seglen, j1 = min(V, j0 + seglen);
    const float* row = m->logits_b + (size_t)r * V;
    float M, Z, ent_unused; int idx;
    select_fold(m, r, nseg, inv_t, M, idx, Z, ent_unused);   // (every warp folds the same row: uniform)
    float ent = 0.f;
    for (int j = j0 + threadIdx.x; j < j1; j += WM_DEC_THREADS) {
      const float p = expf((processed_logit<ADJ>(row, j, m->tok_mask, begin_on, eos, pen, adj) - M) * inv_t) / Z;
      ent += p * logf(p + 1e-5f);
    }
    ent = block_sum(ent, s_val);
    if (threadIdx.x == 0) {
      m->sel_part[((size_t)r * WM_SEL_MAXSEG + sg) * 4 + 3] = ent;
      // probability, under this row's posterior, of the token of every child node (chain: the one node r + 1)
      const int n_lo = tree ? 1 : r + 1, n_hi = tree ? m->n_tree : r + 2;
      for (int n = n_lo; n < n_hi; ++n) {
        if (tree && m->tree->parent[n] != r) continue;
        const int c = ldcg_i(&st->cand[n]);
        if (c >= j0 && c < j1)
          st->row_pc[n] = expf((processed_logit<ADJ>(row, c, m->tok_mask, begin_on, eos, pen, adj) - M) * inv_t) / Z;
      }
    }
  }
}

// Sampled attempt (DecState smp_on).  The rows whose choice decides an emitted token -- the tail's base row 0 (position
// L) and verify rows r < K (position L + r + 1) -- store per segment either the perturbed maximum of
// processed / T + g(position, j) (smp_topk = 0) or the segment's first min(k, finite entries) entries in (value desc,
// index asc) order, their count and whether the segment has more entries equal to the last one (sel_part {max, argmax,
// count, flag}).  The other rows keep the plain argmax (exact-match acceptance: the loop's temperature is 0).
template <bool ADJ>
__device__ __noinline__ void stage_select1_smp_rows(const DecModel* m, int mode, int cta, int ncta, unsigned char* smem_raw) {
  const DecState* st = m->st;
  const int V = m->V, K = m->K;
  float* s_val = reinterpret_cast<float*>(smem_raw);
  int* s_idx = reinterpret_cast<int*>(s_val + 32);
  const int L = st->L;
  const bool begin_on = (L == st->begin_index);
  const float pen = m->pen_tab[L];
  const int eos = st->eos;
  const float* adj = ADJ ? dec_state_adj(st) : nullptr;
  const float* logits = (mode == MODE_A) ? m->logits_a : m->logits_b;
  const int nseg = select_nseg(m, ncta);
  const int seglen = (V + nseg - 1) / nseg;
  const int n_rows = (mode == MODE_A) ? K + 1 : m->n_tree;
  const int kk = st->smp_topk;
  const float temp = st->smp_temp;
  for (int item = cta; item < n_rows * nseg; item += ncta) {
    const int r = item / nseg, sg = item - r * nseg;
    const int j0 = sg * seglen, j1 = min(V, j0 + seglen);
    const float* row = logits + (size_t)r * V;
    const bool sampled = (mode == MODE_A) ? r == 0 : r < K;
    const bool perturb = sampled && kk == 0;
    const int n = (mode == MODE_A) ? L : L + r + 1;
    float bv = -INFINITY;
    int bi = 0x7fffffff;
    for (int j = j0 + threadIdx.x; j < j1; j += WM_DEC_THREADS) {
      float v = processed_logit<ADJ>(row, j, m->tok_mask, begin_on, eos, pen, adj);
      if (perturb) v = __fadd_rn(__fdiv_rn(v, temp), sample_gumbel(st->smp_key, st->smp_window, st->smp_attempt, n, j));
      if (v > bv) { bv = v; bi = j; }
    }
    block_argmax(bv, bi, s_val, s_idx);
    float* o = m->sel_part + ((size_t)r * WM_SEL_MAXSEG + sg) * 4;
    if (!sampled || perturb) {
      if (threadIdx.x == 0) { o[0] = bv; o[1] = __int_as_float(bi); o[2] = 0.f; }
      continue;
    }
    // top-k list: one block-wide selection round per rank, as the tree's candidates (finite values only)
    float* tp = m->topk_part + ((size_t)r * WM_SEL_MAXSEG + sg) * WM_SMP_MAX_TOPK * 2;
    float pv = bv;
    int pi = bi, cnt = (bi != 0x7fffffff) ? 1 : 0;
    if (threadIdx.x == 0) { tp[0] = pv; tp[1] = __int_as_float(pi); }
    while (cnt > 0 && cnt < kk) {
      float cv = -INFINITY;
      int ci = 0x7fffffff;
      for (int j = j0 + threadIdx.x; j < j1; j += WM_DEC_THREADS) {
        const float v = processed_logit<ADJ>(row, j, m->tok_mask, begin_on, eos, pen, adj);
        if (ranks_after(v, j, pv, pi) && (v > cv)) { cv = v; ci = j; }
      }
      block_argmax(cv, ci, s_val, s_idx);
      if (ci == 0x7fffffff) break;   // (uniform)
      pv = cv; pi = ci;
      if (threadIdx.x == 0) { tp[2 * cnt] = pv; tp[2 * cnt + 1] = __int_as_float(pi); }
      ++cnt;
    }
    // a full list may leave out entries equal to its last value: the fold then rescans the segment if that value is tau
    float more = 0.f;
    if (cnt == kk)
      for (int j = pi + 1 + threadIdx.x; j < j1; j += WM_DEC_THREADS)
        if (processed_logit<ADJ>(row, j, m->tok_mask, begin_on, eos, pen, adj) == pv) more = 1.f;
    more = block_sum(more, s_val);
    if (threadIdx.x == 0) { o[0] = bv; o[1] = __int_as_float(bi); o[2] = __int_as_float(cnt); o[3] = __int_as_float(more > 0.f ? 1 : 0); }
  }
}
__device__ __noinline__ void stage_select1_smp(const DecModel* m, int mode, int cta, int ncta, unsigned char* smem_raw) {
  if (dec_state_adj(m->st)) stage_select1_smp_rows<true>(m, mode, cta, ncta, smem_raw);
  else stage_select1_smp_rows<false>(m, mode, cta, ncta, smem_raw);
}

// Fold of sampled row r of `mode` (warp-cooperative, lane = segment; results uniform): the choice at position n, and tau,
// the k-th largest processed value of the row (-inf = the whole row).  tau is the k-th pop of a merge of the sorted
// segment lists; the choice is the perturbed maximum over every entry >= tau (ties on the sum: lowest index).
__device__ __noinline__ void smp_fold(const DecModel* m, int mode, int r, int nseg, int n, int& idx, float& tau) {
  const DecState* st = m->st;
  const int kk = st->smp_topk;
  if (kk == 0) {
    float M, Z, ent;
    select_fold(m, r, nseg, 1.0f, M, idx, Z, ent);
    tau = -INFINITY;
    return;
  }
  const int lane = threadIdx.x & 31;
  const float2 none = make_float2(-INFINITY, __int_as_float(0x7fffffff));
  int cnt = 0, flag = 0;
  if (lane < nseg) {
    const float4 q = __ldcg(reinterpret_cast<const float4*>(m->sel_part + (size_t)r * WM_SEL_MAXSEG * 4) + lane);
    cnt = __float_as_int(q.z);
    flag = __float_as_int(q.w);
  }
  const float* tp = m->topk_part + ((size_t)r * WM_SEL_MAXSEG + lane) * WM_SMP_MAX_TOPK * 2;
  int p = 0;
  float2 cur = cnt > 0 ? ldcg_f2(tp) : none, nxt = cnt > 1 ? ldcg_f2(tp + 2) : none;
  tau = -INFINITY;
  for (int q = 0; q < kk; ++q) {
    float bv = cur.x;
    int bi = __float_as_int(cur.y);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
    }
    if (bi == 0x7fffffff) { tau = -INFINITY; break; }   // fewer than k finite values: the whole row (uniform)
    tau = bv;
    if (__float_as_int(cur.y) == bi) {                  // (indices are unique: one lane pops)
      ++p;
      cur = nxt;
      nxt = (p + 1 < cnt) ? ldcg_f2(tp + 2 * (p + 1)) : none;
    }
  }
  const float temp = st->smp_temp;
  float best = -INFINITY;
  int bidx = 0x7fffffff;
  auto offer = [&](float v, int j) {
    const float s = __fadd_rn(__fdiv_rn(v, temp), sample_gumbel(st->smp_key, st->smp_window, st->smp_attempt, n, j));
    if (s > best || (s == best && j < bidx)) { best = s; bidx = j; }
  };
  float2 last = none;
  for (int e = 0; e < cnt; ++e) {
    last = ldcg_f2(tp + 2 * e);
    if (!(last.x >= tau)) break;
    offer(last.x, __float_as_int(last.y));
  }
  if (flag && cnt == kk && last.x == tau) {   // entries equal to tau beyond the segment's full list
    const int V = m->V, seglen = (V + nseg - 1) / nseg, j1 = min(V, (lane + 1) * seglen);
    const int L = st->L;
    const bool begin_on = (L == st->begin_index);
    const float pen = m->pen_tab[L];
    const float* adj = dec_state_adj(st);
    const float* row = ((mode == MODE_A) ? m->logits_a : m->logits_b) + (size_t)r * V;
    for (int j = __float_as_int(last.y) + 1; j < j1; ++j) {
      const float v = adj ? processed_logit<true>(row, j, m->tok_mask, begin_on, st->eos, pen, adj)
                          : processed_logit<false>(row, j, m->tok_mask, begin_on, st->eos, pen, nullptr);
      if (v == tau) offer(v, j);
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bidx, o);
    if (ov > best || (ov == best && oi < bidx)) { best = ov; bidx = oi; }
  }
  idx = bidx;
}

// The variant with the logits-processor term, or without it, chosen by the uniform DecState adj (on / off for the whole
// call): the stage and persistent kernels.  The ring kernel is instantiated with and without processors instead, so its
// variant without them is the same code as a build without processors.
__device__ __noinline__ void stage_select1(const DecModel* m, int mode, int cta, int ncta, unsigned char* smem_raw) {
  if (dec_state_adj(m->st)) stage_select1_rows<true>(m, mode, cta, ncta, smem_raw);
  else stage_select1_rows<false>(m, mode, cta, ncta, smem_raw);
}
__device__ __noinline__ void stage_select2(const DecModel* m, int cta, int ncta, unsigned char* smem_raw) {
  if (dec_state_adj(m->st)) stage_select2_rows<true>(m, cta, ncta, smem_raw);
  else stage_select2_rows<false>(m, cta, ncta, smem_raw);
}

// tail: candidates = top-1 of every head row (generate_candidates, medusa_utils.py:446-457); SMP (sampled attempt, chain
// only): c0 is the sampled choice of the base row
template <bool SMP = false>
__device__ __noinline__ void stage_select_fin(const DecModel* m, int ncta) {
  DecState* st = m->st;
  const int nseg = select_nseg(m, ncta);
  if (!m->has_tree) {
    for (int r = threadIdx.x >> 5; r <= m->K; r += (WM_DEC_THREADS >> 5)) {   // warp per row
      float M, Z, ent; int idx;
      if (SMP && r == 0) {
        float tau;
        smp_fold(m, MODE_A, 0, nseg, st->L, idx, tau);
        if ((threadIdx.x & 31) == 0) st->tail_tau = tau;
      } else {
        select_fold(m, r, nseg, 1.0f, M, idx, Z, ent);
      }
      if ((threadIdx.x & 31) == 0) st->cand[r] = idx;
    }
    return;
  }
  // tree: merge the per-segment top-k lists of head row r (lane = segment; every list is sorted), k rounds; the q-th
  // winner is the token of every node of level r with rank q (tree_candidates = candidates_flat[tree_indices])
  const DecTree* tr = m->tree;
  const int lane = threadIdx.x & 31;
  for (int r = threadIdx.x >> 5; r <= m->K; r += (WM_DEC_THREADS >> 5)) {
    const int kk = tr->topk[r];
    const float* tp = m->topk_part + ((size_t)r * WM_SEL_MAXSEG + lane) * WM_TREE_MAX_TOPK * 2;
    float lv[WM_TREE_MAX_TOPK]; int li[WM_TREE_MAX_TOPK];
#pragma unroll
    for (int q = 0; q < WM_TREE_MAX_TOPK; ++q) {
      lv[q] = -INFINITY; li[q] = 0x7fffffff;
      if (lane < nseg && q < kk) { lv[q] = __ldcg(tp + 2 * q); li[q] = __float_as_int(__ldcg(tp + 2 * q + 1)); }
    }
    int p = 0;
    for (int q = 0; q < kk; ++q) {
      float v = -INFINITY; int i = 0x7fffffff;
#pragma unroll
      for (int e = 0; e < WM_TREE_MAX_TOPK; ++e)
        if (e == p) { v = lv[e]; i = li[e]; }
      float bv = v; int bi = i;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
      }
      if (v == bv && i == bi) ++p;                    // (indices are unique: exactly one lane advances)
      if (lane < tr->n_tree && tr->depth[lane] == r && tr->rank[lane] == q) st->cand[lane] = bi;
    }
  }
}

// -----------------------------------------------------------------------------------------
// stage: accept + bookkeeping (CTA 0)
//   evaluate_posterior (chain => one candidate), update_inference_inputs (medusa_utils.py:630-652),
//   KV trim (model.py:383-401: chain rows are contiguous => kv_len is just advanced), stop rules
//   (model.py:774-793).
//
//   Sweep elision: the reference re-runs the decoder on the last emitted token (its "pass A") to
//   get the hidden state the heads read.  When accept >= 1 that token is candidate[accept], which
//   the verify sweep just processed at the same position behind the same accepted prefix, so its
//   hidden state and K/V row already exist: we keep accept+1 K/V rows and carry hidden[accept]
//   instead of recomputing them (identical values, half the weight traffic).  Only after an
//   accept-0 iteration (second emitted token = argmax of the verify row, never seen by the
//   decoder) a one-token sweep A is needed (`need_a`).
// -----------------------------------------------------------------------------------------
// SMP (sampled attempt): the choice of verify row r < K is the sampled one (smp_fold at position L + r + 1, its tau kept
// for the scoring kernel); the loop's temperature is 0, so acceptance is the exact match with it
template <bool SMP = false>
__device__ __noinline__ void stage_accept(const DecModel* m, int ncta) {
  __shared__ int s_a;
  __shared__ int s_arg[WM_MAX_T];
  __shared__ float s_thr[WM_MAX_T];
  DecState* st = m->st;
  const int K = m->K;
  const int nseg = select_nseg(m, ncta);
  const int lane = threadIdx.x & 31;
  // fold the scan partials: argmax of every row, acceptance threshold of rows < K
  for (int r = threadIdx.x >> 5; r <= K; r += (WM_DEC_THREADS >> 5)) {   // warp per row
    const float temp = st->temperature;
    float M, Z, ent; int idx;
    if (SMP && r < K) {
      float tau;
      smp_fold(m, MODE_B, r, nseg, st->L + r + 1, idx, tau);
      if (lane == 0) st->row_tau[r] = tau;
    } else {
      select_fold(m, r, nseg, temp > 0.f ? 1.0f / temp : 1.0f, M, idx, Z, ent);
    }
    if (lane == 0) {
      st->row_argmax[r] = idx;
      s_arg[r] = idx;
      if (r < K && temp > 0.f) {
        const float thr = fminf(st->post_thr, expf(ent) * st->post_alpha);   // ent = sum p log(p+1e-5) = -entropy
        st->row_thr[r] = thr;
        s_thr[r] = thr;
      }
    }
  }
  cta_sync();
  // acceptance and loop state: warp 0, one chain position per lane (every cross-CTA value is fetched once, all
  // loads in flight together; a serial walk would pay one L2 round trip per position)
  if (threadIdx.x < 32) {
    const int L = st->L;
    const float temp = st->temperature;
    const int cand_l = (lane <= K) ? ldcg_i(&st->cand[lane]) : 0;
    const float pc_l = (lane < K && temp != 0.f) ? ldcg_f(&st->row_pc[lane + 1]) : 0.f;   // p(cand[lane + 1] | row lane)
    const int cand_next = __shfl_down_sync(0xffffffffu, cand_l, 1);
    bool ok = false;
    if (lane < K) ok = (temp == 0.f) ? (cand_next == s_arg[lane]) : (pc_l > s_thr[lane]);
    const unsigned int bal = __ballot_sync(0xffffffffu, ok);
    const int a = __ffs(~bal) - 1;          // length of the accepted prefix (lanes >= K never vote ok => a <= K)
    int n_new = a + 1;
    int id = cand_l;
    if (a == 0) { n_new = 2; if (lane == 1) id = s_arg[0]; }
    if (lane < n_new) st->ids[L + lane] = id;
    const bool eos = __ballot_sync(0xffffffffu, lane < n_new && id == st->eos) != 0u;
    if (lane == 0) {
      const int newL = L + n_new;
      st->L = newL;
      st->kv_len = (a == 0) ? newL - 1 : newL;
      st->need_a = (a == 0) ? 1 : 0;
      st->keep_n = 0;                        // chain: the surviving K/V rows are already where they belong
      st->accept_last = a;
      const int it = st->n_iter;
      st->accept_hist[it] = a;
      st->n_iter = it + 1;
      bool done = eos || newL >= st->max_length || newL + K >= st->max_length;
      if (st->max_iters > 0 && it + 1 >= st->max_iters) done = true;
      if (done) st->done = 1;
      s_a = a;
    }
  }
  cta_sync();
  const int a = s_a;
  if (a >= 1) {
    const float* src = m->hidden + (size_t)a * m->d;
    for (int j = threadIdx.x; j < m->d; j += WM_DEC_THREADS) m->carry[j] = ldcg_f(src + j);
  }
}

// -----------------------------------------------------------------------------------------
// stage: accept for a candidate TREE (branching medusa_choices; CTA 0)
//   evaluate_posterior over all root-to-leaf paths (medusa_utils.py:526-588): accept length of a path = number of
//   leading edges whose child token passes (typical acceptance: p_parent(child) > threshold(parent); temperature 0:
//   child == argmax(parent)); best = longest, ties broken by the summed log-likelihood (first index at temperature 0,
//   torch.argmax).  update_inference_inputs (:630-652) + _update_medusa_outputs (model.py:383-401): the tokens of the
//   accepted prefix are appended and the K/V rows of its first `accept` nodes (one node when nothing was accepted) are
//   kept -- they are gathered to rows L .. by stage_kv_compact.
//   Reference behaviour (tree_attn = 0): the verify rows attended to ALL earlier tree rows, so the newest token is
//   re-run by sweep A every iteration (need_a = 1), exactly like the reference's pass A.  With true tree attention
//   (tree_attn = 1) a node only saw its ancestors: its hidden state and K/V row are what a re-run would compute, and
//   the sweep is elided as in the chain case.
// -----------------------------------------------------------------------------------------
__device__ __noinline__ void stage_accept_tree(const DecModel* m, int ncta) {
  __shared__ int s_arg[WM_MAX_T];
  __shared__ float s_thr[WM_MAX_T];
  __shared__ int s_a, s_node;
  DecState* st = m->st;
  const DecTree* tr = m->tree;
  const int K = m->K, nt = tr->n_tree;
  const int nseg = select_nseg(m, ncta);
  const int lane = threadIdx.x & 31;
  const float temp = st->temperature;
  for (int r = threadIdx.x >> 5; r < nt; r += (WM_DEC_THREADS >> 5)) {   // warp per tree row
    float M, Z, ent; int idx;
    select_fold(m, r, nseg, temp > 0.f ? 1.0f / temp : 1.0f, M, idx, Z, ent);
    if (lane == 0) {
      st->row_argmax[r] = idx;
      s_arg[r] = idx;
      const float thr = fminf(st->post_thr, expf(ent) * st->post_alpha);
      st->row_thr[r] = thr;
      s_thr[r] = thr;
    }
  }
  cta_sync();
  if (threadIdx.x < 32) {
    const int L = st->L;
    // lane = node: its token and its probability under the parent's posterior
    const int tok_n = (lane < nt) ? ldcg_i(&st->cand[lane]) : 0;
    const float pc_n = (lane >= 1 && lane < nt && temp != 0.f) ? ldcg_f(&st->row_pc[lane]) : 0.f;
    // lane = candidate path: walk its edges (every lane runs the loop -- the shuffles need the full warp --; lanes
    // beyond the last path walk path 0 and are discarded)
    int len = 0;
    float like = 0.f;
    {
      const int c = min(lane, tr->n_cand - 1);
      bool open = true;
      for (int j = 0; j < K; ++j) {
        const int node = tr->retrieve[c][j], child = tr->retrieve[c][j + 1];
        const int ctok = __shfl_sync(0xffffffffu, tok_n, child);
        const float cp = __shfl_sync(0xffffffffu, pc_n, child);
        const bool ok = (temp == 0.f) ? (ctok == s_arg[node]) : (cp > s_thr[node]);
        open = open && ok;
        if (open) { ++len; if (temp != 0.f) like += logf(cp); }
      }
      if (lane >= tr->n_cand) len = -1;
    }
    int a = len;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) a = max(a, __shfl_xor_sync(0xffffffffu, a, o));
    // best path: longest; at temperature 0 the first such path, else the most likely one (first on ties)
    float score = (lane < tr->n_cand && len == a) ? ((temp == 0.f || a == 0) ? 0.f : like) : -INFINITY;
    int best = lane;
    float bs = score;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float os = __shfl_xor_sync(0xffffffffu, bs, o);
      const int ob = __shfl_xor_sync(0xffffffffu, best, o);
      if (os > bs || (os == bs && ob < best)) { bs = os; best = ob; }
    }
    if (a == 0) best = 0;
    int n_new = a + 1;
    // lane = depth along the best path
    const int node_l = (lane <= K) ? tr->retrieve[best][lane] : 0;
    int id = __shfl_sync(0xffffffffu, tok_n, node_l);
    if (a == 0) { n_new = 2; if (lane == 1) id = s_arg[tr->retrieve[best][0]]; }
    if (lane < n_new) st->ids[L + lane] = id;
    const bool eos = __ballot_sync(0xffffffffu, lane < n_new && id == st->eos) != 0u;
    const int keep = (a == 0) ? 1 : a;
    const bool elide = st->tree_attn != 0 && a >= 1;     // true tree attention: node `a` was computed behind exactly its prefix
    const int keep_rows = elide ? a + 1 : keep;
    if (lane < keep_rows) st->keep_src[lane] = L + node_l;
    if (lane == 0) {
      const int newL = L + n_new;
      st->L = newL;
      st->kv_len = elide ? newL : newL - 1;
      st->need_a = elide ? 0 : 1;
      st->keep_n = keep_rows;
      st->accept_last = a;
      const int it = st->n_iter;
      st->accept_hist[it] = a;
      st->n_iter = it + 1;
      bool done = eos || newL >= st->max_length || newL + K >= st->max_length;
      if (st->max_iters > 0 && it + 1 >= st->max_iters) done = true;
      if (done) st->done = 1;
      s_a = elide ? a : -1;
      s_node = tr->retrieve[best][a];
      st->path_node = s_node;
    }
  }
  cta_sync();
  if (s_a >= 1) {
    const float* src = m->hidden + (size_t)s_node * m->d;
    for (int j = threadIdx.x; j < m->d; j += WM_DEC_THREADS) m->carry[j] = ldcg_f(src + j);
  }
}

// stage: gather the surviving K/V rows of a tree verify pass to rows L .. L+keep-1 of every layer's cache (reference
// model.py:383-401: tree_past[:, :, select_indices][..., :accept]).  One (layer, K|V) item per CTA turn; rows move in
// path order (keep_src[j] >= L + j, so a row is always read before a later move can overwrite it), each as the 64
// dims of every head (thread = head, 8 dims).  No-op for chains.
__device__ __noinline__ void stage_kv_compact(const DecModel* m, int cta, int ncta) {
  const DecState* st = m->st;
  const int keep = ldcg_i(&st->keep_n);   // (written by CTA 0 in the previous stage: L2-coherent reads; uniform across the grid)
  if (keep <= 1) return;
  const int d = m->d;
  const int n_l = m->n_layers + (m->has_block ? 1 : 0);
  const int L0 = ldcg_i(&st->keep_src[0]);   // = old L (node 0 is the root)
  const bool on = threadIdx.x < d / 8;
  const int c = 8 * threadIdx.x;   // channel of this thread's 8 dims
  for (int item = cta; item < 2 * n_l; item += ncta) {
    __half* base = (item & 1) ? m->layers[item >> 1].self_v : m->layers[item >> 1].self_k;
    for (int j = 1; j < keep; ++j) {
      const int src = ldcg_i(&st->keep_src[j]), dst = L0 + j;
      if (src != dst) {
        uint4 v = make_uint4(0, 0, 0, 0);
        if (on) v = ldcg_u4(base + self_kv_index(src, c));
        cta_sync();
        if (on) *reinterpret_cast<uint4*>(base + self_kv_index(dst, c)) = v;
      }
      cta_sync();
    }
  }
}

// -----------------------------------------------------------------------------------------
// GEMM descriptors of the stages
// -----------------------------------------------------------------------------------------
enum StageId {
  ST_EMBED = 0, ST_QKV, ST_SELF_ATTN, ST_OPROJ, ST_CROSS_Q, ST_CROSS_ATTN, ST_CROSS_O,
  ST_FC1, ST_FC2, ST_FINAL_LN, ST_COPY_HIDDEN, ST_TAIL_SEED, ST_HEADS, ST_VOCAB, ST_SELECT1, ST_SELECT2, ST_SELECT_FIN,
  ST_ACCEPT, ST_KV_COMPACT
};
enum PhaseId { PH_SWEEP_A = 0, PH_TAIL = 1, PH_VERIFY = 2 };

// Output rows of head layer `layer`: the halves of head_h alternate from layer to layer, so that no layer writes rows
// that a CTA may still be staging as its input, and the last layer is in the first half, where the vocabulary stage
// reads (the block type's base row, stage_tail_seed / stage_final_ln, is there too)
__host__ __device__ inline float* head_layer_out(const DecModel* m, int layer) {
  return m->head_h + (size_t)((m->n_head_layers - 1 - layer) & 1) * WM_MAX_T * m->d;
}

// (host: called with the host copy of the model and an explicit geometry -- x_rows / base of the pass
// are placeholders there, see dec_build_ring_tables)
__host__ __device__ GemmDesc make_gemm_desc(const DecModel* m, int stage, int mode, int layer, const PassGeom* gopt) {
#ifdef __CUDA_ARCH__
  const PassGeom pg = gopt ? *gopt : pass_geom(m, mode);
#else
  const PassGeom pg = *gopt;
#endif
  GemmDesc g;
  const int d = m->d;
  g.d = d;
  g.x_row0 = 0;
  g.x_rows = pg.T;
  g.base = pg.base;
  g.out_row0 = 0;
  g.ln_g = g.ln_b = nullptr;
  g.kc = g.vc = nullptr;
  g.bias = nullptr;
  const DecLayer& L = m->layers[layer];
  switch (stage) {
    case ST_QKV:
      g.W = L.qkv_w; g.bias = L.qkv_b; g.N = 3 * d; g.K = d;
      g.xsrc = XS_LN; g.X = m->x; g.ln_g = L.ln1_g; g.ln_b = L.ln1_b;
      g.epi = EPI_QKV; g.out = m->q; g.ldo = d; g.kc = L.self_k; g.vc = L.self_v;
      break;
    case ST_OPROJ:
      g.W = L.o_w; g.bias = L.o_b; g.N = d; g.K = d;
      g.xsrc = XS_PLAIN; g.X = m->attn;
      g.epi = EPI_RESID; g.out = m->x; g.ldo = d;
      break;
    case ST_CROSS_Q:
      g.W = L.cq_w; g.bias = L.cq_b; g.N = d; g.K = d;
      g.xsrc = XS_LN; g.X = m->x; g.ln_g = L.ln2_g; g.ln_b = L.ln2_b;
      g.epi = EPI_STORE; g.out = m->q; g.ldo = d;
      break;
    case ST_CROSS_O:
      g.W = L.co_w; g.bias = L.co_b; g.N = d; g.K = d;
      g.xsrc = XS_PLAIN; g.X = m->attn;
      g.epi = EPI_RESID; g.out = m->x; g.ldo = d;
      break;
    case ST_FC1:
      g.W = L.fc1_w; g.bias = L.fc1_b; g.N = m->ffn; g.K = d;
      g.xsrc = XS_LN; g.X = m->x; g.ln_g = L.ln3_g; g.ln_b = L.ln3_b;
      g.epi = EPI_GELU; g.out = m->ffn_h; g.ldo = m->ffn;
      break;
    case ST_FC2:
      g.W = L.fc2_w; g.bias = L.fc2_b; g.N = d; g.K = m->ffn;
      g.xsrc = XS_PLAIN; g.X = m->ffn_h;
      g.epi = EPI_RESID; g.out = m->x; g.ldo = d;
      break;
    case ST_HEADS: {
      // head layer `layer` (MedusaResBlock `layer` of every head, reference model.py:235-246): its weights are the
      // layer-major stack's block `layer`
      const int nh = m->has_block ? m->K : m->K + 1;
      g.bias = m->heads_b + (size_t)layer * nh * d; g.W = m->heads_w + (size_t)layer * nh * d * d; g.K = d;
      g.xsrc = XS_PLAIN; g.out = head_layer_out(m, layer); g.ldo = d;
      if (mode == MODE_A) {
        g.N = nh * d; g.out_row0 = m->has_block ? 1 : 0;
        if (layer == 0) {
          // tail: every head on the hidden state of the newest token (generate_candidates reads
          // logits[:, -1]); block type: on the medusa block's output for that token
          g.X = m->has_block ? m->x : m->carry;
          g.x_row0 = 0; g.x_rows = 1;
          g.epi = EPI_HEADS_A;
        } else {
          // later layers: each head on its own row of the previous layer's output
          g.X = head_layer_out(m, layer - 1);
          g.x_row0 = g.out_row0; g.x_rows = nh;
          g.epi = EPI_HEADS_D;
        }
      } else {
        // verify (base_head type only): head 0 on every tree position (disable_medusa, model.py:1281-1284)
        g.X = layer == 0 ? m->hidden : head_layer_out(m, layer - 1); g.N = d; g.epi = EPI_HEAD_B;
      }
      break;
    }
    case ST_VOCAB:
    default:
      g.W = m->embed; g.N = m->V; g.K = d;
      g.xsrc = XS_PLAIN; g.X = m->head_h; g.x_rows = (mode == MODE_A) ? m->K + 1 : m->n_tree;
      g.epi = EPI_LOGITS; g.out = (mode == MODE_A) ? m->logits_a : m->logits_b; g.ldo = m->V;
      break;
  }
  return g;
}

// WITH_GEMM = false: the caller runs the GEMM stages itself (ring kernel) -- keeps stage_gemm out of
// that kernel's code.  ADJ: the logits scans with (1) or without (0) the logits-processor term, or chosen at run time
// from dec_state_adj (-1).  SMP: the sampled scan and folds of a sampled attempt (DecState smp_on; the processor term is
// then chosen at run time)
template <bool WITH_GEMM = true, int ADJ = -1, bool SMP = false>
__device__ void run_stage(const DecModel* m, int stage, int mode, int layer, int cta, int ncta, unsigned char* smem,
                          const PassGeom* gopt = nullptr, unsigned long long* pr = nullptr) {
  switch (stage) {
    case ST_EMBED: stage_embed(m, mode, cta, ncta, gopt); break;
    case ST_SELF_ATTN: stage_self_attn(m, mode, layer, cta, ncta, smem, gopt, pr); break;
    case ST_CROSS_ATTN: stage_cross_attn(m, mode, layer, cta, ncta, smem, gopt); break;
    case ST_FINAL_LN: stage_final_ln(m, mode, cta, ncta, gopt); break;
    case ST_COPY_HIDDEN: stage_copy_hidden_to_x(m, mode, cta, ncta, gopt); break;
    case ST_TAIL_SEED: stage_tail_seed(m, cta, ncta); break;
    case ST_SELECT1:
      if (SMP) stage_select1_smp(m, mode, cta, ncta, smem);
      else if (ADJ < 0) stage_select1(m, mode, cta, ncta, smem);
      else stage_select1_rows<(ADJ > 0)>(m, mode, cta, ncta, smem);
      break;
    case ST_SELECT2:
      if (ADJ < 0) stage_select2(m, cta, ncta, smem);
      else stage_select2_rows<(ADJ > 0)>(m, cta, ncta, smem);
      break;
    case ST_SELECT_FIN:
      if (cta == 0) {
        if (SMP) stage_select_fin<true>(m, ncta);
        else stage_select_fin(m, ncta);
      }
      break;
    case ST_ACCEPT:
      if (cta == 0) {
        if (m->has_tree) stage_accept_tree(m, ncta);
        else if (SMP) stage_accept<true>(m, ncta);
        else stage_accept(m, ncta);
      }
      break;
    case ST_KV_COMPACT: if (m->has_tree) stage_kv_compact(m, cta, ncta); break;
    default:
      if (WITH_GEMM) {
        GemmDesc g = make_gemm_desc(m, stage, mode, layer, gopt);
        stage_gemm(g, cta, ncta, smem);
      }
  }
}

// -----------------------------------------------------------------------------------------
// stage sequences (one definition shared by the graph builder on the host and the persistent
// kernel on the device)
// -----------------------------------------------------------------------------------------
template <class F>
__host__ __device__ void seq_layer(int l, int mode, F&& f) {
  f(ST_QKV, mode, l); f(ST_SELF_ATTN, mode, l); f(ST_OPROJ, mode, l); f(ST_CROSS_Q, mode, l);
  f(ST_CROSS_ATTN, mode, l); f(ST_CROSS_O, mode, l); f(ST_FC1, mode, l); f(ST_FC2, mode, l);
}
// decoder sweep over the rows of `mode` (+ the medusa block's K/V rows for them)
template <class F>
__host__ __device__ void seq_sweep(int n_layers, int has_block, int mode, F&& f) {
  f(ST_EMBED, mode, 0);
  for (int l = 0; l < n_layers; ++l) seq_layer(l, mode, f);
  f(ST_FINAL_LN, mode, 0);
  if (has_block) { f(ST_COPY_HIDDEN, mode, 0); f(ST_QKV, mode, n_layers); }
}
// candidates from the carried hidden state: (block on it,) K+1 heads (one stage per head layer), vocab projection, top-1
template <class F>
__host__ __device__ void seq_tail(int n_layers, int has_block, int n_head_layers, F&& f) {
  if (has_block) { f(ST_TAIL_SEED, MODE_TAIL, 0); seq_layer(n_layers, MODE_TAIL, f); }
  for (int l = 0; l < n_head_layers; ++l) f(ST_HEADS, MODE_A, l);
  f(ST_VOCAB, MODE_A, 0); f(ST_SELECT1, MODE_A, 0); f(ST_SELECT_FIN, MODE_A, 0);
}
// verify: sweep B, base logits of the K+1 positions, acceptance statistics, accept
template <class F>
__host__ __device__ void seq_verify(int n_layers, int has_block, int n_head_layers, F&& f) {
  seq_sweep(n_layers, has_block, MODE_B, f);
  if (!has_block)
    for (int l = 0; l < n_head_layers; ++l) f(ST_HEADS, MODE_B, l);
  f(ST_VOCAB, MODE_B, 0); f(ST_SELECT1, MODE_B, 0); f(ST_SELECT2, MODE_B, 0); f(ST_ACCEPT, MODE_B, 0);
  f(ST_KV_COMPACT, MODE_B, 0);   // (returns at once unless a candidate tree is configured)
}

// -----------------------------------------------------------------------------------------
// mode 0: one kernel per stage (captured into CUDA graphs by the host); SMP: the variant of sampled attempts
// -----------------------------------------------------------------------------------------
template <bool SMP = false>
__global__ void __launch_bounds__(WM_DEC_THREADS, 1)
dec_stage_kernel(const DecModel* __restrict__ m, int stage, int mode, int layer, int phase) {
  extern __shared__ __align__(128) unsigned char smem[];
  const DecState* st = m->st;
  if (st->done) return;
  if (phase == PH_SWEEP_A && !st->need_a) return;
  run_stage<true, -1, SMP>(m, stage, mode, layer, blockIdx.x, gridDim.x, smem);
}

// -----------------------------------------------------------------------------------------
// mode 1: persistent cooperative kernel -- one launch per speculative iteration
// -----------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned int ld_relaxed_u32(const unsigned int* p) {
  unsigned int v;
  asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p));
  return v;
}
// All CTAs are co-resident (cooperative launch).  bar[0] is a monotonically increasing arrival
// counter (reset by the host before every wm_generate): barrier number e completes when it
// reaches ncta * e.  Arrival is a release RED (MEMBAR.ALL.GPU + REDG), the poll a relaxed
// (L2-coherent) load.  ACQUIRE = false (ring kernel): no fence after the poll -- every cross-CTA
// read of that kernel is an L2-coherent load (common.cuh), so L1 need not be invalidated (ncu
// showed CCTL.IVALL after each barrier turning every LN/bias/local-memory access into an L2 trip).
template <bool ACQUIRE>
__device__ __forceinline__ unsigned int grid_barrier_step(unsigned int* bar, unsigned int epoch, int ncta) {
  // the ring kernel's consumers fetch activations with bulk async copies: order this thread's generic-proxy
  // global writes before async-proxy reads that follow the barrier.  In a 2-CTA cluster the peer multicasts the next
  // stage's rows into this CTA's scratch region (also used by the attention stages and the split passes) as soon as
  // the barrier opens: this thread's generic accesses of its shared memory must be ordered before those async writes
  // too.  Unclustered launches skip that fence (every CTA then writes only its own shared memory, after its own fence).
  if (!ACQUIRE) {
    asm volatile("fence.proxy.async.global;" ::: "memory");
    uint32_t ncl;
    asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(ncl));
    if (ncl > 1) asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  cta_sync();
  if (threadIdx.x == 0) {
    const unsigned int target = (unsigned int)ncta * (epoch + 1u);
    red_add_release(&bar[0], 1u);
    while (ld_relaxed_u32(&bar[0]) < target) { }
    if (ACQUIRE) __threadfence();
  }
  cta_sync();
  return epoch + 1u;
}
__device__ __forceinline__ void grid_barrier(unsigned int* bar, unsigned int& epoch, int ncta) {
  epoch = grid_barrier_step<true>(bar, epoch, ncta);
}

template <bool SMP = false>
__global__ void __launch_bounds__(WM_DEC_THREADS, 1)
dec_iteration_kernel(const DecModel* __restrict__ m) {
  extern __shared__ __align__(128) unsigned char smem[];
  const DecState* st = m->st;
  if (st->done) return;   // uniform: `done` / `need_a` only change in the last stage of an iteration
  const int need_a = st->need_a;
  // bar[2] = barrier epoch at kernel entry; only rewritten after the last barrier of a launch,
  // i.e. after every CTA has read it.
  unsigned int epoch = *reinterpret_cast<volatile unsigned int*>(&m->bar[2]);
  unsigned int* bar = m->bar;
  const int cta = blockIdx.x, ncta = gridDim.x;
  auto run = [&](int stage, int mode, int layer) {
    run_stage<true, -1, SMP>(m, stage, mode, layer, cta, ncta, smem);
    grid_barrier(bar, epoch, ncta);
  };
  if (need_a) seq_sweep(m->n_layers, m->has_block, MODE_A, run);
  if (!st->prefill) {   // (prefill: a 16-token chunk of a long prompt -- sweep A only)
    seq_tail(m->n_layers, m->has_block, m->n_head_layers, run);
    seq_verify(m->n_layers, m->has_block, m->n_head_layers, run);
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) m->bar[2] = epoch;
}

#include "decode_ring.cuh"

// -----------------------------------------------------------------------------------------
// host-side launchers
// -----------------------------------------------------------------------------------------
// Flattened stage program {stage, mode, layer} x n, lists: [off0,off1) sweep A, [off1,off2) tail,
// [off2,off3) verify -- what the ring kernel (consumer and producer side) walks.
void dec_build_program(int n_layers, int has_block, int n_head_layers, std::vector<int>& flat, int off[4]) {
  flat.clear();
  auto push = [&](int stage, int mode, int layer) { flat.push_back(stage); flat.push_back(mode); flat.push_back(layer); };
  off[0] = 0;
  seq_sweep(n_layers, has_block, MODE_A, push);
  off[1] = (int)flat.size() / 3;
  seq_tail(n_layers, has_block, n_head_layers, push);
  off[2] = (int)flat.size() / 3;
  seq_verify(n_layers, has_block, n_head_layers, push);
  off[3] = (int)flat.size() / 3;
}

size_t dec_ring_smem_bytes(int d) {
  switch (d) {
#define WM_CASE(DD) case DD: return RingGeom<DD>::TOTAL;
    WM_RING_WIDTHS(WM_CASE)
#undef WM_CASE
    default: return 0;   // width not instantiated: dec_configure / the launch report the error
  }
}

// Derived vectors of the LayerNorm-fed GEMMs (QKV, cross-Q, FC1) of the ring kernel, {b'_n, c_n} with
//     c_n = sum_k gamma_k W_nk,   b'_n = b_n + sum_k beta_k W_nk
// so that LN(x) W^T + b = rstd * ((gamma o x) W^T - mu * c) + b' (stage_gemm_ring).  Layout per decoder layer (the Medusa
// block included): QKV [3d] | cross-Q [d] | FC1 [ffn] float2.
size_t dec_ln_fold_len(int n_dec, int d, int ffn) { return (size_t)n_dec * (4 * (size_t)d + ffn); }
static size_t ln_fold_offset(int stage, int layer, int d, int ffn) {
  const size_t base = (size_t)layer * (4 * (size_t)d + ffn);
  return base + (stage == ST_QKV ? 0 : stage == ST_CROSS_Q ? 3 * (size_t)d : 4 * (size_t)d);
}

// One warp per row of W: lane l sums k = l, l+32, ... in fp64, then a fixed butterfly; rounded once to fp32.  The order
// does not depend on the launch, so every engine and every rank derives the same bits from the same weights.
__global__ void __launch_bounds__(256) ln_fold_kernel(const __half* __restrict__ W, const float* __restrict__ gamma,
                                                      const float* __restrict__ beta, const float* __restrict__ bias, int N, int K,
                                                      float2* __restrict__ out) {
  const int n = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (n >= N) return;
  const __half* w = W + (size_t)n * K;
  double c = 0.0, e = 0.0;
  for (int k = lane; k < K; k += 32) {
    const double wk = (double)__half2float(w[k]);
    c += (double)gamma[k] * wk;
    e += (double)beta[k] * wk;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    c += __shfl_xor_sync(0xffffffffu, c, o);
    e += __shfl_xor_sync(0xffffffffu, e, o);
  }
  if (lane == 0) out[n] = make_float2((float)((bias ? (double)bias[n] : 0.0) + e), (float)c);
}

cudaError_t dec_fold_layernorms(const DecModel& hm, int n_dec, float2* out, cudaStream_t s) {
  const PassGeom dyn{-1, 0};
  for (int l = 0; l < n_dec; ++l)
    for (const int stage : {ST_QKV, ST_CROSS_Q, ST_FC1}) {
      const GemmDesc g = make_gemm_desc(&hm, stage, MODE_B, l, &dyn);
      ln_fold_kernel<<<(g.N + 7) / 8, 256, 0, s>>>(g.W, g.ln_g, g.ln_b, g.bias, g.N, g.K,
                                                   out + ln_fold_offset(stage, l, hm.d, hm.ffn));
    }
  return cudaGetLastError();
}

// The host tables of the ring kernel, built in one walk of the stage program, so that the chunks the producer warp
// streams into the ring and the slots the compute warps take back out come from the same record.  `hm` is the HOST copy
// of the model (device pointers inside); `cluster`: CTAs per cluster of the launch the tables are for
// (dec_ring_cluster_size).
//   stab[ip * ncta + cta]: the resolved record of instruction ip for CTA cta (CtaStage in common.cuh);
//   ctab[off[cta * 4 + list] .. off[cta * 4 + list + 1]): the chunks of CTA cta for program list `list`, in the order
//   they are consumed: one per 16 rows of a GEMM record (stage_gemm_ring), the K and the V rows of every
//   cross-attention item of the CTA (stage_cross_attn_ring).
void dec_build_ring_tables(const DecModel& hm, const float2* ln_fold, int ncta, int cluster, std::vector<CtaStage>& stab,
                           std::vector<ChunkDesc>& ctab, std::vector<int>& off) {
  std::vector<int> flat;
  int poff[4];
  dec_build_program(hm.n_layers, hm.has_block, hm.n_head_layers, flat, poff);
  const int n = poff[3];
  const PassGeom dyn{-1, 0};   // T = -1: "the rows of the pass" (resolved on the device)
  auto desc = [&](int ip) { return make_gemm_desc(&hm, flat[ip * 3], flat[ip * 3 + 1], flat[ip * 3 + 2], &dyn); };
  // bias the ring kernel reads for a GEMM stage: LayerNorm stages read the {b'_n, c_n} pairs (8 bytes per row)
  auto ring_bias = [&](const GemmDesc& g, int ip, size_t& row_bytes) -> const float* {
    if (g.xsrc == XS_LN) {
      row_bytes = sizeof(float2);
      return reinterpret_cast<const float*>(ln_fold + ln_fold_offset(flat[ip * 3], flat[ip * 3 + 2], hm.d, hm.ffn));
    }
    row_bytes = sizeof(float);
    return g.bias;
  };
  auto push_chunk = [&](const void* src, size_t row_bytes, int nrows, size_t copy_bytes) {
    ctab.push_back(ChunkDesc{src, (uint32_t)row_bytes, (uint32_t)nrows, (uint32_t)copy_bytes, 0, 0, 0});
  };
  // LayerNorm gamma of the next instruction (bulk-copied into shared memory while this one runs)
  std::vector<const float*> nx_g(n, nullptr);
  for (int ip = 0; ip + 1 < n; ++ip)
    if (is_gemm_stage(flat[(ip + 1) * 3])) {
      const GemmDesc gn = desc(ip + 1);
      if (gn.xsrc == XS_LN) nx_g[ip] = gn.ln_g;
    }
  stab.assign((size_t)n * ncta, CtaStage{});
  ctab.clear();
  off.assign((size_t)ncta * 4, 0);
  for (int cta = 0; cta < ncta; ++cta) {
    for (int list = 0; list < 3; ++list) {
      off[(size_t)cta * 4 + list] = (int)ctab.size();
      for (int ip = poff[list]; ip < poff[list + 1]; ++ip) {
        const int stage = flat[ip * 3], layer = flat[ip * 3 + 2];
        CtaStage& c = stab[(size_t)ip * ncta + cta];
        c.stage = stage; c.mode = flat[ip * 3 + 1]; c.layer = layer;
        c.nx_g = nx_g[ip];
        // this CTA's bias slice of the next GEMM stage, if one follows within three instructions (L2 prefetch)
        for (int jn = ip + 1; jn < n && jn < ip + 4; ++jn) {
          if (!is_gemm_stage(flat[jn * 3])) continue;
          const GemmDesc gn = desc(jn);
          const GemmWork wn = gemm_work(gn.N, gn.K, hm.d, cta, ncta);
          size_t rb = 0;
          const float* nb = ring_bias(gn, jn, rb);
          if (nb && wn.n_rows > 0) {
            const uintptr_t a0 = ((uintptr_t)nb + wn.n_begin * rb) & ~(uintptr_t)127;
            const uintptr_t a1 = (uintptr_t)nb + (wn.n_begin + wn.n_rows) * rb;
            c.pf_bias = reinterpret_cast<const float*>(a0);
            c.pf_bias_lines = (int)std::min<uintptr_t>(32, (a1 - a0 + 127) / 128);
          }
          break;
        }
        if (stage == ST_CROSS_ATTN) {
          // the K and the V rows of every (head, key chunk) item of this CTA: one contiguous copy each
          const DecLayer& L = hm.layers[layer];
          for (int item = cta; item < hm.H * hm.cross_chunks; item += ncta) {
            const CrossItem it = cross_item(item, hm.S, hm.cross_chunks);
            if (it.nk == 0) continue;
            const size_t row0 = ((size_t)it.h * hm.S_pad + it.j0) * 72;
            push_chunk(L.cross_k + row0, 0, 1, it.nk * 72 * sizeof(__half));
            push_chunk(L.cross_v + row0, 0, 1, it.nk * 72 * sizeof(__half));
          }
          continue;
        }
        if (stage == ST_SELF_ATTN) {
          // per item of this CTA: its prefix blocks' K rows, then their V rows, sized at launch (sa_prefix_chunk).  A
          // sweep-A pass has a row count known only at launch, so every item the CTA can get at some row count is listed.
          const DecLayer& L = hm.layers[layer];
          int items = 0;
          for (int T = 1; T <= WM_MAX_T; ++T) {
            const SelfAttnSplit sp = self_attn_split(hm.H, T, ncta);
            items = std::max(items, (hm.H * sp.groups - cta + ncta - 1) / ncta);
          }
          for (int k = 0; k < items; ++k)
            for (const __half* cache : {L.self_k, L.self_v})
              for (int b = 0; b < WM_SA_BLOCKS; ++b)
                ctab.push_back(ChunkDesc{cache, 0u, 0u, 0u, (uint16_t)k, (uint8_t)c.mode, (uint8_t)b});
          continue;
        }
        if (!is_gemm_stage(stage)) continue;
        const GemmDesc g = desc(ip);
        const GemmWork wk = gemm_work(g.N, g.K, hm.d, cta, ncta);
        c.epi = g.epi;
        c.ln = (g.xsrc == XS_LN) ? 1 : 0;
        c.X = g.X + (size_t)g.x_row0 * g.K + (size_t)wk.seg * hm.d;
        c.x_ld = g.K;
        c.x_rows_fixed = g.x_rows < 0 ? 0 : g.x_rows;
        size_t rb = 0;
        c.bias = ring_bias(g, ip, rb);
        c.out = g.out;
        c.n_begin = wk.n_begin; c.n_rows = wk.n_rows;
        c.N = g.N; c.ldo = g.ldo; c.out_row0 = g.out_row0;
        c.segs = wk.segs; c.seg = wk.seg; c.block = wk.block;
        // activations that only ever feed one GEMM stage travel in the MMA operand format: the attention stages and
        // the GELU epilogue of FC1 write it, O-proj / cross-O / FC2 skip their split pass.  The residual stream feeds a
        // LayerNorm GEMM: the residual epilogue before one also writes gamma o x in that format (xg), and that stage
        // stages xg instead of x (layer 0 and the Medusa block, fed by other stages, split gamma o x themselves)
        const bool resid = (stage == ST_OPROJ || stage == ST_CROSS_O || stage == ST_FC2);
        c.presplit = resid ? 1 : 0;
        c.out_split = (stage == ST_FC1) ? 1 : 0;
        if (resid && c.nx_g) c.out_gx = hm.xg;
        if (c.ln && ip > 0) {
          const int ps = flat[(ip - 1) * 3];
          if (ps == ST_OPROJ || ps == ST_CROSS_O || ps == ST_FC2) { c.presplit = 1; c.X = hm.xg; }
        }
        // the weight rows of the record, 16 per chunk: d columns of k segment `seg`
        for (int r = 0; r < c.n_rows; r += 16)
          push_chunk(g.W + (size_t)(c.n_begin + r) * g.K + (size_t)c.seg * hm.d, g.K * sizeof(__half),
                     std::min(16, c.n_rows - r), hm.d * sizeof(__half));
      }
    }
    off[(size_t)cta * 4 + 3] = (int)ctab.size();
  }
  // 2-CTA clusters (CTAs 2i, 2i + 1): one multicast copy of X for both where they stage the same rows.  Both must have
  // rows: a CTA without rows returns before staging, and the peer's complete_tx would then shift its xbar phase.
  if (cluster == 2)
    for (int ip = 0; ip < n; ++ip) {
      if (!is_gemm_stage(flat[ip * 3])) continue;
      for (int cta = 0; cta + 1 < ncta; cta += 2) {
        CtaStage& a = stab[(size_t)ip * ncta + cta];
        CtaStage& b = stab[(size_t)ip * ncta + cta + 1];
        if (a.n_rows > 0 && b.n_rows > 0 && a.X == b.X && a.x_ld == b.x_ld && a.x_rows_fixed == b.x_rows_fixed) {
          a.x_role = XR_ISSUE;
          b.x_role = XR_RECEIVE;
        }
      }
    }
}

// Host replay of the ring protocol (no GPU): for each CTA and each launch state, the chunks the producer warp copies
// (ring_walk, as ring_producer runs it) against what the compute warps expect in the slots they take (stage_gemm_ring,
// stage_cross_attn_ring, stage_self_attn_ring), compared as (source, rows, bytes).  The walk's L2 prefetches at
// `budget` bytes (< 0: the built WM_RING_L2_AHEAD) are replayed along, chunk by chunk: each must be copied later in the
// same launch, in prefetch order, or be one of the first weight chunks of the tail program (the next launch's); the
// bytes prefetched and not yet copied never exceed the budget; and with a budget every copy was prefetched first.
// Launch states: every kv0 in [0, WM_MAX_POS - 16] with sweep A skipped (L0 = kv0), with sweep A over t_a = 1 ... 16
// rows (L0 = kv0 + t_a), and prefill chunks of 16 rows; those whose verify rows would pass WM_MAX_POS are left out.
// Returns the number of (launch, CTA) pairs whose sequences differ or whose prefetches break a rule; `first` receives
// {kv0, L0, need_a, cta} of the first of them.
int dec_check_ring_schedule(const DecModel& hm, int ncta, long long budget, int first[4]) {
  const uint32_t l2_ahead = budget < 0 ? (uint32_t)WM_RING_L2_AHEAD : (uint32_t)budget;
  std::vector<CtaStage> stab;
  std::vector<ChunkDesc> ctab;
  std::vector<int> off;
  const float2* fold = reinterpret_cast<const float2*>(uintptr_t(1) << 40);   // (never dereferenced)
  dec_build_ring_tables(hm, fold, ncta, 1, stab, ctab, off);
  std::vector<int> flat;
  int poff[4];
  dec_build_program(hm.n_layers, hm.has_block, hm.n_head_layers, flat, poff);
  struct Copy {
    const void* src; uint32_t nrows, bytes;
    bool operator==(const Copy& o) const { return src == o.src && nrows == o.nrows && bytes == o.bytes; }
  };
  const uint32_t kv_bytes = WM_KV_ROW * sizeof(__half);
  // what the GEMM and cross-attention stages of instruction ip take from the ring at CTA cta: fixed for every launch
  std::vector<std::vector<Copy>> fixed((size_t)poff[3] * ncta);
  for (int ip = 0; ip < poff[3]; ++ip) {
    const int stage = flat[ip * 3], mode = flat[ip * 3 + 1], layer = flat[ip * 3 + 2];
    const DecLayer& L = hm.layers[layer];
    const PassGeom dyn{-1, 0};
    if (stage == ST_CROSS_ATTN) {
      for (int item = 0; item < hm.H * hm.cross_chunks; ++item) {
        const CrossItem it = cross_item(item, hm.S, hm.cross_chunks);
        if (it.nk == 0) continue;
        const size_t row0 = ((size_t)it.h * hm.S_pad + it.j0) * 72;
        std::vector<Copy>& f = fixed[(size_t)ip * ncta + item % ncta];
        f.push_back(Copy{L.cross_k + row0, 1u, it.nk * kv_bytes});
        f.push_back(Copy{L.cross_v + row0, 1u, it.nk * kv_bytes});
      }
    }
    if (!is_gemm_stage(stage)) continue;
    const GemmDesc g = make_gemm_desc(&hm, stage, mode, layer, &dyn);
    for (int cta = 0; cta < ncta; ++cta) {
      std::vector<Copy>& f = fixed[(size_t)ip * ncta + cta];
      const CtaStage& sd = stab[(size_t)ip * ncta + cta];
      for (int u = 0; u * 16 < sd.n_rows; ++u)
        f.push_back(Copy{g.W + (size_t)(sd.n_begin + 16 * u) * g.K + (size_t)sd.seg * hm.d,
                         (uint32_t)std::min(16, sd.n_rows - 16 * u), (uint32_t)(hm.d * sizeof(__half))});
    }
  }
  std::vector<Copy> prod, cons;
  // prefetched chunks not yet matched by a copy, in prefetch order: [pf_head, pending.size())
  std::vector<ChunkCopy> pending;
  auto same = [](const ChunkCopy& x, const ChunkCopy& y) {
    return x.src == y.src && x.row_bytes == y.row_bytes && x.nrows == y.nrows && x.copy_bytes == y.copy_bytes;
  };
  int bad = 0;
  auto run = [&](int L0, int kv0, int need_a, int prefill) {
    for (int cta = 0; cta < ncta; ++cta) {
      prod.clear();
      cons.clear();
      pending.clear();
      size_t pf_head = 0;
      const int* o = &off[(size_t)cta * 4];
      bool pf_ok = true;
      uint64_t pending_bytes = 0;
      ring_walk(
          ctab.data(), need_a ? o[0] : o[1], prefill ? o[1] : o[3], o[1], o[3], l2_ahead, hm.H, hm.n_tree, cta, ncta, L0, kv0,
          [&](const ChunkCopy& p) {
            pending.push_back(p);
            pending_bytes += (uint64_t)p.nrows * p.copy_bytes;
            pf_ok = pf_ok && pending_bytes <= l2_ahead;
          },
          [&](const ChunkCopy& cp) {
            prod.push_back(Copy{cp.src, cp.nrows, cp.copy_bytes});
            // the copy must be of the oldest prefetched chunk, or (no budget) of one never prefetched
            if (pf_head < pending.size() && same(pending[pf_head], cp)) {
              pending_bytes -= (uint64_t)cp.nrows * cp.copy_bytes;
              ++pf_head;
            } else {
              pf_ok = pf_ok && l2_ahead == 0;
            }
          });
      // what is left was prefetched for the next launch: the tail program's leading weight chunks, in order
      for (size_t i = pf_head, c = o[1]; i < pending.size() && pf_ok; ++i, ++c) {
        pf_ok = (int)c < o[3] && ctab[c].nrows != 0 &&
                same(pending[i], ChunkCopy{reinterpret_cast<const unsigned char*>(ctab[c].src), ctab[c].row_bytes,
                                           ctab[c].nrows, ctab[c].copy_bytes});
      }
      for (int ip = need_a ? poff[0] : poff[1]; ip < (prefill ? poff[1] : poff[3]); ++ip) {
        const int stage = flat[ip * 3], mode = flat[ip * 3 + 1], layer = flat[ip * 3 + 2];
        if (stage != ST_SELF_ATTN) {
          const std::vector<Copy>& f = fixed[(size_t)ip * ncta + cta];
          cons.insert(cons.end(), f.begin(), f.end());
          continue;
        }
        const DecLayer& L = hm.layers[layer];
        const PassGeom g = pass_geom(mode, L0, kv0, hm.n_tree);
        const SelfAttnSplit sp = self_attn_split(hm.H, g.T, ncta);
        int k = 0;
        for (int item = cta; item < hm.H * sp.groups; item += ncta, ++k) {
          const int h = item / sp.groups, P = std::min(g.base, kv0);
          for (const __half* cache : {L.self_k, L.self_v})
            for (int b = 0; b < WM_SA_BLOCKS; ++b) {
              const SaChunk s = sa_prefix_chunk(hm.H, ncta, cta, mode, L0, kv0, hm.n_tree, k, b);
              if (s.nk == 0) continue;
              const int nk = std::min(WM_SA_BLOCK, P - b * WM_SA_BLOCK);   // the keys the stage reads from this slot
              cons.push_back(Copy{cache + self_kv_index(b * WM_SA_BLOCK, h * 64), 1u, (uint32_t)nk * kv_bytes});
            }
        }
      }
      if (!(prod == cons) || !pf_ok) {
        if (bad++ == 0) { first[0] = kv0; first[1] = L0; first[2] = need_a; first[3] = cta; }
      }
    }
  };
  for (int kv0 = 0; kv0 <= WM_MAX_POS - 16; ++kv0) {
    if (kv0 >= 1 && kv0 + hm.n_tree <= WM_MAX_POS) run(kv0, kv0, 0, 0);
    for (int t_a = 1; t_a <= WM_MAX_T; ++t_a)
      if (kv0 + t_a + hm.n_tree <= WM_MAX_POS) run(kv0 + t_a, kv0, 1, 0);
    run(kv0 + 16, kv0, 1, 1);
  }
  return bad;
}

cudaError_t dec_relayout_cross_kv(const __half* kv, __half* ck, __half* cv, int S, int S_pad, int d, int H, cudaStream_t s,
                                  int64_t* n_launch) {
  relayout_cross_kv_kernel<<<296, 256, 0, s>>>(kv, ck, cv, S, S_pad, d, H);
  if (n_launch) ++*n_launch;
  return cudaGetLastError();
}

// profile: the stage-timeline variant (processors chosen at run time); smp: the variant of sampled attempts (processors
// chosen at run time); lp: the variant with logits processors
static void* ring_kernel_fn(int d, bool profile, bool lp = false, bool smp = false) {
  switch (d) {
#define WM_CASE(DD)                                                                                                          \
  case DD:                                                                                                                   \
    if (smp) return profile ? (void*)dec_iteration_ring_kernel<DD, true, false, true> : (void*)dec_iteration_ring_kernel<DD, false, false, true>; \
    return profile ? (void*)dec_iteration_ring_kernel<DD, true, false>                                                      \
                   : lp ? (void*)dec_iteration_ring_kernel<DD, false, true> : (void*)dec_iteration_ring_kernel<DD, false, false>;
    WM_RING_WIDTHS(WM_CASE)
#undef WM_CASE
    default: return nullptr;
  }
}

// Cooperative launch (the grid barrier needs every CTA resident), as clusters of hi.cluster CTAs along x.
cudaError_t dec_launch_iteration_ring(const DecModel* dm, const DecHostInfo& hi, bool profile, cudaStream_t s) {
  void* fn = ring_kernel_fn(hi.d, profile, hi.lp != 0, hi.smp != 0);
  if (!fn) return cudaErrorInvalidValue;
  void* args[] = {(void*)&dm};
  cudaLaunchAttribute attr[2];
  attr[0].id = cudaLaunchAttributeCooperative;
  attr[0].val.cooperative = 1;
  attr[1].id = cudaLaunchAttributeClusterDimension;
  attr[1].val.clusterDim.x = (unsigned)hi.cluster;
  attr[1].val.clusterDim.y = 1;
  attr[1].val.clusterDim.z = 1;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(hi.n_sm);
  cfg.blockDim = dim3(WM_RING_THREADS);
  cfg.dynamicSmemBytes = hi.smem_ring;
  cfg.stream = s;
  cfg.attrs = attr;
  cfg.numAttrs = hi.cluster > 1 ? 2 : 1;
  return cudaLaunchKernelExC(&cfg, fn, args);
}

// CTAs per cluster of the ring kernel on a grid of hi.n_sm CTAs: 2 when the grid is the whole device (an even number of
// SMs) and the device can hold n_sm / 2 such clusters at once, else 1.  Needs dec_configure first (shared-memory size).
int dec_ring_cluster_size(const DecHostInfo& hi, int n_sm) {
  void* fn = ring_kernel_fn(hi.d, false);
  if (!fn || hi.n_sm != n_sm || n_sm % 2 != 0) return 1;
  cudaLaunchAttribute attr;
  attr.id = cudaLaunchAttributeClusterDimension;
  attr.val.clusterDim.x = 2;
  attr.val.clusterDim.y = 1;
  attr.val.clusterDim.z = 1;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(n_sm);
  cfg.blockDim = dim3(WM_RING_THREADS);
  cfg.dynamicSmemBytes = hi.smem_ring;
  cfg.attrs = &attr;
  cfg.numAttrs = 1;
  int n = 0;
  if (cudaOccupancyMaxActiveClusters(&n, fn, &cfg) != cudaSuccess) {
    (void)cudaGetLastError();
    return 1;
  }
  return n >= n_sm / 2 ? 2 : 1;
}

size_t dec_smem_bytes(int d, int ffn) {
  size_t s = gemm_smem_bytes(d);
  size_t s2 = gemm_smem_bytes(ffn);
  if (s2 > s) s = s2;
  if (self_attn_smem_bytes() > s) s = self_attn_smem_bytes();
  if (cross_attn_smem_bytes() > s) s = cross_attn_smem_bytes();
  return s;
}

cudaError_t dec_configure(int d, size_t smem, size_t smem_ring) {
  for (const void* fn : {(const void*)dec_stage_kernel<false>, (const void*)dec_stage_kernel<true>,
                         (const void*)dec_iteration_kernel<false>, (const void*)dec_iteration_kernel<true>}) {
    const cudaError_t e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
  }
  cudaError_t e;
  if (smem_ring == 0) return cudaSuccess;   // decoder width without a ring instantiation: persistent mode refuses to run
  switch (d) {
#define WM_CASE(DD)                                                                                                          \
  case DD:                                                                                                                   \
    e = cudaFuncSetAttribute(dec_iteration_ring_kernel<DD, false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_ring); \
    if (e != cudaSuccess) return e;                                                                                          \
    e = cudaFuncSetAttribute(dec_iteration_ring_kernel<DD, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_ring); \
    if (e != cudaSuccess) return e;                                                                                          \
    e = cudaFuncSetAttribute(dec_iteration_ring_kernel<DD, false, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_ring); \
    if (e != cudaSuccess) return e;                                                                                          \
    e = cudaFuncSetAttribute(dec_iteration_ring_kernel<DD, true, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_ring); \
    if (e != cudaSuccess) return e;                                                                                          \
    return cudaFuncSetAttribute(dec_iteration_ring_kernel<DD, true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_ring);
    WM_RING_WIDTHS(WM_CASE)
#undef WM_CASE
    default: return cudaErrorInvalidValue;
  }
}

static int stage_grid(int stage, int T, int n_sm, int H, int K) {
  switch (stage) {
    case ST_EMBED: return T;
    case ST_SELF_ATTN: return H * T;
    case ST_CROSS_ATTN: return H * WM_CROSS_CHUNKS;   // upper bound; items = H * m->cross_chunks
    case ST_FINAL_LN: return 1;
    case ST_COPY_HIDDEN: return 8;
    case ST_TAIL_SEED: return 2;
    case ST_SELECT_FIN: return 1;
    case ST_ACCEPT: return 1;
    case ST_KV_COMPACT: return 2 * WM_MAX_DEC_LAYERS;
    default: return n_sm;
  }
}

// Enqueue one phase as individual stage kernels (captured into a graph by the caller).
//   PH_SWEEP_A: sweep over T uncached rows (kernels return at once unless state.need_a)
//   PH_TAIL   : candidates from the carried hidden state
//   PH_VERIFY : sweep B + acceptance
cudaError_t dec_enqueue_phase(const DecModel* dm, const DecHostInfo& hi, int phase, int T, cudaStream_t s, int64_t* n_launch) {
  auto launch = [&](int stage, int mode, int layer) {
    const int rows = pass_geom(mode, T, 0, hi.n_tree).T;   // (sweep A over T rows: L = T, kv_len = 0)
    const int grid = stage_grid(stage, rows, hi.n_sm, hi.H, hi.K);
    // (sweep A has no logits scan: its graphs, shared by every call, keep the kernel without sampling)
    if (hi.smp && phase != PH_SWEEP_A) dec_stage_kernel<true><<<grid, WM_DEC_THREADS, hi.smem, s>>>(dm, stage, mode, layer, phase);
    else dec_stage_kernel<false><<<grid, WM_DEC_THREADS, hi.smem, s>>>(dm, stage, mode, layer, phase);
    if (n_launch) ++*n_launch;
  };
  if (phase == PH_SWEEP_A) seq_sweep(hi.n_layers, hi.has_block, MODE_A, launch);
  else if (phase == PH_TAIL) seq_tail(hi.n_layers, hi.has_block, hi.n_head_layers, launch);
  else seq_verify(hi.n_layers, hi.has_block, hi.n_head_layers, launch);
  return cudaGetLastError();
}

__global__ void sample_noise_kernel(uint2 key, unsigned int window, unsigned int attempt, int n, int j0, int count,
                                    float* __restrict__ out) {
  const unsigned int k[2] = {key.x, key.y};
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < count; i += gridDim.x * blockDim.x)
    out[i] = sample_gumbel(k, window, attempt, n, j0 + i);
}
cudaError_t dec_launch_sample_noise(const unsigned int key[2], unsigned int window, unsigned int attempt, int n, int j0,
                                    int count, float* out, cudaStream_t s) {
  sample_noise_kernel<<<std::min(1024, (count + 255) / 256), 256, 0, s>>>(make_uint2(key[0], key[1]), window, attempt, n,
                                                                          j0, count, out);
  return cudaGetLastError();
}

cudaError_t dec_launch_iteration(const DecModel* dm, const DecHostInfo& hi, cudaStream_t s) {
  void* args[] = {(void*)&dm};
  const void* fn = hi.smp ? (const void*)dec_iteration_kernel<true> : (const void*)dec_iteration_kernel<false>;
  return cudaLaunchCooperativeKernel(fn, dim3(hi.n_sm), dim3(WM_DEC_THREADS), args, hi.smem, s);
}

}  // namespace wm
