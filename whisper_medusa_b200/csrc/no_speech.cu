// No-speech probability of a window (transcribe(no_speech_threshold=..., logprob_threshold=...)).
//
// The loop stores the final-LayerNorm hidden state of the start-of-transcript row (DecModel::ns_hidden, captured by
// stage_final_ln in the first real iteration's sweep A).  After the loop, this file turns it into the base head's raw
// logits row -- what the model's forward returns for that position:
//   base_head type    : proj_out(h + SiLU(W0 h + b0))   (head 0 first, reference model.py:1274-1280)
//   medusa_block type : proj_out(h)                     (reference model.py:1287)
// and the row's log-sum-exp, so that p[token] = exp(logit[token] - lse) (HF WhisperNoSpeechDetection).
//
// Rounding: every matrix-vector product stages its input row as the ring kernel's GEMM stages stage their activations
// (decode.cu stage_gemm): y -> hi = fp16_rn(y), lo = fp16_rn(y - hi), and accumulates w*hi + w*lo in fp32 (each product
// of two fp16 values is exact in fp32).  Only the order of the fp32 sums differs from the loop's mma.sync tiles.
//
// The vocabulary product streams the fp16 matrix once (large-v2: 51865 x 1280 x 2 B = 132.8 MB) with 16-byte
// non-coherent loads, two rows per warp in flight.  An online softmax runs beside it: each of WM_NS_NSEG fixed
// vocabulary segments leaves one (max, sum of exp) pair, and the last CTA to arrive folds them in segment order, so
// neither the logits nor the log-sum-exp depend on the grid size.
#include <algorithm>

#include "common.cuh"
#include "engine.h"

namespace wm {

namespace {

constexpr int NS_NW = WM_NS_THREADS / 32;
constexpr int NS_MAXC = 1280 / 256;   // 16-byte weight chunks per lane and row (d <= 1280)

// (max, sum of exp(v - max)) pairs; -inf max = empty
__device__ __forceinline__ void lse_merge(float& m, float& s, float om, float os) {
  if (om == -INFINITY) return;
  if (m == -INFINITY) { m = om; s = os; return; }
  if (om > m) { s = s * expf(m - om) + os; m = om; }
  else s += os * expf(om - m);
}

// the input row in the GEMM stages' operand format, widened to fp32 (s_hi, s_lo: [d])
__device__ __forceinline__ void stage_row(const float* x, int d, float* s_hi, float* s_lo) {
  for (int k = threadIdx.x; k < d; k += blockDim.x) {
    const float y = __ldcg(x + k);
    const __half h = __float2half_rn(y);
    s_hi[k] = __half2float(h);
    s_lo[k] = __half2float(__float2half_rn(y - __half2float(h)));
  }
}

// sum_k w[k] * (hi[k] + lo[k]) over one 16-byte chunk (8 columns starting at k0), products added hi then lo
__device__ __forceinline__ float dot8(uint4 w, const float* s_hi, const float* s_lo, int k0, float acc) {
  const __half2* wh = reinterpret_cast<const __half2*>(&w);
  const float4 h0 = *reinterpret_cast<const float4*>(s_hi + k0), h1 = *reinterpret_cast<const float4*>(s_hi + k0 + 4);
  const float4 l0 = *reinterpret_cast<const float4*>(s_lo + k0), l1 = *reinterpret_cast<const float4*>(s_lo + k0 + 4);
  const float hv[8] = {h0.x, h0.y, h0.z, h0.w, h1.x, h1.y, h1.z, h1.w};
  const float lv[8] = {l0.x, l0.y, l0.z, l0.w, l1.x, l1.y, l1.z, l1.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 wf = __half22float2(wh[i]);
    acc = fmaf(wf.x, hv[2 * i], acc);
    acc = fmaf(wf.y, hv[2 * i + 1], acc);
    acc = fmaf(wf.x, lv[2 * i], acc);
    acc = fmaf(wf.y, lv[2 * i + 1], acc);
  }
  return acc;
}

// base_head type: head_out[n] = x[n] + SiLU(b0[n] + W0[n] . x), x taken as hi + lo (the heads epilogue, decode.cu
// gemm_epilogue_heads).  One warp per output row.
__global__ void __launch_bounds__(WM_NS_THREADS) no_speech_head_kernel(NoSpeechArgs p) {
  extern __shared__ __align__(16) float s_x[];
  const int d = p.d, nc = d >> 3;
  float* s_hi = s_x;
  float* s_lo = s_x + d;
  stage_row(p.hidden, d, s_hi, s_lo);
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int n = blockIdx.x * NS_NW + warp; n < d; n += gridDim.x * NS_NW) {
    const __half* w = p.head_w + (size_t)n * d;
    float acc = 0.f;
#pragma unroll
    for (int u = 0; u < NS_MAXC; ++u) {
      const int c = lane + 32 * u;
      if (c < nc) acc = dot8(ldg_nc_v4(w + 8 * c), s_hi, s_lo, 8 * c, acc);
    }
    acc = warp_sum(acc);
    if (lane == 0) p.head_out[n] = (s_hi[n] + s_lo[n]) + silu(acc + p.head_b[n]);
  }
}

__global__ void __launch_bounds__(WM_NS_THREADS) no_speech_vocab_kernel(NoSpeechArgs p) {
  extern __shared__ __align__(16) float s_x[];
  __shared__ float s_m[NS_NW], s_s[NS_NW];
  __shared__ int s_last;
  const int d = p.d, nc = d >> 3, V = p.V;
  float* s_hi = s_x;
  float* s_lo = s_x + d;
  stage_row(p.head_w ? p.head_out : p.hidden, d, s_hi, s_lo);
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int seglen = (V + WM_NS_NSEG - 1) / WM_NS_NSEG;

  for (int sg = blockIdx.x; sg < WM_NS_NSEG; sg += gridDim.x) {
    const int j0 = min(V, sg * seglen), j1 = min(V, j0 + seglen);
    float m = -INFINITY, s = 0.f;
    // rows j and j + NS_NW of the segment per step: 2 x d x 2 bytes of weights in flight per warp
    for (int j = j0 + warp; j < j1; j += 2 * NS_NW) {
      const int jb = j + NS_NW;
      const bool has_b = jb < j1;
      const __half* wa = p.embed + (size_t)j * d;
      const __half* wb = p.embed + (size_t)(has_b ? jb : j) * d;
      uint4 ra[NS_MAXC], rb[NS_MAXC];
#pragma unroll
      for (int u = 0; u < NS_MAXC; ++u) {
        const int c = lane + 32 * u;
        if (c < nc) {
          ra[u] = ldg_nc_v4(wa + 8 * c);
          rb[u] = has_b ? ldg_nc_v4(wb + 8 * c) : make_uint4(0, 0, 0, 0);
        }
      }
      float va = 0.f, vb = 0.f;
#pragma unroll
      for (int u = 0; u < NS_MAXC; ++u) {
        const int c = lane + 32 * u;
        if (c < nc) {
          va = dot8(ra[u], s_hi, s_lo, 8 * c, va);
          vb = dot8(rb[u], s_hi, s_lo, 8 * c, vb);
        }
      }
      va = warp_sum(va);
      vb = warp_sum(vb);
      if (lane == 0) {
        p.logits[j] = va;
        if (has_b) p.logits[jb] = vb;
      }
      lse_merge(m, s, va, 1.f);
      if (has_b) lse_merge(m, s, vb, 1.f);
    }
    __syncthreads();   // (s_m / s_s of the previous segment have been read)
    if (lane == 0) { s_m[warp] = m; s_s[warp] = s; }
    __syncthreads();
    if (threadIdx.x == 0) {
      float M = -INFINITY, S = 0.f;
      for (int w = 0; w < NS_NW; ++w) lse_merge(M, S, s_m[w], s_s[w]);
      p.part[2 * sg] = M;
      p.part[2 * sg + 1] = S;
    }
  }

  // last CTA to arrive folds the segment partials in segment order (threadFenceReduction pattern)
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    s_last = (atomicAdd(p.count, 1u) == gridDim.x - 1);
  }
  __syncthreads();
  if (!s_last || warp != 0) return;
  __threadfence();
  float M = -INFINITY, S = 0.f;   // lane l: segments l, l + 32, ...
  for (int sg = lane; sg < WM_NS_NSEG; sg += 32) lse_merge(M, S, __ldcg(p.part + 2 * sg), __ldcg(p.part + 2 * sg + 1));
  float TM = -INFINITY, TS = 0.f;
  for (int l = 0; l < 32; ++l) lse_merge(TM, TS, __shfl_sync(0xffffffffu, M, l), __shfl_sync(0xffffffffu, S, l));
  if (lane == 0) {
    *p.lse = TM + logf(TS);
    *p.count = 0u;
  }
}

}  // namespace

cudaError_t dec_launch_no_speech(const NoSpeechArgs& a, int grid, cudaStream_t s, int64_t* n_launch) {
  const size_t smem = (size_t)2 * a.d * sizeof(float);
  NoSpeechArgs v = a;
  if (a.head_w) {
    // one launch per layer of head 0, alternating between the halves of head_out: a layer's input row is staged by
    // every CTA before any CTA of the next launch writes
    for (int l = 0; l < a.head_layers; ++l) {
      NoSpeechArgs al = a;
      al.hidden = l == 0 ? a.hidden : a.head_out + (size_t)((l - 1) & 1) * a.d;
      al.head_w = a.head_w + (size_t)l * a.head_stride * a.d;
      al.head_b = a.head_b + (size_t)l * a.head_stride;
      al.head_out = a.head_out + (size_t)(l & 1) * a.d;
      no_speech_head_kernel<<<std::max(1, std::min(grid, (a.d + NS_NW - 1) / NS_NW)), WM_NS_THREADS, smem, s>>>(al);
      const cudaError_t e = cudaGetLastError();
      if (e != cudaSuccess) return e;
      ++*n_launch;
    }
    v.head_out = a.head_out + (size_t)((a.head_layers - 1) & 1) * a.d;
  }
  no_speech_vocab_kernel<<<std::max(1, std::min(grid, WM_NS_NSEG)), WM_NS_THREADS, smem, s>>>(v);
  ++*n_launch;
  return cudaGetLastError();
}

}  // namespace wm
