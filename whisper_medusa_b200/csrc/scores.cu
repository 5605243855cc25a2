// Scores and per-token log-probabilities of the speculative loop (generate(return_dict_in_generate=True, ...)).
//
// One launch after every iteration, enqueued only when scoring is on.  It only reads what the loop left behind --
// logits_a (the tail's rows), logits_b (the verify rows) and the loop state -- and keeps its own cursor (the first
// position not scored yet), so an iteration that did not run (the loop ended earlier in the batch) costs one early
// return.  With L0 = the cursor (len(input_ids) at the start of the iteration), a = the accept length and path = the
// best candidate's root-to-leaf nodes, every row is processed with cur_len = L0 (processed_logit, with the iteration's
// logits-processor term adj when processors are on) and:
//   token at L0          (c0)                 <- base row 0 of the tail (logits_a)
//   token at L0 + j, j>=1 (c1..ca / the extra) <- verify row path[j - 1]
//   scores row of the iteration              <- verify row path[a] (the reference's next_token_logits)
// log_softmax at temperature 1: fp32, max-subtracted, in WM_SCORE_NSEG vocabulary segments per row whose partials are
// folded in segment order by the last CTA to arrive, so the result does not depend on the grid size.
// TAU (a sampled attempt with top-k): a token row keeps only its top-k set {v >= tau} (DecState tail_tau for c0, row_tau
// for verify rows), as HF's log_softmax of the warped scores times the temperature; the scores rows stay unrestricted.
#include <algorithm>

#include "common.cuh"
#include "engine.h"

namespace wm {

namespace {

// (max, sum of exp(v - max)) pairs; -inf max = empty
__device__ __forceinline__ void lse_merge(float& m, float& s, float om, float os) {
  if (om == -INFINITY) return;
  if (m == -INFINITY) { m = om; s = os; return; }
  if (om > m) { s = s * expf(m - om) + os; m = om; }
  else s += os * expf(om - m);
}

// node of the best path at depth `dep` (chain: the node is its depth; tree: walk up from path[a], stored by the accept stage)
__device__ __forceinline__ int path_node(const DecState* st, const DecTree* tree, int a, int dep) {
  if (!tree) return dep;
  int node = st->path_node;
  for (int k = a; k > dep; --k) node = tree->parent[node];
  return node;
}

template <bool ADJ, bool TAU = false>
__global__ void __launch_bounds__(WM_SCORE_THREADS) score_iteration_kernel(ScoreArgs p) {
  constexpr int NW = WM_SCORE_THREADS / 32;
  __shared__ float s_m[NW], s_s[NW];
  __shared__ int s_last;
  const DecState* st = p.st;
  const int it = st->n_iter;         // (written by the previous kernel on the stream)
  const int seen = p.state[0];
  if (it == seen) return;            // the loop had already ended: nothing new to score (uniform across the grid)
  const int L0 = seen == 0 ? p.n_prompt : p.state[1];
  const int L = st->L;
  const int a = st->accept_hist[it - 1];
  const int n_lp = p.want_lp ? L - L0 : 0;    // token rows
  const int n_rows = n_lp + (p.want_rows && it - 1 < p.cap_rows ? 1 : 0);
  const bool begin_on = (L0 == st->begin_index);
  const float pen = p.pen_tab[L0];
  const int eos = st->eos;
  const int V = p.V;
  const int seglen = (V + WM_SCORE_NSEG - 1) / WM_SCORE_NSEG;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;

  for (int item = blockIdx.x; item < n_rows * WM_SCORE_NSEG; item += gridDim.x) {
    const int r = item / WM_SCORE_NSEG, sg = item - r * WM_SCORE_NSEG;
    const int j0 = sg * seglen, j1 = min(V, j0 + seglen);
    if (r == n_lp) {   // the scores row: the processed verify row path[a]
      const float* row = p.logits_b + (size_t)path_node(st, p.tree, a, a) * V;
      float* out = p.rows + (size_t)(it - 1) * V;
      for (int j = j0 + threadIdx.x; j < j1; j += WM_SCORE_THREADS) out[j] = processed_logit<ADJ>(row, j, p.tok_mask, begin_on, eos, pen, p.adj);
      continue;
    }
    const float* row = (r == 0) ? p.logits_a : p.logits_b + (size_t)path_node(st, p.tree, a, r - 1) * V;
    const float tau = TAU ? (r == 0 ? st->tail_tau : st->row_tau[r - 1]) : -INFINITY;
    if (threadIdx.x == 0) {   // the segment holding the row's token also records its processed logit for the fold
      const int tok = st->ids[L0 + r];
      if (tok >= j0 && tok < j1) p.part[(size_t)(WM_MAX_T + 1) * WM_SCORE_NSEG * 2 + r] = processed_logit<ADJ>(row, tok, p.tok_mask, begin_on, eos, pen, p.adj);
    }
    float m = -INFINITY, s = 0.f;
    // WM_SCORE_UNROLL elements per thread in flight at once: the segment is read from L2, and one element at a time
    // would pay the load latency per element
    for (int jb = j0 + threadIdx.x; jb < j1; jb += WM_SCORE_UNROLL * WM_SCORE_THREADS) {
      float v[WM_SCORE_UNROLL];
#pragma unroll
      for (int u = 0; u < WM_SCORE_UNROLL; ++u) {
        const int j = jb + u * WM_SCORE_THREADS;
        v[u] = j < j1 ? processed_logit<ADJ>(row, j, p.tok_mask, begin_on, eos, pen, p.adj) : -INFINITY;
        if (TAU && v[u] < tau) v[u] = -INFINITY;
      }
#pragma unroll
      for (int u = 0; u < WM_SCORE_UNROLL; ++u) {
        if (v[u] > m) { s = s * expf(m - v[u]) + 1.f; m = v[u]; }
        else if (v[u] != -INFINITY) s += expf(v[u] - m);
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float om = __shfl_xor_sync(0xffffffffu, m, o), os = __shfl_xor_sync(0xffffffffu, s, o);
      lse_merge(m, s, om, os);
    }
    __syncthreads();   // (s_m / s_s of the previous item have been read)
    if (lane == 0) { s_m[warp] = m; s_s[warp] = s; }
    __syncthreads();
    if (threadIdx.x == 0) {
      float M = -INFINITY, S = 0.f;
      for (int w = 0; w < NW; ++w) lse_merge(M, S, s_m[w], s_s[w]);
      p.part[((size_t)r * WM_SCORE_NSEG + sg) * 2] = M;
      p.part[((size_t)r * WM_SCORE_NSEG + sg) * 2 + 1] = S;
    }
  }

  // last CTA to arrive folds the segment partials of every token row (threadFenceReduction pattern)
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    s_last = (atomicAdd(reinterpret_cast<unsigned int*>(&p.state[2]), 1u) == gridDim.x - 1);
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  for (int r = warp; r < n_lp; r += NW) {   // warp per row, lane = segment, folded in segment order
    float pm = -INFINITY, ps = 0.f;
    if (lane < WM_SCORE_NSEG) {
      pm = __ldcg(p.part + ((size_t)r * WM_SCORE_NSEG + lane) * 2);
      ps = __ldcg(p.part + ((size_t)r * WM_SCORE_NSEG + lane) * 2 + 1);
    }
    const float tok_v = __ldcg(p.part + (size_t)(WM_MAX_T + 1) * WM_SCORE_NSEG * 2 + r);
    float M = -INFINITY, S = 0.f;
    for (int sg = 0; sg < WM_SCORE_NSEG; ++sg)
      lse_merge(M, S, __shfl_sync(0xffffffffu, pm, sg), __shfl_sync(0xffffffffu, ps, sg));
    if (lane == 0) p.lp[L0 + r] = tok_v - (M + logf(S));
  }
  if (threadIdx.x == 0) {
    p.state[0] = it;
    p.state[1] = L;
    p.state[2] = 0;
  }
}

}  // namespace

int dec_score_grid(int n_cta, int K) { return std::min(n_cta, (K + 2) * WM_SCORE_NSEG); }

cudaError_t dec_launch_scores(const ScoreArgs& a, int grid, cudaStream_t s) {
  if (a.tau) {
    if (a.adj) score_iteration_kernel<true, true><<<grid, WM_SCORE_THREADS, 0, s>>>(a);
    else score_iteration_kernel<false, true><<<grid, WM_SCORE_THREADS, 0, s>>>(a);
  } else if (a.adj) score_iteration_kernel<true><<<grid, WM_SCORE_THREADS, 0, s>>>(a);
  else score_iteration_kernel<false><<<grid, WM_SCORE_THREADS, 0, s>>>(a);
  return cudaGetLastError();
}

}  // namespace wm
