// Logits processors of the speculative loop: generate(sequence_bias=..., bad_words_ids=..., no_repeat_ngram_size=...,
// min_length=..., min_new_tokens=...).
//
// One launch before every iteration, enqueued only when processors are on.  The reference calls every processor with
// the sequence at the start of the iteration, for the base row, the head rows and every verify row alike
// (DESIGN.md section 7), and the loop keeps len(input_ids) = st->L fixed from sweep A to the accept stage.  So one dense
// term per iteration reproduces HF's chain for every row of the iteration: processed_logit adds adj[j] to the raw logit
// before the EOS decay and the suppress masks.  With every ban -inf and every bias finite:
//   SequenceBias: scores + bias, bias = single-token biases, then += each multi-token entry (in dict order) whose
//                 prefix ends input_ids                       -> base[j] + the matched values, in table order (fp32)
//   NoBadWords:   the same with -inf                         -> -inf entries of the same tables
//   NoRepeatNGram / MinLength / MinNewTokens: scores[...] = -inf -> adj = -inf
// Each CTA owns a slice of the vocabulary and applies every rule to its slice, so no grid-wide ordering is needed and the
// sums run in table order whatever the grid.
#include <algorithm>

#include "common.cuh"
#include "engine.h"

namespace wm {

namespace {

__global__ void __launch_bounds__(WM_LP_THREADS) logits_proc_kernel(LogitsProcArgs p) {
  __shared__ unsigned char s_hit[WM_LP_MAX_SEQS];
  const DecState* st = p.st;
  if (st->done) return;              // the loop had already ended (uniform across the grid)
  const int L = st->L;
  const int* ids = st->ids;
  const int slice = (p.V + gridDim.x - 1) / gridDim.x;
  const int j0 = blockIdx.x * slice, j1 = min(p.V, j0 + slice);
  for (int j = j0 + threadIdx.x; j < j1; j += WM_LP_THREADS) p.adj[j] = p.base[j];
  // multi-token sequences: does the prefix (all but the last token) end input_ids?  Longer than input_ids: skipped.
  for (int t = threadIdx.x; t < p.n_seq; t += WM_LP_THREADS) {
    const int o = p.seq_off[t], len = p.seq_off[t + 1] - o;
    bool hit = len <= L;
    for (int k = 0; hit && k < len - 1; ++k) hit = ids[L - len + 1 + k] == p.seq_tok[o + k];
    s_hit[t] = hit;
  }
  __syncthreads();
  if (threadIdx.x == 0) {            // one thread adds the matched values in table order (HF's fp32 += in dict order)
    for (int t = 0; t < p.n_seq; ++t) {
      if (!s_hit[t]) continue;
      const int last = p.seq_tok[p.seq_off[t + 1] - 1];
      if (last >= j0 && last < j1) p.adj[last] += p.seq_val[t];
    }
  }
  __syncthreads();
  // no_repeat_ngram_size = n: ban every token that followed the last n - 1 tokens anywhere in input_ids (nothing while
  // L + 1 < n: there is no start i then)
  const int n = p.ngram;
  if (n > 0) {
    for (int i = threadIdx.x; i + n <= L; i += WM_LP_THREADS) {
      bool hit = true;
      for (int k = 0; hit && k < n - 1; ++k) hit = ids[i + k] == ids[L - n + 1 + k];
      const int tok = ids[i + n - 1];
      if (hit && tok >= j0 && tok < j1) p.adj[tok] = -INFINITY;
    }
  }
  if (threadIdx.x == 0 && L < p.eos_min_len) {
    const int eos = st->eos;
    if (eos >= j0 && eos < j1) p.adj[eos] = -INFINITY;
  }
}

}  // namespace

int dec_logits_proc_grid(int n_cta) { return std::max(1, std::min(n_cta, 32)); }

cudaError_t dec_launch_logits_proc(const LogitsProcArgs& a, int grid, cudaStream_t s) {
  logits_proc_kernel<<<grid, WM_LP_THREADS, 0, s>>>(a);
  return cudaGetLastError();
}

}  // namespace wm
