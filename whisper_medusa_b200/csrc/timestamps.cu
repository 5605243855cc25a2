// Token-level timestamps (generate(return_token_timestamps=True)): HF WhisperGenerationMixin._extract_token_timestamps
// on the GPU.
//
// The decode loop captures the raw cross-attention scores of the alignment heads at every position (TsCapture,
// decode.cu ts_capture).  After the loop, for the N rows P .. n-2 of the final sequence:
//   ts_softmax_kernel : each (head, row): softmax over all S encoder frames (the probabilities HF's attention returns)
//   ts_norm_kernel    : each (head, frame < F): mean and std (unbiased=False) over the N rows; normalise in place
//   ts_filter_kernel  : each (row, frame): median of `filter` frames (reflect padding, NaN sorts last as in torch.sort;
//                       skipped when F <= filter / 2), averaged over the heads in list order -> matrix [N][F]
//   ts_dtw_kernel     : one CTA: DTW of -matrix over anti-diagonals, HF's tie rule, 2-bit trace packed by row in
//                       shared memory; the backtrace writes the first frame of every row (the jumps) and the times
//                       f32((double)frame * time_precision), then the last time once more.
// The cost is fp32: for f32 inputs an fp32 add gives the bits of HF's f64 add stored back to f32.
#include <algorithm>

#include "common.cuh"
#include "engine.h"

namespace wm {

namespace {

constexpr int TS_THREADS = 256;
constexpr int TS_STAGE = 17;   // floats per DTW row's staging slice (16 frames, padded against bank conflicts)

__device__ __forceinline__ float block_reduce(float v, bool is_max, float* red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  v = is_max ? warp_max(v) : warp_sum(v);
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float r = is_max ? -INFINITY : 0.f;
  for (int w = 0; w < nw; ++w) r = is_max ? fmaxf(r, red[w]) : r + red[w];
  return r;
}

// grid (N, n_heads): probs[head][i][0..S) = softmax of captured row row0 + i of the head's slot
__global__ void __launch_bounds__(TS_THREADS) ts_softmax_kernel(const float* __restrict__ scores, const int* __restrict__ head_slot,
                                                                int S, int row0, int N, float* __restrict__ probs) {
  __shared__ float red[TS_THREADS / 32];
  const int i = blockIdx.x, hh = blockIdx.y;
  const float* row = scores + ((size_t)head_slot[hh] * WM_TS_ROWS + row0 + i) * S;
  float mx = -INFINITY;
  for (int j = threadIdx.x; j < S; j += blockDim.x) mx = fmaxf(mx, row[j]);
  mx = block_reduce(mx, true, red);
  float sum = 0.f;
  for (int j = threadIdx.x; j < S; j += blockDim.x) sum += expf(row[j] - mx);
  sum = block_reduce(sum, false, red);
  float* out = probs + ((size_t)hh * N + i) * S;
  for (int j = threadIdx.x; j < S; j += blockDim.x) out[j] = expf(row[j] - mx) / sum;
}

// grid (ceil(F / TS_THREADS), n_heads): column statistics over the N rows (fp64 sums), then (p - mean) / std in fp32.
// A column of equal values has std 0 and, with fp64 sums, mean == value: 0 / 0 = NaN.  HF's fp32 torch.mean can land an
// ulp away from the value (e.g. 7 x 0.1f), and then gives +-inf there instead; the two agree when the mean is exact
// (zero columns, N = 1, dyadic values).
__global__ void __launch_bounds__(TS_THREADS) ts_norm_kernel(float* __restrict__ probs, int ldp, int N, int F) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x, hh = blockIdx.y;
  if (j >= F) return;
  float* col = probs + (size_t)hh * N * ldp + j;
  double s = 0.0;
  for (int i = 0; i < N; ++i) s += (double)col[(size_t)i * ldp];
  const double mean = s / N;
  double q = 0.0;
  for (int i = 0; i < N; ++i) {
    const double d = (double)col[(size_t)i * ldp] - mean;
    q += d * d;
  }
  const float mean_f = (float)mean, std_f = (float)sqrt(q / N);
  for (int i = 0; i < N; ++i) col[(size_t)i * ldp] = (col[(size_t)i * ldp] - mean_f) / std_f;
}

// torch.sort order: NaN after every number
__device__ __forceinline__ bool sorts_after(float a, float b) { return (a > b) || (isnan(a) && !isnan(b)); }

// Median of the FW-frame window around j (reflect padding; pad < F, so one reflection suffices).  FW > 0: a compile-time
// width -- the window stays in registers and the median is the element of rank pad in torch.sort's order (ties broken
// by position, so exactly one element has each rank).  FW = 0: any width up to WM_TS_MAX_FILTER, insertion sort in a
// local array.
template <int FW>
__device__ __forceinline__ float window_median(const float* __restrict__ row, int j, int F, int filter) {
  const int pad = filter / 2;
  if constexpr (FW > 0) {
    float w[FW];
#pragma unroll
    for (int k = 0; k < FW; ++k) {
      int x = j - FW / 2 + k;
      if (x < 0) x = -x;
      if (x >= F) x = 2 * (F - 1) - x;
      w[k] = row[x];
    }
    float med = w[0];
#pragma unroll
    for (int k = 0; k < FW; ++k) {
      int rank = 0;
#pragma unroll
      for (int m = 0; m < FW; ++m)
        if (m != k) rank += (sorts_after(w[k], w[m]) || (m < k && !sorts_after(w[m], w[k]))) ? 1 : 0;
      if (rank == FW / 2) med = w[k];
    }
    return med;
  } else {
    float w[WM_TS_MAX_FILTER];
    for (int k = 0; k < filter; ++k) {
      int x = j - pad + k;
      if (x < 0) x = -x;
      if (x >= F) x = 2 * (F - 1) - x;
      const float e = row[x];
      int p = k;
      while (p > 0 && sorts_after(w[p - 1], e)) { w[p] = w[p - 1]; --p; }
      w[p] = e;
    }
    return w[pad];
  }
}

// grid (ceil(F / TS_THREADS), N): matrix[i][j] = mean over the listed heads of the median-filtered normalised weights
template <int FW>
__global__ void __launch_bounds__(TS_THREADS) ts_filter_kernel(const float* __restrict__ probs, int ldp, int n_heads, int N, int F,
                                                               int filter, float* __restrict__ matrix) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x, i = blockIdx.y;
  if (j >= F) return;
  float acc = 0.f;
  for (int hh = 0; hh < n_heads; ++hh) {
    const float* row = probs + ((size_t)hh * N + i) * ldp;
    acc += (F <= filter / 2) ? row[j] : window_median<FW>(row, j, F, filter);
  }
  matrix[(size_t)i * F + j] = acc / (float)n_heads;
}

// One CTA, thread i (0 .. N) owns DTW row i.  Anti-diagonal k holds the cells (i, k - i); three diagonals rotate in
// shared memory and one barrier per diagonal orders them.  Row i - 1 of the matrix is read 16 frames at a time into the
// thread's own staging slice.  trace: 2 bits per cell, row i - 1 in words
// [(i-1) * w16, i * w16), each word written only by its row's thread.
__global__ void ts_dtw_kernel(const float* __restrict__ matrix, int N, int F, double time_precision, int* __restrict__ jumps,
                              float* __restrict__ times) {
  extern __shared__ float smem_f[];
  const int np1 = N + 1;
  float* diag = smem_f;                                                     // [3][N + 1]
  float* stage = smem_f + 3 * np1;                                          // [N + 1][17]
  uint32_t* trace = reinterpret_cast<uint32_t*>(stage + TS_STAGE * np1);    // [N][w16]
  const int w16 = (F + 15) / 16;
  const int i = threadIdx.x;
  const bool active = i <= N;
  if (active) diag[i] = (i == 0) ? 0.f : INFINITY;                          // k = 0: cost[0][0] = 0
  __syncthreads();
  uint32_t word = 0u;
  const float* mrow = matrix + (size_t)(i > 0 ? i - 1 : 0) * F;
  float* my = stage + (size_t)(active ? i : 0) * TS_STAGE;
  // the rows' 16-frame groups start on different diagonals, so a load waited for in its own diagonal would stall every
  // barrier: each group is loaded into registers one group ahead and only stored to the slice when it is due
  float nxt[16];
#pragma unroll
  for (int u = 0; u < 16; ++u) nxt[u] = (active && i > 0 && u < F) ? __ldg(mrow + u) : 0.f;
  for (int k = 1; k <= N + F; ++k) {
    float* cur = diag + (k % 3) * np1;
    const float* prev = diag + ((k - 1) % 3) * np1;
    const float* prev2 = diag + ((k - 2) % 3) * np1;
    const int j = k - i;
    if (active && j >= 0 && j <= F) {
      if (i == 0 || j == 0) {
        cur[i] = INFINITY;
      } else {
        const int q = (j - 1) & 15;
        if (q == 0) {
#pragma unroll
          for (int u = 0; u < 16; ++u) my[u] = nxt[u];
#pragma unroll
          for (int u = 0; u < 16; ++u) nxt[u] = (j + 15 + u < F) ? __ldg(mrow + j + 15 + u) : 0.f;
        }
        const float c0 = prev2[i - 1], c1 = prev[i - 1], c2 = prev[i];
        float c;
        uint32_t t;
        if (c0 < c1 && c0 < c2) { c = c0; t = 0u; }
        else if (c1 < c0 && c1 < c2) { c = c1; t = 1u; }
        else { c = c2; t = 2u; }
        cur[i] = -my[q] + c;
        word |= t << (q * 2);
        if (q == 15 || j == F) {
          trace[(size_t)(i - 1) * w16 + ((j - 1) >> 4)] = word;
          word = 0u;
        }
      }
    }
    __syncthreads();
  }
  if (threadIdx.x != 0) return;
  // backtrace from (N, F) with trace[0][:] = 2 and trace[:][0] = 1 (HF sets them after the sweep).  The last cell of row
  // r the walk visits is the first one going forwards: the jump of text row r - 1.
  int r = N, c = F;
  int last_r = -1, last_c = 0;
  while (r > 0 || c > 0) {
    if (r != last_r && last_r > 0) jumps[last_r - 1] = last_c;
    last_r = r; last_c = c - 1;
    uint32_t t;
    if (r == 0) t = 2u;
    else if (c == 0) t = 1u;
    else t = (trace[(size_t)(r - 1) * w16 + ((c - 1) >> 4)] >> (((c - 1) & 15) * 2)) & 3u;
    if (t == 0u) { --r; --c; }
    else if (t == 1u) --r;
    else --c;
  }
  if (last_r > 0) jumps[last_r - 1] = last_c;
  __threadfence_block();
  for (int q = 0; q < N; ++q) times[q] = (float)((double)jumps[q] * time_precision);
  times[N] = times[N - 1];
}

}  // namespace

size_t ts_dtw_smem_bytes(int N, int F) {
  return (size_t)(3 + TS_STAGE) * (N + 1) * sizeof(float) + (size_t)N * ((F + 15) / 16) * sizeof(uint32_t);
}

cudaError_t ts_launch_softmax(const TsSoftmaxArgs& a, cudaStream_t s) {
  if (a.N <= 0 || a.n_heads <= 0) return cudaSuccess;
  ts_softmax_kernel<<<dim3(a.N, a.n_heads), TS_THREADS, 0, s>>>(a.scores, a.head_slot, a.S, a.row0, a.N, a.probs);
  return cudaGetLastError();
}

cudaError_t ts_launch_extract(const TsExtractArgs& a, cudaStream_t s, int64_t* n_launch) {
  if (a.N <= 0) return cudaSuccess;
  const int gx = std::max(1, (a.F + TS_THREADS - 1) / TS_THREADS);
  if (a.F > 0) {
    ts_norm_kernel<<<dim3(gx, a.n_heads), TS_THREADS, 0, s>>>(a.probs, a.ldp, a.N, a.F);
    if (a.filter == 7)   // HF's default width: the register path
      ts_filter_kernel<7><<<dim3(gx, a.N), TS_THREADS, 0, s>>>(a.probs, a.ldp, a.n_heads, a.N, a.F, a.filter, a.matrix);
    else
      ts_filter_kernel<0><<<dim3(gx, a.N), TS_THREADS, 0, s>>>(a.probs, a.ldp, a.n_heads, a.N, a.F, a.filter, a.matrix);
    if (n_launch) *n_launch += 2;
  }
  const size_t smem = ts_dtw_smem_bytes(a.N, a.F);
  cudaError_t e = cudaFuncSetAttribute(ts_dtw_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  const int threads = (a.N + 1 + 31) / 32 * 32;
  ts_dtw_kernel<<<1, threads, smem, s>>>(a.matrix, a.N, a.F, a.time_precision, a.jumps, a.times);
  if (n_launch) *n_launch += 1;
  return cudaGetLastError();
}

}  // namespace wm
