// Polyphase resampler (sm_90a): torchaudio.functional.resample with its defaults (sinc_interp_hann,
// lowpass_filter_width = 6, rolloff = 0.99) for integer rates.
//
// After dividing both rates by their gcd (orig -> new), output sample o = q * new + p is phase p of block q:
//   y[o] = sum_c K[p][c] * xpad[q * orig + c],   c in [0, 2 * width + orig),   xpad = width zeros | x | width + orig zeros
// (torchaudio's conv1d with stride orig), K[p][c] = sinc(pi t) * cos(pi t / 12)^2 * base / orig with
// t = (-p / new + (c - width) / orig) * base clamped to [-6, 6], base = 0.99 * min(orig, new), width = ceil(6 orig / base).
// The table is built on the host in fp64, in torchaudio's order of operations (its kernel for an fp64 waveform),
// and rounded once to fp32.  Outside |t| < 6 every tap rounds to zero in fp32, so each phase keeps only its support:
// ~2 * width + 1 columns of the 2 * width + orig (475 columns per phase at 44.1 kHz -> 16 kHz, at most 34 non-zero).
//
// Kernel: one CTA per T consecutive outputs.  The input span those outputs read is staged in shared memory (zero
// outside the recording: the padding), then every output is one fp32 FMA chain over its phase's taps, in column order.
// Taps live in global memory as [tap][phase], so the consecutive phases of a warp read consecutive words.
#include <algorithm>
#include <cmath>

#include "common.cuh"
#include "engine.h"

namespace wm {

namespace {

constexpr double kLowpassWidth = 6.0;
constexpr double kRolloff = 0.99;
constexpr size_t kStageFloats = 12288;   // 48 KB of staged input per CTA (no shared-memory opt-in needed)
constexpr int kThreads = 256;

int64_t gcd64(int64_t a, int64_t b) {
  while (b) { const int64_t t = a % b; a = b; b = t; }
  return a;
}

}  // namespace

bool resample_build_table(int orig_hz, int new_hz, ResampleTable& t) {
  if (orig_hz <= 0 || new_hz <= 0) return false;
  const int64_t g = gcd64(orig_hz, new_hz);
  const int orig = (int)(orig_hz / g), nw = (int)(new_hz / g);
  if (orig > kResampleMaxRate || nw > kResampleMaxRate) return false;
  t.orig = orig;
  t.nw = nw;
  const double base = (double)std::min(orig, nw) * kRolloff;
  t.width = (int)std::ceil(kLowpassWidth * orig / base);
  const double scale = base / orig;
  const int cols = 2 * t.width + orig;
  std::vector<std::vector<float>> rows((size_t)nw);
  t.lo.assign((size_t)nw, 0);
  t.n.assign((size_t)nw, 0);
  t.max_taps = 0;
  for (int p = 0; p < nw; ++p) {
    // torchaudio's fp64 kernel: t = arange(0, -new, -1) / new + arange(-width, width + orig) / orig, then * base
    const double t0 = (double)(-p) / (double)nw;
    // columns with |t| < 6, widened by two on each side; beyond them t is clamped to +-6 and the tap is 0 in fp32
    const double c_min = t.width + orig * (-kLowpassWidth / base - t0);
    const double c_max = t.width + orig * (kLowpassWidth / base - t0);
    const int c0 = std::max(0, (int)std::floor(c_min) - 2);
    const int c1 = std::min(cols, (int)std::ceil(c_max) + 3);
    std::vector<float> v;
    v.reserve((size_t)std::max(0, c1 - c0));
    for (int c = c0; c < c1; ++c) {
      double x = t0 + (double)(c - t.width) / (double)orig;
      x *= base;
      x = std::min(std::max(x, -kLowpassWidth), kLowpassWidth);
      double w = std::cos(x * M_PI / kLowpassWidth / 2.0);
      w = w * w;
      x *= M_PI;
      double k = (x == 0.0) ? 1.0 : std::sin(x) / x;
      k *= w * scale;
      v.push_back((float)k);
    }
    int a = 0, b = (int)v.size();
    while (a < b && v[a] == 0.0f) ++a;
    while (b > a && v[b - 1] == 0.0f) --b;
    rows[p].assign(v.begin() + a, v.begin() + b);
    t.lo[p] = c0 + a;
    t.n[p] = b - a;
    t.max_taps = std::max(t.max_taps, b - a);
  }
  t.taps.assign((size_t)nw * t.max_taps, 0.0f);
  for (int p = 0; p < nw; ++p) std::copy(rows[p].begin(), rows[p].end(), t.taps.begin() + (size_t)p * t.max_taps);
  // input reach of output o, relative to floor(o * orig / new): [dlo, dhi)
  t.dlo = INT64_MAX;
  t.dhi = INT64_MIN;
  for (int p = 0; p < nw; ++p) {
    const int64_t f = (int64_t)p * orig / nw;
    t.dlo = std::min(t.dlo, (int64_t)t.lo[p] - t.width - f);
    t.dhi = std::max(t.dhi, (int64_t)t.lo[p] + t.n[p] - t.width - f);
  }
  return true;
}

int64_t resample_out_len(int64_t n_in, const ResampleTable& t) {
  // ceil(n_in * new / orig) without overflow for any n_in < 2^62 / new
  return (n_in / t.orig) * t.nw + ((n_in % t.orig) * t.nw + t.orig - 1) / t.orig;
}

int resample_block_outputs(const ResampleTable& t, size_t* smem_bytes) {
  for (int T = 4 * kThreads; T >= 32; T /= 2) {
    const int64_t span = (int64_t)(T - 1) * t.orig / t.nw + 1 + (t.dhi - t.dlo);
    if (span <= (int64_t)kStageFloats) {
      *smem_bytes = (size_t)span * sizeof(float);
      return T;
    }
  }
  return 0;
}

__global__ void __launch_bounds__(kThreads) resample_poly_kernel(const float* __restrict__ x, int64_t n_in,
                                                                  float* __restrict__ y, int64_t n_out,
                                                                  const float* __restrict__ taps,  // [max_taps][nw]
                                                                  const int2* __restrict__ sup,    // [nw] {lo - width, n}
                                                                  int orig, int nw, int T, int64_t dlo, int64_t dhi) {
  extern __shared__ float s_x[];
  const int64_t o0 = (int64_t)blockIdx.x * T;
  const int64_t o1 = min(o0 + (int64_t)T, n_out);
  const int64_t s_lo = o0 * orig / nw + dlo;
  const int64_t s_hi = (o1 - 1) * orig / nw + dhi;
  for (int64_t i = s_lo + threadIdx.x; i < s_hi; i += blockDim.x)
    s_x[i - s_lo] = (i >= 0 && i < n_in) ? x[i] : 0.0f;
  __syncthreads();
  for (int64_t o = o0 + threadIdx.x; o < o1; o += blockDim.x) {
    const int64_t q = o / nw;
    const int p = (int)(o - q * nw);
    const int2 s = sup[p];
    const float* xs = s_x + (q * orig + s.x - s_lo);
    float acc = 0.0f;
    for (int c = 0; c < s.y; ++c) acc = fmaf(__ldg(taps + (size_t)c * nw + p), xs[c], acc);
    y[o] = acc;
  }
}

cudaError_t resample_launch(const float* x, int64_t n_in, float* y, int64_t n_out, const float* taps_dev,
                            const int2* sup_dev, const ResampleTable& t, int T, size_t smem, cudaStream_t s) {
  if (n_out <= 0) return cudaSuccess;
  const int64_t blocks = (n_out + T - 1) / T;
  resample_poly_kernel<<<(unsigned)blocks, kThreads, smem, s>>>(x, n_in, y, n_out, taps_dev, sup_dev, t.orig, t.nw, T,
                                                                t.dlo, t.dhi);
  return cudaGetLastError();
}

}  // namespace wm
