// Log-mel frontend (sm_90a): framing -> hann -> 400-point real DFT -> power -> slaney mel ->
// log10 -> global max floor -> (x+4)/4.  Follows HF feature_extraction_whisper.py:135-164
// (_torch_extract_fbank_features): torch.stft(n_fft=400, hop=160, hann, center=True, reflect),
// |.|^2, drop the last frame, mel_filters.T @ magnitudes, clamp(1e-10).log10(), max(x, max-8), (x+4)/4.
//
// The 400-point DFT is evaluated directly (201 bins x 400 taps per frame, fp32) from a
// shared-memory twiddle table: ~0.5 GFMA per 30 s clip, far below anything that matters next to
// the encoder.  Two launches: (1) per-frame log-mel + global max via an order-preserving integer
// atomicMax (deterministic), (2) floor/scale + fp16 time-major copy for the conv stem.
#include "common.cuh"
#include "engine.h"

namespace wm {

#define MEL_NFFT 400
#define MEL_HOP 160
#define MEL_NFREQ 201
#define MEL_NMEL 80
#define MEL_FRAMES 3000
#define MEL_NSAMP 480000
#define MEL_FR 4  // frames per CTA

__device__ __forceinline__ int float_key(float v) {
  int b = __float_as_int(v);
  return b >= 0 ? b : (b ^ 0x7fffffff);
}
__device__ __forceinline__ float key_float(int k) {
  return __int_as_float(k >= 0 ? k : (k ^ 0x7fffffff));
}

__global__ void __launch_bounds__(256) mel_power_kernel(const float* __restrict__ pcm, const float* __restrict__ fb,
                                                        float* __restrict__ logspec, int* __restrict__ gmax_bits) {
  __shared__ float s_cos[MEL_NFFT], s_sin[MEL_NFFT];
  __shared__ float s_x[MEL_FR][MEL_NFFT];
  __shared__ float s_pw[MEL_FR][MEL_NFREQ + 3];
  __shared__ int s_max;
  const int tid = threadIdx.x;
  const int f0 = blockIdx.x * MEL_FR;
  if (tid == 0) s_max = float_key(-INFINITY);
  for (int k = tid; k < MEL_NFFT; k += blockDim.x) {
    float s, c;
    sincospif((float)k / 200.0f, &s, &c);  // angle 2*pi*k/400
    s_cos[k] = c;
    s_sin[k] = s;
  }
  __syncthreads();
  for (int idx = tid; idx < MEL_FR * MEL_NFFT; idx += blockDim.x) {
    const int fi = idx / MEL_NFFT, j = idx - fi * MEL_NFFT;
    int i = (f0 + fi) * MEL_HOP + j - MEL_NFFT / 2;
    if (i < 0) i = -i;                                   // reflect padding (center=True)
    if (i >= MEL_NSAMP) i = 2 * (MEL_NSAMP - 1) - i;
    const float w = 0.5f - 0.5f * s_cos[j];              // periodic hann(400)
    s_x[fi][j] = pcm[i] * w;
  }
  __syncthreads();
  for (int idx = tid; idx < MEL_FR * MEL_NFREQ; idx += blockDim.x) {
    const int fi = idx / MEL_NFREQ, k = idx - fi * MEL_NFREQ;
    float re = 0.f, im = 0.f;
    int ph = 0;
#pragma unroll 8
    for (int j = 0; j < MEL_NFFT; ++j) {
      const float x = s_x[fi][j];
      re = fmaf(x, s_cos[ph], re);
      im = fmaf(x, s_sin[ph], im);
      ph += k;
      if (ph >= MEL_NFFT) ph -= MEL_NFFT;
    }
    s_pw[fi][k] = re * re + im * im;
  }
  __syncthreads();
  for (int idx = tid; idx < MEL_FR * MEL_NMEL; idx += blockDim.x) {
    const int fi = idx / MEL_NMEL, mI = idx - fi * MEL_NMEL;
    float acc = 0.f;
    for (int k = 0; k < MEL_NFREQ; ++k) acc = fmaf(fb[k * MEL_NMEL + mI], s_pw[fi][k], acc);
    const float lv = log10f(fmaxf(acc, 1e-10f));
    logspec[(size_t)mI * MEL_FRAMES + f0 + fi] = lv;
    atomicMax(&s_max, float_key(lv));
  }
  __syncthreads();
  if (tid == 0) atomicMax(gmax_bits, s_max);
}

__global__ void mel_init_kernel(int* gmax_bits) { *gmax_bits = float_key(-INFINITY); }

// floor at max-8, scale, and write the fp16 time-major copy (row r+1 = frame r; row 0 stays zero)
__global__ void mel_finalize_kernel(float* __restrict__ mel, __half* __restrict__ x_tm, const int* __restrict__ gmax_bits,
                                    int apply_floor) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= MEL_NMEL * MEL_FRAMES) return;
  const int mI = idx / MEL_FRAMES, f = idx - mI * MEL_FRAMES;
  float v = mel[idx];
  if (apply_floor) {
    const float gmax = key_float(*gmax_bits);
    v = fmaxf(v, gmax - 8.0f);
    v = (v + 4.0f) / 4.0f;
    mel[idx] = v;
  }
  x_tm[(size_t)(f + 1) * MEL_NMEL + mI] = __float2half_rn(v);
}

cudaError_t mel_forward(const float* pcm, const float* filters, float* mel_f32, __half* x_tm, int* gmax_bits,
                        cudaStream_t s, int64_t* n_launch) {
  mel_init_kernel<<<1, 1, 0, s>>>(gmax_bits);
  mel_power_kernel<<<MEL_FRAMES / MEL_FR, 256, 0, s>>>(pcm, filters, mel_f32, gmax_bits);
  const int n = MEL_NMEL * MEL_FRAMES;
  mel_finalize_kernel<<<(n + 255) / 256, 256, 0, s>>>(mel_f32, x_tm, gmax_bits, 1);
  if (n_launch) *n_launch += 3;
  return cudaGetLastError();
}

cudaError_t mel_to_time_major(const float* mel_f32, __half* x_tm, cudaStream_t s, int64_t* n_launch) {
  const int n = MEL_NMEL * MEL_FRAMES;
  mel_finalize_kernel<<<(n + 255) / 256, 256, 0, s>>>(const_cast<float*>(mel_f32), x_tm, nullptr, 0);
  if (n_launch) *n_launch += 1;
  return cudaGetLastError();
}

}  // namespace wm
