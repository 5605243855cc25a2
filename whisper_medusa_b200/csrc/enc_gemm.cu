// Encoder-side dense GEMM  C[M,N] = A[M,K] * W[N,K]^T  (fp16 operands, fp32 accumulate) with fused
// epilogues, plus the row LayerNorm.  Used for: conv1/conv2 as implicit GEMMs over a time-major
// activation (HF modeling_whisper.py:619-625), the encoder layer projections and FFN (:392-408)
// and the cross-attention K/V projection of every decoder layer (:325-336).
//
// This file is the mma.sync (m16n8k16) implementation: 128x128x32 CTA tile, 8 warps (2x4), 4-stage
// cp.async pipeline, XOR-swizzled shared memory read with ldmatrix.  The wgmma/TMA version in
// enc_gemm_tc.cu replaces it on the hot path; this one is its cross-check.
#include "common.cuh"
#include "engine.h"
#include "tc_common.cuh"

namespace wm {

#define EG_BM 128
#define EG_BN 128
#define EG_BK 32
#define EG_STAGES 4
#define EG_THREADS 256

// smem tile: rows of 32 halfs (64 B) = 4 chunks of 16 B; physical chunk = c ^ ((row >> 1) & 3)
__device__ __forceinline__ int eg_swz(int row, int chunk) { return row * 32 + ((chunk ^ ((row >> 1) & 3)) << 3); }

template <int EPI>
__global__ void __launch_bounds__(EG_THREADS) enc_gemm_kernel(EncGemmArgs a) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  __half* sA = reinterpret_cast<__half*>(smem_raw);                  // [STAGES][128*32]
  __half* sB = sA + EG_STAGES * EG_BM * EG_BK;                        // [STAGES][128*32]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int wm_ = warp >> 2, wn_ = warp & 3;                          // 2 x 4 warps
  const int m0 = blockIdx.y * EG_BM, n0 = blockIdx.x * EG_BN;
  const int KT = a.K / EG_BK;

  auto load_stage = [&](int stage, int kt) {
    const __half* Ag = a.A + (size_t)m0 * a.lda + (size_t)kt * EG_BK;
    const __half* Wg = a.W + (size_t)n0 * a.K + (size_t)kt * EG_BK;
    __half* dA = sA + stage * EG_BM * EG_BK;
    __half* dB = sB + stage * EG_BN * EG_BK;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int c = tid + i * EG_THREADS;      // 512 chunks per operand
      const int row = c >> 2, ch = c & 3;
      cp_async16(dA + eg_swz(row, ch), Ag + (size_t)row * a.lda + ch * 8);
      cp_async16(dB + eg_swz(row, ch), Wg + (size_t)row * a.K + ch * 8);
    }
  };

  float acc[4][4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[i][j][e] = 0.f;

#pragma unroll
  for (int s = 0; s < EG_STAGES - 1; ++s) {
    if (s < KT) load_stage(s, s);
    cp_async_commit();
  }

  for (int kt = 0; kt < KT; ++kt) {
    cp_async_wait<EG_STAGES - 2>();
    __syncthreads();
    {
      const int nk = kt + EG_STAGES - 1;
      if (nk < KT) load_stage(nk % EG_STAGES, nk);
      cp_async_commit();
    }
    const __half* tA = sA + (kt % EG_STAGES) * EG_BM * EG_BK;
    const __half* tB = sB + (kt % EG_STAGES) * EG_BN * EG_BK;
#pragma unroll
    for (int k16 = 0; k16 < 2; ++k16) {
      uint32_t af[4][4], bf[4][2];
#pragma unroll
      for (int mi = 0; mi < 4; ++mi) {
        const int row = wm_ * 64 + mi * 16 + (lane & 7) + ((lane >> 3) & 1) * 8;
        const int ch = k16 * 2 + (lane >> 4);
        ldmatrix_x4(af[mi][0], af[mi][1], af[mi][2], af[mi][3], tA + eg_swz(row, ch));
      }
#pragma unroll
      for (int np = 0; np < 2; ++np) {
        const int row = wn_ * 32 + np * 16 + (lane & 7) + ((lane >> 4) << 3);
        const int ch = k16 * 2 + ((lane >> 3) & 1);
        ldmatrix_x4(bf[np * 2][0], bf[np * 2][1], bf[np * 2 + 1][0], bf[np * 2 + 1][1], tB + eg_swz(row, ch));
      }
#pragma unroll
      for (int mi = 0; mi < 4; ++mi)
#pragma unroll
        for (int ni = 0; ni < 4; ++ni)
          mma_16816(acc[mi][ni], af[mi][0], af[mi][1], af[mi][2], af[mi][3], bf[ni][0], bf[ni][1]);
    }
  }
  cp_async_wait<0>();

  // ---- epilogue ----
  const int g = lane >> 2, t = lane & 3;
#pragma unroll
  for (int mi = 0; mi < 4; ++mi) {
#pragma unroll
    for (int half_ = 0; half_ < 2; ++half_) {
      const int row = m0 + wm_ * 64 + mi * 16 + g + half_ * 8;
      if (row >= a.M) continue;
#pragma unroll
      for (int ni = 0; ni < 4; ++ni) {
        const int col = n0 + wn_ * 32 + ni * 8 + 2 * t;
        float v0 = acc[mi][ni][half_ * 2 + 0] + a.bias[col];
        float v1 = acc[mi][ni][half_ * 2 + 1] + a.bias[col + 1];
        if (EPI == ENC_EPI_BIAS_F16) {
          *reinterpret_cast<__half2*>(a.out16 + (size_t)row * a.ldo16 + col) = __floats2half2_rn(v0, v1);
        } else if (EPI == ENC_EPI_BIAS_GELU_F16) {
          *reinterpret_cast<__half2*>(a.out16 + (size_t)row * a.ldo16 + col) =
              __floats2half2_rn(gelu_erf(v0), gelu_erf(v1));
        } else if (EPI == ENC_EPI_BIAS_RES_F32) {
          float2* p = reinterpret_cast<float2*>(a.out32 + (size_t)row * a.ldo32 + col);
          float2 o = *p;
          o.x += v0; o.y += v1;
          *p = o;
        } else {  // ENC_EPI_BIAS_GELU_POS_F32
          const float2 pz = *reinterpret_cast<const float2*>(a.pos + (size_t)row * a.N + col);
          float2 o;
          o.x = gelu_erf(v0) + pz.x;
          o.y = gelu_erf(v1) + pz.y;
          *reinterpret_cast<float2*>(a.out32 + (size_t)row * a.ldo32 + col) = o;
        }
      }
    }
  }
}

static const size_t kEgSmem = (size_t)2 * EG_STAGES * EG_BM * EG_BK * sizeof(__half);

cudaError_t enc_gemm_configure() {
  cudaError_t e;
#define WM_SET(EPI)                                                                                            \
  e = cudaFuncSetAttribute(enc_gemm_kernel<EPI>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kEgSmem); \
  if (e != cudaSuccess) return e;
  WM_SET(ENC_EPI_BIAS_F16)
  WM_SET(ENC_EPI_BIAS_GELU_F16)
  WM_SET(ENC_EPI_BIAS_RES_F32)
  WM_SET(ENC_EPI_BIAS_GELU_POS_F32)
#undef WM_SET
  return cudaSuccess;
}

cudaError_t enc_gemm(const EncGemmArgs& a, cudaStream_t s, int64_t* n_launch) {
  if (a.N % EG_BN != 0 || a.K % EG_BK != 0 || (a.lda % 8) != 0) return cudaErrorInvalidValue;
  dim3 grid(a.N / EG_BN, (a.M + EG_BM - 1) / EG_BM);
  switch (a.epi) {
    case ENC_EPI_BIAS_F16: enc_gemm_kernel<ENC_EPI_BIAS_F16><<<grid, EG_THREADS, kEgSmem, s>>>(a); break;
    case ENC_EPI_BIAS_GELU_F16: enc_gemm_kernel<ENC_EPI_BIAS_GELU_F16><<<grid, EG_THREADS, kEgSmem, s>>>(a); break;
    case ENC_EPI_BIAS_RES_F32: enc_gemm_kernel<ENC_EPI_BIAS_RES_F32><<<grid, EG_THREADS, kEgSmem, s>>>(a); break;
    case ENC_EPI_BIAS_GELU_POS_F32: enc_gemm_kernel<ENC_EPI_BIAS_GELU_POS_F32><<<grid, EG_THREADS, kEgSmem, s>>>(a); break;
    default: return cudaErrorInvalidValue;
  }
  if (n_launch) ++*n_launch;
  return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------
// LayerNorm (eps 1e-5, biased variance): one warp per row; writes the fp16 GEMM operand
// ---------------------------------------------------------------------------------------------
// The row (d <= 1280, a multiple of 128) is read ONCE with 16-byte loads and kept in registers for the two-pass
// statistics and the normalisation; outputs are written as 8-byte (fp16) / 16-byte (fp32) vectors.
__global__ void __launch_bounds__(256) enc_layernorm_kernel(const float* __restrict__ x, const float* __restrict__ g,
                                                            const float* __restrict__ b, __half* __restrict__ y16,
                                                            float* __restrict__ y32, int M, int d) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  tc_grid_dep_launch();                        // (programmatic dependent launch, tc_common.cuh)
  tc_grid_dep_wait();                          // x is the predecessor's output
  if (row >= M) return;
  const int nv = d >> 7;                       // float4 per lane
  const float4* xr = reinterpret_cast<const float4*>(x + (size_t)row * d) + lane;
  float4 v[10];
#pragma unroll
  for (int i = 0; i < 10; ++i)
    if (i < nv) v[i] = xr[i * 32];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < 10; ++i)
    if (i < nv) s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
  const float mean = warp_sum(s) / (float)d;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < 10; ++i)
    if (i < nv) {
      const float a0 = v[i].x - mean, a1 = v[i].y - mean, a2 = v[i].z - mean, a3 = v[i].w - mean;
      q += (a0 * a0 + a1 * a1) + (a2 * a2 + a3 * a3);
    }
  const float rstd = rsqrtf(warp_sum(q) / (float)d + 1e-5f);
  const float4* g4 = reinterpret_cast<const float4*>(g) + lane;
  const float4* b4 = reinterpret_cast<const float4*>(b) + lane;
  uint2* o16 = reinterpret_cast<uint2*>(y16 + (size_t)row * d) + lane;
  float4* o32 = y32 ? reinterpret_cast<float4*>(y32 + (size_t)row * d) + lane : nullptr;
#pragma unroll
  for (int i = 0; i < 10; ++i)
    if (i < nv) {
      const float4 gg = g4[i * 32], bb = b4[i * 32];
      float4 y;
      y.x = (v[i].x - mean) * rstd * gg.x + bb.x;
      y.y = (v[i].y - mean) * rstd * gg.y + bb.y;
      y.z = (v[i].z - mean) * rstd * gg.z + bb.z;
      y.w = (v[i].w - mean) * rstd * gg.w + bb.w;
      o16[i * 32] = make_uint2(pack_half2(y.x, y.y), pack_half2(y.z, y.w));
      if (o32) o32[i * 32] = y;
    }
}

cudaError_t enc_layernorm(const float* x, const float* g, const float* b, __half* y16, float* y32, int M, int d,
                          cudaStream_t s, int64_t* n_launch, bool pdl) {
  const int wpb = 8;
  cudaError_t e = tc_launch(enc_layernorm_kernel, dim3((M + wpb - 1) / wpb), dim3(wpb * 32), 0, s, pdl, x, g, b, y16, y32, M, d);
  if (e != cudaSuccess) return e;
  if (n_launch) ++*n_launch;
  return cudaGetLastError();
}

}  // namespace wm
