// Encoder self-attention on the Hopper tensor cores (sm_90a, wgmma): full (non-causal) softmax(Q K^T / 8) V over
// S = 1500 positions, head_dim 64 (HF modeling_whisper.py:284-357).  Same blocking and rounding points as the mma.sync
// kernel (enc_attn.cu: 64-key blocks, online softmax in fp32 with exp2, un-normalised P rounded to fp16 for the P V
// product, fp32 O), so the two agree to fp32 accumulation order and enc_attn.cu stays the cross-check.
//
// One CTA = one head x 128 query rows, two CTAs per SM.
//   warp 8      : TMA producer -- Q tile once, then per key block the K tile [64 keys][64] and the V^T tile
//                 [64 dims][64 keys] (cp.async.bulk.tensor.2d, SWIZZLE_128B) into a 3-stage ring
//   warps 0-7   : two consumer warpgroups of 64 query rows each: S = Q K^T (wgmma m64n64k16 x4, both operands in shared
//                 memory) into registers, online softmax on the accumulator fragments (a row is spread over the 4
//                 threads of a quad), P rounded to fp16 in registers in the A-fragment layout, O += P V^T (wgmma
//                 m64n64k16 x4, A from registers); the ring stage is released once both products have completed
// V^T ([H*64][S_pad] fp16) is written by the QKV GEMM's epilogue or by enc_transpose_v_kernel, so that both products
// use K-major operands.
#include <cuda.h>

#include <map>
#include <tuple>

#include "common.cuh"
#include "engine.h"
#include "tc_common.cuh"

namespace wm {

#define AT_BQ 128
#define AT_BK 64
#define AT_STAGES 3
#define AT_THREADS 288
#define AT_Q_BYTES (AT_BQ * 64 * 2)        // 16 KB
#define AT_KV_BYTES (2 * AT_BK * 64 * 2)   // K tile 8 KB + V^T tile 8 KB per stage

// 2^x on the SFU without the denormal fix-ups of exp2f (the arguments are <= 0; results below 2^-126 flush to zero and
// round to zero in fp16 anyway)
__device__ __forceinline__ float at_ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

__global__ void __launch_bounds__(AT_THREADS, 2)
enc_attn_tc_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_k,
                   const __grid_constant__ CUtensorMap map_vt, __half* __restrict__ out, int S, int d) {
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  __shared__ __align__(8) uint64_t q_full, kv_full[AT_STAGES], kv_empty[AT_STAGES];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int h = blockIdx.y, q0 = blockIdx.x * AT_BQ;
  const int nkb = (S + AT_BK - 1) / AT_BK;
  const uint32_t smem_base = (tc_smem_u32(smem_raw) + 1023u) & ~1023u;   // (1 KB of slack in the allocation)
  const uint32_t sQ = smem_base;
  const uint32_t sKV = smem_base + AT_Q_BYTES;   // stage s: K at +0, V^T at +8 KB

  if (warp == 8 && lane == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_q) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_k) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_vt) : "memory");
    tc_mbar_init(tc_smem_u32(&q_full), 1);
    for (int s = 0; s < AT_STAGES; ++s) { tc_mbar_init(tc_smem_u32(&kv_full[s]), 1); tc_mbar_init(tc_smem_u32(&kv_empty[s]), 8); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  // programmatic dependent launch (tc_common.cuh): everything above overlapped the QKV GEMM's tail; Q, K and V^T are its
  // outputs
  tc_grid_dep_launch();
  tc_grid_dep_wait();

  if (warp == 8) {
    // ===== TMA producer =====
    if (lane == 0) {
      tc_mbar_expect_tx(tc_smem_u32(&q_full), AT_Q_BYTES);
      tc_tma_load_2d(sQ, &map_q, h * 64, q0, tc_smem_u32(&q_full));
      for (int kb = 0; kb < nkb; ++kb) {
        const int s = kb % AT_STAGES;
        const uint32_t ph = (kb / AT_STAGES) & 1;
        tc_mbar_wait(tc_smem_u32(&kv_empty[s]), ph ^ 1);
        const uint32_t full = tc_smem_u32(&kv_full[s]);
        tc_mbar_expect_tx(full, AT_KV_BYTES);
        tc_tma_load_2d(sKV + s * AT_KV_BYTES, &map_k, d + h * 64, kb * AT_BK, full);
        tc_tma_load_2d(sKV + s * AT_KV_BYTES + AT_BK * 64 * 2, &map_vt, kb * AT_BK, h * 64, full);
      }
    }
    return;
  }

  // ===== consumer warpgroup wg: query rows 64 wg .. 64 wg + 63 of the tile.  This thread holds rows r0 = 16 (warp % 4)
  // + lane / 4 and r0 + 8, columns 8 j + 2 (lane % 4) + {0, 1} (j = 0..7) of the S and O fragments
  const int wg = warp >> 2;
  const int cq = 2 * (lane & 3);
  const uint64_t qdesc = tc_smem_desc(sQ + wg * 64 * 128);
  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  const float L2E = 1.4426950408889634f * 0.125f;   // log2(e) * head_dim^-0.5 (q is NOT pre-scaled)
  tc_mbar_wait(tc_smem_u32(&q_full), 0);
  for (int kb = 0; kb < nkb; ++kb) {
    const int s = kb % AT_STAGES;
    tc_mbar_wait(tc_smem_u32(&kv_full[s]), (kb / AT_STAGES) & 1);
    const uint32_t sK = sKV + s * AT_KV_BYTES;
    float sc[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) sc[i] = 0.f;
    wgmma_fence_regs(sc);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) wgmma_ss_n64(sc, qdesc + (uint64_t)(k * 2), tc_smem_desc(sK) + (uint64_t)(k * 2), k > 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(sc);
    const int nvalid = S - kb * AT_BK;   // existing keys of this block (only the last block is partial)
    if (nvalid < AT_BK) {
#pragma unroll
      for (int j = 0; j < 8; ++j)
#pragma unroll
        for (int e = 0; e < 2; ++e)
          if (8 * j + cq + e >= nvalid) { sc[4 * j + e] = -INFINITY; sc[4 * j + 2 + e] = -INFINITY; }
    }
    uint32_t pa[4][4];   // P in the A-fragment layout of the four k16 steps of P V
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      float mx = -INFINITY;
#pragma unroll
      for (int j = 0; j < 8; ++j) mx = fmaxf(mx, fmaxf(sc[4 * j + 2 * hr], sc[4 * j + 2 * hr + 1]));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float m_new = fmaxf(m_run[hr], mx);
      const float alpha = at_ex2((m_run[hr] - m_new) * L2E);   // first block: 2^-inf = 0
      const float msc = m_new * L2E;
      m_run[hr] = m_new;
      float lsum = 0.f;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        // masked keys: 2^-inf = 0
        const float p0 = at_ex2(fmaf(sc[4 * j + 2 * hr], L2E, -msc));
        const float p1 = at_ex2(fmaf(sc[4 * j + 2 * hr + 1], L2E, -msc));
        lsum += p0 + p1;
        pa[j >> 1][(j & 1) * 2 + hr] = pack_half2(p0, p1);
      }
      l_run[hr] = fmaf(l_run[hr], alpha, lsum);
      if (alpha != 1.0f) {   // the running maximum rarely moves after the first blocks
#pragma unroll
        for (int j = 0; j < 8; ++j) { o[4 * j + 2 * hr] *= alpha; o[4 * j + 2 * hr + 1] *= alpha; }
      }
    }
    const uint64_t vdesc = tc_smem_desc(sK + AT_BK * 64 * 2);
    wgmma_fence_regs(o);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) wgmma_rs_n64(o, pa[k], vdesc + (uint64_t)(k * 2), 1u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(o);
    __syncwarp();
    if (lane == 0) tc_mbar_arrive(tc_smem_u32(&kv_empty[s]));   // K(kb) and V^T(kb) are consumed
  }
  // the four threads of a quad summed disjoint columns with the same running maxima: their sums add up
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    l_run[hr] += __shfl_xor_sync(0xffffffffu, l_run[hr], 1);
    l_run[hr] += __shfl_xor_sync(0xffffffffu, l_run[hr], 2);
  }
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    const int row = q0 + wg * 64 + (warp & 3) * 16 + (lane >> 2) + hr * 8;
    if (row < S) {
      const float inv = 1.0f / l_run[hr];
      __half* dst = out + (size_t)row * d + h * 64 + cq;
#pragma unroll
      for (int j = 0; j < 8; ++j)
        *reinterpret_cast<uint32_t*>(dst + 8 * j) = pack_half2(o[4 * j + 2 * hr] * inv, o[4 * j + 2 * hr + 1] * inv);
    }
  }
}

// V of qkv16 [S_pad][3d] (columns 2d ..) -> vT [d][S_pad]  (rows >= S of qkv16 are zero: never written)
__global__ void __launch_bounds__(256) enc_transpose_v_kernel(const __half* __restrict__ qkv, __half* __restrict__ vt, int S_pad, int d) {
  __shared__ __half tile[64][66];
  const int p0 = blockIdx.x * 64, c0 = blockIdx.y * 64;
  for (int i = threadIdx.x; i < 64 * 32; i += 256) {
    const int r = i >> 5, c2 = (i & 31) * 2;
    const __half2 v = *reinterpret_cast<const __half2*>(qkv + (size_t)(p0 + r) * 3 * d + 2 * d + c0 + c2);
    tile[r][c2] = __low2half(v);
    tile[r][c2 + 1] = __high2half(v);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 64 * 32; i += 256) {
    const int c = i >> 5, r2 = (i & 31) * 2;
    *reinterpret_cast<__half2*>(vt + (size_t)(c0 + c) * S_pad + p0 + r2) = __halves2half2(tile[r2][c], tile[r2 + 1][c]);
  }
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
typedef CUresult (*AtEncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                    const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static AtEncodeTiledFn at_encode_fn() {
  static AtEncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<AtEncodeTiledFn>(p);
  }
  return fn;
}
static bool at_make_map(CUtensorMap* map, const __half* base, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows) {
  AtEncodeTiledFn fn = at_encode_fn();
  if (!fn) return false;
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {ld * sizeof(__half)};
  cuuint32_t box[2] = {64, box_rows};
  cuuint32_t estr[2] = {1, 1};
  return fn(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<__half*>(base), dims, strides, box, estr,
            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

static const size_t kAtSmem = (size_t)AT_Q_BYTES + (size_t)AT_STAGES * AT_KV_BYTES + 1024;

cudaError_t enc_attention_tc_configure() {
  cudaError_t e = cudaFuncSetAttribute(enc_attn_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kAtSmem);
  if (e != cudaSuccess) return e;
  return at_encode_fn() ? cudaSuccess : cudaErrorNotSupported;
}

// qkv: [S_pad][3d] fp16 (q | k | v), vt: scratch [d][S_pad] fp16, out: [S_pad][d] fp16
cudaError_t enc_attention_tc(const __half* qkv, __half* vt, __half* out, int S, int S_pad, int d, int H, bool vt_ready,
                             cudaStream_t s, int64_t* n_launch, bool pdl) {
  typedef std::tuple<const void*, const void*, int, int> Key;
  struct Maps { CUtensorMap q, k, vt; };
  static thread_local std::map<Key, Maps> cache;
  Key key(qkv, vt, S_pad, d);
  auto it = cache.find(key);
  if (it == cache.end()) {
    Maps m;
    if (!at_make_map(&m.q, qkv, (uint64_t)S_pad, (uint64_t)3 * d, (uint64_t)3 * d, AT_BQ)) return cudaErrorInvalidValue;
    if (!at_make_map(&m.k, qkv, (uint64_t)S_pad, (uint64_t)3 * d, (uint64_t)3 * d, AT_BK)) return cudaErrorInvalidValue;
    if (!at_make_map(&m.vt, vt, (uint64_t)d, (uint64_t)S_pad, (uint64_t)S_pad, 64)) return cudaErrorInvalidValue;
    it = cache.emplace(key, m).first;
  }
  if (!vt_ready) {
    enc_transpose_v_kernel<<<dim3(S_pad / 64, d / 64), 256, 0, s>>>(qkv, vt, S_pad, d);
    if (n_launch) ++*n_launch;
  }
  dim3 grid((S + AT_BQ - 1) / AT_BQ, H);
  cudaError_t e = tc_launch(enc_attn_tc_kernel, grid, dim3(AT_THREADS), kAtSmem, s, pdl && vt_ready, it->second.q, it->second.k,
                            it->second.vt, out, S, d);
  if (e != cudaSuccess) return e;
  if (n_launch) ++*n_launch;
  return cudaGetLastError();
}

}  // namespace wm
