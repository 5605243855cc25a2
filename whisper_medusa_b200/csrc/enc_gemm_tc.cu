// Encoder-side dense GEMM on the Hopper tensor cores (sm_90a, wgmma):
//   C[M,N] = A[M,K] * W[N,K]^T   fp16 operands (both K-major), fp32 accumulation in registers.
//
// Structure: one BM x BN output tile per CTA, K swept in 64-column blocks.  At M = 1500 a GEMM has few tiles per SM,
// so the host picks, per GEMM, the tile shape with the fewest operand bytes on the busiest SM (see pick_tile):
//   128 x 128, 6-stage ring, one CTA per SM: outputs of <= 1536 columns and the fp32 read-modify-write epilogues;
//   128 x 128, 3-stage ring, two CTAs per SM (one tile's epilogue overlaps the other's main loop): other narrow tiles;
//   256 x 128, 128 x 192: wide fp16 outputs, one CTA per SM, fewer rounds of tiles over the SMs.
//   warp 8    : TMA producer -- cp.async.bulk.tensor.2d (SWIZZLE_128B) of the A and W tiles into a shared-memory ring,
//                               completion on `full` mbarriers
//   warps 0-7 : two consumer warpgroups, each owning BM / 2 rows of the tile: wgmma.mma_async m64nBNk16 (A and W from
//               shared memory) x4 per stage and 64-row slice, one wgmma group kept in flight; a stage is released
//               (`empty`) once the group that read it has completed.  Epilogue: accumulators + bias -> the idle ring as
//               an fp32 tile -> GELU / residual / positions applied while the tile is copied out row-contiguously.
// The A operand may be an "implicit im2col" view: conv1/conv2 read a time-major activation whose
// GEMM rows overlap (row stride 80 resp. 2d elements) -- the TMA tensor map simply carries that
// stride, no im2col buffer exists.
#include <cuda.h>

#include <cstring>
#include <map>
#include <tuple>

#include "common.cuh"
#include "engine.h"
#include "tc_common.cuh"

namespace wm {

#define TC_BM 128
#define TC_BN 128
#define TC_BK 64
#define TC_THREADS 288   /* two consumer warpgroups + one TMA warp */
__host__ __device__ constexpr int tc_stage_bytes(int bm, int bn) { return (bm + bn) * TC_BK * 2; }
__host__ __device__ constexpr int tc_stage_ld(int bn) { return bn + 8; }   // fp32 epilogue tile row stride (floats)

struct TcArgs {
  int M, N, K;
  int epi;
  const float* bias;
  __half* out16; int ldo16;
  float* out32; int ldo32;
  const float* pos;
  __half* vt; int vt_col0, vt_ld;   // columns >= vt_col0 are ALSO written transposed: vt[col - vt_col0][row] (null: off)
  __half* ck; __half* cv; int kv_spad;   // non-null: the output [pos][k | v] goes to the decode layout [head][kv_spad][72]
};

template <int BN>
__device__ __forceinline__ void tc_wgmma(float (&d)[BN / 2], uint64_t adesc, uint64_t bdesc, uint32_t acc) {
  static_assert(BN == 128 || BN == 192, "tile widths of WM_TC_ALL");
  if constexpr (BN == 128) wgmma_ss_n128(d, adesc, bdesc, acc);
  else wgmma_ss_n192(d, adesc, bdesc, acc);
}

template <int EPI, int BM, int BN, int STAGES>
__global__ void __launch_bounds__(TC_THREADS, (BM == 128 && BN == 128 && STAGES == 3) ? 2 : 1)
enc_gemm_tc_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_w, TcArgs a) {
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  // stage s: A tile [BM rows][64 halfs] at s * STAGE_BYTES, W tile [BN rows][64 halfs] behind it (both 1024-B aligned, SW128)
  constexpr int STAGE_BYTES = tc_stage_bytes(BM, BN);
  constexpr int A_BYTES = BM * TC_BK * 2;
  constexpr int MI = BM / 128;            // 64-row slices per consumer warpgroup
  constexpr int LD = tc_stage_ld(BN);
  static_assert(BM * LD * 4 <= STAGES * STAGE_BYTES, "the fp32 epilogue tile must fit in the ring");
  __shared__ __align__(8) uint64_t s_full[STAGES], s_empty[STAGES];
  __shared__ __align__(16) float s_bias[BN];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
  const int KT = a.K / TC_BK;
  // 1024-B aligned base (the dynamic allocation carries 1 KB of slack)
  const uint32_t smem_base = (tc_smem_u32(smem_raw) + 1023u) & ~1023u;
  unsigned char* const smem = smem_raw + (smem_base - tc_smem_u32(smem_raw));

  if (warp == 8 && lane == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_a) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_w) : "memory");
    for (int s = 0; s < STAGES; ++s) {
      tc_mbar_init(tc_smem_u32(&s_full[s]), 1);
      tc_mbar_init(tc_smem_u32(&s_empty[s]), 8);   // lane 0 of every consumer warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  tc_grid_dep_launch();

  if (warp == 8) {
    // ===== TMA producer =====
    if (lane == 0) {
      // the weight tiles of the first ring round do not depend on the predecessor kernel: they are requested before the
      // grid-dependency wait (programmatic dependent launch, tc_common.cuh), the activation tiles after it
      const int pre = KT < STAGES ? KT : STAGES;
      for (int kt = 0; kt < pre; ++kt) {
        const uint32_t full = tc_smem_u32(&s_full[kt]);
        tc_mbar_expect_tx(full, STAGE_BYTES);
        tc_tma_load_2d(smem_base + kt * STAGE_BYTES + A_BYTES, &map_w, kt * TC_BK, n0, full);
      }
      tc_grid_dep_wait();
      for (int kt = 0; kt < pre; ++kt)
        tc_tma_load_2d(smem_base + kt * STAGE_BYTES, &map_a, kt * TC_BK, m0, tc_smem_u32(&s_full[kt]));
      for (int kt = pre; kt < KT; ++kt) {
        const int s = kt % STAGES;
        const uint32_t ph = (kt / STAGES) & 1;
        tc_mbar_wait(tc_smem_u32(&s_empty[s]), ph ^ 1);
        const uint32_t full = tc_smem_u32(&s_full[s]);
        tc_mbar_expect_tx(full, STAGE_BYTES);
        tc_tma_load_2d(smem_base + s * STAGE_BYTES, &map_a, kt * TC_BK, m0, full);
        tc_tma_load_2d(smem_base + s * STAGE_BYTES + A_BYTES, &map_w, kt * TC_BK, n0, full);
      }
    }
    return;
  }

  // ===== consumer warpgroups =====
  const int wg = warp >> 2;                  // rows [wg * BM / 2, (wg + 1) * BM / 2) of the tile
  const int tid = threadIdx.x;               // 0 .. 255
  for (int i = tid; i < BN; i += 256) s_bias[i] = a.bias[n0 + i];
  float acc[MI][BN / 2];
#pragma unroll
  for (int i = 0; i < MI; ++i)
#pragma unroll
    for (int j = 0; j < BN / 2; ++j) acc[i][j] = 0.f;
  for (int kt = 0; kt < KT; ++kt) {
    const int s = kt % STAGES;
    tc_mbar_wait(tc_smem_u32(&s_full[s]), (kt / STAGES) & 1);
    const uint64_t adesc = tc_smem_desc(smem_base + s * STAGE_BYTES + wg * (BM / 2) * 128);
    const uint64_t bdesc = tc_smem_desc(smem_base + s * STAGE_BYTES + A_BYTES);
#pragma unroll
    for (int i = 0; i < MI; ++i) wgmma_fence_regs(acc[i]);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < TC_BK / 16; ++k)
#pragma unroll
      for (int i = 0; i < MI; ++i)
        tc_wgmma<BN>(acc[i], adesc + (uint64_t)(i * 512 + k * 2), bdesc + (uint64_t)(k * 2), (kt > 0 || k > 0) ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<1>();   // the group of stage kt - 1 has completed: its ring slot may be refilled
#pragma unroll
    for (int i = 0; i < MI; ++i) wgmma_fence_regs(acc[i]);
    if (kt > 0 && lane == 0) tc_mbar_arrive(tc_smem_u32(&s_empty[(kt - 1) % STAGES]));
  }
  wgmma_wait<0>();
#pragma unroll
  for (int i = 0; i < MI; ++i) wgmma_fence_regs(acc[i]);
  tc_grid_dep_wait();   // (the epilogue reads and writes activations)
  // every consumer is done with the ring (and s_bias is complete): the ring becomes the fp32 tile [BM][LD]
  asm volatile("bar.sync 1, 256;" ::: "memory");
  float* const tile = reinterpret_cast<float*>(smem);
  {
    const int r_w = wg * (BM / 2) + (warp & 3) * 16 + (lane >> 2), c_q = 2 * (lane & 3);
#pragma unroll
    for (int i = 0; i < MI; ++i)
#pragma unroll
      for (int j = 0; j < BN / 8; ++j)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int r = r_w + i * 64 + h * 8, c = j * 8 + c_q;
          *reinterpret_cast<float2*>(tile + r * LD + c) =
              make_float2(acc[i][4 * j + 2 * h] + s_bias[c], acc[i][4 * j + 2 * h + 1] + s_bias[c + 1]);
        }
  }
  asm volatile("bar.sync 1, 256;" ::: "memory");
  constexpr bool F32_OUT = (EPI == ENC_EPI_BIAS_RES_F32 || EPI == ENC_EPI_BIAS_GELU_POS_F32);
  if constexpr (!F32_OUT) {
    // 8 consecutive columns of one row per thread: one 16-byte store
    for (int it = tid; it < BM * (BN / 8); it += 256) {
      const int r = it / (BN / 8), c = (it % (BN / 8)) * 8;
      const int row = m0 + r, col = n0 + c;
      if (row >= a.M) continue;
      const float4 x0 = *reinterpret_cast<const float4*>(tile + r * LD + c);
      const float4 x1 = *reinterpret_cast<const float4*>(tile + r * LD + c + 4);
      float x[8] = {x0.x, x0.y, x0.z, x0.w, x1.x, x1.y, x1.z, x1.w};
      if (EPI == ENC_EPI_BIAS_GELU_F16) {
#pragma unroll
        for (int e = 0; e < 8; ++e) x[e] = gelu_erf(x[e]);
      }
      __half* dst = a.out16 + (size_t)row * a.ldo16 + col;
      if (EPI == ENC_EPI_BIAS_F16 && a.ck != nullptr) {
        // cross-attention K/V straight into the layout the decode kernels read: [head][position][64 dims + 8 pad]
        // (pad halfs and positions >= M stay zero from the allocation)
        const int dm = a.N >> 1;
        const int cc = col >= dm ? col - dm : col;
        dst = (col >= dm ? a.cv : a.ck) + ((size_t)(cc >> 6) * a.kv_spad + row) * 72 + (cc & 63);
      }
      *reinterpret_cast<uint4*>(dst) = make_uint4(pack_half2(x[0], x[1]), pack_half2(x[2], x[3]), pack_half2(x[4], x[5]),
                                                  pack_half2(x[6], x[7]));
    }
    if (EPI == ENC_EPI_BIAS_F16 && a.vt != nullptr && n0 + BN > a.vt_col0) {
      // V^T for the attention kernel: two consecutive positions of one column per thread, so a warp writes 128
      // contiguous bytes of a V^T row
      for (int it = tid; it < BN * (BM / 2); it += 256) {
        const int c = it / (BM / 2), r = (it % (BM / 2)) * 2;
        const int row = m0 + r, col = n0 + c;
        if (col < a.vt_col0 || row >= a.M) continue;
        __half* vdst = a.vt + (size_t)(col - a.vt_col0) * a.vt_ld + row;
        const __half2 hh = __floats2half2_rn(tile[r * LD + c], tile[(r + 1) * LD + c]);
        if (row + 1 < a.M) *reinterpret_cast<__half2*>(vdst) = hh;
        else vdst[0] = __low2half(hh);
      }
    }
  } else {
    // fp32 read-modify-write epilogues (residual stream / conv2 + positions): 4 consecutive columns per thread
    for (int it = tid; it < BM * (BN / 4); it += 256) {
      const int r = it / (BN / 4), c = (it % (BN / 4)) * 4;
      const int row = m0 + r, col = n0 + c;
      if (row >= a.M) continue;
      const float4 x = *reinterpret_cast<const float4*>(tile + r * LD + c);
      float* dst = a.out32 + (size_t)row * a.ldo32 + col;
      if (EPI == ENC_EPI_BIAS_RES_F32) {
        const float4 in = *reinterpret_cast<const float4*>(dst);
        *reinterpret_cast<float4*>(dst) = make_float4(in.x + x.x, in.y + x.y, in.z + x.z, in.w + x.w);
      } else {
        const float4 in = *reinterpret_cast<const float4*>(a.pos + (size_t)row * a.N + col);
        *reinterpret_cast<float4*>(dst) =
            make_float4(gelu_erf(x.x) + in.x, gelu_erf(x.y) + in.y, gelu_erf(x.z) + in.z, gelu_erf(x.w) + in.w);
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// host side: tensor maps (cached per operand view) and launch
// ---------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

// 2-D fp16 view [rows][K] with row stride `ld` elements, boxes of [128 rows][64 columns], SWIZZLE_128B
static bool make_map(CUtensorMap* map, const __half* base, uint64_t rows, uint64_t K, uint64_t ld, uint32_t box_rows) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return false;
  cuuint64_t dims[2] = {K, rows};
  cuuint64_t strides[1] = {ld * sizeof(__half)};
  cuuint32_t box[2] = {TC_BK, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<__half*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS;
}

static constexpr size_t tc_smem(int bm, int bn, int stages) { return (size_t)stages * tc_stage_bytes(bm, bn) + 1024; }

// every instantiation: X(EPI, BM, BN, STAGES) -- exactly the tiles pick_tile can return for each epilogue
// (tests/test_encoder_gemm_tiles.py derives this list from the widths the suite runs and compares)
#define WM_TC_F16_TILES(X, EPI) X(EPI, 128, 128, 3) X(EPI, 128, 128, 6) X(EPI, 256, 128, 4) X(EPI, 128, 192, 5)
#define WM_TC_ALL(X)                                                                                             \
  WM_TC_F16_TILES(X, ENC_EPI_BIAS_F16) WM_TC_F16_TILES(X, ENC_EPI_BIAS_GELU_F16)                                 \
  X(ENC_EPI_BIAS_RES_F32, 128, 128, 6) X(ENC_EPI_BIAS_GELU_POS_F32, 128, 128, 6)

cudaError_t enc_gemm_tc_configure() {
  cudaError_t e;
#define WM_SET(EPI, BM, BN, ST)                                                                                          \
  e = cudaFuncSetAttribute(enc_gemm_tc_kernel<EPI, BM, BN, ST>, cudaFuncAttributeMaxDynamicSharedMemorySize,             \
                           (int)tc_smem(BM, BN, ST));                                                                    \
  if (e != cudaSuccess) return e;
  WM_TC_ALL(WM_SET)
#undef WM_SET
  return get_encode_fn() ? cudaSuccess : cudaErrorNotSupported;
}

// Tile shape of one GEMM.  Tiles are dealt to the SMs in ceil(tiles / n_sm) rounds of K * (BM + BN) * 2 operand bytes
// each; the shape with the fewest operand bytes on the busiest SM wins.  The wide candidates exist for the fp16-output
// epilogues only (the fp32 read-modify-write epilogues feed N = d outputs: too few tiles already, always one CTA per SM
// with the deep ring).  128 x 256 is no candidate: at M = 1500 and 3000 it costs exactly what 256 x 128 costs.
struct TcTile { int bm, bn, stages; };
static TcTile pick_tile(const EncGemmArgs& g, int n_sm) {
  const bool f16_out = g.epi == ENC_EPI_BIAS_F16 || g.epi == ENC_EPI_BIAS_GELU_F16;
  const bool narrow = g.N <= 1536 || !f16_out;   // few 128 x 128 tiles per SM and round: one CTA per SM with a deep ring
  TcTile best = {TC_BM, TC_BN, narrow ? 6 : 3};
  if (g.tile == 1 || !f16_out) return best;
  auto cost = [&](int bm, int bn) {
    const long tiles = (long)((g.M + bm - 1) / bm) * (g.N / bn);
    return ((tiles + n_sm - 1) / n_sm) * (long)(bm + bn);
  };
  long c = cost(best.bm, best.bn);
  const TcTile wide[2] = {{256, 128, 4}, {128, 192, 5}};
  for (const TcTile& t : wide) {
    if (g.N % t.bn != 0) continue;
    const long ct = cost(t.bm, t.bn);
    if (ct < c) { c = ct; best = t; }
  }
  return best;
}

void enc_gemm_tc_tile(int M, int N, int K, bool fp16_out, int n_sm, int out[3]) {
  EncGemmArgs g;
  memset(&g, 0, sizeof g);
  g.M = M; g.N = N; g.K = K; g.epi = fp16_out ? ENC_EPI_BIAS_F16 : ENC_EPI_BIAS_RES_F32;
  const TcTile t = pick_tile(g, n_sm > 0 ? n_sm : 132);
  out[0] = t.bm; out[1] = t.bn; out[2] = t.stages;
}

// `a_rows` = rows of the A view that may be touched (the allocation is padded accordingly)
cudaError_t enc_gemm_tc(const EncGemmArgs& g, int a_rows, cudaStream_t s, int64_t* n_launch) {
  if (g.N % TC_BN != 0 || g.K % TC_BK != 0 || (g.lda % 8) != 0) return cudaErrorInvalidValue;
  typedef std::tuple<const void*, uint64_t, uint64_t, uint64_t, uint32_t> Key;
  static thread_local std::map<Key, CUtensorMap> cache;
  auto get = [&](const __half* base, uint64_t rows, uint64_t K, uint64_t ld, uint32_t box_rows, CUtensorMap* out) -> bool {
    Key k(base, rows, K, ld, box_rows);
    auto it = cache.find(k);
    if (it == cache.end()) {
      CUtensorMap m;
      if (!make_map(&m, base, rows, K, ld, box_rows)) return false;
      it = cache.emplace(k, m).first;
    }
    *out = it->second;
    return true;
  };
  static thread_local int n_sm = 0;
  if (n_sm == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess ||
        cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n_sm <= 0)
      n_sm = 132;
  }
  const TcTile t = pick_tile(g, n_sm);
  CUtensorMap ma, mw;
  if (!get(g.A, (uint64_t)a_rows, (uint64_t)g.K, (uint64_t)g.lda, (uint32_t)t.bm, &ma)) return cudaErrorInvalidValue;
  if (!get(g.W, (uint64_t)g.N, (uint64_t)g.K, (uint64_t)g.K, (uint32_t)t.bn, &mw)) return cudaErrorInvalidValue;
  TcArgs a;
  a.M = g.M; a.N = g.N; a.K = g.K; a.epi = g.epi; a.bias = g.bias; a.out16 = g.out16; a.ldo16 = g.ldo16;
  a.out32 = g.out32; a.ldo32 = g.ldo32; a.pos = g.pos;
  a.vt = g.vt; a.vt_col0 = g.vt_col0; a.vt_ld = g.vt_ld;
  a.ck = g.ck; a.cv = g.cv; a.kv_spad = g.kv_spad;
  if (a.ck != nullptr && (g.epi != ENC_EPI_BIAS_F16 || (g.N >> 1) % 64 != 0)) return cudaErrorInvalidValue;
  dim3 grid(g.N / t.bn, (g.M + t.bm - 1) / t.bm);
  bool launched = false;
  cudaError_t le = cudaSuccess;
#define WM_LAUNCH(EPI, BM, BN, ST)                                                                                       \
  if (!launched && g.epi == EPI && t.bm == BM && t.bn == BN && t.stages == ST) {                                          \
    le = tc_launch(enc_gemm_tc_kernel<EPI, BM, BN, ST>, grid, dim3(TC_THREADS), tc_smem(BM, BN, ST), s, g.pdl != 0, ma,  \
                   mw, a);                                                                                               \
    launched = true;                                                                                                     \
  }
  WM_TC_ALL(WM_LAUNCH)
#undef WM_LAUNCH
  if (!launched) return cudaErrorInvalidValue;
  if (le != cudaSuccess) return le;
  if (n_launch) ++*n_launch;
  return cudaGetLastError();
}

}  // namespace wm
