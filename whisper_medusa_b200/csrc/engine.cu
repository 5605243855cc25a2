// C ABI + host orchestration of the Whisper-Medusa decode path (see include/whisper_medusa_b200.h).
//
// Host responsibilities only: own device memory, define the packed-weight layout, enqueue the
// mel / encoder / cross-KV kernels for a clip, and drive the speculative loop (CUDA graphs of
// stage kernels, or the persistent per-iteration kernel).  No arithmetic of the path runs on
// the host; there is no CPU fallback.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <map>
#include <string>
#include <vector>

#include "../../include/whisper_medusa_b200.h"
#include "common.cuh"
#include "engine.h"

using namespace wm;

namespace {

struct TensorInfo {
  std::string name;
  size_t offset, nbytes;
  int dtype;  // 0 f16, 1 f32
};

constexpr int kFrames = 3000;
constexpr int kSamples = 480000;
constexpr int kNFreq = 201;

inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

}  // namespace

struct wm_handle {
  wm_config cfg;
  int device = 0;
  int n_sm = 0;
  int n_cta = 0;           // CTAs of the decode kernels (default: every SM; option "decode_ctas" partitions the GPU between streams)
  cudaStream_t stream = nullptr;
  std::string err;
  // weights
  std::vector<TensorInfo> tensors;
  std::map<std::string, int> tindex;
  size_t wbytes = 0;
  unsigned char* wdev = nullptr;
  bool wowned = false, wready = false;
  // dims
  int S = 0, S_pad = 0, n_dec = 0;  // n_dec = decoder layers + block
  // encoder buffers
  float *pcm = nullptr, *mel32 = nullptr, *melfb = nullptr, *x32 = nullptr, *enc32 = nullptr;
  __half *x_tm = nullptr, *h1 = nullptr, *ln16 = nullptr, *qkv16 = nullptr, *att16 = nullptr, *ffn16 = nullptr,
         *enc16 = nullptr, *vt16 = nullptr;
  int* gmax = nullptr;
  std::vector<__half*> cross_k, cross_v, self_k, self_v;
  // decode buffers
  DecModel hm;             // host copy
  DecModel* dm = nullptr;  // device copy
  DecState* st = nullptr;
  uint8_t* tok_mask = nullptr;
  float* pen_tab = nullptr;
  unsigned int* bar = nullptr;
  int* prog = nullptr;
  unsigned long long* prof = nullptr;
  ChunkDesc* chunk_tab = nullptr;
  int* chunk_off = nullptr;
  CtaStage* stage_tab = nullptr;
  float2* ln_fold = nullptr;     // {b'_n, c_n} of the LayerNorm-fed GEMMs of the ring kernel (derived from the weights)
  DecTree* tree = nullptr;       // device copy of the candidate tree (branching medusa_choices)
  DecHostInfo hi;
  std::map<int, cudaGraphExec_t> graph_a;  // sweep A, keyed by T
  cudaGraphExec_t graph_tail = nullptr, graph_b = nullptr;
  int64_t launches_a[WM_MAX_T + 1] = {0};
  int64_t launches_tail = 0, launches_b = 0;
  int decode_mode = 0;
  int enc_gemm_impl = 0;   // 0 = mma.sync kernel, 1 = wgmma/TMA kernel
  int enc_pdl = 1;         // encoder kernels launched with programmatic stream serialization (option "enc_pdl" = 0: plain launches)
  int enc_gemm_tile = 0;   // wgmma kernel: 0 = tile shape picked per GEMM, 1 = 128 x 128 tiles only (option "enc_gemm" = 2)
  int enc_attn_impl = 0;   // 0 = mma.sync flash attention, 1 = wgmma/TMA attention
  bool tc_ok = false, attn_tc_ok = false;
  bool encoded = false;
  // pinned staging + timing
  int* h_state = nullptr;  // pinned copy of the DecState header
  float* h_stage = nullptr;  // pinned staging for pcm / mel
  DecState* h_init = nullptr;  // pinned initial loop state (uploaded asynchronously by wm_generate)
  float* h_pen = nullptr;      // pinned EOS-penalty table
  cudaEvent_t ev[6] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
  double ms[3] = {0, 0, 0};
  int64_t launches[3] = {0, 0, 0};
  float last_pen_factor = 0.f;
  int last_pen_start = -2, last_pen_prompt = -1;
  // resampler tap tables on the device, one per (orig_hz, new_hz) pair used on this handle
  struct Resampler {
    ResampleTable t;
    float* taps = nullptr;   // [max_taps][nw]
    int2* sup = nullptr;     // [nw] {lo - width, n}
    int T = 0;
    size_t smem = 0;
  };
  std::map<std::pair<int, int>, Resampler> resamplers;
};

static_assert(offsetof(DecState, tree_attn) == 60, "the 16 header words of DecState (L .. tree_attn) are patched as one 64-byte copy");

#define CK(call)                                                                                   \
  do {                                                                                             \
    cudaError_t _e = (call);                                                                       \
    if (_e != cudaSuccess) {                                                                       \
      char _b[512];                                                                                \
      snprintf(_b, sizeof _b, "%s failed at %s:%d: %s", #call, __FILE__, __LINE__, cudaGetErrorString(_e)); \
      h->err = _b;                                                                                 \
      return WM_ERR_CUDA;                                                                          \
    }                                                                                              \
  } while (0)

static int fail(wm_handle* h, int code, const std::string& msg) {
  if (h) h->err = msg;
  return code;
}

// ---------------------------------------------------------------------------------------------
// packed-weight layout
// ---------------------------------------------------------------------------------------------
static void add_tensor(wm_handle* h, const std::string& name, size_t elems, int dtype) {
  TensorInfo t;
  t.name = name;
  t.offset = align_up(h->wbytes, 256);
  t.nbytes = elems * (dtype == 0 ? 2 : 4);
  t.dtype = dtype;
  h->wbytes = t.offset + t.nbytes;
  h->tindex[name] = (int)h->tensors.size();
  h->tensors.push_back(t);
}

static void build_layout(wm_handle* h) {
  const wm_config& c = h->cfg;
  const size_t d = c.d_model, f = c.ffn_dim, V = c.vocab_size;
  add_tensor(h, "enc.conv1_w", d * 256, 0);
  add_tensor(h, "enc.conv1_b", d, 1);
  add_tensor(h, "enc.conv2_w", d * 3 * d, 0);
  add_tensor(h, "enc.conv2_b", d, 1);
  add_tensor(h, "enc.pos", (size_t)c.max_source_positions * d, 1);
  for (int i = 0; i < c.enc_layers; ++i) {
    std::string p = "enc." + std::to_string(i) + ".";
    add_tensor(h, p + "ln1_g", d, 1); add_tensor(h, p + "ln1_b", d, 1);
    add_tensor(h, p + "qkv_w", 3 * d * d, 0); add_tensor(h, p + "qkv_b", 3 * d, 1);
    add_tensor(h, p + "o_w", d * d, 0); add_tensor(h, p + "o_b", d, 1);
    add_tensor(h, p + "ln2_g", d, 1); add_tensor(h, p + "ln2_b", d, 1);
    add_tensor(h, p + "fc1_w", f * d, 0); add_tensor(h, p + "fc1_b", f, 1);
    add_tensor(h, p + "fc2_w", d * f, 0); add_tensor(h, p + "fc2_b", d, 1);
  }
  add_tensor(h, "enc.lnf_g", d, 1); add_tensor(h, "enc.lnf_b", d, 1);
  add_tensor(h, "dec.embed", V * d, 0);
  add_tensor(h, "dec.pos", (size_t)c.max_target_positions * d, 1);
  for (int i = 0; i < h->n_dec; ++i) {
    std::string p = "dec." + std::to_string(i) + ".";
    add_tensor(h, p + "ln1_g", d, 1); add_tensor(h, p + "ln1_b", d, 1);
    add_tensor(h, p + "qkv_w", 3 * d * d, 0); add_tensor(h, p + "qkv_b", 3 * d, 1);
    add_tensor(h, p + "o_w", d * d, 0); add_tensor(h, p + "o_b", d, 1);
    add_tensor(h, p + "ln2_g", d, 1); add_tensor(h, p + "ln2_b", d, 1);
    add_tensor(h, p + "cq_w", d * d, 0); add_tensor(h, p + "cq_b", d, 1);
    add_tensor(h, p + "ckv_w", 2 * d * d, 0); add_tensor(h, p + "ckv_b", 2 * d, 1);
    add_tensor(h, p + "co_w", d * d, 0); add_tensor(h, p + "co_b", d, 1);
    add_tensor(h, p + "ln3_g", d, 1); add_tensor(h, p + "ln3_b", d, 1);
    add_tensor(h, p + "fc1_w", f * d, 0); add_tensor(h, p + "fc1_b", f, 1);
    add_tensor(h, p + "fc2_w", d * f, 0); add_tensor(h, p + "fc2_b", d, 1);
  }
  add_tensor(h, "dec.lnf_g", d, 1); add_tensor(h, "dec.lnf_b", d, 1);
  const size_t nh = c.medusa_block ? c.medusa_num_heads : c.medusa_num_heads + 1;
  add_tensor(h, "heads_w", nh * d * d, 0);
  add_tensor(h, "heads_b", nh * d, 1);
  h->wbytes = align_up(h->wbytes, 256);
}

template <typename T>
static const T* wptr(wm_handle* h, const std::string& name) {
  auto it = h->tindex.find(name);
  if (it == h->tindex.end()) return nullptr;
  return reinterpret_cast<const T*>(h->wdev + h->tensors[it->second].offset);
}

// ---------------------------------------------------------------------------------------------
// slaney mel filter bank [201][80]  (HF audio_utils.py mel_filter_bank, norm="slaney",
// mel_scale="slaney"; called from feature_extraction_whisper.py:95-103)
// ---------------------------------------------------------------------------------------------
static double hz_to_mel(double f) {
  const double min_log_hz = 1000.0, min_log_mel = 15.0, logstep = 27.0 / std::log(6.4);
  return f >= min_log_hz ? min_log_mel + std::log(f / min_log_hz) * logstep : 3.0 * f / 200.0;
}
static double mel_to_hz(double m) {
  const double min_log_hz = 1000.0, min_log_mel = 15.0, logstep = std::log(6.4) / 27.0;
  return m >= min_log_mel ? min_log_hz * std::exp(logstep * (m - min_log_mel)) : 200.0 * m / 3.0;
}
static std::vector<float> build_mel_filters(int n_mels) {
  std::vector<double> ff(n_mels + 2);
  const double m0 = hz_to_mel(0.0), m1 = hz_to_mel(8000.0);
  for (int i = 0; i < n_mels + 2; ++i) ff[i] = mel_to_hz(m0 + (m1 - m0) * i / (n_mels + 1));
  std::vector<float> fb((size_t)kNFreq * n_mels);
  for (int k = 0; k < kNFreq; ++k) {
    const double fk = 8000.0 * k / (kNFreq - 1);
    for (int m = 0; m < n_mels; ++m) {
      const double down = (fk - ff[m]) / (ff[m + 1] - ff[m]);
      const double up = (ff[m + 2] - fk) / (ff[m + 2] - ff[m + 1]);
      double v = std::fmax(0.0, std::fmin(down, up));
      v *= 2.0 / (ff[m + 2] - ff[m]);
      fb[(size_t)k * n_mels + m] = (float)v;
    }
  }
  return fb;
}

// ---------------------------------------------------------------------------------------------
// lifetime
// ---------------------------------------------------------------------------------------------
template <typename T>
static cudaError_t dalloc(T** p, size_t elems) {
  cudaError_t e = cudaMalloc((void**)p, elems * sizeof(T));
  if (e != cudaSuccess) return e;
  return cudaMemset(*p, 0, elems * sizeof(T));
}

// How the decode stages split over the n_cta CTAs of the decode grid: key chunks per head of the cross-attention
// stage (a chunk must fit one ring slot: <= WM_CH_MAX keys) and vocabulary segments per row of the logits scan.
static void set_decode_split(wm_handle* h) {
  DecModel& m = h->hm;
  const int min_chunks = (h->S + WM_CH_MAX_KEYS - 1) / WM_CH_MAX_KEYS;
  m.cross_chunks = h->n_cta / h->cfg.n_heads;
  if (m.cross_chunks < min_chunks) m.cross_chunks = min_chunks;
  if (m.cross_chunks > WM_CROSS_CHUNKS) m.cross_chunks = WM_CROSS_CHUNKS;
  m.sel_nseg = h->n_cta / (h->cfg.medusa_num_heads + 1);
  if (m.sel_nseg < 1) m.sel_nseg = 1;
  if (m.sel_nseg > 32) m.sel_nseg = 32;
}
// graph / persistent_simple stages hold at most 3 16-row units per warp (stage_gemm): the vocabulary projection
// needs enough CTAs for that; the ring kernel has no such limit
static bool simple_modes_fit(const wm_handle* h) {
  const int rows = (h->cfg.vocab_size + h->n_cta - 1) / h->n_cta;
  return (rows + 15) / 16 <= 3 * (WM_DEC_THREADS / 32);
}

extern "C" int wm_create(const wm_config* cfg, int device, wm_handle** out) {
  if (!cfg || !out) return WM_ERR_INVALID;
  *out = nullptr;
  wm_handle* h = new wm_handle();
  h->cfg = *cfg;
  h->device = device;
  const wm_config& c = h->cfg;
  auto bad = [&](const char* m) { h->err = m; *out = h; return WM_ERR_INVALID; };
  if (c.d_model % 128 != 0 || c.n_heads * WM_HEAD_DIM != c.d_model) return bad("d_model must be n_heads*64 and a multiple of 128");
  if (c.ffn_dim % 128 != 0) return bad("ffn_dim must be a multiple of 128");
  if (c.n_mels != 80) return bad("n_mels must be 80");
  if (c.medusa_num_heads < 1 || c.medusa_num_heads + 1 > WM_MAX_T) return bad("medusa_num_heads must be in [1, 15]");
  if (c.dec_layers + 1 > WM_MAX_DEC_LAYERS) return bad("too many decoder layers");
  if (c.max_target_positions + c.medusa_num_heads + 2 > WM_MAX_POS) return bad("max_target_positions too large");
  if (c.max_source_positions != 1500) return bad("max_source_positions must be 1500 (30 s window)");
  *out = h;
  h->S = c.max_source_positions;
  h->S_pad = (int)align_up(h->S, 128);
  h->n_dec = c.dec_layers + (c.medusa_block ? 1 : 0);
  build_layout(h);
  if (device < 0) return WM_OK;  // layout-only handle (weight packing / tests on a box without a GPU)
  CK(cudaSetDevice(device));
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0) return fail(h, WM_ERR_UNSUPPORTED, "this engine is built for sm_90a (H100) only");
  h->n_sm = prop.multiProcessorCount;
  h->n_cta = h->n_sm;
  CK(cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
  for (auto& e : h->ev) CK(cudaEventCreate(&e));

  const size_t d = c.d_model, f = c.ffn_dim, V = c.vocab_size, SP = h->S_pad;
  CK(dalloc(&h->pcm, (size_t)kSamples));
  CK(dalloc(&h->mel32, (size_t)80 * kFrames));
  CK(dalloc(&h->melfb, (size_t)kNFreq * 80));
  CK(dalloc(&h->gmax, 1));
  CK(dalloc(&h->x_tm, (size_t)3080 * 80));
  CK(dalloc(&h->h1, (size_t)3080 * d));
  CK(dalloc(&h->x32, SP * d));
  CK(dalloc(&h->enc32, SP * d));
  CK(dalloc(&h->ln16, SP * d));
  CK(dalloc(&h->qkv16, SP * 3 * d));
  CK(dalloc(&h->att16, SP * d));
  CK(dalloc(&h->ffn16, SP * f));
  CK(dalloc(&h->enc16, SP * d));
  CK(dalloc(&h->vt16, d * SP));
  h->cross_k.resize(h->n_dec);
  h->cross_v.resize(h->n_dec);
  h->self_k.resize(h->n_dec);
  h->self_v.resize(h->n_dec);
  for (int i = 0; i < h->n_dec; ++i) {
    CK(dalloc(&h->cross_k[i], (size_t)c.n_heads * SP * 72));
    CK(dalloc(&h->cross_v[i], (size_t)c.n_heads * SP * 72));
    CK(dalloc(&h->self_k[i], (size_t)WM_MAX_POS * d));
    CK(dalloc(&h->self_v[i], (size_t)WM_MAX_POS * d));
  }
  {
    std::vector<float> fb = build_mel_filters(80);
    CK(cudaMemcpy(h->melfb, fb.data(), fb.size() * sizeof(float), cudaMemcpyHostToDevice));
  }
  // decode buffers
  DecModel& m = h->hm;
  memset(&m, 0, sizeof m);
  m.d = (int)d; m.H = c.n_heads; m.ffn = (int)f; m.V = (int)V; m.S = h->S; m.S_pad = h->S_pad;
  m.n_layers = c.dec_layers; m.has_block = c.medusa_block ? 1 : 0; m.K = c.medusa_num_heads;
  m.n_tree = c.medusa_num_heads + 1; m.has_tree = 0; m.tree = nullptr;
  CK(dalloc(&h->tree, 1));
  CK(dalloc(&m.topk_part, (size_t)WM_MAX_T * 32 * WM_TREE_MAX_TOPK * 2));
  CK(dalloc(&m.x, (size_t)WM_MAX_T * d));
  CK(dalloc(&m.xg, (size_t)WM_MAX_T * d));
  CK(dalloc(&m.q, (size_t)WM_MAX_T * d));
  CK(dalloc(&m.attn, (size_t)WM_MAX_T * d));
  CK(dalloc(&m.ffn_h, (size_t)WM_MAX_T * f));
  CK(dalloc(&m.hidden, (size_t)WM_MAX_T * d));
  CK(dalloc(&m.head_h, (size_t)WM_MAX_T * d));
  CK(dalloc(&m.carry, d));
  CK(dalloc(&m.cross_part, (size_t)c.n_heads * WM_CROSS_CHUNKS * WM_MAX_T * (WM_HEAD_DIM + 2)));
  CK(dalloc(&m.cross_cnt, (size_t)c.n_heads));
  set_decode_split(h);
  if (f % d != 0 || f / d > 8 || h->n_sm < (int)(f / d)) return fail(h, WM_ERR_UNSUPPORTED, "ffn_dim must be a multiple (<= 8x) of d_model");
  CK(dalloc(&m.gemm_part, (size_t)8 * WM_MAX_T * d));
  CK(dalloc(&m.gemm_cnt, (size_t)h->n_sm));
  CK(dalloc(&m.sel_part, (size_t)WM_MAX_T * 32 * 4));
  CK(dalloc(&m.logits_a, (size_t)WM_MAX_T * V));
  CK(dalloc(&m.logits_b, (size_t)WM_MAX_T * V));
  CK(dalloc(&h->st, 1));
  CK(dalloc(&h->tok_mask, V));
  CK(dalloc(&h->pen_tab, (size_t)WM_MAX_POS + 32));
  CK(dalloc(&h->bar, 8));
  CK(dalloc(&h->dm, 1));
  m.st = h->st; m.tok_mask = h->tok_mask; m.pen_tab = h->pen_tab; m.bar = h->bar;
  CK(cudaMallocHost((void**)&h->h_state, 64 * sizeof(int)));
  CK(cudaMallocHost((void**)&h->h_stage, (size_t)kSamples * sizeof(float)));
  CK(cudaMallocHost((void**)&h->h_init, sizeof(DecState)));
  CK(cudaMallocHost((void**)&h->h_pen, (size_t)(WM_MAX_POS + 32) * sizeof(float)));

  h->hi.n_sm = h->n_cta; h->hi.H = c.n_heads; h->hi.K = c.medusa_num_heads; h->hi.n_layers = c.dec_layers;
  h->hi.has_block = m.has_block;
  h->hi.n_tree = m.n_tree;
  h->hi.d = (int)d;
  h->hi.smem = dec_smem_bytes((int)d, (int)f);
  h->hi.smem_ring = dec_ring_smem_bytes((int)d);
  CK(dec_configure((int)d, h->hi.smem, h->hi.smem_ring));
  h->hi.cluster = dec_ring_cluster_size(h->hi, h->n_sm);
  // product path by default: one persistent ring-kernel launch per speculative iteration.  Decoder widths the ring
  // kernel is not instantiated for (WM_RING_WIDTHS) fall back to the stage-kernel graphs.
  h->decode_mode = h->hi.smem_ring ? 2 : 0;
  {
    std::vector<int> flat;
    dec_build_program(c.dec_layers, m.has_block, flat, m.prog_off);
    CK(dalloc(&h->prog, flat.size()));
    CK(cudaMemcpy(h->prog, flat.data(), flat.size() * sizeof(int), cudaMemcpyHostToDevice));
    m.prog = reinterpret_cast<const StageInstr*>(h->prog);
  }
  CK(enc_gemm_configure());
  h->tc_ok = (enc_gemm_tc_configure() == cudaSuccess);
  h->enc_gemm_impl = h->tc_ok ? 1 : 0;   // wgmma/TMA GEMM by default; option "enc_gemm" = 0 selects the mma.sync kernel
  h->attn_tc_ok = (enc_attention_tc_configure() == cudaSuccess);
  h->enc_attn_impl = h->attn_tc_ok ? 1 : 0;   // likewise option "enc_attn"
  (void)cudaGetLastError();
  if (!simple_modes_fit(h) && !h->hi.smem_ring) return fail(h, WM_ERR_UNSUPPORTED, "too few SMs for the vocab projection split");
  return WM_OK;
}

extern "C" int wm_destroy(wm_handle* h) {
  if (!h) return WM_OK;
  if (h->device < 0) { delete h; return WM_OK; }
  cudaSetDevice(h->device);
  if (h->stream) cudaStreamSynchronize(h->stream);
  for (auto& kv : h->graph_a) cudaGraphExecDestroy(kv.second);
  if (h->graph_b) cudaGraphExecDestroy(h->graph_b);
  if (h->graph_tail) cudaGraphExecDestroy(h->graph_tail);
  auto F = [](void* p) { if (p) cudaFree(p); };
  F(h->pcm); F(h->mel32); F(h->melfb); F(h->gmax); F(h->x_tm); F(h->h1); F(h->x32); F(h->enc32); F(h->ln16);
  F(h->qkv16); F(h->att16); F(h->ffn16); F(h->enc16); F(h->vt16);
  for (auto p : h->cross_k) F(p);
  for (auto p : h->cross_v) F(p);
  for (auto p : h->self_k) F(p);
  for (auto p : h->self_v) F(p);
  F(h->hm.x); F(h->hm.xg); F(h->hm.q); F(h->hm.attn); F(h->hm.ffn_h); F(h->hm.hidden); F(h->hm.head_h); F(h->hm.carry); F(h->hm.cross_part); F(h->hm.cross_cnt); F(h->hm.sel_part); F(h->hm.gemm_part); F(h->hm.gemm_cnt);
  F(h->hm.topk_part); F(h->tree); F(h->hm.logits_a); F(h->hm.logits_b); F(h->st); F(h->tok_mask); F(h->pen_tab); F(h->bar); F(h->prog); F(h->prof); F(h->chunk_tab); F(h->chunk_off); F(h->stage_tab); F(h->ln_fold); F(h->dm);
  if (h->wowned) F(h->wdev);
  for (auto& kv : h->resamplers) { F(kv.second.taps); F(kv.second.sup); }
  if (h->h_state) cudaFreeHost(h->h_state);
  if (h->h_stage) cudaFreeHost(h->h_stage);
  if (h->h_init) cudaFreeHost(h->h_init);
  if (h->h_pen) cudaFreeHost(h->h_pen);
  for (auto& e : h->ev) if (e) cudaEventDestroy(e);
  if (h->stream) cudaStreamDestroy(h->stream);
  delete h;
  return WM_OK;
}

extern "C" const char* wm_strerror(int status) {
  switch (status) {
    case WM_OK: return "ok";
    case WM_ERR_INVALID: return "invalid argument or configuration";
    case WM_ERR_CUDA: return "CUDA error";
    case WM_ERR_STATE: return "call order violated";
    case WM_ERR_UNSUPPORTED: return "not supported";
    case WM_ERR_NOMEM: return "out of memory";
    default: return "unknown status";
  }
}
extern "C" const char* wm_last_error(wm_handle* h) { return h ? h->err.c_str() : "null handle"; }

// ---------------------------------------------------------------------------------------------
// weights
// ---------------------------------------------------------------------------------------------
extern "C" int wm_tensor_count(wm_handle* h) { return h ? (int)h->tensors.size() : 0; }
extern "C" const char* wm_tensor_name(wm_handle* h, int i) {
  if (!h || i < 0 || i >= (int)h->tensors.size()) return nullptr;
  return h->tensors[i].name.c_str();
}
extern "C" int wm_tensor_info(wm_handle* h, const char* name, size_t* offset, size_t* nbytes, int32_t* dtype) {
  if (!h || !name) return WM_ERR_INVALID;
  auto it = h->tindex.find(name);
  if (it == h->tindex.end()) return fail(h, WM_ERR_INVALID, std::string("unknown tensor ") + name);
  const TensorInfo& t = h->tensors[it->second];
  if (offset) *offset = t.offset;
  if (nbytes) *nbytes = t.nbytes;
  if (dtype) *dtype = t.dtype;
  return WM_OK;
}
extern "C" size_t wm_weights_nbytes(wm_handle* h) { return h ? h->wbytes : 0; }

static int bind_weights(wm_handle* h) {
  DecModel& m = h->hm;
  for (int i = 0; i < h->n_dec; ++i) {
    std::string p = "dec." + std::to_string(i) + ".";
    DecLayer& L = m.layers[i];
    L.ln1_g = wptr<float>(h, p + "ln1_g"); L.ln1_b = wptr<float>(h, p + "ln1_b");
    L.qkv_w = wptr<__half>(h, p + "qkv_w"); L.qkv_b = wptr<float>(h, p + "qkv_b");
    L.o_w = wptr<__half>(h, p + "o_w"); L.o_b = wptr<float>(h, p + "o_b");
    L.ln2_g = wptr<float>(h, p + "ln2_g"); L.ln2_b = wptr<float>(h, p + "ln2_b");
    L.cq_w = wptr<__half>(h, p + "cq_w"); L.cq_b = wptr<float>(h, p + "cq_b");
    L.co_w = wptr<__half>(h, p + "co_w"); L.co_b = wptr<float>(h, p + "co_b");
    L.ln3_g = wptr<float>(h, p + "ln3_g"); L.ln3_b = wptr<float>(h, p + "ln3_b");
    L.fc1_w = wptr<__half>(h, p + "fc1_w"); L.fc1_b = wptr<float>(h, p + "fc1_b");
    L.fc2_w = wptr<__half>(h, p + "fc2_w"); L.fc2_b = wptr<float>(h, p + "fc2_b");
    L.self_k = h->self_k[i]; L.self_v = h->self_v[i]; L.cross_k = h->cross_k[i]; L.cross_v = h->cross_v[i];
  }
  m.embed = wptr<__half>(h, "dec.embed");
  m.pos = wptr<float>(h, "dec.pos");
  m.lnf_g = wptr<float>(h, "dec.lnf_g"); m.lnf_b = wptr<float>(h, "dec.lnf_b");
  m.heads_w = wptr<__half>(h, "heads_w"); m.heads_b = wptr<float>(h, "heads_b");
  // LayerNorm beta / gamma folded through the weights they feed (ring kernel; a function of the weight values, so
  // derived again at every binding: upload, broadcast, adoption of another engine's weights)
  if (!h->ln_fold) CK(dalloc(&h->ln_fold, dec_ln_fold_len(h->n_dec, h->cfg.d_model, h->cfg.ffn_dim)));
  CK(dec_fold_layernorms(m, h->n_dec, h->ln_fold, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  {
    // weight-chunk schedule of the ring producer (depends on the weight addresses)
    std::vector<ChunkDesc> tab;
    std::vector<int> off;
    dec_build_chunk_table(m, h->n_cta, tab, off);
    if (h->chunk_tab) { cudaFree(h->chunk_tab); h->chunk_tab = nullptr; }
    if (h->chunk_off) { cudaFree(h->chunk_off); h->chunk_off = nullptr; }
    CK(cudaMalloc((void**)&h->chunk_tab, tab.size() * sizeof(ChunkDesc)));
    CK(cudaMalloc((void**)&h->chunk_off, off.size() * sizeof(int)));
    CK(cudaMemcpy(h->chunk_tab, tab.data(), tab.size() * sizeof(ChunkDesc), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(h->chunk_off, off.data(), off.size() * sizeof(int), cudaMemcpyHostToDevice));
    m.chunk_tab = h->chunk_tab;
    m.chunk_off = h->chunk_off;
    std::vector<CtaStage> stab;
    dec_build_stage_table(m, h->ln_fold, h->n_cta, h->hi.cluster, stab);
    if (h->stage_tab) { cudaFree(h->stage_tab); h->stage_tab = nullptr; }
    CK(cudaMalloc((void**)&h->stage_tab, stab.size() * sizeof(CtaStage)));
    CK(cudaMemcpy(h->stage_tab, stab.data(), stab.size() * sizeof(CtaStage), cudaMemcpyHostToDevice));
    m.stage_tab = h->stage_tab;
  }
  CK(cudaMemcpy(h->dm, &m, sizeof m, cudaMemcpyHostToDevice));
  h->wready = true;
  return WM_OK;
}

extern "C" int wm_load_weights(wm_handle* h, const void* blob, size_t nbytes) {
  if (!h || !blob) return WM_ERR_INVALID;
  if (h->device < 0) return fail(h, WM_ERR_STATE, "layout-only handle");
  if (nbytes != h->wbytes) return fail(h, WM_ERR_INVALID, "weight blob size mismatch");
  CK(cudaSetDevice(h->device));
  if (h->wdev && !h->wowned) h->wdev = nullptr;
  if (!h->wdev) { CK(cudaMalloc((void**)&h->wdev, h->wbytes)); h->wowned = true; }
  CK(cudaMemcpy(h->wdev, blob, nbytes, cudaMemcpyHostToDevice));
  return bind_weights(h);
}
extern "C" int wm_adopt_weights(wm_handle* h, void* device_blob, size_t nbytes) {
  if (!h || !device_blob) return WM_ERR_INVALID;
  if (h->device < 0) return fail(h, WM_ERR_STATE, "layout-only handle");
  if (nbytes != h->wbytes) return fail(h, WM_ERR_INVALID, "weight blob size mismatch");
  CK(cudaSetDevice(h->device));
  if (h->wdev && h->wowned) cudaFree(h->wdev);
  h->wdev = reinterpret_cast<unsigned char*>(device_blob);
  h->wowned = false;
  return bind_weights(h);
}

// Candidate tree of branching medusa_choices (reference medusa_utils.py:305-421, restated): choices[i] = how many of
// head i's top tokens are tried at depth i (choices[0] = 1: the base head's argmax).  All ones = the top-1 chain.
extern "C" int wm_set_medusa_choices(wm_handle* h, const int32_t* choices, int32_t n) {
  if (!h || !choices) return WM_ERR_INVALID;
  if (h->device < 0) return fail(h, WM_ERR_STATE, "layout-only handle");
  const int K = h->cfg.medusa_num_heads;
  if (n != K + 1) return fail(h, WM_ERR_INVALID, "medusa_choices must have medusa_num_heads + 1 entries");
  if (choices[0] != 1) return fail(h, WM_ERR_INVALID, "medusa_choices[0] must be 1 (the base head is greedy)");
  static thread_local DecTree t;
  memset(&t, 0, sizeof t);
  bool chain = true;
  long n_tree = 0, level = 1;
  for (int i = 0; i <= K; ++i) {
    if (choices[i] < 1 || choices[i] > WM_TREE_MAX_TOPK) return fail(h, WM_ERR_UNSUPPORTED, "medusa_choices entries must be in 1..4");
    if (choices[i] != 1) chain = false;
    level *= choices[i];
    n_tree += level;
    if (n_tree > WM_MAX_T || level > WM_TREE_MAX_CAND)
      return fail(h, WM_ERR_UNSUPPORTED, "candidate tree too large for this engine (at most 16 nodes and 32 paths)");
  }
  CK(cudaSetDevice(h->device));
  CK(cudaStreamSynchronize(h->stream));
  DecModel& m = h->hm;
  if (chain) {
    m.has_tree = 0; m.tree = nullptr; m.n_tree = K + 1;
  } else {
    t.n_tree = (int)n_tree; t.n_cand = (int)level;
    // nodes level by level; the node with in-level index q at depth i has parent q / choices[i] and carries the
    // (q % choices[i])-th best token of head i (tree_indices repeats each level's top-k block)
    int start = 0, prev_start = 0, size = 1;
    for (int i = 0; i <= K; ++i) {
      if (i > 0) size *= choices[i];
      for (int q = 0; q < size; ++q) {
        const int node = start + q;
        t.depth[node] = i;
        t.rank[node] = q % choices[i];
        t.parent[node] = (i == 0) ? -1 : prev_start + q / choices[i];
        t.anc[node] = (1u << node) | (i == 0 ? 0u : t.anc[t.parent[node]]);
      }
      t.topk[i] = choices[i];
      // retrieve_indices[:, i]: path c passes through in-level node c / (n_cand / size)
      for (int c = 0; c < t.n_cand; ++c) t.retrieve[c][i] = start + c / (t.n_cand / size);
      prev_start = start;
      start += size;
    }
    CK(cudaMemcpy(h->tree, &t, sizeof t, cudaMemcpyHostToDevice));
    m.has_tree = 1; m.tree = h->tree; m.n_tree = t.n_tree;
  }
  h->hi.n_tree = m.n_tree;
  for (auto& kv : h->graph_a) cudaGraphExecDestroy(kv.second);
  h->graph_a.clear();
  if (h->graph_b) { cudaGraphExecDestroy(h->graph_b); h->graph_b = nullptr; }
  if (h->graph_tail) { cudaGraphExecDestroy(h->graph_tail); h->graph_tail = nullptr; }
  if (h->wready) return bind_weights(h);   // the stage records of the verify vocabulary projection carry the row count
  CK(cudaMemcpy(h->dm, &m, sizeof m, cudaMemcpyHostToDevice));
  return WM_OK;
}

extern "C" int wm_set_suppress(wm_handle* h, const int32_t* sup, int32_t n_sup, const int32_t* beg, int32_t n_beg) {
  if (!h) return WM_ERR_INVALID;
  if (h->device < 0) return fail(h, WM_ERR_STATE, "layout-only handle");
  CK(cudaSetDevice(h->device));
  std::vector<uint8_t> mask(h->cfg.vocab_size, 0);
  for (int i = 0; i < n_sup; ++i) {
    if (sup[i] < 0 || sup[i] >= h->cfg.vocab_size) return fail(h, WM_ERR_INVALID, "suppress id out of range");
    mask[sup[i]] |= 1;
  }
  for (int i = 0; i < n_beg; ++i) {
    if (beg[i] < 0 || beg[i] >= h->cfg.vocab_size) return fail(h, WM_ERR_INVALID, "begin-suppress id out of range");
    mask[beg[i]] |= 2;
  }
  CK(cudaMemcpy(h->tok_mask, mask.data(), mask.size(), cudaMemcpyHostToDevice));
  return WM_OK;
}

// ---------------------------------------------------------------------------------------------
// frontend + encoder
// ---------------------------------------------------------------------------------------------
static cudaError_t gemm_dispatch(wm_handle* h, const EncGemmArgs& a, cudaStream_t s, int64_t* nl) {
  if (h->enc_gemm_impl == 1) {
    EncGemmArgs b = a;
    b.tile = h->enc_gemm_tile;
    b.pdl = h->enc_pdl;
    return enc_gemm_tc(b, (int)align_up((size_t)a.M, 128), s, nl);
  }
  return enc_gemm(a, s, nl);
}

static int run_encoder(wm_handle* h) {
  const wm_config& c = h->cfg;
  const int d = c.d_model, f = c.ffn_dim, S = h->S;
  cudaStream_t s = h->stream;
  int64_t* nl = &h->launches[1];
  EncGemmArgs a;
  memset(&a, 0, sizeof a);
  // conv1 (k=3, pad 1) as an implicit GEMM over the time-major mel: row t = frames t-1..t+1
  a.A = h->x_tm; a.lda = 80; a.W = wptr<__half>(h, "enc.conv1_w"); a.bias = wptr<float>(h, "enc.conv1_b");
  a.M = kFrames; a.N = d; a.K = 256; a.epi = ENC_EPI_BIAS_GELU_F16; a.out16 = h->h1 + d; a.ldo16 = d;
  CK(gemm_dispatch(h, a, s, nl));
  // conv2 (k=3, stride 2, pad 1): row t = h1 rows 2t..2t+2 ; + GELU + sinusoid positions
  memset(&a, 0, sizeof a);
  a.A = h->h1; a.lda = 2 * d; a.W = wptr<__half>(h, "enc.conv2_w"); a.bias = wptr<float>(h, "enc.conv2_b");
  a.M = S; a.N = d; a.K = 3 * d; a.epi = ENC_EPI_BIAS_GELU_POS_F32; a.out32 = h->x32; a.ldo32 = d;
  a.pos = wptr<float>(h, "enc.pos");
  CK(gemm_dispatch(h, a, s, nl));
  for (int i = 0; i < c.enc_layers; ++i) {
    std::string p = "enc." + std::to_string(i) + ".";
    CK(enc_layernorm(h->x32, wptr<float>(h, p + "ln1_g"), wptr<float>(h, p + "ln1_b"), h->ln16, nullptr, S, d, s, nl, h->enc_pdl != 0));
    memset(&a, 0, sizeof a);
    a.A = h->ln16; a.lda = d; a.W = wptr<__half>(h, p + "qkv_w"); a.bias = wptr<float>(h, p + "qkv_b");
    a.M = S; a.N = 3 * d; a.K = d; a.epi = ENC_EPI_BIAS_F16; a.out16 = h->qkv16; a.ldo16 = 3 * d;
    const bool vt_fused = (h->enc_attn_impl == 1 && h->enc_gemm_impl == 1);   // the wgmma GEMM epilogue writes V^T too
    if (vt_fused) { a.vt = h->vt16; a.vt_col0 = 2 * d; a.vt_ld = h->S_pad; }
    CK(gemm_dispatch(h, a, s, nl));
    if (h->enc_attn_impl == 1) CK(enc_attention_tc(h->qkv16, h->vt16, h->att16, S, h->S_pad, d, c.n_heads, vt_fused, s, nl, h->enc_pdl != 0));
    else CK(enc_attention(h->qkv16, h->att16, S, d, c.n_heads, s, nl));
    memset(&a, 0, sizeof a);
    a.A = h->att16; a.lda = d; a.W = wptr<__half>(h, p + "o_w"); a.bias = wptr<float>(h, p + "o_b");
    a.M = S; a.N = d; a.K = d; a.epi = ENC_EPI_BIAS_RES_F32; a.out32 = h->x32; a.ldo32 = d;
    CK(gemm_dispatch(h, a, s, nl));
    CK(enc_layernorm(h->x32, wptr<float>(h, p + "ln2_g"), wptr<float>(h, p + "ln2_b"), h->ln16, nullptr, S, d, s, nl, h->enc_pdl != 0));
    memset(&a, 0, sizeof a);
    a.A = h->ln16; a.lda = d; a.W = wptr<__half>(h, p + "fc1_w"); a.bias = wptr<float>(h, p + "fc1_b");
    a.M = S; a.N = f; a.K = d; a.epi = ENC_EPI_BIAS_GELU_F16; a.out16 = h->ffn16; a.ldo16 = f;
    CK(gemm_dispatch(h, a, s, nl));
    memset(&a, 0, sizeof a);
    a.A = h->ffn16; a.lda = f; a.W = wptr<__half>(h, p + "fc2_w"); a.bias = wptr<float>(h, p + "fc2_b");
    a.M = S; a.N = d; a.K = f; a.epi = ENC_EPI_BIAS_RES_F32; a.out32 = h->x32; a.ldo32 = d;
    CK(gemm_dispatch(h, a, s, nl));
  }
  CK(enc_layernorm(h->x32, wptr<float>(h, "enc.lnf_g"), wptr<float>(h, "enc.lnf_b"), h->enc16, h->enc32, S, d, s, nl, h->enc_pdl != 0));
  // cross-attention K/V of every decoder layer, re-laid out per head for the decode kernels (cross_k / cross_v)
  for (int i = 0; i < h->n_dec; ++i) {
    std::string p = "dec." + std::to_string(i) + ".";
    memset(&a, 0, sizeof a);
    a.A = h->enc16; a.lda = d; a.W = wptr<__half>(h, p + "ckv_w"); a.bias = wptr<float>(h, p + "ckv_b");
    a.M = S; a.N = 2 * d; a.K = d; a.epi = ENC_EPI_BIAS_F16; a.out16 = h->qkv16; a.ldo16 = 2 * d;   // (scratch: [pos][k | v])
    if (h->enc_gemm_impl == 1 && d % 64 == 0) {
      // the wgmma GEMM's epilogue writes the decode layout itself (pad entries stay zero from the allocation)
      a.ck = h->cross_k[i]; a.cv = h->cross_v[i]; a.kv_spad = h->S_pad;
      CK(gemm_dispatch(h, a, s, nl));
    } else {
      CK(gemm_dispatch(h, a, s, nl));
      CK(dec_relayout_cross_kv(h->qkv16, h->cross_k[i], h->cross_v[i], S, h->S_pad, d, h->cfg.n_heads, s, nl));
    }
  }
  return WM_OK;
}

static int finish_encode(wm_handle* h) {
  CK(cudaEventRecord(h->ev[2], h->stream));
  CK(cudaStreamSynchronize(h->stream));
  float t0 = 0, t1 = 0;
  CK(cudaEventElapsedTime(&t0, h->ev[0], h->ev[1]));
  CK(cudaEventElapsedTime(&t1, h->ev[1], h->ev[2]));
  h->ms[0] = t0; h->ms[1] = t1;
  h->encoded = true;
  return WM_OK;
}

extern "C" int wm_encode_pcm(wm_handle* h, const float* pcm, int32_t n) {
  if (!h || n < 0 || (!pcm && n > 0)) return WM_ERR_INVALID;   // an empty clip (n == 0) is valid: 30 s of silence
  if (!h->wready) return fail(h, WM_ERR_STATE, "weights not loaded");
  CK(cudaSetDevice(h->device));
  h->launches[0] = h->launches[1] = 0;
  const int m = n < kSamples ? n : kSamples;
  if (m > 0) memcpy(h->h_stage, pcm, (size_t)m * sizeof(float));
  if (m < kSamples) memset(h->h_stage + m, 0, (size_t)(kSamples - m) * sizeof(float));
  CK(cudaEventRecord(h->ev[0], h->stream));
  CK(cudaMemcpyAsync(h->pcm, h->h_stage, (size_t)kSamples * sizeof(float), cudaMemcpyHostToDevice, h->stream));
  CK(mel_forward(h->pcm, h->melfb, h->mel32, h->x_tm, h->gmax, h->stream, &h->launches[0]));
  CK(cudaEventRecord(h->ev[1], h->stream));
  int r = run_encoder(h);
  if (r != WM_OK) return r;
  return finish_encode(h);
}

// Device twin of wm_encode_pcm: the window is copied into the handle's PCM buffer and the rest of the buffer is zeroed,
// so the mel kernels see exactly the samples wm_encode_pcm stages from the host.
extern "C" int wm_encode_pcm_device(wm_handle* h, const float* pcm_dev, int32_t n, void* producer_stream) {
  if (!h || n < 0 || n > kSamples || (!pcm_dev && n > 0)) return WM_ERR_INVALID;
  if (!h->wready) return fail(h, WM_ERR_STATE, "weights not loaded");
  CK(cudaSetDevice(h->device));
  h->launches[0] = h->launches[1] = 0;
  CK(cudaEventRecord(h->ev[5], reinterpret_cast<cudaStream_t>(producer_stream)));
  CK(cudaStreamWaitEvent(h->stream, h->ev[5], 0));
  CK(cudaEventRecord(h->ev[0], h->stream));
  if (n > 0) CK(cudaMemcpyAsync(h->pcm, pcm_dev, (size_t)n * sizeof(float), cudaMemcpyDeviceToDevice, h->stream));
  if (n < kSamples) CK(cudaMemsetAsync(h->pcm + n, 0, (size_t)(kSamples - n) * sizeof(float), h->stream));
  CK(mel_forward(h->pcm, h->melfb, h->mel32, h->x_tm, h->gmax, h->stream, &h->launches[0]));
  CK(cudaEventRecord(h->ev[1], h->stream));
  int r = run_encoder(h);
  if (r != WM_OK) return r;
  return finish_encode(h);
}

extern "C" int wm_resample(wm_handle* h, const float* in_dev, int64_t n_in, int32_t orig_hz, int32_t new_hz,
                           float* out_dev, int64_t out_cap, int64_t* n_out, void* stream) {
  if (!h || !n_out || n_in < 0 || (n_in > 0 && (!in_dev || !out_dev)) || orig_hz <= 0 || new_hz <= 0 || n_in >= (int64_t(1) << 40))
    return WM_ERR_INVALID;
  if (h->device < 0) return fail(h, WM_ERR_STATE, "layout-only handle has no device");
  CK(cudaSetDevice(h->device));
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  if (orig_hz == new_hz) {
    *n_out = n_in;
    if (out_cap < n_in) return fail(h, WM_ERR_INVALID, "out_cap is smaller than the resampled length");
    if (n_in > 0) CK(cudaMemcpyAsync(out_dev, in_dev, (size_t)n_in * sizeof(float), cudaMemcpyDeviceToDevice, s));
    return WM_OK;
  }
  auto key = std::make_pair((int)orig_hz, (int)new_hz);
  auto it = h->resamplers.find(key);
  if (it == h->resamplers.end()) {
    wm_handle::Resampler r;
    if (!resample_build_table(orig_hz, new_hz, r.t))
      return fail(h, WM_ERR_UNSUPPORTED, "rates too large after dividing by their gcd");
    r.T = resample_block_outputs(r.t, &r.smem);
    if (r.T == 0) return fail(h, WM_ERR_UNSUPPORTED, "downsampling ratio too large for the staged input tile");
    const ResampleTable& t = r.t;
    std::vector<float> tt((size_t)t.max_taps * t.nw);
    for (int p = 0; p < t.nw; ++p)
      for (int j = 0; j < t.max_taps; ++j) tt[(size_t)j * t.nw + p] = t.taps[(size_t)p * t.max_taps + j];
    std::vector<int2> sup((size_t)t.nw);
    for (int p = 0; p < t.nw; ++p) sup[p] = make_int2(t.lo[p] - t.width, t.n[p]);
    CK(dalloc(&r.taps, tt.size()));
    CK(dalloc(&r.sup, sup.size()));
    CK(cudaMemcpy(r.taps, tt.data(), tt.size() * sizeof(float), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(r.sup, sup.data(), sup.size() * sizeof(int2), cudaMemcpyHostToDevice));
    it = h->resamplers.emplace(key, r).first;
  }
  const wm_handle::Resampler& r = it->second;
  const int64_t m = resample_out_len(n_in, r.t);
  *n_out = m;
  if (out_cap < m) return fail(h, WM_ERR_INVALID, "out_cap is smaller than the resampled length");
  CK(resample_launch(in_dev, n_in, out_dev, m, r.taps, r.sup, r.t, r.T, r.smem, s));
  return WM_OK;
}

extern "C" int wm_resample_taps(int32_t orig_hz, int32_t new_hz, float* taps, int32_t* lo, int32_t* n_taps, int64_t cap,
                                int32_t* info4) {
  if (!info4) return WM_ERR_INVALID;
  ResampleTable t;
  if (!resample_build_table(orig_hz, new_hz, t)) return WM_ERR_INVALID;
  info4[0] = t.orig; info4[1] = t.nw; info4[2] = t.width; info4[3] = t.max_taps;
  if (!taps && !lo && !n_taps) return WM_OK;
  if (!taps || !lo || !n_taps || cap < (int64_t)t.taps.size()) return WM_ERR_INVALID;
  std::copy(t.taps.begin(), t.taps.end(), taps);
  for (int p = 0; p < t.nw; ++p) { lo[p] = t.lo[p]; n_taps[p] = t.n[p]; }
  return WM_OK;
}

extern "C" int wm_encode_mel_device(wm_handle* h, const float* mel_dev, void* producer_stream) {
  if (!h || !mel_dev) return WM_ERR_INVALID;
  if (!h->wready) return fail(h, WM_ERR_STATE, "weights not loaded");
  CK(cudaSetDevice(h->device));
  h->launches[0] = h->launches[1] = 0;
  // order after the work that produced the features on the caller's stream
  CK(cudaEventRecord(h->ev[5], reinterpret_cast<cudaStream_t>(producer_stream)));
  CK(cudaStreamWaitEvent(h->stream, h->ev[5], 0));
  CK(cudaEventRecord(h->ev[0], h->stream));
  CK(cudaMemcpyAsync(h->mel32, mel_dev, (size_t)80 * kFrames * sizeof(float), cudaMemcpyDeviceToDevice, h->stream));
  CK(mel_to_time_major(h->mel32, h->x_tm, h->stream, &h->launches[0]));
  CK(cudaEventRecord(h->ev[1], h->stream));
  int r = run_encoder(h);
  if (r != WM_OK) return r;
  return finish_encode(h);
}

extern "C" int wm_encode_mel(wm_handle* h, const float* mel) {
  if (!h || !mel) return WM_ERR_INVALID;
  if (!h->wready) return fail(h, WM_ERR_STATE, "weights not loaded");
  CK(cudaSetDevice(h->device));
  h->launches[0] = h->launches[1] = 0;
  memcpy(h->h_stage, mel, (size_t)80 * kFrames * sizeof(float));
  CK(cudaEventRecord(h->ev[0], h->stream));
  CK(cudaMemcpyAsync(h->mel32, h->h_stage, (size_t)80 * kFrames * sizeof(float), cudaMemcpyHostToDevice, h->stream));
  CK(mel_to_time_major(h->mel32, h->x_tm, h->stream, &h->launches[0]));
  CK(cudaEventRecord(h->ev[1], h->stream));
  int r = run_encoder(h);
  if (r != WM_OK) return r;
  return finish_encode(h);
}

// ---------------------------------------------------------------------------------------------
// decode loop
// ---------------------------------------------------------------------------------------------
static int get_graph(wm_handle* h, int phase, int T, cudaGraphExec_t* out, int64_t* n_launch) {
  if (phase == 2 && h->graph_b) { *out = h->graph_b; *n_launch = h->launches_b; return WM_OK; }
  if (phase == 1 && h->graph_tail) { *out = h->graph_tail; *n_launch = h->launches_tail; return WM_OK; }
  if (phase == 0) {
    auto it = h->graph_a.find(T);
    if (it != h->graph_a.end()) { *out = it->second; *n_launch = h->launches_a[T]; return WM_OK; }
  }
  cudaGraph_t g;
  int64_t nl = 0;
  CK(cudaStreamBeginCapture(h->stream, cudaStreamCaptureModeThreadLocal));
  cudaError_t e = dec_enqueue_phase(h->dm, h->hi, phase, T, h->stream, &nl);
  cudaError_t e2 = cudaStreamEndCapture(h->stream, &g);
  CK(e);
  CK(e2);
  cudaGraphExec_t ge;
  CK(cudaGraphInstantiate(&ge, g, 0));
  CK(cudaGraphDestroy(g));
  if (phase == 2) { h->graph_b = ge; h->launches_b = nl; }
  else if (phase == 1) { h->graph_tail = ge; h->launches_tail = nl; }
  else { h->graph_a[T] = ge; h->launches_a[T] = nl; }
  *out = ge; *n_launch = nl;
  return WM_OK;
}

extern "C" int wm_generate(wm_handle* h, const int32_t* prompt, int32_t n_prompt, const wm_gen_params* gp,
                           int32_t* out_ids, int32_t* n_out, int32_t* accept_lens, int32_t* n_iter) {
  if (!h || !prompt || !gp || !out_ids || !n_out) return WM_ERR_INVALID;
  if (!h->encoded) return fail(h, WM_ERR_STATE, "wm_encode_* must be called before wm_generate");
  const int K = h->cfg.medusa_num_heads;
  if (n_prompt < 1 || n_prompt + K + 2 > gp->max_length) return fail(h, WM_ERR_INVALID, "prompt length must be in [1, max_length - K - 2)");
  if (gp->max_length > h->cfg.max_target_positions) return fail(h, WM_ERR_INVALID, "max_length exceeds max_target_positions");
  if (gp->temperature < 0.f) return fail(h, WM_ERR_INVALID, "temperature must be >= 0");
  for (int i = 0; i < n_prompt; ++i)
    if (prompt[i] < 0 || prompt[i] >= h->cfg.vocab_size) return fail(h, WM_ERR_INVALID, "prompt id out of range");
  CK(cudaSetDevice(h->device));
  cudaStream_t s = h->stream;
  h->launches[2] = 0;

  // EOS exponential-decay penalty table (HF logits_process.py:1742-1772): indexed by cur_len
  if (gp->penalty_start != h->last_pen_start || gp->penalty_factor != h->last_pen_factor || n_prompt != h->last_pen_prompt) {
    // (pinned staging, stream-ordered upload: the previous call's copy completed before that call returned)
    const int ntab = WM_MAX_POS + 32;
    for (int L = 0; L < ntab; ++L) h->h_pen[L] = 0.f;
    if (gp->penalty_start >= 0) {
      const int reg = gp->penalty_start + n_prompt;
      for (int L = 0; L < ntab; ++L)
        if (L > reg) h->h_pen[L] = (float)(std::pow((double)gp->penalty_factor, (double)(L - reg)) - 1.0);
    }
    CK(cudaMemcpyAsync(h->pen_tab, h->h_pen, (size_t)ntab * sizeof(float), cudaMemcpyHostToDevice, s));
    h->last_pen_start = gp->penalty_start; h->last_pen_factor = gp->penalty_factor; h->last_pen_prompt = n_prompt;
  }
  // loop state
  {
    DecState& hs = *h->h_init;   // pinned: the upload is asynchronous, no host synchronisation before the first launch
    memset(&hs, 0, sizeof hs);
    hs.L = n_prompt; hs.kv_len = 0; hs.done = 0; hs.n_iter = 0; hs.max_iters = gp->max_iters; hs.need_a = 1;
    hs.max_length = gp->max_length; hs.eos = gp->eos_token_id; hs.pad = gp->pad_token_id;
    hs.begin_index = gp->begin_index; hs.temperature = gp->temperature; hs.post_thr = gp->posterior_threshold;
    hs.post_alpha = gp->posterior_alpha;
    hs.tree_attn = (h->hm.has_tree && gp->tree_attention) ? 1 : 0;
    for (int i = 0; i < n_prompt; ++i) hs.ids[i] = prompt[i];
    // reference stop rule evaluated before the first iteration is never true for sane inputs; the
    // loop always runs at least once (model.py:635).
    CK(cudaMemcpyAsync(h->st, &hs, sizeof hs, cudaMemcpyHostToDevice, s));
    CK(cudaMemsetAsync(h->bar, 0, 8 * sizeof(unsigned int), s));
    CK(cudaMemsetAsync(h->hm.cross_cnt, 0, (size_t)h->cfg.n_heads * sizeof(unsigned int), s));
    CK(cudaMemsetAsync(h->hm.gemm_cnt, 0, (size_t)h->n_sm * sizeof(unsigned int), s));
  }
  // Long prompts (decoder_input_ids beyond the 16 rows of a stage tile): the leading tokens are cached by prefill
  // launches -- sweep A over 16-token chunks, no candidates / verify -- before the loop proper starts on the rest.
  int n_tail = n_prompt;     // rows of the first real iteration's sweep A
  {
    int pos = 0;
    while (n_prompt - pos > WM_MAX_T) {
      DecState& hs = *h->h_init;
      hs.L = pos + WM_MAX_T; hs.kv_len = pos; hs.need_a = 1; hs.prefill = 1;
      CK(cudaMemcpyAsync(h->st, &hs, 64, cudaMemcpyHostToDevice, s));   // the 16 header words (L .. tree_attn)
      if (h->decode_mode == 0) {
        cudaGraphExec_t g = nullptr; int64_t nl = 0; int r;
        if ((r = get_graph(h, 0, WM_MAX_T, &g, &nl)) != WM_OK) return r;
        CK(cudaGraphLaunch(g, s));
        h->launches[2] += nl;
      } else if (h->decode_mode == 1) {
        CK(dec_launch_iteration(h->dm, h->hi, s));
        h->launches[2] += 1;
      } else {
        CK(dec_launch_iteration_ring(h->dm, h->hi, false, s));
        h->launches[2] += 1;
      }
      CK(cudaStreamSynchronize(s));   // the pinned header is rewritten for the next chunk
      pos += WM_MAX_T;
    }
    if (pos > 0) {
      DecState& hs = *h->h_init;
      hs.L = n_prompt; hs.kv_len = pos; hs.need_a = 1; hs.prefill = 0;
      CK(cudaMemcpyAsync(h->st, &hs, 64, cudaMemcpyHostToDevice, s));
      n_tail = n_prompt - pos;
    }
  }
  cudaGraphExec_t gA1 = nullptr, gAp = nullptr, gT = nullptr, gB = nullptr;
  int64_t nA1 = 0, nAp = 0, nT = 0, nB = 0;
  if (h->decode_mode == 0) {
    int r;
    if ((r = get_graph(h, 0, n_tail, &gAp, &nAp)) != WM_OK) return r;
    if ((r = get_graph(h, 0, 1, &gA1, &nA1)) != WM_OK) return r;
    if ((r = get_graph(h, 1, 1, &gT, &nT)) != WM_OK) return r;
    if ((r = get_graph(h, 2, h->hm.n_tree, &gB, &nB)) != WM_OK) return r;
  }
  CK(cudaEventRecord(h->ev[3], s));
  int L = n_prompt, iters = 0, done = 0;
  while (!done) {
    // iterations that are certainly needed unless EOS shows up: each adds at most K+1 tokens and
    // the loop ends once L + K >= max_length
    int lb = (gp->max_length - K - L + K) / (K + 1);
    if (lb < 1) lb = 1;
    if (lb > 32) lb = 32;
    if (gp->max_iters > 0 && lb > gp->max_iters - iters) lb = gp->max_iters - iters;
    if (lb < 1) lb = 1;
    for (int i = 0; i < lb; ++i) {
      if (h->decode_mode == 0) {
        const bool first = (iters + i == 0);
        // sweep A kernels return immediately unless the state says the newest token is uncached
        CK(cudaGraphLaunch(first ? gAp : gA1, s));
        CK(cudaGraphLaunch(gT, s));
        CK(cudaGraphLaunch(gB, s));
        h->launches[2] += (first ? nAp : nA1) + nT + nB;
      } else if (h->decode_mode == 1) {
        CK(dec_launch_iteration(h->dm, h->hi, s));
        h->launches[2] += 1;
      } else {
        CK(dec_launch_iteration_ring(h->dm, h->hi, h->hm.prof != nullptr, s));
        h->launches[2] += 1;
      }
    }
    CK(cudaMemcpyAsync(h->h_state, h->st, 16 * sizeof(int), cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    L = h->h_state[0];
    done = h->h_state[2];
    iters = h->h_state[3];
  }
  CK(cudaEventRecord(h->ev[4], s));
  CK(cudaStreamSynchronize(s));
  float tms = 0;
  CK(cudaEventElapsedTime(&tms, h->ev[3], h->ev[4]));
  h->ms[2] = tms;
  // read back ids / accept lengths
  std::vector<int> ids(L);
  CK(cudaMemcpy(ids.data(), reinterpret_cast<const char*>(h->st) + offsetof(DecState, ids), (size_t)L * sizeof(int),
                cudaMemcpyDeviceToHost));
  // post-EOS fill (model.py:798-810)
  for (int i = 0; i < L; ++i)
    if (ids[i] == gp->eos_token_id) {
      for (int j = i + 1; j < L; ++j) ids[j] = gp->eos_token_id;
      break;
    }
  for (int i = 0; i < L; ++i) out_ids[i] = ids[i];
  *n_out = L;
  if (n_iter) *n_iter = iters;
  if (accept_lens && iters > 0)
    CK(cudaMemcpy(accept_lens, reinterpret_cast<const char*>(h->st) + offsetof(DecState, accept_hist),
                  (size_t)iters * sizeof(int), cudaMemcpyDeviceToHost));
  return WM_OK;
}

// Stacked head logits of a teacher-forced decoder pass (reference WhisperMedusaModel.forward, model.py:1223-1347:
// `logits` [K+1, batch 1, T, V]).  The loop kernels only ever need the heads at the LAST position, so this utility
// entry runs the prefix ids[0..t) through sweep A + the candidate tail for t = 1..T (O(T^2) rows, T <= 16) and
// collects the K+1 rows of each: out[(k * T + t) * V + v].  Raw logits, no processors.
extern "C" int wm_forward(wm_handle* h, const int32_t* ids, int32_t n_ids, float* out) {
  if (!h || !ids || !out) return WM_ERR_INVALID;
  if (!h->encoded) return fail(h, WM_ERR_STATE, "wm_encode_* must be called before wm_forward");
  if (n_ids < 1 || n_ids > WM_MAX_T) return fail(h, WM_ERR_INVALID, "wm_forward takes 1..16 decoder ids");
  for (int i = 0; i < n_ids; ++i)
    if (ids[i] < 0 || ids[i] >= h->cfg.vocab_size) return fail(h, WM_ERR_INVALID, "decoder id out of range");
  CK(cudaSetDevice(h->device));
  cudaStream_t s = h->stream;
  const int K = h->cfg.medusa_num_heads;
  const size_t V = (size_t)h->cfg.vocab_size;
  for (int t = 1; t <= n_ids; ++t) {
    DecState& hs = *h->h_init;
    memset(&hs, 0, sizeof hs);
    hs.L = t; hs.need_a = 1; hs.max_length = h->cfg.max_target_positions; hs.eos = -1; hs.pad = -1; hs.begin_index = -1;
    hs.temperature = 1.f; hs.post_thr = 0.09f; hs.post_alpha = 0.3f;
    for (int i = 0; i < t; ++i) hs.ids[i] = ids[i];
    CK(cudaMemcpyAsync(h->st, &hs, sizeof hs, cudaMemcpyHostToDevice, s));
    CK(cudaMemsetAsync(h->hm.cross_cnt, 0, (size_t)h->cfg.n_heads * sizeof(unsigned int), s));
    CK(cudaMemsetAsync(h->hm.gemm_cnt, 0, (size_t)h->n_sm * sizeof(unsigned int), s));
    if (h->decode_mode == 2) {
      // ring kernel (any decode grid): one speculative iteration = sweep A over the prefix, the candidate tail (whose
      // K+1 logit rows are what we want) and a verify pass whose results are simply not read
      CK(cudaMemsetAsync(h->bar, 0, 8 * sizeof(unsigned int), s));
      CK(dec_launch_iteration_ring(h->dm, h->hi, false, s));
    } else {
      if (!simple_modes_fit(h)) return fail(h, WM_ERR_UNSUPPORTED, "wm_forward: this decode grid needs the ring kernel (decode_mode 2)");
      cudaGraphExec_t gA = nullptr, gT = nullptr;
      int64_t nA = 0, nT = 0;
      int r;
      if ((r = get_graph(h, 0, t, &gA, &nA)) != WM_OK) return r;
      if ((r = get_graph(h, 1, 1, &gT, &nT)) != WM_OK) return r;
      CK(cudaGraphLaunch(gA, s));
      CK(cudaGraphLaunch(gT, s));
    }
    for (int k = 0; k <= K; ++k)
      CK(cudaMemcpyAsync(out + ((size_t)k * n_ids + (t - 1)) * V, h->hm.logits_a + (size_t)k * V, V * sizeof(float),
                         cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));   // h_init is rewritten by the next prefix
  }
  return WM_OK;
}

// ---------------------------------------------------------------------------------------------
// taps
// ---------------------------------------------------------------------------------------------
extern "C" int wm_get_mel(wm_handle* h, float* out) {
  if (!h || !out) return WM_ERR_INVALID;
  CK(cudaSetDevice(h->device));
  CK(cudaMemcpy(out, h->mel32, (size_t)80 * kFrames * sizeof(float), cudaMemcpyDeviceToHost));
  return WM_OK;
}
extern "C" int wm_get_encoder_out(wm_handle* h, float* out) {
  if (!h || !out) return WM_ERR_INVALID;
  if (!h->encoded) return fail(h, WM_ERR_STATE, "nothing encoded yet");
  CK(cudaSetDevice(h->device));
  CK(cudaMemcpy(out, h->enc32, (size_t)h->S * h->cfg.d_model * sizeof(float), cudaMemcpyDeviceToHost));
  return WM_OK;
}
extern "C" int wm_last_logits(wm_handle* h, int32_t which, float* out) {
  if (!h || !out || which < 0 || which > 1) return WM_ERR_INVALID;
  CK(cudaSetDevice(h->device));
  const size_t n = (size_t)(h->cfg.medusa_num_heads + 1) * h->cfg.vocab_size;
  CK(cudaMemcpy(out, which == 0 ? h->hm.logits_a : h->hm.logits_b, n * sizeof(float), cudaMemcpyDeviceToHost));
  return WM_OK;
}
extern "C" double wm_last_ms(wm_handle* h, int32_t what) { return (h && what >= 0 && what < 3) ? h->ms[what] : -1.0; }
extern "C" int64_t wm_last_launches(wm_handle* h, int32_t what) {
  if (!h) return -1;
  if (what == 1) return h->launches[0] + h->launches[1];
  if (what == 2) return h->launches[2];
  return -1;
}
extern "C" int wm_decode_cluster(wm_handle* h) { return h ? h->hi.cluster : 0; }
extern "C" int wm_set_option(wm_handle* h, const char* key, int32_t value) {
  if (!h || !key) return WM_ERR_INVALID;
  const std::string k(key);
  if (k == "decode_mode") {
    if (value < 0 || value > 2) return fail(h, WM_ERR_INVALID, "decode_mode must be 0, 1 or 2");
    if (value < 2 && !simple_modes_fit(h)) return fail(h, WM_ERR_UNSUPPORTED, "decode modes 0 / 1 need more CTAs for the vocabulary projection");
    if (value == 2 && !h->hi.smem_ring) return fail(h, WM_ERR_UNSUPPORTED, "the ring kernel is not instantiated for this decoder width");
    h->decode_mode = value;
    return WM_OK;
  }
  if (k == "decode_ctas") {
    // Size of the decode grid.  Default = every SM (lowest latency for one stream).  Several handles that share one
    // weight blob and use 1/S of the SMs each run S streams CONCURRENTLY (their cooperative kernels are co-resident):
    // a stage chain is latency-bound, so S partitions move S times the bytes in about the same time (DESIGN.md 7).
    if (value < (int)(h->cfg.ffn_dim / h->cfg.d_model) || value > h->n_sm) return fail(h, WM_ERR_INVALID, "decode_ctas out of range");
    CK(cudaSetDevice(h->device));
    CK(cudaStreamSynchronize(h->stream));
    h->n_cta = value;
    h->hi.n_sm = value;
    h->hi.cluster = dec_ring_cluster_size(h->hi, h->n_sm);
    set_decode_split(h);
    for (auto& kv : h->graph_a) cudaGraphExecDestroy(kv.second);
    h->graph_a.clear();
    if (h->graph_b) { cudaGraphExecDestroy(h->graph_b); h->graph_b = nullptr; }
    if (h->graph_tail) { cudaGraphExecDestroy(h->graph_tail); h->graph_tail = nullptr; }
    if (!simple_modes_fit(h)) {
      if (!h->hi.smem_ring) return fail(h, WM_ERR_UNSUPPORTED, "too few CTAs for this model without the ring kernel");
      h->decode_mode = 2;
    }
    if (h->wready) return bind_weights(h);   // the per-CTA stage / chunk tables depend on the grid
    CK(cudaMemcpy(h->dm, &h->hm, sizeof(DecModel), cudaMemcpyHostToDevice));
    return WM_OK;
  }
  if (k == "profile") {
    // stage timeline of the persistent ring kernel (debug): buffer [2][n_instr][3] u64
    CK(cudaSetDevice(h->device));
    if (value && !h->prof) CK(dalloc(&h->prof, (size_t)2 * h->hm.prog_off[3] * 16));
    h->hm.prof = value ? h->prof : nullptr;
    CK(cudaMemcpy(h->dm, &h->hm, sizeof(DecModel), cudaMemcpyHostToDevice));
    return WM_OK;
  }
  if (k == "enc_attn") {
    if (value == 1 && !h->attn_tc_ok) return fail(h, WM_ERR_UNSUPPORTED, "wgmma attention unavailable (cuTensorMapEncodeTiled not found)");
    if (value < 0 || value > 1) return fail(h, WM_ERR_INVALID, "enc_attn must be 0 (mma.sync) or 1 (wgmma)");
    h->enc_attn_impl = value;
    return WM_OK;
  }
  if (k == "enc_pdl") {
    if (value < 0 || value > 1) return fail(h, WM_ERR_INVALID, "enc_pdl must be 0 or 1");
    h->enc_pdl = value;
    return WM_OK;
  }
  if (k == "enc_gemm") {
    if (value == 1 && !h->tc_ok) return fail(h, WM_ERR_UNSUPPORTED, "wgmma GEMM unavailable (cuTensorMapEncodeTiled not found)");
    if (value < 0 || value > 2)
      return fail(h, WM_ERR_INVALID, "enc_gemm must be 0 (mma.sync), 1 (wgmma) or 2 (wgmma, 128 x 128 tiles only)");
    if (value >= 1 && !h->tc_ok) return fail(h, WM_ERR_UNSUPPORTED, "wgmma GEMM unavailable (cuTensorMapEncodeTiled not found)");
    h->enc_gemm_impl = value ? 1 : 0;
    h->enc_gemm_tile = value == 2 ? 1 : 0;
    return WM_OK;
  }
  return fail(h, WM_ERR_INVALID, "unknown option " + k);
}
// Stage timeline of the last persistent-ring iteration (option "profile" = 1): rows of 24 int64
// {stage, mode, layer, body_ns(last cta), barrier_ns(last cta), raw[16] of CTA 0, 0, 0, 0}; raw[k] is a
// timestamp relative to the stage begin (or a flag), see dec_iteration_ring_kernel
extern "C" int wm_get_stage_profile(wm_handle* h, int64_t* out, int32_t cap_rows, int32_t* n_rows) {
  if (!h || !out || !n_rows) return WM_ERR_INVALID;
  if (!h->prof) return fail(h, WM_ERR_STATE, "profiling is off (wm_set_option(h, \"profile\", 1))");
  CK(cudaSetDevice(h->device));
  const int n = h->hm.prog_off[3];
  std::vector<unsigned long long> raw((size_t)2 * n * 16);
  std::vector<int> prog((size_t)n * 3);
  CK(cudaMemcpy(raw.data(), h->prof, raw.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(prog.data(), h->prog, prog.size() * sizeof(int), cudaMemcpyDeviceToHost));
  int rows = 0;
  for (int i = 0; i < n && rows < cap_rows; ++i) {
    const unsigned long long* a = &raw[(size_t)i * 16];
    const unsigned long long* b = &raw[((size_t)n + i) * 16];
    if (a[0] == 0) continue;   // stage never executed (sweep A skipped)
    int64_t* o = out + (size_t)rows * 24;
    o[0] = prog[i * 3]; o[1] = prog[i * 3 + 1]; o[2] = prog[i * 3 + 2];
    o[3] = (int64_t)(b[1] - b[0]); o[4] = (int64_t)(b[2] - b[1]);
    for (int k = 0; k < 16; ++k) {
      const bool flag = (k == 11 || k == 12);
      o[5 + k] = flag ? (int64_t)a[k] : (a[k] >= a[0] ? (int64_t)(a[k] - a[0]) : -1);
    }
    o[21] = o[22] = o[23] = 0;
    ++rows;
  }
  *n_rows = rows;
  return WM_OK;
}
extern "C" int wm_set_decode_mode(wm_handle* h, int32_t mode) {
  if (!h) return WM_ERR_INVALID;
  int prev = h->decode_mode;
  if (mode >= 0 && mode <= 2 && wm_set_option(h, "decode_mode", mode) != WM_OK) return WM_ERR_UNSUPPORTED;
  return prev;
}
// Device address of the packed weights (so that further handles on the same GPU can wm_adopt_weights them: one copy
// of the 3.1 GB blob serves every concurrent stream).
extern "C" int wm_enc_gemm_tile(int32_t M, int32_t N, int32_t K, int32_t fp16_out, int32_t n_sm, int32_t* out3) {
  if (!out3 || M <= 0 || N <= 0 || K <= 0 || N % 128 != 0) return WM_ERR_INVALID;
  int t[3];
  enc_gemm_tc_tile(M, N, K, fp16_out != 0, n_sm, t);
  out3[0] = t[0]; out3[1] = t[1]; out3[2] = t[2];
  return WM_OK;
}
extern "C" void* wm_weights_device_ptr(wm_handle* h) { return (h && h->wready) ? (void*)h->wdev : nullptr; }
