/*
 * whisper_medusa_b200 -- C ABI of the H100-native Whisper-Medusa decode path.
 *
 * The reference (aiola-lab/whisper-medusa) is pure Python and has no FFI of its own; the
 * boundary it exposes for this path is the Python surface of
 *   whisper_medusa/models/model.py:213  class WhisperMedusaModel
 *     :265-291   from_pretrained(path)          -> wm_create + wm_tensor_info/wm_load_weights
 *     :1419-1449 generate(input_features, ...)  -> wm_encode_mel / wm_encode_pcm + wm_generate
 *     :1223-1347 forward(...).logits            -> wm_last_logits (parity tap)
 * Each entry point below names the reference lines it replaces.  The Python host
 * (whisper_medusa_b200/model.py) binds exactly these symbols with ctypes; INTEGRATION.md shows
 * the stub a reference maintainer would add.
 *
 * Conventions: plain pointers and sizes only; the caller owns every host buffer; the handle
 * owns all device memory (unless weights are adopted with wm_adopt_weights); one handle =
 * one CUDA device + one stream; a handle is not thread-safe, distinct handles are
 * independent.  Every function returns 0 on success or a negative wm_status.
 */
#ifndef WHISPER_MEDUSA_B200_H_
#define WHISPER_MEDUSA_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct wm_handle wm_handle;

typedef enum wm_status {
  WM_OK = 0,
  WM_ERR_INVALID = -1,      /* bad argument / unsupported configuration            */
  WM_ERR_CUDA = -2,         /* a CUDA runtime call failed (see wm_last_error)      */
  WM_ERR_STATE = -3,        /* call order violated (e.g. generate before encode)   */
  WM_ERR_UNSUPPORTED = -4,  /* valid in the reference but not implemented here     */
  WM_ERR_NOMEM = -5
} wm_status;

/* Shape of the model: the fields of MedusaConfig the path reads
 * (reference whisper_medusa/utils/config_and_args.py:17-62). */
typedef struct wm_config {
  int32_t vocab_size;
  int32_t d_model;
  int32_t n_heads;            /* encoder == decoder attention heads; head_dim must be 64 */
  int32_t ffn_dim;
  int32_t enc_layers;
  int32_t dec_layers;
  int32_t n_mels;             /* 80 */
  int32_t max_source_positions; /* 1500 */
  int32_t max_target_positions; /* 448 */
  int32_t medusa_num_heads;   /* K */
  int32_t medusa_block;       /* 0 = "base_head" (Medusa-Linear), 1 = "medusa_block" */
} wm_config;

/* What _medusa_greedy_search reads from the generation config and kwargs
 * (reference model.py:404-835; medusa_utils.py:14-18). */
typedef struct wm_gen_params {
  int32_t max_length;          /* generation_config.max_length (448) */
  int32_t eos_token_id;
  int32_t pad_token_id;
  int32_t begin_index;         /* SuppressTokensAtBegin begin_index = len(prompt) */
  float temperature;           /* generate() forces 1.0 (model.py:1878-1881); 0 = exact-match acceptance */
  float posterior_threshold;   /* 0.09 */
  float posterior_alpha;       /* 0.3  */
  int32_t penalty_start;       /* ExponentialDecayLengthPenalty start_index, <0 = off */
  float penalty_factor;
  int32_t max_iters;           /* 0 = run to completion; >0 = stop after this many iterations */
  int32_t tree_attention;      /* branching medusa_choices only: 0 = reference behaviour (verify rows attend causally over
                                * cache order; medusa_attn_mask is built but never applied, model.py / medusa_utils.py:329-358),
                                * 1 = every tree node attends to its ancestors only (true tree attention) */
} wm_gen_params;

/* ---- lifetime ------------------------------------------------------------------------ */
int wm_create(const wm_config* cfg, int device, wm_handle** out);
int wm_destroy(wm_handle* h);
const char* wm_strerror(int status);
const char* wm_last_error(wm_handle* h);

/* ---- weights (replaces from_pretrained, model.py:265-291) ----------------------------- */
/* The packed blob layout is defined by the library; the host packer asks where each engine
 * tensor lives.  dtype: 0 = fp16, 1 = fp32.  Names are listed by wm_tensor_name(0..count-1). */
int wm_tensor_count(wm_handle* h);
const char* wm_tensor_name(wm_handle* h, int index);
int wm_tensor_info(wm_handle* h, const char* name, size_t* offset, size_t* nbytes, int32_t* dtype);
size_t wm_weights_nbytes(wm_handle* h);
/* Copy a packed host blob to the device (the handle allocates and owns the device copy). */
int wm_load_weights(wm_handle* h, const void* host_blob, size_t nbytes);
/* Use a caller-owned DEVICE blob (e.g. one filled by an NCCL broadcast); not freed by the handle. */
int wm_adopt_weights(wm_handle* h, void* device_blob, size_t nbytes);

/* ---- candidate tree (medusa_utils.py:305-421 generate_medusa_buffers, :446-457 per-head top-k) ------------- */
/* choices[0..K]: choices[0] = 1; all ones = top-1 chain (default).  Branching trees: at most 16 nodes, 32 paths, k <= 4. */
int wm_set_medusa_choices(wm_handle* h, const int32_t* choices, int32_t n);

/* ---- logits processors (model.py:1168-1207; HF logits_process.py:1893-1901,1847-1862) -- */
int wm_set_suppress(wm_handle* h, const int32_t* suppress_ids, int32_t n_suppress,
                    const int32_t* begin_suppress_ids, int32_t n_begin);

/* ---- frontend + encoder (HF feature_extraction_whisper.py:135-164; modeling_whisper.py:593-647;
 *      cross-attention K/V projection :325-336) ------------------------------------------- */
/* f32 PCM @16 kHz on the host, any length (zero-padded / truncated to 480000 samples). */
int wm_encode_pcm(wm_handle* h, const float* pcm, int32_t n_samples);
/* f32 log-mel [n_mels][3000] on the host (what WhisperProcessor produces). */
int wm_encode_mel(wm_handle* h, const float* mel);
/* The same features already in DEVICE memory of the handle's GPU (a CUDA `input_features` tensor: the
 * reference's caller does `input_features.to(device)` first, README.md:129-133).  `producer_stream` is the
 * cudaStream_t (NULL = legacy default stream) the features were produced on: the copy is ordered after it. */
int wm_encode_mel_device(wm_handle* h, const float* mel_dev, void* producer_stream);
/* Device twin of wm_encode_pcm: n_samples (0..480000) f32 samples @16 kHz in DEVICE memory of the handle's GPU, e.g. one
 * window in the middle of a long recording.  Samples past the window are zero, as for host PCM, and the log-mel and
 * encoder output are bit-identical to wm_encode_pcm on the same samples.  Ordered after `producer_stream` (as for
 * wm_encode_mel_device). */
int wm_encode_pcm_device(wm_handle* h, const float* pcm_dev, int32_t n_samples, void* producer_stream);

/* ---- resampler (torchaudio.functional.resample with its defaults: sinc_interp_hann, lowpass_filter_width 6,
 *      rolloff 0.99; integer rates) ------------------------------------------------------------------------------ */
/* Mono f32 samples in DEVICE memory, n_in of them at orig_hz -> *n_out = ceil(n_in * new / orig) samples at new_hz in
 * out_dev (orig / new: the rates divided by their gcd; out_cap >= *n_out).  Enqueued on `stream` (cudaStream_t, NULL =
 * legacy default stream); orig_hz == new_hz is a device copy.  The handle keeps the tap table of every rate pair it
 * has resampled; its weights need not be loaded. */
int wm_resample(wm_handle* h, const float* in_dev, int64_t n_in, int32_t orig_hz, int32_t new_hz, float* out_dev,
                int64_t out_cap, int64_t* n_out, void* stream);
/* Host logic, no GPU needed: the polyphase table the resampler runs for orig_hz -> new_hz, built in fp64 and rounded
 * once to fp32.  info4 = {orig, new, width, max_taps} after the gcd reduction.  With taps / lo / n_taps given
 * (cap >= new * max_taps floats): phase p has n_taps[p] taps taps[p * max_taps + j] on columns lo[p] + j of
 * torchaudio's dense [new][2 * width + orig] kernel, whose other columns are zero. */
int wm_resample_taps(int32_t orig_hz, int32_t new_hz, float* taps, int32_t* lo, int32_t* n_taps, int64_t cap,
                     int32_t* info4);

/* ---- the speculative decode loop (model.py:404-835 + medusa_utils.py:424-671) ---------- */
/* prompt: decoder_input_ids, 1 <= n_prompt < max_length - K - 2 (beyond 16 tokens the leading ones are cached by prefill
 * launches of 16-token chunks).  out_ids receives the FULL sequence (prompt + generated, after
 * the post-EOS fill of model.py:798-810); capacity must be >= max_length + medusa_num_heads + 2.
 * accept_lens (capacity >= max_length, may be NULL) receives the per-iteration accept length. */
int wm_generate(wm_handle* h, const int32_t* prompt, int32_t n_prompt, const wm_gen_params* gp,
                int32_t* out_ids, int32_t* n_out, int32_t* accept_lens, int32_t* n_iter);

/* ---- teacher-forced forward (model.py:1223-1347 `forward(...).logits`, shape [K+1, 1, T, V]) -------------- */
/* ids: 1..16 decoder_input_ids; out (host, capacity (K+1) * n_ids * vocab_size floats) receives the raw logits of
 * every head at every position, out[(k * n_ids + t) * V + v]; k = 0 is the base head.  Needs wm_encode_* first. */
int wm_forward(wm_handle* h, const int32_t* ids, int32_t n_ids, float* out);

/* ---- parity taps / measurements --------------------------------------------------------- */
int wm_get_mel(wm_handle* h, float* out /* [n_mels][3000] */);
int wm_get_encoder_out(wm_handle* h, float* out /* [max_source_positions][d_model] */);
/* Raw (pre-processor) logits of the last executed iteration: which = 0 pass A ([K+1][V], rows =
 * heads at the last position), 1 = pass B ([K+1][V], rows = tree positions). */
int wm_last_logits(wm_handle* h, int32_t which, float* out);
/* Device time (CUDA events on the handle's stream) of the last call: 0 = mel, 1 = encoder
 * (+cross K/V), 2 = decode loop.  Milliseconds. */
double wm_last_ms(wm_handle* h, int32_t what);
/* Number of kernel launches issued by the last wm_encode_* (what=1) / wm_generate (what=2). */
int64_t wm_last_launches(wm_handle* h, int32_t what);
/* CTAs per thread-block cluster of the persistent ring kernel: 2 when its grid is the whole GPU and the device can hold
 * all of those 2-CTA clusters at once (activation rows are then multicast to both CTAs of a cluster), else 1. */
int wm_decode_cluster(wm_handle* h);
/* Decode execution mode: 2 (DEFAULT) = one persistent cooperative kernel per speculative iteration with the
 * shared-memory weight ring (bulk-async prefetch across barriers; the product path); 1 = the same without the
 * ring (grid barriers only); 0 = CUDA graphs of stage kernels (debug / per-stage profiling, and the automatic
 * default for a decoder width the ring kernel is not instantiated for).  Returns the previous mode. */
int wm_set_decode_mode(wm_handle* h, int32_t mode);
/* Device address of the packed weights once loaded: a second handle on the same GPU adopts it (wm_adopt_weights)
 * instead of holding its own copy -- how S concurrent streams share one blob. */
void* wm_weights_device_ptr(wm_handle* h);
/* Engine options: "decode_ctas" = CTAs of the decode grid (default: every SM; S handles with n_sm / S each decode S
 * streams concurrently -- SURVEY 8(f) rank 3, the reference is batch 1 at model.py:1451); "decode_mode" (as above); "enc_gemm" 1 = wgmma/TMA encoder GEMM (default),
 * 0 = mma.sync encoder GEMM (cross-check), 2 = wgmma with 128 x 128 tiles only (cross-check of the per-GEMM tile
 * shapes); "enc_attn" 1 = wgmma/TMA encoder attention (default), 0 = mma.sync flash attention (cross-check);
 * "enc_pdl" 1 = encoder kernels under programmatic dependent launch (default), 0 = plain stream-ordered launches;
 * "profile" 1 = record the stage timeline below. */
int wm_set_option(wm_handle* h, const char* key, int32_t value);
/* Host logic, no GPU needed: the tile {rows, columns, ring stages} the wgmma encoder GEMM runs an M x N x K product
 * with on a GPU of n_sm SMs (0: 132) -- the shape with the fewest operand bytes on the busiest SM (DESIGN.md section 4).
 * fp16_out: the bias / bias+GELU epilogues; 0: the fp32 residual-stream epilogues (128 x 128 tiles only). */
int wm_enc_gemm_tile(int32_t M, int32_t N, int32_t K, int32_t fp16_out, int32_t n_sm, int32_t* out3);
/* Debug: per-stage timeline of the last persistent iteration (after wm_set_option(h, "profile", 1)).
 * Rows of 24 int64: stage id, mode, layer; body ns and barrier-wait ns seen by the last CTA; then the
 * 16 raw probes of CTA 0 -- ns offsets from stage begin ([1] end of body, [2] end of barrier, [7] record
 * read, [8] activations landed, [9] LayerNorm statistics, [10] split done, [3] staged, [13] before the
 * weight wait, [4] weights present, [5] MMAs done, [6] epilogue done, [14] unit loop left, [15] stage
 * function left) and two flags ([11], [12]: weights already present at stage begin / before the wait);
 * 3 spare. */
int wm_get_stage_profile(wm_handle* h, int64_t* out, int32_t cap_rows, int32_t* n_rows);

#ifdef __cplusplus
}
#endif
#endif /* WHISPER_MEDUSA_B200_H_ */
