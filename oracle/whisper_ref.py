"""CPU ORACLE (test infrastructure -- never imported by the product path).

A plain-PyTorch fp32 restatement of the arithmetic on the reference's decode path that
lives in the third-party dependency ``transformers==4.49.0`` (reference
``requirements.txt:6``; NOT vendored under /root/reference) plus the reference's own head
stacking.  Each function cites what it follows.  ``HF/`` = transformers
``models/whisper`` (read from the installed 5.5.0; the arithmetic of these functions is
unchanged from 4.49 as far as inspected -- SURVEY.md 8(c)).

Pinning: the reference ships no tests or golden vectors for this path (SURVEY.md section 4),
so this oracle is pinned two ways by ``tests/test_oracle_*.py``:
  * against the installed HF ``WhisperForConditionalGeneration`` / ``WhisperFeatureExtractor``
    run on the same seeded weights and audio (the third-party arithmetic), and
  * against the reference's own ``whisper_medusa/models/medusa_utils.py`` loaded by file path
    (only in the authoring container, where /root/reference exists).
The reference's ``WhisperMedusaModel`` itself cannot be imported here (transformers 5.5.0
vs the pinned 4.49.0), so the loop restatement in ``medusa_ref.py`` is *not* pinned by a run
of the reference model: for that part parity is "unpinned" (see DESIGN.md).

``regime``:
  * ``"fp32"``   -- reference numerics: fp16-rounded checkpoint values, everything fp32.
  * ``"engine"`` -- the same algorithm with the CUDA engine's documented rounding points
    reproduced (fp16 operands of the encoder GEMMs and of encoder attention, fp16 self- and
    cross-attention K/V caches).  Token-id parity is asserted against this regime; logits
    closeness is asserted against both.

Everything also runs in fp64: ``RefWeights(sd, dtype=torch.float64)`` for the encoder, the decoder side
(``decoder_forward``, ``medusa_logits`` and the loop in ``medusa_ref.py``), and
``log_mel_spectrogram(pcm, torch.float64)`` for the frontend.  The engine regime then still rounds to fp16
where the engine does and widens back, and everything else is fp64.  The fp32 results are unchanged by a bit.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Tuple

import numpy as np
import torch
import torch.nn.functional as F

SAMPLE_RATE = 16000
N_FFT = 400
HOP = 160
N_SAMPLES = 480000
N_FRAMES = 3000
LN_EPS = 1e-5


def _r16(x: torch.Tensor) -> torch.Tensor:
    """Round to fp16 and back to the working dtype (an engine rounding point)."""
    return x.to(torch.float16).to(x.dtype)


# --------------------------------------------------------------------------------------
# a1. log-mel frontend
# --------------------------------------------------------------------------------------
def _hz_to_mel_slaney(f):
    """HF ``audio_utils.py:hertz_to_mel`` (mel_scale="slaney")."""
    f = np.asarray(f, dtype=np.float64)
    min_log_hertz, min_log_mel, logstep = 1000.0, 15.0, 27.0 / np.log(6.4)
    mels = 3.0 * f / 200.0
    log_region = f >= min_log_hertz
    mels = np.where(log_region, min_log_mel + np.log(np.maximum(f, 1e-30) / min_log_hertz) * logstep, mels)
    return mels


def _mel_to_hz_slaney(m):
    """HF ``audio_utils.py:mel_to_hertz`` (mel_scale="slaney")."""
    m = np.asarray(m, dtype=np.float64)
    min_log_hertz, min_log_mel, logstep = 1000.0, 15.0, np.log(6.4) / 27.0
    f = 200.0 * m / 3.0
    log_region = m >= min_log_mel
    f = np.where(log_region, min_log_hertz * np.exp(logstep * (m - min_log_mel)), f)
    return f


def mel_filter_bank(n_freq: int = 201, n_mels: int = 80, fmin: float = 0.0, fmax: float = 8000.0,
                    sr: int = SAMPLE_RATE, dtype=np.float32) -> np.ndarray:
    """Slaney-normalised triangular filters ``[n_freq, n_mels]`` (computed in fp64, returned as ``dtype``).

    Follows HF ``audio_utils.py:mel_filter_bank`` (norm="slaney", mel_scale="slaney") as
    called from HF ``feature_extraction_whisper.py:95-103``.
    """
    mel_pts = np.linspace(_hz_to_mel_slaney(fmin), _hz_to_mel_slaney(fmax), n_mels + 2)
    filter_freqs = _mel_to_hz_slaney(mel_pts)
    fft_freqs = np.linspace(0, sr // 2, n_freq)
    fdiff = np.diff(filter_freqs)
    slopes = np.expand_dims(filter_freqs, 0) - np.expand_dims(fft_freqs, 1)
    down = -slopes[:, :-2] / fdiff[:-1]
    up = slopes[:, 2:] / fdiff[1:]
    fb = np.maximum(0.0, np.minimum(down, up))
    enorm = 2.0 / (filter_freqs[2 : n_mels + 2] - filter_freqs[:n_mels])
    fb *= np.expand_dims(enorm, 0)
    return fb.astype(dtype)


def pad_or_trim(pcm: np.ndarray) -> np.ndarray:
    """HF ``feature_extraction_whisper.py:189-342`` ``__call__`` with padding="max_length",
    truncation=True: right-pad with zeros / cut to 480 000 samples."""
    pcm = np.asarray(pcm, dtype=np.float32).reshape(-1)
    if pcm.shape[0] >= N_SAMPLES:
        return pcm[:N_SAMPLES].copy()
    out = np.zeros(N_SAMPLES, dtype=np.float32)
    out[: pcm.shape[0]] = pcm
    return out


def log_mel_spectrogram(pcm: np.ndarray, dtype: torch.dtype = torch.float32) -> np.ndarray:
    """f32 PCM -> ``[80, 3000]`` log-mel in ``dtype``.

    Follows HF ``feature_extraction_whisper.py:135-164`` (``_torch_extract_fbank_features``):
    hann(400) STFT (center, reflect pad), hop 160, |.|^2, drop last frame, mel, log10 with
    clamp 1e-10, floor at global max - 8, (x + 4) / 4.  ``dtype=torch.float64``: window, STFT, filters, log10
    and floor in fp64 (the f32 samples are widened exactly), a reference for the fp32 frontends.
    """
    wav = torch.from_numpy(pad_or_trim(pcm)).to(dtype)
    window = torch.hann_window(N_FFT, dtype=dtype)
    stft = torch.stft(wav, N_FFT, HOP, window=window, return_complex=True)
    mag = stft[..., :-1].abs() ** 2
    fb = torch.from_numpy(mel_filter_bank(dtype=np.float64 if dtype == torch.float64 else np.float32))
    mel = fb.T @ mag
    log_spec = torch.clamp(mel, min=1e-10).log10()
    log_spec = torch.maximum(log_spec, log_spec.max() - 8.0)
    log_spec = (log_spec + 4.0) / 4.0
    return log_spec.numpy().astype(np.float64 if dtype == torch.float64 else np.float32)


# --------------------------------------------------------------------------------------
# weights
# --------------------------------------------------------------------------------------
class RefWeights:
    """View of an fp16 checkpoint state dict (reference key layout, SURVEY.md 3.1) in the working dtype.

    ``dtype`` is the dtype every function computes in: fp32 (default, the reference's numerics) or fp64 (an
    independent high-precision reference for the engine; the engine regime still rounds to fp16 at the engine's
    rounding points and widens back)."""

    def __init__(self, state_dict: Dict[str, torch.Tensor], dtype: torch.dtype = torch.float32):
        self.dtype = dtype
        self.sd = {k: v.detach().to(dtype) for k, v in state_dict.items()}
        self.ln_probe = None     # optional callable(prefix, x): sees every LayerNorm input (statistics in tests)
        # optional callable(name, t): sees every encoder fp16 rounding point before it rounds ("mel", "conv1",
        # "layers.{i}.ln1" / "q" / "k" / "v" / "attn" / "ln2" / "fc1"; "q" carries the head_dim^-0.5 scaling, which the
        # engine applies after its rounding), every encoder LayerNorm input ("layers.{i}.ln1_in" / "ln2_in", "ln_f_in")
        # and the attention scores ("layers.{i}.scores", [H, S, S], scaled)
        self.enc_probe = None

    def __getitem__(self, k: str) -> torch.Tensor:
        return self.sd[k]

    def get(self, k: str) -> Optional[torch.Tensor]:
        return self.sd.get(k)

    def lin(self, x: torch.Tensor, prefix: str) -> torch.Tensor:
        return F.linear(x, self.sd[prefix + ".weight"], self.sd.get(prefix + ".bias"))

    def ln(self, x: torch.Tensor, prefix: str) -> torch.Tensor:
        if self.ln_probe is not None:
            self.ln_probe(prefix, x)
        return F.layer_norm(x, (x.shape[-1],), self.sd[prefix + ".weight"], self.sd[prefix + ".bias"], LN_EPS)


def _split_heads(x: torch.Tensor, n_heads: int) -> torch.Tensor:
    T, d = x.shape
    return x.view(T, n_heads, d // n_heads).transpose(0, 1)  # [H, T, dh]


def _merge_heads(x: torch.Tensor) -> torch.Tensor:
    H, T, dh = x.shape
    return x.transpose(0, 1).reshape(T, H * dh)


# --------------------------------------------------------------------------------------
# a2. encoder
# --------------------------------------------------------------------------------------
def _flash_attention_engine_rounding(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, block: int = 64,
                                     probe=None) -> torch.Tensor:
    """softmax(q k^T) v with the engine's rounding points: the same mathematics as the plain
    softmax, evaluated in 64-key blocks with a running row maximum, the un-normalised
    probabilities rounded to fp16 before they multiply V (they are the fp16 operand of the P*V
    tensor-core MMA in ``enc_attn.cu``), the row sum kept unrounded, in the working dtype.  ``q`` already carries the
    head_dim^-0.5 scaling; ``probe`` (optional) sees the scores."""
    H, S, dh = q.shape
    s = q @ k.transpose(1, 2)
    if probe is not None:
        probe(s)
    like = dict(dtype=q.dtype, device=q.device)
    m = torch.full((H, S), float("-inf"), **like)
    l = torch.zeros(H, S, **like)
    o = torch.zeros(H, S, dh, **like)
    for b in range(0, S, block):
        sb = s[:, :, b : b + block]
        m_new = torch.maximum(m, sb.max(dim=-1).values)
        alpha = torch.exp(m - m_new)
        p = torch.exp(sb - m_new[..., None])
        l = l * alpha + p.sum(dim=-1)
        o = o * alpha[..., None] + _r16(p) @ v[:, b : b + block]
        m = m_new
    return o / l[..., None]



def encoder_forward(w: RefWeights, cfg, mel: torch.Tensor, regime: str = "fp32") -> torch.Tensor:
    """``[80, 3000]`` log-mel -> ``[1500, d]`` encoder states.

    Follows HF ``modeling_whisper.py:593-647`` (``WhisperEncoder.forward``): conv1+GELU,
    conv2(stride 2)+GELU, + sinusoid positions, N pre-LN layers (``:380-414``; attention
    ``:284-357`` with q scaled before QK^T and no k bias), final LayerNorm.

    Computes in ``w.dtype``.  In the engine regime the engine's fp16 rounding points are kept (the mel;
    conv1 + GELU; the LayerNorm outputs; Q, K and V; P; the attention output; the FC1 + GELU output) and everything else
    is in the working dtype.  ``w.enc_probe`` (optional) sees each of them before it is rounded.
    """
    eng = regime == "engine"
    probe = w.enc_probe

    def rq(name: str, t: torch.Tensor) -> torch.Tensor:
        if probe is not None:
            probe(name, t)
        return _r16(t) if eng else t

    def ln(name: str, t: torch.Tensor, prefix: str) -> torch.Tensor:
        if probe is not None:
            probe(name + "_in", t)
        return w.ln(t, prefix)

    p = "whisper_model.model.encoder"
    x = rq("mel", mel.to(w.dtype))[None]  # [1, 80, 3000]
    x = F.gelu(F.conv1d(x, w[f"{p}.conv1.weight"], w[f"{p}.conv1.bias"], padding=1))
    x = rq("conv1", x)
    x = F.gelu(F.conv1d(x, w[f"{p}.conv2.weight"], w[f"{p}.conv2.bias"], stride=2, padding=1))
    x = x[0].transpose(0, 1)  # [1500, d]
    x = x + w[f"{p}.embed_positions.weight"]
    H = cfg.encoder_attention_heads
    dh = cfg.d_model // H
    for i in range(cfg.encoder_layers):
        lp = f"{p}.layers.{i}"
        li = f"layers.{i}."
        h = rq(li + "ln1", ln(li + "ln1", x, f"{lp}.self_attn_layer_norm"))
        q = w.lin(h, f"{lp}.self_attn.q_proj") * (dh ** -0.5)
        k = w.lin(h, f"{lp}.self_attn.k_proj")
        v = w.lin(h, f"{lp}.self_attn.v_proj")
        q, k, v = (_split_heads(rq(li + n, t), H) for n, t in (("q", q), ("k", k), ("v", v)))
        sprobe = (lambda s: probe(li + "scores", s)) if probe is not None else None
        if eng:
            o = _merge_heads(_flash_attention_engine_rounding(q, k, v, probe=sprobe))
        else:
            s = q @ k.transpose(1, 2)
            if sprobe is not None:
                sprobe(s)
            o = _merge_heads(torch.softmax(s, dim=-1) @ v)
        x = x + w.lin(rq(li + "attn", o), f"{lp}.self_attn.out_proj")
        h = rq(li + "ln2", ln(li + "ln2", x, f"{lp}.final_layer_norm"))
        h = rq(li + "fc1", F.gelu(w.lin(h, f"{lp}.fc1")))
        x = x + w.lin(h, f"{lp}.fc2")
    return ln("ln_f", x, f"{p}.layer_norm")


# --------------------------------------------------------------------------------------
# a3/a4. decoder with KV cache
# --------------------------------------------------------------------------------------
class RefCache:
    """Legacy-tuple style KV cache (what flows through the reference loop, SURVEY.md 3.2
    step 9): per layer self K/V ``[n, d]`` and cross K/V ``[1500, d]``."""

    def __init__(self, n_layers: int):
        self.self_k: List[Optional[torch.Tensor]] = [None] * n_layers
        self.self_v: List[Optional[torch.Tensor]] = [None] * n_layers
        self.cross_k: List[Optional[torch.Tensor]] = [None] * n_layers
        self.cross_v: List[Optional[torch.Tensor]] = [None] * n_layers

    @property
    def length(self) -> int:
        return 0 if self.self_k[0] is None else int(self.self_k[0].shape[0])

    def clone(self) -> "RefCache":
        c = RefCache(len(self.self_k))
        c.self_k, c.self_v = list(self.self_k), list(self.self_v)
        c.cross_k, c.cross_v = self.cross_k, self.cross_v  # passed through (model.py:397-400)
        return c

    def keep_rows(self, base_len: int, rows: List[int]) -> None:
        """Reference ``model.py:383-401``: cat(pre-verify KV, gathered tree rows)."""
        idx = torch.tensor(list(range(base_len)) + list(rows), dtype=torch.long)
        for i in range(len(self.self_k)):
            if self.self_k[i] is not None:
                self.self_k[i] = self.self_k[i][idx]
                self.self_v[i] = self.self_v[i][idx]


def _decoder_layer(w: RefWeights, cfg, lp: str, li: int, x: torch.Tensor, enc: torch.Tensor,
                   cache: RefCache, regime: str, causal_offset: Optional[int],
                   new_allowed: Optional[torch.Tensor] = None) -> torch.Tensor:
    """HF ``modeling_whisper.py:449-506`` (``WhisperDecoderLayer.forward``).

    ``causal_offset`` = number of cached positions before this call (query t sees cached
    keys plus new keys 0..t), or None for "no mask" (query sees every key).
    """
    eng = regime == "engine"
    rq = _r16 if eng else (lambda t: t)
    H = cfg.decoder_attention_heads
    dh = cfg.d_model // H
    T = x.shape[0]
    # self attention
    h = w.ln(x, f"{lp}.self_attn_layer_norm")
    q = w.lin(h, f"{lp}.self_attn.q_proj") * (dh ** -0.5)
    k_new = rq(w.lin(h, f"{lp}.self_attn.k_proj"))
    v_new = rq(w.lin(h, f"{lp}.self_attn.v_proj"))
    if cache.self_k[li] is None:
        cache.self_k[li], cache.self_v[li] = k_new, v_new
    else:
        cache.self_k[li] = torch.cat([cache.self_k[li], k_new], dim=0)
        cache.self_v[li] = torch.cat([cache.self_v[li], v_new], dim=0)
    K, V = cache.self_k[li], cache.self_v[li]
    n = K.shape[0]
    scores = _split_heads(q, H) @ _split_heads(K, H).transpose(1, 2)  # [H, T, n]
    if causal_offset is not None:
        past = n - T
        mask = torch.arange(n)[None, :] > (past + torch.arange(T))[:, None]
        if new_allowed is not None:   # true tree attention (NOT what the reference does): new row t sees new row j only if allowed
            mask = mask.clone()
            mask[:, past:] |= ~new_allowed
        scores = scores.masked_fill(mask[None], float("-inf"))
    o = _merge_heads(torch.softmax(scores, dim=-1) @ _split_heads(V, H))
    x = x + w.lin(o, f"{lp}.self_attn.out_proj")
    # cross attention (K/V computed once per clip, HF modeling_whisper.py:325-336)
    h = w.ln(x, f"{lp}.encoder_attn_layer_norm")
    q = w.lin(h, f"{lp}.encoder_attn.q_proj") * (dh ** -0.5)
    if cache.cross_k[li] is None:
        e = rq(enc.to(w.dtype))
        cache.cross_k[li] = rq(w.lin(e, f"{lp}.encoder_attn.k_proj"))
        cache.cross_v[li] = rq(w.lin(e, f"{lp}.encoder_attn.v_proj"))
    scores = _split_heads(q, H) @ _split_heads(cache.cross_k[li], H).transpose(1, 2)
    o = _merge_heads(torch.softmax(scores, dim=-1) @ _split_heads(cache.cross_v[li], H))
    x = x + w.lin(o, f"{lp}.encoder_attn.out_proj")
    # feed forward
    h = w.ln(x, f"{lp}.final_layer_norm")
    x = x + w.lin(F.gelu(w.lin(h, f"{lp}.fc1")), f"{lp}.fc2")
    return x


def decoder_forward(w: RefWeights, cfg, ids: List[int], positions: List[int], enc: torch.Tensor,
                    cache: RefCache, regime: str = "fp32", new_allowed: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Hidden states ``[T, d]`` for ``ids`` at explicit ``positions``; appends to ``cache``.

    Follows HF ``modeling_whisper.py:691-796`` (``WhisperDecoder.forward``): token + learned
    position embedding (``:204-212`` with explicit ``position_ids``), N layers under the
    ordinary causal mask in cache order, final LayerNorm.  This is what reference
    ``model.py:113-129`` (``medusa_forward``) returns as ``outputs[0]``.
    """
    p = "whisper_model.model.decoder"
    idt = torch.tensor(ids, dtype=torch.long)
    pos = torch.tensor(positions, dtype=torch.long)
    x = w[f"{p}.embed_tokens.weight"][idt] + w[f"{p}.embed_positions.weight"][pos]
    past = cache.length
    for i in range(cfg.decoder_layers):
        x = _decoder_layer(w, cfg, f"{p}.layers.{i}", i, x, enc, cache, regime, past, new_allowed)
    return w.ln(x, f"{p}.layer_norm")


# --------------------------------------------------------------------------------------
# a5/a6/a7. Medusa heads
# --------------------------------------------------------------------------------------
def res_block(w: RefWeights, x: torch.Tensor, prefix: str) -> torch.Tensor:
    """Reference ``model.py:180-210``: ``x + SiLU(Linear(x))``."""
    return x + F.silu(w.lin(x, prefix + ".linear"))


def proj_out(w: RefWeights, x: torch.Tensor) -> torch.Tensor:
    return F.linear(x, w["whisper_model.proj_out.weight"])


def medusa_logits(w: RefWeights, cfg, hidden: torch.Tensor, enc: torch.Tensor, cache: RefCache,
                  disable_medusa: bool, regime: str = "fp32") -> torch.Tensor:
    """Stacked logits ``[rows, T, V]`` (reference ``model.py:1272-1301``).

    base_head type: row i = proj_out(medusa_heads[i](hidden)); with ``disable_medusa`` only
    row 0 (``:1281-1284``).  medusa_block type (``:1287`` + ``:1349-1417``): row 0 =
    proj_out(hidden); an extra decoder layer (its own KV slot, index N) runs on the
    final-LayerNorm'ed hidden states -- always, because its KV must be cached
    (``:1410-1413``) -- and the heads read its output.
    """
    n_layers = int(cfg.medusa_num_layers)

    def head(i: int, x: torch.Tensor) -> torch.Tensor:
        for l in range(n_layers):
            x = res_block(w, x, f"medusa_heads.{i}.{l}")
        return x

    rows = []
    if cfg.medusa_heads_type == "base_head":
        for i in range(cfg.medusa_num_heads + 1):
            rows.append(proj_out(w, head(i, hidden)))
            if disable_medusa:
                break
    else:
        rows.append(proj_out(w, hidden))
        li = cfg.decoder_layers
        past = cache.self_k[li].shape[0] if cache.self_k[li] is not None else 0
        # 4.49 SDPA path: attention_mask=None => causal when T > 1, unmasked when T == 1.
        # With a cache and T > 1 (the verify pass) the block's attention output is never
        # consumed (disable_medusa), only its K/V rows; plain causal is used here.
        blk = _decoder_layer(w, cfg, "medusa_block", li, hidden, enc, cache, regime, past)
        if not disable_medusa:
            for i in range(cfg.medusa_num_heads):
                rows.append(proj_out(w, head(i, blk)))
    return torch.stack(rows, dim=0)


def new_cache(cfg) -> RefCache:
    return RefCache(cfg.decoder_layers + (1 if cfg.medusa_heads_type == "medusa_block" else 0))
