"""Seeded synthetic checkpoints and audio (no hub / dataset access in this environment).

The state dict uses the reference's checkpoint key layout (SURVEY.md 3.1 step 3; attribute
names in reference ``model.py:213-256``):

    whisper_model.model.encoder.* / whisper_model.model.decoder.* / whisper_model.proj_out.weight
    medusa_heads.{i}.{l}.linear.{weight,bias}            (reference model.py:235-246)
    medusa_block.*  (a WhisperDecoderLayer)              (reference model.py:248-256)

All tensors are fp16 (an "fp16 checkpoint"); both the oracle and the CUDA engine consume
exactly these values.  Everything is random (including LayerNorm affine and biases) so a
dropped bias or a mis-packed matrix cannot hide behind an identity initialisation.
"""
from __future__ import annotations

import math
from typing import Dict

import numpy as np
import torch

from .config import MedusaConfig

SAMPLE_RATE = 16000


def _sinusoids(length: int, channels: int) -> torch.Tensor:
    """Whisper encoder position table (HF ``modeling_whisper.py`` ``sinusoids``)."""
    inc = math.log(10000.0) / (channels // 2 - 1)
    inv = torch.exp(-inc * torch.arange(channels // 2, dtype=torch.float32))
    t = torch.arange(length, dtype=torch.float32)[:, None] * inv[None, :]
    return torch.cat([t.sin(), t.cos()], dim=1)


def _decoder_layer_keys(prefix: str, d: int, ffn: int):
    yield f"{prefix}.self_attn_layer_norm", "ln", (d,)
    for p in ("q_proj", "k_proj", "v_proj", "out_proj"):
        yield f"{prefix}.self_attn.{p}", "lin" if p != "k_proj" else "lin_nobias", (d, d)
    yield f"{prefix}.encoder_attn_layer_norm", "ln", (d,)
    for p in ("q_proj", "k_proj", "v_proj", "out_proj"):
        yield f"{prefix}.encoder_attn.{p}", "lin" if p != "k_proj" else "lin_nobias", (d, d)
    yield f"{prefix}.final_layer_norm", "ln", (d,)
    yield f"{prefix}.fc1", "lin", (ffn, d)
    yield f"{prefix}.fc2", "lin", (d, ffn)


ACTIVATION_PROFILES = ("default", "offset", "outliers", "gamma_spread", "small", "near_top")
ENCODER_PROFILES = ("default", "offset", "outliers", "small", "peaked", "near_top")


def synthetic_state_dict(config: MedusaConfig, seed: int = 0, enc_gain: float = 1.0,
                         dec_gain: float = 2.0, head_gain: float = 0.8,
                         logit_std: float = 1.75, activation_profile: str = "default",
                         encoder_profile: str = "default") -> Dict[str, torch.Tensor]:
    """Deterministic fp16 state dict of the exact shapes of ``config`` (CPU tensors).

    Linear weights are N(0, gain^2 / fan_in).  The gains are chosen (empirically, see
    DESIGN.md "synthetic checkpoints") so that a random model does not collapse onto one
    repeated token: ``dec_gain`` 2 makes the decoder a strongly non-linear function of the
    previous token, ``logit_std`` sets the spread of the vocabulary logits
    (= std(embedding) * sqrt(d)), and ``head_gain`` makes the Medusa heads disagree with the
    base head often enough that every accept length 0..K occurs under typical acceptance.

    ``activation_profile`` (one of ``ACTIVATION_PROFILES``) reshapes the decoder side so that its residual stream and
    LayerNorm operands have the statistics of real checkpoints (see ``_apply_activation_profile``); ``"default"``
    returns exactly the tensors it always did.  ``encoder_profile`` (one of ``ENCODER_PROFILES``) does the same for the
    encoder's tensors (``_apply_encoder_profile``).
    """
    if activation_profile not in ACTIVATION_PROFILES:
        raise ValueError(f"activation_profile must be one of {ACTIVATION_PROFILES}")
    if encoder_profile not in ENCODER_PROFILES:
        raise ValueError(f"encoder_profile must be one of {ENCODER_PROFILES}")
    g = torch.Generator(device="cpu")
    g.manual_seed(int(seed))
    d, V = config.d_model, config.vocab_size
    sd: Dict[str, torch.Tensor] = {}
    gain = {"v": enc_gain}

    def randn(*shape, scale):
        return (torch.randn(*shape, generator=g, dtype=torch.float32) * scale).to(torch.float16)

    def add(name: str, kind: str, shape):
        if kind == "ln":
            sd[name + ".weight"] = (1.0 + 0.1 * torch.randn(*shape, generator=g)).to(torch.float16)
            sd[name + ".bias"] = randn(*shape, scale=0.1)
        elif kind in ("lin", "lin_nobias"):
            sd[name + ".weight"] = randn(*shape, scale=gain["v"] / math.sqrt(shape[1]))
            if kind == "lin":
                sd[name + ".bias"] = randn(shape[0], scale=0.05)
        else:
            raise AssertionError(kind)

    enc = "whisper_model.model.encoder"
    sd[f"{enc}.conv1.weight"] = randn(d, config.num_mel_bins, 3, scale=enc_gain / math.sqrt(3 * config.num_mel_bins))
    sd[f"{enc}.conv1.bias"] = randn(d, scale=0.05)
    sd[f"{enc}.conv2.weight"] = randn(d, d, 3, scale=enc_gain / math.sqrt(3 * d))
    sd[f"{enc}.conv2.bias"] = randn(d, scale=0.05)
    sd[f"{enc}.embed_positions.weight"] = _sinusoids(config.max_source_positions, d).to(torch.float16)
    for i in range(config.encoder_layers):
        p = f"{enc}.layers.{i}"
        add(f"{p}.self_attn_layer_norm", "ln", (d,))
        for q in ("q_proj", "k_proj", "v_proj", "out_proj"):
            add(f"{p}.self_attn.{q}", "lin" if q != "k_proj" else "lin_nobias", (d, d))
        add(f"{p}.final_layer_norm", "ln", (d,))
        add(f"{p}.fc1", "lin", (config.encoder_ffn_dim, d))
        add(f"{p}.fc2", "lin", (d, config.encoder_ffn_dim))
    add(f"{enc}.layer_norm", "ln", (d,))

    dec = "whisper_model.model.decoder"
    gain["v"] = dec_gain
    sd[f"{dec}.embed_tokens.weight"] = randn(V, d, scale=logit_std / math.sqrt(d))
    sd[f"{dec}.embed_positions.weight"] = randn(config.max_target_positions, d, scale=0.5 * logit_std / math.sqrt(d))
    for i in range(config.decoder_layers):
        for name, kind, shape in _decoder_layer_keys(f"{dec}.layers.{i}", d, config.decoder_ffn_dim):
            add(name, kind, shape)
    add(f"{dec}.layer_norm", "ln", (d,))
    sd["whisper_model.proj_out.weight"] = sd[f"{dec}.embed_tokens.weight"]  # tied

    n_heads = config.medusa_num_heads + (0 if config.is_block else 1)  # reference model.py:235-256
    gain["v"] = head_gain
    for i in range(n_heads):
        for l in range(config.medusa_num_layers):
            add(f"medusa_heads.{i}.{l}.linear", "lin", (config.medusa_hidden_size, d))
    gain["v"] = dec_gain
    if config.is_block:
        for name, kind, shape in _decoder_layer_keys("medusa_block", d, config.decoder_ffn_dim):
            add(name, kind, shape)
    if activation_profile != "default":
        _apply_activation_profile(sd, config, activation_profile, seed)
    if encoder_profile != "default":
        _apply_encoder_profile(sd, config, encoder_profile, seed)
    return sd


def _apply_encoder_profile(sd: Dict[str, torch.Tensor], config: MedusaConfig, profile: str, seed: int) -> None:
    """Reshape the encoder tensors of ``sd`` in place (own generator: the default tensors are drawn first and
    unchanged).  Nothing outside the encoder changes.

    * ``offset``: a DC component common to all channels of the residual stream, through the conv2 bias (+20, which
      GELU passes on), the position table (a per-row level cycling over 1, 10, 100, 300) and the O-proj / FC2 biases
      (+5 each).  |mean| / std at the LayerNorm inputs reaches the hundreds; LayerNorm removes it exactly, so only the
      fp32 residual stream and the LayerNorm statistics see it.
    * ``outliers``: three residual channels 50-300x the others (position table, conv2 / O-proj / FC2 rows).
    * ``small``: the residual stream scaled to std ~ 3e-3 (conv2 weights and bias, position table, O-proj / FC2), so the
      LayerNorm eps of 1e-5 is a large share of the variance.
    * ``peaked``: the Q and K rows of two heads per layer scaled by 3 (scores x 9): score spreads of tens, a near one-hot
      softmax whose row maximum moves from one 64-key block to another.
    * ``near_top``: in every layer one head's Q and V rows and a quarter of the FC1 neurons are scaled by 4000, so Q,
      V and the FC1 + GELU output reach 1e4-3e4 at their fp16 rounding points; that head's K rows and the O-proj / FC2
      columns that read the scaled values are scaled by 1/4000 (the scores and the function stay as they were).
    """
    g = torch.Generator(device="cpu")
    g.manual_seed(2_000_003 * (ENCODER_PROFILES.index(profile) + 1) + int(seed))
    d, f = config.d_model, config.encoder_ffn_dim
    dh = d // config.encoder_attention_heads
    enc = "whisper_model.model.encoder"
    layers = [f"{enc}.layers.{i}" for i in range(config.encoder_layers)]
    writers = ("self_attn.out_proj", "fc2")
    pos = f"{enc}.embed_positions.weight"

    def f32(k):
        return sd[k].to(torch.float32)

    def put(k, v):
        v = v.to(torch.float16)
        assert torch.isfinite(v).all(), k
        sd[k] = v

    if profile == "offset":
        n_pos = sd[pos].shape[0]
        dc = torch.tensor([1.0, 10.0, 100.0, 300.0]).repeat(n_pos // 4 + 1)[:n_pos]
        put(pos, f32(pos) + dc[:, None])
        put(f"{enc}.conv2.bias", f32(f"{enc}.conv2.bias") + 20.0)
        for lp in layers:
            for wr in writers:
                put(f"{lp}.{wr}.bias", f32(f"{lp}.{wr}.bias") + 5.0)
    elif profile == "outliers":
        ch = torch.randperm(d, generator=g)[:3]
        gain = torch.tensor([50.0, 120.0, 300.0])
        p = f32(pos)
        p[:, ch] = p[:, ch] * gain + 0.02 * gain
        put(pos, p)
        for k in ([f"{enc}.conv2"] + [f"{lp}.{wr}" for lp in layers for wr in writers]):
            w, b = f32(f"{k}.weight"), f32(f"{k}.bias")
            w[ch] *= gain.view(-1, *([1] * (w.dim() - 1)))
            b[ch] *= gain
            put(f"{k}.weight", w)
            put(f"{k}.bias", b)
    elif profile == "small":
        s = 3e-3
        for k in ([f"{enc}.conv2.weight", f"{enc}.conv2.bias", pos]
                  + [f"{lp}.{wr}.{t}" for lp in layers for wr in writers for t in ("weight", "bias")]):
            put(k, f32(k) * s)
    elif profile == "peaked":
        for lp in layers:
            heads = torch.randperm(config.encoder_attention_heads, generator=g)[:2]
            for proj in ("q_proj", "k_proj"):
                w = f32(f"{lp}.self_attn.{proj}.weight")
                b = f32(f"{lp}.self_attn.{proj}.bias") if proj == "q_proj" else None
                for h in heads.tolist():
                    w[h * dh:(h + 1) * dh] *= 3.0
                    if b is not None:
                        b[h * dh:(h + 1) * dh] *= 3.0
                put(f"{lp}.self_attn.{proj}.weight", w)
                if b is not None:
                    put(f"{lp}.self_attn.{proj}.bias", b)
    elif profile == "near_top":
        G = 4000.0
        for lp in layers:
            h = int(torch.randint(config.encoder_attention_heads, (1,), generator=g))
            rows = slice(h * dh, (h + 1) * dh)
            for proj, scale in (("q_proj", G), ("k_proj", 1.0 / G), ("v_proj", G)):
                w = f32(f"{lp}.self_attn.{proj}.weight")
                w[rows] *= scale
                put(f"{lp}.self_attn.{proj}.weight", w)
                if proj != "k_proj":
                    b = f32(f"{lp}.self_attn.{proj}.bias")
                    b[rows] *= scale
                    put(f"{lp}.self_attn.{proj}.bias", b)
            wo = f32(f"{lp}.self_attn.out_proj.weight")
            wo[:, rows] /= G
            put(f"{lp}.self_attn.out_proj.weight", wo)
            nrn = torch.randperm(f, generator=g)[: f // 4]
            w1, b1, w2 = f32(f"{lp}.fc1.weight"), f32(f"{lp}.fc1.bias"), f32(f"{lp}.fc2.weight")
            w1[nrn] *= G
            b1[nrn] *= G
            w2[:, nrn] /= G
            put(f"{lp}.fc1.weight", w1)
            put(f"{lp}.fc1.bias", b1)
            put(f"{lp}.fc2.weight", w2)


def _apply_activation_profile(sd: Dict[str, torch.Tensor], config: MedusaConfig, profile: str, seed: int) -> None:
    """Reshape the decoder-side tensors of ``sd`` in place (own generator: the default tensors are drawn first and
    unchanged).  The encoder, the token embedding (tied to proj_out) and the Medusa heads keep their values.

    * ``offset``: a DC component common to all channels of the residual stream, through the position table and the
      out-proj / FC2 biases.  It cycles over three levels per position: the first LayerNorm's rows have |mean| / std
      of about 5, 30 and 300 (d = 512; 1.6x that at d = 1280), the later ones about 1-5.  LayerNorm removes it
      exactly, so only rounding sees it.
    * ``outliers``: three residual channels 50-300x the others (position table, out-proj / FC2 rows).
    * ``gamma_spread``: LayerNorm gamma log-uniform in magnitude over 0.02...5, a tenth of it negative; beta ~ N(0, 0.5^2).
    * ``small``: residual stream scaled to about 1e-2 (token / position embeddings, out-proj / FC2); the final
      LayerNorm's gamma / beta compensate, so the logits keep their spread.  gamma o x then lies where the fp16 lo half
      of the split is subnormal.
    * ``near_top``: one channel of the residual holds about 100 (position table; out-proj / FC2 never write it) and
      every folded LayerNorm has gamma = 300 there, so |gamma o x| is about 3e4, inside fp16 but near its top.  The
      columns of the QKV, cross-Q and FC1 weights that read that channel are scaled by 1/300.
    """
    g = torch.Generator(device="cpu")
    g.manual_seed(1_000_003 * (ACTIVATION_PROFILES.index(profile) + 1) + int(seed))
    d = config.d_model
    dec = "whisper_model.model.decoder"
    layers = [f"{dec}.layers.{i}" for i in range(config.decoder_layers)] + (["medusa_block"] if config.is_block else [])
    folded_ln = ("self_attn_layer_norm", "encoder_attn_layer_norm", "final_layer_norm")
    ln_fed = {"self_attn_layer_norm": ("self_attn.q_proj", "self_attn.k_proj", "self_attn.v_proj"),
              "encoder_attn_layer_norm": ("encoder_attn.q_proj",), "final_layer_norm": ("fc1",)}
    writers = ("self_attn.out_proj", "encoder_attn.out_proj", "fc2")

    def f32(k):
        return sd[k].to(torch.float32)

    def put(k, v):
        v = v.to(torch.float16)
        assert torch.isfinite(v).all(), k
        sd[k] = v

    pos = f"{dec}.embed_positions.weight"
    if profile == "offset":
        n_pos = sd[pos].shape[0]
        dc = torch.tensor([0.5, 2.5, 25.0]).repeat(n_pos // 3 + 1)[:n_pos]
        put(pos, f32(pos) + dc[:, None])
        for lp in layers:
            for wr in writers:
                put(f"{lp}.{wr}.bias", f32(f"{lp}.{wr}.bias") + 5.0)
    elif profile == "outliers":
        ch = torch.randperm(d, generator=g)[:3]
        gain = torch.tensor([50.0, 120.0, 300.0])
        p = f32(pos)
        p[:, ch] = p[:, ch] * gain + 0.02 * gain
        put(pos, p)
        for lp in layers:
            for wr in writers:
                w, b = f32(f"{lp}.{wr}.weight"), f32(f"{lp}.{wr}.bias")
                w[ch] *= gain[:, None]
                b[ch] *= gain
                put(f"{lp}.{wr}.weight", w)
                put(f"{lp}.{wr}.bias", b)
    elif profile == "gamma_spread":
        for lp in layers + [dec]:
            for ln in (folded_ln if lp != dec else ("layer_norm",)):
                mag = torch.exp(torch.empty(d).uniform_(math.log(0.02), math.log(5.0), generator=g))
                sign = torch.where(torch.rand(d, generator=g) < 0.1, -1.0, 1.0)
                put(f"{lp}.{ln}.weight", mag * sign)
                put(f"{lp}.{ln}.bias", 0.5 * torch.randn(d, generator=g))
    elif profile == "small":
        s_emb = 1e-2 / float(f32(f"{dec}.embed_tokens.weight").std())
        for k in (f"{dec}.embed_tokens.weight", pos):
            put(k, f32(k) * s_emb)
        sd["whisper_model.proj_out.weight"] = sd[f"{dec}.embed_tokens.weight"]          # tied
        for lp in layers:
            for wr in writers:
                for t in ("weight", "bias"):
                    put(f"{lp}.{wr}.{t}", f32(f"{lp}.{wr}.{t}") * 0.02)
        for t in ("weight", "bias"):
            put(f"{dec}.layer_norm.{t}", f32(f"{dec}.layer_norm.{t}") / s_emb)
    elif profile == "near_top":
        c = int(torch.randint(d, (1,), generator=g))
        p = f32(pos)
        p[:, c] = 100.0
        put(pos, p)
        for lp in layers:
            for wr in writers:
                w, b = f32(f"{lp}.{wr}.weight"), f32(f"{lp}.{wr}.bias")
                w[c] = 0.0
                b[c] = 0.0
                put(f"{lp}.{wr}.weight", w)
                put(f"{lp}.{wr}.bias", b)
            for ln in folded_ln:
                gm = f32(f"{lp}.{ln}.weight")
                gm[c] = 300.0
                put(f"{lp}.{ln}.weight", gm)
                for fed in ln_fed[ln]:
                    w = f32(f"{lp}.{fed}.weight")
                    w[:, c] /= 300.0
                    put(f"{lp}.{fed}.weight", w)


def synthetic_audio(seconds: float, stream_id: int = 0, seed: int = 1234) -> np.ndarray:
    """Speech-like 16 kHz mono f32 clip (SURVEY.md 8(d)): a few AM-modulated harmonic
    stacks plus low-level noise, peak-normalised to 0.5."""
    rng = np.random.default_rng(seed + stream_id)
    n = int(round(seconds * SAMPLE_RATE))
    t = np.arange(n, dtype=np.float64) / SAMPLE_RATE
    x = np.zeros(n, dtype=np.float64)
    for _ in range(int(rng.integers(3, 6))):
        f0 = rng.uniform(90.0, 260.0)
        am = 0.5 * (1.0 + np.sin(2 * np.pi * rng.uniform(1.5, 6.0) * t + rng.uniform(0, 2 * np.pi)))
        for h in range(1, 9):
            x += am * (rng.uniform(0.2, 1.0) / h) * np.sin(2 * np.pi * f0 * h * t + rng.uniform(0, 2 * np.pi))
    x += 0.02 * rng.standard_normal(n)
    x *= 0.5 / max(np.abs(x).max(), 1e-9)
    return x.astype(np.float32)


def preset_config(name: str, heads: int = 10, heads_type: str = "base_head", head_layers: int = 1, **kw) -> MedusaConfig:
    """BASELINE.json configs: ``large-v2`` (cfg 2-5), ``tiny.en`` (cfg 1), ``micro`` (tests); ``base``, ``small`` and
    ``medium`` (the full-depth tests).  ``head_layers``: MedusaResBlocks per head (``medusa_num_layers``)."""
    table = {
        "large-v2": "openai/whisper-large-v2",
        "tiny.en": "openai/whisper-tiny.en",
        "micro": "synthetic/whisper-micro",
        "base": "openai/whisper-base",
        "small": "openai/whisper-small",
        "medium": "openai/whisper-medium",
    }
    wname = table.get(name, name)
    from .config import WHISPER_PRESETS

    d_model = kw.get("d_model", WHISPER_PRESETS[wname]["d_model"])
    return MedusaConfig(
        medusa_num_heads=heads, medusa_num_layers=head_layers, medusa_hidden_size=d_model,
        whisper_model_name=wname, medusa_choices=[1] * (heads + 1), medusa_heads_type=heads_type, **kw)


def width_config(d_model: int, heads: int = 4, heads_type: str = "base_head", ffn_dim: int = 0,
                 head_layers: int = 1) -> MedusaConfig:
    """A small model at decoder width ``d_model``: micro's vocabulary and special tokens, 2 encoder and 2 decoder layers,
    d_model / 64 attention heads, FFN width ``ffn_dim`` (default 4 * d_model, as in every Whisper size)."""
    ffn = int(ffn_dim) or 4 * d_model
    return preset_config("micro", heads=heads, heads_type=heads_type, head_layers=head_layers, d_model=d_model,
                         encoder_attention_heads=d_model // 64, decoder_attention_heads=d_model // 64,
                         encoder_ffn_dim=ffn, decoder_ffn_dim=ffn)
