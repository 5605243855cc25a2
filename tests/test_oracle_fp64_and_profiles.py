"""CPU tests of the fp64 oracle and of the synthetic checkpoints the decode-numerics GPU tests run on."""
import hashlib

import pytest
import torch

from oracle import medusa_ref as M
from oracle import whisper_ref as W
from whisper_medusa_b200.synthetic import (ACTIVATION_PROFILES, preset_config, synthetic_state_dict,
                                           width_config)


def _digest(sd):
    h = hashlib.sha256()
    for k in sorted(sd):
        h.update(k.encode())
        h.update(sd[k].contiguous().view(torch.uint8).numpy().tobytes())
    return h.hexdigest()[:16]


@pytest.mark.parametrize("preset,heads,htype,seed,digest", [
    ("micro", 4, "base_head", 0, "5be0d18e8d496fa0"),
    ("micro", 10, "medusa_block", 5, "47fcc93c15629a41"),
    ("tiny.en", 4, "base_head", 3, "bdbd12c8ae1d77b7"),
    ("tiny.en", 4, "medusa_block", 7, "ba82255e0e9c4e30"),
])
def test_default_state_dict_is_unchanged(preset, heads, htype, seed, digest):
    """Every golden fixture was made from these tensors: the default profile must keep every bit."""
    cfg = preset_config(preset, heads=heads, heads_type=htype)
    assert _digest(synthetic_state_dict(cfg, seed=seed)) == digest
    assert _digest(synthetic_state_dict(cfg, seed=seed, activation_profile="default")) == digest


def test_width_config_and_d_model_override():
    for d in (128, 256, 512, 640, 768, 1024, 1280):
        cfg = width_config(d)
        assert (cfg.d_model, cfg.decoder_attention_heads, cfg.encoder_attention_heads) == (d, d // 64, d // 64)
        assert (cfg.decoder_ffn_dim, cfg.encoder_ffn_dim, cfg.decoder_layers, cfg.encoder_layers) == (4 * d, 4 * d, 2, 2)
        assert cfg.medusa_hidden_size == d and cfg.vocab_size == 512 and cfg.eos_token_id == 500
    assert width_config(768, ffn_dim=768).decoder_ffn_dim == 768
    # an overridden d_model also sets the Medusa heads' width (the heads are d x d)
    cfg = preset_config("micro", d_model=256, decoder_attention_heads=4)
    assert cfg.medusa_hidden_size == 256
    sd = synthetic_state_dict(width_config(256, heads=2), seed=0)
    assert tuple(sd["medusa_heads.0.0.linear.weight"].shape) == (256, 256)


def _decode_fp64_with_probe(cfg, sd, enc):
    """Runs a 5-token decoder pass + Medusa heads in fp64; returns (logits, per-LayerNorm-input statistics)."""
    w = W.RefWeights(sd, torch.float64)
    stats = {"mu_sigma": [], "gx": [], "outlier": []}

    def probe(prefix, x):
        if not prefix.endswith("layer_norm") or prefix.endswith("decoder.layer_norm"):
            return
        mu, sig = x.mean(-1), x.std(-1, unbiased=False)
        stats["mu_sigma"].append(mu.abs() / sig)
        stats["gx"].append((x * w[prefix + ".weight"]).abs())
        a = x.abs()
        stats["outlier"].append(a.max(-1).values / a.median(-1).values)

    w.ln_probe = probe
    cache = W.new_cache(cfg)
    ids = [cfg.decoder_start_token_id, cfg.no_timestamps_token_id, 17, 33, 64]
    hidden = W.decoder_forward(w, cfg, ids, list(range(len(ids))), enc, cache, "engine")
    logits = W.medusa_logits(w, cfg, hidden, enc, cache, False, "engine")
    return logits, {k: torch.cat([t.reshape(-1) for t in v]) for k, v in stats.items()}


@pytest.mark.parametrize("d", [512, 1280])
@pytest.mark.parametrize("profile", ACTIVATION_PROFILES)
def test_activation_profiles_reach_their_regime(profile, d):
    """Each profile puts the LayerNorm-fed operands of the decoder (gamma o x, split into fp16 hi + lo by the ring
    kernel) where it says, with every checkpoint value finite in fp16 and finite fp64 logits."""
    cfg = width_config(d, heads=4)
    sd = synthetic_state_dict(cfg, seed=1, activation_profile=profile)
    for k, v in sd.items():
        assert v.dtype == torch.float16 and torch.isfinite(v).all(), k
    enc = torch.randn(1500, d, generator=torch.Generator().manual_seed(0), dtype=torch.float64)
    logits, st = _decode_fp64_with_probe(cfg, sd, enc)
    assert torch.isfinite(logits).all() and float(logits.std()) > 0.5
    ms, gx, outl = st["mu_sigma"], st["gx"], st["outlier"]
    assert float(gx.max()) < 65504.0
    if profile == "default":
        assert float(ms.max()) < 0.2 and float(outl.max()) < 20 and 1.0 < float(gx.max()) < 100.0
    elif profile == "offset":
        assert float(ms.max()) > 250 and float(ms.max()) < 600
        assert ((ms > 2) & (ms < 6)).any() and ((ms > 20) & (ms < 60)).any()
    elif profile == "outliers":
        assert float(outl.max()) > 300
    elif profile == "gamma_spread":
        g = sd["whisper_model.model.decoder.layers.0.self_attn_layer_norm.weight"].float()
        assert float(g.abs().min()) < 0.03 and float(g.abs().max()) > 4 and (g < 0).any()
    elif profile == "small":
        assert float(gx.median()) < 0.125 and float(gx.max()) < 1.0       # fp16 lo half subnormal below ~0.125
    elif profile == "near_top":
        assert float(gx.max()) > 2e4


@pytest.mark.parametrize("preset,htype,seed", [("micro", "base_head", 0), ("micro", "medusa_block", 1),
                                               ("tiny.en", "base_head", 0), ("tiny.en", "medusa_block", 2)])
def test_fp64_oracle_agrees_with_fp32(preset, htype, seed):
    """The fp64 oracle is the fp32 one computed in fp64: in the fp32 regime the two agree to fp32 accumulation level
    (measured: at most 5e-6 of max|logit| on these four models, three speculative iterations).  In the engine regime
    an fp16 K/V rounding can fall on either side of a boundary in the two precisions, and a 1-ulp flip of a cross-
    attention key moves the logits of these random models by up to ~1e-3 (measured: 7.5e-4 at tiny.en): that is the
    noise floor of any fp32-accurate implementation against the fp64 engine-regime reference."""
    cfg = preset_config(preset, heads=4, heads_type=htype)
    sd = synthetic_state_dict(cfg, seed=seed)
    enc = torch.randn(1500, cfg.d_model, generator=torch.Generator().manual_seed(seed))
    prompt = M.init_tokens(cfg, None)
    gp = M.gen_params(cfg, prompt, None, 40)
    for regime in ("fp32", "engine"):
        tr = {dt: M.medusa_greedy_search(W.RefWeights(sd, dt), cfg, enc, prompt, gp, regime, capture_logits=3, max_iters=3)
              for dt in (torch.float32, torch.float64)}
        a, b = tr[torch.float32], tr[torch.float64]
        assert a.sequences == b.sequences and a.accept_lengths == b.accept_lengths, regime
        assert b.passA_logits[0].dtype == torch.float64
        for la, lb in zip(a.passA_logits + a.passB_logits, b.passA_logits + b.passB_logits):
            assert la.dtype == torch.float32
            err = float((la.double() - lb).abs().max() / max(1.0, float(lb.abs().max())))
            assert err < (1e-5 if regime == "fp32" else 2e-3), (regime, err)
