"""CPU tests of the fp64 encoder and log-mel oracle, and of the encoder activation profiles the GPU encoder tests run on
(``synthetic_state_dict(encoder_profile=...)``)."""
import numpy as np
import pytest
import torch

from oracle import whisper_ref as W
from whisper_medusa_b200.synthetic import (ENCODER_PROFILES, preset_config, synthetic_audio, synthetic_state_dict,
                                           width_config)

ENC = "whisper_model.model.encoder"


def _rel_max(a, b):
    a, b = a.double(), b.double()
    return float((a - b).abs().max() / max(1.0, float(b.abs().max())))


def _rel_rms(a, b):
    a, b = a.double(), b.double()
    return float((a - b).pow(2).mean().sqrt() / b.pow(2).mean().sqrt())


@pytest.mark.parametrize("d", [128, 384, 1280])
def test_fp64_encoder_agrees_with_fp32(d):
    """The fp64 encoder is the fp32 one computed in fp64.  In the fp32 regime the two agree to fp32 accumulation level
    (measured: at most 6.4e-7 of max(1, max|state|) at d = 128, 384, 1280 on 30 s of audio).  In the engine regime an
    fp16 rounding (QKV, P, FC1 + GELU, ...) can fall on either side of a boundary in the two precisions, so the fp32
    oracle differs from the fp64 reference by flip noise: measured 3.3e-4 max and 2.3e-4 relative RMS.  The bars are
    about 3x those; the GPU tests print this floor beside the engine's error."""
    cfg = width_config(d, heads=4)
    sd = synthetic_state_dict(cfg, seed=1)
    mel = torch.from_numpy(W.log_mel_spectrogram(synthetic_audio(30.0, stream_id=1), torch.float64))
    for regime, bar_max, bar_rms in (("fp32", 2e-6, 2e-6), ("engine", 1e-3, 7e-4)):
        a = W.encoder_forward(W.RefWeights(sd), cfg, mel.float(), regime)
        b = W.encoder_forward(W.RefWeights(sd, torch.float64), cfg, mel, regime)
        assert a.dtype == torch.float32 and b.dtype == torch.float64 and b.shape == (1500, d)
        assert _rel_max(a, b) < bar_max, (regime, _rel_max(a, b))
        assert _rel_rms(a, b) < bar_rms, (regime, _rel_rms(a, b))


@pytest.mark.parametrize("seconds", [5.0, 30.0, 0.37])
def test_fp64_log_mel_matches_hf_feature_extractor(seconds):
    """The fp64 log-mel against the installed HF extractor (which computes in fp32): measured 1.1e-5 at 30 s, the
    extractor's own fp32 error.  The fp32 oracle stays within 1e-5 of the extractor (test_oracle_frontend_and_backbone)."""
    from transformers import WhisperFeatureExtractor

    pcm = synthetic_audio(seconds, stream_id=3)
    hf = WhisperFeatureExtractor()(pcm, sampling_rate=16000, return_tensors="np").input_features[0]
    ours = W.log_mel_spectrogram(pcm, torch.float64)
    assert ours.dtype == np.float64 and ours.shape == (80, 3000)
    assert np.abs(hf - ours).max() < 3e-5
    assert np.abs(W.log_mel_spectrogram(pcm) - ours).max() < 3e-5


def probe_encoder(cfg, sd, mel):
    """fp64 engine-regime encoder with ``enc_probe``: (states, statistics) where the statistics are, over all layers,
    the largest |mean| / std, smallest std and largest max / median |x| of a LayerNorm input row, the largest score
    spread (max - min over the keys of one query row) and the largest |value| at each fp16 rounding point, Q as the
    engine stores it (without the head_dim^-0.5 scaling)."""
    w = W.RefWeights(sd, torch.float64)
    st = {"mu_sigma": 0.0, "std_min": float("inf"), "outlier": 0.0, "spread": 0.0}
    qscale = (cfg.d_model // cfg.encoder_attention_heads) ** 0.5

    def probe(name, t):
        key = name.split(".")[-1]
        if key.endswith("_in"):
            mu, sg = t.mean(-1), t.std(-1, unbiased=False)
            a = t.abs()
            st["mu_sigma"] = max(st["mu_sigma"], float((mu.abs() / sg).max()))
            st["std_min"] = min(st["std_min"], float(sg.min()))
            st["outlier"] = max(st["outlier"], float((a.max(-1).values / a.median(-1).values).max()))
        elif key == "scores":
            st["spread"] = max(st["spread"], float((t.max(-1).values - t.min(-1).values).max()))
        else:
            v = float(t.abs().max()) * (qscale if key == "q" else 1.0)
            st[key] = max(st.get(key, 0.0), v)

    w.enc_probe = probe
    return W.encoder_forward(w, cfg, mel, "engine"), st


def tail_only_mel(seed=0):
    """Content only in frames 2944-2999 (encoder rows 1472-1499), a uniform floor elsewhere."""
    rng = np.random.default_rng(seed)
    mel = np.full((80, 3000), -0.5)
    mel[:, 2944:] = rng.uniform(-1.0, 1.5, (80, 56))
    return mel


@pytest.mark.parametrize("d", [512, 1280])
@pytest.mark.parametrize("profile", ENCODER_PROFILES)
def test_encoder_profiles_reach_their_regime(profile, d):
    """Each encoder profile reaches its regime on 30 s of audio and on the tail-only mel, measured with the fp64 probe;
    every checkpoint value and every fp16 rounding point of the engine stays finite and below 65504, and only encoder
    tensors change."""
    cfg = width_config(d, heads=4)
    sd = synthetic_state_dict(cfg, seed=1, encoder_profile=profile)
    base = synthetic_state_dict(cfg, seed=1)
    for k, v in sd.items():
        assert v.dtype == torch.float16 and torch.isfinite(v).all(), k
        if not k.startswith(ENC + "."):
            assert torch.equal(v, base[k]), k
    assert (profile == "default") == all(torch.equal(sd[k], base[k]) for k in sd)
    mels = (W.log_mel_spectrogram(synthetic_audio(30.0, stream_id=1), torch.float64), tail_only_mel())
    for mel in mels:
        out, st = probe_encoder(cfg, sd, torch.from_numpy(mel))
        assert torch.isfinite(out).all()
        points = {k: v for k, v in st.items() if k not in ("mu_sigma", "std_min", "outlier", "spread")}
        assert set(points) == {"mel", "conv1", "ln1", "q", "k", "v", "attn", "ln2", "fc1"}
        assert max(points.values()) < 65504.0, points
        if profile == "default":
            assert st["mu_sigma"] < 2 and st["std_min"] > 0.3 and st["outlier"] < 20 and st["spread"] < 15
            assert max(points.values()) < 10
        elif profile == "offset":
            assert st["mu_sigma"] > 200
        elif profile == "outliers":
            assert st["outlier"] > 300
        elif profile == "small":
            assert st["std_min"] ** 2 < 1e-5        # eps is more than the variance of some rows
        elif profile == "peaked":
            assert st["spread"] > 30
        elif profile == "near_top":
            assert min(points["q"], points["v"], points["fc1"]) > 1e4 and max(points.values()) < 3.5e4


@pytest.mark.parametrize("profile", ENCODER_PROFILES)
def test_encoder_profiles_at_full_depth(profile):
    """Each encoder profile in every one of medium's 24 layers on 30 s of audio (DESIGN.md section 2, "Profiles at
    depth"): every fp16 rounding point below 65504 (measured at most 2.0e4, near_top) and each profile in its regime in
    every layer, except ``small``, whose eps-dominated rows occur in the first layers only (the residual grows with
    depth: the smallest row std per layer is 1.4e-3 to 1.5e-2)."""
    cfg = preset_config("medium", heads=4)
    sd = synthetic_state_dict(cfg, seed=1, encoder_profile=profile)
    w = W.RefWeights(sd, torch.float64)
    per = {}

    def probe(name, t):
        if not name.startswith("layers."):
            return
        _, layer, key = name.split(".")
        st = per.setdefault(int(layer), {"mu_sigma": 0.0, "std_min": float("inf"), "outlier": 0.0, "spread": 0.0})
        if key.endswith("_in"):
            mu, sg = t.mean(-1), t.std(-1, unbiased=False)
            a = t.abs()
            st["mu_sigma"] = max(st["mu_sigma"], float((mu.abs() / sg).max()))
            st["std_min"] = min(st["std_min"], float(sg.min()))
            st["outlier"] = max(st["outlier"], float((a.max(-1).values / a.median(-1).values).max()))
        elif key == "scores":
            st["spread"] = max(st["spread"], float((t.max(-1).values - t.min(-1).values).max()))
        else:
            st[key] = max(st.get(key, 0.0), float(t.abs().max()) * (64 ** 0.5 if key == "q" else 1.0))

    w.enc_probe = probe
    mel = torch.from_numpy(W.log_mel_spectrogram(synthetic_audio(30.0, stream_id=1), torch.float64))
    assert torch.isfinite(W.encoder_forward(w, cfg, mel, "engine")).all()
    w.enc_probe = None       # the probe refers to w: without this cycle the weights are freed at once
    assert sorted(per) == list(range(cfg.encoder_layers))
    for i, st in per.items():
        points = {k: st[k] for k in ("ln1", "q", "k", "v", "attn", "ln2", "fc1")}
        where = (profile, i, st)
        assert max(points.values()) < 65504.0, where
        if profile == "default":
            assert st["mu_sigma"] < 2 and st["std_min"] > 0.3 and st["outlier"] < 20 and st["spread"] < 15, where
            assert max(points.values()) < 10, where
        elif profile == "offset":
            assert st["mu_sigma"] > 50, where
        elif profile == "outliers":
            assert st["outlier"] > 100, where
        elif profile == "small":
            assert st["std_min"] < 0.02 and (i > 0 or st["std_min"] ** 2 < 1e-5), where
        elif profile == "peaked":
            assert st["spread"] > 10, where
        elif profile == "near_top":
            assert min(points["q"], points["v"], points["fc1"]) > 1e4 and max(points.values()) < 3.5e4, where


def test_encoder_and_decoder_profiles_are_independent():
    """A decoder profile leaves the encoder alone and the other way round."""
    cfg = width_config(512, heads=4)
    base = synthetic_state_dict(cfg, seed=2)
    dec = synthetic_state_dict(cfg, seed=2, activation_profile="offset")
    enc = synthetic_state_dict(cfg, seed=2, encoder_profile="offset")
    both = synthetic_state_dict(cfg, seed=2, activation_profile="offset", encoder_profile="offset")
    for k in base:
        is_enc = k.startswith(ENC + ".")
        assert torch.equal(dec[k], base[k]) or not is_enc, k
        assert torch.equal(enc[k], base[k]) or is_enc, k
        assert torch.equal(both[k], enc[k] if is_enc else dec[k]), k
    with pytest.raises(ValueError):
        synthetic_state_dict(cfg, encoder_profile="gamma_spread")
