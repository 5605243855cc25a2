"""Encoder and log-mel frontend against the fp64 oracle (DESIGN.md section 2, "Encoder and frontend against fp64").

Encoder checks start from the engine's own mel (``model.mel()``), so the frontend is checked on its own (group D).  The
reference is ``encoder_forward`` in fp64 with the engine's fp16 rounding points; the fp32 oracle's error against the
same reference is the floor, printed and recorded beside the engine's.  Two metrics over all 1500 x d states, each with
its own bar: max |diff| / max(1, max|ref|), and the relative RMS, which sees small systematic errors that hide under the
flip noise of single fp16 ulps.  The max metric is also asserted over rows 0-31 and 1408-1499 alone (the first tiles,
and the last query tile of the attention, whose last 64-key block is partial, and the last M tile of every GEMM).
``WM_NUMERICS_RECORD=<file>`` records the errors instead of asserting the bars (tests/_decode_ref.py).

Groups: A widths x inputs (default profile), B encoder activation profiles, C implementation matrix (enc_gemm 1 / 2 / 0
x enc_attn 1 / 0, enc_pdl 0), D frontend, E scratch isolation between clips."""
import numpy as np
import pytest
import torch

from _decode_ref import DECODE_LOGIT_BAR, check_error, check_logits, decode_logits, rel_err
from oracle import whisper_ref as W
from test_oracle_encoder_fp64 import tail_only_mel
from whisper_medusa_b200.synthetic import ENCODER_PROFILES, synthetic_audio, synthetic_state_dict, width_config

pytestmark = pytest.mark.gpu

#: encoder states against the fp64 engine-regime oracle, about 3x the worst measured on an H100 (DESIGN.md section 2):
#: max |diff| / max(1, max|ref|) on the default profile (worst 4.6e-4; the fp32 oracle 4.1e-4) and under the activation
#: profiles (worst 3.0e-3 under `outliers`, whose fp32 oracle is 3.1e-3 off), relative RMS (worst 4.0e-4)
ENC_MAX_BAR = 1.5e-3
ENC_MAX_BAR_PROFILES = 1e-2
ENC_RMS_BAR = 1.2e-3
#: log-mel: max |diff| against the fp64 log-mel (worst 3.7e-5, with a DC offset; the fp32 oracle 3.4e-5)
MEL_BAR = 1.1e-4

WIDTHS = (128, 384, 512, 640, 768, 1024, 1280)
A_MODELS = [(d, 0) for d in WIDTHS] + [(768, 768)]
INPUTS = ("speech30", "clip5", "mel_random", "mel_left", "mel_tail", "mel_const")
B_INPUTS = ("speech30", "mel_tail")
PROFILES = [p for p in ENCODER_PROFILES if p != "default"]
EDGE_ROWS = {"rows0-31": slice(0, 32), "rows1408-1499": slice(1408, 1500)}
_KW = dict(language=None, max_length=60)


def _mid(d, ffn, profile):
    return f"d{d}" + (f"-ffn{ffn}" if ffn else "") + ("" if profile == "default" else f"-{profile}")


def _designed_mel(kind):
    rng = np.random.default_rng(7)
    if kind == "mel_random":
        return rng.uniform(-1.0, 1.5, (80, 3000))
    if kind == "mel_left":                       # content in frames 0-63 only (conv1's left pad, the first tiles)
        m = np.full((80, 3000), -0.5)
        m[:, :64] = rng.uniform(-1.0, 1.5, (80, 64))
        return m
    if kind == "mel_tail":                       # frames 2944-2999: encoder rows 1472-1499
        return tail_only_mel(7)
    if kind == "mel_const":                      # every row the same up to positions: near-uniform attention
        return np.full((80, 3000), 0.3)
    raise AssertionError(kind)


_MODEL = {}


def _model(d, ffn=0, profile="default"):
    """(model, cfg, sd); one engine alive at a time."""
    from whisper_medusa_b200 import WhisperMedusaModel

    key = (d, ffn, profile)
    if key not in _MODEL:
        for m in _MODEL.values():
            m[0].close()
        _MODEL.clear()
        cfg = width_config(d, heads=4, ffn_dim=ffn)
        sd = synthetic_state_dict(cfg, seed=3 + WIDTHS.index(d), encoder_profile=profile)
        _MODEL[key] = (WhisperMedusaModel(cfg, sd).to("cuda:0"), cfg, sd)
    return _MODEL[key]


def _encode(model, inp, seed):
    """Run the engine's frontend + encoder on an input; returns (mel, encoder states) as the engine holds them."""
    if inp.startswith("mel_"):
        feats = torch.from_numpy(_designed_mel(inp).astype(np.float32))[None]
        model.generate(input_features=feats, max_iters=1, **_KW)
    else:
        pcm = synthetic_audio(30.0 if inp == "speech30" else 5.0, stream_id=seed)
        model.generate_from_pcm(pcm, max_iters=1, **_KW)
    return model.mel(), model.encoder_output()


_REF = {}


def _ref(key, cfg, sd, mel):
    """(fp64, fp32) engine-regime oracle states of one (model, input), cached."""
    if key not in _REF:
        torch.set_num_threads(16)
        r64 = W.encoder_forward(W.RefWeights(sd, torch.float64), cfg, mel.double(), "engine")
        r32 = W.encoder_forward(W.RefWeights(sd), cfg, mel, "engine")
        _REF[key] = (r64, r32)
    return _REF[key]


def _rel_rms(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.sqrt(((a - b) ** 2).mean() / (b ** 2).mean()))


def check_states(enc, r64, r32, case, what="states", max_bar=ENC_MAX_BAR):
    """Both metrics over all states, and the max metric over the edge rows; returns the worst max metric."""
    e, r, f = enc.numpy(), r64.numpy(), r32.double().numpy()
    assert np.isfinite(e).all(), (case, what, "non-finite encoder states")
    worst = check_error(rel_err(e, r), max_bar, case, f"{what}/max", rel_err(f, r))
    check_error(_rel_rms(e, r), ENC_RMS_BAR, case, f"{what}/rms", _rel_rms(f, r))
    for name, rows in EDGE_ROWS.items():
        worst = max(worst, check_error(rel_err(e[rows], r[rows]), max_bar, case, f"{what}/max-{name}",
                                       rel_err(f[rows], r[rows])))
    return worst


def _with_options(model, opts, fn):
    try:
        for k, v in opts.items():
            model.set_option(k, v)
        return fn()
    finally:
        for k, v in (("enc_gemm", 1), ("enc_attn", 1), ("enc_pdl", 1)):
            model.set_option(k, v)


def _check_case(d, ffn, profile, inp):
    model, cfg, sd = _model(d, ffn, profile)
    seed = 3 + WIDTHS.index(d)
    mel, enc = _encode(model, inp, seed)
    case = f"{_mid(d, ffn, profile)}/{inp}"
    r64, r32 = _ref(case, cfg, sd, mel)
    worst = check_states(enc, r64, r32, case, max_bar=ENC_MAX_BAR if profile == "default" else ENC_MAX_BAR_PROFILES)
    # 128 x 128 tiles only: a tile's K loop is the same, so the same bits whatever tiles the width picks
    _, enc128 = _with_options(model, {"enc_gemm": 2}, lambda: _encode(model, inp, seed))
    assert torch.equal(enc128, enc), case
    print(f"{case}: worst rel. error vs fp64 {worst:.3g}, fp32 oracle {rel_err(r32.double().numpy(), r64.numpy()):.3g}")


@pytest.mark.parametrize("inp", INPUTS)
@pytest.mark.parametrize("d,ffn", A_MODELS, ids=[_mid(d, f, "default") for d, f in A_MODELS])
def test_a_encoder_every_width_and_input(d, ffn, inp):
    """Group A: every width (and FFN = d at 768) on 30 s of speech-like audio (every row distinct), the 5 s clip, and
    designed mels: random in the real range, content in frames 0-63 only, in frames 2944-2999 only, constant."""
    _check_case(d, ffn, "default", inp)


@pytest.mark.parametrize("inp", B_INPUTS)
@pytest.mark.parametrize("profile", PROFILES)
@pytest.mark.parametrize("d", [512, 1280], ids=["d512", "d1280"])
def test_b_encoder_activation_profiles(d, profile, inp):
    """Group B: every encoder activation profile (synthetic_state_dict(encoder_profile=...)) at d = 512 and 1280."""
    _check_case(d, 0, profile, inp)


@pytest.mark.parametrize("d,ffn", A_MODELS, ids=[_mid(d, f, "default") for d, f in A_MODELS])
def test_c_implementation_matrix(d, ffn):
    """Group C: enc_gemm 1 (wgmma, tiles per GEMM) / 2 (wgmma, 128 x 128) / 0 (mma.sync) x enc_attn 1 (wgmma) / 0
    (mma.sync), and plain launches (enc_pdl 0).  enc_gemm 2 and enc_pdl 0 give the bits of the default; every other
    combination meets the fp64 bars.  enc_gemm 0 writes the cross-K/V through relayout_cross_kv_kernel: the pass-A/B
    logits of one iteration are checked against the fp64 decode oracle from that run's encoder states."""
    model, cfg, sd = _model(d, ffn)
    seed = 3 + WIDTHS.index(d)
    inp = "speech30"
    mel, base = _encode(model, inp, seed)
    case = f"{_mid(d, ffn, 'default')}/{inp}"
    r64, r32 = _ref(case, cfg, sd, mel)
    for g in (1, 2, 0):
        for a in (1, 0):
            _, enc = _with_options(model, {"enc_gemm": g, "enc_attn": a}, lambda: _encode(model, inp, seed))
            if a == 1 and g in (1, 2):
                assert torch.equal(enc, base), (case, g, a)
            else:
                check_states(enc, r64, r32, case, f"enc_gemm{g}-enc_attn{a}")
    _, enc = _with_options(model, {"enc_pdl": 0}, lambda: _encode(model, inp, seed))
    assert torch.equal(enc, base), case

    def run_mma():
        _encode(model, inp, seed)
        return model.encoder_output(), [model.last_logits(i).numpy().copy() for i in (0, 1)]

    enc0, logits = _with_options(model, {"enc_gemm": 0}, run_mma)
    ref = decode_logits(cfg, sd, enc0, _KW, 1)
    for (ab, which) in (("A", 0), ("B", 1)):
        check_logits(logits[which], getattr(ref, f"pass{ab}_logits")[0].numpy(), case, f"enc_gemm0/pass{ab}1")


def _frontend_inputs():
    n = 480000
    t = np.arange(n) / 16000.0
    speech = synthetic_audio(30.0, stream_id=11)
    out = {
        "quiet_1e-4": speech * (1e-4 / 0.5),
        "square_clipped": np.clip(speech * 20.0, -1.0, 1.0),
        "dc_0.3": speech + 0.3,
        "impulse_first": np.eye(1, n, 0)[0],
        "impulse_last": np.eye(1, n, n - 1)[0],
        "tone_bin25": 0.5 * np.sin(2 * np.pi * 1000.0 * t),          # 1000 Hz = bin 25 of the 400-point DFT
        "burst_last_10ms": np.concatenate([np.zeros(n - 160), np.random.default_rng(1).standard_normal(160) * 0.3]),
        "burst_first_10ms": np.concatenate([np.random.default_rng(2).standard_normal(160) * 0.3, np.zeros(n - 160)]),
        "loudest_in_second_half": speech * np.where(t > 22.0, 1.0, 0.05),
    }
    for m in (1, 160, 479999, 480000):
        out[f"n{m}"] = speech[:m]
    return {k: v.astype(np.float32) for k, v in out.items()}


def test_d_frontend_against_fp64_log_mel():
    """Group D: the engine's log-mel against the fp64 log-mel: quiet audio (the floor at max - 8 and the 1e-10 clamp
    engage broadly), clipping, DC offset, impulses at both reflect-padded edges, a tone on a DFT bin, a 10 ms burst as
    the only content in the first or the last frame, the loudest frame in the second half, and clip lengths 1, 160,
    479999 and 480000.  The existing 5e-5 bar against the fp32 oracle holds as well."""
    model, cfg, sd = _model(128)
    for name, pcm in _frontend_inputs().items():
        model.generate_from_pcm(pcm, max_iters=1, **_KW)
        mel = model.mel().numpy()
        ref = W.log_mel_spectrogram(pcm, torch.float64)
        ref32 = W.log_mel_spectrogram(pcm)
        assert np.isfinite(mel).all(), name
        check_error(float(np.abs(mel - ref).max()), MEL_BAR, "frontend", name, float(np.abs(ref32 - ref).max()))
        assert np.abs(mel - ref32).max() < 5e-5, name


def test_e_scratch_does_not_leak_between_clips():
    """Group E: a loud 30 s clip, then a 5 s clip on the same handle: mel, encoder states and one iteration's pass-A/B
    logits are bit-identical to the 5 s clip on a fresh handle (padded rows of the GEMM operands, the attention output,
    conv1's activations and the time-major mel's pad rows carry nothing from the previous clip), for both GEMM kernels."""
    from whisper_medusa_b200 import WhisperMedusaModel

    model, cfg, sd = _model(1280)
    loud = np.clip(synthetic_audio(30.0, stream_id=21) * 2.0, -1.0, 1.0)
    short = synthetic_audio(5.0, stream_id=22)

    def run(m, pcm):
        m.generate_from_pcm(pcm, max_iters=1, **_KW)
        return [m.mel(), m.encoder_output()] + [m.last_logits(i) for i in (0, 1)]

    fresh = WhisperMedusaModel(cfg, sd).to("cuda:0")
    try:
        for g in (1, 0):
            fresh.set_option("enc_gemm", g)
            want = run(fresh, short)
            got = _with_options(model, {"enc_gemm": g}, lambda: (run(model, loud), run(model, short))[1])
            for name, x, y in zip(("mel", "states", "passA", "passB"), got, want):
                assert torch.equal(x, y), (g, name)
    finally:
        fresh.close()
