"""Long-form transcription on the GPU: the resampler kernel against the fp64 oracle (oracle/resample_ref.py), the
device-window frontend against the host-PCM frontend, and transcribe() / StreamGroup.transcribe() against per-window
generate calls and the package's merge.  The CPU suite (test_longform_host.py) pins the oracle to torchaudio and the
window plan and merge to transformers, so nothing here needs either library."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import resample_ref as R
from oracle import whisper_ref as W
from whisper_medusa_b200 import StreamGroup, WhisperMedusaModel, _lib
from whisper_medusa_b200.longform import Window, merge_windows, plan_windows, text_ids, window_params
from whisper_medusa_b200.synthetic import preset_config, synthetic_audio, synthetic_state_dict

pytestmark = pytest.mark.gpu

RATES = (8000, 22050, 44100, 48000, 96000, 16000)
# Worst |engine - oracle| measured over 10 minutes of peak-0.5 audio at each of RATES: 2.3e-7 (96 kHz), on an H100 80GB
# HBM3 at a 700 W power limit (tests/gpu_longform.py; DESIGN.md section 7): the fp32 FMA chain against the fp64 sum of the same fp32 taps.
RESAMPLE_BAR = 1e-6

_MODELS = {}


def _model(preset, heads=4):
    if preset not in _MODELS:
        cfg = preset_config(preset, heads=heads)
        sd = synthetic_state_dict(cfg, seed=11)
        _MODELS[preset] = (WhisperMedusaModel(cfg, sd).to("cuda:0"), sd)
    return _MODELS[preset]


def _recording(seconds, first_stream=0):
    """A 16 kHz recording made of consecutive synthetic clips (each at most 25 s)."""
    parts, left, k = [], float(seconds), first_stream
    while left > 0:
        s = min(25.0, left)
        parts.append(synthetic_audio(s, stream_id=k))
        left -= s
        k += 1
    return np.concatenate(parts).astype(np.float32) if parts else np.zeros(0, np.float32)


def _at_rate(x16, sr):
    """The 16 kHz recording played at another rate (oracle resampling, rounded to f32)."""
    return R.resample(x16, 16000, sr).astype(np.float32)


def _signal(n, sr, seed=0):
    rng = np.random.default_rng(seed)
    t = np.arange(n) / sr
    x = 0.02 * rng.standard_normal(n)
    for f in (110.0, 440.0, 3000.0, 0.45 * sr):
        x += rng.uniform(0.2, 1.0) * np.sin(2 * np.pi * f * t + rng.uniform(0, 2 * np.pi))
    return (0.5 * x / max(1e-9, np.abs(x).max())).astype(np.float32) if n else np.zeros(0, np.float32)


def _resample_dev(model, x_dev, sr_in, sr_out):
    lib = _lib.load()
    n_out = R.resampled_length(x_dev.numel(), sr_in, sr_out)
    y = torch.full((max(1, n_out),), float("nan"), device="cuda:0")
    got = C.c_int64(-1)
    stream = torch.cuda.current_stream().cuda_stream
    rc = lib.wm_resample(model._handle, C.c_void_p(x_dev.data_ptr()), x_dev.numel(), sr_in, sr_out,
                         C.c_void_p(y.data_ptr()), n_out, C.byref(got), C.c_void_p(stream))
    assert rc == 0, lib.wm_last_error(model._handle)
    assert got.value == n_out
    return y[:n_out]


@pytest.mark.parametrize("sr", RATES)
def test_resampler_kernel_vs_oracle(sr):
    model, _ = _model("micro")
    for n in (0, 1, 12347, 60 * sr, 600 * sr):
        x = _signal(n, sr, seed=n % 101)
        xd = torch.from_numpy(x).to("cuda:0")
        y = _resample_dev(model, xd, sr, 16000).cpu().numpy()
        ref = R.resample(x, sr, 16000)
        assert y.shape == ref.shape, (sr, n)
        if n:
            err = float(np.abs(y.astype(np.float64) - ref).max())
            assert err <= RESAMPLE_BAR, (sr, n, err)
        if sr == 16000:
            assert np.array_equal(y.view(np.uint32), x.view(np.uint32))        # a device copy: bit-exact
        # transcribe's upload path: the same kernel, the same bits
        y2 = model._upload_16k(xd, sr).cpu().numpy()
        assert np.array_equal(y2.view(np.uint32), y.view(np.uint32))


def _window_mel(model, x16_dev, w):
    model._encode_window(x16_dev, w, torch.cuda.current_stream().cuda_stream)
    return model.mel().numpy()


@pytest.mark.parametrize("mode", ["persistent", "graph"])
@pytest.mark.parametrize("preset", ["micro", "tiny.en"])
def test_16k_windows_equal_short_clips(preset, mode):
    """75 s at 16 kHz -> 4 windows: every window's mel and tokens are bit-identical to generate_from_pcm on the host-
    sliced samples; the merged ids are the package's merge of those ids; a CUDA tensor input gives the same result."""
    model, _ = _model(preset)
    model.set_decode_mode(mode)
    eos = int(model.generation_config.eos_token_id)
    x = _recording(75.0)
    out = model.transcribe(x, max_length=160)[0].tolist()
    wins = model.last_windows
    plan = plan_windows(len(x), *window_params())
    assert [(r.start, r.end, r.stride_left, r.stride_right) for r in wins] == [tuple(w) for w in plan]
    assert len(wins) == 4
    x_dev = torch.from_numpy(x).to("cuda:0")
    per_window = []
    for r in wins:
        ids = model.generate_from_pcm(x[r.start:r.end], max_length=160)[0].tolist()
        mel_host = model.mel().numpy()
        assert ids == r.ids, (r, ids, r.ids)
        mel_dev = _window_mel(model, x_dev, Window(r.start, r.end, 0, 0))
        assert np.array_equal(mel_dev.view(np.uint32), mel_host.view(np.uint32)), r
        per_window.append(text_ids(ids, eos))
    assert out == merge_windows(per_window)
    assert model.transcribe(x_dev, max_length=160)[0].tolist() == out
    model.set_decode_mode("persistent")


@pytest.mark.parametrize("sr", [44100, 48000])
def test_resampled_windows(sr):
    """At 44.1 / 48 kHz every window's mel is within 5e-5 of the oracle log-mel of the oracle-resampled slice, and its
    tokens are those of generate(input_features=<that window's engine mel>)."""
    model, _ = _model("tiny.en")
    x16 = _recording(70.0, first_stream=5)
    x = _at_rate(x16, sr)
    out = model.transcribe(x, sampling_rate=sr, max_length=160)[0].tolist()
    wins = model.last_windows
    assert len(wins) == len(plan_windows(R.resampled_length(len(x), sr, 16000), *window_params())) >= 3
    ref16 = R.resample(x, sr, 16000).astype(np.float32)
    x16_dev = model._upload_16k(torch.from_numpy(x).to("cuda:0"), sr)
    per_window = []
    for r in wins:
        mel = _window_mel(model, x16_dev, Window(r.start, r.end, 0, 0))
        want = W.log_mel_spectrogram(ref16[r.start:r.end])
        assert np.abs(mel - want).max() <= 5e-5, (r, float(np.abs(mel - want).max()))
        ids = model.generate(torch.from_numpy(mel)[None], max_length=160)[0].tolist()
        assert ids == r.ids, r
        per_window.append(text_ids(ids, int(model.generation_config.eos_token_id)))
    assert out == merge_windows(per_window)
    # generate_from_pcm at the same rate: one clip of at most 30 s, resampled on the GPU
    clip = x[: 20 * sr]
    ids = model.generate_from_pcm(clip, sampling_rate=sr, max_length=160)[0].tolist()
    mel = model.mel().numpy()
    assert np.abs(mel - W.log_mel_spectrogram(R.resample(clip, sr, 16000).astype(np.float32))).max() <= 5e-5
    assert ids == model.generate(torch.from_numpy(mel)[None], max_length=160)[0].tolist()


def test_short_recording_is_one_window():
    model, _ = _model("tiny.en")
    eos = int(model.generation_config.eos_token_id)
    for seconds in (3.0, 30.0):
        x = _recording(seconds, first_stream=9)
        got = model.transcribe(x, max_length=160)[0].tolist()
        assert len(model.last_windows) == 1
        ref = model.generate_from_pcm(x, max_length=160)[0].tolist()
        assert got == text_ids(ref, eos)
    assert model.transcribe(np.zeros(0, np.float32))[0].tolist() == [] and model.last_windows == []
    assert tuple(model.transcribe(np.zeros(0, np.float32), sampling_rate=44100).shape) == (1, 0)


def test_stream_group_transcribe_equals_model_transcribe():
    model, sd = _model("tiny.en")
    cfg = model.config
    recs = [_recording(75.0, first_stream=20), _at_rate(_recording(40.0, first_stream=30), 44100),
            _at_rate(_recording(20.0, first_stream=40), 48000)]
    rates = [16000, 44100, 48000]
    want, want_windows = [], []
    for x, sr in zip(recs, rates):
        want.append(model.transcribe(x, sampling_rate=sr, max_length=160)[0].tolist())
        want_windows.append([r.ids for r in model.last_windows])
    for S in (2, 4):
        grp = StreamGroup(cfg, None, "cuda:0", n_streams=S, weights_from=model)
        one = grp.transcribe(recs[0], max_length=160)
        assert len(one) == 1 and one[0][0].tolist() == want[0], S
        got = grp.transcribe(recs, sampling_rate=rates, max_length=160)
        assert [g[0].tolist() for g in got] == want, S
        assert [[r.ids for r in ws] for ws in grp.last_windows] == want_windows, S
        assert len(grp.last_traces) == sum(len(w) for w in want_windows) == 4 + 2 + 1
        grp.close()


def test_stream_group_transcribe_large_v2():
    for m, _ in _MODELS.values():
        m.close()
    _MODELS.clear()
    cfg = preset_config("large-v2", heads=10)
    sd = synthetic_state_dict(cfg, seed=0)
    model = WhisperMedusaModel(cfg, sd).to("cuda:0")
    kw = dict(language="en", posterior_alpha=100.0)
    x = _recording(70.0, first_stream=50)
    want = model.transcribe(x, **kw)[0].tolist()
    assert len(model.last_windows) == 3
    grp = StreamGroup(cfg, None, "cuda:0", n_streams=2, weights_from=model)
    assert grp.transcribe([x], **kw)[0][0].tolist() == want
    grp.close()
    model.close()
