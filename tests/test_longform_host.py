"""Long-form transcription, host side (no GPU): the window plan and the merge against the installed transformers'
own functions, the resampler oracle against torchaudio, the engine's resampler tap table against the oracle, and the
argument errors."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from oracle import resample_ref as R
from whisper_medusa_b200 import WhisperMedusaModel
from whisper_medusa_b200.longform import (MAX_WINDOW_SAMPLES, merge_windows, plan_windows, resampled_length, text_ids,
                                          window_params)
from whisper_medusa_b200.synthetic import preset_config

RATES = (8000, 22050, 44100, 48000, 96000, 16000)


# ---------------------------------------------------------------------------------------------------- window plan
class _StubExtractor:
    """Stands in for WhisperFeatureExtractor inside chunk_iter: reports where each chunk starts."""
    sampling_rate = 16000

    def __call__(self, chunk, sampling_rate, return_tensors, return_attention_mask):
        return {"first": int(chunk[0]) if len(chunk) else -1}


def _hf_plan(n, chunk_length_s, stride_length_s):
    from transformers.pipelines.automatic_speech_recognition import chunk_iter

    chunk_len, left, right = window_params(chunk_length_s, stride_length_s)
    out = []
    for item in chunk_iter(np.arange(n, dtype=np.int64), _StubExtractor(), chunk_len, left, right):
        length, l, r = item["stride"]
        out.append((item["first"], item["first"] + length, l, r))
    return out


@pytest.mark.parametrize("n", [0, 1, 479999, 480000, 480001, 800000, 720000, 5 * 60 * 16000])
def test_window_plan_matches_chunk_iter(n):
    # 720000: the samples past the last full step (80000 = stride_left) lie inside the previous window, which is the
    # last one
    pytest.importorskip("transformers")
    mine = [tuple(w) for w in plan_windows(n, *window_params(30.0, None))]
    assert mine == _hf_plan(n, 30.0, None)
    assert all(w[1] - w[0] <= MAX_WINDOW_SAMPLES for w in mine)
    if n:
        assert mine[0][2] == 0 and mine[-1][3] == 0 and mine[-1][1] == n
    else:
        assert mine == []


@pytest.mark.parametrize("chunk_s,stride", [(10.0, 2.0), (20.0, [4.0, 1.0]), (30.0, 0.0), (12.5, None), (30.0, [0, 9.5])])
@pytest.mark.parametrize("n", [1, 159999, 160000, 200001, 1234567, 3 * 480000])
def test_window_plan_non_default_strides(chunk_s, stride, n):
    pytest.importorskip("transformers")
    mine = [tuple(w) for w in plan_windows(n, *window_params(chunk_s, stride))]
    assert mine == _hf_plan(n, chunk_s, stride)


def test_window_params():
    assert window_params() == (480000, 80000, 80000)
    assert window_params(30.0, [3.0, 1.0]) == (480000, 48000, 16000)
    assert window_params(15) == (240000, 40000, 40000)
    for bad in (dict(chunk_length_s=30.01), dict(chunk_length_s=0), dict(chunk_length_s=-1.0),
                dict(chunk_length_s=float("nan")), dict(chunk_length_s=10.0, stride_length_s=6.0),
                dict(chunk_length_s=10.0, stride_length_s=5.0), dict(chunk_length_s=10.0, stride_length_s=[-1.0, 1.0])):
        with pytest.raises(ValueError):
            window_params(**bad)


# ---------------------------------------------------------------------------------------------------- merge
def _hf_merge(seqs):
    from transformers.models.whisper.tokenization_whisper import _find_longest_common_sequence

    return [int(t) for t in _find_longest_common_sequence([list(s) for s in seqs])]


def _overlapping_windows(rng, n_tokens, n_windows, overlap, vocab, flip=0.0):
    text = rng.integers(0, vocab, n_tokens).tolist()
    step = max(1, n_tokens // n_windows)
    out = []
    for k in range(n_windows):
        w = list(text[max(0, k * step - overlap): min(n_tokens, (k + 1) * step + overlap)])
        for i in range(len(w)):
            if rng.random() < flip:
                w[i] = int(rng.integers(0, vocab))
        out.append(w)
    return out


def test_merge_matches_find_longest_common_sequence():
    pytest.importorskip("transformers")
    rng = np.random.default_rng(7)
    cases = []
    for seed_case in range(40):
        n_w = int(rng.integers(1, 6))
        cases.append(_overlapping_windows(rng, int(rng.integers(0, 300)), n_w, int(rng.integers(0, 40)),
                                          int(rng.choice([5, 50, 50000])), flip=float(rng.choice([0.0, 0.02, 0.2]))))
    cases += [
        [[1, 2, 3, 4, 5]],                                   # a single window
        [[1, 2, 3, 4], [3, 4, 5, 6], [5, 6, 7, 8]],          # clean overlaps
        [[1, 2, 3], [7, 8, 9]],                              # disjoint windows
        [[], [1, 2, 3], []],                                 # empty windows
        [[], []],
        [[1, 2, 3, 4], [], [3, 4, 5]],
        [[10, 11, 12, 13, 14], [12, 99, 14, 15, 16]],        # the overlap disagrees in one token
        [[10, 11, 12, 13, 14, 15], [12, 13, 77, 15, 16, 17]],
        [[5, 5, 5, 5, 5], [5, 5, 5, 5, 5, 6]],               # runs of one token
        [[1, 7, 7, 7, 7, 2], [7, 7, 7, 2, 3]],
        [[4, 4], [4], [4, 4, 4]],
    ]
    for seqs in cases:
        assert merge_windows(seqs) == _hf_merge(seqs), seqs
    assert merge_windows([]) == []


def test_text_ids_drop_the_special_block():
    assert text_ids([50257, 11, 50362, 300, 50256, 12], 50256) == [11, 300, 12]
    assert text_ids([], 3) == []


# ---------------------------------------------------------------------------------------------------- resampler
def _signal(n, sr, seed=0):
    """Peak-0.5 test audio at rate sr: harmonics up to near Nyquist plus white noise."""
    rng = np.random.default_rng(seed)
    t = np.arange(n) / sr
    x = 0.02 * rng.standard_normal(n)
    for f in (110.0, 440.0, 3000.0, 0.45 * sr):
        x += rng.uniform(0.2, 1.0) * np.sin(2 * np.pi * f * t + rng.uniform(0, 2 * np.pi))
    return (0.5 * x / max(1e-9, np.abs(x).max())).astype(np.float32) if n else np.zeros(0, np.float32)


@pytest.mark.parametrize("sr", RATES)
def test_resample_oracle_matches_torchaudio(sr):
    """The oracle equals torchaudio.functional.resample on the same samples: within 1e-6 of its run on fp64 samples
    (fp64 taps; the oracle's are those taps rounded to fp32, as the engine's), within 2e-5 of its run on fp32 samples
    (taps evaluated in fp32 arithmetic)."""
    AF = pytest.importorskip("torchaudio.functional")
    for n in (0, 1, 12347, 60 * sr):
        x = _signal(n, sr, seed=n % 97)
        y = R.resample(x, sr, 16000)
        assert y.shape == (resampled_length(n, sr, 16000),) == (R.resampled_length(n, sr, 16000),)
        if n == 0:
            continue                             # (torchaudio cannot reshape an empty waveform)
        ref64 = AF.resample(torch.from_numpy(x).double(), sr, 16000).numpy()
        ref32 = AF.resample(torch.from_numpy(x), sr, 16000).double().numpy()
        assert ref64.shape == y.shape
        assert np.abs(y - ref64).max() <= 1e-6, (sr, n, np.abs(y - ref64).max())
        assert np.abs(y - ref32).max() <= 2e-5, (sr, n, np.abs(y - ref32).max())
        if sr == 16000:
            assert np.array_equal(y, x.astype(np.float64))


def _lib_taps(lib, orig_hz, new_hz):
    info = (C.c_int32 * 4)()
    assert lib.wm_resample_taps(orig_hz, new_hz, None, None, None, 0, info) == 0
    orig, new, width, max_taps = list(info)
    taps = np.zeros(new * max_taps, np.float32)
    lo = np.zeros(new, np.int32)
    cnt = np.zeros(new, np.int32)
    P = lambda a, t: a.ctypes.data_as(C.POINTER(t))  # noqa: E731
    assert lib.wm_resample_taps(orig_hz, new_hz, P(taps, C.c_float), P(lo, C.c_int32), P(cnt, C.c_int32), taps.size, info) == 0
    return (orig, new, width, max_taps), taps.reshape(new, max_taps), lo, cnt


@pytest.mark.parametrize("sr", [r for r in RATES if r != 16000] + [16001])
def test_engine_tap_table_matches_the_oracle(engine_lib, sr):
    """wm_resample_taps (fp64 build, one rounding to fp32) holds exactly the oracle's taps, the oracle's taps are
    exactly torchaudio's own fp64 kernel rounded to fp32, and every tap outside a phase's support is zero."""
    dense, width = R.sinc_taps(sr, 16000)
    (orig, new, w, max_taps), taps, lo, cnt = _lib_taps(engine_lib, sr, 16000)
    assert (orig, new) == R.reduced_rates(sr, 16000) and w == width and dense.shape == (new, 2 * width + orig)
    for p in range(new):
        got = taps[p, : cnt[p]]
        assert np.array_equal(got.view(np.uint32), dense[p, lo[p]: lo[p] + cnt[p]].view(np.uint32)), p
        assert not np.any(taps[p, cnt[p]:])
        outside = np.concatenate([dense[p, : lo[p]], dense[p, lo[p] + cnt[p]:]])
        assert np.all(outside == 0), p
        assert cnt[p] > 0 and got[0] != 0 and got[-1] != 0
    assert max_taps <= 2 * width + 2
    if sr != 16001:
        tf = pytest.importorskip("torchaudio.functional.functional")
        k, kw = tf._get_sinc_resample_kernel(sr, 16000, math.gcd(sr, 16000), dtype=torch.float64)
        k32 = k[:, 0, :].float().numpy()
        assert kw == width and np.array_equal(k32.view(np.uint32), dense.view(np.uint32))
    if sr == 44100:
        assert (new, 2 * width + orig) == (160, 475) and 33 <= max_taps <= 35


def test_resample_taps_argument_errors(engine_lib):
    info = (C.c_int32 * 4)()
    assert engine_lib.wm_resample_taps(0, 16000, None, None, None, 0, info) != 0
    assert engine_lib.wm_resample_taps(44100, -1, None, None, None, 0, info) != 0
    assert engine_lib.wm_resample_taps(44100, 16000, None, None, None, 0, None) != 0
    taps = (C.c_float * 10)()
    lo = (C.c_int32 * 160)()
    cnt = (C.c_int32 * 160)()
    assert engine_lib.wm_resample_taps(44100, 16000, taps, lo, cnt, 10, info) != 0      # capacity too small
    n = C.c_int64()
    assert engine_lib.wm_resample(None, None, 0, 44100, 16000, None, 0, C.byref(n), None) != 0


# ---------------------------------------------------------------------------------------------------- host API errors
def _fake_engine(preset="micro"):
    m = WhisperMedusaModel(preset_config(preset, heads=4), None)
    m._handle = C.c_void_p(1)      # pretend an engine exists: the argument checks come first
    return m


def test_transcribe_argument_errors():
    m = _fake_engine()
    try:
        x = np.zeros(16000, np.float32)
        with pytest.raises(ValueError):
            m.transcribe(x, chunk_length_s=31.0)                         # beyond one encoder window
        with pytest.raises(ValueError):
            m.transcribe(np.zeros((2, 16000), np.float32))               # multi-channel: downmix first
        with pytest.raises(ValueError):
            m.transcribe(torch.zeros(1, 16000))
        with pytest.raises(ValueError):
            m.transcribe(x, chunk_length_s=10.0, stride_length_s=6.0)    # HF: chunk_len < left + right
        with pytest.raises(ValueError):
            m.transcribe(x, sampling_rate=44100.5)                       # integer rates only
        with pytest.raises(ValueError):
            m.transcribe(x, sampling_rate=0)
        with pytest.raises(NotImplementedError):
            m.transcribe(x, return_timestamps=True)
        with pytest.raises(NotImplementedError):
            m.transcribe(x, temperature=0.4)
        with pytest.raises(ValueError):
            m.generate_from_pcm(x, sampling_rate=-8000)
    finally:
        m._handle = None
    with pytest.raises(Exception):
        WhisperMedusaModel(preset_config("micro", heads=4), None).transcribe(np.zeros(10, np.float32))   # no engine


def test_short_form_refusals_still_hold():
    """generate() and generate_from_pcm() keep refusing more than 30 s, at 16 kHz and after resampling."""
    m = _fake_engine()
    try:
        with pytest.raises(NotImplementedError):
            m.generate(torch.zeros(1, 80, 6000))
        with pytest.raises(NotImplementedError):
            m.generate_from_pcm(np.zeros(480001, np.float32))
        with pytest.raises(NotImplementedError):
            m.generate_from_pcm(np.zeros(31 * 48000, np.float32), sampling_rate=48000)
        assert resampled_length(30 * 44100, 44100, 16000) == 480000
        with pytest.raises(NotImplementedError):
            m.generate_from_pcm(np.zeros(30 * 44100 + 3, np.float32), sampling_rate=44100)     # 480002 samples at 16 kHz
    finally:
        m._handle = None
