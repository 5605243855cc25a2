"""WER / CER restatement (whisper_medusa_b200/metrics.py, reference whisper_medusa/utils/metrics.py:5-71 on
jiwer 3.0.3) and the evaluation driver (whisper_medusa_b200/eval.py, reference eval_whisper_medusa.py:21-96).
jiwer is not installed here, so the known answers below are worked by hand from its documented transforms."""
import struct
import wave

import numpy as np
import pytest

from whisper_medusa_b200.eval import evaluate_rows, load_audio
from whisper_medusa_b200.metrics import (cer_standardize, compute_cer, compute_wer, edit_distance,
                                          wer_standardize)


def test_edit_distance_known_answers():
    assert edit_distance("kitten", "sitting") == 3
    assert edit_distance([], ["a", "b"]) == 2
    assert edit_distance(["a", "b", "c"], ["a", "b", "c"]) == 0
    assert edit_distance(["a", "b", "c"], ["a", "c"]) == 1
    assert edit_distance("flaw", "lawn") == 2
    # symmetric
    assert edit_distance("intention", "execution") == edit_distance("execution", "intention") == 5


def test_wer_transforms_follow_jiwer_chain():
    # lower-case, contractions ("won't" before the generic n't), kaldi non-words, punctuation, spaces
    assert wer_standardize("I won't  go,\tshe CAN'T!") == ["i", "will", "not", "go", "she", "can", "not"]
    assert wer_standardize("Let's see: it's [laughter] <unk> fine.") == ["let", "us", "see", "it", "is", "fine"]
    assert wer_standardize("they're  we've I'm he'd you'll") == ["they", "are", "we", "have", "i", "am", "he", "would", "you", "will"]
    assert wer_standardize("  ...  ") == []
    # unicode punctuation (category P*) goes, letters with accents stay
    assert wer_standardize("¿Qué tal? — «bien»") == ["qué", "tal", "bien"]


def test_cer_transforms_keep_inner_spaces():
    assert cer_standardize("Ab, c!") == list("ab c")
    assert cer_standardize("a\t\tb") == list("a b")


def test_corpus_scores_match_hand_computation():
    refs = ["the cat sat on the mat", "hello world", ""]
    hyps = ["the cat sat on mat", "hello there world", "something"]
    # utt 0: 1 deletion / 6 words; utt 1: 1 insertion / 2 words; utt 2: reference -> "EMPTY": 1 substitution / 1 word
    wer, wers = compute_wer(hyps, refs)
    assert wers == pytest.approx([1 / 6, 1 / 2, 1.0])
    assert wer == pytest.approx(3 / 9)
    cer, cers = compute_cer(["abc"], ["abd"])
    assert cers == pytest.approx([1 / 3]) and cer == pytest.approx(1 / 3)
    # both sides empty: "EMPTY" vs "EMPTY" -> 0 errors over 1 word
    wer, wers = compute_wer(["", "a"], ["...", "a"])
    assert wers == [0.0, 0.0] and wer == 0.0
    # corpus score is the pooled ratio, not the mean of the ratios
    wer, wers = compute_wer(["a b c d", "x"], ["a b c e", "y"])
    assert wer == pytest.approx(2 / 5) and np.mean(wers) == pytest.approx((1 / 4 + 1) / 2)


def _write_wav(path, x, sr, width=2, channels=1):
    with wave.open(path, "wb") as w:
        w.setnchannels(channels)
        w.setsampwidth(width)
        w.setframerate(sr)
        if width == 2:
            data = (np.clip(x, -1, 1) * 32767).astype("<i2")
        else:
            data = (np.clip(x, -1, 1) * 2147483647).astype("<i4")
        if channels > 1:
            data = np.repeat(data[:, None], channels, axis=1)
        w.writeframes(data.tobytes())


def test_audio_loading_and_driver(tmp_path):
    t = np.arange(16000) / 16000.0
    tone = 0.25 * np.sin(2 * np.pi * 440 * t).astype(np.float32)
    p16 = str(tmp_path / "a.wav")
    _write_wav(p16, tone, 16000)
    x = load_audio(p16)
    assert x.dtype == np.float32 and x.shape == (16000,) and np.abs(x - tone).max() < 1e-4
    p2 = str(tmp_path / "b.wav")
    _write_wav(p2, tone, 16000, width=4, channels=2)     # stereo 32-bit: first channel
    assert np.abs(load_audio(p2) - tone).max() < 1e-6
    p8 = str(tmp_path / "c.wav")
    _write_wav(p8, tone[::2], 8000)                        # 8 kHz -> resampled to 16 kHz
    y = load_audio(p8)
    assert abs(len(y) - 16000) <= 2
    # the driver: transcribe is injected (the GPU path has its own tests), columns as in the reference
    rows = [{"audio": p16, "sentence": "hello world", "language": "en"}, {"audio": p2, "sentence": "good bye"},
            {"audio": p8, "sentence": float("nan")}]
    said = {p16: "hello word", p2: "good bye", p8: ""}
    calls = []

    def transcribe(pcm, lang):
        calls.append((len(pcm), lang))
        return list(said.values())[len(calls) - 1]

    wer, cer, table = evaluate_rows(rows, transcribe, default_language="en")
    assert [c[1] for c in calls] == ["en", "en", "en"]
    assert list(table) == ["audio", "label", "prediction", "wer", "cer", "language"]
    assert table["label"] == ["hello world", "good bye", ""]
    assert table["wer"] == pytest.approx([0.5, 0.0, 0.0])
    assert wer == pytest.approx(1 / 5)          # 1 error over 2 + 2 + 1 ("EMPTY") words
    assert 0 < cer < 0.1
