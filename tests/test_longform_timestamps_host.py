"""Token timestamps of long-form transcription, host side (no GPU): the timed merge, the window offsets and the
(start, end) pairs against the installed transformers' own functions, and the argument errors of
transcribe(return_token_timestamps=True) before any upload.

* The timed merge equals ``_find_longest_common_sequence(sequences, token_timestamp_sequences)``, ids and pairs, on
  randomised overlapping windows with empty windows, ties, repeated ids and times that break a match by their order.
* The offsets and pairs equal what ``_decode_asr(..., return_timestamps="word")`` hands to ``_collate_word_timestamps``
  for the same windows (a stub tokenizer; the strides in seconds as the pipeline's ``postprocess`` converts them).
* A constructed recording on which the timed and the untimed merge disagree, each equal to HF.
* transcribe / StreamGroup.transcribe with the flag on a stand-in engine: each window's frame count reaches the
  extraction, the result is the host functions applied to ``last_windows``, and without the flag nothing changes.
"""
import ctypes as C
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from whisper_medusa_b200 import WhisperMedusaModel, _lib
from whisper_medusa_b200.longform import (SAMPLE_RATE, WindowResult, merge_timed, merge_windows, plan_windows, text_ids,
                                          token_pairs, window_offsets, window_params)
from whisper_medusa_b200.model import GenerateTrace, MedusaGenerateOutput
from whisper_medusa_b200.synthetic import preset_config

EOS = 50257
NOTS = 50363                 # <|notimestamps|>; timestamps begin at NOTS + 1
SOT, SOP = 50258, 50361      # <|startoftranscript|>, <|startofprev|>


def _hf_lcs(seqs, pairs):
    from transformers.models.whisper.tokenization_whisper import _find_longest_common_sequence

    ids, ps = _find_longest_common_sequence([list(s) for s in seqs], [list(p) for p in pairs])
    return [int(t) for t in ids], list(ps)


# ---------------------------------------------------------------------------------------------------- timed merge
def _timed_windows(rng, n_tokens, n_windows, overlap, vocab, flip, jitter):
    """Overlapping windows of one token stream with times: every token has a true (start, end); a window sees it moved
    by up to ``jitter`` s (rounded to 0.01 s as _decode_asr rounds), so overlapping copies are in or out of order."""
    text = rng.integers(0, vocab, n_tokens).tolist()
    t0 = np.cumsum(rng.uniform(0.0, 0.4, n_tokens))
    step = max(1, n_tokens // n_windows)
    seqs, pairs = [], []
    for k in range(n_windows):
        lo, hi = max(0, k * step - overlap), min(n_tokens, (k + 1) * step + overlap)
        ids, ps = [], []
        for j in range(lo, hi):
            tok = int(rng.integers(0, vocab)) if rng.random() < flip else text[j]
            d = float(rng.choice([0.0, jitter * rng.uniform(-1, 1)]))
            s = round(float(t0[j - 1] if j else 0.0) + d, 2)
            ids.append(tok)
            ps.append((s, round(max(s, float(t0[j]) + d), 2)))
        if rng.random() < 0.15:
            ids, ps = [], []                                     # an empty (or skipped) window
        seqs.append(ids)
        pairs.append(ps)
    return seqs, pairs


def test_timed_merge_matches_find_longest_common_sequence():
    pytest.importorskip("transformers")
    rng = np.random.default_rng(11)
    n_cases = 0
    for _ in range(120):
        seqs, pairs = _timed_windows(rng, int(rng.integers(0, 250)), int(rng.integers(1, 6)), int(rng.integers(0, 40)),
                                     int(rng.choice([3, 20, 50000])), float(rng.choice([0.0, 0.05, 0.3])),
                                     float(rng.choice([0.0, 0.02, 0.5])))
        assert merge_windows(seqs, pairs) == _hf_lcs(seqs, pairs), (seqs, pairs)
        n_cases += 1
    a = [(0.0, 0.5), (0.5, 1.0), (1.0, 1.5), (1.5, 2.0)]
    crafted = [
        ([[1, 2, 3, 4]], [a]),                                                   # a single window
        ([[], []], [[], []]),
        ([[1, 2, 3, 4], [], [3, 4, 5]], [a, [], [(1.0, 1.5), (1.5, 2.0), (2.0, 2.5)]]),
        ([[5, 5, 5, 5], [5, 5, 5, 5, 6]], [a, [(1.0, 1.5), (1.0, 1.5), (1.5, 2.0), (1.5, 2.0), (2.0, 2.5)]]),   # ties
        ([[1, 2, 3, 4], [3, 4, 5]], [a, [(1.0, 1.4), (1.5, 2.0), (2.0, 2.5)]]),    # equal start, earlier end: no match
        ([[1, 2, 3, 4], [3, 4, 5]], [a, [(1.0, 1.5), (1.5, 2.0), (2.0, 2.5)]]),    # equal pairs match
        ([[1, 2, 3, 4], [3, 4, 5]], [a, [(0.9, 1.9), (1.4, 2.5), (2.0, 2.5)]]),    # earlier starts: no match
        ([[7, 7, 7, 2], [7, 7, 2, 3]], [a, [(0.5, 1.0), (1.0, 1.5), (1.5, 2.0), (2.0, 2.5)]]),   # repeated ids
    ]
    for seqs, pairs in crafted:
        assert merge_windows(seqs, pairs) == _hf_lcs(seqs, pairs), seqs
    assert merge_windows([], []) == ([], [])
    assert n_cases == 120


def test_timed_and_untimed_merges_can_disagree():
    """The right window hears "3 4 5" earlier than the left one placed them: untimed, the overlap matches and the ids are
    de-duplicated; timed, only "5" is in order (one match is not enough), so both windows are kept whole."""
    pytest.importorskip("transformers")
    from transformers.models.whisper.tokenization_whisper import _find_longest_common_sequence

    seqs = [[1, 2, 3, 4, 5], [3, 4, 5, 6, 7]]
    pairs = [[(0.0, 1.0), (1.0, 2.0), (2.0, 3.0), (3.0, 4.0), (4.0, 5.0)],
             [(1.5, 2.5), (2.5, 3.5), (4.0, 5.0), (5.0, 6.0), (6.0, 7.0)]]
    untimed = merge_windows(seqs)
    timed, timed_pairs = merge_windows(seqs, pairs)
    assert untimed == [1, 2, 3, 4, 5, 6, 7] == [int(t) for t in _find_longest_common_sequence(seqs)]
    assert timed == [1, 2, 3, 4, 5, 3, 4, 5, 6, 7] and timed_pairs == pairs[0] + pairs[1]
    assert (timed, timed_pairs) == _hf_lcs(seqs, pairs)
    assert timed != untimed


# ---------------------------------------------------------------------------------------------------- offsets and pairs
class _StubTokenizer:
    """What _decode_asr reads of a Whisper tokenizer: special ids are the block [EOS, NOTS]; no id decodes to a
    language code."""
    all_special_ids = list(range(EOS, NOTS + 1))

    def convert_tokens_to_ids(self, tok):
        return {"<|notimestamps|>": NOTS, "<|startofprev|>": SOP, "<|startoftranscript|>": SOT}[tok]

    def _strip_prompt(self, token_ids, prompt_token_id, decoder_start_token_id):
        from transformers.models.whisper.tokenization_whisper import WhisperTokenizer

        return WhisperTokenizer._strip_prompt(self, token_ids, prompt_token_id, decoder_start_token_id)

    def decode(self, ids):
        return "".join(f"<|t{int(t)}|>" for t in ids)


def _hf_decode_asr(windows, ids, times, monkeypatch):
    """(tokens, token_timestamps) that _decode_asr(..., return_timestamps="word") hands to _collate_word_timestamps."""
    import transformers.models.whisper.tokenization_whisper as TW

    seen = []
    monkeypatch.setattr(TW, "_collate_word_timestamps",
                        lambda tok, tokens, ts, lang, ret: seen.append((list(tokens), list(ts))) or [])
    outputs = []
    for w, i, t in zip(windows, ids, times):
        stride = (w.end - w.start, w.stride_left, w.stride_right)
        outputs.append({"tokens": torch.tensor([i], dtype=torch.long), "token_timestamps": t[None],
                        "stride": tuple(s / SAMPLE_RATE for s in stride)})      # ASR pipeline postprocess
    TW._decode_asr(_StubTokenizer(), outputs, return_timestamps="word", return_language=False, time_precision=0.02)
    assert len(seen) == 1
    return seen[0]


def _window_tokens(rng, w, text, t_true, specials=True):
    """A window's ids (text from the recording's stream, maybe a special id among them) and its times in seconds from
    the window's start, float32 and non-decreasing, as generate returns them."""
    a, b = w.start / SAMPLE_RATE, w.end / SAMPLE_RATE
    sel = [j for j in range(len(text)) if a <= t_true[j] < b]
    ids = [text[j] for j in sel]
    if specials and ids and rng.random() < 0.5:     # (not <|startofprev|>: HF reads a window starting with it as a prompt)
        ids.insert(int(rng.integers(0, len(ids))), int(rng.choice([t for t in range(EOS, NOTS + 1) if t != SOP])))
    if not ids:
        ids = [int(rng.integers(0, 1000))]
    t = np.sort(np.clip(np.array([t_true[j] - a for j in sel] + [0.0] * (len(ids) - len(sel)))
                        + rng.normal(0, 0.05, len(ids)), 0, (w.end - w.start) / SAMPLE_RATE))
    return ids, torch.from_numpy(t.astype(np.float32))


PLANS = {
    "default_strides": (75 * SAMPLE_RATE, 30.0, None),
    "asymmetric_strides": (100 * SAMPLE_RATE, 30.0, [4.0, 1.0]),
    "short_last_window": (int(61.37 * SAMPLE_RATE), 20.0, [3.5, 2.25]),
    "one_window": (int(17.3 * SAMPLE_RATE), 30.0, None),
}


@pytest.mark.parametrize("plan", list(PLANS))
def test_offsets_and_pairs_match_decode_asr(plan, monkeypatch):
    pytest.importorskip("transformers")
    n, chunk_s, stride = PLANS[plan]
    windows = plan_windows(n, *window_params(chunk_s, stride))
    assert len(windows) >= (1 if plan == "one_window" else 3)
    if plan == "short_last_window":
        assert windows[-1].end - windows[-1].start < windows[0].end - windows[0].start
    for seed in range(4):
        rng = np.random.default_rng(100 * seed + len(plan))
        n_tok = int(n / SAMPLE_RATE * 3)
        t_true = np.sort(rng.uniform(0, n / SAMPLE_RATE, n_tok))
        text = rng.integers(0, [5, 40, 1000, 50000][seed], n_tok).tolist()
        ids, times = zip(*(_window_tokens(rng, w, text, t_true) for w in windows))
        hf_tokens, hf_pairs = _hf_decode_asr(windows, ids, times, monkeypatch)
        offsets = window_offsets(windows)
        pairs = [token_pairs(i, t.tolist(), off, EOS) for i, t, off in zip(ids, times, offsets)]
        got = merge_windows([text_ids(i, EOS) for i in ids], pairs)
        assert got == (hf_tokens, hf_pairs), (plan, seed)
        # the same through the transcription's window results
        results = [WindowResult(w, list(i), None, token_timestamps=t[None], num_frames=0) for w, i, t in zip(windows, ids, times)]
        assert merge_timed(results, EOS) == got
    # HF's offset rule: the first window starts at 0; each next one at the previous start + its step
    assert offsets[0] == 0.0
    for k in range(1, len(windows)):
        assert abs(offsets[k] - windows[k].start / SAMPLE_RATE) < 1e-9


def test_pairs_with_and_without_the_decoder_prompt():
    """HF's short-form sequences carry no decoder prompt; had they carried it, with its times of 0.0, the pairs would be
    the same: the first text id starts at round(0.0 + offset, 2) either way."""
    ids, times = [11, 50359, 12, 13], [0.42, 0.42, 0.97, 1.5]
    for off in (0.0, 24.999999, 53.33):
        plain = token_pairs(ids, times, off, EOS)
        with_prompt = token_pairs([SOT, 50259, 50359, NOTS] + ids, [0.0] * 4 + times, off, EOS)
        assert plain == with_prompt
        assert plain[0] == (round(0.0 + off, 2), round(0.42 + off, 2)) and plain[1] == (round(0.42 + off, 2),
                                                                                            round(0.97 + off, 2))
        assert len(plain) == 3


# ---------------------------------------------------------------------------------------------------- transcribe on a stand-in engine
class _Lib:
    """The C ABI calls a window's decode makes, recorded; token times are 0.25 s per position after the prompt."""

    def __init__(self):
        self.frames = []
        self.heads_sent = []

    def wm_set_option(self, handle, key, value):
        return 0

    def wm_set_alignment_heads(self, handle, arr, n):
        self.heads_sent.append(n)
        return 0

    def wm_token_timestamps(self, handle, n_prompt, n_total, num_frames, width, tp, out, matrix, jumps):
        self.frames.append(num_frames)
        for i in range(n_total):
            out[i] = 0.0 if i < n_prompt else 0.25 * (i - n_prompt + 1) * tp / 0.02
        return 0

    def wm_last_no_speech(self, handle, token, prob, row):
        prob._obj.value = 0.9
        return 0


def _stand_in(monkeypatch, heads=((1, 1),), choices=None):
    """A model whose engine is a stand-in: each window "decodes" ids that depend on its first sample."""
    lib = _Lib()
    monkeypatch.setattr(_lib, "load", lambda: lib)
    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a, **k: SimpleNamespace(cuda_stream=0))
    cfg = preset_config("micro", heads=4)
    if choices is not None:
        cfg.medusa_choices = choices
    m = WhisperMedusaModel(cfg, None)
    m.generation_config.alignment_heads = [list(h) for h in heads] if heads is not None else None
    m._pushed = (tuple(m.generation_config.suppress_tokens or []), tuple(m.generation_config.begin_suppress_tokens or []))
    m._handle = C.c_void_p(1)
    m._upload_16k = lambda audio, sr: torch.as_tensor(audio, dtype=torch.float32).reshape(-1)
    eos = int(m.generation_config.eos_token_id)
    state = {}
    m._encode_window = lambda x16, w, stream: state.update(first=w.start // SAMPLE_RATE)

    def run_loop(prompt, gp):
        k = state["first"]
        tr = GenerateTrace()
        tr.sequences = list(prompt) + [k, k + 1, k + 2, eos, eos]
        tr.n_new_tokens = 4
        return tr

    m._run_loop = run_loop
    m._generate_output = lambda seq, tr, s, lg: MedusaGenerateOutput(seq, None, None, torch.zeros(1, 4), -0.5, [1])
    return m, lib


def test_transcribe_with_timestamps_on_a_stand_in_engine(monkeypatch):
    from whisper_medusa_b200.streams import StreamGroup

    m, lib = _stand_in(monkeypatch)
    eos = int(m.generation_config.eos_token_id)
    x = np.zeros(int(62.5 * SAMPLE_RATE), np.float32)
    plain = m.transcribe(x)
    assert isinstance(plain, torch.Tensor) and lib.frames == []
    assert all(r.token_timestamps is None and r.num_frames is None for r in m.last_windows)
    out = m.transcribe(x, return_token_timestamps=True, time_precision=0.04)
    wins = m.last_windows
    assert [r.num_frames for r in wins] == lib.frames == [WhisperMedusaModel.pcm_num_frames(r.end - r.start) for r in wins]
    assert lib.frames[-1] < 3000                                   # the short last window is cropped to its frames
    assert all(r.token_timestamps.tolist() == [[0.5, 1.0, 1.5]] for r in wins)     # time_precision reaches the extraction
    ids, pairs = merge_timed(wins, eos)
    assert out.keys() == ["sequences", "token_timestamps"]
    assert out.sequences.tolist() == [ids] and out.token_timestamps.shape == (1, len(ids), 2)
    assert torch.equal(out.token_timestamps, torch.tensor(pairs, dtype=torch.float32)[None])
    offs = window_offsets(wins)
    assert out.token_timestamps[0, 0].tolist() == [0.0, 0.5] and pairs[-1] == (round(1.0 + offs[-1], 2),
                                                                             round(1.5 + offs[-1], 2))
    assert torch.equal(m.transcribe(x), plain)                      # and off again
    # the no-speech rule: skipped windows keep their times and add nothing
    out_ns = m.transcribe(x, return_token_timestamps=True, no_speech_threshold=0.5, logprob_threshold=0.0)
    assert all(r.skipped and r.token_timestamps is not None for r in m.last_windows)
    assert out_ns.sequences.shape == (1, 0) and out_ns.token_timestamps.shape == (1, 0, 2)
    # StreamGroup through the shared queue: one output per recording, equal to the model's
    g = object.__new__(StreamGroup)
    g.n_streams, g.models, g.device = 1, [m], torch.device("cpu")
    got = g.transcribe([x, x[: 20 * SAMPLE_RATE]], return_token_timestamps=True, time_precision=0.04)
    assert torch.equal(got[0].sequences, out.sequences) and torch.equal(got[0].token_timestamps, out.token_timestamps)
    assert got[1].sequences.tolist() == [[0, 1, 2]] and len(g.last_windows[1]) == 1
    assert isinstance(g.transcribe(x)[0], torch.Tensor)


def test_argument_errors_before_any_upload(monkeypatch):
    from whisper_medusa_b200.streams import StreamGroup

    def no_upload(*a, **k):
        raise AssertionError("uploaded before the argument checks")

    x = np.zeros(40 * SAMPLE_RATE, np.float32)
    cases = [(dict(heads=None), ValueError, "no `alignment_heads`"),
             (dict(heads=[[0, 1], [2, 0]]), ValueError, "out of range"),           # micro: 2 layers of 2 heads
             (dict(heads=[[1, 1]], choices=[1, 2, 1, 1, 1]), NotImplementedError, "chain"),
             (dict(heads=[[1, 1]], width=6), ValueError, "odd")]
    for kw, err, msg in cases:
        m, lib = _stand_in(monkeypatch, heads=kw["heads"], choices=kw.get("choices"))
        if "width" in kw:
            m.config.median_filter_width = kw["width"]
        m._upload_16k = no_upload
        try:
            with pytest.raises(err, match=msg):
                m.transcribe(x, return_token_timestamps=True)
            with pytest.raises(err, match=msg):
                m.transcribe(x, return_token_timestamps=True, no_speech_threshold=0.6, logprob_threshold=-1.0)
            g = object.__new__(StreamGroup)
            g.n_streams, g.models, g.device = 1, [m], torch.device("cpu")
            with pytest.raises(err, match=msg):
                g.transcribe([x, x], return_token_timestamps=True)
            assert lib.frames == [] and lib.heads_sent == []
        finally:
            m._handle = None
    # segment timestamps still raise
    m, _ = _stand_in(monkeypatch)
    m._upload_16k = no_upload
    with pytest.raises(NotImplementedError):
        m.transcribe(x, return_timestamps=True, return_token_timestamps=True)
    m._handle = None
