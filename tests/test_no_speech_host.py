"""CPU tests of the no-speech rule (transcribe(no_speech_threshold=..., logprob_threshold=...)).

* The skip rule restated in ``longform.skip_window`` agrees with the installed transformers'
  ``WhisperGenerationMixin._need_fallback``, driven by a ``WhisperNoSpeechDetection`` and by scores whose
  ``_retrieve_avg_logprobs`` is the log-probability compared, over a grid that includes exact-equality edges.
* ``oracle.no_speech_ref`` scores the same token as HF and its probability equals ``WhisperNoSpeechDetection`` on the
  same raw row.
* A skipped window merges as an empty one, as HF's ``_find_longest_common_sequence`` does.
* Argument rules of ``transcribe`` / ``generate`` on a fake engine, the output object's fields, and the C ABI symbol.
"""
import ctypes as C
import itertools
import types

import numpy as np
import pytest
import torch

from oracle import no_speech_ref as NS
from oracle import whisper_ref as W
from whisper_medusa_b200 import WhisperMedusaModel
from whisper_medusa_b200.longform import Window, WindowResult, merge_windows, no_speech_rule, skip_window
from whisper_medusa_b200.model import MedusaGenerateOutput
from whisper_medusa_b200.synthetic import preset_config, synthetic_state_dict


def _hf_should_skip(no_speech_prob, avg_logprob_scores, tokens, nst, lpt):
    from transformers.generation.logits_process import WhisperNoSpeechDetection
    from transformers.models.whisper.generation_whisper import WhisperGenerationMixin

    det = WhisperNoSpeechDetection(no_speech_token=5, begin_index=1)
    det._no_speech_prob = [no_speech_prob]
    this = types.SimpleNamespace(_retrieve_avg_logprobs=WhisperGenerationMixin._retrieve_avg_logprobs)
    gc = types.SimpleNamespace(compression_ratio_threshold=None, logprob_threshold=lpt, no_speech_threshold=nst)
    _, skip = WhisperGenerationMixin._need_fallback(this, tokens, [{"scores": avg_logprob_scores}], 0, [det], gc, 8, 0.0)
    return skip


def _scores_for(avg):
    """fp64 scores of two tokens whose average log-probability is about ``avg`` (< 0), and that value as HF computes it."""
    from transformers.models.whisper.generation_whisper import WhisperGenerationMixin

    x = float(np.log(np.expm1(-avg)))       # log_softmax([0, x])[0] = -log(1 + e^x) = avg
    scores = [torch.tensor([0.0, x, -30.0, -30.0, -30.0, -30.0, -30.0, -30.0], dtype=torch.float64)] * 2
    tokens = torch.tensor([0, 0])
    return scores, tokens, float(WhisperGenerationMixin._retrieve_avg_logprobs(scores, tokens, 0.0))


def test_skip_rule_matches_need_fallback():
    pytest.importorskip("transformers")
    n = 0
    for avg_target in (-0.05, -0.7, -1.0, -2.5):
        scores, tokens, avg = _scores_for(avg_target)
        for p in (0.0, 0.3, 0.6, 0.6000001, 0.95, 1.0):
            # thresholds on both sides of each value and exactly at it
            for nst, lpt in itertools.product((0.0, 0.3, 0.6, p, 0.99), (-3.0, -1.0, avg, avg_target, -0.01, 0.0)):
                hf = _hf_should_skip(p, scores, tokens, nst, lpt)
                assert skip_window(p, avg, nst, lpt) == hf, (p, avg, nst, lpt)
                n += 1
    assert n > 500


def test_oracle_probability_matches_no_speech_detection():
    pytest.importorskip("transformers")
    from transformers.generation.logits_process import WhisperNoSpeechDetection

    cfg = preset_config("micro", heads=4)
    sd = synthetic_state_dict(cfg, seed=5)
    enc = torch.randn(cfg.max_source_positions, cfg.d_model, generator=torch.Generator().manual_seed(1), dtype=torch.float64)
    w = W.RefWeights(sd, torch.float64)
    row, prob = NS.no_speech_row(w, cfg, enc)
    assert row.shape == (cfg.vocab_size,) and row.dtype == torch.float64
    det = WhisperNoSpeechDetection(no_speech_token=NS.no_speech_token(cfg), begin_index=1)   # offset 1: reads `scores`
    det(torch.tensor([[int(cfg.decoder_start_token_id)]]), row[None])
    # (HF takes the softmax in fp32: .float().softmax)
    assert float(det.no_speech_prob[0]) == pytest.approx(prob, rel=1e-6)
    det(torch.tensor([[int(cfg.decoder_start_token_id)]]), row[None].float())
    assert float(det.no_speech_prob[0]) == pytest.approx(float(torch.softmax(row.float(), -1)[NS.no_speech_token(cfg)]),
                                                         rel=1e-7)
    # causality: the SOT row of a longer prompt is the same row
    cache = W.new_cache(cfg)
    prompt = [int(cfg.decoder_start_token_id), 7, 9, 11]
    hidden = W.decoder_forward(w, cfg, prompt, list(range(4)), enc, cache)
    full = W.medusa_logits(w, cfg, hidden, enc, cache, True)[0, 0]
    assert torch.allclose(full, row, rtol=0, atol=1e-12)


@pytest.mark.parametrize("preset,token", [("large-v2", 50362), ("tiny.en", 50361), ("micro", 501)])
def test_no_speech_token_is_hfs_choice(preset, token):
    m = WhisperMedusaModel(preset_config(preset, heads=4), None)
    assert NS.no_speech_token(m.config) == token
    assert int(m.generation_config.no_timestamps_token_id) - 1 == token


def test_skipped_window_merges_as_empty():
    pytest.importorskip("transformers")
    from transformers.models.whisper.tokenization_whisper import _find_longest_common_sequence

    rng = np.random.default_rng(3)
    for trial in range(40):
        n = int(rng.integers(3, 6))
        seqs = [rng.integers(0, 20, int(rng.integers(0, 30))).tolist() for _ in range(n)]
        for k in range(n):
            skipped = [s if i != k else [] for i, s in enumerate(seqs)]
            hf = [int(t) for t in _find_longest_common_sequence([list(s) for s in skipped])]
            assert merge_windows(skipped) == hf, (trial, k)
            # the same through WindowResult.merge_ids
            wins = [WindowResult(Window(0, 1, 0, 0), s + [1000], None, skipped=(i == k)) for i, s in enumerate(seqs)]
            assert merge_windows([r.merge_ids(1000) for r in wins]) == hf


def test_argument_rules():
    assert no_speech_rule(None, None) is False
    assert no_speech_rule(0.6, -1.0) is True
    with pytest.raises(ValueError):
        no_speech_rule(0.6, None)
    with pytest.raises(NotImplementedError):
        no_speech_rule(None, -1.0)
    for bad in (float("nan"), float("inf"), "0.6", True):
        with pytest.raises(ValueError):
            no_speech_rule(bad, -1.0)
        with pytest.raises(ValueError):
            no_speech_rule(0.6, bad)


def _fake_engine():
    m = WhisperMedusaModel(preset_config("micro", heads=4), None)
    m._handle = C.c_void_p(1)   # pretend an engine exists: nothing below reaches it
    calls = []
    m._encode_features = lambda feats: None
    m._decode = lambda language, task, kwargs, temperature, generation_config=None, return_dict_in_generate=None: \
        calls.append((dict(kwargs), return_dict_in_generate)) or "decoded"
    return m, calls


def test_transcribe_and_generate_arguments_on_a_fake_engine():
    m, calls = _fake_engine()
    x = np.zeros(16000, np.float32)
    feats = torch.zeros(1, 80, 3000)
    try:
        with pytest.raises(ValueError):
            m.transcribe(x, no_speech_threshold=0.6)
        with pytest.raises(NotImplementedError):
            m.transcribe(x, logprob_threshold=-1.0)
        with pytest.raises(ValueError):
            m.transcribe(x, no_speech_threshold=float("nan"), logprob_threshold=-1.0)
        # generate keeps refusing the threshold (the reference raises at model.py:1201)
        with pytest.raises(NotImplementedError):
            m.generate(feats, no_speech_threshold=0.6, logprob_threshold=-1.0)
        # output_no_speech_prob reaches _decode, with or without the dict (there it has no effect)
        assert m.generate(feats, return_dict_in_generate=True, output_no_speech_prob=True) == "decoded"
        assert m.generate(feats, output_no_speech_prob=True) == "decoded"
        assert calls == [({"output_no_speech_prob": True}, True), ({"output_no_speech_prob": True}, None)]
        # the SOT row of an explicit prompt must be in its last tile
        assert m._no_speech_row([m.config.decoder_start_token_id, 3, 4], m.generation_config) == 0
        long = [7] * 16 + [m.config.decoder_start_token_id, 3]
        assert m._no_speech_row(long, m.generation_config) == 16
        with pytest.raises(NotImplementedError):
            m._no_speech_row([m.config.decoder_start_token_id] + [7] * 17, m.generation_config)
        with pytest.raises(ValueError):
            m._no_speech_row([7, 8], m.generation_config)
    finally:
        m._handle = None


def test_generate_output_fields_unchanged_without_no_speech():
    seq = torch.tensor([[5, 6]])
    lp = torch.tensor([[-0.5, -0.25]])
    out = MedusaGenerateOutput(sequences=seq, scores=None, logits=None, token_logprobs=lp, avg_logprob=-0.375,
                               accept_lengths=[1])
    assert out.keys() == ["sequences", "token_logprobs", "avg_logprob", "accept_lengths"]
    assert out[1] is lp and out[-1] == [1] and out["no_speech_prob"] is None
    out.no_speech_prob = 0.25
    assert out.keys()[-1] == "no_speech_prob" and out[-1] == 0.25 and out[3] == [1]


def test_c_abi_exports_wm_last_no_speech(engine_lib):
    assert hasattr(engine_lib, "wm_last_no_speech")


class _RecordingLib:
    """The C ABI calls ``_decode`` makes around the loop, recorded (no engine behind them)."""

    def __init__(self):
        self.options = []

    def wm_set_option(self, handle, key, value):
        self.options.append((handle.value, key.decode(), int(value)))
        return 0

    def wm_last_no_speech(self, handle, token, prob, row):
        return 0


def test_no_speech_row_is_sent_to_every_engine(monkeypatch):
    """The option reaches the engine on every call, so a new engine (after to() / close()) is configured too."""
    from whisper_medusa_b200 import _lib
    from whisper_medusa_b200.model import GenerateTrace

    lib = _RecordingLib()
    monkeypatch.setattr(_lib, "load", lambda: lib)
    m = WhisperMedusaModel(preset_config("micro", heads=4), None)
    m._pushed = (tuple(m.generation_config.suppress_tokens or []), tuple(m.generation_config.begin_suppress_tokens or []))

    def run_loop(prompt, gp):
        tr = GenerateTrace()
        tr.sequences = list(prompt) + [5, int(gp.eos_token_id)]
        return tr

    m._run_loop = run_loop
    m._generate_output = lambda seq, tr, s, lg: MedusaGenerateOutput(seq, None, None, None, -0.5, [])
    try:
        for handle in (1, 1, 2):        # the same engine twice, then a replacement engine
            m._handle = C.c_void_p(handle)
            out = m._decode(None, None, {"output_no_speech_prob": True}, None, return_dict_in_generate=True)
            assert out.no_speech_prob == 0.0
        m._decode(None, None, {}, None)   # off again on the last engine
        ns = [(h, v) for h, k, v in lib.options if k == "no_speech_row"]
        assert ns == [(1, 0), (1, 0), (2, 0), (2, -1)]
    finally:
        m._handle = None
