"""CPU tests of token-level timestamps (generate(return_token_timestamps=True)).

* ``oracle.timestamps_ref`` -- the extraction restated with a DTW vectorised over anti-diagonals -- equals the installed
  transformers' ``WhisperGenerationMixin._extract_token_timestamps`` and ``_dynamic_time_warping`` exactly, over row
  counts 0 .. 448, prompts of 1 .. 5 ids, crops, NaN columns, duplicate heads and several time precisions.
* Argument errors, the ``alignment_heads`` round trip through ``save_pretrained``, the output object, the frame count
  ``generate_from_pcm`` uses, the C ABI declarations, the one-row ``attention_mask`` rule of ``generate`` and the
  per-row masks of ``StreamGroup.generate``.
"""
import ctypes as C
import os
import re
import types

import numpy as np
import pytest
import torch

from oracle import timestamps_ref as TS
from whisper_medusa_b200 import WhisperMedusaModel, _lib
from whisper_medusa_b200.config import MedusaGenerationConfig
from whisper_medusa_b200.model import GenerateTrace, MedusaGenerateOutput
from whisper_medusa_b200.synthetic import preset_config

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class _Out(dict):
    """What HF's extractor reads from generate outputs (``.cross_attentions``, ``.sequences``, ``"beam_indices" in``)."""
    __getattr__ = dict.__getitem__


def _hf_timestamps(rows_by_layer, n_prompt, pairs, n_layers, num_frames, tp, width=7):
    """HF's ``_extract_token_timestamps`` on rows ``[layers][heads, n - 1, S]`` split the way generate returns them: the
    prompt's rows in one step, then one row per step."""
    from transformers.models.whisper.generation_whisper import WhisperGenerationMixin

    n1 = rows_by_layer[0].shape[1]
    steps = [tuple(r[None, :, :n_prompt] for r in rows_by_layer)]
    steps += [tuple(r[None, :, t : t + 1] for r in rows_by_layer) for t in range(n_prompt, n1)]
    outs = _Out(cross_attentions=tuple(steps), sequences=torch.zeros(1, n1 + 1, dtype=torch.long))
    this = types.SimpleNamespace(config=types.SimpleNamespace(decoder_layers=n_layers, median_filter_width=width))
    return WhisperGenerationMixin._extract_token_timestamps(this, outs, pairs, time_precision=tp, num_frames=num_frames,
                                                            num_input_ids=n_prompt)[0].numpy()


def _rows(n_layers, H, n1, S, seed, sharp=4.0):
    g = torch.Generator().manual_seed(seed)
    return [torch.softmax(sharp * torch.randn(H, n1, S, generator=g), dim=-1) for _ in range(n_layers)]


def _ours(rows_by_layer, n_prompt, pairs, num_frames, tp, width=7):
    probs = torch.stack([rows_by_layer[l][h, n_prompt:] for l, h in pairs])
    ts, _, _ = TS.extract(probs, n_prompt, num_frames, width, tp)
    return ts


@pytest.mark.parametrize("n_gen,n_prompt,num_frames,tp", [
    (1, 1, None, 0.02), (2, 3, None, 0.02), (3, 4, 3000, 0.02), (7, 2, 801, 0.01), (12, 5, 40, 0.02),
    (30, 1, 5, 0.02), (30, 3, 1, 0.02), (60, 4, 3000, 0.04), (120, 2, 1999, 0.02),
])
def test_extract_matches_hf(n_gen, n_prompt, num_frames, tp):
    pytest.importorskip("transformers")
    L, H, S = 4, 6, 1500
    pairs = [[1, 0], [2, 3], [3, 5], [2, 3]]           # a duplicate counts twice
    rows = _rows(L, H, n_prompt + n_gen - 1, S, seed=n_gen * 7 + n_prompt)
    for nf in (num_frames, None if num_frames is None else torch.tensor([num_frames])):
        hf = _hf_timestamps(rows, n_prompt, pairs, L, nf, tp)
        ours = _ours(rows, n_prompt, pairs, None if nf is None else int(nf if isinstance(nf, int) else nf[0]), tp)
        assert ours.shape == hf.shape == (n_prompt + n_gen,)
        np.testing.assert_array_equal(ours, hf)


def test_extract_448_rows_matches_hf():
    pytest.importorskip("transformers")
    L, H, S, P = 2, 2, 1500, 2
    rows = _rows(L, H, P + 448 - 1 + 1, S, seed=3)     # N = 448 rows after the prompt
    pairs = [[0, 1], [1, 0]]
    hf = _hf_timestamps(rows, P, pairs, L, 400, 0.02)   # (F = 200 keeps HF's Python DTW short)
    np.testing.assert_array_equal(_ours(rows, P, pairs, 400, 0.02), hf)
    assert hf.shape == (P + 449,)


def test_nan_columns_and_single_row_match_hf():
    """std = 0 gives NaN (one row, or a column of equal values); NaN propagates through the filter and the DTW."""
    pytest.importorskip("transformers")
    L, H, S, P = 1, 2, 64, 2
    rows = _rows(L, H, P + 2, S, seed=11)
    for n_gen in (2, 3):                   # N = 1 row (all NaN), N = 2 rows with equal columns
        r = [x[:, : P + n_gen - 1].clone() for x in rows]
        r[0][:, P:, 10:20] = 0.25          # exactly representable: the mean is the value, the std 0
        hf = _hf_timestamps(r, P, [[0, 0], [0, 1]], L, None, 0.02)
        np.testing.assert_array_equal(_ours(r, P, [[0, 0], [0, 1]], None, 0.02), hf)


def test_dtw_matches_hf_with_ties_and_nan():
    pytest.importorskip("transformers")
    from transformers.models.whisper.generation_whisper import _dynamic_time_warping

    rng = np.random.default_rng(5)
    for shape in [(1, 1), (1, 9), (9, 1), (5, 7), (17, 40), (40, 17)]:
        for kind in ("float", "ties", "nan"):
            m = rng.standard_normal(shape)
            if kind == "ties":
                m = rng.integers(-2, 2, shape).astype(np.float64)
            if kind == "nan":
                m[rng.random(shape) < 0.2] = np.nan
            m = m.astype(np.float32).astype(np.float64)
            a, b = _dynamic_time_warping(m)
            c, d = TS.dtw(m)
            np.testing.assert_array_equal(a, c)
            np.testing.assert_array_equal(b, d)


def test_median_filter_matches_hf():
    pytest.importorskip("transformers")
    from transformers.models.whisper.generation_whisper import _median_filter

    x = torch.randn(2, 3, 5, 20)
    x[0, 0, 0, 3] = float("nan")
    for w in (1, 3, 7, 9, 41):
        assert torch.equal(torch.nan_to_num(TS.median_filter(x, w), 9.0), torch.nan_to_num(_median_filter(x, w), 9.0))
    with pytest.raises(ValueError, match="odd"):
        TS.median_filter(x, 4)


def test_pcm_frame_count_matches_feature_extractor():
    pytest.importorskip("transformers")
    from transformers import WhisperFeatureExtractor

    fe = WhisperFeatureExtractor()
    for n in (1, 159, 160, 161, 480000):
        mask = fe(np.zeros(n, dtype=np.float32), sampling_rate=16000, return_attention_mask=True)["attention_mask"]
        assert WhisperMedusaModel.pcm_num_frames(n) == int(np.asarray(mask).sum(-1)[0]), n


def test_alignment_heads_round_trip(tmp_path):
    g = MedusaGenerationConfig(alignment_heads=[[2, 1], [3, 0]])
    g.save_pretrained(str(tmp_path))
    assert MedusaGenerationConfig.from_pretrained(str(tmp_path)).alignment_heads == [[2, 1], [3, 0]]
    MedusaGenerationConfig().save_pretrained(str(tmp_path / "none"))
    assert MedusaGenerationConfig.from_pretrained(str(tmp_path / "none")).alignment_heads is None
    assert preset_config("micro", heads=4).median_filter_width == 7


class _RecordingLib:
    """The C ABI calls ``_decode`` makes around the loop, recorded (no engine behind them)."""

    def __init__(self):
        self.pairs = []

    def wm_set_option(self, handle, key, value):
        return 0

    def wm_set_alignment_heads(self, handle, arr, n):
        self.pairs.append((handle.value, [int(arr[i]) for i in range(2 * n)]))
        return 0

    def wm_token_timestamps(self, handle, n_prompt, n_total, num_frames, width, tp, out, matrix, jumps):
        for i in range(n_total):
            out[i] = 0.5 * i
        return 0


def _fake_model(monkeypatch, heads=None, choices=None):
    lib = _RecordingLib()
    monkeypatch.setattr(_lib, "load", lambda: lib)
    cfg = preset_config("micro", heads=4)
    if choices is not None:
        cfg.medusa_choices = choices
    m = WhisperMedusaModel(cfg, None)
    m.generation_config.alignment_heads = heads
    m._pushed = (tuple(m.generation_config.suppress_tokens or []), tuple(m.generation_config.begin_suppress_tokens or []))

    def run_loop(prompt, gp):
        tr = GenerateTrace()
        tr.sequences = list(prompt) + [5, 6, int(gp.eos_token_id)]
        tr.n_new_tokens = 3
        return tr

    m._run_loop = run_loop
    m._generate_output = lambda seq, tr, s, lg: MedusaGenerateOutput(seq, None, None, torch.zeros(1, 3), -0.5, [1])
    return m, lib


def test_argument_errors(monkeypatch):
    m, _ = _fake_model(monkeypatch, heads=None)
    m._handle = C.c_void_p(1)
    try:
        with pytest.raises(ValueError, match="no `alignment_heads`"):
            m.generate_from_pcm(np.zeros(1600, np.float32), return_token_timestamps=True)
        m.generation_config.alignment_heads = [[0, 1], [2, 0]]          # micro: 2 layers of 2 heads
        with pytest.raises(ValueError, match="out of range"):
            m.generate_from_pcm(np.zeros(1600, np.float32), return_token_timestamps=True)
        m.generation_config.alignment_heads = [[1, 1]]
        m.config.median_filter_width = 6
        with pytest.raises(ValueError, match="odd"):
            m.generate_from_pcm(np.zeros(1600, np.float32), return_token_timestamps=True)
    finally:
        m._handle = None
    t, _ = _fake_model(monkeypatch, heads=[[1, 1]], choices=[1, 2, 1, 1, 1])
    t._handle = C.c_void_p(1)
    try:
        with pytest.raises(NotImplementedError, match="chain"):
            t.generate_from_pcm(np.zeros(1600, np.float32), return_token_timestamps=True)
    finally:
        t._handle = None


def test_output_object_and_pairs_sent(monkeypatch):
    m, lib = _fake_model(monkeypatch, heads=[[1, 1], [0, 0], [1, 1]])
    try:
        for handle in (1, 2):
            m._handle = C.c_void_p(handle)
            out = m._decode(None, None, {}, None, token_timestamps=(None, 0.02))
            assert out.keys() == ["sequences", "token_timestamps"]
            assert out[1] is out.token_timestamps and out["sequences"] is out[0]
            # ids = [5, 6] after the EOS strip; prompt [SOT, <|notimestamps|>]: positions 2, 3 of 0.5 * position
            assert out.sequences.tolist() == [[5, 6]]
            assert out.token_timestamps.tolist() == [[1.0, 1.5]]
            full = m._decode(None, None, {}, None, return_dict_in_generate=True, token_timestamps=(None, 0.02))
            assert full.keys() == ["sequences", "token_logprobs", "avg_logprob", "accept_lengths", "token_timestamps"]
            assert full[:4] == (full.sequences, full.token_logprobs, full.avg_logprob, full.accept_lengths)
        plain = m._decode(None, None, {}, None)            # capture switched off on the engine that had it
        assert isinstance(plain, torch.Tensor)
        m._decode(None, None, {}, None)                    # ... once
        assert lib.pairs == [(1, [1, 1, 0, 0, 1, 1])] * 2 + [(2, [1, 1, 0, 0, 1, 1])] * 2 + [(2, [])]
    finally:
        m._handle = None
    assert MedusaGenerateOutput.FIELDS[-1] == "token_timestamps"


def test_c_abi_declares_and_exports_timestamp_entries(engine_lib):
    names = ["wm_set_alignment_heads", "wm_token_timestamps", "wm_token_timestamps_from_probs", "wm_last_alignment_probs"]
    with open(os.path.join(ROOT, "include", "whisper_medusa_b200.h")) as f:
        header = f.read()
    for n in names:
        assert re.search(rf"\bint {n}\(", header), n
        assert n in _lib.SYMBOLS
        assert hasattr(engine_lib, n)


def test_attention_mask_must_be_one_row(monkeypatch):
    """generate takes one clip: a mask of several rows (a batch's) raises instead of cropping by another row."""
    m, _ = _fake_model(monkeypatch, heads=[[1, 1]])
    m._handle = C.c_void_p(1)
    feats = torch.zeros(1, 80, 3000)
    try:
        for bad in (torch.ones(2, 3000), torch.ones(1, 1500), torch.ones(1, 1, 3000)):
            with pytest.raises(ValueError, match="attention_mask"):
                m.generate(feats, attention_mask=bad, return_token_timestamps=True)
        assert m._mask_frames(torch.ones(1, 3000)) == 3000
        assert m._mask_frames(torch.cat([torch.ones(1200), torch.zeros(1800)])) == 1200
    finally:
        m._handle = None


class _MaskRecorder:
    """A stand-in engine of a StreamGroup: records the mask each row's generate receives."""

    def __init__(self, seen):
        self.seen = seen
        self.last_trace = GenerateTrace()

    def generate(self, x, attention_mask=None, **kw):
        self.seen[int(x[0, 0, 0])] = None if attention_mask is None else attention_mask.clone()
        return torch.zeros(1, 1, dtype=torch.long)


def test_stream_group_hands_each_row_its_mask():
    from whisper_medusa_b200.streams import StreamGroup

    seen = {}
    g = object.__new__(StreamGroup)
    g.n_streams, g.models = 2, [_MaskRecorder(seen), _MaskRecorder(seen)]
    feats = torch.zeros(3, 80, 3000)
    for i in range(3):
        feats[i, 0, 0] = i
    mask = torch.zeros(3, 3000, dtype=torch.long)
    for i, n in enumerate((3000, 1200, 40)):
        mask[i, :n] = 1
    g.generate(feats, attention_mask=mask, return_token_timestamps=True)
    assert {i: int(v.sum()) for i, v in seen.items()} == {0: 3000, 1: 1200, 2: 40}
    assert all(v.shape == (1, 3000) for v in seen.values())
    g.generate(feats, return_token_timestamps=True)
    assert all(v is None for v in seen.values())
    with pytest.raises(ValueError, match="one row per clip"):
        g.generate(feats, attention_mask=mask[:2])
