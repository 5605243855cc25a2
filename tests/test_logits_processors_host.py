"""Logits processors without a GPU: ``sequence_bias``, ``bad_words_ids``, ``no_repeat_ngram_size``, ``min_length`` and
``min_new_tokens``.

* The oracle's ``processors_ref.process_logits`` is bit-equal to a ``LogitsProcessorList`` of the installed HF
  processors, and with no processor set it is ``medusa_ref.process_logits``.
* Where the reference checkout is present, the oracle loop equals the reference's own loop (``processors_ref.run_loop``)
  with each processor alone and all of them, in chains and trees, at temperature 0 and 1; every scenario's tokens differ
  from the same stream without processors.
* The host: HF's exception types, the refusals, the tables sent to the engine, and a call without processors.
"""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

from _wm_paths import ROOT
from oracle import make_processors_golden as PG
from oracle import medusa_ref as M
from oracle import processors_ref as PR
from oracle import ref_harness as R
from whisper_medusa_b200 import WhisperMedusaModel, _lib
from whisper_medusa_b200 import processors as P
from whisper_medusa_b200.model import GenerateTrace
from whisper_medusa_b200.synthetic import preset_config

V, EOS = 97, 50


def _hf_list(gp, prompt_len):
    from transformers.generation.logits_process import (LogitsProcessorList, MinLengthLogitsProcessor,
                                                        MinNewTokensLengthLogitsProcessor, NoBadWordsLogitsProcessor,
                                                        NoRepeatNGramLogitsProcessor, SequenceBiasLogitsProcessor)
    procs = LogitsProcessorList()
    if gp.sequence_bias:
        procs.append(SequenceBiasLogitsProcessor([[list(ids), v] for ids, v in gp.sequence_bias]))
    if gp.no_repeat_ngram_size:
        procs.append(NoRepeatNGramLogitsProcessor(gp.no_repeat_ngram_size))
    if gp.bad_words_ids:
        procs.append(NoBadWordsLogitsProcessor(gp.bad_words_ids, EOS))
    if gp.min_length:
        procs.append(MinLengthLogitsProcessor(gp.min_length, EOS))
    if gp.min_new_tokens:
        procs.append(MinNewTokensLengthLogitsProcessor(prompt_len, gp.min_new_tokens, EOS))
    return procs


def _check_equal(gp, ids, prompt_len, seed=0):
    g = torch.Generator().manual_seed(seed)
    rows = torch.randn(5, V, generator=g) * 4
    ref = _hf_list(gp, prompt_len)(torch.tensor([ids]).expand(5, -1), rows.clone())
    got = PR.process_logits(rows, len(ids), gp, ids)
    assert torch.equal(got, ref)
    return got, rows


def _gp(prompt_len, **kw):
    gp = M.GenParams(eos_token_id=EOS, pad_token_id=EOS, prompt_len=prompt_len, begin_index=prompt_len)
    kw = dict(dict(sequence_bias=None, no_repeat_ngram_size=0, bad_words_ids=None, min_length=0, min_new_tokens=0), **kw)
    for k, v in kw.items():
        setattr(gp, k, v)
    return gp


def test_sequence_bias_sums_in_dict_order_on_one_last_token():
    rng = np.random.default_rng(1)
    ids = [3, 9, 4, 7, 11, 7]
    vals = [float(v) for v in rng.normal(0, 3, 6)]
    sb = [((7,), vals[0]), ((11, 7, 20), vals[1]), ((7, 20), vals[2]), ((4, 7, 11, 7, 20), vals[3]),
          ((5, 20), vals[4]), ((20,), vals[5])]
    got, rows = _check_equal(_gp(2, sequence_bias=sb), ids, 2)
    # (the sum runs from the single-token bias through the matched entries in order, in fp32)
    want = torch.tensor(0.0) + torch.tensor(vals[5])
    for v in (vals[1], vals[2], vals[3]):
        want = want + torch.tensor(v)
    assert torch.equal(got[:, 20], rows[:, 20] + want)


def test_sequences_longer_than_the_context_are_skipped():
    sb = [((1, 2, 3, 4, 5), 2.5), ((2, 3), -1.25)]
    _check_equal(_gp(2, sequence_bias=sb), [1, 2], 2)
    _check_equal(_gp(2, bad_words_ids=[[1, 2, 3, 9], [2, 8]]), [1, 2], 2, seed=3)


@pytest.mark.parametrize("n", [1, 2, 3])
@pytest.mark.parametrize("cur_len", [1, 2, 3, 12])
def test_no_repeat_ngram(n, cur_len):
    ids = [5, 6, 5, 6, 7, 5, 6, 8, 5, 6, 5, 6][:cur_len]
    got, _ = _check_equal(_gp(1, no_repeat_ngram_size=n), ids, 1, seed=n * 10 + cur_len)
    if cur_len + 1 < n:
        assert torch.isfinite(got).all()


def test_bad_words_filter_the_lone_eos():
    ids = [3, 4, 5]
    got, _ = _check_equal(_gp(1, bad_words_ids=[[EOS], [8], [5, 9], [4, 5, 10], [EOS, 12]]), ids, 1)
    assert torch.isfinite(got[:, EOS]).all() and torch.isinf(got[:, 8]).all() and torch.isinf(got[:, 9]).all()
    assert torch.isinf(got[:, 10]).all() and torch.isfinite(got[:, 12]).all()


@pytest.mark.parametrize("cur_len", [20, 24, 25, 26, 30])
def test_min_length_and_min_new_tokens_with_a_long_prompt(cur_len):
    ids = list(range(1, cur_len + 1))
    _check_equal(_gp(20, min_length=26), ids, 20)
    got, _ = _check_equal(_gp(20, min_new_tokens=5), ids, 20)
    assert bool(torch.isinf(got[:, EOS]).all()) == (cur_len - 20 < 5)


def test_all_processors_together():
    ids = [1, 2, 3, 1, 2, 4, 1, 2]
    gp = _gp(3, sequence_bias=[((2, 6), 1.5), ((6,), -0.75), ((1, 2, 6), 0.125)], no_repeat_ngram_size=2,
             bad_words_ids=[[2, 4], [13]], min_length=12, min_new_tokens=2)
    _check_equal(gp, ids, 3)


def test_without_processors_it_is_the_existing_oracle():
    rows = torch.randn(3, V) * 4
    gp = _gp(2, suppress_tokens=[3, 9], begin_suppress_tokens=[4], exponential_decay_length_penalty=(1, 1.2))
    for L in (2, 4):
        assert torch.equal(PR.process_logits(rows, L, gp, list(range(L))), M.process_logits(rows, L, gp))
    # the loop and the scores record compiled with the processors are the existing ones when none is set
    from oracle import make_ref_golden as G
    from oracle import scores_ref as S
    from oracle import whisper_ref as W

    cfg, sd, pcm, max_len, pen, temp, alpha, thr = G.stream_inputs("micro_lin_pen", 0)
    w = W.RefWeights(sd)
    enc = W.encoder_forward(w, cfg, torch.from_numpy(W.log_mel_spectrogram(pcm)), "fp32")
    prompt = M.init_tokens(cfg, None)
    gp = M.gen_params(cfg, prompt, pen, max_len, temperature=temp, posterior_alpha=alpha, posterior_threshold=thr)
    a = M.medusa_greedy_search(w, cfg, enc, prompt, gp, "fp32", capture_logits=1 << 20)
    b = PR.medusa_greedy_search(w, cfg, enc, prompt, gp, "fp32", capture_logits=1 << 20)
    assert (a.sequences, a.accept_lengths) == (b.sequences, b.accept_lengths)
    sa = S.loop_scores(a, len(prompt), gp, cfg.medusa_choices)
    sb = PR.loop_scores(b, len(prompt), gp, cfg.medusa_choices)
    assert sa.token_logprobs == sb.token_logprobs and all(torch.equal(x, y) for x, y in zip(sa.rows, sb.rows))


# ---------------------------------------------------------------------------- the loop against the reference's loop
@pytest.mark.skipif(not R.available(), reason="the reference checkout is not present")
@pytest.mark.parametrize("name", sorted(PG.SCENARIOS))
def test_oracle_loop_matches_the_reference_loop(name):
    torch.set_num_threads(min(8, os.cpu_count() or 1))
    ref_seq, ref_acc, seq, acc, plain = PG.run_scenario(name, with_reference=True)
    assert seq == ref_seq and acc == ref_acc
    assert seq != plain, "the processors do not change this stream"


def test_fixture_matches_the_oracle():
    """The frozen fixtures are what the oracle loop computes now (micro scenarios; the larger ones run on the GPU)."""
    fx = np.load(PG.FIXTURE)
    for name in sorted(PG.SCENARIOS):
        if not name.startswith("micro"):
            continue
        _, _, seq, acc, plain = PG.run_scenario(name)
        assert seq == fx[f"{name}/sequences"].tolist() and acc == fx[f"{name}/accept"].tolist()
        assert plain == fx[f"{name}/plain"].tolist() and seq != plain


# ---------------------------------------------------------------------------- host
class _Lib:
    def __init__(self):
        self.calls = []

    def wm_set_option(self, handle, key, value):
        return 0

    def wm_set_suppress(self, *a):
        return 0

    def wm_set_logits_processors(self, handle, toks, offs, vals, n, ngram, eos_min):
        o = [offs[i] for i in range(n + 1)]
        self.calls.append((handle.value, [tuple(toks[o[i]:o[i + 1]]) for i in range(n)], [vals[i] for i in range(n)],
                           ngram, eos_min))
        return 0


def _fake(monkeypatch):
    lib = _Lib()
    monkeypatch.setattr(_lib, "load", lambda: lib)
    m = WhisperMedusaModel(preset_config("micro", heads=4), None)
    m._pushed = (tuple(m.generation_config.suppress_tokens or []), tuple(m.generation_config.begin_suppress_tokens or []))
    runs = []

    def run_loop(prompt, gp):
        runs.append(list(prompt))
        tr = GenerateTrace()
        tr.sequences = list(prompt) + [5, 6, int(gp.eos_token_id)]
        tr.n_new_tokens = 3
        return tr

    m._run_loop = run_loop
    return m, lib, runs


def _errors(kw, m):
    g = m.generation_config
    return P.build(P.options(kw, g), int(g.eos_token_id), m.config.vocab_size, 2, 448, None)


@pytest.mark.parametrize("kw", [
    {"sequence_bias": []}, {"sequence_bias": {(1, 2): 1}}, {"sequence_bias": {(): 1.0}}, {"sequence_bias": {(-1,): 1.0}},
    {"sequence_bias": {"a": 1.0}}, {"sequence_bias": [[[0], 1.0]]}, {"sequence_bias": [[[1, 2], 1]]},
    {"sequence_bias": [[(1, 2), 1.0]]}, {"bad_words_ids": []}, {"bad_words_ids": [3]}, {"bad_words_ids": [[3, -1]]},
    {"no_repeat_ngram_size": 2.0}, {"min_length": 3.0}, {"min_new_tokens": 1.5},
])
def test_argument_errors_have_hf_types(kw, monkeypatch):
    """The same exception type as the installed HF processor's constructor on the same argument."""
    from transformers.generation.logits_process import (MinLengthLogitsProcessor, MinNewTokensLengthLogitsProcessor,
                                                        NoBadWordsLogitsProcessor, NoRepeatNGramLogitsProcessor,
                                                        SequenceBiasLogitsProcessor)
    m, _, _ = _fake(monkeypatch)
    (k, v), = kw.items()
    make = {"sequence_bias": lambda: SequenceBiasLogitsProcessor(v), "bad_words_ids": lambda: NoBadWordsLogitsProcessor(v, 3),
            "no_repeat_ngram_size": lambda: NoRepeatNGramLogitsProcessor(v),
            "min_length": lambda: MinLengthLogitsProcessor(v, 3),
            "min_new_tokens": lambda: MinNewTokensLengthLogitsProcessor(2, v, 3)}[k]
    with pytest.raises(Exception) as hf:
        make()
    with pytest.raises(type(hf.value)):
        _errors(kw, m)


def test_vocab_values_capacity_and_nan_refusals(monkeypatch):
    m, lib, runs = _fake(monkeypatch)
    m._handle = C.c_void_p(1)
    feats = torch.zeros(1, 80, 3000)
    Vm = m.config.vocab_size
    try:
        with pytest.raises(ValueError, match="vocabulary size"):
            m.generate(feats, sequence_bias=[[[Vm], 1.0]])
        with pytest.raises(ValueError, match="vocabulary size"):
            m.generate(feats, bad_words_ids=[[1, Vm + 3]])
        for bad in (float("inf"), float("nan")):
            with pytest.raises(ValueError, match="finite"):
                m.generate(feats, sequence_bias=[[[4], bad]])
        with pytest.raises(NotImplementedError, match="at most 256"):
            m.generate(feats, bad_words_ids=[[1, 2 + i] for i in range(257)])
        with pytest.raises(NotImplementedError, match="4096"):
            m.generate(feats, bad_words_ids=[[1] * 100 + [i] for i in range(2, 44)])
        # an EOS ban inside the decay region: min_length 10 on a 2-token prompt, penalty from length 2 + 3
        with pytest.raises(NotImplementedError, match="overlaps"):
            m.generate(feats, min_length=10, exponential_decay_length_penalty=(3, 1.2))
        with pytest.raises(NotImplementedError, match="overlaps"):
            m.generate(feats, min_new_tokens=5, exponential_decay_length_penalty=(2, 0.9))
        eos = int(m.generation_config.eos_token_id)
        with pytest.raises(NotImplementedError, match="ending in EOS"):
            m.generate(feats, bad_words_ids=[[7, eos]], exponential_decay_length_penalty=(30, 1.2))
        with pytest.raises(NotImplementedError, match="not implemented"):
            m.generate(feats, repetition_penalty=1.3)
        with pytest.raises(NotImplementedError, match="not implemented"):
            m.transcribe(np.zeros(1600, np.float32), repetition_penalty=1.3)
        assert not runs and not lib.calls           # every check ran before any engine call
        # no overlap: the ban ends (length 5) before the region starts (lengths above 2 + 3)
        m._encode_features = lambda f: None
        m.generate(feats, min_length=5, exponential_decay_length_penalty=(3, 1.2))
        assert lib.calls[-1] == (1, [], [], 0, 5)
    finally:
        m._handle = None


def test_tables_sent_and_switched_off(monkeypatch):
    m, lib, runs = _fake(monkeypatch)
    m._encode_features = lambda f: None
    feats = torch.zeros(1, 80, 3000)
    eos = int(m.generation_config.eos_token_id)
    try:
        m._handle = C.c_void_p(1)
        m.generate(feats)                                          # no processors, never had any: nothing sent
        assert lib.calls == []
        m.generate(feats, sequence_bias={(3, 4): 1.5, (9,): -2.0}, bad_words_ids=[[eos], [5, 6], [3, 4]],
                   no_repeat_ngram_size=3, min_new_tokens=4, decoder_input_ids=torch.tensor([[1, 2, 3, 4, 5]]))
        ninf = float("-inf")
        assert lib.calls == [(1, [(3, 4), (9,), (5, 6), (3, 4)], [1.5, -2.0, ninf, ninf], 3, 9)]
        m.generation_config.min_length = 7                         # the generation config is a source too
        m.generate(feats)
        assert lib.calls[-1] == (1, [], [], 0, 7)
        del m.generation_config.min_length
        m.generate(feats)                                          # switched off on the engine that had them ...
        m.generate(feats)                                          # ... once
        assert lib.calls[-1] == (1, [], [], 0, 0) and len(lib.calls) == 3
        m._handle = C.c_void_p(2)
        m.generate(feats, min_length=0, no_repeat_ngram_size=0)    # HF: 0 = off
        assert len(lib.calls) == 3
    finally:
        m._handle = None


def test_no_preset_or_fixture_sets_a_processor():
    """Every existing call is unchanged: no built-in preset's generation config sets any of the options."""
    from whisper_medusa_b200.config import MedusaGenerationConfig

    for name in ("large-v2", "tiny.en", "micro", "base", "small", "medium"):
        g = MedusaGenerationConfig.from_model_config(preset_config(name))
        assert P.build(P.options({}, g), int(g.eos_token_id), 10 ** 6, 4, 448, None) is None, name


def test_c_abi_declares_the_entry(engine_lib):
    with open(os.path.join(ROOT, "include", "whisper_medusa_b200.h")) as f:
        header = f.read()
    assert re.search(r"\bint wm_set_logits_processors\(", header)
    assert "wm_set_logits_processors" in _lib.SYMBOLS and hasattr(engine_lib, "wm_set_logits_processors")
