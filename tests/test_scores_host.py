"""Scores and per-token log-probabilities without a GPU: the oracle's record of them (oracle/scores_ref.py) is pinned
to the reference's own loop run with ``return_dict_in_generate=True, output_scores=True, output_logits=True``, and the
host accepts ``output_scores`` / ``output_logits`` while every pinned refusal still raises."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from _wm_paths import GOLDEN
from oracle import make_ref_golden as G
from oracle import make_scores_golden as SG
from oracle import medusa_ref as M
from oracle import ref_harness as R
from oracle import scores_ref as S
from oracle import whisper_ref as W
from whisper_medusa_b200 import MedusaGenerateOutput, WhisperMedusaModel
from whisper_medusa_b200.synthetic import preset_config

FIX = os.path.join(GOLDEN, "ref_loop_scores_micro.npz")


def _oracle(group, s, enc=None):
    """fp32 oracle run of a make_ref_golden stream with every iteration's logits captured, and its scores record."""
    cfg, sd, pcm, max_len, pen, temp, alpha, thr = G.stream_inputs(group, s)
    w = W.RefWeights(sd)
    if enc is None:
        enc = W.encoder_forward(w, cfg, torch.from_numpy(W.log_mel_spectrogram(pcm)), "fp32")
    prompt = M.init_tokens(cfg, "en" if cfg.is_multilingual else None)
    gp = M.gen_params(cfg, prompt, pen, max_len, temperature=temp, posterior_alpha=alpha, posterior_threshold=thr)
    tr = M.medusa_greedy_search(w, cfg, enc, prompt, gp, "fp32", capture_logits=1 << 20)
    return cfg, prompt, tr, S.loop_scores(tr, len(prompt), gp, cfg.medusa_choices)


def _rows_close(got, ref, bar):
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    assert got.shape == ref.shape
    assert np.array_equal(np.isneginf(got), np.isneginf(ref)), "suppressed ids differ"
    fin = np.isfinite(ref)
    assert np.isfinite(got[fin]).all()
    err = np.abs(got[fin] - ref[fin]).max() / max(1.0, np.abs(ref[fin]).max())
    assert err <= bar, err
    return err


@pytest.mark.parametrize("group,s", SG.STREAMS)
def test_oracle_scores_match_the_frozen_reference_rows(group, s):
    """One processed row per iteration, equal (to fp32 summation order) to the reference's ``scores``; -inf exactly at
    the suppressed ids."""
    fx = np.load(FIX)
    torch.set_num_threads(min(8, os.cpu_count() or 1))
    cfg, prompt, tr, sc = _oracle(group, s)
    assert tr.sequences == fx[f"{group}/{s}/sequences"].tolist()
    assert tr.accept_lengths == fx[f"{group}/{s}/accept"].tolist()
    ref_rows = fx[f"{group}/{s}/scores"]
    assert len(sc.rows) == len(tr.accept_lengths) == ref_rows.shape[0]
    _rows_close(torch.stack(sc.rows).numpy(), ref_rows, 1e-5)
    # one log-probability per generated position, each <= 0
    assert len(sc.token_logprobs) == len(tr.sequences) - len(prompt)
    assert max(sc.token_logprobs) <= 0.0


@pytest.mark.skipif(not R.available(), reason="the reference checkout is not present")
@pytest.mark.parametrize("group", ["micro_lin_t1", "micro_blk_pen", "micro_tree122_t1", "tiny_lin_t1"])
def test_oracle_scores_match_the_reference_loop(group):
    """The reference's loop run live (oracle/ref_harness.py) with output_scores / output_logits: ``len(scores)`` is the
    number of iterations, both tuples hold the same tensors, and the oracle record reproduces them, on the micro and tiny
    presets (chain, Block heads with the length penalty, a branching tree)."""
    torch.set_num_threads(min(8, os.cpu_count() or 1))
    prompt, seq, out, enc = SG.run_stream(group, 0)
    cfg, _, tr, sc = _oracle(group, 0, enc=enc)
    assert tr.sequences == seq
    assert len(out.scores) == len(tr.accept_lengths) and out.logits is not None
    assert all(a is b for a, b in zip(out.scores, out.logits))
    assert all(tuple(r.shape) == (1, 1, cfg.vocab_size) for r in out.scores)
    _rows_close(torch.stack(sc.rows).numpy(), torch.cat([r.reshape(1, -1) for r in out.scores]).numpy(), 1e-5)


def test_exact_match_tokens_are_row_maxima():
    """With exact-match acceptance every emitted token is the argmax of the row it was chosen from, so its
    log-probability is that row's largest log_softmax entry."""
    cfg, prompt, tr, sc = _oracle("micro_lin_t0", 0)
    gp = M.gen_params(cfg, prompt, None, G.GROUPS["micro_lin_t0"][5], temperature=0.0)
    L, k = len(prompt), 0
    for i, a in enumerate(tr.accept_lengths):
        rows_a = M.process_logits(tr.passA_logits[i], L, gp).double()
        rows_b = M.process_logits(tr.passB_logits[i], L, gp).double()
        n_new = a + 1 if a else 2
        for j in range(n_new):
            row = rows_a[0] if j == 0 else rows_b[sc.paths[i][j - 1]]
            assert sc.token_logprobs[k] == pytest.approx(float(torch.log_softmax(row, -1).max()), abs=1e-12)
            k += 1
        L += n_new


def _fake_engine():
    m = WhisperMedusaModel(preset_config("micro", heads=4), None)
    m._handle = C.c_void_p(1)   # pretend an engine exists: nothing below reaches it
    calls = []
    m._encode_features = lambda feats: None
    m._decode = lambda language, task, kwargs, temperature, generation_config=None, return_dict_in_generate=None: \
        calls.append((dict(kwargs), return_dict_in_generate)) or "decoded"
    return m, calls


def test_output_scores_and_logits_are_accepted_and_refusals_hold():
    m, calls = _fake_engine()
    feats = torch.zeros(1, 80, 3000)
    try:
        assert m.generate(feats, output_scores=True, output_logits=True) == "decoded"    # no effect without the dict
        assert m.generate(feats, return_dict_in_generate=True, output_scores=True) == "decoded"
        assert calls == [({"output_scores": True, "output_logits": True}, None), ({"output_scores": True}, True)]
        for bad in (dict(output_attentions=True), dict(output_hidden_states=True), dict(return_timestamps=True),
                    dict(no_speech_threshold=0.6), dict(temperature=0.4), dict(do_sample=True)):
            with pytest.raises(NotImplementedError):
                m.generate(feats, return_dict_in_generate=True, output_scores=True, **bad)
        with pytest.raises(NotImplementedError):   # transcribe has no output objects
            m.transcribe(np.zeros(16000, np.float32), return_dict_in_generate=True)
    finally:
        m._handle = None


def test_generate_output_is_attribute_and_key_indexable():
    seq = torch.tensor([[5, 6]])
    rows = (torch.zeros(1, 4),)
    out = MedusaGenerateOutput(sequences=seq, scores=rows, logits=None, token_logprobs=torch.tensor([[-0.5, -0.25]]),
                               avg_logprob=-0.375, accept_lengths=[1])
    assert out["sequences"] is out.sequences is out[0] is seq
    assert out["scores"] is rows and out[1] is rows
    assert out["logits"] is None and out.keys() == ["sequences", "scores", "token_logprobs", "avg_logprob", "accept_lengths"]
    assert out[2] is out.token_logprobs and out[-1] == [1]
    with pytest.raises(KeyError):
        out["attentions"]
