"""Medusa heads of several ResBlocks (``medusa_num_layers`` = 2, 3 and WM_MAX_HEAD_LAYERS) on the H100, against the fp64
engine-regime oracle and the reference's own loop.

* Raw rows: pass A (every head's row) and every verify row of two iterations, at every ring width, Linear and Block
  heads, K = 1, 4, 10 and 15, through ``_check_two_iterations`` (DECODE_LOGIT_BAR); every decode mode and a 33-CTA grid
  at d = 512; 16-node trees under both attention rules.  Then a whole generate equals the fp32 oracle.
* Tokens against tests/golden/ref_loop_head_layers.npz in all three decode modes, on the whole GPU and on 33 CTAs: a
  stream matches the fixture, or, where the fp16 operand rounding flips an oracle near-tie, the oracle run in the
  engine's regime from the engine's encoder states.
* whisper-large-v2 dimensions at full depth with 2 layers per head and K = 10.
* What reads the heads' output composes: no-speech row, scores and token log-probabilities, token timestamps, logits
  processors, a sampled attempt of temperature fallback, and a StreamGroup of two engines.
"""
import math

import numpy as np
import pytest
import torch

from _decode_ref import DECODE_LOGIT_BAR, check_error, rel_err
from oracle import make_head_layers_golden as G
from oracle import medusa_ref as M
from oracle import no_speech_ref as NS
from oracle import processors_ref as PR
from oracle import sampling_ref as SR
from oracle import timestamps_ref as TS
from oracle import whisper_ref as W
from test_gpu_decode_rows_and_depth import ALL_MODES, MAX_LEN, RING_WIDTHS, _check_two_iterations
from test_gpu_sampling import _sampled
from whisper_medusa_b200 import _lib
from whisper_medusa_b200.synthetic import preset_config, synthetic_audio, synthetic_state_dict, width_config

pytestmark = pytest.mark.gpu

MAXL = _lib.WM_MAX_HEAD_LAYERS
SEED = 3

_MODELS = {}


def _model(cfg, seed=SEED):
    """(model, cfg, sd, pcm); one engine alive at a time."""
    from whisper_medusa_b200 import WhisperMedusaModel

    key = (repr(cfg.to_dict()), seed)
    if key not in _MODELS:
        for m in _MODELS.values():
            m[0].close()
        _MODELS.clear()
        sd = synthetic_state_dict(cfg, seed=seed)
        _MODELS[key] = (WhisperMedusaModel(cfg, sd).to("cuda:0"), cfg, sd, synthetic_audio(5.0, stream_id=seed))
    return _MODELS[key]


def _close_all():
    for m in _MODELS.values():
        m[0].close()
    _MODELS.clear()


# ------------------------------------------------------------------------------------------------------------ raw rows
ROW_CASES = [(d, n, htype, (1, 4, 10, 15)[i % 4])
             for i, (d, n, htype) in enumerate((d, n, h) for d in RING_WIDTHS for n in (2, 3, MAXL)
                                               for h in ("base_head", "medusa_block"))]


@pytest.mark.parametrize("case", ROW_CASES, ids=lambda c: f"d{c[0]}-l{c[1]}-{c[2]}-k{c[3]}")
def test_rows_of_two_iterations(case):
    d, n, htype, k = case
    cfg = width_config(d, heads=k, heads_type=htype, head_layers=n)
    model, cfg, sd, pcm = _model(cfg)
    runs = [("persistent", None)]
    if d == 512:
        runs += [("persistent_simple", None), ("graph", None), ("persistent", 33)]
    _check_two_iterations(model, cfg, sd, pcm, dict(language=None, max_length=MAX_LEN), f"heads{n}/d{d}-{htype}-k{k}",
                          runs)


@pytest.mark.parametrize("case", [(512, 2, (1, 3, 4)), (1280, 3, (1, 3, 2, 1)), (384, MAXL, (1, 3, 4))],
                         ids=lambda c: f"d{c[0]}-l{c[1]}-tree{''.join(map(str, c[2]))}")
def test_tree_rows_both_attention_rules(case):
    d, n, choices = case
    cfg = width_config(d, heads=len(choices) - 1, head_layers=n)
    cfg.medusa_choices = list(choices)
    model, cfg, sd, pcm = _model(cfg)
    runs = [(m, None) for m in ALL_MODES] if d == 512 else [("persistent", None), ("persistent", 33)]
    for ta in (False, True):
        _check_two_iterations(model, cfg, sd, pcm, dict(language=None, max_length=MAX_LEN),
                              f"heads{n}/d{d}-tree" + ("-tree_attn" if ta else ""), runs, tree_attention=ta)


@pytest.mark.parametrize("htype", ["base_head", "medusa_block"])
def test_whole_generate_equals_the_fp32_oracle(htype):
    model, cfg, sd, pcm = _model(width_config(512, heads=4, heads_type=htype, head_layers=3))
    kw = dict(language=None, max_length=MAX_LEN)
    for mode in ALL_MODES:
        model.set_decode_mode(mode)
        out = model.generate_from_pcm(pcm, **kw)[0].tolist()
        tr = model.last_trace
        enc = model.encoder_output()
        prompt = M.init_tokens(cfg, None)
        gp = M.gen_params(cfg, prompt, None, MAX_LEN)
        ref = M.medusa_greedy_search(W.RefWeights(sd), cfg, enc, prompt, gp, "engine")
        assert (tr.sequences, tr.accept_lengths) == (ref.sequences, ref.accept_lengths), mode
        assert out == M.strip_output(ref.sequences, len(prompt), gp)
    model.set_decode_mode("persistent")


# ------------------------------------------------------------------------------------------------ the reference's loop
@pytest.mark.parametrize("mode,ctas", [(m, None) for m in ALL_MODES] + [("persistent", 33)],
                         ids=lambda v: str(v))
def test_engine_matches_the_reference_streams(mode, ctas):
    from whisper_medusa_b200 import WhisperMedusaModel

    _close_all()
    fx = np.load(G.FIXTURE)
    total = flips = 0
    for g, spec in G.GROUPS.items():
        for s in range(spec[5]):
            cfg, sd, pcm, max_len, pen, temp = G.stream_inputs(g, s)
            m = WhisperMedusaModel(cfg, sd).to("cuda:0")
            try:
                m.set_decode_mode(mode)
                if ctas:
                    m.set_option("decode_ctas", ctas)
                m.generate_from_pcm(pcm, max_length=max_len, exponential_decay_length_penalty=pen,
                                    medusa_temperature=temp)
                seq, acc = m.last_trace.sequences, m.last_trace.accept_lengths
                enc = m.encoder_output()
            finally:
                m.close()
            total += 1
            if seq == fx[f"{g}/{s}/sequences"].tolist() and acc == fx[f"{g}/{s}/accept"].tolist():
                continue
            flips += 1
            prompt = M.init_tokens(cfg, "en" if cfg.is_multilingual else None)
            gp = M.gen_params(cfg, prompt, pen, max_len, temperature=temp)
            tr = M.medusa_greedy_search(W.RefWeights(sd), cfg, enc, prompt, gp, "engine")
            assert (seq, acc) == (tr.sequences, tr.accept_lengths), (g, s, mode, ctas)
    print(f"head layers {mode}@{ctas}: {flips} of {total} streams differ from the fixture by a numeric-regime flip")
    assert flips <= total // 5, (flips, total)


# ------------------------------------------------------------------------------------------------------- large-v2 depth
def test_large_v2_full_depth():
    """whisper-large-v2 (d = 1280, 32 layers, 51865 tokens), two ResBlocks per head, K = 10: pass A and the verify rows
    of two iterations against fp64, then the tokens of a 60-token generate against the fp32 oracle."""
    model, cfg, sd, pcm = _model(preset_config("large-v2", heads=10, head_layers=2), seed=7)
    kw = dict(language="en", max_length=60)
    enc = _check_two_iterations(model, cfg, sd, pcm, kw, "heads2/large-v2-k10", [("persistent", None)])
    model.generate_from_pcm(pcm, **kw)
    prompt = M.init_tokens(cfg, "en")
    ref = M.medusa_greedy_search(W.RefWeights(sd), cfg, enc, prompt, M.gen_params(cfg, prompt, None, 60), "engine")
    assert model.last_trace.sequences == ref.sequences
    _close_all()


# ------------------------------------------------------------------------------------------------ what reads the heads
def test_no_speech_row():
    """The no-speech row runs head 0 through all of its layers (one launch each) before the vocabulary product."""
    for n in (2, 3):
        model, cfg, sd, pcm = _model(width_config(512, heads=4, head_layers=n), seed=21)
        out = model.generate_from_pcm(pcm, max_length=60, return_dict_in_generate=True, output_scores=True,
                                      output_no_speech_prob=True)
        prob, row = model.last_no_speech()
        assert prob == out.no_speech_prob
        ref, ref_p = NS.no_speech_row(W.RefWeights(sd, torch.float64), cfg, model.encoder_output().double(),
                                      regime="engine")
        ref = ref.numpy()
        check_error(rel_err(row.numpy(), ref), DECODE_LOGIT_BAR, f"heads{n}/no_speech", "sot_row")
        scale = max(1.0, float(np.abs(ref).max()))
        check_error(abs(math.log(prob) - math.log(ref_p)) / scale, 2 * DECODE_LOGIT_BAR, f"heads{n}/no_speech", "log_p")


@pytest.mark.parametrize("htype", ["base_head", "medusa_block"])
def test_scores_and_processors(htype):
    """Scores rows and token log-probabilities, with logits processors on, against the oracle's record."""
    model, cfg, sd, pcm = _model(preset_config("micro", heads=4, heads_type=htype, head_layers=2), seed=5)
    plain = model.generate_from_pcm(pcm, max_length=100)[0].tolist()
    args = dict(sequence_bias=[[[plain[0]], -30.0], [[plain[0], plain[1]], 2.5]], bad_words_ids=[[plain[2]]],
                no_repeat_ngram_size=2, min_new_tokens=4)
    out = model.generate_from_pcm(pcm, max_length=100, return_dict_in_generate=True, output_scores=True, **args)
    tr_e = model.last_trace
    enc = model.encoder_output()
    prompt = M.init_tokens(cfg, None)
    over = dict(sequence_bias=[((plain[0],), -30.0), ((plain[0], plain[1]), 2.5)], bad_words_ids=[[plain[2]]],
                no_repeat_ngram_size=2, min_new_tokens=4)
    gp = M.gen_params(cfg, prompt, None, 100, **over)
    tr = PR.medusa_greedy_search(W.RefWeights(sd), cfg, enc, prompt, gp, "engine", capture_logits=1 << 20)
    assert (tr.sequences, tr.accept_lengths) == (tr_e.sequences, tr_e.accept_lengths)
    assert out.sequences[0].tolist() != plain
    sc = PR.loop_scores(tr, len(prompt), gp, cfg.medusa_choices)
    n_tok = min(tr_e.n_new_tokens, len(sc.token_logprobs))
    lp = out.token_logprobs[0, :n_tok].cpu().double().numpy()
    err = max(abs(float(lp[j]) - sc.token_logprobs[j]) / sc.token_scales[j] for j in range(n_tok))
    check_error(err, 2 * DECODE_LOGIT_BAR, f"heads2/{htype}", "token_logprobs")
    worst = 0.0
    for i, row in enumerate(out.scores):
        got, ref = row[0].cpu().double(), sc.rows[i].double()
        assert torch.equal(torch.isneginf(got), torch.isneginf(ref)), i
        fin = torch.isfinite(ref)
        worst = max(worst, float((got[fin] - ref[fin]).abs().max()) / max(1.0, float(ref[fin].abs().max())))
    check_error(worst, DECODE_LOGIT_BAR, f"heads2/{htype}", "scores")


def test_token_timestamps_capture():
    model, cfg, sd, pcm = _model(width_config(384, heads=4, head_layers=3), seed=8)
    H = cfg.decoder_attention_heads
    model.generation_config.alignment_heads = [[cfg.decoder_layers - 1, h] for h in range(H)] + [[0, H - 1]]
    out = model.generate_from_pcm(pcm, max_length=80, return_token_timestamps=True, return_dict_in_generate=True)
    tr = model.last_trace
    seq = tr.sequences[: len(model._init_tokens(None, None)) + tr.n_new_tokens]
    got = model.last_alignment_probs(0, len(seq) - 1).double()
    ref, scores = TS.alignment_probs(W.RefWeights(sd, torch.float64), cfg, seq[:-1], model.encoder_output().double(),
                                     model.generation_config.alignment_heads, regime="engine", return_scores=True)
    mask = ref > 1e-20
    err = float((got.clamp_min(1e-300).log() - ref.log())[mask].abs().max())
    check_error(err / max(1.0, float(scores.abs().max())), 2 * DECODE_LOGIT_BAR, "heads3/timestamps", "alignment")
    assert out.token_timestamps.shape == out.sequences.shape


@pytest.mark.parametrize("htype", ["base_head", "medusa_block"])
def test_sampled_attempt(htype):
    """A sampled attempt of temperature fallback against the oracle's sampled loop: tokens equal, or the oracle met a
    near-tie; most seeds match in full, with top-k-restricted token log-probabilities within 2 x DECODE_LOGIT_BAR."""
    model, cfg, sd, pcm = _model(preset_config("micro", heads=4, heads_type=htype, head_layers=2), seed=4)
    model.generate_from_pcm(pcm, max_length=20)
    enc = model.encoder_output()
    prompt = M.init_tokens(cfg)
    gp = M.gen_params(cfg, prompt, None, 72)
    full = 0
    for s in range(4):
        seed = (s, 2000 + s)
        ref = SR.sampled_search(W.RefWeights(sd), cfg, enc, prompt, gp, 0.6, 50, seed, 0, 1, regime="engine")
        out = _sampled(model, 0.6, 50, seed=seed, max_length=72)
        got = model.last_trace.sequences
        if got == ref.sequences:
            full += 1
            n = model.last_trace.n_new_tokens
            lp = out.token_logprobs[0, :n].cpu().double().numpy()
            err = max(abs(float(lp[j]) - ref.token_logprobs[j]) / ref.token_scales[j] for j in range(n))
            assert err <= 2 * DECODE_LOGIT_BAR, (seed, err)
        else:
            assert ref.min_gap < 2e-3 * max(ref.token_scales), (seed, got, ref.sequences)
    assert full >= 3, full


def test_stream_group_equals_single_engine():
    from whisper_medusa_b200 import WhisperMedusaModel
    from whisper_medusa_b200.streams import StreamGroup

    _close_all()
    cfg = preset_config("tiny.en", heads=4, head_layers=3)
    sd = synthetic_state_dict(cfg, seed=3)
    clips = [synthetic_audio(6.0, stream_id=s) for s in range(3)]
    m = WhisperMedusaModel(cfg, sd).to("cuda:0")
    try:
        single = [m.generate_from_pcm(c)[0].tolist() for c in clips]
    finally:
        m.close()
    g = StreamGroup(cfg, sd, "cuda:0", n_streams=2)
    try:
        assert [o[0].tolist() for o in g.generate_from_pcm(clips)] == single
    finally:
        g.close()
