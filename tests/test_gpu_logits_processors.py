"""GPU tests of the logits processors: generate(sequence_bias=..., bad_words_ids=..., no_repeat_ngram_size=...,
min_length=..., min_new_tokens=...).

* Tokens and accept lengths against tests/golden/ref_loop_processors.npz (oracle/make_processors_golden.py, held there to
  the reference's own loop): micro and tiny.en synthetic weights, Linear and Block heads, chains and branching trees,
  temperature 0 and 1, the EOS decay on.  As in test_gpu_parity's unselected streams, a stream either matches the
  fixture or the oracle run in the engine's rounding regime from the engine's encoder states.
* whisper-large-v2 synthetic weights: the engine against that oracle directly (its CPU run takes the place of a fixture).
* Scores rows and token log-probabilities carry the processing.
* transcribe and StreamGroup give what per-window / single-engine generate gives with the same options.
"""
import numpy as np
import pytest
import torch

from _decode_ref import DECODE_LOGIT_BAR, check_error
from oracle import make_processors_golden as PG
from oracle import make_ref_golden as G
from oracle import medusa_ref as M
from oracle import processors_ref as PR
from oracle import whisper_ref as W
from whisper_medusa_b200.synthetic import preset_config, synthetic_audio, synthetic_state_dict

pytestmark = pytest.mark.gpu


def _oracle_engine_regime(cfg, sd, enc, prompt, gp, capture=0):
    return PR.medusa_greedy_search(W.RefWeights(sd), cfg, enc, prompt, gp, "engine", capture_logits=capture)


def _gp(cfg, prompt, pen, max_len, temp, alpha, thr, args):
    return M.gen_params(cfg, prompt, pen, max_len, temperature=temp, posterior_alpha=alpha, posterior_threshold=thr,
                        **PG._gp_over(args, int(cfg.eos_token_id)))


def test_engine_matches_the_fixtures():
    from whisper_medusa_b200 import WhisperMedusaModel

    fx = np.load(PG.FIXTURE)
    total = flips = 0
    for name, (group, _) in PG.SCENARIOS.items():
        cfg, sd, pcm, max_len, pen, temp, alpha, thr = G.stream_inputs(group, 0)
        args = PG.scenario_args(name, fx[f"{name}/plain"].tolist())
        m = WhisperMedusaModel(cfg, sd).to("cuda:0")
        m.generate_from_pcm(pcm, max_length=max_len, exponential_decay_length_penalty=pen, medusa_temperature=temp,
                            posterior_alpha=alpha, posterior_threshold=thr, **args)
        seq, acc = m.last_trace.sequences, m.last_trace.accept_lengths
        enc = m.encoder_output()
        m.close()
        total += 1
        if seq == fx[f"{name}/sequences"].tolist() and acc == fx[f"{name}/accept"].tolist():
            continue
        flips += 1
        prompt = M.init_tokens(cfg, None)
        tr = _oracle_engine_regime(cfg, sd, enc, prompt, _gp(cfg, prompt, pen, max_len, temp, alpha, thr, args))
        assert seq == tr.sequences and acc == tr.accept_lengths, name
    print(f"processors: {flips} of {total} scenarios differ from the fixture by a numeric-regime flip")
    assert flips <= total // 5, (flips, total)


def test_large_v2_against_the_oracle():
    from whisper_medusa_b200 import WhisperMedusaModel

    cfg = preset_config("large-v2", heads=4)
    sd = synthetic_state_dict(cfg, seed=7)
    pcm = synthetic_audio(8.0, stream_id=7)
    m = WhisperMedusaModel(cfg, sd).to("cuda:0")
    kw = dict(language="en", max_length=60, exponential_decay_length_penalty=(40, 1.05))
    plain = m.generate_from_pcm(pcm, **kw)[0].tolist()
    args = dict(sequence_bias=[[[plain[0]], -30.0], [[plain[0], plain[1]], 2.5]], bad_words_ids=[[plain[2]]],
                no_repeat_ngram_size=2, min_new_tokens=6)
    out = m.generate_from_pcm(pcm, **kw, **args)[0].tolist()
    seq, acc = m.last_trace.sequences, m.last_trace.accept_lengths
    enc = m.encoder_output()
    m.close()
    assert out != plain
    prompt = M.init_tokens(cfg, "en")
    gp = _gp(cfg, prompt, (40, 1.05), 60, 1.0, 0.3, 0.09, args)
    tr = _oracle_engine_regime(cfg, sd, enc, prompt, gp)
    assert seq == tr.sequences and acc == tr.accept_lengths


@pytest.mark.parametrize("name", ["micro_lin_t1/all", "micro_tree122_t1/all", "micro_lin_pen/all"])
def test_scores_carry_the_processing(name):
    from whisper_medusa_b200 import WhisperMedusaModel

    fx = np.load(PG.FIXTURE)
    group, _ = PG.SCENARIOS[name]
    cfg, sd, pcm, max_len, pen, temp, alpha, thr = G.stream_inputs(group, 0)
    args = PG.scenario_args(name, fx[f"{name}/plain"].tolist())
    m = WhisperMedusaModel(cfg, sd).to("cuda:0")
    out = m.generate_from_pcm(pcm, max_length=max_len, exponential_decay_length_penalty=pen, medusa_temperature=temp,
                              posterior_alpha=alpha, posterior_threshold=thr, return_dict_in_generate=True,
                              output_scores=True, **args)
    tr_e = m.last_trace
    enc = m.encoder_output()
    m.close()
    prompt = M.init_tokens(cfg, None)
    gp = _gp(cfg, prompt, pen, max_len, temp, alpha, thr, args)
    tr = _oracle_engine_regime(cfg, sd, enc, prompt, gp, capture=1 << 20)
    assert tr.sequences == tr_e.sequences
    sc = PR.loop_scores(tr, len(prompt), gp, cfg.medusa_choices)
    n_tok = min(tr_e.n_new_tokens, len(sc.token_logprobs))
    lp = out.token_logprobs[0, :n_tok].cpu().double().numpy()
    err = max(abs(float(lp[j]) - sc.token_logprobs[j]) / sc.token_scales[j] for j in range(n_tok))
    check_error(err, 2 * DECODE_LOGIT_BAR, name, "token_logprobs")
    worst = 0.0
    for i, row in enumerate(out.scores):
        got, ref = row[0].cpu().double(), sc.rows[i].double()
        assert torch.equal(torch.isneginf(got), torch.isneginf(ref)), (name, i)
        fin = torch.isfinite(ref)
        worst = max(worst, float((got[fin] - ref[fin]).abs().max()) / max(1.0, float(ref[fin].abs().max())))
    check_error(worst, DECODE_LOGIT_BAR, name, "scores")


def test_transcribe_and_stream_group_equal_generate():
    from whisper_medusa_b200 import WhisperMedusaModel
    from whisper_medusa_b200.streams import StreamGroup

    cfg = preset_config("tiny.en", heads=4)
    sd = synthetic_state_dict(cfg, seed=3)
    audio = np.concatenate([synthetic_audio(20.0, stream_id=s) for s in (3, 4)])
    opts = dict(sequence_bias=[[[300], 1.5], [[11, 300], -0.5]], bad_words_ids=[[13], [220, 11]],
                no_repeat_ngram_size=3, min_new_tokens=3)
    m = WhisperMedusaModel(cfg, sd).to("cuda:0")
    merged = m.transcribe(audio, **opts)
    assert merged.shape[1] > 0
    for w in m.last_windows:
        assert w.ids == m.generate_from_pcm(audio[w.start:w.end], **opts)[0].tolist()
    clips = [synthetic_audio(6.0, stream_id=s) for s in range(3)]
    single = [m.generate_from_pcm(c, **opts)[0].tolist() for c in clips]
    plain = [m.generate_from_pcm(c)[0].tolist() for c in clips]
    assert single != plain
    m.close()
    g = StreamGroup(cfg, sd, "cuda:0", n_streams=2)
    try:
        assert [o[0].tolist() for o in g.generate_from_pcm(clips, **opts)] == single
        assert [o[0].tolist() for o in g.transcribe(audio, **opts)] == [merged[0].tolist()]
    finally:
        g.close()
