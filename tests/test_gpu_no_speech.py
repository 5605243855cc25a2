"""GPU tests of the no-speech probability (generate(..., output_no_speech_prob=True), transcribe(no_speech_threshold=...)).

* The raw SOT row from the kernel against the fp64 oracle (oracle/no_speech_ref.py, engine regime) decoding from the
  engine's own encoder states, at every ring-kernel width with the realistic activation profiles: within
  DECODE_LOGIT_BAR of the row's logit scale; log p[no_speech] (a logit minus a log-sum-exp) within twice that.
* The same row against the engine's own forward(decoder_input_ids=[[SOT]], disable_medusa=True) in the same decode
  mode.  The decoder's arithmetic on the SOT row does not depend on the rows after it (causal attention, row-wise GEMM
  tiles), so both paths feed the same fp32 hidden row to the last products and differ only in their summation order:
  mma.sync tiles in the loop, an FMA chain in csrc/no_speech.cu.  For a d-term fp32 sum of exact products either order
  is within gamma_d = d u / (1 - d u) of the exact sum relative to sum |w_k x_k| (u = 2^-23: one bit more than
  round-to-nearest, for the tensor cores' truncating adds).  The bar of logit j is therefore
  2 gamma_d sum_k |E_jk| |y_k|, plus, for the base_head type, head 0's own bound carried through |SiLU'| <= 1.1 and the
  vocabulary matrix.  It is computed from the oracle's hidden row before the comparison.  The engine sets the capture
  buffer to NaN before each loop, so a decode mode whose loop missed the row fails instead of reusing an older one.
* Capture changes nothing: sequences, accept lengths and token log-probabilities are bit-identical with the capture on
  and off, in every decode mode, on chains (K = 1, 4, 10), 16-node trees under both attention rules and a 20-token prompt
  whose SOT row is in the final tile; a SOT row in a prefill chunk raises NotImplementedError.
* transcribe on a recording of synthetic speech and exact silence, with thresholds set between the windows' measured
  values: the skipped set is the rule's, kept windows equal the run without thresholds, the merge treats skipped windows
  as empty, StreamGroup (S = 1, 2, 4) equals model.transcribe, and without thresholds nothing changes.
"""
import math

import numpy as np
import pytest
import torch

from _decode_ref import DECODE_LOGIT_BAR, check_error, rel_err
from oracle import no_speech_ref as NS
from oracle import whisper_ref as W
from whisper_medusa_b200.longform import merge_windows, skip_window, text_ids
from whisper_medusa_b200.synthetic import ACTIVATION_PROFILES, synthetic_audio, synthetic_state_dict, width_config

pytestmark = pytest.mark.gpu

RING_WIDTHS = (128, 384, 512, 768, 1024, 1280)
ALL_MODES = ("persistent", "graph", "persistent_simple")
NS_DICT = dict(return_dict_in_generate=True, output_scores=True, output_no_speech_prob=True)
SCORE_DICT = dict(return_dict_in_generate=True, output_scores=True)

_MODELS = {}


def _model(cfg, seed, profile="default"):
    """One engine alive at a time."""
    from whisper_medusa_b200 import WhisperMedusaModel

    key = (repr(cfg.to_dict()), seed, profile)
    if key not in _MODELS:
        for m in _MODELS.values():
            m[0].close()
        _MODELS.clear()
        sd = synthetic_state_dict(cfg, seed=seed, activation_profile=profile)
        _MODELS[key] = (WhisperMedusaModel(cfg, sd).to("cuda:0"), sd)
    return _MODELS[key]


def _sot(model):
    return int(model.generation_config.decoder_start_token_id)


# ------------------------------------------------------------------------------------------------ against the oracle
CASES = [(d, ACTIVATION_PROFILES[1 + i % (len(ACTIVATION_PROFILES) - 1)], "base_head") for i, d in enumerate(RING_WIDTHS)]
CASES += [(512, "outliers", "medusa_block"), (1280, "near_top", "medusa_block")]


@pytest.mark.parametrize("case", CASES, ids=[f"d{c[0]}_{c[1]}_{c[2]}" for c in CASES])
def test_row_against_fp64_oracle(case):
    d, profile, heads_type = case
    cfg = width_config(d, heads=4, heads_type=heads_type)
    model, sd = _model(cfg, 20 + RING_WIDTHS.index(d), profile)
    out = model.generate_from_pcm(synthetic_audio(5.0, stream_id=2), max_length=60, **NS_DICT)
    prob, row = model.last_no_speech()
    assert prob == out.no_speech_prob
    ref, ref_p = NS.no_speech_row(W.RefWeights(sd, torch.float64), cfg, model.encoder_output().double(), regime="engine")
    ref = ref.numpy()
    name = f"no_speech d{d} {profile} {heads_type}"
    check_error(rel_err(row.numpy(), ref), DECODE_LOGIT_BAR, name, "sot_row")
    scale = max(1.0, float(np.abs(ref).max()))
    check_error(abs(math.log(prob) - math.log(ref_p)) / scale, 2 * DECODE_LOGIT_BAR, name, "log_p_no_speech")


def _sum_bound(Wm, x, d):
    """gamma_d sum_k |W_jk| |x_k| per row j, with u = 2^-23."""
    u = 2.0 ** -23
    gamma = d * u / (1 - d * u)
    return gamma * (np.abs(Wm) @ np.abs(x))


@pytest.mark.parametrize("heads_type", ["base_head", "medusa_block"])
def test_row_against_engine_forward(heads_type):
    cfg = width_config(512, heads=4, heads_type=heads_type)
    model, sd = _model(cfg, 5, "gamma_spread")
    pcm = synthetic_audio(5.0, stream_id=4)
    # the bar, from the oracle's hidden row (fp64) before anything runs on the engine's side
    model.generate_from_pcm(pcm, max_length=40)
    w = W.RefWeights(sd, torch.float64)
    enc = model.encoder_output().double()
    hidden = W.decoder_forward(w, cfg, [_sot(model)], [0], enc, W.new_cache(cfg), "engine")[0].numpy()
    E = sd["whisper_model.proj_out.weight"].double().numpy()
    if heads_type == "base_head":
        W0 = sd["medusa_heads.0.0.linear.weight"].double().numpy()
        b0 = sd["medusa_heads.0.0.linear.bias"].double().numpy()
        y = hidden + torch.nn.functional.silu(torch.from_numpy(W0 @ hidden + b0)).numpy()
        bar = 2 * _sum_bound(E, y, cfg.d_model) + np.abs(E) @ (1.1 * 2 * _sum_bound(W0, hidden, cfg.d_model))
    else:
        bar = 2 * _sum_bound(E, hidden, cfg.d_model)
    ran = []
    for mode in ALL_MODES:
        model.set_decode_mode(mode)
        model.generate_from_pcm(pcm, max_length=40, **NS_DICT)
        # (the capture buffer is NaN before each loop: a mode whose loop missed the row would raise here)
        p0, row = model.last_no_speech()
        fwd = model.forward(decoder_input_ids=torch.tensor([[_sot(model)]]), disable_medusa=True).logits
        fwd = fwd.reshape(-1).float().cpu().numpy()
        p1, row1 = model.last_no_speech()      # forward passes leave the captured row alone
        assert p1 == p0 and torch.equal(row1, row)
        diff = np.abs(row.numpy().astype(np.float64) - fwd)
        assert (diff <= bar).all(), (mode, float(diff.max()), float(bar[diff.argmax()]), float((diff / bar).max()))
        ran.append(mode)
    model.set_decode_mode("persistent")
    assert len(ran) == 3


# ------------------------------------------------------------------------------------------------ capture changes nothing
CAPTURE_CASES = [
    ("chain_k1", 1, None, dict(max_length=200)),
    ("chain_k4", 4, None, dict(max_length=200)),
    ("chain_k10", 10, None, dict(max_length=200)),
    ("tree_134_causal", 2, (1, 3, 4), dict(max_length=200, tree_attention=False)),
    ("tree_134_ancestors", 2, (1, 3, 4), dict(max_length=200, tree_attention=True)),
    ("tree_1321_causal", 3, (1, 3, 2, 1), dict(max_length=200, tree_attention=False)),
    ("tree_1321_ancestors", 3, (1, 3, 2, 1), dict(max_length=200, tree_attention=True)),
    ("prompt20", 4, None, dict(max_length=200)),
]


@pytest.mark.parametrize("case", CAPTURE_CASES, ids=[c[0] for c in CAPTURE_CASES])
def test_capture_changes_nothing(case):
    from whisper_medusa_b200 import EngineError

    name, k, choices, kw = case
    cfg = width_config(512, heads=k)
    if choices:
        cfg.medusa_choices = list(choices)
    model, sd = _model(cfg, 3)
    pcm = synthetic_audio(5.0, stream_id=3)
    kw = dict(kw)
    if name == "prompt20":     # SOT at index 17 of 20: the final tile (rows 16..19); 16 rows are prefilled first
        rng = np.random.default_rng(20)
        prompt = [int(t) for t in rng.integers(20, 400, size=20)]
        prompt[17] = _sot(model)
        kw["decoder_input_ids"] = torch.tensor([prompt])
    ran = []
    try:
        for mode in ALL_MODES:
            try:
                model.set_decode_mode(mode)
            except EngineError:
                continue
            off = model.generate_from_pcm(pcm, **SCORE_DICT, **kw)
            tr_off = model.last_trace
            on = model.generate_from_pcm(pcm, **NS_DICT, **kw)
            tr_on = model.last_trace
            assert tr_on.sequences == tr_off.sequences and tr_on.accept_lengths == tr_off.accept_lengths, (name, mode)
            assert torch.equal(on.sequences, off.sequences)
            assert torch.equal(on.token_logprobs, off.token_logprobs), (name, mode)
            assert all(torch.equal(a, b) for a, b in zip(on.scores, off.scores))
            assert off.no_speech_prob is None and 0.0 <= on.no_speech_prob <= 1.0
            assert tr_on.launches_decode == tr_off.launches_decode + (1 if cfg.is_block else 2)
            # switched off again: the launches of a call without it
            model.generate_from_pcm(pcm, **SCORE_DICT, **kw)
            assert model.last_trace.launches_decode == tr_off.launches_decode
            ran.append(mode)
    finally:
        model.set_decode_mode("persistent")
    assert "persistent" in ran and len(ran) >= 2, ran


def test_sot_row_in_a_prefill_chunk_raises():
    cfg = width_config(512, heads=4)
    model, sd = _model(cfg, 3)
    prompt = [_sot(model)] + [30 + i for i in range(19)]        # 20 tokens, SOT in the first (prefilled) chunk
    with pytest.raises(NotImplementedError):
        model.generate_from_pcm(synthetic_audio(5.0, stream_id=3), max_length=100,
                                decoder_input_ids=torch.tensor([prompt]), **NS_DICT)
    # the engine is left usable and the option off
    plain = model.generate_from_pcm(synthetic_audio(5.0, stream_id=3), max_length=100)
    assert plain.shape[0] == 1


# ------------------------------------------------------------------------------------------------ transcribe
def _recording():
    """Synthetic speech with stretches of exact silence, 16 kHz."""
    parts = [synthetic_audio(6.0, stream_id=1), np.zeros(14 * 16000, np.float32), synthetic_audio(7.0, stream_id=2),
             np.zeros(12 * 16000, np.float32), synthetic_audio(5.0, stream_id=5)]
    return np.concatenate(parts).astype(np.float32)


def test_transcribe_skips_silent_windows():
    from whisper_medusa_b200 import StreamGroup

    cfg = width_config(384, heads=4)
    model, sd = _model(cfg, 7)
    x = _recording()
    kw = dict(chunk_length_s=10.0, max_length=80)
    base = model.transcribe(x, **kw)
    base_wins = [(r.ids, r.trace.launches_decode) for r in model.last_windows]
    assert all(r.no_speech_prob is None and r.skipped is None for r in model.last_windows)
    # measure every window's values with thresholds that skip nothing
    model.transcribe(x, no_speech_threshold=1.0, logprob_threshold=-1e9, **kw)
    probe = [(r.no_speech_prob, r.avg_logprob) for r in model.last_windows]
    assert not any(r.skipped for r in model.last_windows)
    ps = sorted(set(p for p, _ in probe))
    assert len(ps) >= 2, probe
    # thresholds between measured values: skip on p alone (every avg_logprob < 1.0), cut between two distinct probabilities
    cut = len(ps) // 2
    nst, lpt = (ps[cut - 1] + ps[cut]) / 2, 1.0
    got = model.transcribe(x, no_speech_threshold=nst, logprob_threshold=lpt, **kw)
    wins = model.last_windows
    skipped = [r.skipped for r in wins]
    assert skipped == [skip_window(r.no_speech_prob, r.avg_logprob, nst, lpt) for r in wins]
    assert any(skipped) and not all(skipped), probe
    eos = int(model.generation_config.eos_token_id)
    for r, (ids, _) in zip(wins, base_wins):
        assert r.ids == ids           # decoding is the same with the rule on; only the merge drops skipped windows
    assert got[0].tolist() == merge_windows([[] if s else text_ids(ids, eos) for s, (ids, _) in zip(skipped, base_wins)])
    # without thresholds: results and launches are today's
    again = model.transcribe(x, **kw)
    assert torch.equal(again, base)
    assert [(r.ids, r.trace.launches_decode) for r in model.last_windows] == base_wins
    model.close()
    _MODELS.clear()
    for S in (1, 2, 4):
        group = StreamGroup(cfg, sd, "cuda:0", n_streams=S)
        try:
            out = group.transcribe(x, no_speech_threshold=nst, logprob_threshold=lpt, **kw)[0]
            assert torch.equal(out.cpu(), got.cpu()), S
            assert [r.skipped for r in group.last_windows[0]] == skipped, S
        finally:
            group.close()
