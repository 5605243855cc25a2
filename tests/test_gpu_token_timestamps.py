"""GPU tests of token-level timestamps (generate(return_token_timestamps=True)), against the fp64 oracle.

* Capture: the cross-attention probabilities the loop kept at every position of the engine's own sequence against the
  oracle's teacher-forced rows of that sequence (oracle/timestamps_ref.py, engine regime, the engine's encoder states),
  at every ring width and at a width without a ring kernel, both head types, all three decode modes, chains K = 1, 4,
  10 and 15, the realistic, accept-0 and all-accept regimes, a 20-token prompt (prefill), a partial grid and a run to
  max_length 448.  Bar: a cross-attention score is a decoder logit and is held to DECODE_LOGIT_BAR of the row's score
  scale (DESIGN.md section 2).  A log-probability is the score minus the row's log-sum-exp, which moves by at most the
  largest score error, so |log p - log p_ref| <= 2 DECODE_LOGIT_BAR max(1, max|s_ref|) wherever p_ref > 1e-20.
* Extraction on the engine's rows: the matrix within 1e-4 of max(1, max|matrix|) of HF's fp32 torch computation on the
  same rows (only the order and width of the mean / std sums differ); the DTW jumps and the timestamps bit-equal to
  HF's _dynamic_time_warping on the engine's matrix; crafted rows (NaN columns, N = 0 / 1, crops, a filter wider than
  the crop, filter widths 1 / 5 / 7 / 9) equal HF.
* End to end against HF's extraction on the fp64 oracle's rows: identical except at DTW near-ties the matrix bar
  explains, and those are counted and kept rare.
* Timestamps change nothing: tokens, accept lengths, scores, token log-probabilities, no-speech probability and the
  launch count are bit-identical with them on and off; two runs are bit-equal; a forward() after generate does not
  change them; StreamGroup.generate with a batch of feature-extractor masks equals batch-1 runs with each row's mask.
"""
import numpy as np
import pytest
import torch

from _decode_ref import DECODE_LOGIT_BAR, check_error
from oracle import timestamps_ref as TS
from oracle import whisper_ref as W
from whisper_medusa_b200.synthetic import ACTIVATION_PROFILES, synthetic_audio, synthetic_state_dict, width_config

pytestmark = pytest.mark.gpu

RING_WIDTHS = (128, 384, 512, 768, 1024, 1280)
FALLBACK_WIDTH = 256          # no ring-kernel instantiation: the stage / iteration kernels
REGIMES = {
    "realistic": {},
    "accept0": dict(posterior_threshold=1.5, posterior_alpha=1e9),   # no candidate passes
    "allaccept": dict(posterior_threshold=0.0, posterior_alpha=0.0),  # every candidate passes
}
_MODELS = {}


def _model(cfg, seed, profile="default"):
    from whisper_medusa_b200 import WhisperMedusaModel

    key = (repr(cfg.to_dict()), seed, profile)
    if key not in _MODELS:
        for m in _MODELS.values():
            m[0].close()
        _MODELS.clear()
        sd = synthetic_state_dict(cfg, seed=seed, activation_profile=profile)
        m = WhisperMedusaModel(cfg, sd).to("cuda:0")
        H = cfg.decoder_attention_heads
        # every head of the last layer, one of the first, and a duplicate
        m.generation_config.alignment_heads = [[cfg.decoder_layers - 1, h] for h in range(H)] + [[0, H - 1], [0, H - 1]]
        _MODELS[key] = (m, sd)
    return _MODELS[key]


def _check_capture(model, sd, cfg, seq, n_prompt, case):
    n = len(seq)
    got = model.last_alignment_probs(0, n - 1).double()
    pairs = model.generation_config.alignment_heads
    ref, scores = TS.alignment_probs(W.RefWeights(sd, torch.float64), cfg, seq[: n - 1], model.encoder_output().double(),
                                     pairs, regime="engine", return_scores=True)
    mask = ref > 1e-20
    err = float((got.clamp_min(1e-300).log() - ref.log())[mask].abs().max())
    scale = max(1.0, float(scores.abs().max()))
    check_error(err / scale, 2 * DECODE_LOGIT_BAR, case, "alignment_log_probs")
    return got, ref


CASES = []
for i, d in enumerate(RING_WIDTHS + (FALLBACK_WIDTH,)):
    CASES.append((d, "base_head" if i % 2 == 0 else "medusa_block", (1, 4, 10, 15)[i % 4], list(REGIMES)[i % 3],
                  ACTIVATION_PROFILES[i % len(ACTIVATION_PROFILES)]))


@pytest.mark.parametrize("case", CASES, ids=[f"d{c[0]}_{c[1]}_k{c[2]}_{c[3]}" for c in CASES])
def test_capture_against_fp64_oracle(case):
    d, heads_type, K, regime, profile = case
    cfg = width_config(d, heads=K, heads_type=heads_type)
    model, sd = _model(cfg, 40 + d % 97, profile)
    modes = ("persistent", "graph", "persistent_simple") if d != FALLBACK_WIDTH else ("graph", "persistent_simple")
    for mode in modes:
        model.set_decode_mode(mode)
        out = model.generate_from_pcm(synthetic_audio(6.0, stream_id=d % 7), max_length=80, return_token_timestamps=True,
                                      return_dict_in_generate=True, **REGIMES[regime])
        tr = model.last_trace
        n_prompt = len(model._init_tokens(None, None))
        seq = tr.sequences[: n_prompt + tr.n_new_tokens]
        _check_capture(model, sd, cfg, seq, n_prompt, f"{case} {mode}")
        assert out.token_timestamps.shape == out.sequences.shape
    model.set_decode_mode("persistent" if d != FALLBACK_WIDTH else "graph")


@pytest.mark.parametrize("what", ["prefill_prompt", "partial_grid", "max_length"])
def test_capture_long_prompt_partial_grid_and_long_run(what):
    cfg = width_config(512, heads=4)
    model, sd = _model(cfg, 7, "gamma_spread")
    kw = dict(max_length=120)
    if what == "prefill_prompt":
        base = model._init_tokens(None, None)
        kw["decoder_input_ids"] = torch.tensor([list(range(3, 3 + 18)) + base])
    if what == "partial_grid":
        model.set_option("decode_ctas", 40)
    if what == "max_length":
        kw = dict(max_length=448, **REGIMES["allaccept"])
    try:
        out = model.generate_from_pcm(synthetic_audio(8.0, stream_id=3), return_token_timestamps=True, **kw)
        tr = model.last_trace
        n_prompt = len(kw["decoder_input_ids"][0]) if "decoder_input_ids" in kw else len(model._init_tokens(None, None))
        seq = tr.sequences[: n_prompt + tr.n_new_tokens]
        _check_capture(model, sd, cfg, seq, n_prompt, what)
        assert out.keys() == ["sequences", "token_timestamps"]
    finally:
        if what == "partial_grid":
            model.set_option("decode_ctas", torch.cuda.get_device_properties(0).multi_processor_count)


def test_extraction_matches_hf_on_engine_rows():
    from transformers.models.whisper.generation_whisper import _dynamic_time_warping

    cfg = width_config(1280, heads=10)
    model, sd = _model(cfg, 3, "default")
    pcm = synthetic_audio(12.0, stream_id=1)
    nf = model.pcm_num_frames(pcm.size)
    out = model.generate_from_pcm(pcm, max_length=200, return_token_timestamps=True)
    tr = model.last_trace
    P = len(model._init_tokens(None, None))
    n = P + tr.n_new_tokens
    for num_frames in (nf, None):
        ts, mat, jumps = model.last_timestamp_matrix(P, n, num_frames)
        N = n - 1 - P
        probs = model.last_alignment_probs(P, N)
        ref = TS.alignment_matrix(probs, num_frames)
        err = float((mat - ref).abs().max()) / max(1.0, float(ref.abs().max()))
        assert err <= 1e-4, err
        text, time = _dynamic_time_warping(-mat.double().numpy())
        hf_j = TS.jumps_of(text, time)
        np.testing.assert_array_equal(jumps.numpy(), hf_j)
        np.testing.assert_array_equal(ts.numpy(), TS.assemble(hf_j, P, 0.02))
        if num_frames == nf:
            np.testing.assert_array_equal(out.token_timestamps[0].cpu().numpy(), ts.numpy()[P : P + out.sequences.shape[1]])


def test_crafted_rows_match_hf():
    cfg = width_config(512, heads=4)
    model, _ = _model(cfg, 7, "gamma_spread")
    g = torch.Generator().manual_seed(0)
    cases = []
    for N, W_, nf, tp in [(0, 30, None, 0.02), (1, 30, None, 0.02), (2, 40, None, 0.02), (9, 200, 101, 0.01),
                          (20, 1500, 5, 0.02), (33, 1500, 1, 0.02), (448, 1500, None, 0.02), (57, 90, 3000, 0.04)]:
        p = torch.softmax(3 * torch.randn(3, N, W_, generator=g), dim=-1)
        if N >= 2:
            p[1, :, 5:9] = 0.25                       # all-equal columns: std 0, NaN
        cases.append((p, nf, tp))
    for (p, nf, tp), width in [(c, 7) for c in cases] + [(c, w) for c in cases[2:5] for w in (1, 5, 9)]:
        P = 3
        ts, mat, jumps = model.timestamps_from_probs(p, P, nf, tp, filter_width=width)
        ref_ts, ref_mat, _ = TS.extract(p, P, nf, width, tp)
        if p.shape[1] == 0:
            np.testing.assert_array_equal(ts.numpy(), ref_ts)
            continue
        both_nan = torch.isnan(mat) & torch.isnan(ref_mat)
        assert torch.equal(torch.isnan(mat), torch.isnan(ref_mat))
        d = (mat - ref_mat).abs()[~both_nan]
        assert d.numel() == 0 or float(d.max()) <= 1e-4 * max(1.0, float(ref_mat[~both_nan].abs().max()))
        np.testing.assert_array_equal(ts.numpy(), ref_ts, err_msg=str((p.shape, nf, tp)))


def test_end_to_end_against_fp64_oracle():
    """Engine timestamps against HF's extraction of the fp64 oracle's rows: differences only at DTW near-ties."""
    n_diff, n_all = 0, 0
    for d, seed, K in ((1280, 3, 10), (768, 5, 4)):
        cfg = width_config(d, heads=K)
        model, sd = _model(cfg, seed, "default")
        pcm = synthetic_audio(10.0, stream_id=seed)
        nf = model.pcm_num_frames(pcm.size)
        model.generate_from_pcm(pcm, max_length=160, return_token_timestamps=True)
        tr = model.last_trace
        P = len(model._init_tokens(None, None))
        n = P + tr.n_new_tokens
        ts, _, _ = model.last_timestamp_matrix(P, n, nf)
        ref = TS.alignment_probs(W.RefWeights(sd, torch.float64), cfg, tr.sequences[: n - 1], model.encoder_output().double(),
                                 model.generation_config.alignment_heads, regime="engine")
        ref_ts, _, _ = TS.extract(ref[:, P:].float(), P, nf, 7, 0.02)
        n_diff += int((ts.numpy() != ref_ts).sum())
        n_all += n - P
        assert float(np.abs(ts.numpy() - ref_ts).max()) <= 0.1, (d, ts, ref_ts)
    print(f"end to end: {n_diff} of {n_all} timestamps differ from the fp64 oracle's")
    assert n_diff <= max(2, n_all // 20), (n_diff, n_all)


def test_timestamps_change_nothing():
    from whisper_medusa_b200.streams import StreamGroup

    cfg = width_config(1280, heads=10)
    model, sd = _model(cfg, 3, "default")
    pcm = synthetic_audio(9.0, stream_id=6)
    kw = dict(max_length=150, return_dict_in_generate=True, output_scores=True, output_no_speech_prob=True)
    for mode in ("persistent", "graph", "persistent_simple"):
        model.set_decode_mode(mode)
        off = model.generate_from_pcm(pcm, **kw)
        l_off = model.last_trace.launches_decode
        on = model.generate_from_pcm(pcm, return_token_timestamps=True, **kw)
        l_on = model.last_trace.launches_decode
        on2 = model.generate_from_pcm(pcm, return_token_timestamps=True, **kw)
        assert l_on == l_off, mode
        assert torch.equal(on.sequences, off.sequences) and on.accept_lengths == off.accept_lengths
        assert torch.equal(on.token_logprobs, off.token_logprobs) and on.no_speech_prob == off.no_speech_prob
        assert all(torch.equal(a, b) for a, b in zip(on.scores, off.scores))
        assert torch.equal(on.token_timestamps, on2.token_timestamps)
        P = len(model._init_tokens(None, None))
        n = P + model.last_trace.n_new_tokens
        before = model.last_timestamp_matrix(P, n)
        model.forward(decoder_input_ids=torch.tensor([model._init_tokens(None, None)]))
        after = model.last_timestamp_matrix(P, n)
        assert all(torch.equal(a, b) for a, b in zip(before, after))
    model.set_decode_mode("persistent")
    # the engine reads back the pairs it captured with, whatever the config holds now
    heads = model.generation_config.alignment_heads
    model.generation_config.alignment_heads = heads[:1]
    try:
        assert model.last_alignment_probs(0, 2).shape[0] == len(heads)
    finally:
        model.generation_config.alignment_heads = heads
    # a batch with the feature extractor's masks: each row is cropped by its own mask, as its batch-1 run is
    feats = torch.zeros(2, 80, 3000)
    masks = torch.zeros(2, 3000, dtype=torch.long)
    singles = []
    for i, (sid, sec) in enumerate(((1, 7.0), (2, 4.0))):
        pcm_i = synthetic_audio(sec, stream_id=sid)
        model.generate_from_pcm(pcm_i, max_length=100)
        feats[i] = model.mel()
        masks[i, : model.pcm_num_frames(pcm_i.size)] = 1
        singles.append(model.generate(feats[i : i + 1], attention_mask=masks[i : i + 1], max_length=100,
                                      return_token_timestamps=True))
    assert (singles[1].token_timestamps <= (400 // 2 - 1) * 0.02 + 1e-6).all()   # 4 s = 400 frames: 200 columns
    group = StreamGroup(cfg, None, "cuda:0", n_streams=2, weights_from=model)
    try:
        outs = group.generate(feats, attention_mask=masks, max_length=100, return_token_timestamps=True)
    finally:
        group.close()
    for a, b in zip(outs, singles):
        assert torch.equal(a.sequences, b.sequences) and torch.equal(a.token_timestamps, b.token_timestamps)
