"""GPU tests of token timestamps in long-form transcription (transcribe(return_token_timestamps=True)).

* Windows: every window's token times are bit-identical to generate_from_pcm(window samples, return_token_timestamps=
  True), cropped to the window's own frame count (the short last window included); its ids, accept lengths and decode
  launch count are those of the same transcription without timestamps; a plain transcribe returns what it returned.
* The returned object is the package's host functions (longform.merge_timed, pinned to transformers by
  test_longform_timestamps_host.py) applied to last_windows.
* Each window's times against HF's extraction of the fp64 oracle's teacher-forced rows (oracle/timestamps_ref.py) on the
  engine's ids and encoder states: the count of differing times is printed and held to the short-form test's bar.
* At 48 kHz with the no-speech rule on and language=None (a multilingual vocabulary on a small model, so every window
  detects its language through forward()): skipped windows keep their times and add nothing; StreamGroup.transcribe with
  S = 1, 2 and 4 equals model.transcribe, ids, times and per-window times.
"""
import numpy as np
import pytest
import torch

from oracle import resample_ref as R
from oracle import timestamps_ref as TS
from oracle import whisper_ref as W
from whisper_medusa_b200.longform import merge_timed, merge_windows, skip_window, text_ids
from whisper_medusa_b200.synthetic import synthetic_audio, synthetic_state_dict, width_config

pytestmark = pytest.mark.gpu

_MODELS = {}


def _model(d, K, seed, profile="default"):
    """One engine alive at a time; alignment heads: every head of the last decoder layer and one of the first."""
    from whisper_medusa_b200 import WhisperMedusaModel

    key = (d, K, seed, profile)
    if key not in _MODELS:
        for m in _MODELS.values():
            m[0].close()
        _MODELS.clear()
        cfg = width_config(d, heads=K)
        sd = synthetic_state_dict(cfg, seed=seed, activation_profile=profile)
        m = WhisperMedusaModel(cfg, sd).to("cuda:0")
        H = cfg.decoder_attention_heads
        m.generation_config.alignment_heads = [[cfg.decoder_layers - 1, h] for h in range(H)] + [[0, H - 1]]
        _MODELS[key] = (m, sd)
    return _MODELS[key]


def _recording(seconds, first_stream=0):
    parts, left, k = [], float(seconds), first_stream
    while left > 0:
        s = min(25.0, left)
        parts.append(synthetic_audio(s, stream_id=k))
        left -= s
        k += 1
    return np.concatenate(parts).astype(np.float32)


def _window_state(r):
    return r.ids, r.trace.accept_lengths, r.trace.launches_decode


def _check_output(model, out):
    ids, pairs = merge_timed(model.last_windows, int(model.generation_config.eos_token_id))
    assert out.keys() == ["sequences", "token_timestamps"]
    assert out.sequences.tolist() == [ids]
    assert torch.equal(out.token_timestamps.cpu(), torch.tensor(pairs, dtype=torch.float32).reshape(1, -1, 2))


CASES = [(384, 4, 21, "default"), (768, 10, 22, "gamma_spread"), (1280, 10, 3, "default")]


@pytest.mark.parametrize("case", CASES, ids=[f"d{c[0]}_k{c[1]}" for c in CASES])
def test_windows_equal_short_clips_and_the_oracle(case):
    d, K, seed, profile = case
    model, sd = _model(d, K, seed, profile)
    cfg = model.config
    eos = int(model.generation_config.eos_token_id)
    x = _recording(62.5, first_stream=d % 11)            # windows 0-30, 20-50, 40-62.5 s: the last one is short
    kw = dict(max_length=120)
    plain = model.transcribe(x, **kw)
    plain_wins = [_window_state(r) for r in model.last_windows]
    assert all(r.token_timestamps is None and r.num_frames is None for r in model.last_windows)
    out = model.transcribe(x, return_token_timestamps=True, **kw)
    wins = model.last_windows
    assert len(wins) == 3 and wins[-1].end - wins[-1].start == 22.5 * 16000
    assert [_window_state(r) for r in wins] == plain_wins
    _check_output(model, out)
    assert merge_windows([text_ids(r.ids, eos) for r in wins]) == plain[0].tolist()
    assert torch.equal(model.transcribe(x, **kw), plain)
    assert [_window_state(r) for r in model.last_windows] == plain_wins
    # every window against its short clip, and against the fp64 oracle's alignment of the engine's ids
    ref_w = W.RefWeights(sd, torch.float64)
    n_diff, n_all = 0, 0
    P = len(model._init_tokens(None, None))
    for r in wins:
        nf = model.pcm_num_frames(r.end - r.start)
        assert r.num_frames == nf
        clip = model.generate_from_pcm(x[r.start:r.end], return_token_timestamps=True, **kw)
        assert clip.sequences[0].tolist() == r.ids
        assert torch.equal(clip.token_timestamps, r.token_timestamps), r
        tr = model.last_trace
        n = P + tr.n_new_tokens
        ts, _, _ = model.last_timestamp_matrix(P, n, nf)
        assert torch.equal(ts[P : P + len(r.ids)], r.token_timestamps[0].cpu())
        ref = TS.alignment_probs(ref_w, cfg, tr.sequences[: n - 1], model.encoder_output().double(),
                                 model.generation_config.alignment_heads, regime="engine")
        ref_ts, _, _ = TS.extract(ref[:, P:].float(), P, nf, 7, 0.02)
        n_diff += int((ts.numpy() != ref_ts).sum())
        n_all += n - P
        assert float(np.abs(ts.numpy() - ref_ts).max()) <= 0.1, (r, ts, ref_ts)
        assert float(ts.max()) <= (nf // 2) * 0.02 + 1e-6          # cropped to the window's frames
    print(f"d{d}: {n_diff} of {n_all} window token times differ from the fp64 oracle's")
    assert n_diff <= max(2, n_all // 20), (n_diff, n_all)


def _multilingual(model):
    """The micro vocabulary's free ids above <|notimestamps|> as language and task tokens: language=None then detects
    each window's language with one forward() on <|startoftranscript|>."""
    g = model.generation_config
    g.is_multilingual = True
    g.lang_to_id = {"<|en|>": 503, "<|de|>": 504, "<|fr|>": 506, "<|es|>": 508}
    g.task_to_id = {"transcribe": 505, "translate": 507}


def _speech_and_silence():
    parts = [synthetic_audio(6.0, stream_id=1), np.zeros(14 * 16000, np.float32), synthetic_audio(7.0, stream_id=2),
             np.zeros(12 * 16000, np.float32), synthetic_audio(5.3, stream_id=5)]
    return np.concatenate(parts).astype(np.float32)


def test_48k_no_speech_language_detection_and_stream_groups():
    from whisper_medusa_b200 import StreamGroup

    model, sd = _model(512, 4, 7, "default")
    _multilingual(model)
    cfg = model.config
    x16 = _speech_and_silence()
    x48 = R.resample(x16, 16000, 48000).astype(np.float32)
    kw = dict(sampling_rate=48000, chunk_length_s=10.0, max_length=80, language=None)
    base = model.transcribe(x48, **kw)
    base_wins = [_window_state(r) for r in model.last_windows]
    langs = {r.trace.sequences[1] for r in model.last_windows}
    assert langs <= {503, 504, 506, 508}
    last = model.last_windows[-1]
    assert last.end - last.start < model.last_windows[0].end - model.last_windows[0].start
    # thresholds between the windows' measured no-speech probabilities
    model.transcribe(x48, no_speech_threshold=1.0, logprob_threshold=-1e9, **kw)
    ps = sorted(set(r.no_speech_prob for r in model.last_windows))
    assert len(ps) >= 2, ps
    nst, lpt = (ps[len(ps) // 2 - 1] + ps[len(ps) // 2]) / 2, 1.0
    ns = dict(no_speech_threshold=nst, logprob_threshold=lpt)
    untimed = model.transcribe(x48, **ns, **kw)
    untimed_wins = [_window_state(r) for r in model.last_windows]
    skipped = [r.skipped for r in model.last_windows]
    assert any(skipped) and not all(skipped)
    out = model.transcribe(x48, return_token_timestamps=True, **ns, **kw)
    wins = model.last_windows
    assert [r.skipped for r in wins] == skipped
    assert [r.skipped for r in wins] == [skip_window(r.no_speech_prob, r.avg_logprob, nst, lpt) for r in wins]
    # the rule adds its own launches; timestamps add none
    assert [_window_state(r) for r in wins] == untimed_wins
    assert [s[:2] for s in untimed_wins] == [s[:2] for s in base_wins]
    assert all(r.token_timestamps is not None and r.token_timestamps.shape == (1, len(r.ids)) for r in wins)
    _check_output(model, out)
    eos = int(model.generation_config.eos_token_id)
    kept = [[] if r.skipped else text_ids(r.ids, eos) for r in wins]
    assert untimed[0].tolist() == merge_windows(kept)
    # each window (16 kHz samples after the GPU resampler) against its short clip, language detected the same way
    x16_dev = model._upload_16k(torch.from_numpy(x48).to("cuda:0"), 48000)
    for r in wins:
        clip = model.generate_from_pcm(x16_dev[r.start:r.end].cpu().numpy(), return_token_timestamps=True,
                                       max_length=80, language=None)
        assert clip.sequences[0].tolist() == r.ids
        assert torch.equal(clip.token_timestamps, r.token_timestamps), r
    assert torch.equal(model.transcribe(x48, **kw), base)
    # StreamGroup: the shared queue gives each recording what model.transcribe gives it
    recs, rates = [x48, _recording(47.0, first_stream=3)], [48000, 16000]
    want = []
    for x, sr in zip(recs, rates):
        o = model.transcribe(x, return_token_timestamps=True, **ns, **dict(kw, sampling_rate=sr))
        want.append((o, [(r.ids, r.token_timestamps, r.num_frames) for r in model.last_windows]))
    for S in (1, 2, 4):
        group = StreamGroup(cfg, None, "cuda:0", n_streams=S, weights_from=model)
        try:
            got = group.transcribe(recs, sampling_rate=rates, return_token_timestamps=True, **ns,
                                   **{k: v for k, v in kw.items() if k != "sampling_rate"})
            for g, ws, (o, o_ws) in zip(got, group.last_windows, want):
                assert torch.equal(g.sequences, o.sequences) and torch.equal(g.token_timestamps, o.token_timestamps), S
                assert len(ws) == len(o_ws)
                for r, (ids, ts, nf) in zip(ws, o_ws):
                    assert r.ids == ids and torch.equal(r.token_timestamps, ts) and r.num_frames == nf, S
        finally:
            group.close()
