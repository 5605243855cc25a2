"""GPU tests of the sampled attempts of temperature fallback (csrc/decode.cu stage_select1_smp_rows / smp_fold) and of
transcribe(temperature=(0.0, ...), compression_ratio_threshold=..., logprob_threshold=...).

* wm_sample_noise is bit-equal to the numpy restatement (oracle/sampling_ref.py).
* The first sampled token equals the oracle's Gumbel-max choice on the engine's own processed base row, at T in
  {0.2, 0.6, 1.0} and top_k in {50, 0}; its frequencies over many seeds follow softmax(row / T) over the top-k set.
* top_k = 1 at any temperature and seed decodes exactly what medusa_temperature=0 decodes.
* Sampled tokens are the same in the three decode modes.
* transcribe: windows that pass at T = 0 are bit-identical to plain transcribe; a forced fallback runs every attempt,
  keeps the last, is reproducible under torch.manual_seed and equals StreamGroup.transcribe with S = 2 and 4.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import sampling_ref as SR
from whisper_medusa_b200.synthetic import synthetic_audio, synthetic_state_dict, width_config

pytestmark = pytest.mark.gpu

ALL_MODES = ("persistent", "graph", "persistent_simple")
_MODELS = {}


def _model(heads=4):
    from whisper_medusa_b200 import WhisperMedusaModel

    if heads not in _MODELS:
        for m in _MODELS.values():
            m[0].close()
        _MODELS.clear()
        cfg = width_config(384, heads=heads)
        sd = synthetic_state_dict(cfg, seed=7)
        _MODELS[heads] = (WhisperMedusaModel(cfg, sd).to("cuda:0"), sd, cfg)
    return _MODELS[heads]


def _encode(model, stream_id=1):
    model.generate_from_pcm(synthetic_audio(6.0, stream_id=stream_id), max_length=20)


def _sampled(model, t, k, seed=(11, 22), window=0, attempt=1, **kw):
    out = model._decode(None, None, dict(kw, medusa_temperature=0.0), None, return_dict_in_generate=True,
                        sampling=(t, k, seed[0], seed[1], window, attempt))
    return out


def test_noise_matches_numpy():
    from whisper_medusa_b200 import _lib

    model, _, _ = _model()
    lib = _lib.load()
    for seed, win, att, n, j0, cnt in [((0, 0), 0, 0, 0, 0, 4096), ((0xFFFFFFFF, 1), 7, 3, 447, 51000, 865),
                                       ((123456789, 987654321), 2, 5, 20, 3, 1001)]:
        out = np.zeros(cnt, np.float32)
        assert lib.wm_sample_noise(model._handle, seed[0], seed[1], win, att, n, j0, cnt,
                                   out.ctypes.data_as(C.POINTER(C.c_float))) == 0
        assert np.array_equal(out, SR.gumbel(seed, win, att, n, np.arange(j0, j0 + cnt)))


def _processed_base_row(model, n_prompt):
    """The processed base row of the first iteration (suppress and begin-suppress at L == begin_index)."""
    g = model.generation_config
    row = model.last_logits(0)[0].double().cpu().numpy().astype(np.float32)
    row[list(g.suppress_tokens or [])] = -np.inf
    if n_prompt == int(getattr(g, "begin_index", n_prompt) or n_prompt):
        row[list(g.begin_suppress_tokens or [])] = -np.inf
    return row


@pytest.mark.parametrize("t", [0.2, 0.6, 1.0])
@pytest.mark.parametrize("k", [50, 0])
def test_first_token_is_the_gumbel_max_choice(t, k):
    model, _, _ = _model()
    _encode(model)
    for s in range(6):
        out = _sampled(model, t, k, seed=(s, 3), max_iters=1)
        prompt = model._init_tokens(None, None)
        row = _processed_base_row(model, len(prompt))
        want, _ = SR.choose(row, t, k, SR.gumbel((s, 3), 0, 1, len(prompt), np.arange(len(row))))
        assert model.last_trace.sequences[len(prompt)] == want, (s, t, k)


def test_first_token_frequencies():
    from scipy.stats import chi2

    model, _, _ = _model()
    _encode(model)
    prompt = model._init_tokens(None, None)
    t, k = 1.0, 50
    counts = {}
    for s in range(1500):
        _sampled(model, t, k, seed=(s, 77), max_iters=1)
        tok = model.last_trace.sequences[len(prompt)]
        counts[tok] = counts.get(tok, 0) + 1
    row = _processed_base_row(model, len(prompt))
    p = SR.exact_probs(row, t, k)
    n = sum(counts.values())
    obs = np.array([counts.get(j, 0) for j in range(len(p))], np.float64)
    assert obs[p == 0].sum() == 0
    big = p * n >= 5
    o = np.append(obs[big], obs[~big].sum())
    e = np.append(p[big] * n, p[~big].sum() * n)
    keep = e > 0
    stat = float(((o[keep] - e[keep]) ** 2 / e[keep]).sum())
    assert stat < chi2.ppf(1 - 1e-4, int(keep.sum()) - 1), (stat, int(keep.sum()))


def test_top_k_one_is_greedy_in_every_mode():
    model, _, _ = _model()
    for mode in ALL_MODES:
        model.set_decode_mode(mode)
        _encode(model)
        greedy = model._decode(None, None, dict(medusa_temperature=0.0, max_length=60), None)[0].tolist()
        for t, s in ((0.2, 1), (1.0, 9)):
            out = _sampled(model, t, 1, seed=(s, s), max_length=60)
            assert out.sequences[0].tolist() == greedy, (mode, t)
    model.set_decode_mode("persistent")


@pytest.mark.parametrize("heads", [1, 4, 10])
def test_sampled_tokens_do_not_depend_on_the_decode_mode(heads):
    model, _, _ = _model(heads)
    got = {}
    for mode in ALL_MODES:
        model.set_decode_mode(mode)
        _encode(model)
        for t, k in ((0.6, 50), (1.0, 0)):
            out = _sampled(model, t, k, seed=(5, 6), max_length=60)
            got.setdefault((t, k), []).append((out.sequences[0].tolist(), float(out.avg_logprob)))
    model.set_decode_mode("persistent")
    for key, runs in got.items():
        assert all(r[0] == runs[0][0] for r in runs), key
        assert all(abs(r[1] - runs[0][1]) < 1e-4 for r in runs), key


def test_transcribe_with_a_schedule():
    from whisper_medusa_b200 import StreamGroup

    model, sd, cfg = _model()
    x = np.concatenate([synthetic_audio(12.0, stream_id=s) for s in (1, 2)]).astype(np.float32)
    kw = dict(chunk_length_s=10.0, max_length=60)
    sched = (0.0, 0.2, 0.6, 1.0)
    plain = model.transcribe(x, **kw)
    plain_ids = [r.ids for r in model.last_windows]
    # every window passes at T = 0: the plain result, one attempt each
    got = model.transcribe(x, temperature=sched, compression_ratio_threshold=1e9, logprob_threshold=-1e9, **kw)
    assert torch.equal(got, plain)
    assert [r.ids for r in model.last_windows] == plain_ids
    assert all(len(r.attempts) == 1 and r.temperature == 0.0 for r in model.last_windows)
    first = [r.attempts[0] for r in model.last_windows]
    # forced fallback: every attempt runs, the last is kept, the first is the plain decode's, and the encoder runs
    # once per window
    encodes = []
    encode = model._encode_window
    model._encode_window = lambda *a: encodes.append(a[1]) or encode(*a)
    torch.manual_seed(1234)
    forced = model.transcribe(x, temperature=sched, logprob_threshold=1e9, **kw)
    del model._encode_window
    wins = model.last_windows
    assert len(encodes) == len(wins)
    assert [(w.start, w.end) for w in encodes] == [(r.start, r.end) for r in wins]
    assert all([a[0] for a in r.attempts] == list(sched) and r.temperature == 1.0 for r in wins)
    assert [r.attempts[0] for r in wins] == first
    # a threshold between the attempts' values: each window keeps the attempt HF's driver keeps
    lpt = float(np.median([a[2] for r in wins for a in r.attempts]))
    torch.manual_seed(1234)
    model.transcribe(x, temperature=sched, logprob_threshold=lpt, **kw)
    for r, f in zip(model.last_windows, wins):
        kept, skipped, att = SR.fallback(lambda a, t: (None, f.attempts[a][2], f.attempts[a][1]), sched, None, lpt)
        assert r.attempts == f.attempts[:len(att)] and r.temperature == sched[kept] and not skipped
        assert r.avg_logprob == f.attempts[kept][2]
    torch.manual_seed(1234)
    again = model.transcribe(x, temperature=sched, logprob_threshold=1e9, **kw)
    assert torch.equal(again, forced)
    assert [r.attempts for r in model.last_windows] == [r.attempts for r in wins]
    # the combination with the no-speech rule and with token timestamps runs the same attempts
    model.generation_config.alignment_heads = [[0, 0], [1, 3]]
    torch.manual_seed(1234)
    ts = model.transcribe(x, temperature=sched, logprob_threshold=1e9, no_speech_threshold=1.0,
                          return_token_timestamps=True, **kw)
    assert [r.ids for r in model.last_windows] == [r.ids for r in wins]
    assert ts.token_timestamps.shape[1] == ts.sequences.shape[1]
    model.close()
    _MODELS.clear()
    for S in (2, 4):
        group = StreamGroup(cfg, sd, "cuda:0", n_streams=S)
        try:
            torch.manual_seed(1234)
            out = group.transcribe([x, x[: 16000 * 9]], temperature=sched, logprob_threshold=1e9, **kw)
            assert torch.equal(out[0].cpu(), forced.cpu()), S
            # same attempts and ratios; avg_logprob to the last bits of the rows a partial grid computes
            for r, w in zip(group.last_windows[0], wins):
                assert [a[:2] for a in r.attempts] == [a[:2] for a in w.attempts], S
                assert all(abs(a[2] - b[2]) < 1e-4 for a, b in zip(r.attempts, w.attempts)), S
        finally:
            group.close()


# (preset, heads, heads type, temperature, top_k, EOS decay): chains of 1, 4 and 10 heads, Linear and Block heads
PARITY = [("micro", 1, "base_head", 0.2, 50, None), ("micro", 4, "base_head", 0.6, 0, None),
          ("micro", 10, "medusa_block", 1.0, 50, None), ("micro", 4, "medusa_block", 0.2, 0, (5, 1.2)),
          ("tiny.en", 4, "base_head", 1.0, 50, (5, 1.2)), ("tiny.en", 10, "base_head", 0.6, 50, None)]


@pytest.mark.parametrize("preset,heads,htype,t,k,decay", PARITY)
def test_sampled_loop_matches_the_oracle(preset, heads, htype, t, k, decay):
    """Engine tokens and top-k-restricted token log-probabilities of sampled attempts against the oracle's sampled loop
    (engine regime, from the engine's own encoder states), on the whole GPU and on a partial grid.  A run may diverge
    only where the oracle met a near-tie (a choice margin below 2e-3 of the logit scale: the engine's rows are within
    DECODE_LOGIT_BAR of the oracle's); most runs must match in full."""
    from _decode_ref import DECODE_LOGIT_BAR
    from oracle import medusa_ref as M
    from oracle import whisper_ref as W
    from whisper_medusa_b200 import WhisperMedusaModel
    from whisper_medusa_b200.synthetic import preset_config

    for m in _MODELS.values():
        m[0].close()
    _MODELS.clear()
    cfg = preset_config(preset, heads=heads, heads_type=htype)
    sd = synthetic_state_dict(cfg, seed=4)
    model = WhisperMedusaModel(cfg, sd).to("cuda:0")
    try:
        model.generate_from_pcm(synthetic_audio(5.0, stream_id=3), max_length=20)
        enc = model.encoder_output()
        w = W.RefWeights(sd)
        prompt = M.init_tokens(cfg)
        max_length = 72
        gp = M.gen_params(cfg, prompt, decay, max_length)
        full = 0
        runs = 0
        for ctas in (None, 33):
            if ctas:
                model.set_option("decode_ctas", ctas)
            for s in range(4):
                seed = (s, 1000 + s)
                ref = SR.sampled_search(w, cfg, enc, prompt, gp, t, k, seed, 0, 1, regime="engine")
                out = _sampled(model, t, k, seed=seed, max_length=max_length, exponential_decay_length_penalty=decay)
                got = model.last_trace.sequences
                runs += 1
                if got == ref.sequences:
                    full += 1
                    n = model.last_trace.n_new_tokens
                    lp = out.token_logprobs[0, :n].cpu().double().numpy()
                    err = max(abs(float(lp[j]) - ref.token_logprobs[j]) / ref.token_scales[j] for j in range(n))
                    assert err <= 2 * DECODE_LOGIT_BAR, (seed, ctas, err)
                else:
                    assert ref.min_gap < 2e-3 * max(ref.token_scales), (seed, ctas, got, ref.sequences)
        assert full >= runs * 3 // 4, (full, runs)
    finally:
        model.close()
