"""CPU tests of temperature fallback: the noise, the Gumbel-max top-k choice, HF's fallback quantities and the
per-window attempt loop of transcribe (on a fake engine)."""
import ctypes as C
import math
import types

import numpy as np
import pytest
import torch

from oracle import sampling_ref as SR
from whisper_medusa_b200 import WhisperMedusaModel
from whisper_medusa_b200.longform import Fallback, compression_ratio, fallback_rule, needs_fallback
from whisper_medusa_b200.synthetic import preset_config


def test_philox_known_answers():
    """Random123's published known-answer vectors of Philox4x32-10."""
    cases = [((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
             ((0xFFFFFFFF,) * 4, (0xFFFFFFFF, 0xFFFFFFFF), (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
             ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0),
              (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1))]
    for ctr, key, want in cases:
        assert SR.philox4x32_10(np.array(ctr, np.uint32), key).tolist() == list(want)


def test_noise_is_finite_and_keyed():
    g = SR.gumbel((123, 456), 3, 1, 17, np.arange(60000))
    assert g.dtype == np.float32 and np.isfinite(g).all()
    # the extreme words: u = 2^-25 and 1 - 2^-25
    u = (np.array([0, (1 << 24) - 1], np.float64) + 0.5) * 2.0 ** -24
    assert np.isfinite(-np.log(-np.log(u))).all()
    assert not np.array_equal(g[:100], SR.gumbel((123, 456), 3, 2, 17, np.arange(100)))
    assert not np.array_equal(g[:100], SR.gumbel((123, 456), 3, 1, 18, np.arange(100)))
    assert np.array_equal(g[40:50], SR.gumbel((123, 456), 3, 1, 17, np.arange(40, 50)))


def _chi2_ok(counts: np.ndarray, p: np.ndarray) -> bool:
    """Pearson's test over the cells with expectation >= 5 (the rest pooled), at the fixed bound of p = 1e-4."""
    from scipy.stats import chi2
    n = counts.sum()
    e = p * n
    big = e >= 5
    obs = np.append(counts[big], counts[~big].sum())
    exp = np.append(e[big], e[~big].sum())
    keep = exp > 0
    stat = float(((obs[keep] - exp[keep]) ** 2 / exp[keep]).sum())
    return stat < chi2.ppf(1 - 1e-4, max(1, int(keep.sum()) - 1))


@pytest.mark.parametrize("temperature", [0.2, 1.0])
@pytest.mark.parametrize("top_k", [50, 0, 1])
def test_gumbel_top_k_frequencies_match_softmax(temperature, top_k):
    rng = np.random.default_rng(7)
    V = 300
    row = (rng.standard_normal(V) * 1.5).astype(np.float32)
    row[5] = -np.inf                                    # a suppressed token
    n_draws = 6000
    counts = np.zeros(V, np.int64)
    for s in range(n_draws):
        idx, _ = SR.choose(row, temperature, top_k, SR.gumbel((s, 99), 0, 1, 4, np.arange(V)))
        counts[idx] += 1
    p = SR.exact_probs(row, temperature, top_k)
    assert counts[p == 0].sum() == 0
    assert _chi2_ok(counts, p)


def test_ties_at_the_kth_value_are_kept():
    row = np.array([3.0, 1.0, 2.0, 2.0, 2.0, 0.5], np.float32)   # k = 2: tau = 2.0, and all three 2.0 stay
    assert SR.top_k_tau(row, 2) == 2.0
    p = SR.exact_probs(row, 1.0, 2)
    assert (p[[0, 2, 3, 4]] > 0).all() and p[1] == 0 and p[5] == 0
    seen = set()
    for s in range(400):
        idx, tau = SR.choose(row, 1.0, 2, SR.gumbel((s, 0), 0, 1, 0, np.arange(6)))
        assert tau == 2.0
        seen.add(idx)
    assert seen == {0, 2, 3, 4}


def test_top_k_at_least_the_vocabulary_is_the_whole_row():
    rng = np.random.default_rng(3)
    row = rng.standard_normal(64).astype(np.float32)
    for s in range(50):
        g = SR.gumbel((s, 1), 2, 3, 9, np.arange(64))
        assert SR.choose(row, 0.6, 64, g) == SR.choose(row, 0.6, 0, g)
        assert SR.choose(row, 0.6, 1000, g) == SR.choose(row, 0.6, 0, g)
    assert fallback_rule((0.0, 0.2), 2.4, None, 70000, 51865).top_k == 0


def test_compression_ratio_and_avg_logprob_match_hf():
    from transformers.generation.logits_process import TemperatureLogitsWarper, TopKLogitsWarper
    from transformers.models.whisper.generation_whisper import WhisperGenerationMixin as HF

    rng = np.random.default_rng(11)
    for V in (51865, 51864, 300):
        ids = rng.integers(0, V, 80).tolist()
        ids = ids + ids[:40]
        assert compression_ratio(ids, V) == HF._retrieve_compression_ratio(torch.tensor(ids), V)
    # avg_logprob at T > 0: log_softmax of HF's warped scores times T = the row restricted to its top-k set at T = 1
    V, T, k = 300, 0.6, 50
    rows = torch.tensor(rng.standard_normal((6, V)).astype(np.float32))
    toks = torch.tensor([int(torch.argsort(r, descending=True)[i * 7]) for i, r in enumerate(rows)])   # in the top-k set
    warped = TopKLogitsWarper(k)(None, TemperatureLogitsWarper(T)(None, rows.clone()))
    hf = float(HF._retrieve_avg_logprobs(list(warped), toks, T))
    mine = []
    for r, t in zip(rows.numpy(), toks.tolist()):
        z = np.where(r >= SR.top_k_tau(r, k), r.astype(np.float64), -np.inf)
        mine.append(z[t] - (z.max() + np.log(np.exp(z - z.max()).sum())))
    assert abs(hf - float(np.mean(mine))) < 1e-5


def test_fallback_rule_arguments():
    V = 51865
    assert fallback_rule(None, None, None, None, V) is None
    assert fallback_rule(0.0, None, None, None, V) is None
    fb = fallback_rule((0.0, 0.2, 0.4), 2.4, -1.0, None, V)
    assert fb == Fallback((0.0, 0.2, 0.4), 2.4, -1.0, 50)
    assert fallback_rule([None, 0.5], None, -1.0, 0, V).temperatures == (0.0, 0.5)
    assert fallback_rule((0.0, 0.2), None, None, None, V) is None        # no threshold: the first entry only (HF)
    assert fallback_rule((0.0, 0.2), 2.4, None, None, V, default_top_k=20).top_k == 20
    with pytest.raises(NotImplementedError):
        fallback_rule((0.2, 0.4), 2.4, None, None, V)                   # sampling on the first attempt
    with pytest.raises(NotImplementedError):
        fallback_rule(None, 2.4, None, None, V)                         # a threshold with no schedule
    with pytest.raises(NotImplementedError):
        fallback_rule((0.0, 0.2), 2.4, None, 65, V)                     # above the engine's bound
    for bad in ((0.0, -0.2), (0.0, float("nan")), (0.0, float("inf")), ()):
        with pytest.raises(ValueError):
            fallback_rule(bad, 2.4, None, None, V)
    for bad in (float("nan"), "2.4", True):
        with pytest.raises(ValueError):
            fallback_rule((0.0, 0.2), bad, None, None, V)
    with pytest.raises(ValueError):
        fallback_rule((0.0, 0.2), 2.4, None, -1, V)
    fb = Fallback((0.0, 0.2), 2.4, -1.0, 50)
    assert needs_fallback(2.5, 0.0, fb) and needs_fallback(1.0, -1.5, fb) and not needs_fallback(2.4, -1.0, fb)


class _Engine:
    """A fake engine behind _decode: each attempt returns scripted (ids, avg_logprob, no_speech_prob)."""

    def __init__(self, m, script):
        self.m, self.script, self.calls = m, script, []

    def decode(self, language, task, kwargs, temperature, generation_config=None, return_dict_in_generate=None,
               token_timestamps=None, sampling=None):
        from whisper_medusa_b200.model import GenerateTrace, MedusaGenerateOutput
        a = sampling[5] if sampling is not None else 0
        self.calls.append((sampling, dict(kwargs)))
        ids, avg, nsp = self.script(a, sampling)
        eos = int(self.m.generation_config.eos_token_id)
        prompt = list(kwargs.get("decoder_input_ids") or self.m._init_tokens(language, task))
        tr = GenerateTrace()
        tr.sequences = prompt + ids + [eos]
        tr.n_new_tokens = len(ids) + 1
        self.m.last_trace = tr
        if not return_dict_in_generate:
            return torch.tensor([ids])
        out = MedusaGenerateOutput(torch.tensor([ids]), None, None, None, avg, [])
        out.no_speech_prob = nsp
        return out


def _fake(script, monkeypatch):
    monkeypatch.setattr(torch.cuda, "current_stream", lambda device=None: types.SimpleNamespace(cuda_stream=0))
    m = WhisperMedusaModel(preset_config("micro", heads=4), None)
    m._handle = C.c_void_p(1)
    m._encode_window = lambda x16, w, s: None
    m._upload_16k = lambda audio, sr: torch.zeros(int(np.asarray(audio).size))
    e = _Engine(m, script)
    m._decode = e.decode
    return m, e


_REPEAT = [7, 8] * 60        # compression ratio far above 2.4
_PLAIN = list(range(10, 50))


@pytest.mark.parametrize("case", ["pass_first", "pass_third", "keep_last", "skip"])
def test_attempt_loop(case, monkeypatch):
    script = {
        "pass_first": lambda a, s: (_PLAIN, -0.2, 0.0),
        "pass_third": lambda a, s: (_REPEAT if a < 2 else _PLAIN, -0.2, 0.0),
        "keep_last": lambda a, s: (_REPEAT + [a], -0.2, 0.0),
        "skip": lambda a, s: (_PLAIN, -2.0 if a == 1 else -1.5, 0.9 if a == 1 else 0.1),
    }[case]
    m, e = _fake(script, monkeypatch)
    try:
        torch.manual_seed(0)
        ns = dict(no_speech_threshold=0.6) if case == "skip" else {}
        m.transcribe(np.zeros(16000, np.float32), temperature=(0.0, 0.2, 0.4, 0.6),
                     compression_ratio_threshold=2.4, logprob_threshold=-1.0, **ns)
        w = m.last_windows[0]
        n = {"pass_first": 1, "pass_third": 3, "keep_last": 4, "skip": 2}[case]
        assert len(w.attempts) == n and len(e.calls) == n
        assert [a[0] for a in w.attempts] == [0.0, 0.2, 0.4, 0.6][:n]
        assert w.temperature == w.attempts[-1][0] and w.compression_ratio == w.attempts[-1][1]
        assert e.calls[0][0] is None                                   # the first attempt is the ordinary decode
        for a, (smp, kw) in enumerate(e.calls[1:], start=1):
            assert smp[0] == [0.0, 0.2, 0.4, 0.6][a] and smp[1] == 50 and smp[4] == 0 and smp[5] == a
            assert kw["medusa_temperature"] == 0.0
            assert kw["decoder_input_ids"] == e.calls[0][1]["decoder_input_ids"]   # attempt 0's prompt
        if case == "keep_last":
            assert w.ids == _REPEAT + [3]
        assert w.skipped is (True if case == "skip" else None)
    finally:
        m._handle = None


def test_seeds_follow_torch_and_do_not_depend_on_dispatch(monkeypatch):
    m, e = _fake(lambda a, s: (_REPEAT, -0.2, 0.0), monkeypatch)
    try:
        x = np.zeros(16000 * 50, np.float32)       # two windows
        kw = dict(temperature=(0.0, 0.5), compression_ratio_threshold=2.4)
        torch.manual_seed(5)
        m.transcribe(x, **kw)
        first = [c[0] for c in e.calls if c[0] is not None]
        assert [s[4] for s in first] == [0, 1] and len({s[2:4] for s in first}) == 1
        torch.manual_seed(5)
        want = tuple(int(v) for v in torch.randint(0, 2 ** 32, (2,), dtype=torch.int64))
        assert first[0][2:4] == want
        e.calls.clear()
        torch.manual_seed(5)
        m.transcribe(x, **kw)
        assert [c[0] for c in e.calls if c[0] is not None] == first
    finally:
        m._handle = None


def test_no_fallback_leaves_torch_rng_alone(monkeypatch):
    m, e = _fake(lambda a, s: (_REPEAT, -2.0, 0.0), monkeypatch)
    try:
        for kw in ({}, {"temperature": (0.0, 0.2)}, {"temperature": 0.0}):
            torch.manual_seed(1)
            m.transcribe(np.zeros(16000, np.float32), **kw)
            assert torch.rand(1).item() == (torch.manual_seed(1), torch.rand(1).item())[1]
        assert all(c[0] is None for c in e.calls)
    finally:
        m._handle = None


def test_refusals(monkeypatch):
    m, e = _fake(lambda a, s: (_PLAIN, -0.2, 0.0), monkeypatch)
    x = np.zeros(16000, np.float32)
    try:
        with pytest.raises(NotImplementedError):
            m.transcribe(x, temperature=0.4)
        with pytest.raises(NotImplementedError):
            m.transcribe(x, logprob_threshold=-1.0)
        with pytest.raises(NotImplementedError):
            m.transcribe(x, compression_ratio_threshold=2.4)
        with pytest.raises(NotImplementedError):
            m.transcribe(x, temperature=(0.2, 0.4), compression_ratio_threshold=2.4)
        with pytest.raises(NotImplementedError):
            m.transcribe(x, temperature=(0.0, 0.4), compression_ratio_threshold=2.4, top_k=100)
        with pytest.raises(NotImplementedError):
            m.transcribe(x, temperature=(0.0, 0.4), compression_ratio_threshold=2.4, top_p=0.9)
        with pytest.raises(ValueError):
            m.transcribe(x, temperature=(0.0, -0.4), compression_ratio_threshold=2.4)
        with pytest.raises(NotImplementedError):
            m.generate(torch.zeros(1, 80, 3000), temperature=(0.0, 0.2), compression_ratio_threshold=2.4)
        assert e.calls == []
        m.config.medusa_choices = [1, 2, 1, 1]
        with pytest.raises(NotImplementedError):
            m.transcribe(x, temperature=(0.0, 0.4), compression_ratio_threshold=2.4)
    finally:
        m._handle = None


def test_oracle_fallback_driver_matches_hf_rule():
    seqs = {0: _REPEAT, 1: _PLAIN}
    kept, skipped, att = SR.fallback(lambda a, t: (seqs.get(a, _PLAIN), -0.5, None), (0.0, 0.2, 0.4), 2.4, -1.0)
    assert kept == 1 and not skipped and len(att) == 2
    assert att[0][1] == compression_ratio(_REPEAT, 51865)
    kept, skipped, att = SR.fallback(lambda a, t: (_PLAIN, -2.0, None), (0.0, 0.2), None, -1.0, 0.6, 0.9)
    assert kept == 0 and skipped
    assert math.isclose(att[0][2], -2.0)


@pytest.mark.parametrize("heads,htype", [(1, "base_head"), (4, "base_head"), (10, "base_head"), (4, "medusa_block"),
                                         (10, "medusa_block")])
def test_sampled_loop_equals_one_token_decode(heads, htype):
    """The oracle's sampled speculative loop gives the tokens of a one-token-at-a-time Gumbel-max decode (suppression
    only, begin-suppress cleared: every position's row is then processed the same way in every iteration)."""
    from oracle import medusa_ref as M
    from oracle import whisper_ref as W
    from whisper_medusa_b200.synthetic import synthetic_audio, synthetic_state_dict

    cfg = preset_config("micro", heads=heads, heads_type=htype)
    w = W.RefWeights(synthetic_state_dict(cfg, seed=3))
    enc = W.encoder_forward(w, cfg, torch.from_numpy(W.log_mel_spectrogram(synthetic_audio(5.0))), "fp32")
    prompt = M.init_tokens(cfg)
    gp = M.gen_params(cfg, prompt, max_length=70, begin_suppress_tokens=None)
    accepted = 0
    for t, k in ((0.2, 50), (0.6, 0), (1.0, 50), (1.0, 1)):
        for s in range(4):
            tr = SR.sampled_search(w, cfg, enc, prompt, gp, t, k, (s, 17), 2, 1)
            n_new = len(tr.sequences) - len(prompt)
            one = SR.one_token_search(w, cfg, enc, prompt, gp, t, k, (s, 17), 2, 1, n_new)
            assert tr.sequences[:len(one)] == one, (t, k, s)
            assert len(tr.token_logprobs) >= len(one) - len(prompt)
            accepted += sum(tr.accept_lengths)
    if htype == "base_head":     # the verify rows' choices accepted candidates, not only accept-0 iterations
        assert accepted > 0


def test_top_k_and_one_entry_schedules(monkeypatch):
    """top_k is refused where nothing samples (as an unknown option was); a one-entry schedule with thresholds is HF's
    call that never falls back."""
    V = 51865
    for args in ((None, None, None), (0.0, None, None), ((0.0,), 2.4, None), ((0.0, 0.2), None, None)):
        with pytest.raises(NotImplementedError):
            fallback_rule(*args, 5, V)
    assert fallback_rule((0.0,), 2.4, -1.0, None, V) is None
    m, e = _fake(lambda a, s: (_REPEAT, -2.0, 0.0), monkeypatch)
    x = np.zeros(16000, np.float32)
    try:
        with pytest.raises(NotImplementedError):
            m.transcribe(x, top_k=5)
        m.transcribe(x, temperature=(0.0,), logprob_threshold=-1.0)
        m.transcribe(x, temperature=[0.0], compression_ratio_threshold=2.4, logprob_threshold=-1.0)
        assert [c[0] for c in e.calls] == [None, None]
    finally:
        m._handle = None


def test_eval_driver_passes_the_schedule(monkeypatch):
    from whisper_medusa_b200 import eval as E

    got = {}
    monkeypatch.setattr(E, "evaluate_model", lambda *a: got.setdefault("args", a))
    E.main(["--model-name", "m", "--data-path", "d", "--out-file-path", "o", "--chunk-length-s", "30",
            "--temperature", "0,0.2,0.4", "--compression-ratio-threshold", "2.4", "--logprob-threshold", "-1"])
    assert got["args"][-2:] == ([0.0, 0.2, 0.4], 2.4) and got["args"][-3] == -1.0
    monkeypatch.undo()
    with pytest.raises(ValueError):        # the schedule is a chunked-mode option
        E.evaluate_model("m", "d", "o", temperature=[0.0, 0.2], compression_ratio_threshold=2.4)
