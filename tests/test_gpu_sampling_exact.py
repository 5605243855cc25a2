"""Every sampled decision of temperature fallback, judged exactly against the engine's own raw rows.

A run with ``max_iters=i`` stops after iteration i, so ``last_logits(0)`` (the tail's rows) and ``last_logits(1)`` (the
verify rows) are iteration i's raw rows.  They are processed on the host (``oracle.processors_ref.process_logits`` with
the iteration's ids; the EOS decay factor as the fp32 the C ABI carries) and every decision is restated from them with
``oracle.sampling_ref.choose``.  The inputs are identical, so the expected answer is exact: no near-tie exemption and no
quota of runs that may differ.  For every iteration:

* c0 is the Gumbel-max choice of processed base row 0 at position L; head candidate h is the argmax of processed head
  row h (first maximum); verify row r < K chooses at position L + r + 1 (``last_accept()["row_argmax"]``, all K rows);
* the accept length is the number of leading candidates equal to their verify row's choice, the emitted tokens are
  those candidates plus, at accept 0, verify row 0's choice; each shorter run is a prefix of the longer one;
* the scores row equals the host-processed verify row ``accept`` bit for bit (-inf included), and each token
  log-probability is the fp64 ``log_softmax`` over the token row's top-k set ``{v >= tau}`` (all ties kept) within fp32
  rounding (1e-5 of the row's logit scale).

Scenarios: plain rows (K = 1, 4, 10, Linear and Block heads, T = 0.2 / 1.0 / 1.7, top_k = 1 / 2 / 50 / 63 / 64 / 0,
EOS decay on and off); exact ties at tau from ``sequence_bias={(j,): 2^20 or 2^24}`` (which quantizes every row to steps
of 1/8 or 2) -- each scenario asserts from the rows and the grid's segment count that it reached the path it is named for
(the segment rescan of ``smp_fold``, ties across segments, ties on the perturbed sum); rows with fewer than k finite
values and segments that are entirely -inf (``bad_words_ids``, ``min_length``, ``no_repeat_ngram_size``); every decoder
width at its real vocabulary; grids from 4 CTAs (one vocabulary segment) to the whole GPU (32 segments) in every decode
mode; the order of greedy, sampled and processor calls on one engine; a 40-token prompt (prefill launches) and a run to
max_length 448.
"""
import numpy as np
import pytest
import torch

from oracle import medusa_ref as M
from oracle import processors_ref as P
from oracle import sampling_ref as SR
from whisper_medusa_b200.synthetic import preset_config, synthetic_audio, synthetic_state_dict

pytestmark = pytest.mark.gpu

ALL_MODES = ("persistent", "persistent_simple", "graph")
WINDOW, ATTEMPT = 3, 2
DECAY = (5, 1.2)
_MODELS = {}


@pytest.fixture(scope="module", autouse=True)
def _close_engines():
    yield
    for m in _MODELS.values():
        m[0].close()
    _MODELS.clear()


def _model(cfg, seed=4):
    """One engine alive at a time, encoded once (the sampled calls decode from its encoder states)."""
    from whisper_medusa_b200 import WhisperMedusaModel

    key = (repr(cfg.to_dict()), seed)
    if key not in _MODELS:
        for m in _MODELS.values():
            m[0].close()
        _MODELS.clear()
        sd = synthetic_state_dict(cfg, seed=seed)
        model = WhisperMedusaModel(cfg, sd).to("cuda:0")
        _encode(model)
        _MODELS[key] = (model, sd)
    return _MODELS[key]


def _language(model):
    return "en" if model.config.is_multilingual else None


def _encode(model):
    model.generate_from_pcm(synthetic_audio(5.0, stream_id=3), max_length=20, language=_language(model))


def _micro(heads, htype="base_head"):
    return preset_config("micro", heads=heads, heads_type=htype)


def _preset(name, heads=4, htype="base_head"):
    return preset_config(name, heads=heads, heads_type=htype, decoder_layers=2, encoder_layers=2)


def _n_sm():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _nseg(n_cta, K):
    """Vocabulary segments per row of the logits scan, as the engine derives them from the decode grid."""
    return min(32, max(1, n_cta // (K + 1)))


def _set_grid(model, ctas):
    """``ctas`` CTAs (None: every SM), set explicitly; returns the grid's segment count."""
    n = _n_sm() if ctas is None else ctas
    model.set_option("decode_ctas", n)
    return _nseg(n, model.config.medusa_num_heads)


def _new(a):
    return a + 1 if a else 2


def _upto_eos(toks, eos):
    toks = list(toks)
    return toks[: toks.index(eos) + 1] if eos in toks else toks


def _gp(model, n_prompt, pen, procs):
    """The processors the engine applied (oracle GenParams).  The penalty factor crosses the C ABI as an fp32
    (``wm_gen_params.penalty_factor``), and the engine's EOS table is built from that value."""
    g = model.generation_config
    if pen is not None:
        pen = (int(pen[0]), float(np.float32(pen[1])))
    gp = M.GenParams(eos_token_id=int(g.eos_token_id), pad_token_id=int(g.pad_token_id),
                     suppress_tokens=list(g.suppress_tokens or []) or None,
                     begin_suppress_tokens=list(g.begin_suppress_tokens or []) or None, begin_index=n_prompt,
                     exponential_decay_length_penalty=pen, prompt_len=n_prompt)
    for key, v in procs.items():
        setattr(gp, key, list(v.items()) if key == "sequence_bias" else v)
    return gp


def _choose(row, t, k, seed, n):
    return SR.choose(row, t, k, SR.gumbel(seed, WINDOW, ATTEMPT, n, np.arange(len(row))))


def _paths(row, t, k, nseg, seed, n):
    """The selection paths a sampled row takes on a grid of ``nseg`` vocabulary segments."""
    V = len(row)
    seglen = -(-V // nseg)
    segs = [row[s * seglen:(s + 1) * seglen] for s in range(nseg)]
    fin = np.isfinite(row)
    hit = set()
    if any(not np.isfinite(s).any() for s in segs):
        hit.add("empty_segment")
    if k and fin.sum() < k:
        hit.add("fewer_than_k")
    tau = SR.top_k_tau(row, k)
    if np.isfinite(tau):
        if (row >= tau).sum() > k:
            hit.add("tie_at_tau")                      # the k-th value is tied beyond the k-th entry: all kept
            if len({int(j) // seglen for j in np.flatnonzero(row == tau)}) > 1:
                hit.add("tie_across_segments")
        # a segment's full list ends at tau and more entries equal to tau follow it: the fold rescans the segment
        if any((s >= tau).sum() > k for s in segs):
            hit.add("rescan")
    noise = SR.gumbel(seed, WINDOW, ATTEMPT, n, np.arange(V))
    s = np.where(row >= tau, (row / np.float32(t)).astype(np.float32) + noise, -np.inf).astype(np.float32)
    if (s == s.max()).sum() > 1:
        hit.add("sum_tie")
        if len({int(j) // seglen for j in np.flatnonzero(s == s.max())}) > 1:
            hit.add("sum_tie_across_segments")
    return hit


def _restricted_logprob(row, tau, tok):
    z = np.where(row >= tau, row.astype(np.float64), -np.inf)
    m = z.max()
    return float(z[tok] - (m + np.log(np.exp(z - m).sum())))


def _scale(row):
    return max(1.0, float(np.abs(row[np.isfinite(row)]).max()))


def _sampled(model, t, k, seed, kw, **extra):
    call = dict(kw, medusa_temperature=0.0, output_scores=True, **extra)
    return model._decode(_language(model), None, call, None, return_dict_in_generate=True,
                         sampling=(t, k, seed[0], seed[1], WINDOW, ATTEMPT))


def _check_runs(model, t, k, seed, n_iters, kw=None, procs=None, pen=None, nseg=None, hits=None, first=1):
    """Runs with max_iters = first .. n_iters; checks the last iteration of each exactly (module docstring).  Returns
    (the last run's sequences, the number of iterations checked)."""
    cfg = model.config
    K, V = cfg.medusa_num_heads, cfg.vocab_size
    kw = dict(kw or {})
    procs = dict(procs or {})
    nseg = nseg if nseg is not None else _nseg(_n_sm(), K)
    eos = int(model.generation_config.eos_token_id)
    prev, checked, ref_lp, scales = None, 0, [], []
    for i in range(first, n_iters + 1):
        out = _sampled(model, t, k, seed, dict(kw, exponential_decay_length_penalty=pen, **procs), max_iters=i)
        tr = model.last_trace
        if tr.iterations < i:           # the run had already ended (EOS or max_length)
            break
        ids, acc = tr.sequences, tr.accept_lengths
        n_prompt = len(ids) - sum(_new(a) for a in acc)
        L = len(ids) - _new(acc[-1])
        where = (seed, t, k, i, L)
        if prev is not None:
            assert len(prev) == L and ids[:L] == prev, where
        prev = list(ids)
        gp = _gp(model, n_prompt, pen, procs)
        A = P.process_logits(model.last_logits(0), L, gp, ids[:L]).numpy()
        B = P.process_logits(model.last_logits(1), L, gp, ids[:L]).numpy()
        tap = model.last_accept()
        cand, rarg = tap["cand"].tolist(), tap["row_argmax"].tolist()
        c0, tau0 = _choose(A[0], t, k, seed, L)
        assert cand[0] == c0, (where, cand[0], c0)
        for h in range(1, K + 1):
            assert cand[h] == int(np.argmax(A[h])), (where, h)
        ch = [_choose(B[r], t, k, seed, L + r + 1) for r in range(K)]
        assert rarg[:K] == [c for c, _ in ch], (where, rarg[:K], ch)
        accept = 0
        while accept < K and cand[accept + 1] == ch[accept][0]:
            accept += 1
        if accept < K:
            assert cand[accept + 1] != ch[accept][0]
        assert acc[-1] == accept, (where, acc[-1], accept)
        new = cand[: accept + 1] + ([ch[0][0]] if accept == 0 else [])
        assert _upto_eos(ids[L:], eos) == _upto_eos(new, eos), (where, ids[L:], new)
        if hits is not None:
            for row, n in [(A[0], L)] + [(B[r], L + r + 1) for r in range(K)]:
                for p in _paths(row, t, k, nseg, seed, n):
                    hits[p] = hits.get(p, 0) + 1
        # scores: the rows bit for bit, the token log-probabilities over the top-k set at fp32 rounding
        got_row = out.scores[-1][0].cpu().numpy()
        assert np.array_equal(got_row, B[accept]), (where, np.flatnonzero(got_row != B[accept])[:8])
        n_tok = len(_upto_eos(new, eos))
        lp = out.token_logprobs[0, L - n_prompt:].cpu().double().numpy()
        assert len(lp) == n_tok, (where, len(lp), n_tok)
        srcs = [(A[0], tau0)] + [(B[r], ch[r][1]) for r in range(K)]
        for j in range(n_tok):
            row, tau = srcs[j]
            ref = _restricted_logprob(row, tau, new[j])
            assert abs(float(lp[j]) - ref) <= 1e-5 * _scale(row), (where, j, float(lp[j]), ref)
        ref_lp.append([_restricted_logprob(*srcs[j], new[j]) for j in range(n_tok)])
        scales.append(max([_scale(srcs[j][0]) for j in range(n_tok)] + [1.0]))
        checked += 1
        if first == 1:     # every iteration of this run checked: its whole average
            flat = [v for it in ref_lp for v in it]
            assert abs(out.avg_logprob - float(np.mean(flat))) <= 1e-5 * max(scales), (where, out.avg_logprob)
    return prev, checked


def _check_seeds(model, t, k, kw=None, procs=None, pen=None, nseg=None, hits=None, min_iters=8, n_iters=10):
    """At least ``min_iters`` iterations checked exactly, over as many seeds as the runs' EOS stops need."""
    total, seqs = 0, []
    for s in range(6):
        seq, n = _check_runs(model, t, k, (17 + s, 4000 + s), n_iters, kw, procs, pen, nseg, hits)
        seqs.append(seq)
        total += n
        if total >= min_iters:
            break
    assert total >= min_iters, total
    return seqs


# ---------------------------------------------------------------------------------------------------- 1. plain rows
# (K, heads type, temperature, top_k, EOS decay)
PLAIN = [(1, "base_head", 0.2, 1, None), (1, "medusa_block", 1.7, 64, DECAY), (4, "base_head", 1.0, 2, DECAY),
         (4, "medusa_block", 0.2, 63, None), (10, "base_head", 1.7, 50, None), (10, "medusa_block", 1.0, 0, DECAY),
         (4, "base_head", 1.7, 0, None), (10, "base_head", 0.2, 64, DECAY), (4, "medusa_block", 1.0, 50, DECAY),
         (1, "base_head", 1.0, 0, DECAY)]


@pytest.mark.parametrize("K,htype,t,k,pen", PLAIN)
def test_plain_rows(K, htype, t, k, pen):
    model, _ = _model(_micro(K, htype))
    _set_grid(model, None)
    _check_seeds(model, t, k, dict(max_length=120), pen=pen)


# ---------------------------------------------------------------------------------------------------- 2. ties at tau
def _bias_all(V, b):
    return {(j,): float(b) for j in range(V)}


# (id, config, bias, temperature, top_k, decode_ctas (None: every SM), paths that must be reached)
TIES = [
    ("k50_one_segment", ("micro", 10, "medusa_block"), 2 ** 20, 1.0, 50, 4, {"tie_at_tau", "rescan"}),
    ("k64_one_segment", ("micro", 10, "base_head"), 2 ** 24, 0.2, 64, 4, {"tie_at_tau", "rescan", "sum_tie"}),
    ("k1_32_segments", ("micro", 1, "base_head"), 2 ** 24, 1.0, 1, None,
     {"tie_at_tau", "rescan", "tie_across_segments", "sum_tie"}),
    ("k64_tiny", ("tiny.en", 4, "base_head"), 2 ** 24, 0.2, 64, None,
     {"tie_at_tau", "tie_across_segments", "sum_tie_across_segments"}),
    ("k50_tiny", ("tiny.en", 1, "medusa_block"), 2 ** 20, 0.2, 50, None, {"tie_at_tau", "tie_across_segments"}),
    ("k1_tiny", ("tiny.en", 4, "base_head"), 2 ** 24, 0.2, 1, None, {"tie_at_tau", "tie_across_segments", "sum_tie"}),
]


def _cfg(spec):
    name, K, htype = spec
    return _micro(K, htype) if name == "micro" else _preset(name, K, htype)


@pytest.mark.parametrize("case", TIES, ids=[c[0] for c in TIES])
def test_ties_at_tau(case):
    _, spec, bias, t, k, ctas, need = case
    model, _ = _model(_cfg(spec))
    nseg = _set_grid(model, ctas)
    hits = {}
    try:
        _check_seeds(model, t, k, dict(max_length=120), dict(sequence_bias=_bias_all(model.config.vocab_size, bias)),
                     nseg=nseg, hits=hits, min_iters=6, n_iters=6)
    finally:
        _set_grid(model, None)
    assert need <= set(hits), (need - set(hits), hits)


# ---------------------------------------------------------------------------------------- 3. fewer than k finite values
def _allowed(cfg, m, seed=0):
    """EOS and m - 1 other ids spread over the lower half of the vocabulary (the upper segments are then all -inf)."""
    eos = int(cfg.eos_token_id)
    skip = set(cfg.suppress_tokens or []) | set(cfg.begin_suppress_tokens or []) | {eos}
    pool = [j for j in range(cfg.vocab_size // 2) if j not in skip]
    pick = np.random.default_rng(seed).choice(len(pool), m - 1, replace=False)
    return {eos} | {pool[int(i)] for i in pick}


# (id, K, top_k, |allowed|, further processors, paths that must be reached)
FEW = [("k_minus_1", 4, 50, 49, {}, {"fewer_than_k"}), ("k", 4, 50, 50, {}, {"fewer_than_k"}),
       ("k_plus_1", 4, 50, 51, {}, set()), ("twenty", 4, 50, 20, {}, {"fewer_than_k"}),
       ("min_length", 4, 50, 50, dict(min_length=119), {"fewer_than_k"}),
       ("no_repeat_ngram", 1, 20, 24, dict(no_repeat_ngram_size=1), {"fewer_than_k"})]


@pytest.mark.parametrize("case", FEW, ids=[c[0] for c in FEW])
def test_fewer_than_k_finite_values(case):
    _, K, k, m, extra, need = case
    model, _ = _model(_micro(K))
    cfg = model.config
    allowed = _allowed(cfg, m)
    procs = dict(bad_words_ids=[[j] for j in range(cfg.vocab_size) if j not in allowed], **extra)
    hits = {}
    for t in (0.2, 1.0):
        _check_seeds(model, t, k, dict(max_length=120), procs, nseg=_set_grid(model, None), hits=hits, min_iters=6,
                     n_iters=8)
    assert ({"empty_segment"} | need) <= set(hits), hits


# ---------------------------------------------------------------------------------------- 4. every width, real vocabulary
@pytest.mark.parametrize("name", ["tiny.en", "base", "small", "medium", "large-v2"])
def test_every_width(name):
    """Every sampled ring-kernel instantiation (each width; processors on and off; top-k and whole-row)."""
    model, _ = _model(_preset(name, 4))
    model.set_decode_mode("persistent")
    _set_grid(model, None)
    V = model.config.vocab_size
    _check_runs(model, 1.0, 50, (5, 6), 4, dict(max_length=120))
    _check_runs(model, 0.6, 0, (7, 8), 4, dict(max_length=120), pen=DECAY)
    hits = {}
    _check_runs(model, 0.2, 64, (9, 10), 4, dict(max_length=120), dict(sequence_bias=_bias_all(V, 2 ** 24)), hits=hits)
    _check_runs(model, 1.0, 0, (11, 12), 4, dict(max_length=120), dict(sequence_bias=_bias_all(V, 2 ** 20)), hits=hits)
    assert {"tie_at_tau", "sum_tie"} <= set(hits), hits


# ---------------------------------------------------------------------------------------------- 5. grids and modes
@pytest.mark.parametrize("K,htype", [(10, "medusa_block"), (3, "base_head")])
def test_every_grid_and_mode(K, htype):
    """The whole GPU, 33 CTAs and the smallest grid every mode accepts (ffn_dim / d_model CTAs: one segment at
    K = 10 and K = 3); K = 3 on the whole GPU has 32 segments.  Tokens are identical everywhere."""
    model, _ = _model(_micro(K, htype))
    cfg = model.config
    smallest = cfg.decoder_ffn_dim // cfg.d_model
    V = cfg.vocab_size
    runs = {}
    segs = set()
    try:
        for ctas in (None, 33, smallest):
            for mode in ALL_MODES:
                nseg = _set_grid(model, ctas)
                model.set_decode_mode(mode)
                segs.add(nseg)
                hits = {}
                for name, t, k, procs in (("ties", 1.0, 50, dict(sequence_bias=_bias_all(V, 2 ** 20))),
                                          ("plain", 0.2, 64, {})):
                    seq, n = _check_runs(model, t, k, (21, 22), 6, dict(max_length=120), procs, nseg=nseg, hits=hits)
                    assert n >= 4, (name, ctas, mode, n)
                    runs.setdefault(name, []).append(((ctas, mode), seq))
                if nseg == 1:
                    assert "rescan" in hits, (ctas, mode, hits)
    finally:
        model.set_decode_mode("persistent")
        _set_grid(model, None)
    assert 1 in segs and (K != 3 or 32 in segs), segs
    for name, got in runs.items():
        assert all(s == got[0][1] for _, s in got), (name, [(w, s) for w, s in got if s != got[0][1]])


# ---------------------------------------------------------------------------------------------------- 6. call order
def test_call_order_on_one_engine():
    """Greedy, sampled, sampled with processors, greedy with processors and greedy again on one engine: each call
    equals the same call on a fresh engine (cached sampled stage-kernel graphs, the host-chosen scores variant)."""
    from whisper_medusa_b200 import WhisperMedusaModel

    cfg = _micro(4)
    model, sd = _model(cfg)
    procs = dict(sequence_bias={(j,): 2.5 for j in range(0, 512, 7)}, bad_words_ids=[[j] for j in range(300, 420)])
    calls = [(None, {}), ((1.0, 50), {}), ((0.6, 2), procs), (None, procs), (None, {})]

    def run(m, smp, extra):
        kw = dict(max_length=80, output_scores=True, **extra)
        if smp is None:
            out = m._decode(None, None, kw, None, return_dict_in_generate=True)
        else:
            out = m._decode(None, None, dict(kw, medusa_temperature=0.0), None, return_dict_in_generate=True,
                            sampling=(smp[0], smp[1], 31, 32, WINDOW, ATTEMPT))
        return (m.last_trace.sequences, m.last_trace.accept_lengths, out.token_logprobs.cpu().tolist(),
                [r.cpu() for r in out.scores])

    try:
        for mode in ALL_MODES:
            model.set_decode_mode(mode)
            got = [run(model, smp, extra) for smp, extra in calls]
            for (smp, extra), g in zip(calls, got):
                fresh = WhisperMedusaModel(cfg, sd).to("cuda:0")
                try:
                    fresh.set_decode_mode(mode)
                    _encode(fresh)
                    want = run(fresh, smp, extra)
                finally:
                    fresh.close()
                assert g[:3] == want[:3], (mode, smp, bool(extra))
                assert all(torch.equal(a, b) for a, b in zip(g[3], want[3])), (mode, smp, bool(extra))
            assert got[0][0] == got[4][0]
    finally:
        model.set_decode_mode("persistent")


# -------------------------------------------------------------------------------------------- 7. long prompts, depth
def test_sampled_after_a_long_prompt():
    """A 40-token decoder_input_ids prompt (prefill launches of the stage kernel without sampling), then the first and
    second sampled iterations exactly, with and without processors."""
    model, _ = _model(_micro(4))
    cfg = model.config
    rng = np.random.default_rng(40)
    skip = set(cfg.suppress_tokens) | {int(cfg.eos_token_id)}
    prompt = [int(cfg.decoder_start_token_id)] + [int(j) for j in rng.choice(
        [j for j in range(cfg.vocab_size) if j not in skip], 39, replace=False)]
    kw = dict(max_length=120, decoder_input_ids=torch.tensor([prompt]))
    for mode in ALL_MODES:
        model.set_decode_mode(mode)
        for t, k, procs in ((1.0, 50, {}), (0.2, 64, dict(sequence_bias=_bias_all(cfg.vocab_size, 2 ** 20))),
                            (1.7, 0, dict(no_repeat_ngram_size=2))):
            seq, n = _check_runs(model, t, k, (41, 42), 2, kw, procs)
            assert n == 2 and seq[:40] == prompt, (mode, t, k)
    model.set_decode_mode("persistent")


def test_sampled_to_max_length():
    """A sampled run to max_length 448 (EOS suppressed): its last two iterations exactly (positions up to 447)."""
    model, _ = _model(_micro(4))
    g = model.generation_config
    saved = list(g.suppress_tokens or [])
    g.suppress_tokens = saved + [int(g.eos_token_id)]
    try:
        for t, k in ((1.0, 50), (0.6, 0)):
            _sampled(model, t, k, (51, 52), dict(max_length=448))
            n = model.last_trace.iterations
            assert len(model.last_trace.sequences) + 4 >= 448
            seq, checked = _check_runs(model, t, k, (51, 52), n, dict(max_length=448), first=n - 1)
            assert checked == 2 and len(seq) + 4 >= 448 and len(seq) > 440, (t, k, len(seq))
    finally:
        g.suppress_tokens = saved
