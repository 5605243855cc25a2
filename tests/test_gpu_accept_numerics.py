"""GPU tests of the logits scan, candidate selection and typical acceptance against the host reference
(tests/_accept_ref.py) on the engine's own logits.

A run with ``max_iters=i`` stops after iteration i, so the accept-step tap (``last_accept()``, ``wm_last_accept``) and
the raw-logits tap (``last_logits``) hold iteration i; its tokens and accept lengths must be a prefix of the full run's.
On every checked iteration:

* ``cand`` (every node's token) and ``row_argmax`` (every verify row) are bit-equal to the fp32 replica of the scan,
  with the engine's tie rules (first index; top-k by value descending, index ascending);
* ``|row_pc - ref| <= PC_BAR * max(ref_pc, ref_thr)`` (relative to the decision; a hopeless candidate may underflow in
  fp32) and ``|row_thr - ref| <= THR_BAR * ref_thr``, with fp64 references;
* the accept length, the best path's node ``path_node`` (trees) and the emitted tokens equal the host decision on the
  engine's rows.  The only allowed exception is an iteration where a compared candidate probability lies within
  ``NEAR * max(PC_BAR, THR_BAR)`` of its threshold (relative); such iterations are counted and must stay rare.  At temperature 0 there is none.

Groups (DESIGN.md section 2, "Candidates and acceptance against fp64"): A chains under temperature, both branches of
the threshold's min, begin-suppress and a length penalty that makes EOS a candidate; B vocabulary segment geometry
(partial grids, an empty last segment at V = 513, V = 51866, large-v2 in the benchmark regime); C branching trees under
both attention rules; D exact ties from twin embedding rows; E flat and peaked posteriors.

``WM_NUMERICS_RECORD=<file>`` records the worst errors per case instead of asserting the bars (tests/_decode_ref.py).
"""
import numpy as np
import pytest
import torch

import _accept_ref as A
from _decode_ref import check_error
from test_gpu_scores import _host_gp, _load
from whisper_medusa_b200.synthetic import preset_config, synthetic_audio, synthetic_state_dict, width_config

pytestmark = pytest.mark.gpu

#: |row_pc - ref| / max(ref_pc, ref_thr) and |row_thr - ref| / ref_thr: about 3x the worst values measured on an H100
#: over every case of this file, 5.4e-7 and 4.0e-6 (DESIGN.md section 2)
PC_BAR = 1.5e-6
THR_BAR = 1.2e-5
#: decisions may differ from the host's only where |pc - thr| <= NEAR * max(PC_BAR, THR_BAR) * thr
NEAR = 10.0

_MODELS = {}


def _model(cfg, seed, twins=None, **sd_kw):
    """One engine alive at a time.  ``twins = (src, dst, n)``: embedding rows dst..dst+n copy rows src..src+n (proj_out is
    tied), so their logits are exact ties."""
    from whisper_medusa_b200 import WhisperMedusaModel

    key = (repr(cfg.to_dict()), seed, twins, tuple(sorted(sd_kw.items())))
    if key not in _MODELS:
        for m in _MODELS.values():
            m.close()
        _MODELS.clear()
        sd = synthetic_state_dict(cfg, seed=seed, **sd_kw)
        if twins:
            src, dst, n = twins
            e = sd["whisper_model.model.decoder.embed_tokens.weight"].clone()
            e[dst: dst + n] = e[src: src + n]
            sd["whisper_model.model.decoder.embed_tokens.weight"] = e
            sd["whisper_model.proj_out.weight"] = e
        _MODELS[key] = WhisperMedusaModel(cfg, sd).to("cuda:0")
    return _MODELS[key]


def _new_tokens(a):
    return a + 1 if a else 2


def _eos_fill(toks, eos):
    if eos in toks:
        j = toks.index(eos)
        return toks[: j + 1] + [eos] * (len(toks) - j - 1)
    return list(toks)


class Stats:
    def __init__(self):
        self.iters = self.typical = self.near = self.ties = 0
        self.pc = self.thr = 0.0


def _check_iteration(model, pcm, kw, i, full, st, twins=None):
    """Run to iteration i and hold its scan and accept step to the host reference."""
    cfg = model.config
    model.generate_from_pcm(pcm, max_iters=i, **kw)
    tr = model.last_trace
    assert tr.iterations == i and tr.accept_lengths == full.accept_lengths[:i]
    a = tr.accept_lengths[-1]
    L = len(tr.sequences) - _new_tokens(a)
    n_prompt = len(tr.sequences) - sum(_new_tokens(x) for x in tr.accept_lengths)
    assert tr.sequences == full.sequences[: len(tr.sequences)]
    tap = model.last_accept()
    raw_a, raw_b = model.last_logits(0).numpy(), model.last_logits(2).numpy()
    if twins:
        src, dst, n = twins
        assert np.array_equal(raw_a[:, src: src + n], raw_a[:, dst: dst + n]), "twin logits differ (pass A)"
        assert np.array_equal(raw_b[:, src: src + n], raw_b[:, dst: dst + n]), "twin logits differ (verify)"
    gp = _host_gp(model, n_prompt, kw.get("exponential_decay_length_penalty"))
    T = A.f32(kw.get("medusa_temperature", 1.0))
    thr = A.f32(kw.get("posterior_threshold", model.generation_config.posterior_threshold))
    alpha = A.f32(kw.get("posterior_alpha", model.generation_config.posterior_alpha))
    tree = A.tree_tables(cfg.medusa_choices)
    rows_a, rows_b = A.process_rows(raw_a, L, gp), A.process_rows(raw_b, L, gp)
    ref = A.decide(rows_a, rows_b, tree, T, thr, alpha)
    where = (i, L)
    assert tap["cand"].tolist() == ref.cand.tolist(), where
    assert tap["row_argmax"].tolist() == ref.row_argmax.tolist(), where
    if twins:   # rows whose maximum is an exact tie
        st.ties += sum(int(np.sum(r == r.max()) > 1) for r in np.concatenate([rows_a, rows_b]) if np.isfinite(r.max()))
    st.iters += 1
    near = []
    if T != 0.0:
        assert tap["row_pc"] is not None
        pc, thr_e = tap["row_pc"].double().numpy(), tap["row_thr"].double().numpy()
        for child, parent in ref.edges:
            scale = max(ref.row_pc[child], ref.row_thr[parent])
            st.pc = max(st.pc, abs(pc[child] - ref.row_pc[child]) / scale)
        for r in ref.stat_rows:
            st.thr = max(st.thr, abs(thr_e[r] - ref.row_thr[r]) / ref.row_thr[r])
        near = A.margin_rows(ref, NEAR * max(PC_BAR, THR_BAR))
        st.typical += 1
    else:
        assert tap["row_pc"] is None and tap["row_thr"] is None
    got_path = None if tree.chain else tap["path_node"]
    got_toks = tr.sequences[L:]
    same = (a == ref.accept and got_toks == _eos_fill(ref.new_tokens, gp.eos_token_id)
            and (got_path is None or got_path == ref.path_node))
    if not same:
        assert near, ("decision differs away from the threshold", where, a, ref.accept, got_toks, ref.new_tokens,
                      got_path, ref.path_node)
        st.near += 1


def _run(name, model, pcm, kw, iters=None, twins=None):
    """Full run, then iterations ``iters`` (default: every one) checked; returns the stats."""
    model.generate_from_pcm(pcm, **kw)
    full = model.last_trace
    n = full.iterations
    its = range(1, n + 1) if iters is None else sorted({min(max(1, i if i > 0 else n + i + 1), n) for i in iters})
    st = Stats()
    for i in its:
        _check_iteration(model, pcm, kw, i, full, st, twins)
    if st.typical:
        check_error(st.pc, PC_BAR, name, "row_pc")
        check_error(st.thr, THR_BAR, name, "row_thr")
    # decisions that differ at the threshold are rare: at most one in 20 typical iterations, none at temperature 0
    assert st.near <= max(1, st.typical // 20), (name, st.near, st.typical)
    print(f"{name}: {st.iters} iterations, pc {st.pc:.2e}, thr {st.thr:.2e}, near-threshold {st.near}, tie rows {st.ties}")
    return st


def _kw(T, thr_alpha, pen=(10, 1.15), max_length=100):
    return dict(max_length=max_length, medusa_temperature=T, posterior_threshold=thr_alpha[0],
                posterior_alpha=thr_alpha[1], exponential_decay_length_penalty=pen)


PAIRS = [(0.09, 0.3), (0.09, 100.0), (0.01, 100.0)]
TEMPS = [0.0, 0.5, 1.0, 2.0]


# ------------------------------------------------------------------------------------------------ A: chains
@pytest.mark.parametrize("K", [1, 3, 4, 10, 15])
def test_a_chains_micro(K):
    """d = 128 (V = 512): every iteration, every temperature and threshold / alpha pair; the length penalty makes EOS a
    candidate, iteration 1 runs under begin-suppress."""
    model = _model(width_config(128, heads=K), 3)
    pcm = synthetic_audio(5.0, stream_id=K)
    for T in TEMPS:
        for pair in PAIRS:
            _run(f"A/micro/K{K}/T{T}/{pair}", model, pcm, _kw(T, pair))


@pytest.mark.parametrize("K", [1, 4, 15])
def test_a_chains_tiny(K):
    """tiny.en (V = 51864): iterations 1, 2, n/2 and n."""
    model = _model(preset_config("tiny.en", heads=K), 4)
    pcm = synthetic_audio(5.0, stream_id=10 + K)
    for T in TEMPS:
        for pair in PAIRS:
            kw = _kw(T, pair, max_length=120)
            model.generate_from_pcm(pcm, **kw)
            n = model.last_trace.iterations
            _run(f"A/tiny/K{K}/T{T}/{pair}", model, pcm, kw, iters=[1, 2, n // 2, n])


# ------------------------------------------------------------------------------------------------ B: segment geometry
@pytest.mark.parametrize("K", [3, 15])
@pytest.mark.parametrize("ctas", [0, 37, 8])
def test_b_partial_grids(K, ctas):
    """Vocabulary segments per row: clamp(n_cta / (K+1), 1, 32) -- 32 / 9 / 2 at K = 3, 8 / 2 / 1 at K = 15."""
    model = _model(width_config(128, heads=K), 5)
    pcm = synthetic_audio(5.0, stream_id=20 + K)
    if ctas:
        model.set_option("decode_ctas", ctas)
    try:
        for T in (0.0, 0.5, 1.0):
            _run(f"B/ctas{ctas or 'full'}/K{K}/T{T}", model, pcm, _kw(T, PAIRS[0]))
    finally:
        model.close()
        _MODELS.clear()


@pytest.mark.parametrize("V,K", [(513, 1), (513, 3), (51866, 4)])
def test_b_vocabulary_sizes(V, K):
    """V = 513 on the full grid: 32 segments of 17, the last one empty; V = 51866 (large-v3's vocabulary) at d = 128 on
    the full grid and on 8 CTAs."""
    cfg = width_config(128, heads=K)
    cfg.vocab_size = V
    model = _model(cfg, 6)
    pcm = synthetic_audio(5.0, stream_id=30 + K)
    for T in (0.0, 0.5, 1.0, 2.0):
        _run(f"B/V{V}/K{K}/T{T}", model, pcm, _kw(T, PAIRS[0]), iters=None if V < 1000 else [1, 2, 3, -1])
    if V > 1000:
        model.set_option("decode_ctas", 8)
        try:
            _run(f"B/V{V}/K{K}/ctas8", model, pcm, _kw(1.0, PAIRS[0]), iters=[1, 2, 3, -1])
        finally:
            model.close()
            _MODELS.clear()


def test_b_large_v2_benchmark_regime():
    """large-v2, 10 heads, the large_linear_k10_mixed fixture's options: iterations 1-3, n/2 and n."""
    g, cfg, seed, stream, kw = _load("large_linear_k10_mixed")
    model = _model(cfg, seed)
    pcm = synthetic_audio(float(g["audio_seconds"]), stream_id=stream)
    n = len(g["accept_lengths"])
    try:
        _run("B/large_linear_k10_mixed", model, pcm, kw, iters=[1, 2, 3, n // 2, n])
        assert model.last_trace.accept_lengths == g["accept_lengths"].tolist()[: model.last_trace.iterations]
    finally:
        model.close()
        _MODELS.clear()


# ------------------------------------------------------------------------------------------------ C: trees
TREES = [(1, 3, 4), (1, 3, 2, 1), (1, 4, 2), (1, 2, 2, 2)]


@pytest.mark.parametrize("choices", TREES, ids=["-".join(map(str, c)) for c in TREES])
@pytest.mark.parametrize("tree_attention", [False, True])
def test_c_trees(choices, tree_attention):
    """Every node's candidate, row_pc and row_thr, and path_node, every iteration, T = 0 and 1."""
    cfg = width_config(128, heads=len(choices) - 1)
    cfg.medusa_choices = list(choices)
    model = _model(cfg, 7)
    pcm = synthetic_audio(5.0, stream_id=40)
    for T in (0.0, 1.0):
        kw = _kw(T, PAIRS[0])
        kw["tree_attention"] = tree_attention
        _run(f"C/{choices}/attn{int(tree_attention)}/T{T}", model, pcm, kw)


# ------------------------------------------------------------------------------------------------ D: exact ties
TIE_CASES = [
    # (id, preset / width, V, choices, twins (src, dst, n), decode_ctas for nseg = 1)
    ("micro_chain", 128, None, (1, 1, 1, 1, 1), (0, 256, 256), 8),
    ("micro_142", 128, None, (1, 4, 2), (0, 256, 256), 4),
    ("tiny_chain", "tiny.en", None, (1, 1, 1, 1, 1), (0, 25932, 25932), 8),
]


@pytest.mark.parametrize("case", TIE_CASES, ids=[c[0] for c in TIE_CASES])
def test_d_exact_ties(case):
    """Twin embedding rows give bit-equal logits (asserted first); argmax and top-k then follow the tie rule with the
    twins in different segments (full grid) and in one segment, on different threads of one CTA (nseg = 1)."""
    name, width, V, choices, twins, ctas1 = case
    K = len(choices) - 1
    cfg = width_config(width, heads=K) if isinstance(width, int) else preset_config(width, heads=K)
    cfg.medusa_choices = list(choices)
    model = _model(cfg, 8, twins=twins)
    pcm = synthetic_audio(5.0, stream_id=50)
    its = None if isinstance(width, int) else [1, 2, 3, -1]
    total = 0
    try:
        for T in (0.0, 1.0):
            total += _run(f"D/{name}/full/T{T}", model, pcm, _kw(T, PAIRS[0]), iters=its, twins=twins).ties
        model.set_option("decode_ctas", ctas1)
        for T in (0.0, 1.0):
            total += _run(f"D/{name}/nseg1/T{T}", model, pcm, _kw(T, PAIRS[0]), iters=its, twins=twins).ties
    finally:
        model.close()
        _MODELS.clear()
    assert total > 0, "no row had a tied maximum"


# ------------------------------------------------------------------------------------------------ E: posterior shape
@pytest.mark.parametrize("preset,logit_std,alpha", [("tiny.en", 0.05, 1.0), ("tiny.en", 12.0, 0.3), (128, 12.0, 0.3)])
def test_e_posterior_shape(preset, logit_std, alpha):
    """Flat rows (entropy ~ log V, alpha = 1: p and thr both ~ 1/V) and peaked rows (p ~ 1, other candidates
    underflow)."""
    K = 4
    cfg = width_config(preset, heads=K) if isinstance(preset, int) else preset_config(preset, heads=K)
    model = _model(cfg, 9, logit_std=logit_std)
    pcm = synthetic_audio(5.0, stream_id=60)
    its = None if isinstance(preset, int) else [1, 2, 3, 4, -2, -1]
    for T in (0.5, 1.0, 2.0):
        _run(f"E/{preset}/std{logit_std}/T{T}", model, pcm, _kw(T, (0.09, alpha), max_length=80), iters=its)
