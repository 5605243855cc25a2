"""GPU tests of generate(return_dict_in_generate=True, output_scores=True, output_logits=True).

* Scoring only reads the loop's buffers: sequences, token ids and accept lengths are identical with it on and off, in
  every decode mode the engine offers, on chains (K = 1, 4, 10), 16-node trees under both attention rules, a 45-token
  prompt (prefill launches), a run to max_length and max_iters = 1.
* The kernel in isolation: the last iteration's processed rows are rebuilt on the host from its raw logits
  (``last_logits``) and ``log_softmax`` is taken in fp64; token log-probabilities and the scores row agree at fp32
  rounding (1e-5 of the row's logit scale).
* Against references: the scores rows against the reference loop's own rows (tests/golden/ref_loop_scores_micro.npz,
  made by oracle/make_scores_golden.py), and token log-probabilities against the fp64 oracle decoding from the engine's
  encoder states.  A log-probability is a logit minus a log-sum-exp, so its error is at most twice the logit error:
  the bar is 2 x DECODE_LOGIT_BAR of the row's logit scale.
"""
import os

import numpy as np
import pytest
import torch

from _decode_ref import DECODE_LOGIT_BAR, check_error, decode_logits
from _wm_paths import GOLDEN
from oracle import make_ref_golden as G
from oracle import make_scores_golden as SG
from oracle import medusa_ref as M
from oracle import scores_ref as S
from whisper_medusa_b200.synthetic import preset_config, synthetic_audio, synthetic_state_dict, width_config

pytestmark = pytest.mark.gpu

ALL_MODES = ("persistent", "graph", "persistent_simple")
DICT = dict(return_dict_in_generate=True, output_scores=True, output_logits=True)

_MODELS = {}


def _model(cfg, seed):
    """One engine alive at a time."""
    from whisper_medusa_b200 import WhisperMedusaModel

    key = (repr(cfg.to_dict()), seed)
    if key not in _MODELS:
        for m in _MODELS.values():
            m[0].close()
        _MODELS.clear()
        sd = synthetic_state_dict(cfg, seed=seed)
        _MODELS[key] = (WhisperMedusaModel(cfg, sd).to("cuda:0"), sd)
    return _MODELS[key]


def _load(name):
    g = np.load(os.path.join(GOLDEN, name + ".npz"))
    seed, stream, max_len, heads, is_block = [int(v) for v in g["meta"]]
    preset = {"micro": "micro", "tiny": "tiny.en", "large": "large-v2"}[name.split("_")[0]]
    cfg = preset_config(preset, heads=heads, heads_type="medusa_block" if is_block else "base_head")
    pen = None if g["penalty"][0] < 0 else (int(g["penalty"][0]), float(g["penalty"][1]))
    kw = dict(language="en" if cfg.is_multilingual else None, max_length=max_len,
              exponential_decay_length_penalty=pen, medusa_temperature=float(g["temperature"]))
    if "posterior" in g.files:
        kw.update(posterior_alpha=float(g["posterior"][0]), posterior_threshold=float(g["posterior"][1]))
    return g, cfg, seed, stream, kw


def _new_tokens(accept_lengths):
    return [a + 1 if a else 2 for a in accept_lengths]


def _host_gp(model, prompt_len, pen):
    """The processors the engine applied (oracle GenParams).  The penalty factor crosses the C ABI as an fp32
    (``wm_gen_params.penalty_factor``), and the engine's EOS table is built from that value."""
    g = model.generation_config
    pen = pen if pen is not None else g.exponential_decay_length_penalty
    if pen is not None:
        pen = (int(pen[0]), float(np.float32(pen[1])))
    return M.GenParams(eos_token_id=int(g.eos_token_id), pad_token_id=int(g.pad_token_id),
                       suppress_tokens=list(g.suppress_tokens or []) or None,
                       begin_suppress_tokens=list(g.begin_suppress_tokens or []) or None, begin_index=prompt_len,
                       exponential_decay_length_penalty=None if pen is None else tuple(pen), prompt_len=prompt_len)


def _row_err(got, ref):
    """Largest difference of two processed rows relative to the row's logit scale; -inf (suppressed ids) must match."""
    got = np.asarray(torch.as_tensor(got).cpu(), np.float64)
    ref = np.asarray(torch.as_tensor(ref).cpu(), np.float64)
    assert np.array_equal(np.isneginf(got), np.isneginf(ref)), "suppressed ids differ"
    fin = np.isfinite(ref)
    assert np.isfinite(got[fin]).all()
    return float(np.abs(got[fin] - ref[fin]).max() / max(1.0, np.abs(ref[fin]).max()))


def _check_output_shape(model, out, plain):
    """The dict result against the plain call's result and the loop's trace."""
    tr = model.last_trace
    V = model.config.vocab_size
    assert torch.equal(out.sequences, plain)
    assert out.accept_lengths == tr.accept_lengths
    assert len(out.scores) == len(out.logits) == tr.iterations
    assert all(a is b for a, b in zip(out.scores, out.logits))
    assert all(tuple(r.shape) == (1, V) for r in out.scores)
    lp = out.token_logprobs.cpu()
    assert tuple(lp.shape) == (1, tr.n_new_tokens)
    assert torch.isfinite(lp).all() and (lp <= 0).all()
    assert out.avg_logprob == pytest.approx(float(lp.double().mean()), rel=1e-12)
    # stops at the first EOS
    n_prompt = len(tr.sequences) - sum(_new_tokens(tr.accept_lengths))
    gen = tr.sequences[n_prompt:]
    eos = int(model.generation_config.eos_token_id)
    assert tr.n_new_tokens == (gen.index(eos) + 1 if eos in gen else len(gen))
    return n_prompt


def _check_last_iteration(model, out, n_prompt, pen, tol=1e-5):
    """Rebuild the last iteration's processed rows from its raw logits and compare the kernel's results with an fp64
    log_softmax of them.  Returns the largest error relative to the row's logit scale."""
    tr = model.last_trace
    cfg = model.config
    a = tr.accept_lengths[-1]
    n_new = _new_tokens([a])[0]
    L = len(tr.sequences) - n_new
    gp = _host_gp(model, n_prompt, pen)
    rows_a = M.process_logits(model.last_logits(0), L, gp)
    rows_b = M.process_logits(model.last_logits(2), L, gp)
    toks = tr.sequences[L:]
    n_tok = tr.n_new_tokens - (L - n_prompt)           # tokens of this iteration up to the first EOS
    chosen = toks[: min(a + 1, n_tok)]
    chain = all(int(c) == 1 for c in cfg.medusa_choices)
    path = list(range(cfg.medusa_num_heads + 1)) if chain else S.best_path(rows_a, cfg.medusa_choices, chosen)
    lp = out.token_logprobs[0, L - n_prompt:].cpu().double()
    assert len(lp) == n_tok
    worst = 0.0
    for j in range(n_tok):
        row = (rows_a[0] if j == 0 else rows_b[path[j - 1]]).double()
        ref = float(torch.log_softmax(row, -1)[toks[j]])
        scale = max(1.0, float(row[torch.isfinite(row)].abs().max()))
        worst = max(worst, abs(float(lp[j]) - ref) / scale)
    assert worst <= tol, worst
    if chain or len(chosen) == a + 1:    # path[a] is known (a tree path is only known up to the first EOS)
        assert _row_err(out.scores[-1][0], rows_b[path[a]]) <= 1e-6
    return worst


# ---------------------------------------------------------------------------------------------- on / off, all modes
# (case id, K, medusa_choices, generate kwargs, EOS suppressed => the run goes to max_length)
_PROMPT45 = [int(t) for t in np.random.default_rng(45).integers(20, 400, size=45)]
CASES = [
    ("chain_k1", 1, None, dict(max_length=200), False),
    ("chain_k4", 4, None, dict(max_length=200), False),
    ("chain_k10", 10, None, dict(max_length=200), False),
    ("tree_134_causal", 2, (1, 3, 4), dict(max_length=200, tree_attention=False), False),
    ("tree_134_ancestors", 2, (1, 3, 4), dict(max_length=200, tree_attention=True), False),
    ("tree_1321_causal", 3, (1, 3, 2, 1), dict(max_length=200, tree_attention=False), False),
    ("tree_1321_ancestors", 3, (1, 3, 2, 1), dict(max_length=200, tree_attention=True), False),
    ("prompt45", 4, None, dict(max_length=200, decoder_input_ids=torch.tensor([_PROMPT45])), False),
    ("to_max_length", 4, None, dict(max_length=448), True),
    ("max_iters1", 4, None, dict(max_length=200, max_iters=1), False),
    ("penalty_t0", 4, None, dict(max_length=200, exponential_decay_length_penalty=(5, 1.2), medusa_temperature=0.0),
     False),
]


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_scoring_changes_no_token_and_is_exact(case):
    from whisper_medusa_b200 import EngineError

    name, k, choices, kw, no_eos = case
    cfg = width_config(512, heads=k)
    if choices:
        cfg.medusa_choices = list(choices)
    model, sd = _model(cfg, 3)
    pcm = synthetic_audio(5.0, stream_id=3)
    g = model.generation_config
    saved = list(g.suppress_tokens or [])
    if no_eos:
        g.suppress_tokens = saved + [int(g.eos_token_id)]
    ran = []
    try:
        for mode in ALL_MODES:
            try:
                model.set_decode_mode(mode)
            except EngineError:
                continue
            plain = model.generate_from_pcm(pcm, **kw)
            ref_tr = model.last_trace
            out = model.generate_from_pcm(pcm, **DICT, **kw)
            tr = model.last_trace
            assert tr.sequences == ref_tr.sequences and tr.accept_lengths == ref_tr.accept_lengths, (name, mode)
            # one scoring launch per enqueued iteration (the persistent modes launch one kernel per iteration and one per
            # 16-token prefill chunk, which is not scored; iterations enqueued after the loop ended in a batch return at
            # once, and so does their scoring launch)
            if mode == "graph":
                assert tr.launches_decode > ref_tr.launches_decode
            else:
                n_prefill = (len(_PROMPT45) - 1) // 16 if "decoder_input_ids" in kw else 0
                assert tr.launches_decode == 2 * ref_tr.launches_decode - n_prefill
            n_prompt = _check_output_shape(model, out, plain)
            if "decoder_input_ids" in kw:
                assert n_prompt == 45
            _check_last_iteration(model, out, n_prompt, kw.get("exponential_decay_length_penalty"))
            # the same call again without the dict: nothing of the scoring remains switched on
            again = model.generate_from_pcm(pcm, **kw)
            assert torch.equal(again, plain) and model.last_trace.launches_decode == ref_tr.launches_decode
            ran.append(mode)
            if no_eos:
                assert int(g.eos_token_id) not in tr.sequences and len(tr.sequences) + k >= kw["max_length"]
            if "max_iters" in kw:
                assert tr.iterations == 1
    finally:
        g.suppress_tokens = saved
        model.set_decode_mode("persistent")
    assert "persistent" in ran and len(ran) >= 2, ran


def test_exact_match_tokens_are_row_maxima():
    """medusa_temperature = 0: every token is its row's argmax, so its log-probability is the row's largest
    log_softmax entry (checked on the last iteration of runs of 1..6 iterations)."""
    g, cfg, seed, stream, kw = _load("micro_linear_k4_t0")
    assert kw["medusa_temperature"] == 0.0
    model, sd = _model(cfg, seed)
    pcm = synthetic_audio(float(g["audio_seconds"]), stream_id=stream)
    for it in range(1, 7):
        out = model.generate_from_pcm(pcm, max_iters=it, **DICT, **kw)
        tr = model.last_trace
        n_prompt = len(tr.sequences) - sum(_new_tokens(tr.accept_lengths))
        a = tr.accept_lengths[-1]
        L = len(tr.sequences) - _new_tokens([a])[0]
        gp = _host_gp(model, n_prompt, kw["exponential_decay_length_penalty"])
        rows_a = M.process_logits(model.last_logits(0), L, gp).double()
        rows_b = M.process_logits(model.last_logits(2), L, gp).double()
        lp = out.token_logprobs[0, L - n_prompt:].cpu().double()
        for j in range(len(lp)):
            row = rows_a[0] if j == 0 else rows_b[j - 1]
            assert tr.sequences[L + j] == int(row.argmax())
            assert abs(float(lp[j]) - float(torch.log_softmax(row, -1).max())) <= 1e-5 * max(1.0, float(row[torch.isfinite(row)].abs().max()))


# ---------------------------------------------------------------------------------------------- against references
def test_scores_match_the_reference_loop_rows():
    """The scores rows against the reference loop's own rows, on every iteration up to the first one where the engine's
    decisions leave the reference's (fp16 K/V caches and operands against fp32: a decision within ~1e-3 of a tie can
    flip).  Bar: 2e-2 of the logit scale, the end-to-end bar of the engine's logits against an fp32 golden
    (tests/test_gpu_parity.py), since the reference also runs its own fp32 encoder."""
    fx = np.load(os.path.join(GOLDEN, "ref_loop_scores_micro.npz"))
    compared = total = eos_stops = 0
    worst = 0.0
    for group, s in SG.STREAMS:
        cfg, sd, pcm, max_len, pen, temp, alpha, thr = G.stream_inputs(group, s)
        from whisper_medusa_b200 import WhisperMedusaModel

        m = WhisperMedusaModel(cfg, sd).to("cuda:0")
        try:
            kw = dict(max_length=max_len, exponential_decay_length_penalty=pen, medusa_temperature=temp,
                      posterior_alpha=alpha, posterior_threshold=thr)
            plain = m.generate_from_pcm(pcm, **kw)
            out = m.generate_from_pcm(pcm, **DICT, **kw)
            n_prompt = _check_output_shape(m, out, plain)
            _check_last_iteration(m, out, n_prompt, pen)
            tr = m.last_trace
        finally:
            m.close()
        ref_acc = fx[f"{group}/{s}/accept"].tolist()
        ref_rows = fx[f"{group}/{s}/scores"]
        seq_ref = fx[f"{group}/{s}/sequences"].tolist()
        eos_stops += int(cfg.eos_token_id in seq_ref[n_prompt:])
        total += len(ref_acc)
        L = n_prompt
        for i, (a, b) in enumerate(zip(tr.accept_lengths, ref_acc)):
            if a != b or tr.sequences[: L + _new_tokens([a])[0]] != seq_ref[: L + _new_tokens([a])[0]]:
                break
            err = _row_err(out.scores[i][0], ref_rows[i])
            worst = max(worst, err)
            assert err <= 2e-2, (group, i, err)
            compared += 1
            L += _new_tokens([a])[0]
    print(f"scores vs the reference loop: {compared} of {total} iterations compared, worst {worst:.2e}")
    assert compared >= 0.8 * total and eos_stops >= 1


FP64_CASES = [("micro_linear_k4", None), ("micro_block_k10", None), ("tiny_linear_k4", None),
              ("large_linear_k10_mixed", 3)]


@pytest.mark.parametrize("name,n_iters", FP64_CASES, ids=[c[0] for c in FP64_CASES])
def test_token_logprobs_match_the_fp64_oracle(name, n_iters):
    """Token log-probabilities (and the scores rows) of the golden streams against the fp64 engine-regime oracle
    decoding from the engine's own encoder states (all iterations; the first ``n_iters`` at large-v2)."""
    if not os.path.isfile(os.path.join(GOLDEN, name + ".npz")):
        pytest.skip("fixture missing")
    g, cfg, seed, stream, kw = _load(name)
    model, sd = _model(cfg, seed)
    model.set_decode_mode("persistent")
    pcm = synthetic_audio(float(g["audio_seconds"]), stream_id=stream)
    plain = model.generate_from_pcm(pcm, **kw)
    out = model.generate_from_pcm(pcm, **DICT, **kw)
    tr = model.last_trace
    assert tr.accept_lengths == g["accept_lengths"].tolist()
    n_prompt = _check_output_shape(model, out, plain)
    _check_last_iteration(model, out, n_prompt, kw["exponential_decay_length_penalty"])
    n = tr.iterations if n_iters is None else min(n_iters, tr.iterations)
    ref = decode_logits(cfg, sd, model.encoder_output(), kw, n)
    assert ref.accept_lengths == tr.accept_lengths[:n]
    prompt = M.init_tokens(cfg, kw.get("language"))
    extra = {k: kw[k] for k in ("posterior_alpha", "posterior_threshold") if k in kw}
    gp = M.gen_params(cfg, prompt, kw["exponential_decay_length_penalty"], kw["max_length"],
                      temperature=kw["medusa_temperature"], **extra)
    sc = S.loop_scores(ref, len(prompt), gp, cfg.medusa_choices)
    n_tok = min(tr.n_new_tokens, len(sc.token_logprobs))
    lp = out.token_logprobs[0, :n_tok].cpu().double().numpy()
    err = max(abs(float(lp[j]) - sc.token_logprobs[j]) / sc.token_scales[j] for j in range(n_tok))
    check_error(err, 2 * DECODE_LOGIT_BAR, name, "token_logprobs")
    rows_err = max(_row_err(out.scores[i][0], sc.rows[i]) for i in range(n))
    check_error(rows_err, DECODE_LOGIT_BAR, name, "scores")
    print(f"{name}: {n_tok} token log-probabilities, worst error {err:.2e} of the logit scale")
