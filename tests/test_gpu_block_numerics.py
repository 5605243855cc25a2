"""Medusa-Block heads against the fp64 engine-regime oracle: every width, row count, tree, prompt depth and accept step.

The Block type runs code the Medusa-Linear type never touches: its own decoder layer ``n_layers`` with its own
self-attention K/V cache (appended by every sweep through ``ST_COPY_HIDDEN`` + ``ST_QKV``, prefill chunks and verify
sweeps included), the tail (``ST_TAIL_SEED``, then the block re-run on the carried hidden state at position L - 1 over
that cache), tree compaction over ``n_layers + 1`` layers, heads written from row 1, and a LayerNorm fold whose split
operand is γ∘x of the copied hidden state.  A fault in any of these changes only the heads' rows 1..K, so the groups
below check logits, not just tokens.  They reuse the checks of tests/test_gpu_decode_rows_and_depth.py,
tests/test_gpu_decode_numerics.py and tests/test_gpu_accept_numerics.py with ``heads_type="medusa_block"``:

* A: ``forward()`` with 1..16 ids at every width, every mode, the ring on 8 / 37 CTAs at 512 and 1280;
* B: chains K = 1, 7, 15 at d = 128, 512, 1280: two iterations, then a whole generate against the fp32 oracle;
* C: 16-node trees under both attention rules, all verify rows, at the first iteration whose ``stage_kv_compact`` moves
  a row (so the block layer's cache is gathered) and at the one after it;
* D: prompts cached by prefill chunks up to position 446;
* E: iterations n/2 and n of runs to length >= 400 against one oracle iteration from the engine's history;
  E': reference-attention trees deep in the loop (both head types) against the accumulated oracle run;
* F: every activation profile at d = 512 and 1280;
* G: candidates and typical acceptance (``last_accept()``) against tests/_accept_ref.py.

Every case uses checkpoint seed 3 and audio stream 3 unless a fixture fixes them.  Bars: DECODE_LOGIT_BAR through
check_logits (``WM_NUMERICS_RECORD`` records every case), PC_BAR / THR_BAR for the accept step."""
import pytest
import torch

import _accept_ref as A
from _decode_ref import decode_logits
from test_gpu_accept_numerics import PAIRS, TEMPS, _kw, _run
from test_gpu_decode_numerics import _logits_vs_fp64
from test_gpu_decode_rows_and_depth import (ALL_MODES, FALLBACK_WIDTH, MAX_LEN, RING_WIDTHS, _chain_verify_and_generate,
                                            _check_pass_logits, _deep_in_the_loop, _e_id, _engine_enc,
                                            _forward_sweeps, _n_tree, _prefilled_prompts)
from test_gpu_scores import _load
from whisper_medusa_b200.synthetic import (ACTIVATION_PROFILES, preset_config, synthetic_audio, synthetic_state_dict,
                                           width_config)

pytestmark = pytest.mark.gpu

SEED = 3
BLOCK = "medusa_block"

_MODELS = {}


def _cfg(d, k, choices=None, heads_type=BLOCK):
    cfg = width_config(d, heads=k, heads_type=heads_type)
    if choices:
        cfg.medusa_choices = list(choices)
    return cfg


def _model(cfg, profile="default", seed=SEED):
    """(model, cfg, sd, pcm); one engine alive at a time."""
    from whisper_medusa_b200 import WhisperMedusaModel

    key = (repr(cfg.to_dict()), profile, seed)
    if key not in _MODELS:
        for m in _MODELS.values():
            m[0].close()
        _MODELS.clear()
        sd = synthetic_state_dict(cfg, seed=seed, activation_profile=profile)
        model = WhisperMedusaModel(cfg, sd).to("cuda:0")
        _MODELS[key] = (model, cfg, sd, synthetic_audio(5.0, stream_id=seed))
    return _MODELS[key]


def _tree_id(ch):
    return "tree" + "".join(map(str, ch))


# ---------------------------------------------------------------------------------------------------------------- A
@pytest.mark.parametrize("d", RING_WIDTHS + (FALLBACK_WIDTH,))
def test_a_forward_sweeps_of_every_row_count(d):
    """forward() with the first 1..16 of 16 ids: heads rows 1..K of every position come from the block re-run at that
    position over a block cache written by a T-row sweep."""
    _forward_sweeps(_model(_cfg(d, 4)), d, f"A/d{d}-block")


# ---------------------------------------------------------------------------------------------------------------- B
@pytest.mark.parametrize("d,k", [(d, k) for d in (128, 512, 1280) for k in (1, 7, 15)], ids=lambda v: str(v))
def test_b_chain_verify_sweeps_of_2_8_16_rows(d, k):
    """Pass A and all K+1 verify rows of two iterations (every mode at d = 512, the ring elsewhere), then a whole
    generate to max_length 448 with the tokens and accept lengths of the fp32 engine-regime oracle."""
    _chain_verify_and_generate(_model(_cfg(d, k)), d, f"B/d{d}-k{k}-block")


# ---------------------------------------------------------------------------------------------------------------- C
def _compaction_moves_rows(tree, a, path_node, tree_attention):
    """Whether the accept step of an iteration with accept length ``a`` and best-path node ``path_node`` makes
    stage_kv_compact move a K/V row (kept row j comes from tree row path[j]; it moves unless path[j] == j)."""
    path = [int(path_node)]
    while tree.parent[path[-1]] >= 0:
        path.append(int(tree.parent[path[-1]]))
    path.reverse()
    keep = a + 1 if (tree_attention and a >= 1) else max(a, 1)
    return any(path[j] != j for j in range(keep))


C_CASES = [(d, ch) for d in (128, 512, 1280) for ch in ((1, 3, 4), (1, 3, 2, 1))]


@pytest.mark.parametrize("case", C_CASES, ids=lambda c: f"d{c[0]}-{_tree_id(c[1])}")
def test_c_tree_verify_rows_across_compaction(case):
    """16-node trees under reference and true tree attention: pass A and all 16 verify rows at iteration i, the first
    one whose accept step moves a kept K/V row in every layer's cache (the block's included), and at iteration i + 1,
    which runs on the compacted caches.  The oracle runs from the start with the same kept rows (its ``keep_rows``)."""
    d, choices = case
    model, cfg, sd, pcm = _model(_cfg(d, len(choices) - 1, choices))
    assert _n_tree(cfg) == 16
    tree = A.tree_tables(choices)
    kw = dict(language=None, max_length=MAX_LEN)
    runs = ALL_MODES if d == 512 else ("persistent",)
    model.set_decode_mode("persistent")
    enc = _engine_enc(model, pcm, kw)
    for ta in (False, True):
        cid = f"C/d{d}-{_tree_id(choices)}" + ("-tree_attn" if ta else "") + "-block"
        first = None
        for it in range(1, 21):
            model.generate_from_pcm(pcm, max_iters=it, tree_attention=ta, **kw)
            tr = model.last_trace
            assert tr.iterations == it, (cid, it)
            if _compaction_moves_rows(tree, tr.accept_lengths[-1], model.last_accept()["path_node"], ta):
                first = it
                break
        assert first is not None, (cid, "no K/V row moved in the first 20 iterations", tr.accept_lengths)
        ref64 = decode_logits(cfg, sd, enc, kw, first + 1, tree_attention=ta)
        ref32 = decode_logits(cfg, sd, enc, kw, first + 1, dtype=torch.float32, tree_attention=ta)
        for mode in runs:
            model.set_decode_mode(mode)
            for it in (first, first + 1):
                model.generate_from_pcm(pcm, max_iters=it, tree_attention=ta, **kw)
                tr = model.last_trace
                assert tr.iterations == it
                assert tr.sequences == ref64.sequences[: len(tr.sequences)], (cid, mode, it)
                _check_pass_logits(model, cfg, ref64, ref32, it, cid, f"{mode}/iter{it}")
        model.set_decode_mode("persistent")


# ---------------------------------------------------------------------------------------------------------------- D
@pytest.mark.parametrize("d,k", [(d, k) for d in RING_WIDTHS for k in (4, 15)], ids=lambda v: str(v))
def test_d_prefilled_prompts_to_full_depth(d, k):
    """Random-id prompts of 16, 17, 32, 33, 255, 256, 257 and max_length - K - 2 tokens: the prefill chunks append the
    block's K/V rows too.  Iteration-1 pass-A and verify logits and tokens (every mode at 512 and 1280, 8 / 37 CTAs at
    1280)."""
    _prefilled_prompts(_model(_cfg(d, k)), d, k, f"D/d{d}-k{k}-block")


# ---------------------------------------------------------------------------------------------------------------- E
# (d, K, medusa_choices, tree_attention, medusa_temperature); seed 3 reaches a length of 434 or more in every case
E_CASES = ([(d, 4, None, False, 1.0) for d in (128, 512, 1280)] + [(512, 15, None, False, 1.0)]
           + [(d, 2, (1, 3, 4), True, 1.0) for d in (128, 512, 1280)] + [(512, 4, None, False, 0.0)])


@pytest.mark.parametrize("case", E_CASES, ids=_e_id)
def test_e_logits_deep_in_the_real_loop(case):
    """A whole generate to max_length 448 reaches a length of 400 or more; at iterations ~n/2 and n the engine's
    logits and continuation equal one iteration of the fp64 oracle started from the engine's own history (the method
    tests/test_oracle_history_prompt.py pins for Block heads)."""
    d, k, choices, ta, temp = case
    _deep_in_the_loop(_model(_cfg(d, k, choices)), ta, temp, "E/" + _e_id(case) + "-block")


E2_CASES = [(ch, ht) for ch in ((1, 3, 4), (1, 3, 2, 1)) for ht in ("base_head", BLOCK)]


@pytest.mark.parametrize("choices,heads_type", E2_CASES, ids=lambda v: _tree_id(v) if isinstance(v, tuple) else v)
def test_e2_reference_attention_trees_deep_in_the_loop(choices, heads_type):
    """Trees under reference attention (the default) keep verify rows computed behind rows that are not their
    ancestors, so the history-prompt identity does not hold for them.  At d = 128 the accumulated fp64 oracle runs the
    whole loop: the engine's run to length >= 400 has its tokens and accept lengths, and iterations ~n/2 and n its
    pass-A and verify logits."""
    model, cfg, sd, pcm = _model(_cfg(128, len(choices) - 1, choices, heads_type))
    cid = f"E2/d128-{_tree_id(choices)}" + ("-block" if heads_type == BLOCK else "")
    kw = dict(language=None, max_length=MAX_LEN)
    model.set_decode_mode("persistent")
    model.generate_from_pcm(pcm, **kw)
    full = model.last_trace
    n = full.iterations
    assert len(full.sequences) >= 400, (cid, len(full.sequences), n)
    enc = model.encoder_output()
    ref64 = decode_logits(cfg, sd, enc, kw, n)
    ref32 = decode_logits(cfg, sd, enc, kw, n, dtype=torch.float32)
    for ref in (ref64, ref32):
        assert ref.sequences == full.sequences and ref.accept_lengths == full.accept_lengths, cid
    for it in sorted({n // 2, n}):
        model.generate_from_pcm(pcm, max_iters=it, **kw)
        assert model.last_trace.iterations == it
        assert model.last_trace.sequences == full.sequences[: len(model.last_trace.sequences)], (cid, it)
        _check_pass_logits(model, cfg, ref64, ref32, it, cid, f"persistent/iter{it}of{n}")


# ---------------------------------------------------------------------------------------------------------------- F
#: ``outliers`` at d = 1280: one verify row of iteration 2 is ill-conditioned.  The fp64 reference itself moves by up to
#: 6.3e-4 there when the encoder states are perturbed by a relative 2^-24, and the fp32 oracle is 4.9e-4 off; the
#: explicit-LayerNorm modes measured 1.04e-3 on an H100 (DESIGN.md section 2, "Medusa-Block against fp64").
F_BARS = {(1280, "outliers"): 3e-3}


@pytest.mark.parametrize("profile", ACTIVATION_PROFILES)
@pytest.mark.parametrize("d", [512, 1280])
def test_f_activation_profiles(d, profile):
    """Pass A and pass B of two iterations and forward() in every mode.  The block's QKV splits γ∘x of the copied
    hidden state in place: the operand most exposed to ``small`` (subnormal lo half) and ``near_top``."""
    _logits_vs_fp64(_model(_cfg(d, 4), profile=profile), d, f"F/d{d}-{profile}-block", F_BARS.get((d, profile)))


# ---------------------------------------------------------------------------------------------------------------- G
@pytest.mark.parametrize("K", [1, 4, 10, 15])
def test_g_chains_micro(K):
    """d = 128: every iteration, every temperature and (threshold, alpha) pair, length penalty (10, 1.15)."""
    model, cfg, sd, pcm = _model(_cfg(128, K))
    for T in TEMPS:
        for pair in PAIRS:
            _run(f"G/micro/K{K}/T{T}/{pair}-block", model, pcm, _kw(T, pair))


@pytest.mark.parametrize("choices", [(1, 3, 4), (1, 3, 2, 1)], ids=_tree_id)
@pytest.mark.parametrize("tree_attention", [False, True])
def test_g_trees(choices, tree_attention):
    """Every node's candidate, row_pc, row_thr and path_node, every iteration, T = 0 and 1."""
    model, cfg, sd, pcm = _model(_cfg(128, len(choices) - 1, choices))
    for T in (0.0, 1.0):
        kw = _kw(T, PAIRS[0])
        kw["tree_attention"] = tree_attention
        _run(f"G/{_tree_id(choices)}/attn{int(tree_attention)}/T{T}-block", model, pcm, kw)


def test_g_tiny_chain():
    """tiny.en, K = 4: iterations 1, 2, n/2 and n under every temperature and (threshold, alpha) pair."""
    model, cfg, sd, pcm = _model(preset_config("tiny.en", heads=4, heads_type=BLOCK))
    for T in TEMPS:
        for pair in PAIRS:
            kw = _kw(T, pair, max_length=120)
            model.generate_from_pcm(pcm, **kw)
            n = model.last_trace.iterations
            _run(f"G/tiny/K4/T{T}/{pair}-block", model, pcm, kw, iters=[1, 2, n // 2, n])


def test_g_large_v2_mixed_fixture():
    """large-v2, 10 Block heads, the large_block_k10_mixed fixture's options: iterations 1-3, n/2 and n."""
    g, cfg, seed, stream, kw = _load("large_block_k10_mixed")
    model = _model(cfg, seed=seed)[0]
    pcm = synthetic_audio(float(g["audio_seconds"]), stream_id=stream)
    n = len(g["accept_lengths"])
    _run("G/large_block_k10_mixed", model, pcm, kw, iters=[1, 2, 3, n // 2, n])
    assert model.last_trace.accept_lengths == g["accept_lengths"].tolist()[: model.last_trace.iterations]
    model.close()
    _MODELS.clear()
