"""Decode passes at every row count a stage tile holds (1..16), at full context depth (up to position 446) and on
16-node candidate trees, against the fp64 engine-regime oracle decoding from the engine's own encoder states.

Every stage of the decode kernels is written for T <= 16 rows and a self-attention context of up to 448 positions;
the checks of test_gpu_decode_numerics.py look at 1..5-row forward() sweeps and at the first two iterations (at most
about 15 cached keys).  Here:

* A: forward() with 1..16 ids (pass-A sweeps of every row count) at every decoder width, in every mode it supports,
  and the ring kernel on partial grids (decode_ctas 8 and 37);
* B: chains with K = 1, 7, 15 (verify sweeps of 2, 8 and 16 rows: K = 15 fills every row of the tile, of the accept
  ballot and of the selection arrays), then a whole generate to max_length 448;
* C: 16-node trees, all 16 verify rows through ``last_logits(2)``;
* D: long decoder prompts (cached by 16-row prefill sweeps) up to the deepest one allowed, so that the verify rows of
  the first iteration sit at positions up to 446;
* E: the real loop to a length of 400 and more, checked at about half way and at its last iteration against one
  iteration of the oracle run from the engine's own history (the method pinned on the CPU by
  tests/test_oracle_history_prompt.py): this checks a self-attention cache built up from kept verify rows, elided
  sweeps, one-token sweeps after accept length 0 and tree compaction moves.

Bar: DECODE_LOGIT_BAR for every logit check (through check_logits, so WM_NUMERICS_RECORD records them); tokens and
accept lengths equal to the oracle.  The engine numbers tree nodes level by level, which is the order of the oracle's
``tree_indices``: verify rows are compared index for index, without a mapping."""
import numpy as np
import pytest
import torch

from _decode_ref import check_logits, decode_logits, forward_logits
from oracle import medusa_ref as M
from oracle import whisper_ref as W
from whisper_medusa_b200.synthetic import synthetic_audio, synthetic_state_dict, width_config

pytestmark = pytest.mark.gpu

RING_WIDTHS = (128, 384, 512, 768, 1024, 1280)
FALLBACK_WIDTH = 640
MAX_LEN = 448
SEED = 3               # checkpoint seed and audio stream: every case below decodes to a length of 434 or more
ALL_MODES = ("persistent", "persistent_simple", "graph")


def _modes(d):
    return ALL_MODES if d in RING_WIDTHS else ("graph", "persistent_simple")


_MODELS = {}


def _model(d, k, choices=None, heads_type="base_head"):
    """(model, cfg, sd, pcm); one engine alive at a time."""
    from whisper_medusa_b200 import WhisperMedusaModel

    key = (d, k, tuple(choices or ()), heads_type)
    if key not in _MODELS:
        for m in _MODELS.values():
            m[0].close()
        _MODELS.clear()
        cfg = width_config(d, heads=k, heads_type=heads_type)
        if choices:
            cfg.medusa_choices = list(choices)
        sd = synthetic_state_dict(cfg, seed=SEED)
        model = WhisperMedusaModel(cfg, sd).to("cuda:0")
        _MODELS[key] = (model, cfg, sd, synthetic_audio(5.0, stream_id=SEED))
    return _MODELS[key]


def _n_tree(cfg):
    n, level = 0, 1
    for c in cfg.medusa_choices:
        level *= int(c)
        n += level
    return n


class _Grid:
    """The ring kernel on ``ctas`` CTAs for the duration of a with-block (None: the full grid)."""

    def __init__(self, model, ctas):
        self.model, self.ctas = model, ctas

    def __enter__(self):
        if self.ctas is not None:
            self.model.set_option("decode_ctas", self.ctas)

    def __exit__(self, *exc):
        if self.ctas is not None:
            self.model.set_option("decode_ctas", torch.cuda.get_device_properties(0).multi_processor_count)


def _engine_enc(model, pcm, kw):
    model.generate_from_pcm(pcm, max_iters=1, **kw)
    return model.encoder_output()


def _check_pass_logits(model, cfg, ref64, ref32, it, case, what):
    """Pass A and every verify row of the engine's last iteration against iteration ``it`` of the references."""
    a = model.last_logits(0).numpy()
    b = model.last_logits(2).numpy()
    assert b.shape == (_n_tree(cfg), cfg.vocab_size)
    assert np.array_equal(model.last_logits(1).numpy(), b[: cfg.medusa_num_heads + 1])
    errs = [check_logits(a, ref64.passA_logits[it - 1].numpy(), case, f"{what}/passA{it}",
                         ref32.passA_logits[it - 1].numpy()),
            check_logits(b, ref64.passB_logits[it - 1].numpy(), case, f"{what}/passB{it}",
                         ref32.passB_logits[it - 1].numpy())]
    return max(errs)


def _check_two_iterations(model, cfg, sd, pcm, kw, case, runs, tree_attention=False):
    """Pass-A and all pass-B logits of iterations 1 and 2 for every (mode, ctas) of ``runs``."""
    model.set_decode_mode("persistent")
    enc = _engine_enc(model, pcm, kw)
    ref64 = decode_logits(cfg, sd, enc, kw, 2, tree_attention=tree_attention)
    ref32 = decode_logits(cfg, sd, enc, kw, 2, dtype=torch.float32, tree_attention=tree_attention)
    worst = {}
    for mode, ctas in runs:
        model.set_decode_mode(mode)
        tag = mode if ctas is None else f"{mode}@{ctas}"
        with _Grid(model, ctas):
            for it in (1, 2):
                model.generate_from_pcm(pcm, max_iters=it, tree_attention=tree_attention, **kw)
                tr = model.last_trace
                assert tr.iterations == it
                assert tr.sequences == ref64.sequences[: len(tr.sequences)], (case, tag, it)
                worst[tag] = max(worst.get(tag, 0.0), _check_pass_logits(model, cfg, ref64, ref32, it, case, tag))
    model.set_decode_mode("persistent")
    print(f"{case}: worst rel. error vs fp64 {worst}")
    return enc


# ---------------------------------------------------------------------------------------------------------------- A
_FWD_IDS = [501, 502] + [int(t) for t in np.random.default_rng(SEED).integers(20, 400, size=14)]


@pytest.mark.parametrize("d", RING_WIDTHS + (FALLBACK_WIDTH,))
def test_forward_sweeps_of_every_row_count(d):
    """forward() with the first 1..16 of 16 ids: a pass-A sweep of every row count a stage tile holds, every head at
    every position, in each decode mode of the width (and the ring on 8 and 37 CTAs at d = 512 / 1280).  The decoder is
    causal, so the fp64 reference of the first n ids is the first n rows of the 16-id reference."""
    _forward_sweeps(_model(d, 4), d, f"A/d{d}")


def _forward_sweeps(entry, d, cid):
    model, cfg, sd, pcm = entry
    kw = dict(language=None, max_length=MAX_LEN)
    model.set_decode_mode(_modes(d)[0])
    enc = _engine_enc(model, pcm, kw)
    fwd64 = forward_logits(cfg, sd, enc, _FWD_IDS).numpy()
    fwd32 = forward_logits(cfg, sd, enc, _FWD_IDS, torch.float32).numpy()
    runs = [(mode, None) for mode in _modes(d)]
    if d in (512, 1280):
        runs += [("persistent", 8), ("persistent", 37)]
    for mode, ctas in runs:
        model.set_decode_mode(mode)
        tag = mode if ctas is None else f"{mode}@{ctas}"
        with _Grid(model, ctas):
            for n in range(1, 17):
                out = model.forward(decoder_input_ids=torch.tensor([_FWD_IDS[:n]])).logits.cpu()[:, 0].numpy()
                assert out.shape == (cfg.medusa_num_heads + 1, n, cfg.vocab_size)
                check_logits(out, fwd64[:, :n], cid, f"{tag}/forward{n}", fwd32[:, :n])
    model.set_decode_mode(_modes(d)[0])


# ---------------------------------------------------------------------------------------------------------------- B
B_CASES = [(d, k, "base_head") for d in (128, 512, 1280) for k in (1, 7, 15)] + [(512, 15, "medusa_block")]


@pytest.mark.parametrize("case", B_CASES, ids=lambda c: f"d{c[0]}-k{c[1]}" + ("-block" if c[2] == "medusa_block" else ""))
def test_chain_verify_sweeps_of_2_8_16_rows(case):
    """Chains of K = 1, 7, 15 heads: pass A and all K+1 verify rows of two iterations against fp64 (every mode at
    d = 512, the ring elsewhere); then a whole generate to max_length 448 gives the tokens and accept lengths of the
    fp32 engine-regime oracle."""
    d, k, htype = case
    cid = f"B/d{d}-k{k}" + ("-block" if htype == "medusa_block" else "")
    tr = _chain_verify_and_generate(_model(d, k, heads_type=htype), d, cid)
    if k == 15 and htype == "base_head":
        assert max(tr.accept_lengths) == 15, cid          # a 16-row verify sweep accepted whole


def _chain_verify_and_generate(entry, d, cid):
    """Two iterations against fp64, then a whole generate against the fp32 oracle; returns the generate's trace."""
    model, cfg, sd, pcm = entry
    kw = dict(language=None, max_length=MAX_LEN)
    runs = [(m, None) for m in (ALL_MODES if d == 512 else ("persistent",))]
    enc = _check_two_iterations(model, cfg, sd, pcm, kw, cid, runs)
    out = model.generate_from_pcm(pcm, **kw)[0].tolist()
    tr = model.last_trace
    prompt = M.init_tokens(cfg, None)
    gp = M.gen_params(cfg, prompt, None, MAX_LEN)
    ref = M.medusa_greedy_search(W.RefWeights(sd), cfg, enc, prompt, gp, "engine")
    assert tr.sequences == ref.sequences, cid
    assert tr.accept_lengths == ref.accept_lengths, cid
    assert out == M.strip_output(ref.sequences, len(prompt), gp)
    return tr


# ---------------------------------------------------------------------------------------------------------------- C
C_CASES = [(d, ch) for d in (128, 512, 1280) for ch in ((1, 3, 4), (1, 3, 2, 1))]


@pytest.mark.parametrize("case", C_CASES, ids=lambda c: f"d{c[0]}-tree{''.join(map(str, c[1]))}")
def test_tree_verify_rows_all_16(case):
    """16-node trees ([1,3,4]: 1 + 3 + 12 nodes; [1,3,2,1]: 1 + 3 + 6 + 6), reference attention and true tree attention:
    pass A and all 16 verify rows of two iterations against the fp64 oracle with the same mask (every mode at d = 512,
    the ring elsewhere)."""
    d, choices = case
    model, cfg, sd, pcm = _model(d, len(choices) - 1, choices)
    assert _n_tree(cfg) == 16
    kw = dict(language=None, max_length=MAX_LEN)
    runs = [(m, None) for m in (ALL_MODES if d == 512 else ("persistent",))]
    for ta in (False, True):
        cid = f"C/d{d}-tree{''.join(map(str, choices))}" + ("-tree_attn" if ta else "")
        _check_two_iterations(model, cfg, sd, pcm, kw, cid, runs, tree_attention=ta)


# ---------------------------------------------------------------------------------------------------------------- D
D_LENGTHS = (16, 17, 32, 33, 255, 256, 257)
D_CASES = [(d, k) for d in RING_WIDTHS for k in (4, 15)]


@pytest.mark.parametrize("case", D_CASES, ids=lambda c: f"d{c[0]}-k{c[1]}")
def test_prefilled_prompts_to_full_depth(case):
    """Decoder prompts of random ids cached by 16-row prefill sweeps, up to the deepest one allowed (max_length - K - 2:
    the verify rows of the first iteration then sit at positions up to 446): iteration-1 pass-A and pass-B logits and
    tokens against the fp64 oracle from the same prompt.  The ring at every width; every mode at 512 and 1280, and the
    ring on 8 and 37 CTAs at 1280."""
    d, k = case
    _prefilled_prompts(_model(d, k), d, k, f"D/d{d}-k{k}")


def _prefilled_prompts(entry, d, k, cid):
    model, cfg, sd, pcm = entry
    deepest = MAX_LEN - k - 2
    assert deepest + k == MAX_LEN - 2          # the last verify position is 446
    runs = [(m, None) for m in (ALL_MODES if d in (512, 1280) else ("persistent",))]
    if d == 1280:
        runs += [("persistent", 8), ("persistent", 37)]
    rng = np.random.default_rng(SEED + k)
    model.set_decode_mode("persistent")
    enc = _engine_enc(model, pcm, dict(language=None, max_length=MAX_LEN))
    for n in D_LENGTHS + (deepest,):
        prompt = [int(t) for t in rng.integers(20, 400, size=n)]
        kw = dict(language=None, max_length=MAX_LEN)
        ref64 = decode_logits(cfg, sd, enc, kw, 1, prompt=prompt)
        ref32 = decode_logits(cfg, sd, enc, kw, 1, dtype=torch.float32, prompt=prompt)
        for mode, ctas in runs:
            model.set_decode_mode(mode)
            tag = mode if ctas is None else f"{mode}@{ctas}"
            with _Grid(model, ctas):
                model.generate_from_pcm(pcm, max_iters=1, decoder_input_ids=torch.tensor([prompt]), **kw)
            tr = model.last_trace
            assert tr.iterations == 1 and tr.sequences == ref64.sequences, (n, tag)
            _check_pass_logits(model, cfg, ref64, ref32, 1, cid, f"{tag}/prompt{n}")
    model.set_decode_mode("persistent")


# ---------------------------------------------------------------------------------------------------------------- E
# (d, K, medusa_choices, tree_attention, medusa_temperature)
E_CASES = ([(d, 4, None, False, 1.0) for d in (128, 512, 1280)] + [(512, 15, None, False, 1.0)]
           + [(d, 2, (1, 3, 4), True, 1.0) for d in (128, 512, 1280)] + [(512, 4, None, False, 0.0)])


def _e_id(c):
    d, k, ch, ta, temp = c
    return f"d{d}-k{k}" + (f"-tree{''.join(map(str, ch))}" if ch else "") + ("-tree_attn" if ta else "") + \
        ("-t0" if temp == 0 else "")


@pytest.mark.parametrize("case", E_CASES, ids=_e_id)
def test_logits_deep_in_the_real_loop(case):
    """A whole generate to max_length 448 (ring kernel) reaches a length of 400 or more; at its iteration ~n/2 and at
    its last iteration n, the engine's logits (pass A, every verify row) and its continuation equal one iteration of the
    fp64 oracle started from the engine's own history, with the original prompt's begin-suppress index and
    length-penalty origin."""
    d, k, choices, ta, temp = case
    _deep_in_the_loop(_model(d, k, choices), ta, temp, "E/" + _e_id(case))


def _deep_in_the_loop(entry, ta, temp, cid):
    model, cfg, sd, pcm = entry
    kw = dict(language=None, max_length=MAX_LEN, medusa_temperature=temp)
    model.set_decode_mode("persistent")
    model.generate_from_pcm(pcm, tree_attention=ta, **kw)
    full = model.last_trace
    n = full.iterations
    assert len(full.sequences) >= 400, (cid, len(full.sequences), n)
    enc = model.encoder_output()
    p = len(M.init_tokens(cfg, None))
    for it in sorted({n // 2, n}):
        model.generate_from_pcm(pcm, max_iters=it - 1, tree_attention=ta, **kw)
        hist = list(model.last_trace.sequences)
        assert model.last_trace.iterations == it - 1 and hist == full.sequences[: len(hist)], (cid, it)
        model.generate_from_pcm(pcm, max_iters=it, tree_attention=ta, **kw)
        tr = model.last_trace
        assert tr.iterations == it
        ref64 = decode_logits(cfg, sd, enc, kw, 1, prompt=hist, begin_index=p, prompt_len=p, tree_attention=ta)
        ref32 = decode_logits(cfg, sd, enc, kw, 1, dtype=torch.float32, prompt=hist, begin_index=p, prompt_len=p,
                              tree_attention=ta)
        assert ref64.sequences == tr.sequences, (cid, it)
        assert ref64.accept_lengths == tr.accept_lengths[-1:], (cid, it)
        _check_pass_logits(model, cfg, ref64, ref32, 1, cid, f"persistent/iter{it}of{n}@L{len(hist)}")
