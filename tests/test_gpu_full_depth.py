"""Every Whisper size at its full depth and vocabulary against the fp64 engine-regime oracle (DESIGN.md section 2,
"Full depth").

The other fp64 files build 2-layer models with micro's 512-token vocabulary (``width_config``).  Here the real sizes
(``preset_config``: tiny.en, base, small, medium, large-v2; 4 to 32 layers, V = 51864 / 51865) and a d = 128 model
with 39 decoder layers plus a Medusa-Block layer (every one of the 40 decoder-layer records) run end to end.  What
depth reaches: the ring kernel's folded LayerNorms (3 per layer; the fold magnifies each row's error by about
sqrt(1 + mu^2 / sigma^2), and under ``offset`` the residual DC grows with every layer), the encoder GEMMs' fp16
operands over 32 layers, per-layer tables (self-K/V caches, stage records, the timestamp slot map), and with the real
vocabulary the vocabulary stage's multi-chunk rows per CTA (about 393 rows: 24 full 16-row chunks and a partial one).

Every comparison starts from the engine's own mel and encoder states; the fp32 oracle's error against the same fp64
reference is recorded beside the engine's (``WM_NUMERICS_RECORD``, tests/_decode_ref.py).  Bars: DECODE_LOGIT_BAR for
logits and the no-speech row, twice that for log-probabilities, the encoder bars of test_gpu_encoder_numerics.py.
Tokens and accept lengths equal the oracle's.  One engine is alive at a time, and one fp64 / fp32 copy of its weights
(``RefWeights``) is built per engine and shared by every oracle call (12 GB in fp64 at large-v2).

* A: encoder states at every size (30 s of speech and the tail-only mel), at medium and large-v2 under every encoder
  profile; enc_gemm 2 and enc_pdl 0 give the same bits as the default.
* B: decoder logits at every size in every decode mode: forward() with 1, 5 and 16 ids, pass A and every verify row of
  iterations 1 and 2 at K = 10 (also in the ring kernel on 37 CTAs) and K = 4, and iterations n/2 and n of a run of
  400 new tokens or more (rebuilt from the engine's history); at medium and large-v2 under every decoder activation
  profile in persistent (folded LayerNorm) and persistent_simple (explicit LayerNorm).
* C: Medusa-Block at base and large-v2 (the block layer is decoder record 6 / 32): forward() with 1...16 ids and two
  iterations of a chain, and a 16-node tree at the first iteration whose compaction moves a K/V row in every layer's
  cache and the next one, in every mode.
* D: token log-probabilities and scores rows at base and medium, the no-speech row at every size, timestamp capture at
  medium and large-v2 with 64 alignment pairs over the upper half of the decoder.
* E: d = 128 with 39 decoder layers and a Block layer in every mode: forward(), two iterations and a run of 440 new
  tokens or more.
"""
import math

import numpy as np
import pytest
import torch

from _decode_ref import DECODE_LOGIT_BAR, check_error, check_logits, decode_logits, forward_logits, rel_err
from oracle import medusa_ref as M
from oracle import no_speech_ref as NS
from oracle import scores_ref as S
from oracle import timestamps_ref as TS
from oracle import whisper_ref as W
import _accept_ref as A
from test_gpu_block_numerics import _compaction_moves_rows
from test_gpu_decode_rows_and_depth import _Grid, _check_pass_logits, _n_tree
from test_gpu_encoder_numerics import ENC_MAX_BAR, ENC_MAX_BAR_PROFILES, check_states
from test_gpu_scores import _row_err
from test_oracle_encoder_fp64 import tail_only_mel
from whisper_medusa_b200.synthetic import preset_config, synthetic_audio, synthetic_state_dict

pytestmark = pytest.mark.gpu

GEOMS = ("tiny.en", "base", "small", "medium", "large-v2")
ALL_MODES = ("persistent", "persistent_simple", "graph")
MAX_LEN = 448
#: (decoder activation profile, encoder profile) pairs sharing one checkpoint: the two never touch the same tensor
#: (tests/test_oracle_encoder_fp64.py), and the decoder checks start from the engine's own encoder states
PROFILE_PAIRS = (("offset", "offset"), ("outliers", "outliers"), ("gamma_spread", "small"), ("small", "peaked"),
                 ("near_top", "near_top"))


class _Entry:
    """An engine and what its checks share: config, state dict, fp64 / fp32 oracle weights, a 5 s clip."""

    def __init__(self, cfg, seed, act="default", enc="default"):
        from whisper_medusa_b200 import WhisperMedusaModel

        self.cfg, self.seed = cfg, seed
        self.sd = synthetic_state_dict(cfg, seed=seed, activation_profile=act, encoder_profile=enc)
        self.model = WhisperMedusaModel(cfg, self.sd).to("cuda:0")
        self.w64 = W.RefWeights(self.sd, torch.float64)
        self.w32 = W.RefWeights(self.sd)
        self.pcm = synthetic_audio(5.0, stream_id=seed)
        self.prompt = M.init_tokens(cfg, _lang(cfg))

    def close(self):
        self.model.close()


_ENTRY = {}


def _entry(name, k=10, htype="base_head", act="default", enc="default", choices=None, **kw):
    key = (name, k, htype, act, enc, choices, tuple(sorted(kw.items())))
    if key not in _ENTRY:
        for e in _ENTRY.values():
            e.close()
        _ENTRY.clear()
        cfg = preset_config(name, heads=k, heads_type=htype, **kw)
        if choices:
            cfg.medusa_choices = list(choices)
        seed = 60 + (GEOMS.index(name) if name in GEOMS else 7)
        _ENTRY[key] = _Entry(cfg, seed, act, enc)
    return _ENTRY[key]


def _lang(cfg):
    return "en" if cfg.is_multilingual else None


def _kw(cfg):
    return dict(language=_lang(cfg), max_length=MAX_LEN)


def _engine_enc(e, mode="persistent"):
    e.model.set_decode_mode(mode)
    e.model.generate_from_pcm(e.pcm, max_iters=1, **_kw(e.cfg))
    return e.model.encoder_output()


def _fwd_ids(cfg):
    rng = np.random.default_rng(cfg.d_model)
    hi = min(cfg.vocab_size, 50000)
    return [cfg.decoder_start_token_id, cfg.no_timestamps_token_id] + [int(t) for t in rng.integers(220, hi, size=14)]


# ------------------------------------------------------------------------------------------------------------ checks
def _encoder(e, case, inputs=("speech30", "mel_tail"), profile=False, bit_options=False):
    """Encoder states on each input against fp64, the fp32 oracle's error beside it."""
    model, cfg = e.model, e.cfg
    for inp in inputs:
        if inp == "speech30":
            run = lambda: model.generate_from_pcm(synthetic_audio(30.0, stream_id=e.seed), max_iters=1, **_kw(e.cfg))
        else:
            feats = torch.from_numpy(tail_only_mel(e.seed).astype(np.float32))[None]
            run = lambda: model.generate(input_features=feats, max_iters=1, **_kw(e.cfg))
        run()
        mel, enc = model.mel(), model.encoder_output()
        r64 = W.encoder_forward(e.w64, cfg, mel.double(), "engine")
        r32 = W.encoder_forward(e.w32, cfg, mel, "engine")
        worst = check_states(enc, r64, r32, f"{case}/{inp}", max_bar=ENC_MAX_BAR_PROFILES if profile else ENC_MAX_BAR)
        print(f"A {case}/{inp}: encoder worst rel. error vs fp64 {worst:.3g}, "
              f"fp32 oracle {rel_err(r32.double().numpy(), r64.numpy()):.3g}")
        if bit_options:
            for opt in ("enc_gemm", "enc_pdl"):
                try:
                    model.set_option(opt, 2 if opt == "enc_gemm" else 0)
                    run()
                    assert torch.equal(model.encoder_output(), enc), (case, inp, opt)
                finally:
                    model.set_option(opt, 1)


def _forward(e, case, modes, lengths):
    """forward() with the first n of 16 ids for each n in ``lengths``, in each mode."""
    cfg = e.cfg
    enc = _engine_enc(e)
    ids = _fwd_ids(cfg)
    f64 = forward_logits(cfg, e.w64, enc, ids).numpy()
    f32 = forward_logits(cfg, e.w32, enc, ids).numpy()
    worst = {}
    for mode in modes:
        e.model.set_decode_mode(mode)
        for n in lengths:
            out = e.model.forward(decoder_input_ids=torch.tensor([ids[:n]])).logits.cpu()[:, 0].numpy()
            assert out.shape == (cfg.medusa_num_heads + 1, n, cfg.vocab_size)
            err = check_logits(out, f64[:, :n], case, f"{mode}/forward{n}", f32[:, :n])
            worst[mode] = max(worst.get(mode, 0.0), err)
    e.model.set_decode_mode("persistent")
    print(f"B {case}: forward worst rel. error vs fp64 {worst}")


def _two_iterations(e, case, modes, grid=None):
    """Pass A and every verify row of iterations 1 and 2 in each mode, and in the ring kernel on ``grid`` CTAs if given
    (on 37 CTAs a vocabulary-stage CTA holds about 1400 rows of the 51865; every layer's records are striped anew)."""
    cfg, model = e.cfg, e.model
    enc = _engine_enc(e)
    kw = _kw(e.cfg)
    r64 = decode_logits(cfg, e.w64, enc, kw, 2)
    r32 = decode_logits(cfg, e.w32, enc, kw, 2)
    worst = {}
    for mode, ctas in [(m, None) for m in modes] + ([("persistent", grid)] if grid else []):
        model.set_decode_mode(mode)
        tag = mode if ctas is None else f"{mode}@{ctas}"
        with _Grid(model, ctas):
            for it in (1, 2):
                model.generate_from_pcm(e.pcm, max_iters=it, **kw)
                tr = model.last_trace
                assert tr.iterations == it
                assert tr.sequences == r64.sequences[: len(tr.sequences)], (case, tag, it)
                worst[tag] = max(worst.get(tag, 0.0), _check_pass_logits(model, cfg, r64, r32, it, case, tag))
    model.set_decode_mode("persistent")
    ring = worst.get("persistent")
    explicit = max([worst[m] for m in ("persistent_simple", "graph") if m in worst] or [0.0])
    ratio = f"{ring / explicit:.2f}" if ring is not None and explicit > 0 else "n/a"
    print(f"B {case}: iterations 1-2 worst rel. error vs fp64 {worst}; ring / explicit-LN = {ratio}")


def _deep(e, case, modes, min_new):
    """A run to MAX_LEN makes at least ``min_new`` new tokens (the prompt not counted); iterations ~n/2 and n of it, in each mode, equal one iteration of
    the oracle started from the engine's history with the original prompt's begin-suppress index and length-penalty
    origin (tokens, accept length, pass-A and every verify row)."""
    cfg, model = e.cfg, e.model
    kw = _kw(e.cfg)
    model.set_decode_mode("persistent")
    model.generate_from_pcm(e.pcm, **kw)
    full = model.last_trace
    n = full.iterations
    p = len(e.prompt)
    assert len(full.sequences) - p >= min_new, (case, len(full.sequences), n)
    enc = model.encoder_output()
    refs = {}
    for mode in modes:
        model.set_decode_mode(mode)
        model.generate_from_pcm(e.pcm, **kw)
        assert model.last_trace.sequences == full.sequences and model.last_trace.accept_lengths == full.accept_lengths, \
            (case, mode)
        for it in sorted({n // 2, n}):
            model.generate_from_pcm(e.pcm, max_iters=it - 1, **kw)
            hist = list(model.last_trace.sequences)
            assert hist == full.sequences[: len(hist)], (case, mode, it)
            model.generate_from_pcm(e.pcm, max_iters=it, **kw)
            tr = model.last_trace
            assert tr.iterations == it
            if it not in refs:
                refs[it] = tuple(decode_logits(cfg, w, enc, kw, 1, prompt=hist, begin_index=p, prompt_len=p)
                                 for w in (e.w64, e.w32))
            r64, r32 = refs[it]
            assert r64.sequences == tr.sequences, (case, mode, it)
            assert r64.accept_lengths == tr.accept_lengths[-1:], (case, mode, it)
            _check_pass_logits(model, cfg, r64, r32, 1, case, f"{mode}/iter{it}of{n}@L{len(hist)}")
    model.set_decode_mode("persistent")
    print(f"B {case}: run of {len(full.sequences)} tokens in {n} iterations checked at {sorted(refs)}")


def _no_speech(e, case):
    """The raw SOT row and log p[no_speech] in each decode mode."""
    model, cfg = e.model, e.cfg
    for mode in ALL_MODES:
        model.set_decode_mode(mode)
        out = model.generate_from_pcm(e.pcm, language=_lang(cfg), max_length=60, return_dict_in_generate=True, output_scores=True,
                                      output_no_speech_prob=True)
        prob, row = model.last_no_speech()
        assert prob == out.no_speech_prob
        ref, ref_p = NS.no_speech_row(e.w64, cfg, model.encoder_output().double(), regime="engine")
        ref = ref.numpy()
        check_error(rel_err(row.numpy(), ref), DECODE_LOGIT_BAR, case, f"{mode}/no_speech_row")
        scale = max(1.0, float(np.abs(ref).max()))
        check_error(abs(math.log(prob) - math.log(ref_p)) / scale, 2 * DECODE_LOGIT_BAR, case, f"{mode}/log_p_no_speech")
    model.set_decode_mode("persistent")


def _scores(e, case, n_iters=3):
    """Token log-probabilities and scores rows of the first ``n_iters`` iterations of a run."""
    model, cfg = e.model, e.cfg
    kw = _kw(e.cfg)
    model.set_decode_mode("persistent")
    out = model.generate_from_pcm(e.pcm, return_dict_in_generate=True, output_scores=True, **kw)
    tr = model.last_trace
    ref = decode_logits(cfg, e.w64, model.encoder_output(), kw, n_iters)
    assert ref.accept_lengths == tr.accept_lengths[:n_iters], case
    gp = M.gen_params(cfg, e.prompt, None, MAX_LEN)
    sc = S.loop_scores(ref, len(e.prompt), gp, cfg.medusa_choices)
    n_tok = min(tr.n_new_tokens, len(sc.token_logprobs))
    lp = out.token_logprobs[0, :n_tok].cpu().double().numpy()
    err = max(abs(float(lp[j]) - sc.token_logprobs[j]) / sc.token_scales[j] for j in range(n_tok))
    check_error(err, 2 * DECODE_LOGIT_BAR, case, "token_logprobs")
    check_error(max(_row_err(out.scores[i][0], sc.rows[i]) for i in range(n_iters)), DECODE_LOGIT_BAR, case, "scores")


def _alignment_pairs(cfg, n=64):
    """``n`` distinct (layer, head) pairs over the upper half of the decoder, every head of the last layer included."""
    L, H = cfg.decoder_layers, cfg.decoder_attention_heads
    rest = [[l, h] for l in range(L // 2, L - 1) for h in range(H)]
    pick = np.random.default_rng(L).permutation(len(rest))[: n - H]
    return [[L - 1, h] for h in range(H)] + [rest[i] for i in sorted(pick)]


def _tree_compaction(e, case, modes):
    """A 16-node tree under reference and true tree attention: pass A and all 16 verify rows at iteration i, the first
    one whose accept step makes stage_kv_compact move a kept K/V row in every layer's cache (the block's included), and
    at iteration i + 1, which runs on the compacted caches, against the oracle run from the start with the same kept
    rows (test_gpu_block_numerics.py group C at depth)."""
    cfg, model = e.cfg, e.model
    assert _n_tree(cfg) == 16
    tree = A.tree_tables(cfg.medusa_choices)
    kw = _kw(cfg)
    enc = _engine_enc(e)
    for ta in (False, True):
        cid = case + ("-tree_attn" if ta else "")
        first = None
        for it in range(1, 21):
            model.generate_from_pcm(e.pcm, max_iters=it, tree_attention=ta, **kw)
            tr = model.last_trace
            assert tr.iterations == it, (cid, it)
            if _compaction_moves_rows(tree, tr.accept_lengths[-1], model.last_accept()["path_node"], ta):
                first = it
                break
        assert first is not None, (cid, "no K/V row moved in the first 20 iterations", tr.accept_lengths)
        r64 = decode_logits(cfg, e.w64, enc, kw, first + 1, tree_attention=ta)
        r32 = decode_logits(cfg, e.w32, enc, kw, first + 1, tree_attention=ta)
        for mode in modes:
            model.set_decode_mode(mode)
            for it in (first, first + 1):
                model.generate_from_pcm(e.pcm, max_iters=it, tree_attention=ta, **kw)
                tr = model.last_trace
                assert tr.iterations == it
                assert tr.sequences == r64.sequences[: len(tr.sequences)], (cid, mode, it)
                _check_pass_logits(model, cfg, r64, r32, it, cid, f"{mode}/iter{it}")
        model.set_decode_mode("persistent")
        print(f"C {cid}: compaction first moves a row at iteration {first}")


def _timestamps(e, case):
    """Alignment-head cross-attention probabilities captured during the decode loop (64 pairs) against fp64."""
    model, cfg = e.model, e.cfg
    pairs = _alignment_pairs(cfg)
    assert len(pairs) == 64 and len({tuple(p) for p in pairs}) == 64
    model.generation_config.alignment_heads = pairs
    try:
        for mode in ("persistent", "persistent_simple"):
            model.set_decode_mode(mode)
            model.generate_from_pcm(e.pcm, language=_lang(cfg), max_length=80, return_token_timestamps=True, return_dict_in_generate=True)
            tr = model.last_trace
            seq = tr.sequences[: len(e.prompt) + tr.n_new_tokens]
            n = len(seq)
            got = model.last_alignment_probs(0, n - 1).double()
            ref, scores = TS.alignment_probs(e.w64, cfg, seq[: n - 1], model.encoder_output().double(), pairs,
                                             regime="engine", return_scores=True)
            assert got.shape == ref.shape
            mask = ref > 1e-20
            err = float((got.clamp_min(1e-300).log() - ref.log())[mask].abs().max())
            check_error(err / max(1.0, float(scores.abs().max())), 2 * DECODE_LOGIT_BAR, case,
                        f"{mode}/alignment_log_probs")
    finally:
        model.generation_config.alignment_heads = None
        model.set_decode_mode("persistent")


# ------------------------------------------------------------------------------------------------------------- tests
@pytest.mark.parametrize("name", GEOMS)
def test_default_profile_every_size(name):
    """A, B (K = 10), D at one size: the encoder on two inputs (and its bit-identical options), forward() with 1, 5 and
    16 ids, iterations 1-2 and a deep run in every mode, the no-speech row, scores at base / medium and timestamps at
    medium / large-v2."""
    e = _entry(name)
    case = f"{name}-k10"
    _encoder(e, case, bit_options=True)
    _forward(e, case, ALL_MODES, (1, 5, 16))
    _two_iterations(e, case, ALL_MODES, grid=37)
    _deep(e, case, ALL_MODES, min_new=400)
    _no_speech(e, case)
    if name in ("base", "medium"):
        _scores(e, case)


@pytest.mark.parametrize("name", GEOMS)
def test_k4_every_size(name):
    """B at K = 4: pass A and the 5 verify rows of iterations 1 and 2 in every mode."""
    _two_iterations(_entry(name, k=4), f"{name}-k4", ALL_MODES)


@pytest.mark.parametrize("name", ("base", "large-v2"))
def test_block_at_depth(name):
    """C: the Medusa-Block layer after 6 / 32 decoder layers, K = 10: forward() with 1...16 ids and two iterations in
    every mode."""
    e = _entry(name, htype="medusa_block")
    case = f"{name}-block-k10"
    _forward(e, case, ALL_MODES, range(1, 17))
    _two_iterations(e, case, ALL_MODES)
    _tree_compaction(_entry(name, k=2, htype="medusa_block", choices=(1, 3, 4)), f"{name}-block-tree134", ALL_MODES)


@pytest.mark.parametrize("name", ("medium", "large-v2"))
def test_timestamps_at_depth(name):
    """D: alignment probabilities captured during the decode loop, 64 pairs over the upper half of a 24 / 32-layer
    decoder (every head of the last layer included), in persistent and persistent_simple."""
    _timestamps(_entry(name), f"{name}-k10")


def test_39_layers_and_a_block_layer():
    """E: all 40 decoder-layer records (39 layers + the Block layer) at d = 128: forward() with 1...16 ids, two
    iterations and a run of 440 new tokens or more (measured: 442 in 221 iterations) in every mode."""
    e = _entry("micro", k=4, htype="medusa_block", decoder_layers=39)
    assert e.cfg.decoder_layers == 39 and e.cfg.is_block
    case = "micro-39layers-block-k4"
    _forward(e, case, ALL_MODES, range(1, 17))
    _two_iterations(e, case, ALL_MODES)
    _deep(e, case, ALL_MODES, min_new=440)


@pytest.mark.parametrize("pair", PROFILE_PAIRS, ids=[f"{a}+enc_{b}" for a, b in PROFILE_PAIRS])
@pytest.mark.parametrize("name", ("medium", "large-v2"))
def test_profiles_at_depth(name, pair):
    """A and B under the activation profiles at 24 and 32 layers: the encoder under its profile, and the ring kernel
    (folded LayerNorm) and persistent_simple (explicit LayerNorm) under the decoder profile: forward() with 16 ids and
    iterations 1-2."""
    act, enc = pair
    e = _entry(name, act=act, enc=enc)
    case = f"{name}-k10-{act}+enc_{enc}"
    _encoder(e, case, inputs=("speech30",), profile=True)
    modes = ("persistent", "persistent_simple")
    _forward(e, case, modes, (16,))
    _two_iterations(e, case, modes)
