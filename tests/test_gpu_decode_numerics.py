"""Decoder and encoder numerics at every decoder width the engine ships, against an fp64 reference, on checkpoints
whose residual stream has the statistics of real ones (``synthetic_state_dict(activation_profile=...)``).

Widths: the ring kernel's instantiations (WM_RING_WIDTHS: 128, 384, 512, 768, 1024, 1280 = micro, tiny, base, small,
medium, large) and 640, a valid width without a ring instantiation (decodes in graph / persistent_simple mode).  Every
width runs the default profile; 512 and 1280 also run every activation profile.  Bars: decode logits within
DECODE_LOGIT_BAR of the fp64 engine-regime oracle in every decode mode; tokens and accept lengths equal to the fp32
engine-regime oracle; encoder states within 5e-3 of the engine-regime oracle over all 1500 rows."""
import ctypes as C

import numpy as np
import pytest
import torch

from _decode_ref import check_logits, decode_logits, forward_logits, rel_err
from oracle import medusa_ref as M
from oracle import whisper_ref as W
from whisper_medusa_b200.synthetic import ACTIVATION_PROFILES, synthetic_audio, synthetic_state_dict, width_config

pytestmark = pytest.mark.gpu

RING_WIDTHS = (128, 384, 512, 768, 1024, 1280)
FALLBACK_WIDTH = 640
PROFILES = [p for p in ACTIVATION_PROFILES if p != "default"]

# (d_model, activation profile, heads type, ffn_dim (0 = 4 d))
CASES = ([(d, "default", "base_head", 0) for d in RING_WIDTHS + (FALLBACK_WIDTH,)]
         + [(d, p, "base_head", 0) for d in (512, 1280) for p in PROFILES]
         + [(512, "default", "medusa_block", 0), (1280, "offset", "medusa_block", 0), (768, "default", "base_head", 768)])


def _case_id(case):
    d, prof, ht, ffn = case
    return f"d{d}-{prof}" + ("-block" if ht == "medusa_block" else "") + (f"-ffn{ffn}" if ffn else "")


_KW = dict(language=None, max_length=60)
_FWD_IDS = (501, 502, 17, 33, 64)        # micro's <|startoftranscript|> <|notimestamps|> and three text tokens


def _modes(d):
    return ("persistent", "persistent_simple", "graph") if d in RING_WIDTHS else ("graph", "persistent_simple")


_MODELS = {}


def _model(case):
    """(model, cfg, sd, pcm) of a case; one engine alive at a time."""
    from whisper_medusa_b200 import WhisperMedusaModel

    if case not in _MODELS:
        for m in _MODELS.values():
            m[0].close()
        _MODELS.clear()
        d, prof, ht, ffn = case
        cfg = width_config(d, heads=4, heads_type=ht, ffn_dim=ffn)
        seed = 3 + RING_WIDTHS.index(d) if d in RING_WIDTHS else 9
        sd = synthetic_state_dict(cfg, seed=seed, activation_profile=prof)
        model = WhisperMedusaModel(cfg, sd).to("cuda:0")
        _MODELS[case] = (model, cfg, sd, synthetic_audio(5.0, stream_id=seed))
    return _MODELS[case]


@pytest.mark.parametrize("case", CASES, ids=_case_id)
def test_decode_logits_vs_fp64_reference(case):
    """Pass-A / pass-B logits of two speculative iterations and forward() logits, in every decode mode the width
    supports, against the fp64 oracle decoding from the engine's own encoder states.  Prints the error of the ring
    kernel (folded LayerNorm) over that of the explicit-LayerNorm modes."""
    model, cfg, sd, pcm = _model(case)
    cid = _case_id(case)
    modes = _modes(case[0])
    model.set_decode_mode(modes[0])
    model.generate_from_pcm(pcm, max_iters=1, **_KW)
    enc = model.encoder_output()
    ref64 = decode_logits(cfg, sd, enc, _KW, 2)
    ref32 = decode_logits(cfg, sd, enc, _KW, 2, dtype=torch.float32)
    ids = list(_FWD_IDS)
    fwd64 = forward_logits(cfg, sd, enc, ids).numpy()
    fwd32 = forward_logits(cfg, sd, enc, ids, torch.float32).numpy()
    worst = {}
    for mode in modes:
        model.set_decode_mode(mode)
        errs = []
        for it in (1, 2):
            model.generate_from_pcm(pcm, max_iters=it, **_KW)
            assert model.last_trace.iterations == it
            # iteration 2 starts from what iteration 1 accepted: the same tokens, or the logits are not comparable
            assert model.last_trace.sequences == ref64.sequences[: len(model.last_trace.sequences)], (cid, mode)
            for ab, which in (("A", 0), ("B", 1)):
                r64 = getattr(ref64, f"pass{ab}_logits")[it - 1].numpy()
                r32 = getattr(ref32, f"pass{ab}_logits")[it - 1].numpy()
                errs.append(check_logits(model.last_logits(which).numpy(), r64, cid, f"{mode}/pass{ab}{it}", r32))
        out = model.forward(decoder_input_ids=torch.tensor([ids])).logits.cpu()[:, 0].numpy()
        errs.append(check_logits(out, fwd64, cid, f"{mode}/forward", fwd32))
        worst[mode] = max(errs)
    explicit = max(worst[m] for m in ("persistent_simple", "graph"))
    ratio = f"{worst['persistent'] / explicit:.2f}" if "persistent" in worst and explicit > 0 else "n/a"
    print(f"{cid}: worst rel. error vs fp64 {worst}; ring / explicit-LN = {ratio}")
    model.set_decode_mode(modes[0])


@pytest.mark.parametrize("case", CASES, ids=_case_id)
def test_tokens_vs_engine_regime_oracle(case):
    """A short generate (typical acceptance, the reference's defaults) in the width's default decode mode: tokens and
    accept lengths equal the fp32 engine-regime oracle decoding from the engine's encoder states."""
    model, cfg, sd, pcm = _model(case)
    model.set_decode_mode(_modes(case[0])[0])
    out = model.generate_from_pcm(pcm, **_KW)[0].tolist()
    tr = model.last_trace
    enc = model.encoder_output()
    prompt = M.init_tokens(cfg, None)
    gp = M.gen_params(cfg, prompt, None, _KW["max_length"])
    ref = M.medusa_greedy_search(W.RefWeights(sd), cfg, enc, prompt, gp, "engine")
    assert tr.sequences == ref.sequences, _case_id(case)
    assert tr.accept_lengths == ref.accept_lengths, _case_id(case)
    assert out == M.strip_output(ref.sequences, len(prompt), gp)


@pytest.mark.parametrize("d", [512, 768, 1024])
def test_partial_grids_at_base_small_medium_widths(d):
    """decode_ctas 8 and 37 at d = 512 / 768 / 1024 (8 / 12 / 16 heads: fewer CTAs than heads, and a grid that does
    not divide by the head count, in the cross-attention chunking and every stage's row split): same tokens and
    accept lengths as the full grid."""
    model, cfg, sd, pcm = _model((d, "default", "base_head", 0))
    model.set_decode_mode("persistent")
    want = model.generate_from_pcm(pcm, **_KW)[0].tolist()
    want_acc = model.last_trace.accept_lengths
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    try:
        for ctas in (8, 37):
            model.set_option("decode_ctas", ctas)
            assert model.generate_from_pcm(pcm, **_KW)[0].tolist() == want, (d, ctas)
            assert model.last_trace.accept_lengths == want_acc, (d, ctas)
            assert model.last_trace.launches_decode == model.last_trace.iterations
    finally:
        model.set_option("decode_ctas", n_sm)


@pytest.mark.parametrize("d", RING_WIDTHS + (FALLBACK_WIDTH,))
def test_encoder_states_every_width(d):
    """All 1500 rows of the encoder output against the engine-regime oracle (5e-3; the wgmma GEMM tiles each width
    picks: N = 3d for QKV, 4d for FC1).  The mma.sync GEMM (enc_gemm = 0) agrees with the default to the same level;
    128 x 128 tiles only (enc_gemm = 2) give the same bits as the width's default tile choice."""
    model, cfg, sd, pcm = _model((d, "default", "base_head", 0))
    model.generate_from_pcm(pcm, max_iters=1, **_KW)
    enc = model.encoder_output()
    w = W.RefWeights(sd)
    ref = W.encoder_forward(w, cfg, torch.from_numpy(W.log_mel_spectrogram(pcm)), "engine")
    assert np.isfinite(enc.numpy()).all()
    assert float((enc - ref).abs().max()) < 5e-3, d
    try:
        model.set_option("enc_gemm", 0)
        model.generate_from_pcm(pcm, max_iters=1, **_KW)
        enc_mma = model.encoder_output()
        model.set_option("enc_gemm", 2)
        model.generate_from_pcm(pcm, max_iters=1, **_KW)
        enc_128 = model.encoder_output()
    finally:
        model.set_option("enc_gemm", 1)
    assert float((enc_mma - enc).abs().max()) < 5e-3, d
    assert torch.equal(enc_128, enc), d


def test_fallback_width_decodes_without_the_ring_kernel():
    """d = 640 is valid (multiple of 128, 64-wide heads) but has no ring-kernel instantiation: the engine starts in
    graph mode and refuses the persistent mode instead of ignoring the request."""
    from whisper_medusa_b200 import _lib
    from whisper_medusa_b200.model import EngineError

    model, cfg, sd, pcm = _model((FALLBACK_WIDTH, "default", "base_head", 0))
    lib = _lib.load()
    model.set_decode_mode("persistent_simple")
    model.set_decode_mode("graph")
    with pytest.raises(EngineError):
        model.set_decode_mode("persistent")
    assert lib.wm_set_decode_mode(model._handle, -1) == 0          # -1 queries the mode: still graph
    from whisper_medusa_b200 import WhisperMedusaModel

    fresh = WhisperMedusaModel(cfg, sd).to("cuda:0")
    try:
        assert lib.wm_set_decode_mode(fresh._handle, -1) == 0      # graph from construction
    finally:
        fresh.close()


def _pass_logits(model, pcm):
    model.generate_from_pcm(pcm, max_iters=2, **_KW)
    return [model.last_logits(i).numpy().copy() for i in (0, 1)]


def test_folded_layernorms_follow_every_weight_binding():
    """The ring kernel's folded LayerNorm vectors (c = W gamma, b' = b + W beta) are derived at every binding.
    (i) An engine adopting another's device weights (to(weights_from=)) gives the same bits.  (ii) Loading weights B
    through the C ABI into a handle that held weights A gives the bits of a fresh engine built with B."""
    from whisper_medusa_b200 import WhisperMedusaModel, _lib
    from whisper_medusa_b200.weights import pack_blob

    d = 512
    cfg = width_config(d, heads=4)
    sd_a = synthetic_state_dict(cfg, seed=11)
    sd_b = synthetic_state_dict(cfg, seed=12, activation_profile="gamma_spread")
    pcm = synthetic_audio(5.0, stream_id=11)
    lib = _lib.load()
    a = WhisperMedusaModel(cfg, sd_a).to("cuda:0")
    adopted = WhisperMedusaModel(cfg, sd_a).to("cuda:0", weights_from=a)
    fresh_b = WhisperMedusaModel(cfg, sd_b).to("cuda:0")
    reloaded = WhisperMedusaModel(cfg, sd_a).to("cuda:0")
    try:
        la = _pass_logits(a, pcm)
        for x, y in zip(la, _pass_logits(adopted, pcm)):
            assert np.array_equal(x, y)
        before = _pass_logits(reloaded, pcm)
        blob = pack_blob(reloaded._handle, cfg, sd_b)
        nbytes = lib.wm_weights_nbytes(reloaded._handle)
        assert lib.wm_load_weights(reloaded._handle, C.c_void_p(blob.data_ptr()), nbytes) == 0
        want = _pass_logits(fresh_b, pcm)
        got = _pass_logits(reloaded, pcm)
        for x, y, z in zip(got, want, before):
            assert np.array_equal(x, y)
            assert rel_err(x, z) > 1e-2          # weights B really decode differently from A
    finally:
        for m in (adopted, a, fresh_b, reloaded):
            m.close()
