"""GPU parity tests: the CUDA engine, called through the reference-facing Python host and the C
ABI, against (i) the committed golden fixtures and (ii) the CPU oracle run on the same seeded
inputs.  Bars: token ids and accept lengths bit-exact; log-mel within 5e-5; encoder states within
5e-3 of the engine-regime oracle; decode-path logits within DECODE_LOGIT_BAR of the fp64 engine-regime oracle decoding
from the engine's encoder states (tests/_decode_ref.py)."""
import os

import numpy as np
import pytest
import torch

from _decode_ref import check_logits, decode_logits, forward_logits
from _decode_ref import rel_err as _rel_err
from _wm_paths import GOLDEN
from oracle import medusa_ref as M
from oracle import whisper_ref as W
from whisper_medusa_b200.synthetic import preset_config, synthetic_audio, synthetic_state_dict

pytestmark = pytest.mark.gpu

SMALL = ["micro_linear_k4", "micro_block_k10", "micro_linear_k4_t0", "tiny_linear_k4", "tiny_block_k4"]


def _load(name):
    g = np.load(os.path.join(GOLDEN, name + ".npz"))
    seed, stream, max_len, heads, is_block = [int(v) for v in g["meta"]]
    preset = {"micro": "micro", "tiny": "tiny.en", "large": "large-v2"}[name.split("_")[0]]
    cfg = preset_config(preset, heads=heads, heads_type="medusa_block" if is_block else "base_head")
    pen = None if g["penalty"][0] < 0 else (int(g["penalty"][0]), float(g["penalty"][1]))
    kw = dict(language="en" if cfg.is_multilingual else None, max_length=max_len,
              exponential_decay_length_penalty=pen, medusa_temperature=float(g["temperature"]))
    if "posterior" in g.files:      # acceptance constants other than the defaults (mixed-acceptance large-v2 fixtures)
        kw.update(posterior_alpha=float(g["posterior"][0]), posterior_threshold=float(g["posterior"][1]))
    return g, cfg, seed, stream, kw


_MODELS = {}


def _model(name):
    from whisper_medusa_b200 import WhisperMedusaModel

    if name not in _MODELS:
        for m in _MODELS.values():
            m[0].close()
        _MODELS.clear()
        g, cfg, seed, stream, kw = _load(name)
        sd = synthetic_state_dict(cfg, seed=seed)
        model = WhisperMedusaModel(cfg, sd).to("cuda:0")
        _MODELS[name] = (model, sd)
    return _MODELS[name]


@pytest.mark.parametrize("mode", ["graph", "persistent_simple", "persistent"])
@pytest.mark.parametrize("name", SMALL)
def test_tokens_bit_exact_vs_golden_and_oracle(name, mode):
    g, cfg, seed, stream, kw = _load(name)
    model, sd = _model(name)
    model.set_decode_mode(mode)
    pcm = synthetic_audio(float(g["audio_seconds"]), stream_id=stream)
    out = model.generate_from_pcm(pcm, **kw)[0].tolist()
    assert out == g["tokens"].tolist()
    assert model.last_trace.accept_lengths == g["accept_lengths"].tolist()
    assert model.last_trace.sequences == g["sequences"].tolist()
    # the oracle itself, run here on the same inputs (micro only: seconds on the host cores)
    if name.startswith("micro"):
        w = W.RefWeights(sd)
        mel = torch.from_numpy(W.log_mel_spectrogram(pcm))
        ref, tr = M.generate(w, cfg, mel, language=kw["language"], regime="engine", max_length=kw["max_length"],
                             exponential_decay_length_penalty=kw["exponential_decay_length_penalty"],
                             temperature=kw["medusa_temperature"])
        assert out == ref and model.last_trace.accept_lengths == tr.accept_lengths
    # same clip through the reference's entry point: generate(input_features) with CPU-made features
    feats = torch.from_numpy(W.log_mel_spectrogram(pcm))[None]
    assert model.generate(feats, **kw)[0].tolist() == out


@pytest.mark.parametrize("mode", ["graph", "persistent"])
@pytest.mark.parametrize("name", ["micro_linear_k4", "micro_block_k10", "tiny_linear_k4", "tiny_block_k4"])
def test_mel_encoder_logits_close(name, mode):
    """Tolerances (DESIGN.md section 2):
    * log-mel: 5e-5 abs;
    * encoder states: 5e-3 abs vs the engine-regime oracle (values reach ~5).  The encoder rounds every
      GEMM operand to fp16; an fp32 accumulation-order difference of 1e-7 flips ~0.2 % of those
      roundings by one fp16 ulp (1e-3 relative), which no restatement can reproduce bit-for-bit;
    * logits of the DECODE path: DECODE_LOGIT_BAR (relative) against the fp64 engine-regime oracle decoding from the
      SAME encoder states (the engine's own), which isolates the path that runs every iteration;
    * end-to-end logits vs the committed golden (oracle encoder + oracle decoder): 5e-3 / 2e-2 (fp32)."""
    g, cfg, seed, stream, kw = _load(name)
    model, sd = _model(name)
    model.set_decode_mode(mode)
    pcm = synthetic_audio(float(g["audio_seconds"]), stream_id=stream)
    model.generate_from_pcm(pcm, max_iters=1, **kw)
    enc = model.encoder_output()
    tr = decode_logits(cfg, sd, enc, kw, 2)
    for it in (1, 2):
        model.generate_from_pcm(pcm, max_iters=it, **kw)
        assert model.last_trace.iterations == it
        for ab, which, ref in (("A", 0, tr.passA_logits[it - 1]), ("B", 1, tr.passB_logits[it - 1])):
            lg = model.last_logits(which).numpy()
            check_logits(lg, ref.numpy(), f"{name}/{mode}", f"pass{ab}{it}")
            assert _rel_err(lg[:, ::97], g[f"logits{ab}{it - 1}_strided"]) < 5e-3, (ab, it)
            assert _rel_err(lg[:, ::97], g[f"logits{ab}{it - 1}_strided_fp32"]) < 2e-2, (ab, it)
            assert lg.argmax(1).tolist() == g[f"logits{ab}{it - 1}_topi"][:, 0].tolist()
    mel = model.mel().numpy()
    assert np.abs(mel[:, ::8] - g["mel_sample"]).max() < 5e-5
    enc = enc.numpy()
    assert np.abs(enc[::50] - g["enc_sample"]).max() < 5e-3
    assert np.abs(enc[::50] - g["enc_sample_fp32"]).max() < 3e-2


@pytest.mark.parametrize("name", ["micro_linear_k4", "tiny_linear_k4"])
def test_encoder_gemm_implementations_agree(name):
    """The encoder GEMMs run on the wgmma / TMA kernel by default; the mma.sync kernel
    (option enc_gemm = 0) is the cross-check: same fp16 operands, fp32 accumulation in a different
    order => the outputs agree to the fp16-rounding-flip level (DESIGN.md section 2) and both stay
    within the oracle tolerance; the tokens are identical."""
    g, cfg, seed, stream, kw = _load(name)
    model, sd = _model(name)
    pcm = synthetic_audio(float(g["audio_seconds"]), stream_id=stream)
    outs, toks = [], []
    for impl in (1, 0):
        model.set_option("enc_gemm", impl)
        toks.append(model.generate_from_pcm(pcm, **kw).cpu().numpy())
        outs.append(model.encoder_output().numpy())
    model.set_option("enc_gemm", 1)
    assert np.abs(outs[0] - outs[1]).max() < 5e-3
    for o in outs:
        assert np.abs(o[::50] - g["enc_sample"]).max() < 5e-3
    assert toks[0].tolist() == toks[1].tolist()
    # plain stream-ordered launches instead of programmatic dependent launch: same bits
    model.set_option("enc_pdl", 0)
    model.generate_from_pcm(pcm, **kw)
    plain = model.encoder_output().numpy()
    model.set_option("enc_pdl", 1)
    assert np.array_equal(plain, outs[0])


@pytest.mark.parametrize("name", ["micro_linear_k4", "tiny_linear_k4"])
def test_encoder_attention_implementations_agree(name):
    """Encoder self-attention runs on the wgmma / TMA kernel by default (enc_attn_tc.cu); the mma.sync flash
    attention (option enc_attn = 0) is the cross-check: same 64-key blocking and fp16 rounding of P, fp32 accumulation
    in a different order => encoder states agree to the fp16-rounding-flip level, both within the oracle tolerance, and
    the tokens are identical."""
    g, cfg, seed, stream, kw = _load(name)
    model, sd = _model(name)
    pcm = synthetic_audio(float(g["audio_seconds"]), stream_id=stream)
    outs, toks = [], []
    for impl in (1, 0):
        model.set_option("enc_attn", impl)
        toks.append(model.generate_from_pcm(pcm, **kw).cpu().numpy())
        outs.append(model.encoder_output().numpy())
    model.set_option("enc_attn", 1)
    assert np.abs(outs[0] - outs[1]).max() < 5e-3
    for o in outs:
        assert np.abs(o[::50] - g["enc_sample"]).max() < 5e-3
    assert toks[0].tolist() == toks[1].tolist() == [g["tokens"].tolist()]


def test_frontend_edge_cases():
    """Empty, very short and maximum-length clips (the extractor pads / truncates to 30 s)."""
    g, cfg, seed, stream, kw = _load("micro_linear_k4")
    model, sd = _model("micro_linear_k4")
    for pcm in (np.zeros(0, np.float32), synthetic_audio(0.05), synthetic_audio(30.0, stream_id=5)):
        model.generate_from_pcm(pcm, max_iters=1, **kw)
        assert np.abs(model.mel().numpy() - W.log_mel_spectrogram(pcm)).max() < 5e-5
    with pytest.raises(NotImplementedError):
        model.generate_from_pcm(np.zeros(480001, np.float32), **kw)      # long-form, model.py:1213


def test_reruns_are_deterministic_and_streams_independent():
    g, cfg, seed, stream, kw = _load("micro_linear_k4")
    model, sd = _model("micro_linear_k4")
    a = synthetic_audio(5.0, stream_id=0)
    b = synthetic_audio(5.0, stream_id=7)
    model.set_decode_mode("persistent")
    ra1 = model.generate_from_pcm(a, **kw)[0].tolist()
    rb = model.generate_from_pcm(b, **kw)[0].tolist()
    ra2 = model.generate_from_pcm(a, **kw)[0].tolist()
    assert ra1 == ra2 == g["tokens"].tolist() and rb != ra1
    # a second engine on the same device gives the same answer (handles are independent)
    from whisper_medusa_b200 import WhisperMedusaModel

    other = WhisperMedusaModel(cfg, sd).to("cuda:0")
    assert other.generate_from_pcm(b, **kw)[0].tolist() == rb
    other.close()


def test_length_properties_large_budget():
    """Size-independent invariants (SURVEY.md 3.3) at the full decode budget: tokens per iteration
    = accept+1 (or 2 when accept = 0); the loop stops once L + K >= max_length; prompt preserved."""
    g, cfg, seed, stream, kw = _load("tiny_block_k4")
    model, sd = _model("tiny_block_k4")
    kw = dict(kw, max_length=448)
    model.generate_from_pcm(synthetic_audio(5.0, stream_id=2), **kw)
    tr = model.last_trace
    n_prompt = 2
    assert tr.sequences[:n_prompt] == [50257, 50362]
    assert len(tr.sequences) - n_prompt == sum(a + 1 if a else 2 for a in tr.accept_lengths)
    assert len(tr.sequences) + cfg.medusa_num_heads >= 448 or cfg.eos_token_id in tr.sequences
    assert len(tr.sequences) <= 448 + cfg.medusa_num_heads + 1


@pytest.mark.skipif(not os.path.isfile(os.path.join(GOLDEN, "large_linear_k10.npz")), reason="fixture missing")
@pytest.mark.parametrize("mode", ["persistent", "persistent_simple", "graph"])
def test_large_v2_tokens_bit_exact_vs_golden(mode):
    """BASELINE.json configs[1]: whisper-large-v2 + 10 Medusa-Linear heads, 30 s clip."""
    g, cfg, seed, stream, kw = _load("large_linear_k10")
    model, sd = _model("large_linear_k10")
    model.set_decode_mode(mode)
    pcm = synthetic_audio(float(g["audio_seconds"]), stream_id=stream)
    out = model.generate_from_pcm(pcm, **kw)[0].tolist()
    assert out == g["tokens"].tolist()
    assert model.last_trace.accept_lengths == g["accept_lengths"].tolist()
    if mode == "persistent":
        model.generate_from_pcm(pcm, max_iters=1, **kw)
        enc = model.encoder_output()
        assert np.abs(enc.numpy()[::50] - g["enc_sample"]).max() < 5e-3
        # decode path in isolation: oracle decoding one iteration from the engine's encoder states
        tr = decode_logits(cfg, sd, enc, kw, 1)
        for ab, which, ref in (("A", 0, tr.passA_logits[0]), ("B", 1, tr.passB_logits[0])):
            lg = model.last_logits(which).numpy()
            check_logits(lg, ref.numpy(), "large_linear_k10/persistent", f"pass{ab}1")
            assert _rel_err(lg[:, ::97], g[f"logits{ab}0_strided"]) < 5e-3, ab
        # wgmma GEMM tile shapes: at d = 1280 the wide outputs run as 128 x 192 / 256 x 128 tiles; option enc_gemm = 2
        # forces 128 x 128 tiles.  Same operands, same K order per output element => identical encoder states.
        model.set_option("enc_gemm", 2)
        model.generate_from_pcm(pcm, max_iters=1, **kw)
        enc128 = model.encoder_output()
        model.set_option("enc_gemm", 1)
        assert torch.equal(enc128, enc)
        # programmatic dependent launch (default): every encoder kernel may start while its predecessor drains and does
        # its set-up and first weight loads before the grid-dependency wait; plain stream-ordered launches (enc_pdl = 0)
        # must give the same bits, run after run
        model.set_option("enc_pdl", 0)
        model.generate_from_pcm(pcm, max_iters=1, **kw)
        enc_plain = model.encoder_output()
        model.set_option("enc_pdl", 1)
        assert torch.equal(enc_plain, enc)
        for _ in range(3):
            model.generate_from_pcm(pcm, max_iters=1, **kw)
            assert torch.equal(model.encoder_output(), enc)


@pytest.mark.skipif(not os.path.isfile(os.path.join(GOLDEN, "large_block_k10.npz")), reason="fixture missing")
@pytest.mark.parametrize("mode", ["persistent", "graph"])
def test_large_v2_block_heads_tokens_bit_exact_vs_golden(mode):
    """whisper-large-v2 + the Medusa-Block head type (one extra decoder layer feeding 10 heads; reference
    model.py:1285-1301), short token budget."""
    g, cfg, seed, stream, kw = _load("large_block_k10")
    model, sd = _model("large_block_k10")
    model.set_decode_mode(mode)
    pcm = synthetic_audio(float(g["audio_seconds"]), stream_id=stream)
    out = model.generate_from_pcm(pcm, **kw)[0].tolist()
    assert out == g["tokens"].tolist()
    assert model.last_trace.accept_lengths == g["accept_lengths"].tolist()


# ---------------------------------------------------------------------------------------------------------
# round 2: mixed acceptance at large-v2, K sweep, the reference's own loop, default mode, forward, f1 / f2
# ---------------------------------------------------------------------------------------------------------
LARGE_MIXED = ["large_linear_k10_mixed", "large_linear_k10_a0mix", "large_linear_k6_mixed", "large_linear_k4_mixed",
               "large_linear_k2_mixed", "large_block_k10_mixed"]


@pytest.mark.parametrize("name", LARGE_MIXED)
def test_large_v2_mixed_acceptance_tokens_bit_exact(name):
    """whisper-large-v2, K in {2, 4, 6, 10}, accept lengths mixed (posterior_alpha = 100: 1 and 4; = 230: 0..4 with
    two-sweep iterations interleaved), the eval script's length penalty (140, 1.01) and an EOS stop on the K = 10 case:
    the carry / KV-keep / sweep-elision logic at d = 1280, in the default (persistent ring) mode and in graph mode."""
    if not os.path.isfile(os.path.join(GOLDEN, name + ".npz")):
        pytest.skip("fixture missing")
    g, cfg, seed, stream, kw = _load(name)
    model, sd = _model(name)
    pcm = synthetic_audio(float(g["audio_seconds"]), stream_id=stream)
    for mode in (("persistent", "graph") if name == "large_linear_k10_mixed" else ("persistent",)):
        model.set_decode_mode(mode)
        out = model.generate_from_pcm(pcm, **kw)[0].tolist()
        assert model.last_trace.accept_lengths == g["accept_lengths"].tolist(), mode
        assert out == g["tokens"].tolist(), mode
        assert model.last_trace.sequences == g["sequences"].tolist(), mode
    acc = g["accept_lengths"].tolist()
    assert len(set(acc)) >= (2 if cfg.medusa_num_heads > 2 else 1)   # (Block fixture: accept 0 / 1 / 2 => carry + block tail)
    if name == "large_linear_k10_mixed":
        assert cfg.eos_token_id in g["sequences"].tolist()[4:], "fixture must end by EOS"
        assert len(g["sequences"]) > 144 + 4, "the length penalty must have been active"


def test_engine_vs_the_reference_loop_on_unselected_streams():
    """The CUDA engine against outputs of the REFERENCE'S OWN loop code (tests/golden/ref_loop_streams.npz, made by
    oracle/make_ref_golden.py from the reference checkout): 82 streams whose seeds were not selected for decision margins.
    The engine computes with fp16 K/V caches and fp16 hi/lo operands, the reference in fp32, so a decision that sits
    within ~1e-3 of a tie can flip (and changes the rest of that stream).  Asserted: a stream either matches the
    reference bit-for-bit or matches the oracle run in the engine's rounding regime on the same inputs (i.e. the
    difference is the numeric regime, not the algorithm); and the mismatch RATE against the reference stays small.
    The oracle's encoder sums in another order than the engine's tensor-core tiles, so a decode decision within that
    rounding noise of a tie can also separate the engine from the oracle's own encoder states: such a stream must then
    match the oracle decoding from the engine's encoder states (as in the branching-tree and prefill tests)."""
    from oracle import make_ref_golden as G
    from whisper_medusa_b200 import WhisperMedusaModel

    fx = np.load(os.path.join(GOLDEN, "ref_loop_streams.npz"))
    total = mism = 0
    report = []
    for group, spec in G.GROUPS.items():
        for s in range(spec[3]):
            cfg, sd, pcm, max_len, pen, temp, alpha, thr = G.stream_inputs(group, s)
            m = WhisperMedusaModel(cfg, sd).to("cuda:0")
            m.generate_from_pcm(pcm, max_length=max_len, exponential_decay_length_penalty=pen, medusa_temperature=temp,
                                posterior_alpha=alpha, posterior_threshold=thr)
            seq, acc = m.last_trace.sequences, m.last_trace.accept_lengths
            enc_engine = m.encoder_output()
            m.close()
            total += 1
            if seq == fx[f"{group}/{s}/sequences"].tolist() and acc == fx[f"{group}/{s}/accept"].tolist():
                continue
            mism += 1
            w = W.RefWeights(sd)
            mel = torch.from_numpy(W.log_mel_spectrogram(pcm))
            enc = W.encoder_forward(w, cfg, mel, "engine")
            prompt = M.init_tokens(cfg, None)
            gp = M.gen_params(cfg, prompt, pen, max_len, temperature=temp, posterior_alpha=alpha, posterior_threshold=thr)
            tr = M.medusa_greedy_search(w, cfg, enc, prompt, gp, "engine")
            same_encoder = seq == tr.sequences and acc == tr.accept_lengths
            if not same_encoder:
                tr = M.medusa_greedy_search(w, cfg, enc_engine, prompt, gp, "engine")
            report.append((group, s, "oracle" if same_encoder else "oracle from the engine's encoder states"))
            assert seq == tr.sequences and acc == tr.accept_lengths, (group, s)
    print(f"engine vs reference loop: {mism} of {total} streams differ (numeric-regime flips: {report})")
    assert total >= 80 and mism <= total // 10, (mism, total, report)


def test_default_mode_is_the_persistent_ring_kernel():
    """from construction, without set_decode_mode: one launch per speculative iteration (GPUTEST launch lists must
    show dec_iteration_ring_kernel for the drop-in API, not the stage-kernel graphs)."""
    from whisper_medusa_b200 import WhisperMedusaModel

    g, cfg, seed, stream, kw = _load("tiny_linear_k4")
    m = WhisperMedusaModel(cfg, synthetic_state_dict(cfg, seed=seed)).to("cuda:0")
    out = m.generate_from_pcm(synthetic_audio(float(g["audio_seconds"]), stream_id=stream), **kw)[0].tolist()
    assert out == g["tokens"].tolist()
    assert m.last_trace.launches_decode == m.last_trace.iterations
    m.close()


def test_device_features_and_forward_logits():
    """generate(input_features) with a CUDA tensor (device-to-device, no host bounce) == host features; forward() returns
    the stacked head logits [K+1, 1, T, V] of reference model.py:1223-1347, within DECODE_LOGIT_BAR of the fp64 oracle."""
    g, cfg, seed, stream, kw = _load("micro_linear_k4")
    model, sd = _model("micro_linear_k4")
    pcm = synthetic_audio(float(g["audio_seconds"]), stream_id=stream)
    feats = torch.from_numpy(W.log_mel_spectrogram(pcm))[None]
    a = model.generate(feats, **kw)[0].tolist()
    b = model.generate(feats.to("cuda:0"), **kw)[0].tolist()
    assert a == b == g["tokens"].tolist()
    ids = [cfg.decoder_start_token_id, cfg.no_timestamps_token_id, 17, 33, 64]
    out = model.forward(input_features=feats.to("cuda:0"), decoder_input_ids=torch.tensor([ids])).logits.cpu()
    assert tuple(out.shape) == (cfg.medusa_num_heads + 1, 1, len(ids), cfg.vocab_size)
    ref = forward_logits(cfg, sd, model.encoder_output(), ids)                     # [K+1, T, V]
    check_logits(out[:, 0].numpy(), ref.numpy(), "micro_linear_k4", "forward")
    assert tuple(model.forward(decoder_input_ids=torch.tensor([ids]), disable_medusa=True).logits.shape) == (1, 1, len(ids), cfg.vocab_size)
    with pytest.raises(NotImplementedError):
        model.generate(feats, temperature=0.7, **kw)
    with pytest.raises(NotImplementedError):
        model.generate(feats, some_unknown_option=1, **kw)


def test_language_detection_multilingual():
    """generate(language=None) on a multilingual model runs the detection pass (HF generation_whisper.py:1559-1566):
    argmax of the base logits of <|startoftranscript|> over the language tokens."""
    from whisper_medusa_b200 import WhisperMedusaModel

    lang = {"<|en|>": 300, "<|de|>": 301, "<|fr|>": 302, "<|ja|>": 303}
    cfg = preset_config("micro", heads=4, is_multilingual=True, lang_to_id=lang,
                        task_to_id={"transcribe": 310, "translate": 311})
    sd = synthetic_state_dict(cfg, seed=21)
    m = WhisperMedusaModel(cfg, sd).to("cuda:0")
    pcm = synthetic_audio(5.0, stream_id=9)
    m.generate_from_pcm(pcm, language=None, max_length=40)
    w = W.RefWeights(sd)
    enc = m.encoder_output()
    cache = W.new_cache(cfg)
    hidden = W.decoder_forward(w, cfg, [cfg.decoder_start_token_id], [0], enc, cache, "engine")
    base = W.medusa_logits(w, cfg, hidden, enc, cache, True, "engine")[0, -1]
    ids = sorted(lang.values())
    want = ids[int(torch.argmax(base[torch.tensor(ids)]))]
    assert m.last_trace.sequences[1] == want
    assert m.last_trace.sequences[:4] == [cfg.decoder_start_token_id, want, 310, cfg.no_timestamps_token_id]
    explicit = m.generate_from_pcm(pcm, language="german", max_length=40)
    assert m.last_trace.sequences[1] == 301 and explicit.shape[0] == 1
    m.close()


def test_checkpoint_directory_and_eval_driver_on_gpu(tmp_path):
    """SURVEY 8(f) ranks 1-2 on the GPU path: save_pretrained -> from_pretrained(dir).to(cuda).generate == the directly
    constructed model; the evaluation driver (CSV -> wav -> generate -> WER/CER) runs end to end on synthetic wavs."""
    import wave

    from whisper_medusa_b200 import WhisperMedusaModel
    from whisper_medusa_b200 import eval as E

    g, cfg, seed, stream, kw = _load("micro_linear_k4")
    model, sd = _model("micro_linear_k4")
    pcm = synthetic_audio(float(g["audio_seconds"]), stream_id=stream)
    want = model.generate_from_pcm(pcm, **kw)[0].tolist()
    d = str(tmp_path / "ckpt")
    model.save_pretrained(d)
    m2 = WhisperMedusaModel.from_pretrained(d).to("cuda:0")
    assert m2.generate_from_pcm(pcm, **kw)[0].tolist() == want == g["tokens"].tolist()
    rows = []
    for i in range(3):
        p = str(tmp_path / f"clip{i}.wav")
        x = (synthetic_audio(2.0 + i, stream_id=30 + i) * 32767).astype(np.int16)
        with wave.open(p, "wb") as f:
            f.setnchannels(1); f.setsampwidth(2); f.setframerate(16000); f.writeframes(x.tobytes())
        rows.append({"audio": p, "sentence": "hello world", "language": ""})

    def transcribe(pcm_, lang_):
        ids = m2.generate_from_pcm(pcm_, max_length=40)[0].tolist()
        return " ".join(f"t{t}" for t in ids)

    wer, cer, table = E.evaluate_rows(rows, transcribe, default_language="en")
    assert len(table["prediction"]) == 3 and all(p for p in table["prediction"]) and wer > 0
    m2.close()


@pytest.mark.parametrize("ctas", [8, 37])
@pytest.mark.parametrize("name", ["micro_linear_k4", "micro_block_k10", "tiny_linear_k4", "tiny_block_k4"])
def test_partial_grids_give_the_same_tokens(name, ctas):
    """option "decode_ctas": the persistent kernel on a fraction of the SMs (every CTA then owns several attention items /
    more weight rows per stage) must produce the tokens of the full grid."""
    from whisper_medusa_b200 import WhisperMedusaModel

    g, cfg, seed, stream, kw = _load(name)
    m = WhisperMedusaModel(cfg, synthetic_state_dict(cfg, seed=seed)).to("cuda:0")
    m.set_option("decode_ctas", ctas)
    out = m.generate_from_pcm(synthetic_audio(float(g["audio_seconds"]), stream_id=stream), **kw)[0].tolist()
    assert out == g["tokens"].tolist() and m.last_trace.accept_lengths == g["accept_lengths"].tolist()
    assert m.last_trace.launches_decode == m.last_trace.iterations
    m.close()


def test_stream_group_equals_single_stream_runs():
    """SURVEY 8(f) rank 3 (the reference is batch 1, model.py:1451): S engines share one weight blob, each decodes on
    n_sm / S CTAs, S streams concurrently; every stream's tokens are those of its batch-1 run.  Also the batched
    generate(input_features[B, 80, 3000])."""
    from whisper_medusa_b200 import StreamGroup

    g, cfg, seed, stream, kw = _load("tiny_linear_k4")
    sd = synthetic_state_dict(cfg, seed=seed)
    single, _ = _model("tiny_linear_k4")
    clips = [synthetic_audio(5.0, stream_id=40 + i) for i in range(6)]
    want = [single.generate_from_pcm(c, **kw)[0].tolist() for c in clips]
    for S in (2, 4):
        grp = StreamGroup(cfg, sd, "cuda:0", n_streams=S)
        got = [o[0].tolist() for o in grp.generate_from_pcm(clips, **kw)]
        assert got == want, S
        feats = torch.stack([torch.from_numpy(W.log_mel_spectrogram(c)) for c in clips[:3]])
        assert [o[0].tolist() for o in grp.generate(feats, **kw)] == want[:3]
        # forward() (and with it language detection) works on a partial decode grid too
        ids = torch.tensor([[cfg.decoder_start_token_id, cfg.no_timestamps_token_id, 11]])
        lg_part = grp.models[-1].forward(input_features=feats[:1], decoder_input_ids=ids).logits.cpu().numpy()
        lg_full = single.forward(input_features=feats[:1], decoder_input_ids=ids).logits.cpu().numpy()
        ref = forward_logits(cfg, sd, single.encoder_output(), ids[0].tolist()).numpy()
        check_logits(lg_part[:, 0], ref, f"tiny_linear_k4/stream_group{S}", "forward, partial grid")
        check_logits(lg_full[:, 0], ref, f"tiny_linear_k4/stream_group{S}", "forward, full grid")
        assert all(t.launches_decode == t.iterations for t in grp.last_traces)
        grp.close()


@pytest.mark.parametrize("htype,heads,choices", [("base_head", 2, [1, 2, 2]), ("base_head", 3, [1, 3, 2, 1]),
                                                 ("medusa_block", 2, [1, 2, 2]), ("base_head", 4, [1, 2, 1, 2, 1])])
def test_branching_trees_both_attention_modes(htype, heads, choices):
    """SURVEY 8(f) rank 4.  Branching medusa_choices: per-head top-k candidates, the tree verified in one pass, best
    path by accept length / likelihood, surviving K/V rows gathered.  (i) tree_attention=False reproduces what the
    reference does (its medusa_attn_mask is never applied) -- against the oracle here and against the reference's own
    loop in test_engine_vs_the_reference_loop_on_unselected_streams; (ii) tree_attention=True (every node attends to
    its ancestors only; sweep elision as for the chain) against the oracle with the mask; (iii) the property that makes
    it speculative decoding proper: with exact-match acceptance the tree output IS the base model's greedy output, i.e.
    the same tokens as the top-1 chain at temperature 0."""
    from whisper_medusa_b200 import WhisperMedusaModel

    for seed in (2, 3):
        cfg = preset_config("micro", heads=heads, heads_type=htype)
        cfg.medusa_choices = list(choices)
        sd = synthetic_state_dict(cfg, seed=seed)
        pcm = synthetic_audio(5.0, stream_id=seed)
        m = WhisperMedusaModel(cfg, sd).to("cuda:0")
        w = W.RefWeights(sd)
        # the oracle decodes from the ENGINE's encoder states: the test is about the decode path (the streams are not
        # selected for decision margins, and encoder rounding noise would otherwise decide near-ties)
        m.generate_from_pcm(pcm, max_length=100, max_iters=1)
        enc = m.encoder_output()
        prompt = M.init_tokens(cfg, None)
        for temp in (1.0, 0.0):
            gp = M.gen_params(cfg, prompt, None, 100, temperature=temp)
            for tree_attn in (False, True):
                for mode in (("persistent", "graph") if (seed == 2 and temp == 1.0) else ("persistent",)):
                    m.set_decode_mode(mode)
                    m.generate_from_pcm(pcm, max_length=100, medusa_temperature=temp, tree_attention=tree_attn)
                    tr = M.medusa_greedy_search(w, cfg, enc, prompt, gp, "engine", tree_attention=tree_attn)
                    assert m.last_trace.accept_lengths == tr.accept_lengths, (seed, temp, tree_attn, mode)
                    assert m.last_trace.sequences == tr.sequences, (seed, temp, tree_attn, mode)
        m.set_decode_mode("persistent")
        m.generate_from_pcm(pcm, max_length=100, medusa_temperature=0.0, tree_attention=True)
        tree_greedy = m.last_trace.sequences
        m.close()
        if htype == "base_head":
            cfg1 = preset_config("micro", heads=heads, heads_type=htype)          # top-1 chain, same weights
            m1 = WhisperMedusaModel(cfg1, sd).to("cuda:0")
            m1.generate_from_pcm(pcm, max_length=100, medusa_temperature=0.0)
            chain_greedy = m1.last_trace.sequences
            m1.close()
            n = min(len(tree_greedy), len(chain_greedy))
            assert tree_greedy[:n] == chain_greedy[:n], seed


def test_tree_limits_are_reported():
    from whisper_medusa_b200 import WhisperMedusaModel

    cfg = preset_config("micro", heads=4)
    cfg.medusa_choices = [1, 6, 5, 4, 3]            # the example of the reference's docstring: 511 nodes
    with pytest.raises(NotImplementedError):
        WhisperMedusaModel(cfg, synthetic_state_dict(cfg, seed=0)).to("cuda:0")


@pytest.mark.parametrize("name", ["micro_linear_k4", "micro_block_k10", "tiny_linear_k4"])
def test_long_decoder_prompt_is_prefilled_in_chunks(name):
    """decoder_input_ids longer than the 16 rows of a stage tile (previous-text conditioning): the leading tokens are cached
    by prefill launches (sweep A over 16-token chunks).  Tokens / accept lengths against the oracle decoding from the
    engine's encoder states, in the three execution modes; prompt lengths around the chunk boundaries."""
    g, cfg, seed, stream, kw = _load(name)
    model, sd = _model(name)
    pcm = synthetic_audio(float(g["audio_seconds"]), stream_id=stream)
    w = W.RefWeights(sd)
    rng = np.random.default_rng(5)
    base = M.init_tokens(cfg, kw["language"])
    for n_extra, modes in ((13, ("persistent",)), (14, ("persistent", "graph", "persistent_simple")), (45, ("persistent", "graph"))):
        prompt = [int(t) for t in rng.integers(20, 400, size=n_extra)] + base      # 15 / 16 / 17 ... / 47+ tokens
        kw2 = dict(kw, max_length=min(int(kw["max_length"]) + n_extra, 200), decoder_input_ids=torch.tensor([prompt]))
        want = None
        for mode in modes:
            model.set_decode_mode(mode)
            out = model.generate_from_pcm(pcm, **kw2)[0].tolist()
            tr = model.last_trace
            if want is None:
                enc = model.encoder_output()
                gp = M.gen_params(cfg, prompt, kw["exponential_decay_length_penalty"], kw2["max_length"],
                                  temperature=kw["medusa_temperature"])
                ref = M.medusa_greedy_search(w, cfg, enc, prompt, gp, "engine")
                want = (ref.sequences, ref.accept_lengths)
            assert tr.sequences == want[0] and tr.accept_lengths == want[1], (n_extra, mode)
            assert tr.sequences[: len(prompt)] == prompt and out == M.strip_output(want[0], len(prompt), gp)
    model.set_decode_mode("persistent")
