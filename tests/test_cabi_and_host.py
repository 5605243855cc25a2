"""C-ABI surface and host-side logic that need no GPU: the library loads, exports every symbol the
header declares, defines a consistent weight layout, and the Python host mirrors the reference's
error behaviour."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

from _wm_paths import ROOT
from whisper_medusa_b200 import MedusaConfig, WhisperMedusaModel, _lib
from whisper_medusa_b200.model import EngineError
from whisper_medusa_b200.synthetic import preset_config, synthetic_state_dict
from whisper_medusa_b200.weights import engine_tensors, pack_blob


def test_library_exports_every_declared_symbol(engine_lib):
    hdr = open(os.path.join(ROOT, "include", "whisper_medusa_b200.h")).read()
    declared = set(re.findall(r"\b(wm_[a-z_]+)\s*\(", hdr))
    assert declared, "no declarations parsed"
    assert declared == set(_lib.SYMBOLS), declared ^ set(_lib.SYMBOLS)
    for name in declared:
        assert hasattr(engine_lib, name)


def test_strerror_and_null_handles(engine_lib):
    assert engine_lib.wm_strerror(0) == b"ok"
    assert b"CUDA" in engine_lib.wm_strerror(-2)
    assert engine_lib.wm_destroy(None) == 0
    assert engine_lib.wm_tensor_count(None) == 0


def test_encoder_gemm_tile_choice(engine_lib):
    """Host logic of csrc/enc_gemm_tc.cu::pick_tile: the tile with the fewest operand bytes, K (BM + BN) 2 per tile x
    ceil(tiles / n_sm) tiles, on the busiest SM.  whisper-large-v2 (M = 1500 positions) on the 132 SMs of an H100: the
    wide GEMMs run in at most two rounds of tiles."""
    def tile(M, N, K, fp16_out, n_sm=132):
        out = (C.c_int32 * 3)()
        assert engine_lib.wm_enc_gemm_tile(M, N, K, int(fp16_out), n_sm, out) == 0
        return tuple(out)

    assert tile(1500, 3840, 1280, True) == (128, 192, 5)     # QKV: 12 x 20 tiles
    assert tile(1500, 5120, 1280, True) == (256, 128, 4)     # FC1: 6 x 40
    assert tile(1500, 2560, 1280, True) == (256, 128, 4)     # cross-K/V: 6 x 20
    assert tile(1500, 1280, 1280, False) == (128, 128, 6)    # O-proj: 12 x 10, one CTA per SM, deep ring
    assert tile(1500, 1280, 5120, False) == (128, 128, 6)    # FC2
    assert tile(3000, 1280, 256, True) == (256, 128, 4)      # conv1 as an implicit GEMM: 12 x 10
    # tiny (d = 384): 128 x 128 tiles fit one round where N <= 1408; FC1 (N = 1536) takes 128 x 192 instead
    assert tile(1500, 1152, 384, True)[:2] == (128, 128)
    assert tile(1500, 1536, 384, True)[:2] == (128, 192)
    # the cost model itself: no candidate may beat the chosen tile
    for (M, N, K) in [(1500, 3840, 1280), (1500, 5120, 1280), (1500, 2560, 1280), (1500, 2048, 512), (700, 3072, 768)]:
        bm, bn, _ = tile(M, N, K, True)
        cost = lambda a, b: -(-((-(-M // a)) * (N // b)) // 132) * (a + b)
        for a, b in [(128, 128), (256, 128), (128, 192)]:
            if N % b == 0:
                assert cost(bm, bn) <= cost(a, b), (M, N, K, bm, bn, a, b)
    assert engine_lib.wm_enc_gemm_tile(1500, 1000, 1280, 1, 132, (C.c_int32 * 3)()) != 0   # N must be a multiple of 128
    assert engine_lib.wm_enc_gemm_tile(1500, 1280, 1280, 1, 132, None) != 0


def _layout_handle(lib, cfg):
    m = WhisperMedusaModel(cfg, None)
    h = C.c_void_p()
    wc = m._wm_config()
    assert lib.wm_create(C.byref(wc), -1, C.byref(h)) == 0
    return h


@pytest.mark.parametrize("preset,htype", [("micro", "base_head"), ("micro", "medusa_block"), ("tiny.en", "base_head")])
def test_weight_layout_and_packing(engine_lib, preset, htype):
    cfg = preset_config(preset, heads=4, heads_type=htype)
    sd = synthetic_state_dict(cfg, seed=0)
    h = _layout_handle(engine_lib, cfg)
    try:
        blob = pack_blob(h, cfg, sd)
        assert blob.numel() == engine_lib.wm_weights_nbytes(h)
        # non-overlapping, 256-byte aligned tensors
        spans = []
        off, nb, dt = C.c_size_t(), C.c_size_t(), C.c_int32()
        for i in range(engine_lib.wm_tensor_count(h)):
            name = engine_lib.wm_tensor_name(h, i)
            assert engine_lib.wm_tensor_info(h, name, C.byref(off), C.byref(nb), C.byref(dt)) == 0
            assert off.value % 256 == 0
            spans.append((off.value, off.value + nb.value))
        spans.sort()
        assert all(a[1] <= b[0] for a, b in zip(spans, spans[1:]))
        # q/k/v fused without touching the values, k bias zero, conv weights re-ordered [out][kw*in]
        t = dict(engine_tensors(cfg, sd))
        d = cfg.d_model
        assert torch.equal(t["dec.0.qkv_w"][:d], sd["whisper_model.model.decoder.layers.0.self_attn.q_proj.weight"])
        assert torch.equal(t["dec.0.qkv_w"][2 * d:], sd["whisper_model.model.decoder.layers.0.self_attn.v_proj.weight"])
        assert torch.count_nonzero(t["dec.0.qkv_b"][d:2 * d]) == 0
        c1 = sd["whisper_model.model.encoder.conv1.weight"]
        assert torch.equal(t["enc.conv1_w"][:, 80:160], c1[:, :, 1])
        assert torch.count_nonzero(t["enc.conv1_w"][:, 240:]) == 0
        nh = cfg.medusa_num_heads + (0 if cfg.is_block else 1)
        assert t["heads_w"].shape == (nh * d, d)
        assert engine_lib.wm_tensor_info(h, b"nope", None, None, None) == -1
    finally:
        engine_lib.wm_destroy(h)


def test_create_takes_39_decoder_layers_and_a_block_layer_but_not_40_layers(engine_lib):
    """The per-layer tables hold 40 decoder layers (WM_MAX_DEC_LAYERS): 39 layers plus the Medusa-Block layer fill them;
    40 layers leave no record for a Block layer and are rejected for either head type."""
    for htype in ("base_head", "medusa_block"):
        h = _layout_handle(engine_lib, preset_config("micro", heads=4, heads_type=htype, decoder_layers=39))
        engine_lib.wm_destroy(h)
        wc = WhisperMedusaModel(preset_config("micro", heads=4, heads_type=htype, decoder_layers=40), None)._wm_config()
        h = C.c_void_p()
        assert engine_lib.wm_create(C.byref(wc), -1, C.byref(h)) == -1, htype
        assert b"decoder layers" in engine_lib.wm_last_error(h)
        engine_lib.wm_destroy(h)


def test_create_rejects_unsupported_shapes(engine_lib):
    cfg = preset_config("micro", heads=4)
    m = WhisperMedusaModel(cfg, None)
    for field, value in (("d_model", 100), ("n_mels", 128), ("medusa_num_heads", 16), ("max_source_positions", 750)):
        wc = m._wm_config()
        setattr(wc, field, value)
        h = C.c_void_p()
        assert engine_lib.wm_create(C.byref(wc), -1, C.byref(h)) == -1
        assert engine_lib.wm_last_error(h)
        engine_lib.wm_destroy(h)


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU behaviour")
def test_no_silent_cpu_fallback(engine_lib):
    """Without a GPU the engine must fail loudly, not compute on the host."""
    cfg = preset_config("micro", heads=4)
    model = WhisperMedusaModel(cfg, synthetic_state_dict(cfg, seed=0))
    with pytest.raises(EngineError):
        model.generate(torch.zeros(1, 80, 3000))
    with pytest.raises(EngineError):
        model.to("cpu")
    with pytest.raises(EngineError):
        model.to("cuda:0")


def test_product_code_never_imports_the_oracle():
    pkg = os.path.join(ROOT, "whisper_medusa_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle|import_module\(.oracle|oracle/_ref", src, re.M), f


def test_config_roundtrip_and_reference_errors(tmp_path):
    cfg = preset_config("micro", heads=4, heads_type="medusa_block")
    cfg.save_pretrained(str(tmp_path))
    back = MedusaConfig.from_pretrained(str(tmp_path))
    assert back.to_dict() == cfg.to_dict()
    with pytest.raises(ValueError):
        MedusaConfig(medusa_heads_type="nope", whisper_model_name="synthetic/whisper-micro")   # model.py:224-228
    with pytest.raises(OSError):
        WhisperMedusaModel.from_pretrained(str(tmp_path / "missing"))
    # branching choices construct (the tree is checked against the engine's limits when the engine is created)
    WhisperMedusaModel(MedusaConfig(medusa_num_heads=2, medusa_hidden_size=128, medusa_choices=[1, 2, 2],
                                    whisper_model_name="synthetic/whisper-micro"), None)
    with pytest.raises(ValueError):
        WhisperMedusaModel(MedusaConfig(medusa_num_heads=2, medusa_hidden_size=128, medusa_choices=[1, 2],
                                        whisper_model_name="synthetic/whisper-micro"), None)


def test_checkpoint_directory_roundtrip(tmp_path):
    """from_pretrained reads the reference's checkpoint layout (config.json + model.safetensors with
    tied proj_out omitted, SURVEY.md 3.1)."""
    cfg = preset_config("micro", heads=4)
    sd = synthetic_state_dict(cfg, seed=3)
    WhisperMedusaModel(cfg, sd).save_pretrained(str(tmp_path))
    m = WhisperMedusaModel.from_pretrained(str(tmp_path))
    assert m.config.to_dict() == cfg.to_dict()
    assert set(m._state_dict) == set(sd)
    for k in sd:
        assert torch.equal(m._state_dict[k], sd[k]), k
    assert m.generation_config.posterior_threshold == 0.09 and m.generation_config.posterior_alpha == 0.3
    assert m.get_medusa_choice() == [1] * 5


def test_checkpoint_directory_variants(tmp_path):
    """The layouts HF's save_pretrained produces for the reference's checkpoints (SURVEY.md 8(f) rank 2): sharded
    safetensors with an index, the legacy pytorch_model.bin, fp32 tensors.  The packed engine tensors must be
    the same whichever container the weights came in."""
    import json

    from safetensors.torch import save_file

    from whisper_medusa_b200.weights import engine_tensors

    cfg = preset_config("micro", heads=4)
    sd = synthetic_state_dict(cfg, seed=5)
    ref = {k: v.clone() for k, v in engine_tensors(cfg, sd)}
    tied = "whisper_model.proj_out.weight"

    def check(path):
        m = WhisperMedusaModel.from_pretrained(str(path))
        got = dict(engine_tensors(m.config, m._state_dict))
        assert set(got) == set(ref)
        for k in ref:
            assert got[k].dtype == ref[k].dtype and torch.equal(got[k], ref[k]), k

    # (1) two safetensors shards + index, tensors stored in fp32 (the reference's default dtype)
    d1 = tmp_path / "sharded"
    d1.mkdir()
    cfg.save_pretrained(str(d1))
    keys = sorted(k for k in sd if k != tied)
    half = len(keys) // 2
    wm = {}
    for i, part in enumerate((keys[:half], keys[half:])):
        fn = f"model-{i + 1:05d}-of-00002.safetensors"
        save_file({k: sd[k].to(torch.float32).contiguous() for k in part}, str(d1 / fn))
        wm.update({k: fn for k in part})
    (d1 / "model.safetensors.index.json").write_text(json.dumps({"metadata": {}, "weight_map": wm}))
    check(d1)
    # (2) legacy pytorch_model.bin
    d2 = tmp_path / "bin"
    d2.mkdir()
    cfg.save_pretrained(str(d2))
    torch.save({k: v for k, v in sd.items() if k != tied}, str(d2 / "pytorch_model.bin"))
    check(d2)
    # (3) nothing to load
    d3 = tmp_path / "empty"
    d3.mkdir()
    cfg.save_pretrained(str(d3))
    with pytest.raises(OSError):
        WhisperMedusaModel.from_pretrained(str(d3))


def test_generate_argument_errors_match_reference():
    cfg = preset_config("micro", heads=4)
    m = WhisperMedusaModel(cfg, None)
    m._handle = C.c_void_p(1)  # pretend an engine exists: the argument checks come first
    try:
        with pytest.raises(AssertionError):
            m.generate(torch.zeros(2, 80, 3000))                          # model.py:1451
        with pytest.raises(NotImplementedError):
            m.generate(torch.zeros(1, 80, 3000), return_timestamps=True)  # model.py:1171
        with pytest.raises(NotImplementedError):
            m.generate(torch.zeros(1, 80, 3000), no_speech_threshold=0.6)  # model.py:1201
        with pytest.raises(NotImplementedError):
            m.generate(torch.zeros(1, 80, 6000))                          # model.py:1213
        with pytest.raises(Exception):
            m.generate(torch.zeros(1, 80, 3000), num_beams=4)             # model.py:1153
        # options the reference takes but this path cannot honour fail loudly instead of being dropped (ADVICE r1)
        with pytest.raises(NotImplementedError):
            m.generate(torch.zeros(1, 80, 3000), temperature=0.4)         # -> do_sample (model.py:1878-1881): no sampling branch
        with pytest.raises(NotImplementedError):
            m.generate(torch.zeros(1, 80, 3000), temperature=(0.0, 0.2, 0.4))
        with pytest.raises(NotImplementedError):
            m.generate(torch.zeros(1, 80, 3000), do_sample=True)
        with pytest.raises(NotImplementedError):
            m.generate(torch.zeros(1, 80, 3000), repetition_penalty=1.2)
    finally:
        m._handle = None
    big = WhisperMedusaModel(preset_config("large-v2", heads=10), None)
    assert big._init_tokens("en", None) == [50258, 50259, 50359, 50363]   # SURVEY.md 3.2 step 4
    assert big._init_tokens("german", "translate") == [50258, 50261, 50358, 50363]   # names as HF accepts them
    assert big._init_tokens("<|ja|>", None)[1] == 50266
    with pytest.raises(ValueError):
        big._init_tokens("klingon", None)
    small = WhisperMedusaModel(preset_config("tiny.en", heads=4), None)
    assert small._init_tokens(None, None) == [50257, 50362]
    assert WhisperMedusaModel._strip([1, 2, 5, 6, 9, 9], 2, 9, 9) == [5, 6]


def test_language_tables_match_the_installed_transformers():
    """The embedded Whisper language table (config.py) against transformers' own (tokenization_whisper.py)."""
    tw = pytest.importorskip("transformers.models.whisper.tokenization_whisper")
    from whisper_medusa_b200.config import WHISPER_LANGUAGE_CODES, WHISPER_LANGUAGE_NAMES, WHISPER_PRESETS, language_token

    codes = list(tw.LANGUAGES.keys())
    assert codes[:99] == WHISPER_LANGUAGE_CODES          # (large-v3 appended "yue"; v2 checkpoints have 99)
    assert {k: v for k, v in tw.TO_LANGUAGE_CODE.items()} == WHISPER_LANGUAGE_NAMES
    lang = WHISPER_PRESETS["openai/whisper-large-v2"]["lang_to_id"]
    assert lang["<|en|>"] == 50259 and lang["<|su|>"] == 50357 and len(lang) == 99
    assert language_token("English") == "<|en|>" and language_token("fr") == "<|fr|>"


def test_preset_suppress_lists_have_the_public_shape():
    """The suppress-token lists of the built-in presets are reproduced from the public openai/whisper generation configs
    (no hub access here to diff them; a checkpoint's own generation_config.json takes precedence): at least their shape is
    pinned -- 88 ids for the multilingual models, 90 for the English-only ones, strictly increasing, inside the vocabulary,
    containing the special-token block (sot ... notimestamps excluded, translate / transcribe / startoflm / startofprev /
    nospeech included) and never the EOS token."""
    from whisper_medusa_b200.config import WHISPER_PRESETS

    for name, n in (("openai/whisper-large-v2", 88), ("openai/whisper-tiny.en", 90)):
        p = WHISPER_PRESETS[name]
        s = p["suppress_tokens"]
        assert len(s) == n and s == sorted(set(s)) and 0 < s[0] and s[-1] < p["vocab_size"]
        assert p["eos_token_id"] not in s and p["no_timestamps_token_id"] not in s
        assert p["decoder_start_token_id"] in s            # <|startoftranscript|> may not be re-emitted
        assert p["begin_suppress_tokens"] == [220, p["eos_token_id"]]
    big = WHISPER_PRESETS["openai/whisper-large-v2"]
    assert {big["task_to_id"]["translate"], big["task_to_id"]["transcribe"]} <= set(big["suppress_tokens"])
