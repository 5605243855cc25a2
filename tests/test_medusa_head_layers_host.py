"""Medusa heads of several ResBlocks (``medusa_num_layers`` > 1) on the host, no GPU needed.

* Weight layout: ``heads_w`` / ``heads_b`` are layer-major, ``[L][heads][d][d]`` and ``[L][heads][d]``; every engine
  tensor agrees with ``wm_tensor_info`` at L = 1 ... WM_MAX_HEAD_LAYERS, and at L = 1 the packed blob is byte for
  byte the single-layer layout (digests of blobs packed by the single-layer engine).
* ``wm_create`` and ``engine_tensors`` refuse L = 0 and L = WM_MAX_HEAD_LAYERS + 1.
* The weight ring of the persistent decode kernel replayed with one head stage per layer (tail, and verify for
  base_head).
* The oracle reproduces every stream of ``tests/golden/ref_loop_head_layers.npz``, which
  ``oracle/make_head_layers_golden.py`` froze from the reference's own loop; where the reference checkout is present,
  the oracle is held to that loop directly as well.
"""
import ctypes as C
import hashlib
import os

import numpy as np
import pytest
import torch

from _wm_paths import GOLDEN
from oracle import make_head_layers_golden as G
from oracle import ref_harness as R
from whisper_medusa_b200 import _lib
from whisper_medusa_b200.model import WhisperMedusaModel
from whisper_medusa_b200.synthetic import preset_config, synthetic_state_dict
from whisper_medusa_b200.weights import engine_tensors, pack_blob

FIX = os.path.join(GOLDEN, "ref_loop_head_layers.npz")
MAXL = _lib.WM_MAX_HEAD_LAYERS

# (preset, heads type, K) -> (wm_weights_nbytes, sha256 of pack_blob) of checkpoint seed 5 with one layer per head, as
# the engine packed it before heads could have more than one layer
SINGLE_LAYER_BLOBS = {
    ("micro", "base_head", 4): (2801152, "3668f82f6f5be1262c66bc24690ee94002ac9b756e0aafa0e6a3901296313df2"),
    ("micro", "medusa_block", 4): (3169792, "b3694215fef12719847391ecb99006832d573544deaafd78f41f156e3b2874f3"),
    ("tiny.en", "base_head", 10): (80401920, "05cdee8b89c76e24fcd4678068da3f23a5283234496b08e051ad0b5118acaa7a"),
}


def _create(lib, cfg):
    h = C.c_void_p()
    wc = WhisperMedusaModel(cfg, None)._wm_config()
    rc = lib.wm_create(C.byref(wc), -1, C.byref(h))
    return rc, h


@pytest.mark.parametrize("key", list(SINGLE_LAYER_BLOBS), ids=lambda k: f"{k[0]}-{k[1]}-k{k[2]}")
def test_single_layer_blob_is_unchanged(engine_lib, key):
    preset, htype, k = key
    cfg = preset_config(preset, heads=k, heads_type=htype)
    rc, h = _create(engine_lib, cfg)
    assert rc == 0
    try:
        blob = pack_blob(h, cfg, synthetic_state_dict(cfg, seed=5))
        nbytes, digest = SINGLE_LAYER_BLOBS[key]
        assert engine_lib.wm_weights_nbytes(h) == nbytes
        assert hashlib.sha256(blob.numpy().tobytes()).hexdigest() == digest
    finally:
        engine_lib.wm_destroy(h)


@pytest.mark.parametrize("htype", ["base_head", "medusa_block"])
@pytest.mark.parametrize("layers", list(range(1, MAXL + 1)))
def test_layer_major_heads_layout(engine_lib, layers, htype):
    cfg = preset_config("micro", heads=4, heads_type=htype, head_layers=layers)
    sd = synthetic_state_dict(cfg, seed=1)
    rc, h = _create(engine_lib, cfg)
    assert rc == 0
    try:
        blob = pack_blob(h, cfg, sd)   # (checks every tensor's byte count against wm_tensor_info)
        d, nh = cfg.d_model, cfg.medusa_num_heads + (0 if cfg.is_block else 1)
        off, nb, dt = C.c_size_t(), C.c_size_t(), C.c_int32()
        assert engine_lib.wm_tensor_info(h, b"heads_w", C.byref(off), C.byref(nb), C.byref(dt)) == 0
        assert (nb.value, dt.value) == (layers * nh * d * d * 2, 0)
        w = blob[off.value: off.value + nb.value].view(torch.float16).reshape(layers, nh, d, d)
        assert engine_lib.wm_tensor_info(h, b"heads_b", C.byref(off), C.byref(nb), C.byref(dt)) == 0
        assert (nb.value, dt.value) == (layers * nh * d * 4, 1)
        b = blob[off.value: off.value + nb.value].view(torch.float32).reshape(layers, nh, d)
        for l in range(layers):
            for i in range(nh):
                assert torch.equal(w[l, i], sd[f"medusa_heads.{i}.{l}.linear.weight"].to(torch.float16)), (l, i)
                assert torch.equal(b[l, i], sd[f"medusa_heads.{i}.{l}.linear.bias"].to(torch.float32)), (l, i)
        # every other tensor is the one of the single-layer checkpoint drawn from the same seed
        if layers > 1:
            one = dict(engine_tensors(preset_config("micro", heads=4, heads_type=htype), sd))
            for name, t in engine_tensors(cfg, sd):
                if not name.startswith("heads_"):
                    assert torch.equal(t, one[name]), name
    finally:
        engine_lib.wm_destroy(h)


@pytest.mark.parametrize("layers", [0, MAXL + 1])
def test_out_of_range_layer_counts_are_refused(engine_lib, layers):
    cfg = preset_config("micro", heads=4, head_layers=layers)
    rc, h = _create(engine_lib, cfg)
    try:
        assert rc == -1
        assert b"medusa_num_layers" in engine_lib.wm_last_error(h)
    finally:
        engine_lib.wm_destroy(h)
    with pytest.raises(NotImplementedError, match="medusa_num_layers"):
        dict(engine_tensors(cfg, synthetic_state_dict(preset_config("micro", heads=4), seed=0)))


def test_hidden_size_other_than_d_model_stays_refused():
    cfg = preset_config("micro", heads=4, head_layers=2)
    sd = synthetic_state_dict(cfg, seed=0)
    cfg.medusa_hidden_size = cfg.d_model // 2
    with pytest.raises(ValueError, match="medusa_hidden_size"):
        dict(engine_tensors(cfg, sd))


def _ring(lib, d, grid, layers, block=0, K=10, n_tree=11, n_layers=2):
    bad = C.c_int32(-1)
    first = (C.c_int32 * 4)()
    assert lib.wm_ring_schedule_check_head_layers(d, n_layers, block, K, n_tree, grid, layers, C.byref(bad), first) == 0
    assert bad.value == 0, (d, grid, layers, block, n_tree, "first mismatch {kv_len, L, need_a, cta}:", list(first))


@pytest.mark.parametrize("layers", [2, 3, MAXL])
@pytest.mark.parametrize("d", [128, 512, 1280])
def test_ring_schedule_with_head_layers(engine_lib, d, layers):
    """Chains (K = 10, Linear and Block) on the full grid and on 33 CTAs, and a 16-node tree on 37 CTAs: the chunks
    the producer warp streams for every head stage are the slots the compute warps take."""
    for grid in (132, 33):
        _ring(engine_lib, d, grid, layers)
        _ring(engine_lib, d, grid, layers, block=1)
    _ring(engine_lib, d, 37, layers, K=3, n_tree=16)


def test_ring_schedule_rejects_out_of_range_layer_counts(engine_lib):
    bad = C.c_int32(-1)
    first = (C.c_int32 * 4)()
    for layers in (0, MAXL + 1):
        assert engine_lib.wm_ring_schedule_check_head_layers(512, 2, 0, 10, 11, 132, layers, C.byref(bad), first) != 0


def _fixture_streams():
    return [(g, s) for g, spec in G.GROUPS.items() for s in range(spec[5])]


@pytest.mark.parametrize("group", list(G.GROUPS))
def test_oracle_reproduces_frozen_reference_streams(group):
    fx = np.load(FIX)
    torch.set_num_threads(min(8, os.cpu_count() or 1))
    for s in range(G.GROUPS[group][5]):
        seq, acc = G.oracle_stream(group, s)
        assert seq == fx[f"{group}/{s}/sequences"].tolist(), (group, s)
        assert acc == fx[f"{group}/{s}/accept"].tolist(), (group, s)


def test_fixture_covers_layers_head_types_and_trees():
    fx = np.load(FIX)
    assert sorted(fx.files) == sorted(f"{g}/{s}/{k}" for g, s in _fixture_streams() for k in ("sequences", "accept"))
    layers = {(spec[2], spec[3], spec[4] is not None) for spec in G.GROUPS.values()}
    for htype in ("base_head", "medusa_block"):
        assert {l for t, l, _ in layers if t == htype} >= {2, 3}, htype
        assert any(t == htype and tree for t, _, tree in layers), htype
    # the heads' proposals get accepted: the extra layers are on the path of the decisions
    assert max(int(fx[f"{g}/{s}/accept"].max()) for g, s in _fixture_streams()) >= 2


@pytest.mark.skipif(not R.available(), reason="needs the reference checkout")
@pytest.mark.parametrize("group", ["micro_lin_l2_t1", "micro_blk_l3_k10", "micro_tree122_l2_t1"])
def test_oracle_equals_reference_loop(group):
    torch.set_num_threads(min(8, os.cpu_count() or 1))
    assert G.reference_stream(group, 0) == G.oracle_stream(group, 0)
