"""Host logic of the wgmma encoder GEMM's tile choice (csrc/enc_gemm_tc.cu: pick_tile) against the instantiated kernels.

Every kernel WM_TC_ALL compiles must be one that the widths the GPU encoder tests run (test_gpu_encoder_numerics.py,
group A, with enc_gemm 1 and 2) actually launch, so no compiled kernel ships untested."""
import ctypes as C
import os
import re

from _wm_paths import ROOT

# wm_enc_gemm_tile(M, N = 128 j, fp16_out = 1, n_sm) for j = 1..80 as returned before the never-winning 128 x 256
# candidate was removed.  a = 128 x 128 (6 stages), b = 128 x 128 (3 stages), w = 256 x 128, c = 128 x 192.
CODES = {"a": (128, 128, 6), "b": (128, 128, 3), "w": (256, 128, 4), "c": (128, 192, 5)}
FROZEN_F16 = {
    (1500, 132): "aaaaaaaaaaacwwcwwwwwwwbcbbcbbcbbcwwwwwwwwwwwcwwcwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwww",
    (1500, 114): "aaaaaaaaawwcwwwwwwwbcbbcbbcbwwwwwwwwwwcwwcwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwww",
    (1500, 66): "aaaaacwwwwwcbbcbwwwwwwwcwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwcwwwwwwwwwwwwwwwwwwwwwww",
    (1500, 33): "aacwwcaawwwcwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwww",
    (3000, 132): "aaaaacwwwwwcbbcbwwwwwwwcwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwcwwwwwwwwwwwwwwwwwwwwwww",
    (3000, 114): "aaaawcwwwaacbbwwwwwwcwwwwwwwwwwwwwwwwwwwwwwwwwwcwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwww",
    (3000, 66): "aacwwcaawwwcwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwww",
    (3000, 33): "awcawcwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwww",
}

WIDTHS = tuple(range(128, 1281, 128))
GROUP_A = [(d, 4 * d) for d in (128, 384, 512, 640, 768, 1024, 1280)] + [(768, 768)]


def _tile(lib, M, N, K, fp16_out, n_sm):
    out = (C.c_int32 * 3)()
    assert lib.wm_enc_gemm_tile(M, N, K, int(fp16_out), n_sm, out) == 0
    return tuple(out)


def _gemms(d, f):
    """(epilogue, M, N) of every encoder GEMM at width d, FFN f (engine.cu: run_encoder)."""
    return [("ENC_EPI_BIAS_GELU_F16", 3000, d),       # conv1, implicit GEMM over 3000 frames
            ("ENC_EPI_BIAS_GELU_POS_F32", 1500, d),   # conv2 + positions
            ("ENC_EPI_BIAS_F16", 1500, 3 * d),        # QKV
            ("ENC_EPI_BIAS_RES_F32", 1500, d),        # O-proj
            ("ENC_EPI_BIAS_GELU_F16", 1500, f),       # FC1
            ("ENC_EPI_BIAS_RES_F32", 1500, d),        # FC2
            ("ENC_EPI_BIAS_F16", 1500, 2 * d)]        # cross-K/V of every decoder layer


def test_tile_choice_is_unchanged_over_the_whole_grid(engine_lib):
    """Every width d = 128...1280, FFN ratio 1-8, M = 1500 and 3000, on 132 / 114 / 66 / 33 SMs: the same tile as before
    the 128 x 256 candidate and the fp32-output 3-stage kernels were removed."""
    for (M, n_sm), row in FROZEN_F16.items():
        for d in WIDTHS:
            for N in {d, 2 * d, 3 * d} | {r * d for r in range(1, 9)}:
                assert _tile(engine_lib, M, N, d, True, n_sm) == CODES[row[N // 128 - 1]], (M, N, n_sm)
            # the fp32 read-modify-write epilogues (N = d): always one CTA per SM with the deep ring
            assert _tile(engine_lib, M, d, 4 * d, False, n_sm) == (128, 128, 6), (M, d, n_sm)


def _instantiations():
    """(epilogue, BM, BN, STAGES) of every kernel WM_TC_ALL instantiates, read from the source."""
    src = open(os.path.join(ROOT, "whisper_medusa_b200", "csrc", "enc_gemm_tc.cu")).read()
    body = src[src.index("#define WM_TC_F16_TILES"):src.index("cudaError_t enc_gemm_tc_configure")]
    f16_def, all_def = body.split("#define WM_TC_ALL")
    f16_tiles = [tuple(map(int, t)) for t in re.findall(r"X\(EPI, (\d+), (\d+), (\d+)\)", f16_def)]
    out = {(epi,) + t for epi in re.findall(r"WM_TC_F16_TILES\(X, (\w+)\)", all_def) for t in f16_tiles}
    out |= {(epi, int(a), int(b), int(c)) for epi, a, b, c in re.findall(r"X\((ENC_EPI_\w+), (\d+), (\d+), (\d+)\)", all_def)}
    return out


def test_every_instantiated_kernel_is_launched_by_the_tested_widths(engine_lib):
    """Derive (epilogue, tile, stages) of every encoder GEMM at the widths of the GPU encoder tests (group A) on 132 SMs,
    with the per-GEMM tile choice (enc_gemm = 1) and with 128 x 128 tiles only (enc_gemm = 2, which keeps the 3-stage
    ring for fp16 outputs wider than 1536 columns): the set equals the instantiation list exactly."""
    used = set()
    for d, f in GROUP_A:
        for epi, M, N in _gemms(d, f):
            f16 = epi in ("ENC_EPI_BIAS_F16", "ENC_EPI_BIAS_GELU_F16")
            used.add((epi,) + _tile(engine_lib, M, N, d, f16, 132))
            used.add((epi, 128, 128, 3 if (f16 and N > 1536) else 6))
    inst = _instantiations()
    assert len(inst) == 10
    assert used == inst, (sorted(used - inst), sorted(inst - used))
