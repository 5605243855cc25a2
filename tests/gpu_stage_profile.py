"""Per-stage timeline of the persistent decode kernel (device %globaltimer, CTA 0 and last CTA).

    python tests/gpu_stage_profile.py [--preset large-v2] [--heads 10] [--block] [--iters 6] [--tc] [--temp0] [--seed 0]

Prints, per stage type, the mean body time and barrier-wait time over the layers of the LAST
iteration, and the critical-path sum.  Used to decide what to optimise next.
"""
from __future__ import annotations

import ctypes as C
import os
import sys
from collections import OrderedDict

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from whisper_medusa_b200 import WhisperMedusaModel, _lib  # noqa: E402
from whisper_medusa_b200.synthetic import preset_config, synthetic_audio, synthetic_state_dict  # noqa: E402

STAGES = ["EMBED", "QKV", "SELF_ATTN", "OPROJ", "CROSS_Q", "CROSS_ATTN", "CROSS_O", "FC1", "FC2", "FINAL_LN",
          "COPY_HIDDEN", "TAIL_SEED", "HEADS", "VOCAB", "SELECT1", "SELECT2", "SELECT_FIN", "ACCEPT", "KV_COMPACT"]
MODES = ["A", "B", "TAIL"]


def arg(name, default):
    return type(default)(sys.argv[sys.argv.index(name) + 1]) if name in sys.argv else default


def main():
    preset = arg("--preset", "large-v2")
    heads = arg("--heads", 10)
    iters = arg("--iters", 6)
    cfg = preset_config(preset, heads=heads, heads_type="medusa_block" if "--block" in sys.argv else "base_head")
    for _ in range(arg("--warm-instances", 0)):   # earlier engine instances in the same process (then closed)
        w = WhisperMedusaModel(cfg, synthetic_state_dict(cfg, seed=arg("--seed", 0))).to("cuda:0")
        w.set_decode_mode("persistent")
        w.generate_from_pcm(synthetic_audio(5.0), language="en" if cfg.is_multilingual else None, max_iters=iters,
                            **({"medusa_temperature": 0.0} if "--temp0" in sys.argv else {}))
        print(f"warm instance: decode {w.last_trace.ms_decode:.3f} ms for {w.last_trace.iterations} iterations")
        if "--keep" not in sys.argv:
            w.close()
    model = WhisperMedusaModel(cfg, synthetic_state_dict(cfg, seed=arg("--seed", 0))).to("cuda:0")
    gen_kw = {"medusa_temperature": 0.0} if "--temp0" in sys.argv else {}
    model.set_decode_mode("persistent")
    if "--ctas" in sys.argv:      # decode grid smaller than the GPU (one partition of a StreamGroup)
        model.set_option("decode_ctas", arg("--ctas", 37))
    if "--tc" in sys.argv:
        model.set_option("enc_gemm", 1)
    if "--no-prof" in sys.argv:     # plain run (e.g. under ncu): no timeline
        pcm = synthetic_audio(30.0 if preset == "large-v2" else 5.0)
        model.generate_from_pcm(pcm, language="en" if cfg.is_multilingual else None, max_iters=iters, **gen_kw)
        print(f"decode {model.last_trace.ms_decode:.3f} ms for {model.last_trace.iterations} iterations")
        model.close()
        return
    model.set_option("profile", 1)
    pcm = synthetic_audio(30.0 if preset == "large-v2" else 5.0)
    lang = "en" if cfg.is_multilingual else None
    model.generate_from_pcm(pcm, language=lang, max_iters=iters, **gen_kw)
    tr = model.last_trace
    lib = _lib.load()
    cap = 4096
    buf = (C.c_int64 * (cap * 24))()
    n = C.c_int32(0)
    rc = lib.wm_get_stage_profile(model._handle, buf, cap, C.byref(n))
    assert rc == 0, lib.wm_last_error(model._handle)
    rows = np.frombuffer(buf, dtype=np.int64)[: n.value * 24].reshape(-1, 24)
    # probes in timeline order (see include/whisper_medusa_b200.h)
    order = [7, 8, 9, 10, 3, 13, 4, 5, 6, 14, 15, 1, 2]
    names = ["desc", "x-land", "ln-stat", "split", "staged", "pre-w", "w-ok", "mma", "epi", "units", "fn-end", "body", "barrier"]
    agg = OrderedDict()
    agg2 = OrderedDict()
    gemm = {"QKV", "OPROJ", "CROSS_Q", "CROSS_O", "FC1", "FC2", "HEADS", "VOCAB"}
    for row in rows:
        st, mode, layer, bN, wN = row[:5]
        raw = row[5:21]
        if STAGES[st] not in gemm:
            b = agg2.setdefault((STAGES[st], MODES[mode]), np.zeros(12))
            b[0] += 1
            for k in range(8):
                b[1 + k] += max(raw[3 + k], 0)
            b[9] += max(raw[1], 0); b[10] += max(raw[2], 0); b[11] += raw[11]
        a = agg.setdefault((STAGES[st], MODES[mode]), np.zeros(3 + len(order) + 2))
        a[0] += 1; a[1] += bN; a[2] += wN
        for k, idx in enumerate(order):
            a[3 + k] += max(raw[idx], 0)
        a[3 + len(order)] += raw[11]; a[4 + len(order)] += raw[12]
    print(f"{preset} K={heads} iterations={tr.iterations} decode {tr.ms_decode:.3f} ms "
          f"({tr.ms_decode / max(1, tr.iterations):.3f} ms/iter), encoder {tr.ms_encoder:.3f} ms, mel {tr.ms_mel:.3f} ms")
    print(f"{'stage':<12}{'mode':<5}{'n':>3}" + "".join(f"{x:>8}" for x in names) + f"{'bodyN':>8}{'waitN':>8}  w@begin w@wait"
          "   (us; CTA 0 offsets from stage begin; bodyN/waitN = last CTA)")
    tot = 0.0
    for (st, mode), a in agg.items():
        cnt = a[0]
        tot += a[3 + len(order) - 1] / 1e3
        print(f"{st:<12}{mode:<5}{int(cnt):>3}" + "".join(f"{a[3 + k] / cnt / 1e3:>8.2f}" for k in range(len(order)))
              + f"{a[1] / cnt / 1e3:>8.2f}{a[2] / cnt / 1e3:>8.2f}  {a[3 + len(order)] / cnt / 1e3:>7.2f} {a[4 + len(order)] / cnt / 1e3:>6.2f}")
    print(f"sum over stages of the last iteration (CTA 0): {tot / 1e3:.3f} ms")
    # raw probe offsets (us from stage begin, CTA 0) of the non-GEMM stages: pr[3..10], body end, barrier end
    print("raw probes of the attention / select stages (us): p3 p4 p5 p6 p7 p8 p9 p10 | body barrier | flag11")
    for (st, mode), a in agg2.items():
        cnt = a[0]
        print(f"{st:<12}{mode:<5}{int(cnt):>3}" + "".join(f"{a[1 + k] / cnt / 1e3:>8.2f}" for k in range(8))
              + f" |{a[9] / cnt / 1e3:>8.2f}{a[10] / cnt / 1e3:>8.2f} |{a[11] / cnt / 1e3:>6.2f}")
    model.close()


if __name__ == "__main__":
    main()
