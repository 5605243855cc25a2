"""Cost of Medusa heads with several ResBlocks (medusa_num_layers) on the benchmark clip.

    python tests/gpu_head_layers.py [--rounds 8] [--alpha 100] [--out FILE]

whisper-large-v2 + 10 Medusa-Linear heads with 1, 2 and 3 ResBlocks per head, the 30 s clip of bench.py (stream 0),
typical acceptance in the realistic regime (posterior_alpha = 100), the benchmark's length penalty.  Layer 0 of every
head is the benchmark checkpoint's (seed 0); the layers after it have zero weights and a bias of -200, so each is
x + SiLU(-200) = x exactly (expf(200) overflows to inf and SiLU returns -0).  The kernels do their full work on those
layers -- every weight byte is streamed, every product computed -- but all three arms decode the same tokens with the
same accept lengths (asserted), so their times per iteration compare the same decisions; with trained or random extra
layers the acceptance, and with it the share of iterations that need a sweep over uncached rows, would differ.  The
three engines live in one process and their calls alternate; each call reports the decode loop's device time (CUDA
events) per speculative iteration, and the medians over the rounds are compared.  Every extra layer adds one head stage
to the candidate pass and one to the verify pass, each with its own grid barrier; they stream (K+1) d^2 x 2 B and
d^2 x 2 B of weights.  Prints the card's name and power limit beside the numbers.
"""
from __future__ import annotations

import ctypes as C
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import bench  # noqa: E402
from gpu_scores import arg, card  # noqa: E402
from whisper_medusa_b200 import WhisperMedusaModel, _lib  # noqa: E402
from whisper_medusa_b200.synthetic import preset_config, synthetic_audio, synthetic_state_dict  # noqa: E402

LAYERS = (1, 2, 3)
ST_HEADS = 12   # StageId in csrc/decode.cu


def main():
    rounds, alpha, out_path = arg("--rounds", 8), arg("--alpha", 100.0), arg("--out", "")
    pcm = synthetic_audio(30.0, stream_id=0)
    kw = dict(language="en", exponential_decay_length_penalty=bench.PENALTY, posterior_alpha=alpha)
    base = synthetic_state_dict(preset_config("large-v2", heads=10), seed=0)
    models = {}
    for n in LAYERS:
        cfg = preset_config("large-v2", heads=10, head_layers=n)
        sd = dict(base)
        for i in range(cfg.medusa_num_heads + 1):
            w, b = base[f"medusa_heads.{i}.0.linear.weight"], base[f"medusa_heads.{i}.0.linear.bias"]
            for l in range(1, n):
                sd[f"medusa_heads.{i}.{l}.linear.weight"] = w.new_zeros(w.shape)
                sd[f"medusa_heads.{i}.{l}.linear.bias"] = b.new_full(b.shape, -200.0)
        models[n] = WhisperMedusaModel(cfg, sd).to("cuda:0")
        models[n].generate_from_pcm(pcm, **kw)
    d = models[1].config.d_model
    ms, runs = {n: [] for n in LAYERS}, {}
    for _ in range(rounds):
        for n in LAYERS:
            models[n].generate_from_pcm(pcm, **kw)
            tr = models[n].last_trace
            ms[n].append(tr.ms_decode / tr.iterations)
            runs.setdefault(n, (tr.sequences, tr.accept_lengths, tr.iterations))
            assert (tr.sequences, tr.accept_lengths, tr.iterations) == runs[n]
    assert all(runs[n] == runs[1] for n in LAYERS), "the extra layers changed the tokens: the arms differ in work"
    med = {n: float(np.median(ms[n])) for n in LAYERS}
    res = {"card": card(), "rounds": rounds, "posterior_alpha": alpha,
           "iterations": runs[1][2], "tokens": len(runs[1][0]),
           "ms_per_iter": ms, "median_ms_per_iter": med,
           "extra_us_per_iter_per_layer": {n: (med[n] - med[1]) * 1e3 / (n - 1) for n in LAYERS if n > 1},
           "extra_weight_mb_per_layer": (11 * d * d * 2 + d * d * 2) / 1e6}
    # the head stages' share of one iteration, from the ring kernel's stage timeline (option "profile", a run of its own
    # after the timed rounds): body + barrier wait of the last CTA, summed over the stages of the last iteration
    res["stage_timeline_us"] = {}
    for n in LAYERS:
        m = models[n]
        m.set_option("profile", 1)
        m.generate_from_pcm(pcm, max_iters=6, **kw)
        cap = 4096
        buf = (C.c_int64 * (cap * 24))()
        cnt = C.c_int32(0)
        assert _lib.load().wm_get_stage_profile(m._handle, buf, cap, C.byref(cnt)) == 0
        rows = np.frombuffer(buf, dtype=np.int64)[: cnt.value * 24].reshape(-1, 24)
        t = (rows[:, 3] + rows[:, 4]) / 1e3
        heads = rows[:, 0] == ST_HEADS
        res["stage_timeline_us"][n] = {"head_stages": int(heads.sum()), "heads_us": float(t[heads].sum()),
                                       "iteration_us": float(t.sum())}
        m.set_option("profile", 0)
    print(json.dumps(res))
    if out_path:
        os.makedirs(os.path.dirname(os.path.abspath(out_path)), exist_ok=True)
        with open(out_path, "w") as f:
            json.dump(res, f, indent=1)
    for m in models.values():
        m.close()


if __name__ == "__main__":
    main()
