"""Cost of token timestamps (generate(return_token_timestamps=True)) on the benchmark clip.

    python tests/gpu_token_timestamps.py [--rounds 8] [--alpha 100] [--out FILE]

whisper-large-v2 + 10 Medusa-Linear heads, the 30 s clip of bench.py (stream 0), typical acceptance in the realistic
regime (posterior_alpha = 100), the benchmark's length penalty, and a synthetic alignment table of 16 (layer, head)
pairs from the upper half of the decoder (real checkpoints list 6 to 30).  Calls with timestamps off and on alternate in
one process; each reports the decode loop's device time per speculative iteration (CUDA events).  The tokens of both
arms must be identical.  Then: the extraction kernels' device times (torch.profiler), and HF's host DTW
(_dynamic_time_warping, a CPU number) on the same matrix.  Prints the card's name and power limit beside the numbers.
"""
from __future__ import annotations

import json
import os
import re
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import bench  # noqa: E402
from gpu_scores import arg, card  # noqa: E402
from whisper_medusa_b200 import WhisperMedusaModel  # noqa: E402
from whisper_medusa_b200.synthetic import preset_config, synthetic_audio, synthetic_state_dict  # noqa: E402


def main():
    rounds, alpha, out_path = arg("--rounds", 8), arg("--alpha", 100.0), arg("--out", "")
    cfg = preset_config("large-v2", heads=10)
    model = WhisperMedusaModel(cfg, synthetic_state_dict(cfg, seed=0)).to("cuda:0")
    rng = np.random.default_rng(0)
    cells = rng.choice(16 * 20, 16, replace=False)
    model.generation_config.alignment_heads = [[16 + int(c) // 20, int(c) % 20] for c in sorted(cells)]
    pcm = synthetic_audio(30.0, stream_id=0)
    kw = dict(language="en", exponential_decay_length_penalty=bench.PENALTY, posterior_alpha=alpha)
    arms = {"off": {}, "on": dict(return_token_timestamps=True)}
    for extra in arms.values():                       # warm-up of both arms (buffers, modules)
        model.generate_from_pcm(pcm, **kw, **extra)
    ms, toks, wall = {k: [] for k in arms}, {}, {k: [] for k in arms}
    for _ in range(rounds):
        for name, extra in arms.items():
            t0 = time.perf_counter()
            model.generate_from_pcm(pcm, **kw, **extra)
            wall[name].append((time.perf_counter() - t0) * 1e3)
            tr = model.last_trace
            ms[name].append(tr.ms_decode / tr.iterations)
            toks.setdefault(name, (tr.sequences, tr.accept_lengths, tr.iterations))
            assert (tr.sequences, tr.accept_lengths, tr.iterations) == toks[name]
    assert toks["off"] == toks["on"], "timestamps changed the tokens"
    tr = model.last_trace
    P = len(model._init_tokens("en", None))
    n = P + tr.n_new_tokens
    res = {"card": card(), "iterations": toks["off"][2], "tokens": tr.n_new_tokens, "dtw_rows": n - 1 - P,
           "pairs": len(model.generation_config.alignment_heads), "rounds": rounds,
           "ms_per_iter_off": ms["off"], "ms_per_iter_on": ms["on"],
           "median_off": float(np.median(ms["off"])), "median_on": float(np.median(ms["on"])),
           "wall_ms_median_off": float(np.median(wall["off"])), "wall_ms_median_on": float(np.median(wall["on"]))}
    res["capture_cost_us_per_iter"] = (res["median_on"] - res["median_off"]) * 1e3
    # extraction kernels (torch.profiler, CUDA activities) on the last call's capture
    from torch.profiler import ProfilerActivity, profile

    model.last_timestamp_matrix(P, n, 3000)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            ts, mat, jumps = model.last_timestamp_matrix(P, n, 3000)
    per = {}
    for e in prof.events():
        k = re.search(r"ts_\w+_kernel", e.name) if e.device_type.name == "CUDA" else None
        if k:
            k = k.group(0)
            c, t = per.get(k, (0, 0.0))
            per[k] = (c + 1, t + e.device_time)
    res["extract_kernels_us"] = {k: t / c for k, (c, t) in per.items()}   # mean device time per launch
    res["extract_total_us"] = sum(res["extract_kernels_us"].values())
    # HF's host DTW on the same matrix (CPU)
    from transformers.models.whisper.generation_whisper import _dynamic_time_warping

    t0 = time.perf_counter()
    _dynamic_time_warping(-mat.double().numpy())
    res["hf_host_dtw_ms_cpu"] = (time.perf_counter() - t0) * 1e3
    print(json.dumps(res))
    if out_path:
        os.makedirs(os.path.dirname(os.path.abspath(out_path)), exist_ok=True)
        with open(out_path, "w") as f:
            json.dump(res, f, indent=1)
    model.close()


if __name__ == "__main__":
    main()
