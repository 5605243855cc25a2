"""Cost of the no-speech rule (transcribe(no_speech_threshold=..., logprob_threshold=...)) on large-v2.

    python tests/gpu_no_speech.py [--rounds 6] [--alpha 100] [--out FILE]

(README and DESIGN section 7 quote a run of ``python tests/gpu_no_speech.py --rounds 5``.)

whisper-large-v2 + 10 Medusa-Linear heads, typical acceptance in the realistic regime (posterior_alpha = 100), the
benchmark's length penalty.  Reports:
* the no-speech kernels' device time (torch.profiler, CUDA activities, a run of its own) and the vocabulary kernel's
  achieved bytes/s against the 51865 x 1280 fp16 matrix it streams (132.8 MB);
* the per-window cost of transcribe with the thresholds on and off (a 60 s recording of synthetic speech, 30 s windows),
  calls alternating in one process, medians of the decode loop's device time per window.  "On" includes the scores
  kernel the rule needs (avg_logprob).  The ids of both arms must be identical.
Prints the card's name and power limit beside the numbers.
"""
from __future__ import annotations

import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from whisper_medusa_b200 import WhisperMedusaModel  # noqa: E402
from whisper_medusa_b200.synthetic import preset_config, synthetic_audio, synthetic_state_dict  # noqa: E402


def arg(name, default):
    return type(default)(sys.argv[sys.argv.index(name) + 1]) if name in sys.argv else default


def card() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        return "unknown"


def main():
    rounds, alpha, out_path = arg("--rounds", 6), arg("--alpha", 100.0), arg("--out", "")
    cfg = preset_config("large-v2", heads=10)
    model = WhisperMedusaModel(cfg, synthetic_state_dict(cfg, seed=0)).to("cuda:0")
    x = np.concatenate([synthetic_audio(30.0, stream_id=0), synthetic_audio(30.0, stream_id=1)])
    kw = dict(language="en", exponential_decay_length_penalty=bench.PENALTY, posterior_alpha=alpha)
    arms = {"off": {}, "on": dict(no_speech_threshold=0.6, logprob_threshold=-1.0)}
    for extra in arms.values():                       # warm-up of both arms
        model.transcribe(x, **kw, **extra)
    ms, wall, ids = {k: [] for k in arms}, {k: [] for k in arms}, {}
    for _ in range(rounds):
        for name, extra in arms.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            model.transcribe(x, **kw, **extra)
            torch.cuda.synchronize()
            wins = model.last_windows
            wall[name].append((time.perf_counter() - t0) * 1e3 / len(wins))
            ms[name].append(float(np.mean([r.trace.ms_decode for r in wins])))
            got = [r.ids for r in wins]
            ids.setdefault(name, got)
            assert got == ids[name]
    assert ids["off"] == ids["on"], "the rule changed the decoded ids"
    res = {"card": card(), "windows": len(ids["off"]), "rounds": rounds,
           "decode_ms_per_window_off": ms["off"], "decode_ms_per_window_on": ms["on"],
           "median_decode_ms_off": float(np.median(ms["off"])), "median_decode_ms_on": float(np.median(ms["on"])),
           "median_wall_ms_per_window_off": float(np.median(wall["off"])),
           "median_wall_ms_per_window_on": float(np.median(wall["on"]))}
    res["cost_decode_us_per_window"] = (res["median_decode_ms_on"] - res["median_decode_ms_off"]) * 1e3
    res["cost_wall_us_per_window"] = (res["median_wall_ms_per_window_on"] - res["median_wall_ms_per_window_off"]) * 1e3
    # kernel time in a run of its own
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(rounds):
            model.transcribe(x, **kw, **arms["on"])
        torch.cuda.synchronize()
    per = {}
    for e in prof.events():
        if e.device_type.name == "CUDA" and "no_speech" in e.name:
            n, t = per.get(e.name, (0, 0.0))
            per[e.name] = (n + 1, t + e.device_time)
    kernels = {k: {"count": n, "mean_us": t / n} for k, (n, t) in per.items()}
    res["kernels"] = kernels
    vocab = [v for k, v in kernels.items() if "vocab" in k]
    if vocab:
        bytes_ = cfg.vocab_size * cfg.d_model * 2
        res["vocab_bytes"] = bytes_
        res["vocab_GBps"] = bytes_ / (vocab[0]["mean_us"] * 1e-6) / 1e9
    print(json.dumps(res))
    if out_path:
        os.makedirs(os.path.dirname(os.path.abspath(out_path)), exist_ok=True)
        with open(out_path, "w") as f:
            json.dump(res, f, indent=1)
    model.close()


if __name__ == "__main__":
    main()
