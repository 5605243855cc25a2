"""Cost of temperature fallback (transcribe(temperature=(0.0, ...), ...)) on large-v2 (development aid; not a test).

    python tests/gpu_temperature_fallback.py [--rounds 3] [--minutes 10] [--out FILE]

whisper-large-v2 + 10 Medusa-Linear heads, the benchmark clip and length penalty, typical acceptance in the realistic
regime (posterior_alpha = 100) for the unsampled loop.  Reports, with the card's name and power limit:
* per-iteration decode time and accept-length histogram of the unsampled loop and of sampled attempts at T = 0.2 / 1.0
  with top_k 50 / 0, calls alternating in one process, medians over the rounds;
* the in-kernel time of the logits-scan and fold stages (SELECT1, SELECT_FIN, ACCEPT) from the stage profile, CTA 0,
  per iteration, sampled (T = 1.0, top_k 50 and 0) against unsampled;
* transcribe of a synthetic recording of --minutes minutes with OpenAI's defaults (0.0 ... 1.0, 2.4, -1.0, 0.6):
  attempts per window and wall time against plain transcribe.
"""
from __future__ import annotations

import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import bench  # noqa: E402
from gpu_stage_profile import MODES, STAGES  # noqa: E402
from whisper_medusa_b200 import WhisperMedusaModel, _lib  # noqa: E402
from whisper_medusa_b200.synthetic import preset_config, synthetic_audio, synthetic_state_dict  # noqa: E402


def arg(name, default):
    return type(default)(sys.argv[sys.argv.index(name) + 1]) if name in sys.argv else default


def card() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        return "unknown"


def decode(model, kw, sampling):
    extra = {"medusa_temperature": 0.0} if sampling else {}
    model._decode("en", None, dict(kw, **extra), None, sampling=sampling)
    tr = model.last_trace
    return tr.ms_decode / max(1, tr.iterations), tr.accept_lengths


def stage_times(model, kw, sampling):
    """us per iteration of the select / fold stages (CTA 0 body time) over a 6-iteration profiled run."""
    model.set_option("profile", 1)
    extra = {"medusa_temperature": 0.0} if sampling else {}
    model._decode("en", None, dict(kw, max_iters=6, **extra), None, sampling=sampling)
    model.set_option("profile", 0)
    lib = _lib.load()
    cap = 4096
    buf = (C.c_int64 * (cap * 24))()
    n = C.c_int32(0)
    assert lib.wm_get_stage_profile(model._handle, buf, cap, C.byref(n)) == 0
    rows = np.frombuffer(buf, dtype=np.int64)[: n.value * 24].reshape(-1, 24)
    out = {}
    for row in rows:
        st, mode = STAGES[row[0]], MODES[row[1]]
        if st in ("SELECT1", "SELECT2", "SELECT_FIN", "ACCEPT"):
            out[f"{st}/{mode}"] = out.get(f"{st}/{mode}", 0.0) + max(int(row[5 + 1]), 0) / 1e3
    return {k: round(v, 2) for k, v in out.items()}     # (the profile keeps the last iteration's timeline)


def main():
    rounds, minutes, out_path = arg("--rounds", 3), arg("--minutes", 10), arg("--out", "")
    res = {"card": card()}
    cfg = preset_config("large-v2", heads=10)
    model = WhisperMedusaModel(cfg, synthetic_state_dict(cfg, seed=0)).to("cuda:0")
    model.set_decode_mode("persistent")
    kw = dict(exponential_decay_length_penalty=bench.PENALTY, posterior_alpha=100.0)
    model.generate_from_pcm(synthetic_audio(30.0, stream_id=0), language="en", **kw)
    arms = {"unsampled": None}
    for t in (0.2, 1.0):
        for k in (50, 0):
            arms[f"T={t},top_k={k}"] = (t, k, 1, 2, 0, 1)
    for s in arms.values():
        decode(model, kw, s)                                # warm-up
    ms = {a: [] for a in arms}
    hist = {}
    for _ in range(rounds):
        for a, s in arms.items():
            m, acc = decode(model, kw, s)
            ms[a].append(m)
            hist[a] = np.bincount(acc, minlength=11).tolist()
    res["ms_per_iteration"] = {a: round(float(np.median(v)), 4) for a, v in ms.items()}
    res["accept_hist"] = hist
    res["stage_us_last_iteration"] = {a: stage_times(model, kw, s) for a, s in
                                      (("unsampled", None), ("T=1.0,top_k=50", (1.0, 50, 1, 2, 0, 1)),
                                       ("T=1.0,top_k=0", (1.0, 0, 1, 2, 0, 1)))}
    print(json.dumps(res), flush=True)
    # long recording
    x = np.concatenate([synthetic_audio(30.0, stream_id=i) for i in range(2 * minutes)]).astype(np.float32)
    tkw = dict(language="en", exponential_decay_length_penalty=bench.PENALTY, posterior_alpha=100.0)
    fb = dict(temperature=(0.0, 0.2, 0.4, 0.6, 0.8, 1.0), compression_ratio_threshold=2.4, logprob_threshold=-1.0,
              no_speech_threshold=0.6)
    wall = {}
    for name, extra in (("plain", {}), ("fallback", fb)):
        torch.manual_seed(0)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        model.transcribe(x, **tkw, **extra)
        torch.cuda.synchronize()
        wall[name] = round(time.perf_counter() - t0, 3)
        if extra:
            att = [len(r.attempts) for r in model.last_windows]
            res["attempts_per_window"] = np.bincount(att, minlength=7).tolist()[1:]
            res["windows"] = len(att)
            res["skipped"] = sum(bool(r.skipped) for r in model.last_windows)
    res["transcribe_wall_s"] = wall
    print(json.dumps(res), flush=True)
    if out_path:
        with open(out_path, "w") as f:
            json.dump(res, f)
    model.close()


if __name__ == "__main__":
    main()
