"""Cost of scoring (generate(return_dict_in_generate=True, output_scores=True)) on the benchmark clip.

    python tests/gpu_scores.py [--rounds 8] [--alpha 100] [--out FILE]

whisper-large-v2 + 10 Medusa-Linear heads, the 30 s clip of bench.py (stream 0), typical acceptance in the realistic
regime (posterior_alpha = 100), the benchmark's length penalty.  Calls with scoring off and on alternate in one process;
each reports the decode loop's device time (CUDA events) per speculative iteration.  The tokens of both arms must be
identical.  Prints the card's name and power limit beside the numbers.
"""
from __future__ import annotations

import json
import os
import subprocess
import sys

import numpy as np

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
    rounds, alpha, out_path = arg("--rounds", 8), arg("--alpha", 100.0), arg("--out", "")
    cfg = preset_config("large-v2", heads=10)
    model = WhisperMedusaModel(cfg, synthetic_state_dict(cfg, seed=0)).to("cuda:0")
    pcm = synthetic_audio(30.0, stream_id=0)
    kw = dict(language="en", exponential_decay_length_penalty=bench.PENALTY, posterior_alpha=alpha)
    arms = {"off": {}, "on": dict(return_dict_in_generate=True, output_scores=True, output_logits=True)}
    for extra in arms.values():                       # warm-up of both arms (buffers, modules)
        model.generate_from_pcm(pcm, **kw, **extra)
    ms, toks = {k: [] for k in arms}, {}
    for _ in range(rounds):
        for name, extra in arms.items():
            model.generate_from_pcm(pcm, **kw, **extra)
            tr = model.last_trace
            ms[name].append(tr.ms_decode / tr.iterations)
            toks.setdefault(name, (tr.sequences, tr.accept_lengths, tr.iterations))
            assert (tr.sequences, tr.accept_lengths, tr.iterations) == toks[name]
    assert toks["off"] == toks["on"], "scoring changed the tokens"
    res = {"card": card(), "iterations": toks["off"][2], "tokens": len(toks["off"][0]), "rounds": rounds,
           "ms_per_iter_off": ms["off"], "ms_per_iter_on": ms["on"],
           "median_off": float(np.median(ms["off"])), "median_on": float(np.median(ms["on"]))}
    res["cost_us_per_iter"] = (res["median_on"] - res["median_off"]) * 1e3
    if "--profile" in sys.argv:
        # device time per kernel name (torch.profiler, CUDA activities), one call per arm, in a run of its own
        from torch.profiler import ProfilerActivity, profile

        for name, extra in arms.items():
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                model.generate_from_pcm(pcm, **kw, **extra)
            per = {}
            for e in prof.events():
                if e.device_type.name == "CUDA":
                    n, t = per.get(e.name, (0, 0.0))
                    per[e.name] = (n + 1, t + e.device_time)
            res[f"kernels_{name}"] = {k[:60]: {"count": n, "mean_us": t / n} for k, (n, t) in per.items()
                                      if n >= 10}
    print(json.dumps(res))
    if out_path:
        os.makedirs(os.path.dirname(os.path.abspath(out_path)), exist_ok=True)
        with open(out_path, "w") as f:
            json.dump(res, f, indent=1)
    model.close()


if __name__ == "__main__":
    main()
