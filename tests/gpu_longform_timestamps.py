"""Cost of token timestamps in long-form transcription (transcribe(return_token_timestamps=True)).

    python tests/gpu_longform_timestamps.py [--minutes 10] [--rounds 3] [--alpha 100] [--out FILE]

whisper-large-v2 + 10 Medusa-Linear heads, a recording of --minutes minutes made of 30 s `synthetic_audio` clips (30
windows at 10 minutes), the realistic acceptance regime (posterior_alpha = 100, language + length penalty as bench.py)
and the synthetic alignment table of tests/gpu_token_timestamps.py (16 pairs from the upper half of the decoder).
Transcriptions with timestamps off and on alternate in one process, after a warm-up of both.  Reported, as medians:
the wall time of a transcription, and per window the decode loop's device time (CUDA events), its time per speculative
iteration, and the extraction (wm_token_timestamps: kernels, the copy of the times and the stream synchronisation, timed
on the host around the call).  Also the host time of the timed merge.  Every window's ids must be equal in both arms.
Prints the card's name and power limit beside the numbers.
"""
from __future__ import annotations

import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import bench  # noqa: E402
from gpu_scores import arg, card  # noqa: E402
from whisper_medusa_b200 import WhisperMedusaModel  # noqa: E402
from whisper_medusa_b200.longform import merge_timed  # noqa: E402
from whisper_medusa_b200.synthetic import preset_config, synthetic_audio, synthetic_state_dict  # noqa: E402


def main():
    minutes, rounds, alpha, out_path = arg("--minutes", 10.0), arg("--rounds", 3), arg("--alpha", 100.0), arg("--out", "")
    cfg = preset_config("large-v2", heads=10)
    model = WhisperMedusaModel(cfg, synthetic_state_dict(cfg, seed=0)).to("cuda:0")
    model.release_state_dict()
    rng = np.random.default_rng(0)
    cells = rng.choice(16 * 20, 16, replace=False)
    model.generation_config.alignment_heads = [[16 + int(c) // 20, int(c) % 20] for c in sorted(cells)]
    x = np.concatenate([synthetic_audio(30.0, stream_id=i) for i in range(int(round(minutes * 2)))]).astype(np.float32)
    kw = dict(language="en", exponential_decay_length_penalty=bench.PENALTY, posterior_alpha=alpha)
    arms = {"off": {}, "on": dict(return_token_timestamps=True)}

    extract_ms = []                     # host time of every extraction call of the current transcription
    extract = model._token_timestamps

    def timed_extract(*a, **k):
        t0 = time.perf_counter()
        r = extract(*a, **k)
        extract_ms.append((time.perf_counter() - t0) * 1e3)
        return r

    model._token_timestamps = timed_extract
    for extra in arms.values():                                   # warm-up of both arms
        model.transcribe(x[: 35 * 16000], **kw, **extra)
    wall = {k: [] for k in arms}
    dec, dec_it, ext = ({k: [] for k in arms} for _ in range(3))
    ids = {}
    merge_ms = []
    for _ in range(rounds):
        for name, extra in arms.items():
            extract_ms.clear()
            t0 = time.perf_counter()
            model.transcribe(x, **kw, **extra)
            wall[name].append(time.perf_counter() - t0)
            wins = model.last_windows
            dec[name] += [w.trace.ms_decode for w in wins]
            dec_it[name] += [w.trace.ms_decode / w.trace.iterations for w in wins]
            ext[name] += list(extract_ms)
            got = [w.ids for w in wins]
            assert ids.setdefault(name, got) == got
            if name == "on":
                assert len(extract_ms) == len(wins)
                t0 = time.perf_counter()
                merge_timed(wins, int(model.generation_config.eos_token_id))
                merge_ms.append((time.perf_counter() - t0) * 1e3)
    assert ids["off"] == ids["on"], "timestamps changed a window's ids"
    med = lambda v: float(np.median(v)) if v else 0.0  # noqa: E731
    res = {"card": card(), "minutes": minutes, "windows": len(ids["on"]), "rounds": rounds,
           "pairs": len(model.generation_config.alignment_heads),
           "window_ids": int(sum(len(i) for i in ids["on"])),
           "wall_s_off": wall["off"], "wall_s_on": wall["on"],
           "wall_s_median_off": med(wall["off"]), "wall_s_median_on": med(wall["on"]),
           "decode_ms_per_window_median_off": med(dec["off"]), "decode_ms_per_window_median_on": med(dec["on"]),
           "decode_ms_per_iter_median_off": med(dec_it["off"]), "decode_ms_per_iter_median_on": med(dec_it["on"]),
           "extract_ms_per_window_median": med(ext["on"]), "extract_ms_per_window_max": max(ext["on"]),
           "timed_merge_ms_median": med(merge_ms)}
    res["wall_overhead_pct"] = 100 * (res["wall_s_median_on"] / res["wall_s_median_off"] - 1)
    res["decode_per_iter_overhead_pct"] = 100 * (res["decode_ms_per_iter_median_on"] / res["decode_ms_per_iter_median_off"] - 1)
    res["wall_ms_per_window_overhead"] = (res["wall_s_median_on"] - res["wall_s_median_off"]) * 1e3 / res["windows"]
    print(json.dumps(res))
    if out_path:
        os.makedirs(os.path.dirname(os.path.abspath(out_path)), exist_ok=True)
        with open(out_path, "w") as f:
            json.dump(res, f, indent=1)
    model.close()


if __name__ == "__main__":
    main()
