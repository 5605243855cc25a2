"""Cost of the logits processors (generate(sequence_bias=..., bad_words_ids=..., no_repeat_ngram_size=...,
min_new_tokens=...)) on the benchmark clip.

    python tests/gpu_logits_processors.py [--rounds 8] [--alpha 100] [--out FILE]

whisper-large-v2 + 10 Medusa-Linear heads, the 30 s clip of bench.py (stream 0), typical acceptance in the realistic
regime (posterior_alpha = 100), the benchmark's length penalty.  Calls with all five processors and without any alternate
in one process; each reports the decode loop's device time (CUDA events) per speculative iteration.  The processors do
their full work but leave the clip's tokens as they are (asserted), so both arms decode the same sequence.  The
processors' own kernel time comes from torch.profiler (CUDA activities) in a call of its own.  Prints the card's name
and power limit beside the numbers.
"""
from __future__ import annotations

import json
import os
import sys

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
    pcm = synthetic_audio(30.0, stream_id=0)
    kw = dict(language="en", exponential_decay_length_penalty=bench.PENALTY, posterior_alpha=alpha)
    model.generate_from_pcm(pcm, **kw)
    full = model.last_trace.sequences
    plain = full[4:]
    # the shortest m whose m-grams are all distinct in the clip's sequence: n-grams of size m + 1 then ban nothing
    m = next(m for m in range(1, len(full)) if len({tuple(full[i:i + m]) for i in range(len(full) - m + 1)})
             == len(full) - m + 1)
    # every processor on with its full per-iteration work -- 64 two-token biases and 64 bad words matched against the
    # sequence, 64 single-token biases, an n-gram scan over the whole sequence, an EOS ban -- but aimed at suppressed ids
    # (already -inf) and with n-grams longer than any repeat in the clip, so both arms decode the same tokens and their
    # per-iteration times compare the same work
    sup = [int(t) for t in cfg.suppress_tokens if int(t) < cfg.vocab_size][:64]
    seq_bias = [[[int(a), s], 0.5] for a, s in zip(plain[:64], sup * 8)] + [[[s], -0.5] for s in sup]
    procs = dict(sequence_bias=seq_bias, bad_words_ids=[[int(a), s] for a, s in zip(plain[1:65], sup * 8)],
                 no_repeat_ngram_size=m + 1, min_new_tokens=1)
    arms = {"off": {}, "on": procs}
    for extra in arms.values():
        model.generate_from_pcm(pcm, **kw, **extra)
    ms, toks = {k: [] for k in arms}, {}
    for _ in range(rounds):
        for name, extra in arms.items():
            model.generate_from_pcm(pcm, **kw, **extra)
            tr = model.last_trace
            ms[name].append(tr.ms_decode / tr.iterations)
            toks.setdefault(name, (tr.sequences, tr.accept_lengths, tr.iterations))
            assert (tr.sequences, tr.accept_lengths, tr.iterations) == toks[name]
    assert toks["off"] == toks["on"], "the processors changed the tokens: the arms would not do the same work"
    res = {"card": card(), "iterations": toks["off"][2], "tokens": len(toks["off"][0]), "rounds": rounds,
           "no_repeat_ngram_size": m + 1,
           "ms_per_iter_off": ms["off"], "ms_per_iter_on": ms["on"],
           "median_off": float(np.median(ms["off"])), "median_on": float(np.median(ms["on"]))}
    res["cost_us_per_iter"] = (res["median_on"] - res["median_off"]) * 1e3
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        model.generate_from_pcm(pcm, **kw, **procs)
    per = {}
    for e in prof.events():
        if e.device_type.name == "CUDA" and "logits_proc" in e.name:
            n, t = per.get("logits_proc_kernel", (0, 0.0))
            per["logits_proc_kernel"] = (n + 1, t + e.device_time)
    res["prep_kernel"] = {k: {"count": n, "mean_us": t / n} for k, (n, t) in per.items()}
    print(json.dumps(res))
    if out_path:
        os.makedirs(os.path.dirname(os.path.abspath(out_path)), exist_ok=True)
        with open(out_path, "w") as f:
            json.dump(res, f, indent=1)
    model.close()


if __name__ == "__main__":
    main()
