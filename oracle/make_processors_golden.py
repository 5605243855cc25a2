"""Freeze the oracle loop with logits processors (``sequence_bias``, ``bad_words_ids``, ``no_repeat_ngram_size``,
``min_length``, ``min_new_tokens``) as fixtures for the engine's tests.

    python -m oracle.make_processors_golden        # writes tests/golden/ref_loop_processors.npz

Each scenario is seed 0 of a group of ``oracle/make_ref_golden.py`` with processors whose arguments are derived from
that stream's own tokens without processors (so every scenario changes the tokens).  Where the reference checkout is
present, the script first holds the oracle to the reference's own loop (``processors_ref.run_loop``) on every
scenario it freezes.  The file holds, per scenario, the sequences and accept lengths with and without processors.
Consumers: tests/test_logits_processors_host.py (CPU), tests/test_gpu_logits_processors.py (H100).
"""
from __future__ import annotations

import os
import sys
from typing import Dict, List, Tuple

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import make_ref_golden as G  # noqa: E402
from oracle import medusa_ref as M  # noqa: E402
from oracle import processors_ref as PR  # noqa: E402
from oracle import ref_harness as R  # noqa: E402
from oracle import whisper_ref as W  # noqa: E402

FIXTURE = os.path.join(ROOT, "tests", "golden", "ref_loop_processors.npz")

# scenario -> (make_ref_golden group, processors); each processor alone and all together, chains and trees, Linear and
# Block heads, temperature 0 and 1, the EOS decay on
_KINDS = ("bias", "bad", "ngram", "minlen", "all")
SCENARIOS: Dict[str, Tuple[str, str]] = {}
for _g in ("micro_lin_t1", "micro_lin_t0", "micro_tree122_t1"):
    for _k in _KINDS:
        SCENARIOS[f"{_g}/{_k}"] = (_g, _k)
for _g, _k in (("micro_blk_t1", "all"), ("micro_lin_pen", "all"), ("micro_tree122_t0", "all"), ("tiny_lin_t1", "all"),
               ("tiny_blk_pen", "bias")):
    SCENARIOS[f"{_g}/{_k}"] = (_g, _k)


def processor_args(kind: str, plain: List[int], prompt_len: int, eos: int, max_len: int, pen=None) -> Dict:
    """The processors of a scenario, from the stream's tokens without them (``plain``, prompt included).  With the EOS
    decay (``pen``) the EOS ban ends where the decay starts: the engine refuses an overlap (the reference's rows are NaN
    there)."""
    gen = plain[prompt_len:]
    g0, g1, g2 = gen[0], gen[1], gen[2]
    ended = eos in gen
    args: Dict = {}
    if kind in ("bias", "all"):
        # push the first generated token down; the two-token entries share a last token, so their sum is in dict order
        args["sequence_bias"] = [[[g0], -40.0], [[g0, g1], 3.25], [[g2, g1], -1.5], [[plain[prompt_len - 1], g1], 0.75]]
    if kind in ("bad", "all"):
        args["bad_words_ids"] = [[eos], [g1], [g0, g2], [3, 4, 5]]
    if kind in ("ngram", "all"):
        args["no_repeat_ngram_size"] = 1 if kind == "ngram" else 2
    if kind in ("minlen", "all"):
        n = len(gen[: gen.index(eos)]) if ended else len(gen) // 2
        if kind == "minlen":
            args["min_length"] = min(prompt_len + n + 6, max_len - 8)
        else:
            args["min_new_tokens"] = min(n + 4, max_len - prompt_len - 8)
        if pen is not None:
            args.pop("min_length", None)
            args["min_new_tokens"] = int(pen[0])
    if kind == "minlen" and not ended:
        # the stream does not end by itself: ban the token that follows its first token as well, so it changes
        args["bad_words_ids"] = [[g0, g1]]
    return args


def _gp_over(args: Dict, eos: int) -> Dict:
    over = {}
    if "sequence_bias" in args:
        over["sequence_bias"] = [(tuple(ids), float(v)) for ids, v in {tuple(a[0]): a[1] for a in args["sequence_bias"]}.items()]
    for k in ("bad_words_ids", "no_repeat_ngram_size", "min_length", "min_new_tokens"):
        if k in args:
            over[k] = args[k]
    return over


def run_scenario(name: str, with_reference: bool = False):
    """(reference sequences, reference accepts or None, oracle sequences, oracle accepts, oracle sequences without
    processors) of a scenario; the reference's are None unless ``with_reference``."""
    group, kind = SCENARIOS[name]
    cfg, sd, pcm, max_len, pen, temp, alpha, thr = G.stream_inputs(group, 0)
    w = W.RefWeights(sd)
    enc = W.encoder_forward(w, cfg, torch.from_numpy(W.log_mel_spectrogram(pcm)), "fp32")
    prompt = M.init_tokens(cfg, "en" if cfg.is_multilingual else None)
    kw = dict(temperature=temp, posterior_alpha=alpha, posterior_threshold=thr)
    plain = M.medusa_greedy_search(w, cfg, enc, prompt, M.gen_params(cfg, prompt, pen, max_len, **kw), "fp32")
    args = processor_args(kind, plain.sequences, len(prompt), int(cfg.eos_token_id), max_len, pen)
    gp = M.gen_params(cfg, prompt, pen, max_len, **kw, **_gp_over(args, int(cfg.eos_token_id)))
    tr = PR.medusa_greedy_search(w, cfg, enc, prompt, gp, "fp32")
    ref_seq = ref_acc = None
    if with_reference:
        ref = R.RefLoop(cfg, sd)
        ref_enc = ref.encode(torch.from_numpy(W.log_mel_spectrogram(pcm)))
        ref_seq, ref_acc = PR.run_loop(ref, ref_enc, prompt, processor_args=args, suppress_tokens=cfg.suppress_tokens,
                                       begin_suppress_tokens=cfg.begin_suppress_tokens,
                                       exponential_decay_length_penalty=pen, max_length=max_len, temperature=temp,
                                       posterior_threshold=thr, posterior_alpha=alpha)
    return ref_seq, ref_acc, tr.sequences, tr.accept_lengths, plain.sequences


def scenario_args(name: str, plain: List[int]) -> Dict:
    """The generate() kwargs of a scenario given its frozen stream without processors."""
    group, kind = SCENARIOS[name]
    cfg, _, _, max_len, pen, _, _, _ = G.stream_inputs(group, 0)
    prompt = M.init_tokens(cfg, "en" if cfg.is_multilingual else None)
    return processor_args(kind, list(plain), len(prompt), int(cfg.eos_token_id), max_len, pen)


def main():
    torch.set_num_threads(min(16, os.cpu_count() or 1))
    out = {}
    for name in SCENARIOS:
        ref_seq, ref_acc, seq, acc, plain = run_scenario(name, with_reference=R.available())
        if ref_seq is not None:
            assert (seq, acc) == (ref_seq, ref_acc), f"{name}: the oracle loop differs from the reference's loop"
        assert seq != plain, f"{name}: the processors do not change the stream"
        out[f"{name}/sequences"] = np.array(seq, np.int32)
        out[f"{name}/accept"] = np.array(acc, np.int32)
        out[f"{name}/plain"] = np.array(plain, np.int32)
        print(f"{name}: {len(plain)} -> {len(seq)} ids, reference {'checked' if ref_seq is not None else 'absent'}",
              flush=True)
    np.savez_compressed(FIXTURE, **out)


if __name__ == "__main__":
    main()
