"""Freeze the REFERENCE loop's ``scores`` (``_medusa_greedy_search(..., return_dict_in_generate=True,
output_scores=True, output_logits=True)``, run through oracle/ref_harness.py on the installed Whisper modules) as a
fixture that travels to boxes without the reference checkout.

    python -m oracle.make_scores_golden            # writes tests/golden/ref_loop_scores_micro.npz

Streams: seed 0 of some groups of ``oracle/make_ref_golden.py`` on the micro preset (V = 512), so the rows stay small.
For every stream the file holds the reference's full ``input_ids``, its accept lengths and its ``scores`` rows
``[iterations, V]`` (fp32, ``-inf`` at suppressed ids).  Consumers:
  * tests/test_scores_host.py (CPU): the oracle record (oracle/scores_ref.py) reproduces the rows;
  * tests/test_gpu_scores.py  (H100): the engine's ``scores`` against the same rows.
"""
from __future__ import annotations

import os
import sys
import warnings
from typing import List, Tuple

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import make_ref_golden as G  # noqa: E402
from oracle import medusa_ref as M  # noqa: E402
from oracle import ref_harness as R  # noqa: E402
from oracle import whisper_ref as W  # noqa: E402

FIXTURE = os.path.join(ROOT, "tests", "golden", "ref_loop_scores_micro.npz")
# chains (Linear / Block heads, both acceptance rules, length penalty) and a branching tree
STREAMS = [("micro_lin_t1", 0), ("micro_lin_t0", 0), ("micro_lin_pen", 0), ("micro_blk_t1", 0),
           ("micro_tree1321_t1", 0)]


def reference_scores(ref: "R.RefLoop", enc: torch.Tensor, prompt, *, suppress_tokens=None, begin_suppress_tokens=None,
                     exponential_decay_length_penalty=None, max_length: int = 448, temperature: float = 1.0,
                     posterior_threshold: float = 0.09, posterior_alpha: float = 0.3):
    """The reference's ``_medusa_greedy_search`` called as ``RefLoop.run_loop`` calls it, with
    ``return_dict_in_generate=True, output_scores=True, output_logits=True``.  Returns its output object."""
    from transformers.generation.logits_process import (ExponentialDecayLengthPenalty, LogitsProcessorList,
                                                        SuppressTokensAtBeginLogitsProcessor,
                                                        SuppressTokensLogitsProcessor)
    from transformers.generation.stopping_criteria import EosTokenCriteria, MaxLengthCriteria, StoppingCriteriaList
    from transformers.modeling_outputs import BaseModelOutput

    procs = LogitsProcessorList()
    if exponential_decay_length_penalty is not None:
        procs.append(ExponentialDecayLengthPenalty(tuple(exponential_decay_length_penalty), ref.mcfg.eos_token_id,
                                                   len(prompt)))
    if suppress_tokens:
        procs.append(SuppressTokensLogitsProcessor(list(suppress_tokens)))
    if begin_suppress_tokens:
        procs.append(SuppressTokensAtBeginLogitsProcessor(list(begin_suppress_tokens), len(prompt)))
    stop = StoppingCriteriaList([MaxLengthCriteria(max_length=max_length),
                                 EosTokenCriteria(eos_token_id=ref.mcfg.eos_token_id)])
    ref.generation_config.max_length = max_length
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return ref._medusa_greedy_search(
            torch.tensor([list(prompt)], dtype=torch.long), logits_processor=procs, stopping_criteria=stop,
            pad_token_id=ref.mcfg.pad_token_id, eos_token_id=ref.mcfg.eos_token_id, output_scores=True,
            output_logits=True, return_dict_in_generate=True, temperature=temperature,
            posterior_threshold=posterior_threshold, posterior_alpha=posterior_alpha, synced_gpus=False,
            streamer=None, encoder_outputs=BaseModelOutput(last_hidden_state=enc[None]), use_cache=True)


def run_stream(group: str, s: int) -> Tuple[List[int], List[int], "object", torch.Tensor]:
    """(prompt, sequences, reference output, reference encoder states) of stream s of a make_ref_golden group."""
    cfg, sd, pcm, max_len, pen, temp, alpha, thr = G.stream_inputs(group, s)
    ref = R.RefLoop(cfg, sd)
    enc = ref.encode(torch.from_numpy(W.log_mel_spectrogram(pcm)))
    prompt = M.init_tokens(cfg, "en" if cfg.is_multilingual else None)
    out = reference_scores(ref, enc, prompt, suppress_tokens=cfg.suppress_tokens,
                           begin_suppress_tokens=cfg.begin_suppress_tokens, exponential_decay_length_penalty=pen,
                           max_length=max_len, temperature=temp, posterior_threshold=thr, posterior_alpha=alpha)
    return prompt, out.sequences[0].tolist(), out, enc


def main():
    if not R.available():
        raise SystemExit("the reference checkout is not present: fixtures can only be made where it is")
    fx = {}
    for group, s in STREAMS:
        prompt, seq, out, _ = run_stream(group, s)
        assert len(out.scores) == len(out.logits)
        assert all(a is b for a, b in zip(out.scores, out.logits))   # the same tensor in both tuples
        rows = torch.cat([r.reshape(1, -1) for r in out.scores]).float().numpy()
        ref_seq, ref_acc = G.run_reference(group, s)[1:]
        assert seq == ref_seq, group
        fx[f"{group}/{s}/sequences"] = np.array(seq, dtype=np.int32)
        fx[f"{group}/{s}/accept"] = np.array(ref_acc, dtype=np.int32)
        fx[f"{group}/{s}/prompt_len"] = np.int32(len(prompt))
        fx[f"{group}/{s}/scores"] = rows
        print(f"{group}/{s}: {rows.shape[0]} iterations, {len(seq) - len(prompt)} tokens", flush=True)
    np.savez_compressed(FIXTURE, **fx)


if __name__ == "__main__":
    main()
