"""Freeze the reference's own loop on checkpoints whose Medusa heads are stacks of several ResBlocks
(``medusa_num_layers`` > 1) as fixtures for the engine's tests.

    python -m oracle.make_head_layers_golden        # writes tests/golden/ref_loop_head_layers.npz

Streams are not selected: stream s of a group is checkpoint seed and audio stream ``base_seed + s``.  For every stream
the script runs the reference's loop (``ref_harness.RefLoop``, which builds ``medusa_num_layers`` ResBlocks per head)
and the oracle's restatement (``medusa_ref.medusa_greedy_search``, fp32) and requires them to agree; the file holds the
full ``input_ids`` and the accept lengths.  Consumers: tests/test_medusa_head_layers_host.py (CPU: the oracle
reproduces every stream), tests/test_gpu_head_layers.py (H100: the engine against the same streams).
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import medusa_ref as M  # noqa: E402
from oracle import ref_harness as R  # noqa: E402
from oracle import whisper_ref as W  # noqa: E402
from whisper_medusa_b200.synthetic import preset_config, synthetic_audio, synthetic_state_dict  # noqa: E402

FIXTURE = os.path.join(ROOT, "tests", "golden", "ref_loop_head_layers.npz")

# group -> (preset, heads, heads_type, head layers, medusa_choices or None, n_streams, base_seed, max_length, penalty,
#           temperature): Linear and Block heads, 2, 3 and 4 layers, chains and trees, typical and exact-match acceptance
GROUPS = {
    "micro_lin_l2_t1": ("micro", 4, "base_head", 2, None, 4, 2100, 120, None, 1.0),
    "micro_lin_l3_t0": ("micro", 4, "base_head", 3, None, 3, 2200, 100, None, 0.0),
    "micro_lin_l4_k10": ("micro", 10, "base_head", 4, None, 3, 2300, 140, (20, 1.05), 1.0),
    "micro_blk_l2_t1": ("micro", 4, "medusa_block", 2, None, 4, 2400, 120, None, 1.0),
    "micro_blk_l3_k10": ("micro", 10, "medusa_block", 3, None, 3, 2500, 140, None, 1.0),
    "micro_tree122_l2_t1": ("micro", 2, "base_head", 2, [1, 2, 2], 3, 2600, 100, None, 1.0),
    "micro_blk_tree122_l3_t0": ("micro", 2, "medusa_block", 3, [1, 2, 2], 3, 2700, 100, None, 0.0),
    "tiny_lin_l2_t1": ("tiny.en", 4, "base_head", 2, None, 2, 2800, 120, None, 1.0),
}


def stream_inputs(group: str, s: int):
    """(cfg, state dict, pcm, max_length, penalty, temperature) of stream ``s`` of ``group``."""
    preset, heads, htype, layers, choices, _, base, max_len, pen, temp = GROUPS[group]
    cfg = preset_config(preset, heads=heads, heads_type=htype, head_layers=layers)
    if choices:
        cfg.medusa_choices = list(choices)
    sd = synthetic_state_dict(cfg, seed=base + s)
    pcm = synthetic_audio(5.0, stream_id=base + s)
    return cfg, sd, pcm, max_len, pen, temp


def oracle_stream(group: str, s: int, regime: str = "fp32"):
    cfg, sd, pcm, max_len, pen, temp = stream_inputs(group, s)
    w = W.RefWeights(sd)
    enc = W.encoder_forward(w, cfg, torch.from_numpy(W.log_mel_spectrogram(pcm)), regime)
    prompt = M.init_tokens(cfg, "en" if cfg.is_multilingual else None)
    tr = M.medusa_greedy_search(w, cfg, enc, prompt, M.gen_params(cfg, prompt, pen, max_len, temperature=temp), regime)
    return tr.sequences, tr.accept_lengths


def reference_stream(group: str, s: int):
    cfg, sd, pcm, max_len, pen, temp = stream_inputs(group, s)
    ref = R.RefLoop(cfg, sd)
    enc = ref.encode(torch.from_numpy(W.log_mel_spectrogram(pcm)))
    prompt = M.init_tokens(cfg, "en" if cfg.is_multilingual else None)
    return ref.run_loop(enc, prompt, suppress_tokens=cfg.suppress_tokens, begin_suppress_tokens=cfg.begin_suppress_tokens,
                        exponential_decay_length_penalty=pen, max_length=max_len, temperature=temp)


def main():
    if not R.available():
        raise SystemExit("the reference checkout is not present: the fixture can only be made where it is")
    torch.set_num_threads(min(16, os.cpu_count() or 1))
    out = {}
    for g, spec in GROUPS.items():
        for s in range(spec[5]):
            seq, acc = reference_stream(g, s)
            assert (seq, acc) == oracle_stream(g, s), f"{g}/{s}: the oracle loop differs from the reference's loop"
            out[f"{g}/{s}/sequences"] = np.array(seq, np.int32)
            out[f"{g}/{s}/accept"] = np.array(acc, np.int32)
            print(f"{g}/{s}: {len(seq)} ids, {len(acc)} iterations, accept {acc[:10]}", flush=True)
    np.savez_compressed(FIXTURE, **out)


if __name__ == "__main__":
    main()
