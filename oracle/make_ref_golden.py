"""Freeze outputs of the REFERENCE's own loop code (oracle/ref_harness.py: the verbatim functions of
/root/reference bound onto the installed Whisper modules) as fixtures that travel to boxes without the
reference checkout.

    python -m oracle.make_ref_golden            # writes tests/golden/ref_loop_streams.npz

Streams are NOT selected: seed s of every group is simply ``base_seed + s``.  For every stream the file holds
the reference's full ``input_ids`` (prompt + emitted tokens + post-EOS fill) and its accept-length list,
fp32 on CPU.  Consumers:
  * tests/test_ref_loop_pin.py (CPU): the oracle restatement reproduces every stream bit-for-bit;
  * tests/test_gpu_parity.py  (H100): the CUDA engine against the same streams -- mismatch RATE over all
    of them (fp16-operand rounding can flip a near-tie; a flipped decision changes the rest of the stream).
"""
from __future__ import annotations

import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import medusa_ref as M  # noqa: E402
from oracle import ref_harness as R  # noqa: E402
from oracle import whisper_ref as W  # noqa: E402
from whisper_medusa_b200.synthetic import preset_config, synthetic_audio, synthetic_state_dict  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")

# group -> (preset, heads, heads_type, n_streams, base_seed, max_length, penalty, temperature, posterior_alpha, thr)
GROUPS = {
    "micro_lin_t1": ("micro", 4, "base_head", 12, 100, 120, None, 1.0, 0.3, 0.09),
    "micro_lin_t0": ("micro", 4, "base_head", 10, 200, 100, None, 0.0, 0.3, 0.09),
    "micro_lin_pen": ("micro", 4, "base_head", 10, 300, 140, (20, 1.05), 1.0, 0.3, 0.09),
    "micro_lin_k10": ("micro", 10, "base_head", 10, 400, 160, None, 1.0, 0.3, 0.09),
    "micro_blk_t1": ("micro", 4, "medusa_block", 12, 500, 120, None, 1.0, 0.3, 0.09),
    "micro_blk_t0": ("micro", 4, "medusa_block", 10, 600, 100, None, 0.0, 0.3, 0.09),
    "micro_blk_pen": ("micro", 10, "medusa_block", 10, 700, 140, (20, 1.05), 1.0, 0.3, 0.09),
    "tiny_lin_t1": ("tiny.en", 4, "base_head", 4, 800, 120, None, 1.0, 0.3, 0.09),
    "tiny_blk_pen": ("tiny.en", 4, "medusa_block", 4, 900, 120, (30, 1.03), 1.0, 0.3, 0.09),
    # branching medusa_choices (TREE_CHOICES below): per-head top-k, tree verify in the reference's own way (its
    # medusa_attn_mask is never applied), gathered KV rows, best-path selection by likelihood
    "micro_tree122_t1": ("micro", 2, "base_head", 8, 1000, 100, None, 1.0, 0.3, 0.09),
    "micro_tree122_t0": ("micro", 2, "base_head", 8, 1100, 100, None, 0.0, 0.3, 0.09),
    "micro_tree1321_t1": ("micro", 3, "base_head", 8, 1200, 100, (20, 1.05), 1.0, 0.3, 0.09),
    "micro_tree12121_t0": ("micro", 4, "base_head", 6, 1300, 100, None, 0.0, 0.3, 0.09),
    "micro_blk_tree122_t1": ("micro", 2, "medusa_block", 8, 1400, 100, None, 1.0, 0.3, 0.09),
}
TREE_CHOICES = {"micro_tree122_t1": [1, 2, 2], "micro_tree122_t0": [1, 2, 2], "micro_tree1321_t1": [1, 3, 2, 1],
                "micro_tree12121_t0": [1, 2, 1, 2, 1], "micro_blk_tree122_t1": [1, 2, 2]}


def stream_inputs(group: str, s: int):
    preset, heads, htype, n, base, max_len, pen, temp, alpha, thr = GROUPS[group]
    cfg = preset_config(preset, heads=heads, heads_type=htype)
    if group in TREE_CHOICES:
        cfg.medusa_choices = list(TREE_CHOICES[group])
    sd = synthetic_state_dict(cfg, seed=base + s)
    pcm = synthetic_audio(5.0, stream_id=base + s)
    return cfg, sd, pcm, max_len, pen, temp, alpha, thr


def run_reference(group: str, s: int):
    cfg, sd, pcm, max_len, pen, temp, alpha, thr = stream_inputs(group, s)
    ref = R.RefLoop(cfg, sd)
    mel = torch.from_numpy(W.log_mel_spectrogram(pcm))
    enc = ref.encode(mel)
    prompt = M.init_tokens(cfg, "en" if cfg.is_multilingual else None)
    seq, acc = ref.run_loop(enc, prompt, suppress_tokens=cfg.suppress_tokens,
                            begin_suppress_tokens=cfg.begin_suppress_tokens, exponential_decay_length_penalty=pen,
                            max_length=max_len, temperature=temp, posterior_threshold=thr, posterior_alpha=alpha)
    return prompt, seq, acc


def main():
    if not R.available():
        raise SystemExit("the reference checkout is not present: fixtures can only be made in the authoring container")
    out = {}
    t0 = time.time()
    for group, spec in GROUPS.items():
        n = spec[3]
        hist = np.zeros(spec[1] + 1, dtype=np.int64)
        for s in range(n):
            prompt, seq, acc = run_reference(group, s)
            out[f"{group}/{s}/sequences"] = np.array(seq, dtype=np.int32)
            out[f"{group}/{s}/accept"] = np.array(acc, dtype=np.int32)
            out[f"{group}/{s}/prompt_len"] = np.int32(len(prompt))
            hist += np.bincount(np.array(acc), minlength=spec[1] + 1)
        print(f"{group}: {n} streams, accept histogram {hist.tolist()} ({time.time() - t0:.0f}s)", flush=True)
    np.savez_compressed(os.path.join(GOLDEN, "ref_loop_streams.npz"), **out)


if __name__ == "__main__":
    main()
