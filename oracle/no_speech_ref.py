"""fp64 oracle of the no-speech probability (HF ``WhisperNoSpeechDetection``, ``logits_process.py:2046-2107``).

HF reads the raw (unprocessed) logits of the model at the start-of-transcript position, takes their softmax and keeps
the entry of ``no_timestamps_token_id - 1`` (``generation_whisper.py`` ``_setup_no_speech_detection``).  The model's
logits there are the base head's: ``proj_out(hidden)`` for the medusa_block type, ``proj_out(medusa_heads[0](hidden))``
for the base_head type (reference ``model.py:1274-1288``), which ``whisper_ref.medusa_logits`` with
``disable_medusa=True`` computes.

Causality makes the SOT row independent of the tokens after it: self-attention masks every later position, and
cross-attention, LayerNorm and the MLP act row by row.  So the row the engine keeps from a whole prompt (its first
iteration's sweep A) equals this one-token pass over ``[SOT]`` at position 0.
"""
from __future__ import annotations

from typing import Optional, Tuple

import torch

from . import whisper_ref as W


def no_speech_token(cfg) -> int:
    """The id HF scores: ``no_timestamps_token_id - 1`` (``<|nospeech|>`` / ``<|nocaptions|>``)."""
    return int(cfg.no_timestamps_token_id) - 1


def no_speech_row(w: W.RefWeights, cfg, enc: torch.Tensor, sot: Optional[int] = None,
                  regime: str = "fp32") -> Tuple[torch.Tensor, float]:
    """Raw base-head logits ``[V]`` of the SOT row decoded from encoder states ``enc``, and ``p[no_speech_token]``.

    ``w`` in fp64 (``RefWeights(sd, torch.float64)``) gives the fp64 reference; ``regime="engine"`` applies the
    engine's fp16 roundings of the K/V caches."""
    sot = int(cfg.decoder_start_token_id) if sot is None else int(sot)
    cache = W.new_cache(cfg)
    hidden = W.decoder_forward(w, cfg, [sot], [0], enc, cache, regime)
    row = W.medusa_logits(w, cfg, hidden, enc, cache, True, regime)[0, 0]
    prob = float(torch.softmax(row.double(), dim=-1)[no_speech_token(cfg)])
    return row, prob
