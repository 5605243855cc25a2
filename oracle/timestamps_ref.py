"""Oracle of token-level timestamps (HF ``WhisperGenerationMixin._extract_token_timestamps``,
``generation_whisper.py:241-381``).

* ``alignment_probs``: an fp64 teacher-forced decoder pass (the layers of ``whisper_ref``) over a whole sequence that
  returns the cross-attention probabilities of the alignment heads at every position.  For a chain, the rows the engine
  keeps are these: causally, the row at position p only sees ids[0..p], whichever pass computed it.
* ``extract``: the extraction restated step by step -- crop, normalise, median filter, head average (the same torch
  fp32 operations as HF, so the matrix is bit-equal), DTW vectorised over anti-diagonals in numpy, backtrace, and the
  assembly ``[zeros(P), jump_times, jump_times[-1]]``.
"""
from __future__ import annotations

from typing import List, Optional, Sequence, Tuple

import numpy as np
import torch
import torch.nn.functional as F

from . import whisper_ref as W


def alignment_probs(w: W.RefWeights, cfg, ids: Sequence[int], enc: torch.Tensor, pairs: Sequence[Sequence[int]],
                    regime: str = "fp32", return_scores: bool = False):
    """``[len(pairs), len(ids), S]``: softmax over the S encoder frames of each listed (layer, head) at every position of
    ``ids`` (positions 0 .. n-1, causal self-attention, no cache).  ``regime="engine"`` rounds the K/V caches to fp16
    as the engine stores them.  ``return_scores``: also the raw scores q . k / 8 (same shape)."""
    rq = W._r16 if regime == "engine" else (lambda t: t)
    H = cfg.decoder_attention_heads
    dh = cfg.d_model // H
    p = "whisper_model.model.decoder"
    n = len(ids)
    x = w[f"{p}.embed_tokens.weight"][torch.tensor(list(ids))] + w[f"{p}.embed_positions.weight"][torch.arange(n)]
    e = rq(enc.to(w.dtype))
    mask = torch.arange(n)[None, :] > torch.arange(n)[:, None]
    keep, raw = {}, {}
    for li in range(cfg.decoder_layers):
        lp = f"{p}.layers.{li}"
        h = w.ln(x, f"{lp}.self_attn_layer_norm")
        q = w.lin(h, f"{lp}.self_attn.q_proj") * (dh ** -0.5)
        k = rq(w.lin(h, f"{lp}.self_attn.k_proj"))
        v = rq(w.lin(h, f"{lp}.self_attn.v_proj"))
        s = (W._split_heads(q, H) @ W._split_heads(k, H).transpose(1, 2)).masked_fill(mask[None], float("-inf"))
        x = x + w.lin(W._merge_heads(torch.softmax(s, dim=-1) @ W._split_heads(v, H)), f"{lp}.self_attn.out_proj")
        h = w.ln(x, f"{lp}.encoder_attn_layer_norm")
        q = w.lin(h, f"{lp}.encoder_attn.q_proj") * (dh ** -0.5)
        ck = rq(w.lin(e, f"{lp}.encoder_attn.k_proj"))
        cv = rq(w.lin(e, f"{lp}.encoder_attn.v_proj"))
        sc = W._split_heads(q, H) @ W._split_heads(ck, H).transpose(1, 2)   # [H, n, S]
        a = torch.softmax(sc, dim=-1)
        for (l, hd) in pairs:
            if int(l) == li:
                keep[(li, int(hd))], raw[(li, int(hd))] = a[int(hd)], sc[int(hd)]
        x = x + w.lin(W._merge_heads(a @ W._split_heads(cv, H)), f"{lp}.encoder_attn.out_proj")
        h = w.ln(x, f"{lp}.final_layer_norm")
        x = x + w.lin(F.gelu(w.lin(h, f"{lp}.fc1")), f"{lp}.fc2")
    probs = torch.stack([keep[(int(l), int(hd))] for (l, hd) in pairs])
    if return_scores:
        return probs, torch.stack([raw[(int(l), int(hd))] for (l, hd) in pairs])
    return probs


def median_filter(x: torch.Tensor, width: int) -> torch.Tensor:
    """HF ``_median_filter``: along the last axis, reflect padding, unchanged when the axis is at most width // 2."""
    if width <= 0 or width % 2 != 1:
        raise ValueError("`filter_width` should be an odd number")
    pad = width // 2
    if x.shape[-1] <= pad:
        return x
    x = F.pad(x, (pad, pad, 0, 0), mode="reflect")
    return x.unfold(-1, width, 1).sort()[0][..., pad]


def alignment_matrix(probs: torch.Tensor, num_frames: Optional[int], filter_width: int = 7) -> torch.Tensor:
    """``probs [heads, N, W]`` (fp32, rows P .. n-2) -> the DTW input ``[N, F]``: crop to ``num_frames // 2``,
    normalise each (head, frame) column over the rows, median filter, mean over the heads."""
    m = probs.to(torch.float32)
    if num_frames is not None:
        m = m[..., : int(num_frames) // 2]
    std = torch.std(m, dim=-2, keepdim=True, unbiased=False)
    mean = torch.mean(m, dim=-2, keepdim=True)
    m = (m - mean) / std
    m = median_filter(m, filter_width)
    return m.mean(dim=0)


def dtw(matrix: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
    """HF ``_dynamic_time_warping(matrix)`` (the caller passes ``-matrix``): the cost over anti-diagonals, the same f32
    cost array, tie rule and backtrace.  Returns ``(text_indices, time_indices)``."""
    m = np.asarray(matrix, dtype=np.float64)
    N, Fr = m.shape
    cost = np.full((N + 1, Fr + 1), np.inf, dtype=np.float32)
    trace = -np.ones((N + 1, Fr + 1), dtype=np.float32)
    cost[0, 0] = 0
    for k in range(2, N + Fr + 1):
        i = np.arange(max(1, k - Fr), min(N, k - 1) + 1)
        if i.size == 0:
            continue
        j = k - i
        c0, c1, c2 = cost[i - 1, j - 1], cost[i - 1, j], cost[i, j - 1]
        t0 = (c0 < c1) & (c0 < c2)
        t1 = ~t0 & (c1 < c0) & (c1 < c2)
        c = np.where(t0, c0, np.where(t1, c1, c2))
        cost[i, j] = (m[i - 1, j - 1] + c.astype(np.float64)).astype(np.float32)
        trace[i, j] = np.where(t0, 0, np.where(t1, 1, 2))
    trace[0, :] = 2
    trace[:, 0] = 1
    i, j = N, Fr
    text, time = [], []
    while i > 0 or j > 0:
        text.append(i - 1)
        time.append(j - 1)
        t = trace[i, j]
        if t == 0:
            i, j = i - 1, j - 1
        elif t == 1:
            i -= 1
        else:
            j -= 1
    return np.array(text)[::-1], np.array(time)[::-1]


def jumps_of(text: np.ndarray, time: np.ndarray) -> np.ndarray:
    """The frame where the DTW path enters each text row (HF: ``time_indices[jumps]``)."""
    jumps = np.pad(np.diff(text), (1, 0), constant_values=1).astype(bool)
    return time[jumps]


def assemble(jump_frames: np.ndarray, n_prompt: int, time_precision: float) -> np.ndarray:
    """``[zeros(P), jump_times, jump_times[-1]]`` in f32, jump times = f32((double)frame * time_precision)."""
    jt = np.asarray(jump_frames, dtype=np.int64) * float(time_precision)
    return np.concatenate([np.zeros(n_prompt), jt, jt[-1:]]).astype(np.float32)


def extract(probs: torch.Tensor, n_prompt: int, num_frames: Optional[int] = None, filter_width: int = 7,
            time_precision: float = 0.02) -> Tuple[np.ndarray, Optional[torch.Tensor], Optional[np.ndarray]]:
    """Timestamps ``[P + N + 1]`` (f32) from the alignment rows ``probs [heads, N, W]`` of positions P .. n-2, with the
    matrix and the jump frames (None when N = 0: all zeros, as HF)."""
    N = int(probs.shape[1])
    if N == 0:
        return np.zeros(n_prompt + 1, dtype=np.float32), None, None
    mat = alignment_matrix(probs, num_frames, filter_width)
    text, time = dtw(-mat.double().numpy())
    j = jumps_of(text, time)
    return assemble(j, n_prompt, time_precision), mat, j


def pairs_list(alignment_heads: Sequence[Sequence[int]]) -> List[Tuple[int, int]]:
    return [(int(l), int(h)) for l, h in alignment_heads]
