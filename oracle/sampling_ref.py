"""CPU ORACLE of the sampled attempts of temperature fallback (test infrastructure -- never imported by the product path).

* ``philox4x32_10`` / ``gumbel``: the engine's counter-based noise (``csrc/common.cuh`` ``sample_gumbel``) restated in
  numpy, bit for bit: word ``j % 4`` of Philox4x32-10(key = the seed's words, counter = (j / 4, n, window, attempt)),
  ``u = ((x >> 8) + 0.5) 2^-24`` and ``g = -log(-log u)`` in float64, rounded once to float32.
* ``choose``: the Gumbel-max choice of one processed fp32 row at temperature T over its top-k set
  ``{j : row_j >= tau}`` (tau = the k-th largest value, ties kept, HF ``TopKLogitsWarper``), ties on the sum to the
  lowest index.  ``exact_probs`` is the distribution it samples: ``softmax(row / T)`` over the same set.
* ``fallback``: HF ``generate_with_fallback`` / ``_need_fallback`` for one window, over a callable that decodes one
  attempt.
* ``sampled_search``: ``medusa_ref.medusa_greedy_search``'s loop on a chain with the sampled choice, and
  ``one_token_search``: the one-token-at-a-time Gumbel-max decode it must equal.  Both record the token
  log-probabilities over each token's top-k set (what the scores kernel gives a sampled attempt) and the smallest
  margin of any choice, for the near-tie accounting of the GPU comparison.
"""
from __future__ import annotations

import math
from typing import Callable, List, Optional, Sequence, Tuple

import numpy as np

_M0, _M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
_W0, _W1 = np.uint32(0x9E3779B9), np.uint32(0xBB67AE85)
_LO = np.uint64(0xFFFFFFFF)


def philox4x32_10(counter, key) -> np.ndarray:
    """Philox4x32-10 of counters ``[..., 4]`` (uint32) under ``key`` (two uint32): ``[..., 4]`` uint32."""
    c = np.asarray(counter, dtype=np.uint32).astype(np.uint64)
    k0, k1 = np.uint32(key[0]), np.uint32(key[1])
    with np.errstate(over="ignore"):
        for i in range(10):
            if i:
                k0, k1 = np.uint32(k0 + _W0), np.uint32(k1 + _W1)
            p0, p1 = _M0 * c[..., 0], _M1 * c[..., 2]
            c = np.stack([((p1 >> np.uint64(32)) ^ c[..., 1] ^ np.uint64(k0)) & _LO, p1 & _LO,
                          ((p0 >> np.uint64(32)) ^ c[..., 3] ^ np.uint64(k1)) & _LO, p0 & _LO], axis=-1)
    return c.astype(np.uint32)


def gumbel(seed: Tuple[int, int], window: int, attempt: int, n: int, js) -> np.ndarray:
    """The noise of tokens ``js`` at position ``n``: float32, as the engine computes it."""
    js = np.asarray(js, dtype=np.int64)
    ctr = np.stack([js >> 2, np.full_like(js, n), np.full_like(js, window), np.full_like(js, attempt)], axis=-1)
    x = philox4x32_10(ctr.astype(np.uint32), seed)
    w = x[np.arange(len(js)), js & 3]
    u = ((w >> np.uint32(8)).astype(np.float64) + 0.5) * 2.0 ** -24
    return (-np.log(-np.log(u))).astype(np.float32)


def top_k_tau(row: np.ndarray, top_k: int) -> float:
    """The k-th largest value of ``row`` (k = min(top_k, V)); -inf for top_k = 0 (the whole row)."""
    if top_k == 0 or top_k >= len(row):
        return -math.inf
    return float(np.sort(row)[::-1][top_k - 1])


def choose(row: np.ndarray, temperature: float, top_k: int, noise: np.ndarray) -> Tuple[int, float]:
    """Gumbel-max choice of a processed fp32 row: ``(index, tau)``."""
    row = np.asarray(row, dtype=np.float32)
    tau = top_k_tau(row, top_k)
    s = (row / np.float32(temperature)).astype(np.float32) + noise.astype(np.float32)
    s = np.where(row >= tau, s, -np.inf).astype(np.float32)
    return int(np.argmax(s)), tau       # (np.argmax: the first maximum)


def exact_probs(row: np.ndarray, temperature: float, top_k: int) -> np.ndarray:
    """``softmax(row / T)`` over the top-k set, in float64."""
    row = np.asarray(row, dtype=np.float64)
    tau = top_k_tau(np.asarray(row, dtype=np.float32), top_k)
    z = np.where(row >= tau, row / temperature, -np.inf)
    p = np.exp(z - z.max())
    return p / p.sum()


def fallback(decode: Callable[[int, float], Tuple[List[int], float, float]], temperatures: Sequence[float],
             compression_ratio_threshold: Optional[float], logprob_threshold: Optional[float],
             no_speech_threshold: Optional[float] = None, no_speech_prob: Optional[float] = None, vocab_size: int = 51865):
    """HF ``generate_with_fallback`` for one window.  ``decode(attempt, temperature)`` returns ``(seek_sequence,
    avg_logprob, compression_ratio or None)``; returns ``(kept attempt index, skipped, [(T, ratio, avg_logprob)])``."""
    import zlib

    attempts = []
    kept, skipped = len(temperatures) - 1, False
    for a, t in enumerate(temperatures):
        seq, avg, ratio = decode(a, t)
        if ratio is None:
            length = int(math.log2(vocab_size) / 8) + 1
            b = b"".join(int(x).to_bytes(length, "little") for x in seq)
            ratio = len(b) / len(zlib.compress(b))
        attempts.append((float(t), ratio, avg))
        needs = False
        if compression_ratio_threshold is not None and ratio > compression_ratio_threshold:
            needs = True
        if logprob_threshold is not None and avg < logprob_threshold:
            needs = True
        if no_speech_threshold is not None and logprob_threshold is not None:
            if avg < logprob_threshold and no_speech_prob > no_speech_threshold:
                needs, skipped = False, True
        if not needs:
            kept = a
            break
    return kept, skipped, attempts


# --------------------------------------------------------------------------------------
# the sampled loop and its one-token-at-a-time restatement
# --------------------------------------------------------------------------------------
class SampledTrace:
    def __init__(self, sequences):
        self.sequences = sequences
        self.accept_lengths: List[int] = []
        self.iters = 0
        self.token_logprobs: List[float] = []   # log_softmax at T = 1 over each emitted token's top-k set
        self.token_scales: List[float] = []     # max(1, max |finite logit|) of each token's row
        self.min_gap = math.inf                  # smallest perturbed margin of a choice that decided a token


def _choice(row, temperature: float, top_k: int, seed, window: int, attempt: int, n: int, tr: SampledTrace):
    """Choice of processed row ``row`` (torch) for position n; records its margin and returns (index, tau)."""
    r = row.detach().float().numpy()
    g = gumbel(seed, window, attempt, n, np.arange(len(r)))
    idx, tau = choose(r, temperature, top_k, g)
    s = np.where(r >= tau, (r / np.float32(temperature)).astype(np.float32) + g, -np.inf)
    top2 = np.sort(s)[-2:]
    tr.min_gap = min(tr.min_gap, float(top2[1] - top2[0]) * temperature)
    if np.isfinite(tau):      # the k-th and (k+1)-th values decide the set
        srt = np.sort(r)[::-1]
        kk = int(top_k)
        if kk < len(srt) and np.isfinite(srt[kk]):
            tr.min_gap = min(tr.min_gap, float(srt[kk - 1] - srt[kk]) if srt[kk - 1] != srt[kk] else math.inf)
    return idx, tau


def _restricted_logprob(row, tau: float, tok: int) -> float:
    z = row.detach().double().numpy()
    z = np.where(z >= tau, z, -np.inf)
    m = z.max()
    return float(z[tok] - (m + np.log(np.exp(z - m).sum())))


def sampled_search(w, cfg, enc, prompt: Sequence[int], gp, temperature: float, top_k: int, seed, window: int,
                   attempt: int, regime: str = "fp32", max_iters: Optional[int] = None) -> SampledTrace:
    """``medusa_ref.medusa_greedy_search`` on a chain with the sampled choice: c0 is the Gumbel-max choice of the
    processed base row at position L, the heads propose their argmax, verify row r's choice at position L + r + 1
    decides whether cand[r + 1] is accepted, and verify row 0's choice is the extra token of an accept-0 iteration."""
    import torch

    from . import medusa_ref as M
    from . import whisper_ref as W

    H = cfg.medusa_num_heads
    assert all(int(c) == 1 for c in cfg.medusa_choices), "chains only"
    ids = [int(t) for t in prompt]
    cache = W.new_cache(cfg)
    tr = SampledTrace(ids)
    unfinished = True
    key = (temperature, top_k, seed, window, attempt)
    while True:
        L = len(ids)
        kv = cache.length
        hidden = W.decoder_forward(w, cfg, ids[kv:], list(range(kv, L)), enc, cache, regime)
        rows = M.process_logits(W.medusa_logits(w, cfg, hidden, enc, cache, False, regime)[:, -1, :], L, gp)
        c0, tau0 = _choice(rows[0], *key, L, tr)
        cand = [c0] + [int(torch.argmax(rows[1 + h])) for h in range(H)]
        vcache = cache.clone()
        hidden_b = W.decoder_forward(w, cfg, cand, list(range(L, L + H + 1)), enc, vcache, regime)
        rows_b = M.process_logits(W.medusa_logits(w, cfg, hidden_b, enc, vcache, True, regime)[0], L, gp)
        ch = [_choice(rows_b[r], *key, L + r + 1, tr) for r in range(H)]
        accept = 0
        while accept < H and cand[accept + 1] == ch[accept][0]:
            accept += 1
        new = cand[: accept + 1] + ([ch[0][0]] if accept == 0 else [])
        taus = [tau0] + [c[1] for c in ch]
        srcs = [rows[0]] + [rows_b[r] for r in range(H)]
        if unfinished:
            tr.token_logprobs += [_restricted_logprob(srcs[j], taus[j], t) for j, t in enumerate(new)]
            tr.token_scales += [max(1.0, float(srcs[j][srcs[j].isfinite()].abs().max())) for j in range(len(new))]
        else:
            new = [gp.pad_token_id] * len(new)
        ids = ids + new
        keep = 1 if accept == 0 else accept
        vcache.keep_rows(L, list(range(L, L + keep)))
        cache = vcache
        tr.accept_lengths.append(accept)
        tr.iters += 1
        if gp.eos_token_id in new or len(ids) >= gp.max_length:
            unfinished = False
        if (not unfinished) or len(ids) + H >= gp.max_length:
            break
        if max_iters is not None and tr.iters >= max_iters:
            break
    if gp.eos_token_id in ids:
        j = ids.index(gp.eos_token_id)
        ids = ids[: j + 1] + [gp.eos_token_id] * (len(ids) - j - 1)
    tr.sequences = ids
    return tr


def one_token_search(w, cfg, enc, prompt: Sequence[int], gp, temperature: float, top_k: int, seed, window: int,
                     attempt: int, max_new: int, regime: str = "fp32") -> List[int]:
    """One token per step: the Gumbel-max choice of the processed base row at position len(ids), until EOS or
    ``max_new`` tokens."""
    from . import medusa_ref as M
    from . import whisper_ref as W

    ids = [int(t) for t in prompt]
    cache = W.new_cache(cfg)
    tr = SampledTrace(ids)
    for _ in range(max_new):
        L = len(ids)
        hidden = W.decoder_forward(w, cfg, ids[cache.length:], list(range(cache.length, L)), enc, cache, regime)
        row = M.process_logits(W.medusa_logits(w, cfg, hidden, enc, cache, True, regime)[0, -1:, :], L, gp)[0]
        tok, _ = _choice(row, temperature, top_k, seed, window, attempt, L, tr)
        ids.append(tok)
        if tok == gp.eos_token_id:
            break
    return ids
