"""fp64 numpy restatement of ``torchaudio.functional.resample`` with its defaults (``sinc_interp_hann``,
``lowpass_filter_width=6``, ``rolloff=0.99``) for integer rates: the oracle of the engine's resampler
(``csrc/resample.cu``).

The tap table follows torchaudio's ``_get_sinc_resample_kernel`` operation by operation in fp64 (its kernel for an
fp64 waveform) with ``math.sin`` / ``math.cos``, and is rounded once to fp32, as the engine does.  (For an fp32
waveform torchaudio evaluates the same formula in fp32 arithmetic, which moves its output by up to ~1e-5.)  The
convolution (``_apply_sinc_resample_kernel``: zero padding of ``width`` on the left and ``width + orig`` on the right,
stride ``orig``) then runs in fp64 on those fp32 taps.
"""
from __future__ import annotations

import math
from typing import Tuple

import numpy as np

LOWPASS_FILTER_WIDTH = 6
ROLLOFF = 0.99


def reduced_rates(orig_hz: int, new_hz: int) -> Tuple[int, int]:
    g = math.gcd(int(orig_hz), int(new_hz))
    return int(orig_hz) // g, int(new_hz) // g


def sinc_taps(orig_hz: int, new_hz: int) -> Tuple[np.ndarray, int]:
    """fp32 kernel ``[new, 2 * width + orig]`` (torchaudio's ``kernel[:, 0, :]``) and ``width``."""
    orig, new = reduced_rates(orig_hz, new_hz)
    base = min(orig, new)
    base *= ROLLOFF
    width = math.ceil(LOWPASS_FILTER_WIDTH * orig / base)
    scale = base / orig
    cols = 2 * width + orig
    idx = np.arange(-width, width + orig, dtype=np.float64) / orig
    out = np.empty((new, cols), dtype=np.float32)
    for p in range(new):
        t0 = -p / new
        t = (t0 + idx) * base
        t = np.clip(t, -LOWPASS_FILTER_WIDTH, LOWPASS_FILTER_WIDTH)
        w = np.array([math.cos(v) for v in t * math.pi / LOWPASS_FILTER_WIDTH / 2])
        w = w * w
        t = t * math.pi
        k = np.array([1.0 if v == 0 else math.sin(v) / v for v in t])
        k = k * (w * scale)
        out[p] = k.astype(np.float32)
    return out, width


def resampled_length(n: int, orig_hz: int, new_hz: int) -> int:
    orig, new = reduced_rates(orig_hz, new_hz)
    return -(-int(n) * new // orig)


def resample(x: np.ndarray, orig_hz: int, new_hz: int) -> np.ndarray:
    """1-D samples at ``orig_hz`` -> fp64 samples at ``new_hz``."""
    x = np.asarray(x, dtype=np.float64).reshape(-1)
    if orig_hz == new_hz:
        return x.copy()
    orig, new = reduced_rates(orig_hz, new_hz)
    taps, width = sinc_taps(orig_hz, new_hz)
    n = x.shape[0]
    m = resampled_length(n, orig_hz, new_hz)
    if m == 0:
        return np.zeros(0)
    n_blocks = -(-m // new)
    cols = taps.shape[1]
    xp = np.zeros((n_blocks - 1) * orig + cols)
    xp[width:width + n] = x[: len(xp) - width]
    y = np.zeros((n_blocks, new))
    span = (n_blocks - 1) * orig + 1
    for p in range(new):
        for c in np.flatnonzero(taps[p]):      # the zero taps outside each phase's support add nothing
            y[:, p] += float(taps[p, c]) * xp[c: c + span: orig]
    return y.reshape(-1)[:m]
