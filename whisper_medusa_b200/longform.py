"""Host logic of long-form transcription: the window plan and the merge of the windows' token ids.

Both restate HF's chunked ASR pipeline (``pipeline("automatic-speech-recognition", ..., chunk_length_s=30)``) without
timestamps, so that a recording of any length transcribes as that pipeline would cut and stitch it:

* ``plan_windows`` is ``transformers.pipelines.automatic_speech_recognition.chunk_iter`` at 16 kHz: windows of
  ``chunk_len`` samples advancing by ``chunk_len - stride_left - stride_right``; the first window has no left stride,
  the last no right stride, and a window is kept only while it is longer than its left stride;
* ``merge_windows`` is ``transformers.models.whisper.tokenization_whisper._find_longest_common_sequence`` without
  token timestamps: consecutive windows are aligned where their ids agree best, the left window's ids are kept up to
  the middle of the overlap and the right window's from there on.

With ``no_speech_threshold`` and ``logprob_threshold``, a window is skipped by HF's no-speech rule (``skip_window``) and
contributes no ids to the merge.

The CPU tests pin both to the installed transformers; the package does not import it.
"""
from __future__ import annotations

import math
from typing import List, NamedTuple, Optional, Sequence, Tuple, Union

import numpy as np

SAMPLE_RATE = 16000
MAX_WINDOW_SAMPLES = 480000      # 30 s: what one encoder pass covers


class Window(NamedTuple):
    start: int           # first sample of the window in the 16 kHz recording
    end: int             # one past its last sample
    stride_left: int     # samples at its start that overlap the previous window (0 for the first)
    stride_right: int    # samples at its end that overlap the next window (0 for the last)


def window_params(chunk_length_s: float = 30.0,
                  stride_length_s: Optional[Union[float, Sequence[float]]] = None) -> Tuple[int, int, int]:
    """``(chunk_len, stride_left, stride_right)`` in 16 kHz samples, as HF's pipeline derives them (stride default:
    ``chunk_length_s / 6`` on each side).  Raises ``ValueError`` for a window longer than 30 s, a non-positive window,
    negative strides, or strides that leave no step (``chunk_len <= stride_left + stride_right``)."""
    chunk_length_s = float(chunk_length_s)
    if not math.isfinite(chunk_length_s) or chunk_length_s <= 0:
        raise ValueError(f"chunk_length_s must be positive, got {chunk_length_s}")
    chunk_len = int(round(chunk_length_s * SAMPLE_RATE))
    if chunk_len > MAX_WINDOW_SAMPLES:
        raise ValueError(f"chunk_length_s must be at most 30 s (one encoder window), got {chunk_length_s}")
    if stride_length_s is None:
        stride_length_s = chunk_length_s / 6
    if isinstance(stride_length_s, (int, float)):
        stride_length_s = [stride_length_s, stride_length_s]
    left, right = (int(round(float(s) * SAMPLE_RATE)) for s in stride_length_s)
    if left < 0 or right < 0:
        raise ValueError("stride_length_s must not be negative")
    if chunk_len < left + right:
        raise ValueError("Chunk length must be superior to stride length")           # HF's check and message
    if chunk_len == left + right:
        raise ValueError("Chunk length must be superior to stride length (the windows would not advance)")
    return chunk_len, left, right


def plan_windows(n_samples: int, chunk_len: int, stride_left: int, stride_right: int) -> List[Window]:
    """The windows HF ``chunk_iter`` yields for a recording of ``n_samples`` 16 kHz samples."""
    step = chunk_len - stride_left - stride_right
    if step <= 0:
        raise ValueError("Chunk length must be superior to stride length")
    out: List[Window] = []
    for start in range(0, int(n_samples), step):
        end = min(start + chunk_len, int(n_samples))
        left = 0 if start == 0 else stride_left
        is_last = start + chunk_len >= n_samples
        right = 0 if is_last else stride_right
        if end - start > left:
            out.append(Window(start, end, left, right))
        if is_last:
            break
    return out


def merge_windows(sequences: Sequence[Sequence[int]]) -> List[int]:
    """Longest-common-sequence merge of the windows' ids, left to right (no windows: no ids)."""
    if len(sequences) == 0:
        return []
    left = np.asarray(sequences[0], dtype=np.int64)
    total: List[int] = []
    for right_seq in sequences[1:]:
        right = np.asarray(right_seq, dtype=np.int64)
        n_l, n_r = len(left), len(right)
        best = 0.0
        best_idx = (n_l, n_l, 0, 0)
        for i in range(1, n_l + n_r):
            eps = i / 10000.0                      # favours long perfect matches
            l0, l1 = max(0, n_l - i), min(n_l, n_l + n_r - i)
            r0, r1 = max(0, i - n_l), min(n_r, i)
            matches = int(np.count_nonzero(left[l0:l1] == right[r0:r1]))
            matching = matches / i + eps
            if matches > 1 and matching > best:
                best = matching
                best_idx = (l0, l1, r0, r1)
        l0, l1, r0, r1 = best_idx
        # the left window is trusted for the first half of the overlap, the right window for the second
        total.extend(left[: (l0 + l1) // 2].tolist())
        left = right[(r0 + r1) // 2:]
    total.extend(left.tolist())
    return total


def text_ids(ids: Sequence[int], eos_token_id: int) -> List[int]:
    """A window's ids without the special and timestamp block (every id >= EOS in a Whisper vocabulary)."""
    return [int(t) for t in ids if int(t) < eos_token_id]


def no_speech_rule(no_speech_threshold, logprob_threshold) -> bool:
    """Check the no-speech arguments of ``transcribe``; True when windows are to be tested for silence.

    HF's rule needs both thresholds: ``no_speech_threshold`` alone raises ``ValueError`` (HF itself fails comparing
    with ``None`` there).  ``logprob_threshold`` alone means temperature fallback, which greedy-only Medusa decoding
    cannot do: ``NotImplementedError``.  Both must be finite numbers."""
    if no_speech_threshold is None and logprob_threshold is None:
        return False
    if logprob_threshold is None:
        raise ValueError("no_speech_threshold needs logprob_threshold: a window is skipped when its no-speech "
                         "probability is above the first and its average log-probability below the second")
    if no_speech_threshold is None:
        raise NotImplementedError("logprob_threshold without no_speech_threshold asks for temperature fallback, which "
                                  "is not supported with medusa (greedy search only)")
    for name, v in (("no_speech_threshold", no_speech_threshold), ("logprob_threshold", logprob_threshold)):
        if isinstance(v, bool) or not isinstance(v, (int, float, np.floating, np.integer)) or not math.isfinite(float(v)):
            raise ValueError(f"{name} must be a finite float, got {v!r}")
    return True


def skip_window(no_speech_prob: float, avg_logprob: float, no_speech_threshold: float,
                logprob_threshold: float) -> bool:
    """HF ``WhisperGenerationMixin._need_fallback``'s ``should_skip``: the window is silent when the probability of
    ``<|nospeech|>`` at the start-of-transcript position is above ``no_speech_threshold`` and the average log-probability
    of its tokens is below ``logprob_threshold`` (both strict)."""
    return avg_logprob < logprob_threshold and no_speech_prob > no_speech_threshold


def resampled_length(n: int, orig_hz: int, new_hz: int) -> int:
    """``ceil(n * new / orig)`` with the rates divided by their gcd (torchaudio's output length)."""
    g = math.gcd(int(orig_hz), int(new_hz))
    orig, new = int(orig_hz) // g, int(new_hz) // g
    return -(-int(n) * new // orig)


class WindowResult:
    """One window of a long-form transcription (``WhisperMedusaModel.last_windows``)."""

    def __init__(self, window: Window, ids: List[int], trace, no_speech_prob: Optional[float] = None,
                 avg_logprob: Optional[float] = None, skipped: Optional[bool] = None):
        self.start, self.end = window.start, window.end
        self.stride_left, self.stride_right = window.stride_left, window.stride_right
        self.ids = ids            # what generate() returns for the window (prompt and trailing EOS stripped)
        self.trace = trace        # its GenerateTrace
        # no-speech rule (transcribe(no_speech_threshold=..., logprob_threshold=...); all None without it)
        self.no_speech_prob = no_speech_prob
        self.avg_logprob = avg_logprob
        self.skipped = skipped    # True: the window counts as silence and adds no ids to the merge

    def merge_ids(self, eos_token_id: int) -> List[int]:
        """What the window contributes to ``merge_windows``: its text ids, or none for a skipped window (its
        neighbours are then both kept whole: no overlap is de-duplicated across it)."""
        return [] if self.skipped else text_ids(self.ids, eos_token_id)

    def __repr__(self) -> str:
        return (f"WindowResult(samples {self.start}:{self.end}, strides ({self.stride_left}, {self.stride_right}), "
                f"{len(self.ids)} ids)")
