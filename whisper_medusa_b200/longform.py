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

Token timestamps (``transcribe(return_token_timestamps=True)``) restate what HF's ``tokenization_whisper._decode_asr``
does with ``return_timestamps="word"`` for windows without timestamp tokens: ``window_offsets`` places each window on the
recording's time axis, ``token_pairs`` turns its token times into ``(start, end)`` pairs, and ``merge_windows`` with
``pairs`` is ``_find_longest_common_sequence(sequences, token_timestamp_sequences)``, whose match rule is stricter
(equal ids whose times are in order), so its ids can differ from the untimed merge's.

With a temperature schedule and ``compression_ratio_threshold`` / ``logprob_threshold``, a window is decoded again by
sampling at the schedule's next temperature while its result needs fallback (``fallback_rule``, ``needs_fallback``:
HF's ``generate_with_fallback`` and ``_need_fallback``).

The CPU tests pin all of it to the installed transformers; the package does not import it.
"""
from __future__ import annotations

import math
import zlib
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


Pair = Tuple[float, float]


def merge_windows(sequences: Sequence[Sequence[int]], pairs: Optional[Sequence[Sequence[Pair]]] = None):
    """Longest-common-sequence merge of the windows' ids, left to right (no windows: no ids).

    ``pairs``: one ``(start, end)`` per id of every window (``token_pairs``).  A position of the overlap then matches only
    when the ids are equal and the left window's pair is ``<=`` the right window's (Python's tuple order, as HF compares
    them), and the pairs are cut where the ids are; returns ``(ids, pairs)`` instead of ``ids``."""
    timed = pairs is not None
    if len(sequences) == 0:
        return ([], []) if timed else []
    left = np.asarray(sequences[0], dtype=np.int64)
    total: List[int] = []
    if timed:
        left_p = [tuple(p) for p in pairs[0]]
        total_p: List[Pair] = []
    for k, right_seq in enumerate(sequences[1:], start=1):
        right = np.asarray(right_seq, dtype=np.int64)
        n_l, n_r = len(left), len(right)
        # Shift i (1 <= i < n_l + n_r) lays the last i ids of the left window over the first ones of the right window:
        # left[a] faces right[b] where b - a = i - n_l.  Its match count is the sum of that diagonal of the match matrix.
        same = left[:, None] == right[None, :]
        if timed:     # (ls, le) <= (rs, re) in tuple order
            right_p = [tuple(p) for p in pairs[k]]
            ls, le = (np.array([p[j] for p in left_p], dtype=np.float64).reshape(-1, 1) for j in (0, 1))
            rs, re = (np.array([p[j] for p in right_p], dtype=np.float64).reshape(1, -1) for j in (0, 1))
            same &= (ls < rs) | ((ls == rs) & (le <= re))
        diag = (np.arange(n_r)[None, :] - np.arange(n_l)[:, None] + n_l - 1).ravel()       # = i - 1
        matches = np.bincount(diag, weights=same.ravel(), minlength=max(0, n_l + n_r - 1)).astype(np.int64)
        i = np.arange(1, n_l + n_r)
        matching = matches / i + i / 10000.0       # the second term favours long perfect matches
        matching[matches <= 1] = -np.inf
        best_idx = (n_l, n_l, 0, 0)
        if len(i) and matching.max() > 0.0:        # the first shift of the largest score, as a strict left-to-right scan
            i = int(i[int(np.argmax(matching))])
            best_idx = (max(0, n_l - i), min(n_l, n_l + n_r - i), max(0, i - n_l), min(n_r, i))
        l0, l1, r0, r1 = best_idx
        # the left window is trusted for the first half of the overlap, the right window for the second
        total.extend(left[: (l0 + l1) // 2].tolist())
        left = right[(r0 + r1) // 2:]
        if timed:
            total_p.extend(left_p[: (l0 + l1) // 2])
            left_p = right_p[(r0 + r1) // 2:]
    total.extend(left.tolist())
    if timed:
        total_p.extend(left_p)
        return total, total_p
    return total


def window_offsets(windows: Sequence) -> List[float]:
    """Where each window starts on the recording's time axis, in seconds, as HF's ``_decode_asr`` accumulates it
    (``window``: anything with ``start``, ``end``, ``stride_left`` and ``stride_right`` in 16 kHz samples).  The strides
    are in seconds, as the pipeline's ``postprocess`` converts them; the offset drops by the left stride before a
    window and grows by its length less its right stride after it, in the same order and in Python floats."""
    offset, out = 0.0, []
    for w in windows:
        offset -= w.stride_left / SAMPLE_RATE
        out.append(offset)
        offset += (w.end - w.start) / SAMPLE_RATE - w.stride_right / SAMPLE_RATE
    return out


def token_pairs(ids: Sequence[int], times: Sequence[float], offset: float, eos_token_id: int) -> List[Pair]:
    """``(start, end)`` in recording seconds of every text id of a window (``text_ids``' ids, in order), as HF's
    ``_decode_asr`` forms them: ``start = round(times[i - 1] + offset, 2)`` (``round(0.0 + offset, 2)`` at ``i = 0``) and
    ``end = round(times[i] + offset, 2)``.  ``ids`` and ``times`` are what ``generate(..., return_token_timestamps=True)``
    returns for the window: HF's short-form ``sequences`` and ``token_timestamps`` carry no decoder prompt either, so
    ``i`` indexes the same list here as there (the prompt's times are 0.0, so ``i = 0`` gives the same start either
    way)."""
    out: List[Pair] = []
    for i, t in enumerate(ids):
        if int(t) < eos_token_id:
            start = round(0.0 + offset, 2) if i == 0 else round(float(times[i - 1]) + offset, 2)
            out.append((start, round(float(times[i]) + offset, 2)))
    return out


def merge_timed(results: Sequence["WindowResult"], eos_token_id: int) -> Tuple[List[int], List[Pair]]:
    """The timed merge of a transcription's windows (``WindowResult`` with ``token_timestamps``): every window is
    placed by ``window_offsets``; a skipped window takes part as an empty one, as in the untimed merge."""
    seqs, pairs = [], []
    for r, offset in zip(results, window_offsets(results)):
        if r.skipped:
            seqs.append([])
            pairs.append([])
        else:
            seqs.append(text_ids(r.ids, eos_token_id))
            pairs.append(token_pairs(r.ids, r.token_timestamps.reshape(-1).tolist(), offset, eos_token_id))
    return merge_windows(seqs, pairs)


def text_ids(ids: Sequence[int], eos_token_id: int) -> List[int]:
    """A window's ids without the special and timestamp block (every id >= EOS in a Whisper vocabulary)."""
    return [int(t) for t in ids if int(t) < eos_token_id]


def no_speech_rule(no_speech_threshold, logprob_threshold) -> bool:
    """Check the no-speech arguments of ``transcribe``; True when windows are to be tested for silence.

    HF's rule needs both thresholds: ``no_speech_threshold`` alone raises ``ValueError`` (HF itself fails comparing
    with ``None`` there).  ``logprob_threshold`` alone means temperature fallback, which needs a temperature schedule
    (``fallback_rule``; callers with one do not pass it here): ``NotImplementedError``.  Both must be finite numbers."""
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


# largest top_k of a sampled attempt other than 0 (the whole vocabulary): the engine's per-segment candidate lists
MAX_TOP_K = 64


class Fallback(NamedTuple):
    """Temperature fallback of ``transcribe``: the schedule (first entry 0.0) and the thresholds (None = not tested)."""
    temperatures: Tuple[float, ...]
    compression_ratio_threshold: Optional[float]
    logprob_threshold: Optional[float]
    top_k: int                # 0 = the whole vocabulary


def _finite(name: str, v) -> float:
    if isinstance(v, bool) or not isinstance(v, (int, float, np.floating, np.integer)) or not math.isfinite(float(v)):
        raise ValueError(f"{name} must be a finite float, got {v!r}")
    return float(v)


def fallback_rule(temperature, compression_ratio_threshold, logprob_threshold, top_k, vocab_size: int,
                  default_top_k=None) -> Optional[Fallback]:
    """Check the temperature-fallback arguments of ``transcribe``; the fallback to run, or None.

    A schedule is a tuple or list of finite temperatures >= 0 (``None`` entries are 0.0) whose first entry is 0.0: the
    first attempt is the window's ordinary decode.  A first entry above 0 raises ``NotImplementedError`` (as a scalar
    temperature does); a negative, infinite or NaN entry ``ValueError``.  A fallback needs a schedule of two or more
    entries and at least one threshold; with neither threshold, or with one entry, only the first entry runs (HF), and
    ``compression_ratio_threshold`` without a schedule raises ``NotImplementedError``.  ``top_k``: the call's, else
    ``default_top_k`` (the generation config's), else 50 (HF); 0 or at least ``vocab_size`` is the whole vocabulary, and
    1 .. 64 is supported.  The call's ``top_k`` without a fallback to sample in raises ``NotImplementedError``, as an
    option the engine does not honour.  Scalar temperatures are left to the caller's sampling refusal."""
    no_sampling = NotImplementedError("top_k is only used by the sampled attempts of temperature fallback: pass a "
                                      "temperature schedule and compression_ratio_threshold / logprob_threshold")
    if not isinstance(temperature, (tuple, list)):
        if compression_ratio_threshold is not None:
            raise NotImplementedError("compression_ratio_threshold asks for temperature fallback: pass a temperature "
                                      "schedule, e.g. temperature=(0.0, 0.2, 0.4, 0.6, 0.8, 1.0)")
        if top_k is not None:
            raise no_sampling
        return None
    if len(temperature) == 0:
        raise ValueError("the temperature schedule is empty")
    temps = tuple(0.0 if t is None else _finite("temperature", t) for t in temperature)
    if any(t < 0 for t in temps):
        raise ValueError(f"temperatures must be >= 0, got {temps}")
    if temps[0] != 0.0:
        raise NotImplementedError("sampling (temperature > 0 / do_sample) is not supported with medusa: the first entry "
                                  "of a temperature schedule must be 0.0 (greedy search); sampling runs only on fallback")
    crt = None if compression_ratio_threshold is None else _finite("compression_ratio_threshold", compression_ratio_threshold)
    lpt = None if logprob_threshold is None else _finite("logprob_threshold", logprob_threshold)
    if len(temps) == 1 or (crt is None and lpt is None):
        if top_k is not None:
            raise no_sampling
        return None                 # HF: nothing to fall back to, the first entry is the decode
    k = top_k if top_k is not None else (default_top_k if default_top_k is not None else 50)
    if isinstance(k, bool) or not isinstance(k, (int, np.integer)) or k < 0:
        raise ValueError(f"top_k must be a non-negative integer, got {k!r}")
    k = 0 if int(k) >= vocab_size else int(k)
    if k > MAX_TOP_K:
        raise NotImplementedError(f"top_k must be at most {MAX_TOP_K}, 0 or at least the vocabulary size, got {k}")
    return Fallback(temps, crt, lpt, k)


def compression_ratio(ids: Sequence[int], vocab_size: int) -> float:
    """HF ``_retrieve_compression_ratio``: the ids as little-endian integers of ``int(log2(vocab) / 8) + 1`` bytes, over
    their zlib-compressed length."""
    length = int(math.log2(vocab_size) / 8) + 1
    token_bytes = b"".join(int(t).to_bytes(length, "little") for t in ids)
    return len(token_bytes) / len(zlib.compress(token_bytes))


def needs_fallback(ratio: float, avg_logprob: float, fb: Fallback) -> bool:
    """HF ``_need_fallback`` without the no-speech rule: the compression ratio above its threshold, or the average
    log-probability below its threshold (both strict)."""
    return ((fb.compression_ratio_threshold is not None and ratio > fb.compression_ratio_threshold)
            or (fb.logprob_threshold is not None and avg_logprob < fb.logprob_threshold))


def resampled_length(n: int, orig_hz: int, new_hz: int) -> int:
    """``ceil(n * new / orig)`` with the rates divided by their gcd (torchaudio's output length)."""
    g = math.gcd(int(orig_hz), int(new_hz))
    orig, new = int(orig_hz) // g, int(new_hz) // g
    return -(-int(n) * new // orig)


class WindowResult:
    """One window of a long-form transcription (``WhisperMedusaModel.last_windows``)."""

    def __init__(self, window: Window, ids: List[int], trace, no_speech_prob: Optional[float] = None,
                 avg_logprob: Optional[float] = None, skipped: Optional[bool] = None, token_timestamps=None,
                 num_frames: Optional[int] = None, temperature: Optional[float] = None,
                 compression_ratio: Optional[float] = None, attempts: Optional[List[Tuple[float, float, float]]] = None):
        self.start, self.end = window.start, window.end
        self.stride_left, self.stride_right = window.stride_left, window.stride_right
        self.ids = ids            # what generate() returns for the window (prompt and trailing EOS stripped)
        self.trace = trace        # its GenerateTrace
        # no-speech rule (transcribe(no_speech_threshold=..., logprob_threshold=...); all None without it)
        self.no_speech_prob = no_speech_prob
        self.avg_logprob = avg_logprob
        self.skipped = skipped    # True: the window counts as silence and adds no ids to the merge
        # transcribe(return_token_timestamps=True); both None without it
        self.token_timestamps = token_timestamps   # FloatTensor[1, len(ids)], seconds from the window's start
        self.num_frames = num_frames               # feature frames the alignment was cropped to
        # temperature fallback (transcribe(temperature=(0.0, ...), ...)); all None without it: the kept attempt's
        # temperature and compression ratio, and (temperature, compression_ratio, avg_logprob) of every attempt
        self.temperature = temperature
        self.compression_ratio = compression_ratio
        self.attempts = attempts

    def merge_ids(self, eos_token_id: int) -> List[int]:
        """What the window contributes to ``merge_windows``: its text ids, or none for a skipped window (its
        neighbours are then both kept whole: no overlap is de-duplicated across it)."""
        return [] if self.skipped else text_ids(self.ids, eos_token_id)

    def __repr__(self) -> str:
        return (f"WindowResult(samples {self.start}:{self.end}, strides ({self.stride_left}, {self.stride_right}), "
                f"{len(self.ids)} ids)")
