"""Logits processors of ``generate``: ``sequence_bias``, ``bad_words_ids``, ``no_repeat_ngram_size``, ``min_length`` and
``min_new_tokens``, as HF's ``SequenceBiasLogitsProcessor``, ``NoBadWordsLogitsProcessor``,
``NoRepeatNGramLogitsProcessor``, ``MinLengthLogitsProcessor`` and ``MinNewTokensLengthLogitsProcessor`` apply them.

This module checks the options (with the exception types of the HF processors' argument checks) and turns them into
the tables of ``wm_set_logits_processors``; the engine applies them on the GPU (``csrc/logits_proc.cu``).  The package
does not import transformers; the CPU tests pin these checks and the processing to the installed HF processors.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Any, Dict, List, Optional, Sequence, Tuple

import numpy as np

KEYS = ("sequence_bias", "bad_words_ids", "no_repeat_ngram_size", "min_length", "min_new_tokens")
MAX_SEQS = 256        # sequences of two or more tokens (WM_LP_MAX_SEQS)
MAX_TOKENS = 4096     # their tokens in all (WM_LP_MAX_TOKENS)


@dataclass
class Processors:
    """What ``wm_set_logits_processors`` takes: ``seqs`` in chain order (the sequence_bias entries in dict order, then
    the bad words with ``-inf``), ``ngram`` = no_repeat_ngram_size (0 = off) and ``eos_min_length``: EOS is banned
    while ``len(input_ids)`` is below it."""

    seqs: List[Tuple[Tuple[int, ...], float]]
    ngram: int
    eos_min_length: int


def options(kwargs: Dict[str, Any], g) -> Dict[str, Any]:
    """The five options of one call: a ``generate`` kwarg wins over the generation config's attribute."""
    return {k: kwargs[k] if kwargs.get(k) is not None else getattr(g, k, None) for k in KEYS}


def _is_int(v) -> bool:
    return isinstance(v, (int, np.integer))


def _sequence_bias_dict(sequence_bias) -> Dict[Tuple[int, ...], float]:
    """HF ``SequenceBiasLogitsProcessor._validate_arguments`` (ValueError) and ``_convert_list_arguments_into_dict``."""
    sb = sequence_bias
    if not isinstance(sb, dict) and not isinstance(sb, list) or len(sb) == 0:
        raise ValueError(f"`sequence_bias` has to be a non-empty dictionary, or non-empty list of lists but is {sb}.")
    if isinstance(sb, dict):
        if any(not isinstance(ids, tuple) for ids in sb):
            raise ValueError(f"`sequence_bias` has to be a dict with tuples as keys, but is {sb}.")
        if any(any(not _is_int(t) or t < 0 for t in ids) or len(ids) == 0 for ids in sb):
            raise ValueError(f"Each key in `sequence_bias` has to be a non-empty tuple of positive integers, but is {sb}.")
        if any(not isinstance(v, float) for v in sb.values()):
            raise ValueError(f"`sequence_bias` has to be a dict with floats as values, but is {sb}.")
        return dict(sb)

    def pair_ok(seq):
        return isinstance(seq[0], list) and all(_is_int(t) and t > 0 for t in seq[0]) and isinstance(seq[1], float)

    if any((not pair_ok(seq)) or len(seq) == 0 for seq in sb):
        raise ValueError(f"Each element in `sequence_bias` has to be a non-empty list of lists of positive integers and "
                         f"float, but is {sb}.")
    return {tuple(s[0]): s[1] for s in sb}


def _bad_words_dict(bad_words_ids, eos: int) -> Dict[Tuple[int, ...], float]:
    """HF ``NoBadWordsLogitsProcessor``: its argument checks (ValueError), the ``[eos]`` filter, ``-inf`` biases."""
    bw = bad_words_ids
    if not isinstance(bw, list) or len(bw) == 0:
        raise ValueError(f"`bad_words_ids` has to be a non-empty list, but is {bw}.")
    if any(not isinstance(w, list) for w in bw):
        raise ValueError(f"`bad_words_ids` has to be a list of lists, but is {bw}.")
    if any(any(not _is_int(t) or t < 0 for t in w) for w in bw):
        raise ValueError(f"Each list in `bad_words_ids` has to be a list of positive integers, but is {bw}.")
    if any(len(w) == 0 for w in bw):
        raise ValueError(f"`bad_words_ids` holds an empty list: {bw}.")
    return {tuple(w): float("-inf") for w in bw if w != [eos]}


def build(opts: Dict[str, Any], eos: int, vocab_size: int, prompt_len: int, max_length: int,
          penalty: Optional[Sequence] = None) -> Optional[Processors]:
    """Check the options of one call and build its tables; ``None`` when no processor is on (HF's conditions:
    ``no_repeat_ngram_size``, ``min_length`` and ``min_new_tokens`` only count when > 0).  ``prompt_len`` is the
    decoder prompt's length (``min_new_tokens`` counts from its end), ``penalty`` the call's
    ``exponential_decay_length_penalty``.  Raises before any GPU work."""
    seqs: List[Tuple[Tuple[int, ...], float]] = []
    if opts.get("sequence_bias") is not None:
        for ids, v in _sequence_bias_dict(opts["sequence_bias"]).items():
            if math.isnan(v) or v == math.inf:
                raise ValueError(f"sequence_bias value {v} for {list(ids)}: biases must be finite or -inf")
            seqs.append((tuple(int(t) for t in ids), float(v)))
    if opts.get("bad_words_ids") is not None:
        seqs += [(tuple(int(t) for t in ids), v) for ids, v in _bad_words_dict(opts["bad_words_ids"], eos).items()]
    bad = sorted({t for ids, _ in seqs for t in ids if t >= vocab_size})
    if bad:
        raise ValueError(f"The model vocabulary size is {vocab_size}, but the following tokens were being biased: {bad}")
    multi = [ids for ids, _ in seqs if len(ids) > 1]
    if len(multi) > MAX_SEQS or sum(len(ids) for ids in multi) > MAX_TOKENS:
        raise NotImplementedError(f"sequence_bias / bad_words_ids: at most {MAX_SEQS} sequences of two or more tokens "
                                  f"and {MAX_TOKENS} tokens among them are supported")
    ngram = opts.get("no_repeat_ngram_size")
    if ngram is not None and ngram > 0:
        if not isinstance(ngram, int):
            raise ValueError(f"`ngram_size` has to be a strictly positive integer, but is {ngram}")
    else:
        ngram = 0
    eos_min = 0
    min_length = opts.get("min_length")
    if min_length is not None and min_length > 0:
        if not isinstance(min_length, int):
            raise ValueError(f"`min_length` has to be a non-negative integer, but is {min_length}")
        eos_min = int(min_length)
    min_new = opts.get("min_new_tokens")
    if min_new is not None and min_new > 0:
        if not isinstance(min_new, int):
            raise ValueError(f"`min_new_tokens` has to be a positive integer, but is {min_new}")
        eos_min = max(eos_min, prompt_len + int(min_new))
    if not seqs and not ngram and eos_min <= 0:
        return None
    if penalty is not None:
        # The reference adds |-inf| * (factor^k - 1) to a banned EOS inside the penalty region (cur_len > start +
        # prompt): NaN whenever factor >= 1.  The engine does not reproduce that NaN row; it refuses the combination.
        reg = int(penalty[0]) + prompt_len
        if max(prompt_len, reg + 1) < min(eos_min, max_length):
            raise NotImplementedError(
                f"min_length / min_new_tokens ban EOS up to length {eos_min}, which overlaps the "
                f"exponential_decay_length_penalty region (lengths above {reg}): the reference computes NaN there")
        if any(ids[-1] == eos and v == -math.inf for ids, v in seqs):
            raise NotImplementedError("a bad word or a -inf sequence_bias ending in EOS together with "
                                      "exponential_decay_length_penalty: the reference computes NaN there")
    return Processors(seqs, int(ngram), int(eos_min))
