"""CPU ORACLE of the logits processors (test infrastructure -- never imported by the product path).

HF's ``SequenceBiasLogitsProcessor``, ``NoRepeatNGramLogitsProcessor``, ``NoBadWordsLogitsProcessor``,
``MinLengthLogitsProcessor`` and ``MinNewTokensLengthLogitsProcessor`` restated for the batch-1 loop, in the order of
``_get_logits_processor``, ahead of the EOS decay and the suppress processors of ``medusa_ref.process_logits``.  They
read the sequence at the start of the iteration (``input_ids``), which the reference passes for every row of it
(``model.py:653-665, 689-694``).  The options are attributes of a ``medusa_ref.GenParams`` (``gen_params(...,
sequence_bias=[(ids, bias), ...], bad_words_ids=[[...]], no_repeat_ngram_size=n, min_length=n, min_new_tokens=n)``);
absent attributes are off.

The loop (``medusa_greedy_search``), the scores record (``loop_scores``) and the reference harness (``run_loop``) are
those of ``medusa_ref``, ``scores_ref`` and ``ref_harness``, compiled from their own source with the one change each
needs -- the processors get ``input_ids``, or the harness takes extra HF processors -- so they cannot drift apart.
Pinned in ``tests/test_logits_processors_host.py``: ``process_logits`` bit-equal to the installed HF processors, and the
loop equal to the reference's own loop with them.
"""
from __future__ import annotations

import __future__
import inspect
import textwrap
from typing import Dict, List, Optional, Sequence

import torch

from . import medusa_ref as M
from . import ref_harness as R
from . import scores_ref as S


def _sequence_bias(V: int, entries, input_ids: Sequence[int]) -> torch.Tensor:
    """HF ``SequenceBiasLogitsProcessor``'s ``bias`` row: the single-token biases, then ``+=`` (fp32) each longer entry,
    in dict order, whose prefix ends ``input_ids`` (entries longer than ``input_ids`` skipped; others add 0.0)."""
    bias = torch.zeros(V, dtype=torch.float32)
    singles = [(ids[0], v) for ids, v in entries if len(ids) == 1]
    if singles:
        one = torch.zeros(V, dtype=torch.float32)
        one[torch.tensor([t for t, _ in singles])] = torch.tensor([v for _, v in singles])
        bias += one
    for ids, v in entries:
        if len(ids) == 1 or len(ids) > len(input_ids):
            continue
        hit = list(input_ids[len(input_ids) - len(ids) + 1:]) == list(ids[:-1])
        bias[ids[-1]] += torch.tensor(v if hit else 0.0)
    return bias


def process_logits(rows: torch.Tensor, cur_len: int, gp: M.GenParams,
                   input_ids: Optional[Sequence[int]] = None) -> torch.Tensor:
    """``medusa_ref.process_logits`` preceded by the five processors of ``gp``; ``input_ids`` = the sequence at the start
    of the iteration (``cur_len = len(input_ids)``), needed by sequence_bias, bad_words_ids and no_repeat_ngram_size."""
    rows = rows.clone()
    V = rows.shape[-1]
    eos = gp.eos_token_id
    if getattr(gp, "sequence_bias", None):
        rows = rows + _sequence_bias(V, gp.sequence_bias, input_ids)
    n = getattr(gp, "no_repeat_ngram_size", 0)
    if n and cur_len + 1 >= n:
        key = list(input_ids[cur_len + 1 - n: cur_len])
        banned = [input_ids[i + n - 1] for i in range(cur_len - n + 1) if list(input_ids[i: i + n - 1]) == key]
        if banned:
            rows[:, torch.tensor(banned)] = float("-inf")
    if getattr(gp, "bad_words_ids", None):
        bad = {tuple(w): float("-inf") for w in gp.bad_words_ids if list(w) != [eos]}
        if bad:
            rows = rows + _sequence_bias(V, list(bad.items()), input_ids)
    if getattr(gp, "min_length", 0) > 0 and cur_len < gp.min_length:
        rows[:, eos] = float("-inf")
    if getattr(gp, "min_new_tokens", 0) > 0 and cur_len - gp.prompt_len < gp.min_new_tokens:
        rows[:, eos] = float("-inf")
    return M.process_logits(rows, cur_len, gp)


def _recompile(fn, edits, namespace: Dict):
    """``fn`` compiled from its own source with ``edits`` (each ``old`` must occur exactly once) in ``namespace``."""
    src = textwrap.dedent(inspect.getsource(fn))
    for old, new in edits:
        assert src.count(old) == 1, f"{fn.__name__}: {old!r} occurs {src.count(old)} times"
        src = src.replace(old, new)
    ns = dict(namespace)
    exec(compile(src, inspect.getsourcefile(fn), "exec", __future__.annotations.compiler_flag, dont_inherit=True), ns)
    return ns[fn.__name__]


# the loop of medusa_ref with input_ids handed to the processors (A1 / B1)
medusa_greedy_search = _recompile(
    M.medusa_greedy_search,
    [("process_logits(rows_raw, L, gp)", "process_logits(rows_raw, L, gp, input_ids)"),
     ("process_logits(logits_b_raw, L, gp)", "process_logits(logits_b_raw, L, gp, input_ids)")],
    dict(vars(M), process_logits=process_logits))

# the scores record of scores_ref with the iteration's input_ids (the trace's first L ids) handed to the processors
loop_scores = _recompile(
    S.loop_scores,
    [("M.process_logits(tr.passA_logits[i], L, gp)", "process_logits(tr.passA_logits[i], L, gp, tr.sequences[:L])"),
     ("M.process_logits(tr.passB_logits[i], L, gp)", "process_logits(tr.passB_logits[i], L, gp, tr.sequences[:L])")],
    dict(vars(S), process_logits=process_logits))

# RefLoop.run_loop with HF processors placed ahead of the ones it builds (the 4.49 order of _get_logits_processor)
_run_loop = _recompile(
    R.RefLoop.run_loop,
    [("posterior_alpha: float = 0.3) ->", "posterior_alpha: float = 0.3, processors=()) ->"),
     ("procs = LogitsProcessorList()", "procs = LogitsProcessorList(list(processors))")],
    vars(R))


class _PerRow:
    """The reference calls its processors with one ``input_ids`` row for all the rows of a pass (``[K+1, V]`` or
    ``[n_tree, V]``).  Every processor broadcasts it, except HF's ``NoRepeatNGramLogitsProcessor``, which indexes
    ``input_ids`` per score row and raises IndexError.  This hands it the same row once per score row -- what the others
    compute by broadcasting."""

    def __init__(self, proc):
        self.proc = proc

    def __call__(self, input_ids, scores):
        return self.proc(input_ids.expand(scores.shape[0], -1), scores)


def hf_processors(eos: int, prompt_len: int, sequence_bias=None, no_repeat_ngram_size=None, bad_words_ids=None,
                  min_length=None, min_new_tokens=None) -> List:
    """The installed HF processors for ``generate``'s options (``sequence_bias`` in HF's list form), in
    ``_get_logits_processor``'s order."""
    from transformers.generation.logits_process import (MinLengthLogitsProcessor, MinNewTokensLengthLogitsProcessor,
                                                        NoBadWordsLogitsProcessor, NoRepeatNGramLogitsProcessor,
                                                        SequenceBiasLogitsProcessor)
    procs: List = []
    if sequence_bias is not None:
        procs.append(SequenceBiasLogitsProcessor(sequence_bias))
    if no_repeat_ngram_size:
        procs.append(_PerRow(NoRepeatNGramLogitsProcessor(no_repeat_ngram_size)))
    if bad_words_ids is not None:
        procs.append(NoBadWordsLogitsProcessor(bad_words_ids, eos))
    if min_length:
        procs.append(MinLengthLogitsProcessor(min_length, eos))
    if min_new_tokens:
        procs.append(MinNewTokensLengthLogitsProcessor(prompt_len, min_new_tokens, eos))
    return procs


def run_loop(ref: "R.RefLoop", enc: torch.Tensor, prompt: Sequence[int], *, processor_args: Optional[Dict] = None,
             **kw):
    """The reference's loop (``RefLoop.run_loop``, same keyword arguments) with the HF processors of
    ``processor_args`` (``generate``'s keyword names) ahead of the ones it builds.  Returns (sequences, accept lengths)."""
    procs = hf_processors(int(ref.mcfg.eos_token_id), len(prompt), **(processor_args or {}))
    return _run_loop(ref, enc, prompt, processors=procs, **kw)
