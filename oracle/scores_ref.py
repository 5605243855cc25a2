"""CPU ORACLE (test infrastructure -- never imported by the product path).

Scores and per-token log-probabilities of a run of ``medusa_ref.medusa_greedy_search``, rebuilt from its trace
(``capture_logits`` >= the number of iterations), so the loop itself stays as it is.

Per iteration, with ``L`` = len(input_ids) at its start, ``a`` = its accept length and ``path`` = the best candidate's
root-to-leaf nodes, every row processed with ``cur_len = L`` (``medusa_ref.process_logits``):

* scores row: the processed verify row ``path[a]`` -- ``vlog[best, a]``, the reference's ``next_token_logits``
  (``medusa_utils.py:663-664``) that ``model.py:737-742`` appends to ``scores`` and ``logits``;
* token log-probabilities: ``log_softmax`` at temperature 1 of the row each new token was chosen from -- the base row
  of pass A for the first token, verify row ``path[j - 1]`` for the j-th (accepted candidates, or the extra token of
  an accept-0 iteration).
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import List, Sequence

import torch

from . import medusa_ref as M


@dataclass
class LoopScores:
    rows: List[torch.Tensor] = field(default_factory=list)     # one processed [V] row per iteration
    token_logprobs: List[float] = field(default_factory=list)  # one per position after the prompt (before truncation)
    token_scales: List[float] = field(default_factory=list)    # max(1, max |finite entry|) of each token's row
    paths: List[List[int]] = field(default_factory=list)       # best path nodes of every iteration


def best_path(rows_a: torch.Tensor, choices: Sequence[int], chosen: Sequence[int]) -> List[int]:
    """Node ids of the candidate path the loop chose (``LoopTrace.candidates[i]``, or only its first tokens), recovered
    from the processed pass-A rows of that iteration: the first path whose tokens start with ``chosen``.  Sibling nodes
    carry distinct tokens, so the nodes at the depths ``chosen`` covers are unique."""
    bufs = M.generate_medusa_buffers(choices)
    cands, _ = M.generate_candidates(rows_a[1:], rows_a[0], list(choices)[1:], bufs["tree_indices"])
    for c in range(cands.shape[0]):
        if cands[c, : len(chosen)].tolist() == list(chosen):
            return bufs["retrieve_indices"][c].tolist()
    raise AssertionError("the chosen candidate is not a path of the tree")


def loop_scores(tr: M.LoopTrace, prompt_len: int, gp: M.GenParams, choices: Sequence[int]) -> LoopScores:
    """Scores rows and token log-probabilities of ``tr`` (which must hold the raw logits of every iteration)."""
    assert len(tr.passA_logits) == len(tr.accept_lengths), "run medusa_greedy_search with capture_logits >= iterations"
    out = LoopScores()
    L = prompt_len
    for i, a in enumerate(tr.accept_lengths):
        rows_a = M.process_logits(tr.passA_logits[i], L, gp)
        rows_b = M.process_logits(tr.passB_logits[i], L, gp)
        path = best_path(rows_a, choices, tr.candidates[i])
        out.paths.append(path)
        out.rows.append(rows_b[path[a]].clone())
        n_new = a + 1 if a > 0 else 2
        for j in range(n_new):
            row = rows_a[0] if j == 0 else rows_b[path[j - 1]]
            tok = int(tr.sequences[L + j])
            out.token_logprobs.append(float(torch.log_softmax(row.double(), -1)[tok]))
            out.token_scales.append(max(1.0, float(row[torch.isfinite(row)].abs().max())))
        L += n_new
    return out
