"""Pins the oracle's restatement of medusa_utils.py against what the reference file itself returns for the same inputs
(frozen in tests/golden/reference/medusa_utils.npz by oracle/make_medusa_utils_golden.py) and against known answers
recorded from it (SURVEY.md section 4)."""
import os

import numpy as np
import pytest
import torch

from _wm_paths import GOLDEN
from oracle import make_medusa_utils_golden as G
from oracle import medusa_ref as M


def _ref():
    return np.load(os.path.join(GOLDEN, "reference", "medusa_utils.npz"))


def test_buffers_known_answer():
    # probed from the reference: generate_medusa_buffers([1, 2, 2])
    b = M.generate_medusa_buffers([1, 2, 2])
    assert b["tree_indices"].tolist() == [0, 1, 2, 3, 4, 3, 4]
    assert b["medusa_position_ids"].tolist() == [0, 1, 1, 2, 2, 2, 2]
    assert b["retrieve_indices"].tolist() == [[0, 1, 3], [0, 1, 4], [0, 2, 5], [0, 2, 6]]
    c = M.generate_medusa_buffers([1] * 11)
    assert c["tree_indices"].tolist() == list(range(11))
    assert c["medusa_position_ids"].tolist() == list(range(11))
    assert c["retrieve_indices"].tolist() == [list(range(11))]


@pytest.mark.parametrize("choices", G.BUFFER_CHOICES)
def test_buffers_match_reference(choices):
    r = _ref()
    o = M.generate_medusa_buffers(choices)
    for k in ("tree_indices", "medusa_position_ids", "retrieve_indices"):
        assert torch.equal(torch.from_numpy(r[f"buffers/{G.key(choices)}/{k}"]), o[k].long()), k


@pytest.mark.parametrize("choices", G.CANDIDATE_CHOICES)
def test_candidates_match_reference(choices):
    r = _ref()
    med, base = G.candidate_inputs(choices)
    bufs = M.generate_medusa_buffers(choices)
    oc, ot = M.generate_candidates(med[:, 0, -1], base[0, -1], choices[1:], bufs["tree_indices"])
    assert torch.equal(torch.from_numpy(r[f"candidates/{G.key(choices)}/cart"]), oc.long())
    assert torch.equal(torch.from_numpy(r[f"candidates/{G.key(choices)}/tree"]), ot.long())


@pytest.mark.parametrize("temperature", G.POSTERIOR_TEMPERATURES)
@pytest.mark.parametrize("choices", G.POSTERIOR_CHOICES)
def test_evaluate_posterior_matches_reference(choices, temperature):
    want = _ref()[f"posterior/{G.key(choices)}/{temperature}"]
    n_cand, depth = M.generate_medusa_buffers(choices)["retrieve_indices"].shape
    inputs = G.posterior_inputs(n_cand, depth)
    assert len(want) == len(inputs) == G.POSTERIOR_TRIALS
    for (logits, cands), (rb, ra) in zip(inputs, want.tolist()):
        ob, oa = M.evaluate_posterior(logits, cands, temperature, 0.09, 0.3)
        assert ra == oa and rb == ob


def test_processors_match_hf():
    from transformers.generation.logits_process import (ExponentialDecayLengthPenalty,
                                                        SuppressTokensAtBeginLogitsProcessor,
                                                        SuppressTokensLogitsProcessor)

    g = torch.Generator().manual_seed(1)
    V, eos = 100, 50
    gp = M.GenParams(eos_token_id=eos, pad_token_id=eos, suppress_tokens=[1, 5, 9], begin_suppress_tokens=[2, eos],
                     begin_index=4, exponential_decay_length_penalty=(6, 1.3), prompt_len=4)
    procs = [ExponentialDecayLengthPenalty((6, 1.3), eos, 4), SuppressTokensLogitsProcessor([1, 5, 9]),
             SuppressTokensAtBeginLogitsProcessor([2, eos], 4)]
    for cur_len in (4, 5, 10, 11, 17):
        rows = torch.randn(3, V, generator=g)
        ids = torch.zeros(3, cur_len, dtype=torch.long)
        want = rows.clone()
        for p in procs:
            want = p(ids, want)
        got = M.process_logits(rows, cur_len, gp)
        assert torch.equal(torch.nan_to_num(want, neginf=-1e30), torch.nan_to_num(got, neginf=-1e30))


def test_strip_output_rules():
    gp = M.GenParams(eos_token_id=9, pad_token_id=9)
    assert M.strip_output([1, 2, 5, 6, 9, 9, 9], 2, gp) == [5, 6]      # post-EOS fill removed, EOS removed
    assert M.strip_output([1, 2, 5, 6], 2, gp) == [5, 6]                # no EOS
    assert M.strip_output([1, 2, 9, 9], 2, gp) == []                    # only EOS
    gp2 = M.GenParams(eos_token_id=9, pad_token_id=8)
    assert M.strip_output([1, 2, 5, 9, 8, 8], 2, gp2) == [5]
