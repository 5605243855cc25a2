"""The host reference of the logits scan and the accept step (tests/_accept_ref.py) pinned to the oracle
(oracle/medusa_ref.py): ``generate_candidates``, ``evaluate_posterior`` and ``process_logits``.

* On random rows without ties the helper's candidates and decisions equal the oracle's, and its posterior
  probabilities and thresholds are the oracle's formulas in fp64 within 1e-12, for chains and the trees ``[1,3,4]``,
  ``[1,3,2,1]``, ``[1,4,2]`` at T = 0, 0.5, 1, 2.
* It reproduces the oracle's own candidates and accept lengths from the oracle loop's captured raw rows on micro
  streams (chains, Block heads, length penalty, trees, both acceptance rules).
* The processors: equal to ``process_logits`` everywhere except the EOS entry under the length penalty, where the
  engine rounds ``v + |v| * pen`` once (an FMA) and the oracle twice; the two are at most 1 ulp apart.

Reference-parity note on ties: ``torch.topk`` does not promise an order among equal values, and on the CPU it does not
return them by ascending index (torch 2.11: ``topk([1, 3, -inf, 3, 2, 3, 2], 4)`` gives indices ``[1, 5, 3, 4]``, and
``topk(zeros(1000), 5)`` gives ``[3, 4, 1, 0, 2]``).  So on rows with exact ties the reference's tree candidates are
an order the engine does not promise to reproduce.  The engine (and the helper) order top-k by (value descending, index
ascending) and take the first index for argmax (``torch.argmax`` does the same); ``test_tie_rules`` pins the helper's rule
on rows with exact ties without asking torch.topk to agree.
"""
import os

import numpy as np
import pytest
import torch

import _accept_ref as A
from oracle import make_ref_golden as G
from oracle import medusa_ref as M
from oracle import whisper_ref as W

CHOICES = [(1, 1), (1, 1, 1, 1), (1, 1, 1, 1, 1), (1, 3, 4), (1, 3, 2, 1), (1, 4, 2)]
TEMPS = [0.0, 0.5, 1.0, 2.0]


def _rows(rng, tree, V, T):
    """Pass-A rows and verify rows without ties.  Verify row r puts its children's tokens near the top with a random
    boost, so that every accept length and both sides of the threshold occur."""
    K = len(tree.choices) - 1

    def distinct(n, spread):   # a permutation of evenly spaced values: no two equal in fp32
        return np.stack([(rng.permutation(V) / V * 2.0 - 1.0) * spread for _ in range(n)]).astype(np.float32)

    rows_a = distinct(K + 1, 8.0)
    cand = A.candidates(rows_a, tree)
    rows_b = distinct(tree.n_tree, rng.uniform(1.0, 12.0))
    share = rng.uniform(0.1, 1.0)
    for n in range(1, tree.n_tree):
        p = tree.parent[n]
        if rng.uniform() < share:    # else the child keeps a random logit and is rejected
            rows_b[p, cand[n]] = rows_b[p].max() + np.float32(rng.uniform(-3.0, 3.0) * max(T, 0.5))
    rows_a[:, 7] = -np.inf                # a suppressed id
    rows_b[:, 7] = -np.inf
    for r in (rows_a, rows_b):
        for row in r:
            fin = row[np.isfinite(row)]
            assert np.unique(fin).size == fin.size, "tie in a random row"
    return rows_a, rows_b


def _oracle_quantities(rows_b, tree, cand, T, thr, alpha):
    """evaluate_posterior's formulas (medusa_utils.py:526-588) in fp64 on every candidate path."""
    vlog = torch.from_numpy(rows_b.astype(np.float64))[torch.from_numpy(tree.retrieve)]
    cands = torch.from_numpy(cand[tree.retrieve])
    prob = torch.softmax(vlog[:, :-1] / T, dim=-1)
    cprob = torch.gather(prob, -1, cands[:, 1:].unsqueeze(-1)).squeeze(-1)
    ent = -torch.sum(prob * torch.log(prob + A.ENT_EPS), dim=-1)
    thr_t = torch.minimum(torch.full_like(ent, thr), torch.exp(-ent) * alpha)
    return cprob.numpy(), thr_t.numpy()


@pytest.mark.parametrize("choices", CHOICES, ids=["-".join(map(str, c)) for c in CHOICES])
@pytest.mark.parametrize("T", TEMPS)
def test_decide_equals_the_oracle_on_random_rows(choices, T):
    tree = A.tree_tables(choices)
    thr, alpha = A.f32(0.09), A.f32(0.3)
    rng = np.random.default_rng(hash((choices, T)) & 0xFFFF)
    seen = set()
    for trial in range(12):
        V = int(rng.choice([512, 513, 2000]))
        rows_a, rows_b = _rows(rng, tree, V, T)
        ref = A.decide(rows_a, rows_b, tree, T, thr, alpha)
        # candidates: generate_candidates on the same processed rows
        ra = torch.from_numpy(rows_a)
        cands, tree_cands = M.generate_candidates(ra[1:], ra[0], choices[1:], torch.from_numpy(tree.tree_indices))
        assert ref.cand.tolist() == tree_cands.tolist()
        assert ref.row_argmax.tolist() == [int(torch.argmax(torch.from_numpy(r))) for r in rows_b]
        # decision: evaluate_posterior on [n_cand, K+1, V]
        vlog = torch.from_numpy(rows_b.astype(np.float64))[torch.from_numpy(tree.retrieve)]
        best, accept = M.evaluate_posterior(vlog, cands, T, thr, alpha)
        assert (ref.best, ref.accept) == (best, accept), trial
        assert ref.path_node == int(tree.retrieve[best][accept])
        seen.add(accept)
        if T == 0.0:
            assert ref.row_pc is None and ref.row_thr is None
            continue
        cprob, thr_o = _oracle_quantities(rows_b, tree, ref.cand, T, thr, alpha)
        for c, path in enumerate(tree.retrieve):
            for j in range(len(path) - 1):
                node, child = int(path[j]), int(path[j + 1])
                assert abs(ref.row_pc[child] - cprob[c, j]) <= 1e-12 * max(cprob[c, j], 1e-300) + 1e-300
                assert abs(ref.row_thr[node] - thr_o[c, j]) <= 1e-12 * thr_o[c, j]
    assert len(seen) >= 2, seen      # the rows exercise more than one accept length


def test_accept_tap_needs_a_handle():
    from whisper_medusa_b200 import _lib

    assert _lib.load().wm_last_accept(None, None, None, None, None, None) == -1    # WM_ERR_INVALID


def test_tie_rules():
    """Exact ties: argmax keeps the first index, top-k orders equal values by ascending index."""
    row = np.array([1.0, 3.0, -np.inf, 3.0, 2.0, 3.0, 2.0], np.float32)
    assert A.first_argmax(row) == 1
    assert A.topk_ordered(row, 4) == [1, 3, 5, 4]
    assert A.topk_ordered(row, 6) == [1, 3, 5, 4, 6, 0]
    tree = A.tree_tables((1, 4, 2))
    rows_a = np.stack([row, row[::-1].copy(), row])
    cand = A.candidates(rows_a, tree)
    # root = argmax of row 0; level 1 = top-4 of head 1 (the reversed row: 3.0 at 1, 3, 5, then 2.0 at 0 and 2); level 2
    # = top-2 of head 2 under every level-1 node
    assert cand.tolist() == [1, 1, 3, 5, 0, 1, 3, 1, 3, 1, 3, 1, 3]


def test_processors_match_process_logits_and_round_the_penalty_once():
    rng = np.random.default_rng(5)
    V, eos = 600, 550
    gp = M.GenParams(eos_token_id=eos, pad_token_id=eos, suppress_tokens=[3, 17, 590], begin_suppress_tokens=[220, eos],
                     begin_index=4, exponential_decay_length_penalty=(2, A.f32(1.07)), prompt_len=4)
    raw = (rng.standard_normal((16, V)) * 5).astype(np.float32)
    for L in (4, 5, 6, 7, 30, 200):
        got = A.process_rows(raw, L, gp)
        ref = M.process_logits(torch.from_numpy(raw), L, gp).numpy()
        assert np.array_equal(np.isneginf(got), np.isneginf(ref))
        keep = np.ones(V, bool)
        keep[eos] = False
        assert np.array_equal(got[:, keep], ref[:, keep])
        if L == gp.begin_index:
            assert np.isneginf(got[:, eos]).all()
            continue
        pen = A.engine_pen(gp, L)
        assert (pen == 0.0) == (L <= gp.exponential_decay_length_penalty[0] + gp.prompt_len)
        v = raw[:, eos].astype(np.longdouble)
        exact = v + np.abs(v) * np.longdouble(pen)           # exact in the 64-bit significand: |pen| < 1, |v| > 2^-10
        assert np.array_equal(got[:, eos], exact.astype(np.float32))
        assert np.all(np.abs(got[:, eos].view(np.int32).astype(np.int64) - ref[:, eos].view(np.int32)) <= 1)


def test_fma_rounds_once():
    # (1 + 2^-12)^2 = 1 + 2^-11 + 2^-24: rounded first (a tie, to even) it loses the 2^-24 the fused result keeps
    a = 1.0 + 2.0 ** -12
    assert float(A.fma_f32(a, a, -1.0)) == 2.0 ** -11 + 2.0 ** -24
    assert float(np.float32(np.float32(a) * np.float32(a)) - np.float32(1.0)) == 2.0 ** -11
    # ties of the final rounding go to the even neighbour
    assert float(A.fma_f32(1.0, 1.0, 2.0 ** -24)) == 1.0
    assert float(A.fma_f32(1.0 + 2.0 ** -23, 1.0, 2.0 ** -24)) == 1.0 + 2.0 ** -22
    assert float(A.fma_f32(3.0, 0.5, -1.5)) == 0.0


MICRO_STREAMS = [("micro_lin_t1", 0), ("micro_lin_t0", 0), ("micro_lin_pen", 1), ("micro_blk_t1", 0),
                 ("micro_tree122_t1", 0), ("micro_tree1321_t1", 0), ("micro_tree12121_t0", 0)]


@pytest.mark.parametrize("group,s", MICRO_STREAMS, ids=[f"{g}-{s}" for g, s in MICRO_STREAMS])
def test_reproduces_the_oracle_loop(group, s):
    """Every iteration of an oracle run, from its captured raw rows: the helper's best-path tokens and accept length are
    the oracle's."""
    torch.set_num_threads(min(8, os.cpu_count() or 1))
    cfg, sd, pcm, max_len, pen, temp, alpha, thr = G.stream_inputs(group, s)
    w = W.RefWeights(sd)
    enc = W.encoder_forward(w, cfg, torch.from_numpy(W.log_mel_spectrogram(pcm)), "fp32")
    prompt = M.init_tokens(cfg, "en" if cfg.is_multilingual else None)
    gp = M.gen_params(cfg, prompt, pen, max_len, temperature=temp, posterior_alpha=alpha, posterior_threshold=thr)
    tr = M.medusa_greedy_search(w, cfg, enc, prompt, gp, "fp32", capture_logits=1 << 20)
    L = len(prompt)
    for i, a in enumerate(tr.accept_lengths):
        ref = A.accept_ref(tr.passA_logits[i].numpy(), tr.passB_logits[i].numpy(), L, gp, gp.medusa_choices, temp, thr,
                           alpha)
        assert ref.accept == a, (i, ref.accept, a)
        assert [int(ref.cand[n]) for n in ref.path] == tr.candidates[i], i
        n_new = a + 1 if a else 2
        assert ref.new_tokens == tr.sequences[L: L + n_new] or gp.eos_token_id in tr.sequences[L: L + n_new]
        L += n_new
    assert len(tr.accept_lengths) >= 3
