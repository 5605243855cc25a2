"""Host reference of the logits scan and the accept step of one loop iteration (``stage_select1/2``, ``select_fold``,
``stage_select_fin``, ``stage_accept``, ``stage_accept_tree`` in csrc/decode.cu).

Two precisions, each where the engine's result is defined by it:

* The processed logits are an fp32 replica of ``processed_logit`` (csrc/common.cuh): suppressed ids -inf, and the EOS
  length penalty ``v + |v| * pen`` rounded ONCE (nvcc contracts it to ``FFMA pen, |v|, v``; the replica rounds the exact
  value to fp32, ties to even), with ``pen`` the fp32 of ``factor^(L - start) - 1`` taken in fp64 as ``wm_generate``
  builds its table.  Candidates and argmaxes are comparisons of these fp32 values and must match the engine exactly,
  with the engine's tie rules: argmax keeps the first index, top-k orders by (value descending, index ascending).
* Probabilities, entropies, thresholds and path likelihoods are fp64 on those processed rows, with T, the threshold and
  alpha as the engine received them (fp32 values).

``decide`` takes processed rows, so the CPU test can pin it to ``oracle/medusa_ref.py`` on the same rows;
``accept_ref`` takes the raw rows the engine exposes (``last_logits(0)`` and ``last_logits(2)``).
"""
from __future__ import annotations

from dataclasses import dataclass
from fractions import Fraction
from typing import List, Optional, Sequence

import numpy as np

from oracle import medusa_ref as M

#: the kernel's entropy term is p * log(p + 1e-5f) (medusa_utils.py evaluate_posterior: + 1e-5)
ENT_EPS = float(np.float32(1e-5))


def f32(x) -> float:
    return float(np.float32(x))


def engine_pen(gp: M.GenParams, L: int) -> float:
    """``pen_tab[L]`` of ``wm_generate``: (factor^(L - start - n_prompt) - 1) in fp64 from the fp32 factor, rounded to fp32;
    0 where the penalty is inactive."""
    if gp.exponential_decay_length_penalty is None:
        return 0.0
    start, factor = gp.exponential_decay_length_penalty
    reg = int(start) + int(gp.prompt_len)
    if start < 0 or L <= reg:
        return 0.0
    return f32(float(np.float32(factor)) ** (L - reg) - 1.0)


def _round_f32(x: Fraction) -> np.float32:
    """Round an exact rational to the nearest fp32, ties to even."""
    c = np.float32(float(x))
    best, best_d = c, abs(Fraction(float(c)) - x)
    for n in (np.nextafter(c, np.float32(-np.inf)), np.nextafter(c, np.float32(np.inf))):
        d = abs(Fraction(float(n)) - x)
        if d < best_d or (d == best_d and int(np.float32(n).view(np.uint32)) & 1 == 0):
            best, best_d = n, d
    return np.float32(best)


def fma_f32(a: float, b: float, c: float) -> np.float32:
    """fp32 a * b + c with one rounding (the GPU's FFMA)."""
    return _round_f32(Fraction(float(np.float32(a))) * Fraction(float(np.float32(b))) + Fraction(float(np.float32(c))))


def process_rows(raw, L: int, gp: M.GenParams) -> np.ndarray:
    """fp32 replica of ``processed_logit`` applied to raw rows ``[R, V]`` at cur_len = L."""
    rows = np.array(np.asarray(raw, np.float32), np.float32, copy=True)
    pen = engine_pen(gp, L)
    eos = int(gp.eos_token_id)
    if pen != 0.0 and 0 <= eos < rows.shape[1]:
        for r in range(rows.shape[0]):
            v = float(rows[r, eos])
            rows[r, eos] = fma_f32(abs(v), pen, v)
    if gp.suppress_tokens:
        rows[:, np.asarray(gp.suppress_tokens, np.int64)] = -np.inf
    if gp.begin_suppress_tokens and L == gp.begin_index:
        rows[:, np.asarray(gp.begin_suppress_tokens, np.int64)] = -np.inf
    return rows


def first_argmax(row) -> int:
    """Index of the maximum, the first one on ties (np.argmax's rule, and the engine's)."""
    return int(np.argmax(np.asarray(row)))


def topk_ordered(row, k: int) -> List[int]:
    """The first k entries in (value descending, index ascending) order."""
    v = np.asarray(row, np.float64)
    return [int(i) for i in np.argsort(-v, kind="stable")[:k]]


@dataclass
class Tree:
    choices: List[int]
    tree_indices: np.ndarray   # node -> index into [c0 | top-k of head 1 | ...]
    retrieve: np.ndarray       # [n_cand, K + 1] node ids along each candidate path
    parent: np.ndarray         # [n_tree], -1 for the root

    @property
    def n_tree(self) -> int:
        return int(self.tree_indices.shape[0])

    @property
    def chain(self) -> bool:
        return all(c == 1 for c in self.choices)


def tree_tables(choices: Sequence[int]) -> Tree:
    ch = [int(c) for c in choices]
    b = M.generate_medusa_buffers(ch)
    ti = b["tree_indices"].numpy().astype(np.int64)
    ret = b["retrieve_indices"].numpy().astype(np.int64)
    parent = np.full(ti.shape[0], -1, np.int64)
    for path in ret:
        for j in range(1, len(path)):
            parent[path[j]] = path[j - 1]
    return Tree(ch, ti, ret, parent)


@dataclass
class AcceptRef:
    cand: np.ndarray            # [n_tree] node tokens
    row_argmax: np.ndarray      # [n_tree]
    row_pc: Optional[np.ndarray]   # [n_tree] fp64, p(node token | parent row); nan at the root; None at T = 0
    row_thr: Optional[np.ndarray]  # [n_tree] fp64 thresholds (chain: rows < K; tree: every row); None at T = 0
    stat_rows: List[int]        # rows whose threshold the engine computes
    accept: int
    best: int                   # candidate path
    path: List[int]             # its nodes
    path_node: int              # path[accept]
    new_tokens: List[int]
    edges: List[tuple]          # (child, parent) pairs the decision compared


def candidates(rows_a: np.ndarray, tree: Tree) -> np.ndarray:
    """Node tokens: argmax of the base row, top-k of every head row (generate_candidates)."""
    flat = [first_argmax(rows_a[0])]
    for i, k in enumerate(tree.choices[1:], start=1):
        flat += topk_ordered(rows_a[i], k)
    return np.asarray(flat, np.int64)[tree.tree_indices]


def posterior(row: np.ndarray, T: float):
    """fp64 softmax of ``row / T`` (suppressed ids -> 0) and the engine's entropy term sum p log(p + 1e-5) (= -entropy)."""
    v = np.asarray(row, np.float64)
    fin = np.isfinite(v)
    z = np.zeros_like(v)
    m = v[fin].max()
    z[fin] = np.exp((v[fin] - m) / T)
    p = z / z.sum()
    ent = float(np.sum(p * np.log(p + ENT_EPS)))
    return p, ent


def decide(rows_a, rows_b, tree: Tree, T: float, threshold: float, alpha: float) -> AcceptRef:
    """The scan and the accept step on processed fp32 rows: ``rows_a [K+1, V]`` (pass A: base row, head rows),
    ``rows_b [n_tree, V]`` (verify rows).  ``T``, ``threshold``, ``alpha``: the fp32 values the engine received."""
    rows_a = np.asarray(rows_a, np.float32)
    rows_b = np.asarray(rows_b, np.float32)
    T, threshold, alpha = f32(T), f32(threshold), f32(alpha)
    nt = tree.n_tree
    K = len(tree.choices) - 1
    cand = candidates(rows_a, tree)
    arg = np.asarray([first_argmax(rows_b[r]) for r in range(nt)], np.int64)
    stat_rows = list(range(K)) if tree.chain else list(range(nt))
    pc = thr = None
    if T != 0.0:
        pc = np.full(nt, np.nan)
        thr = np.full(nt, np.nan)
        for r in stat_rows:
            p, ent = posterior(rows_b[r], T)
            thr[r] = min(threshold, float(np.exp(ent)) * alpha)
            for n in range(1, nt):
                if tree.parent[n] == r:
                    pc[n] = p[cand[n]]
    lens, likes, edges = [], [], set()
    for path in tree.retrieve:
        n_ok, like = 0, 0.0
        for j in range(K):
            node, child = int(path[j]), int(path[j + 1])
            edges.add((child, node))
            ok = (cand[child] == arg[node]) if T == 0.0 else (pc[child] > thr[node])
            if not ok:
                break
            n_ok += 1
            if T != 0.0:
                like += float(np.log(pc[child]))
        lens.append(n_ok)
        likes.append(like)
    a = max(lens)
    if a == 0:
        best = 0
    elif T == 0.0:
        best = lens.index(a)
    else:
        best = max((i for i in range(len(lens)) if lens[i] == a), key=lambda i: (likes[i], -i))
    path = [int(x) for x in tree.retrieve[best]]
    toks = [int(cand[n]) for n in path[: a + 1]]
    if a == 0:
        toks.append(int(arg[path[0]]))
    return AcceptRef(cand, arg, pc, thr, stat_rows, a, best, path, path[a], toks, sorted(edges))


def accept_ref(raw_a, raw_b, L: int, gp: M.GenParams, choices: Sequence[int], T: float, threshold: float,
               alpha: float) -> AcceptRef:
    """``decide`` on the raw rows of an iteration that starts at length L (``last_logits(0)``, ``last_logits(2)``)."""
    return decide(process_rows(raw_a, L, gp), process_rows(raw_b, L, gp), tree_tables(choices), T, threshold, alpha)


def margin_rows(ref: AcceptRef, rel: float) -> List[tuple]:
    """Compared edges (child, parent) whose candidate probability lies within ``rel`` (relative to the threshold) of its
    threshold: a decision there may go either way at fp32 resolution."""
    if ref.row_pc is None:
        return []
    return [(c, p) for c, p in ref.edges if abs(ref.row_pc[c] - ref.row_thr[p]) <= rel * ref.row_thr[p]]
