"""Freezes what the reference's ``whisper_medusa/models/medusa_utils.py`` returns for the inputs of
tests/test_oracle_medusa_utils.py into tests/golden/reference/medusa_utils.npz, so that the oracle's restatement is pinned to
the reference's own code on machines without a reference checkout.

    WM_REFERENCE_ROOT=<reference checkout> python -m oracle.make_medusa_utils_golden

The inputs are made here (seeded) and by the tests through the same functions.
"""
from __future__ import annotations

import os

import numpy as np
import torch

GOLDEN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "reference",
                      "medusa_utils.npz")

BUFFER_CHOICES = [[1, 1, 1, 1, 1], [1] * 11, [1, 2, 2], [1, 3, 2, 1], [1, 6, 5, 4, 3]]
CANDIDATE_CHOICES = [[1, 1, 1, 1, 1], [1, 2, 2], [1, 3, 2, 1]]
POSTERIOR_CHOICES = [[1, 1, 1, 1, 1], [1, 2, 2]]
POSTERIOR_TEMPERATURES = [0.0, 1.0, 0.7]
POSTERIOR_TRIALS = 40


def key(choices) -> str:
    return "-".join(str(c) for c in choices)


def candidate_inputs(choices):
    g = torch.Generator().manual_seed(7)
    H, V, T = len(choices) - 1, 300, 3
    med = torch.randn(H, 1, T, V, generator=g)
    base = torch.randn(1, T, V, generator=g)
    return med, base


def posterior_inputs(n_cand: int, depth: int):
    """(logits, candidates) of every trial: random rows, a third of them with argmax-matching prefixes so that
    accepts happen."""
    g = torch.Generator().manual_seed(3)
    V = 200
    out = []
    for trial in range(POSTERIOR_TRIALS):
        logits = torch.randn(n_cand, depth, V, generator=g) * (0.5 + trial % 4)
        cands = torch.randint(0, V, (n_cand, depth), generator=g)
        if trial % 3 == 0:
            cands[:, 1:] = logits[:, :-1].argmax(-1)
            cands[:, 1 + trial % depth:] = 0
        out.append((logits, cands))
    return out


def main() -> None:
    import importlib.util

    from oracle import medusa_ref as M
    from oracle import ref_harness as R

    if not os.path.isfile(R.REF_UTILS):
        raise SystemExit(f"{R.REF_UTILS} not found: set WM_REFERENCE_ROOT to a reference checkout")
    spec = importlib.util.spec_from_file_location("ref_medusa_utils", R.REF_UTILS)
    ref = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ref)
    out = {}
    for ch in BUFFER_CHOICES:
        b = ref.generate_medusa_buffers(ch, device="cpu")
        for k in ("tree_indices", "medusa_position_ids", "retrieve_indices"):
            out[f"buffers/{key(ch)}/{k}"] = b[k].long().numpy()
    for ch in CANDIDATE_CHOICES:
        med, base = candidate_inputs(ch)
        bufs = M.generate_medusa_buffers(ch)
        rc, rt = ref.generate_candidates(med, base, ch[1:], bufs["tree_indices"])
        out[f"candidates/{key(ch)}/cart"] = rc.long().numpy()
        out[f"candidates/{key(ch)}/tree"] = rt[0].long().numpy()
    for ch in POSTERIOR_CHOICES:
        n_cand, depth = M.generate_medusa_buffers(ch)["retrieve_indices"].shape
        for temp in POSTERIOR_TEMPERATURES:
            res = [ref.evaluate_posterior(lg, cd, temp, 0.09, 0.3) for lg, cd in posterior_inputs(n_cand, depth)]
            out[f"posterior/{key(ch)}/{temp}"] = np.array([[int(b), int(a)] for b, a in res], dtype=np.int64)
    os.makedirs(os.path.dirname(GOLDEN), exist_ok=True)
    np.savez_compressed(GOLDEN, **out)
    print(f"wrote {GOLDEN}: {len(out)} arrays")


if __name__ == "__main__":
    main()
