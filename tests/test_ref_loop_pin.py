"""Pins the oracle's loop restatement (oracle/medusa_ref.py::medusa_greedy_search) to the REFERENCE'S OWN CODE.

oracle/ref_harness.py executes the verbatim source of the reference's ``_medusa_greedy_search``, ``forward``,
``_forward_medusa_block``, ``_update_medusa_outputs`` (model.py) and the whole of ``medusa_utils.py`` on the installed
Whisper modules.  Its outputs for 82 UNSELECTED streams (seed = base + index; Linear and Block heads, typical
acceptance, exact-match acceptance, length penalty / EOS stop, K = 4 and 10) are frozen in
tests/golden/ref_loop_streams.npz by oracle/make_ref_golden.py.

* the oracle, fp32 regime, reproduces every frozen reference stream bit-for-bit, i.e. the oracle is pinned to
  executable reference code, not to itself;
* every committed golden made by the oracle has identical tokens / accept lengths in its two numeric regimes.
"""
import glob
import os

import numpy as np
import pytest
import torch

from _wm_paths import GOLDEN
from oracle import make_ref_golden as G
from oracle import medusa_ref as M
from oracle import whisper_ref as W

FIX = os.path.join(GOLDEN, "ref_loop_streams.npz")


def _streams(groups=None):
    out = []
    for g, spec in G.GROUPS.items():
        if groups is None or g in groups:
            out += [(g, s) for s in range(spec[3])]
    return out


def _oracle_stream(group, s, regime="fp32"):
    cfg, sd, pcm, max_len, pen, temp, alpha, thr = G.stream_inputs(group, s)
    w = W.RefWeights(sd)
    mel = torch.from_numpy(W.log_mel_spectrogram(pcm))
    enc = W.encoder_forward(w, cfg, mel, regime)
    prompt = M.init_tokens(cfg, "en" if cfg.is_multilingual else None)
    gp = M.gen_params(cfg, prompt, pen, max_len, temperature=temp, posterior_alpha=alpha, posterior_threshold=thr)
    tr = M.medusa_greedy_search(w, cfg, enc, prompt, gp, regime)
    return tr.sequences, tr.accept_lengths


@pytest.mark.parametrize("group", list(G.GROUPS))
def test_oracle_reproduces_frozen_reference_streams(group):
    fx = np.load(FIX)
    torch.set_num_threads(min(8, os.cpu_count() or 1))
    for _, s in _streams([group]):
        seq, acc = _oracle_stream(group, s)
        assert seq == fx[f"{group}/{s}/sequences"].tolist(), (group, s)
        assert acc == fx[f"{group}/{s}/accept"].tolist(), (group, s)


def test_reference_streams_cover_the_decision_space():
    fx = np.load(FIX)
    seen, eos_stops, total = set(), 0, 0
    for g, s in _streams():
        acc = fx[f"{g}/{s}/accept"].tolist()
        seen |= set(acc)
        seq = fx[f"{g}/{s}/sequences"].tolist()
        cfg = G.stream_inputs(g, s)[0]
        eos_stops += int(cfg.eos_token_id in seq[int(fx[f"{g}/{s}/prompt_len"]):])
        total += 1
        # SURVEY.md 3.3: tokens per iteration = accept + 1, or 2 when nothing was accepted
        assert len(seq) - int(fx[f"{g}/{s}/prompt_len"]) == sum(a + 1 if a else 2 for a in acc)
    assert total >= 80 and set(range(11)) <= seen
    assert eos_stops >= 10, "the EOS stop / post-EOS fill must be exercised"


def test_goldens_agree_between_numeric_regimes():
    """Token ids / accept lengths of every oracle-made fixture are the same in the "engine" rounding regime (what the
    CUDA engine is asserted against) and in the fp32 regime (the reference's numerics)."""
    files = [f for f in sorted(glob.glob(os.path.join(GOLDEN, "*.npz"))) if "ref_loop" not in f]
    assert len(files) >= 7
    for f in files:
        g = np.load(f)
        assert g["tokens"].tolist() == g["tokens_fp32"].tolist(), f
        assert g["sequences"].tolist() == g["sequences_fp32"].tolist(), f
        assert g["accept_lengths"].tolist() == g["accept_lengths_fp32"].tolist(), f
