"""fp64 reference of the decode path and the logit bar it is held to (DESIGN.md section 2).

The engine's decode path keeps about 22 mantissa bits of every activation (fp16 hi + lo) and rounds on purpose only
where the K/V caches are stored in fp16.  The reference here is the oracle in fp64 with exactly those roundings
(regime "engine"), decoding from the engine's own encoder states, so what is left is the engine's own error.

Setting ``WM_NUMERICS_RECORD=<file>`` turns the logit bar into a measurement: every checked error is appended to that
file as one JSON line (case, what, error, and the error of the fp32 oracle against the same fp64 reference) and the bar
is not asserted.  DESIGN.md section 2 records such a run and the bar derived from it.
"""
import json
import os

import numpy as np
import torch

from oracle import medusa_ref as M
from oracle import whisper_ref as W

#: Decode-path logits against the fp64 engine-regime reference, relative to max(1, max|logit|).  The worst value
#: measured over every width, activation profile and decode mode is 3.0e-4 (DESIGN.md section 2); most of it is 1-ulp
#: flips of fp16 K/V roundings, which the fp32 oracle shows too (up to 1.5e-4 against the same reference).
DECODE_LOGIT_BAR = 1e-3

RECORD = os.environ.get("WM_NUMERICS_RECORD")


def rel_err(a, b):
    """max |a - b| relative to the scale of the logits (>= 1): the fp16 K/V caches round with 2^-11 relative
    precision, and Medusa-Block rows (heads on an un-normalised residual stream) reach |logit| ~ 30."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(1.0, float(np.abs(b).max())))


def check_logits(engine, ref64, case, what, ref32=None, bar=None):
    """Assert finite engine logits within ``bar`` (default DECODE_LOGIT_BAR) of the fp64 reference; returns the error.
    In recording mode the error is written out instead of asserted."""
    engine = np.asarray(engine)
    assert np.isfinite(engine).all(), (case, what, "non-finite logits")
    return check_error(rel_err(engine, ref64), DECODE_LOGIT_BAR if bar is None else bar, case, what,
                       None if ref32 is None else rel_err(ref32, ref64))


def check_error(err, bar, case, what, oracle_fp32_err=None):
    """Assert ``err <= bar``; in recording mode append the error (and the fp32 oracle's error against the same fp64
    reference, if given) to the record file instead.  Returns ``err``."""
    if RECORD:
        rec = {"case": case, "what": what, "err": err}
        if oracle_fp32_err is not None:
            rec["oracle_fp32_err"] = oracle_fp32_err
        with open(RECORD, "a") as f:
            f.write(json.dumps(rec) + "\n")
    else:
        assert err <= bar, (case, what, err, bar)
    return err


def decode_logits(cfg, sd, enc, kw, n_iters, dtype=torch.float64, threads=16, prompt=None, begin_index=None,
                  prompt_len=None, tree_attention=False):
    """Oracle decode loop (engine regime, working dtype ``dtype``) started from the given encoder states; the trace
    holds the raw pass-A / pass-B logits of the first ``n_iters`` iterations.  ``sd`` may also be a ``RefWeights``
    already in the working dtype (``dtype`` is then ignored): at large-v2 a conversion costs seconds and 12 GB in fp64.

    ``prompt``: decoder ids to start from (default: the model's start tokens).  Given an engine's history up to the start
    of iteration n together with ``begin_index`` / ``prompt_len`` of the ORIGINAL prompt (so that the begin-suppress and
    length-penalty processors see what they saw in the real run), one iteration of this loop gives the logits and the
    tokens of iteration n of the real run: pass A recomputes every cached row from the ids alone, which for chains and
    for ``tree_attention=True`` is what the real loop's cache holds (tests/test_oracle_history_prompt.py)."""
    torch.set_num_threads(threads)
    w = sd if isinstance(sd, W.RefWeights) else W.RefWeights(sd, dtype)
    if prompt is None:
        prompt = M.init_tokens(cfg, kw.get("language"))
    extra = {k: kw[k] for k in ("posterior_alpha", "posterior_threshold") if k in kw}
    if begin_index is not None:
        extra["begin_index"] = int(begin_index)
    if prompt_len is not None:
        extra["prompt_len"] = int(prompt_len)
    gp = M.gen_params(cfg, prompt, kw.get("exponential_decay_length_penalty"), kw["max_length"],
                      temperature=kw.get("medusa_temperature", 1.0), **extra)
    return M.medusa_greedy_search(w, cfg, enc, [int(t) for t in prompt], gp, "engine", capture_logits=n_iters,
                                  max_iters=n_iters, tree_attention=tree_attention)


def forward_logits(cfg, sd, enc, ids, dtype=torch.float64):
    """Oracle of ``forward(decoder_input_ids=[ids])``: stacked head logits ``[K+1, T, V]`` from an empty cache (``sd``: a
    state dict or a ``RefWeights``, as in ``decode_logits``)."""
    w = sd if isinstance(sd, W.RefWeights) else W.RefWeights(sd, dtype)
    cache = W.new_cache(cfg)
    hidden = W.decoder_forward(w, cfg, list(ids), list(range(len(ids))), enc, cache, "engine")
    return W.medusa_logits(w, cfg, hidden, enc, cache, False, "engine")
