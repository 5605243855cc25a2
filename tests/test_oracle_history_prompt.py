"""CPU pin of the method the deep logit checks of tests/test_gpu_decode_rows_and_depth.py rest on.

Iteration n of a real decode loop runs on a self-attention K/V cache that the loop built up piece by piece: the rows
of the verify passes it kept, one-token sweeps after an accept length of 0 and, for trees, rows gathered out of tree
order.  One iteration of the fp64 oracle started from the loop's own history (prompt + every token accepted before
iteration n), with the begin-suppress index and the length-penalty origin of the ORIGINAL prompt, recomputes that cache
from the ids alone.  For chains and for ``tree_attention=True`` (every kept row was computed behind exactly its
ancestors) it gives the same logits, to fp64 rounding, and the same tokens.  These runs go to a length of 400 and more,
so the self-attention of the checked iterations spans hundreds of keys.

The identity holds for Medusa-Block heads too: the block's K/V row at position p depends only on the decoder's
final-LayerNorm state at p (the block's attention output is never cached), so recomputing it from the ids gives what the
loop appended sweep by sweep."""
import pytest
import torch

from _decode_ref import decode_logits
from oracle import medusa_ref as M
from oracle import whisper_ref as W
from whisper_medusa_b200.synthetic import synthetic_audio, synthetic_state_dict, width_config

MAX_LEN = 448

# (d_model, K, medusa_choices or None for the top-1 chain, tree_attention, heads type)
CASES = [(128, 4, None, False, "base_head"), (128, 2, [1, 3, 4], True, "base_head"),
         (512, 15, None, False, "base_head"), (128, 3, [1, 3, 2, 1], True, "base_head"),
         (128, 4, None, False, "medusa_block"), (512, 15, None, False, "medusa_block"),
         (128, 2, [1, 3, 4], True, "medusa_block"), (128, 3, [1, 3, 2, 1], True, "medusa_block")]


def _case_id(case):
    d, k, ch, ta, ht = case
    return f"d{d}-k{k}" + (f"-tree{''.join(map(str, ch))}" if ch else "") + ("-tree_attn" if ta else "") + \
        ("-block" if ht == "medusa_block" else "")


def _iter_lengths(prompt_len, accepts):
    """Sequence length at the start of every iteration (an accept length a appends a + 1 tokens, 0 appends 2)."""
    out = [prompt_len]
    for a in accepts:
        out.append(out[-1] + (a + 1 if a > 0 else 2))
    return out


def _rel(a, b):
    return float((a - b).abs().max()) / max(1.0, float(b.abs().max()))


@pytest.mark.parametrize("case", CASES, ids=_case_id)
def test_one_iteration_from_the_history_equals_the_accumulated_run(case):
    d, k, choices, tree_attn, heads_type = case
    cfg = width_config(d, heads=k, heads_type=heads_type)
    if choices:
        cfg.medusa_choices = list(choices)
    sd = synthetic_state_dict(cfg, seed=3)
    pcm = synthetic_audio(5.0, stream_id=3)
    enc = W.encoder_forward(W.RefWeights(sd), cfg, torch.from_numpy(W.log_mel_spectrogram(pcm)), "engine")
    kw = dict(language=None, max_length=MAX_LEN)
    full = decode_logits(cfg, sd, enc, kw, 10 ** 6, tree_attention=tree_attn)
    n = full.iters
    p = len(M.init_tokens(cfg, None))
    starts = _iter_lengths(p, full.accept_lengths)
    assert starts[-1] == len(full.sequences) >= 400, (starts[-1], n)
    for it in sorted({(n + 1) // 2, n}):
        lo, hi = starts[it - 1], starts[it]
        hist = decode_logits(cfg, sd, enc, kw, 1, prompt=full.sequences[:lo], begin_index=p, prompt_len=p,
                             tree_attention=tree_attn)
        assert hist.iters == 1
        assert hist.accept_lengths == [full.accept_lengths[it - 1]], it
        assert hist.sequences == full.sequences[:hi], it
        for ab in ("A", "B"):
            ref = getattr(full, f"pass{ab}_logits")[it - 1]
            got = getattr(hist, f"pass{ab}_logits")[0]
            assert got.dtype == torch.float64 and got.shape == ref.shape
            assert _rel(got, ref) <= 1e-12, (it, ab, _rel(got, ref))
