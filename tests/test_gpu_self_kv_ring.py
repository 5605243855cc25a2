"""Self-attention through the weight ring against the stage kernels.

In the ring kernel (`persistent`) the cached keys and values [0, min(base, kv_len)) of every self-attention item arrive
as ring chunks (sa_prefix_chunk, stage_self_attn_ring) and only the rest comes from L2; `graph` reads the whole head-major
cache from L2 (stage_self_attn).  The two modes also differ in their LayerNorm arithmetic (the ring kernel folds it into
its GEMMs, DESIGN.md section 2), so their logits are not the same bits: on the build before the ring carried the prefix,
tokens and accept lengths of these runs were equal and every logit within DECODE_LOGIT_BAR (relative to the logit
scale) of `graph`'s, and that is what is pinned here.  The runs go past 256 cached keys, so both prefix blocks of an item
are used, and the Block runs compact the caches after every accepted tree path."""
import numpy as np
import pytest

from _decode_ref import DECODE_LOGIT_BAR, rel_err
from whisper_medusa_b200.synthetic import preset_config, synthetic_audio, synthetic_state_dict, width_config

pytestmark = pytest.mark.gpu

PENALTY = (140, 1.01)


def _runs(model, pcm, kw, iters):
    """{max_iters: (sequence, accept lengths, pass-A logits, verify logits)} in the model's current decode mode."""
    out = {}
    for it in iters:
        model.generate_from_pcm(pcm, max_iters=it, **kw)
        tr = model.last_trace
        out[it] = (list(tr.sequences), list(tr.accept_lengths), model.last_logits(0).numpy().copy(),
                   model.last_logits(2).numpy().copy())
    return out


def _compare(model, pcm, kw, case):
    model.set_decode_mode("persistent")
    model.generate_from_pcm(pcm, **kw)
    n = model.last_trace.iterations
    length = len(model.last_trace.sequences)
    assert length > 256 + 16, (case, length)   # past the first prefix block
    iters = (1, n // 2, n)
    ring = _runs(model, pcm, kw, iters)
    model.set_decode_mode("graph")
    graph = _runs(model, pcm, kw, iters)
    model.set_decode_mode("persistent")
    worst = 0.0
    for it in iters:
        rs, ra, rla, rlb = ring[it]
        gs, ga, gla, glb = graph[it]
        assert rs == gs, (case, it)
        assert ra == ga, (case, it)
        assert np.isfinite(rla).all() and np.isfinite(rlb).all(), (case, it)
        worst = max(worst, rel_err(rla, gla), rel_err(rlb, glb))
    print(f"{case}: {n} iterations, {length} positions; ring vs graph logits {worst:.3g}")
    assert worst <= DECODE_LOGIT_BAR, (case, worst)


def test_large_v2_ring_equals_graph():
    """The benchmark's workload: large-v2, 10 Linear heads, realistic acceptance, 30 s clip (342 tokens)."""
    from whisper_medusa_b200 import WhisperMedusaModel

    cfg = preset_config("large-v2", heads=10)
    model = WhisperMedusaModel(cfg, synthetic_state_dict(cfg, seed=0)).to("cuda:0")
    try:
        kw = dict(language="en", exponential_decay_length_penalty=PENALTY, posterior_alpha=100.0)
        _compare(model, synthetic_audio(30.0), kw, "large-v2")
    finally:
        model.close()


@pytest.mark.parametrize("tree_attention", [False, True])
def test_block_16_node_tree_ring_equals_graph(tree_attention):
    """Medusa-Block heads on the 16-node tree [1, 3, 4] at d = 512, to max_length 448: the tail's block self-attention,
    sweep A after every iteration (reference attention) or elided sweeps (tree attention), and compaction moves."""
    from whisper_medusa_b200 import WhisperMedusaModel

    cfg = width_config(512, heads=2, heads_type="medusa_block")
    cfg.medusa_choices = [1, 3, 4]
    model = WhisperMedusaModel(cfg, synthetic_state_dict(cfg, seed=3)).to("cuda:0")
    try:
        kw = dict(language=None, max_length=448, tree_attention=tree_attention)
        _compare(model, synthetic_audio(5.0, stream_id=3), kw, f"block/tree_attention={tree_attention}")
    finally:
        model.close()
