"""2-CTA clusters of the persistent ring kernel: the full-GPU grid runs as clusters whose CTAs share one multicast copy of
each GEMM stage's activation rows; any other grid runs unclustered with private copies.  Every output row is computed by
one CTA with a fixed k slicing, FC2 folds its k segments in segment order, and both grids below use the same number of
cross-attention key chunks, so the clustered full grid and the unclustered n_sm - 1 grid must agree bit for bit."""
import os

import numpy as np
import pytest
import torch

from _wm_paths import GOLDEN
from whisper_medusa_b200.synthetic import preset_config, synthetic_audio, synthetic_state_dict

pytestmark = pytest.mark.gpu


def _load(name):
    g = np.load(os.path.join(GOLDEN, name + ".npz"))
    seed, stream, max_len, heads, is_block = [int(v) for v in g["meta"]]
    preset = {"micro": "micro", "tiny": "tiny.en", "large": "large-v2"}[name.split("_")[0]]
    cfg = preset_config(preset, heads=heads, heads_type="medusa_block" if is_block else "base_head")
    pen = None if g["penalty"][0] < 0 else (int(g["penalty"][0]), float(g["penalty"][1]))
    kw = dict(language="en" if cfg.is_multilingual else None, max_length=max_len,
              exponential_decay_length_penalty=pen, medusa_temperature=float(g["temperature"]))
    if "posterior" in g.files:
        kw.update(posterior_alpha=float(g["posterior"][0]), posterior_threshold=float(g["posterior"][1]))
    return g, cfg, seed, stream, kw


@pytest.fixture(scope="module")
def n_sm():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _outputs(model, pcm, kw, ids):
    """tokens, accept lengths, raw logits of both passes of the last iteration, and forward() logits."""
    tokens = model.generate_from_pcm(pcm, **kw)[0].cpu().numpy()
    acc = np.array(model.last_trace.accept_lengths)
    lg0, lg1 = model.last_logits(0).numpy(), model.last_logits(1).numpy()
    fwd = model.forward(decoder_input_ids=torch.tensor([ids])).logits.cpu().numpy()
    return {"tokens": tokens, "accept_lengths": acc, "last_logits0": lg0, "last_logits1": lg1, "forward": fwd}


def test_full_grid_runs_as_two_cta_clusters(n_sm):
    from whisper_medusa_b200 import WhisperMedusaModel

    g, cfg, seed, stream, kw = _load("micro_linear_k4")
    m = WhisperMedusaModel(cfg, synthetic_state_dict(cfg, seed=seed)).to("cuda:0")
    pcm = synthetic_audio(float(g["audio_seconds"]), stream_id=stream)
    try:
        for ctas, want in ((n_sm, 2 if n_sm % 2 == 0 else 1), (n_sm - 1, 1), (33, 1), (n_sm, 2 if n_sm % 2 == 0 else 1)):
            m.set_option("decode_ctas", ctas)
            out = m.generate_from_pcm(pcm, **kw)[0].tolist()
            assert m.last_trace.cluster_decode == want, ctas
            assert out == g["tokens"].tolist() and m.last_trace.accept_lengths == g["accept_lengths"].tolist(), ctas
            assert m.last_trace.launches_decode == m.last_trace.iterations
    finally:
        m.close()


@pytest.mark.parametrize("name", ["large_linear_k10_mixed", "tiny_block_k4"])
def test_multicast_staging_equals_private_staging(name, n_sm):
    """large-v2 with 10 Medusa-Linear heads on the benchmark clip, and a Medusa-Block model (whose block QKV splits
    gamma o x in place in each CTA of a pair): the full grid (clustered) against n_sm - 1 CTAs (unclustered)."""
    from whisper_medusa_b200 import WhisperMedusaModel

    g, cfg, seed, stream, kw = _load(name)
    m = WhisperMedusaModel(cfg, synthetic_state_dict(cfg, seed=seed)).to("cuda:0")
    pcm = synthetic_audio(float(g["audio_seconds"]), stream_id=stream)
    ids = [cfg.decoder_start_token_id, cfg.no_timestamps_token_id, 17, 33, 64, 250, 1000]
    try:
        full = _outputs(m, pcm, kw, ids)
        assert full["tokens"].tolist() == g["tokens"].tolist()
        m.set_option("decode_ctas", n_sm - 1)
        part = _outputs(m, pcm, kw, ids)
    finally:
        m.close()
    for k in full:
        assert np.array_equal(full[k], part[k]), k
