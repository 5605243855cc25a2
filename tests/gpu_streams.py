"""Concurrent streams on one GPU (development aid / measurement; the test is in test_gpu_parity.py).

    python tests/gpu_streams.py [--preset large-v2] [--heads 10] [--clips 8] [--configs 1x132,2x66,4x33] [--alpha 100]

For every configuration SxC (S engines sharing one weight blob, C CTAs each): runs the clips, checks every clip's tokens
against the single-stream run, prints ms per iteration per stream, aggregate tokens/s and achieved HBM GB/s
(algorithmic bytes of every iteration of every stream / wall time of the decode phase).
"""
from __future__ import annotations

import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from whisper_medusa_b200 import StreamGroup  # noqa: E402
from whisper_medusa_b200.synthetic import preset_config, synthetic_audio, synthetic_state_dict  # noqa: E402


def arg(name, default):
    return type(default)(sys.argv[sys.argv.index(name) + 1]) if name in sys.argv else default


def main():
    preset, heads, n_clips = arg("--preset", "large-v2"), arg("--heads", 10), arg("--clips", 8)
    alpha = arg("--alpha", 100.0)
    configs = [tuple(int(v) for v in c.split("x")) for c in arg("--configs", "1x132,2x66,4x33").split(",")]
    cfg = preset_config(preset, heads=heads)
    sd = synthetic_state_dict(cfg, seed=0)
    secs = 30.0 if preset == "large-v2" else 5.0
    clips = [synthetic_audio(secs, stream_id=i) for i in range(n_clips)]
    kw = dict(language="en" if cfg.is_multilingual else None, exponential_decay_length_penalty=bench.PENALTY, posterior_alpha=alpha)
    peak, _ = bench.measured_peak_gbs()
    ref = None
    for S, C in configs:
        try:
            grp = StreamGroup(cfg, sd, "cuda:0", n_streams=S, ctas_per_stream=C)
            grp.generate_from_pcm(clips[:S], **dict(kw, max_iters=4))                      # warm-up
            torch.cuda.synchronize()
            outs = grp.generate_from_pcm(clips, **kw)
            wall = grp.last_wall_s
            toks = [o[0].tolist() for o in outs]
            if ref is None:
                ref = toks
            ok = toks == ref
            tr = grp.last_traces
            sm = bench.summarize(cfg, tr, peak)
            # decode phase: the streams overlap; approximate its wall time by the busiest engine's summed decode windows
            per_iter = [t.ms_decode / max(1, t.iterations) for t in tr]
            enc = sum(t.ms_encoder + t.ms_mel for t in tr)
            dec_wall_ms = max(1e-9, grp.last_decode_phase_s * 1e3)   # busiest engine's summed decode-loop device times
            print(f"{S}x{C:<4d} tokens {'OK ' if ok else 'BAD'} clips {n_clips}  ms/iter/stream {np.mean(per_iter):.3f}  "
                  f"e2e {sm['tokens'] / wall:8.1f} tok/s  decode-phase {sm['tokens'] / (dec_wall_ms / 1e3):8.1f} tok/s  "
                  f"HBM {sm['bytes_eng'] / (dec_wall_ms / 1e3) / 1e9:7.1f} GB/s = {sm['bytes_eng'] / (dec_wall_ms / 1e3) / 1e9 / peak:.3f} of peak  "
                  f"(wall {wall * 1e3:.1f} ms, encoders {enc:.1f} ms, mean accept {sm['mean_accept']:.2f})", flush=True)
            grp.close()
        except Exception as e:  # noqa: BLE001
            print(f"{S}x{C} FAILED: {type(e).__name__}: {e}", flush=True)


if __name__ == "__main__":
    main()
