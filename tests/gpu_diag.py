"""GPU diagnostics: stage-by-stage comparison of the CUDA engine with the CPU oracle.

    python tests/gpu_diag.py [case ...] [--mode graph|persistent] [--large]

Prints one line per check (never raises on a numeric mismatch) so a single GPU run shows
where a divergence starts: mel -> encoder -> first-iteration logits -> token ids.
"""
from __future__ import annotations

import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import medusa_ref as M  # noqa: E402
from oracle import whisper_ref as W  # noqa: E402
from whisper_medusa_b200 import WhisperMedusaModel  # noqa: E402
from whisper_medusa_b200.synthetic import preset_config, synthetic_audio, synthetic_state_dict  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")
TC = "--tc" in sys.argv


def first_diff(a, b):
    for i, (x, y) in enumerate(zip(a, b)):
        if x != y:
            return i
    return None if len(a) == len(b) else min(len(a), len(b))


def run_case(name: str, mode: str, use_oracle: bool = True):
    g = np.load(os.path.join(GOLDEN, name + ".npz"))
    seed, stream, max_len, heads, is_block = [int(v) for v in g["meta"]]
    preset = {"micro": "micro", "tiny": "tiny.en", "large": "large-v2"}[name.split("_")[0]]
    cfg = preset_config(preset, heads=heads, heads_type="medusa_block" if is_block else "base_head")
    t0 = time.time()
    sd = synthetic_state_dict(cfg, seed=seed)
    pcm = synthetic_audio(float(g["audio_seconds"]), stream_id=stream)
    temp = float(g["temperature"])
    pen = None if g["penalty"][0] < 0 else (int(g["penalty"][0]), float(g["penalty"][1]))
    model = WhisperMedusaModel(cfg, sd).to("cuda:0")
    model.set_decode_mode(mode)
    if TC:
        model.set_option("enc_gemm", 1)   # wgmma / TMA encoder GEMM
    print(f"[{name}/{mode}] setup {time.time() - t0:.1f}s", flush=True)
    language = "en" if cfg.is_multilingual else None
    kw = dict(language=language, max_length=max_len, exponential_decay_length_penalty=pen, medusa_temperature=temp)

    # one-iteration run for the logits taps
    model.generate_from_pcm(pcm, max_iters=1, **kw)
    mel_e = model.mel().numpy()
    print(f"[{name}] mel       max|d| vs golden sample = {np.abs(mel_e[:, ::8] - g['mel_sample']).max():.3e}")
    enc_e = model.encoder_output().numpy()
    print(f"[{name}] encoder   max|d| vs golden(engine regime) = {np.abs(enc_e[::50] - g['enc_sample']).max():.3e}"
          f"   vs fp32 regime = {np.abs(enc_e[::50] - g['enc_sample_fp32']).max():.3e}   (|x|max {np.abs(enc_e).max():.2f})")
    for ab, which in (("A", 0), ("B", 1)):
        lg = model.last_logits(which).numpy()
        ref = g[f"logits{ab}0_strided"]
        d = np.abs(lg[:, ::97] - ref)
        rows = d.max(axis=1)
        print(f"[{name}] logits{ab}0  max|d| = {d.max():.3e}  per-row {np.array2string(rows, precision=1)}")
        topi = g[f"logits{ab}0_topi"][:, 0]
        print(f"[{name}] logits{ab}0  raw argmax engine {lg.argmax(1).tolist()} golden {topi.tolist()}")
    if use_oracle and preset != "large-v2":
        w = W.RefWeights(sd)
        melt = torch.from_numpy(W.log_mel_spectrogram(pcm))
        print(f"[{name}] mel       max|d| vs oracle (full) = {np.abs(mel_e - melt.numpy()).max():.3e}")
        enc_o = W.encoder_forward(w, cfg, melt, "engine").numpy()
        print(f"[{name}] encoder   max|d| vs oracle (full) = {np.abs(enc_e - enc_o).max():.3e}")

    # full run
    t0 = time.time()
    out = model.generate_from_pcm(pcm, **kw)[0].tolist()
    tr = model.last_trace
    gold = g["tokens"].tolist()
    fd = first_diff(out, gold)
    print(f"[{name}/{mode}] tokens: engine {len(out)} golden {len(gold)} first_diff {fd}  "
          f"accept_match {tr.accept_lengths == g['accept_lengths'].tolist()}  iters {tr.iterations}")
    if fd is not None:
        print(f"   engine[{max(0, fd - 3)}:{fd + 5}] = {out[max(0, fd - 3):fd + 5]}\n   golden = {gold[max(0, fd - 3):fd + 5]}")
        print(f"   engine accept {tr.accept_lengths[:20]}\n   golden accept {g['accept_lengths'][:20].tolist()}")
    print(f"[{name}/{mode}] ms: mel {tr.ms_mel:.3f} encoder {tr.ms_encoder:.3f} decode {tr.ms_decode:.3f} "
          f"({tr.ms_decode / max(1, tr.iterations):.3f} ms/iter, {tr.n_new_tokens / max(tr.ms_decode, 1e-9) * 1e3:.1f} tok/s) "
          f"launches enc {tr.launches_encode} dec {tr.launches_decode}  wall {time.time() - t0:.2f}s", flush=True)
    # through input_features (mel computed by the oracle frontend on the CPU)
    melt = torch.from_numpy(W.log_mel_spectrogram(pcm))[None]
    out2 = model.generate(melt, **kw)[0].tolist()
    print(f"[{name}/{mode}] generate(input_features) == golden: {out2 == gold}")
    model.close()
    return fd is None


def main():
    argv = sys.argv[1:]
    mode = "graph"
    if "--mode" in argv:
        i = argv.index("--mode")
        mode = argv[i + 1]
        del argv[i:i + 2]
    args = [a for a in argv if not a.startswith("--")]
    names = args or ["micro_linear_k4", "micro_block_k10", "micro_linear_k4_t0", "tiny_linear_k4", "tiny_block_k4"]
    ok = True
    for n in names:
        try:
            ok &= bool(run_case(n, mode))
        except Exception as e:  # noqa: BLE001
            import traceback

            traceback.print_exc()
            print(f"[{n}/{mode}] EXCEPTION {e}", flush=True)
            ok = False
    print("DIAG", "ALL-MATCH" if ok else "MISMATCH")


if __name__ == "__main__":
    main()
