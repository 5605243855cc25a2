"""Long-form transcription on one GPU (development aid / measurement; the tests are in test_gpu_longform.py).

    python tests/gpu_longform.py [--preset large-v2] [--heads 10] [--minutes 10] [--alpha 100] [--out DIR]

A recording of --minutes minutes made by concatenating 30 s `synthetic_audio` clips, transcribed at 16 kHz and at
48 kHz (the same recording, oracle-resampled to 48 kHz on the host) in the realistic acceptance regime
(posterior_alpha = 100, language + length penalty as bench.py).  Reports the GPU resample time, the per-window encode
and decode times, and wall time and merged tokens/s of `model.transcribe` and of `StreamGroup.transcribe` with S = 1,
2 and 4; every StreamGroup result is checked against `model.transcribe`.  Also the resampler's worst |error| against the
fp64 oracle (oracle/resample_ref.py) over 10 minutes of peak-0.5 audio at 8, 22.05, 44.1, 48 and 96 kHz.  One JSON
object goes to DIR/longform.json (default: a new temporary directory; the path is printed).
"""
from __future__ import annotations

import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from oracle import resample_ref as R  # noqa: E402
from whisper_medusa_b200 import StreamGroup, WhisperMedusaModel  # noqa: E402
from whisper_medusa_b200.synthetic import preset_config, synthetic_audio, synthetic_state_dict  # noqa: E402


def arg(name, default):
    return type(default)(sys.argv[sys.argv.index(name) + 1]) if name in sys.argv else default


def gpu_label():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,enforced.power.limit,power.default_limit",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
        return q.splitlines()[0]
    except Exception:  # noqa: BLE001
        return torch.cuda.get_device_name(0)


def signal(n, sr, seed=0):
    rng = np.random.default_rng(seed)
    t = np.arange(n) / sr
    x = 0.02 * rng.standard_normal(n)
    for f in (110.0, 440.0, 3000.0, 0.45 * sr):
        x += rng.uniform(0.2, 1.0) * np.sin(2 * np.pi * f * t + rng.uniform(0, 2 * np.pi))
    return (0.5 * x / np.abs(x).max()).astype(np.float32)


def time_resample(model, x_dev, sr, reps=20):
    """Median device time (CUDA events) of the resampling kernel alone, input already on the device."""
    model._upload_16k(x_dev, sr)
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        model._upload_16k(x_dev, sr)
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def window_stats(windows):
    enc = [w.trace.ms_mel + w.trace.ms_encoder for w in windows]
    dec = [w.trace.ms_decode for w in windows]
    return dict(windows=len(windows), encode_ms_median=float(np.median(enc)), encode_ms_sum=float(np.sum(enc)),
                decode_ms_median=float(np.median(dec)), decode_ms_sum=float(np.sum(dec)),
                decode_ms_max=float(np.max(dec)), window_ids=int(sum(len(w.ids) for w in windows)))


def main():
    preset, heads, minutes, alpha = arg("--preset", "large-v2"), arg("--heads", 10), arg("--minutes", 10.0), arg("--alpha", 100.0)
    out_dir = arg("--out", "") or tempfile.mkdtemp(prefix="wm_longform_")
    os.makedirs(out_dir, exist_ok=True)
    res = dict(gpu=gpu_label(), preset=preset, heads=heads, minutes=minutes, posterior_alpha=alpha)
    print(res["gpu"], flush=True)

    cfg = preset_config(preset, heads=heads)
    model = WhisperMedusaModel(cfg, synthetic_state_dict(cfg, seed=0)).to("cuda:0")
    model.release_state_dict()

    # resampler accuracy and speed over 10 minutes of audio
    acc = {}
    for sr in (8000, 22050, 44100, 48000, 96000):
        x = signal(600 * sr, sr, seed=sr)
        xd = torch.from_numpy(x).to("cuda:0")
        y = model._upload_16k(xd, sr).cpu().numpy().astype(np.float64)
        err = float(np.abs(y - R.resample(x, sr, 16000)).max())
        acc[sr] = dict(max_abs_err=err, kernel_ms=time_resample(model, xd, sr), n_in=len(x), n_out=len(y))
        print(f"resample {sr:>6} Hz -> 16 kHz, 10 min: max |err| {err:.3e}  kernel {acc[sr]['kernel_ms']:.3f} ms", flush=True)
        del xd
    res["resample"] = acc

    kw = dict(language="en" if cfg.is_multilingual else None, exponential_decay_length_penalty=bench.PENALTY,
              posterior_alpha=alpha)
    n_clips = int(round(minutes * 2))
    x16 = np.concatenate([synthetic_audio(30.0, stream_id=i) for i in range(n_clips)]).astype(np.float32)
    x48 = R.resample(x16, 16000, 48000).astype(np.float32)
    warm = x16[: 35 * 16000]
    model.transcribe(warm, **kw)                                           # warm-up (one short recording)
    runs = {}
    for name, x, sr in (("16k", x16, 16000), ("48k", x48, 48000)):
        x_dev = torch.from_numpy(x).to("cuda:0")
        t_up = time_resample(model, x_dev, sr) if sr != 16000 else 0.0
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        ref = model.transcribe(x, sampling_rate=sr, **kw)[0].tolist()
        wall = time.perf_counter() - t0
        row = dict(resample_kernel_ms=t_up, model=dict(wall_s=wall, merged_tokens=len(ref), tok_s=len(ref) / wall,
                                                       **window_stats(model.last_windows)))
        row["model"]["window_tok_s"] = row["model"]["window_ids"] / wall
        print(f"{name}: model.transcribe   wall {wall:7.2f} s  merged {len(ref)} tokens  {len(ref) / wall:7.1f} tok/s  "
              f"(window ids decoded {row['model']['window_tok_s']:.1f} /s)  "
              f"{row['model']['windows']} windows: encode {row['model']['encode_ms_median']:.2f} ms, "
              f"decode {row['model']['decode_ms_median']:.1f} ms (median per window)", flush=True)
        for S in (1, 2, 4):
            grp = StreamGroup(cfg, None, "cuda:0", n_streams=S, weights_from=model)
            grp.transcribe(warm, **kw)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            got = grp.transcribe(x, sampling_rate=sr, **kw)[0][0].tolist()
            wall = time.perf_counter() - t0
            row[f"group{S}"] = dict(wall_s=wall, tok_s=len(got) / wall, equal=got == ref, decode_phase_s=grp.last_decode_phase_s,
                                    **window_stats(grp.last_windows[0]))
            print(f"{name}: StreamGroup S={S}  wall {wall:7.2f} s  {len(got) / wall:7.1f} tok/s  "
                  f"{'equal' if got == ref else 'DIFFERENT'} to model.transcribe  decode phase {grp.last_decode_phase_s:.2f} s",
                  flush=True)
            grp.close()
        runs[name] = row
        del x_dev
    res["runs"] = runs
    with open(os.path.join(out_dir, "longform.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(f"results: {os.path.join(out_dir, 'longform.json')}")
    model.close()


if __name__ == "__main__":
    main()
