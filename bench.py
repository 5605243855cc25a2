#!/usr/bin/env python
"""Benchmark of the hot path: effective decoded tokens/sec (post-verify), Whisper-large-v2 + 10
Medusa-Linear heads, batch 1, 30 s synthetic audio  (BASELINE.json metric; configs[1]).

    python bench.py --gpus 1 --steps 5 --warmup 3
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N ... bench.py --gpus N ...
    python bench.py --impl reference            # the CPU oracle (port of the reference) on host cores

One "step" = one 30 s clip through the whole path (PCM -> log-mel -> encoder -> cross-K/V -> Medusa speculative
loop until EOS / max_length), called the way the reference's evaluation script calls generate()
(eval_whisper_medusa.py:61-65: language + exponential_decay_length_penalty=(140, 1.01)).  Streams are independent
(reference asserts batch 1, model.py:1451), so N GPUs run N streams per step with no data-path collective ("weak"
scaling); the only collective is the NCCL broadcast of the packed weights at start-up.

Acceptance regimes.  Seeded random weights have no real acceptance statistics: under the default typical-acceptance
constants the synthetic large-v2 model accepts all K candidates every iteration.  `posterior_alpha` (a field of the
reference's MedusaGenerationConfig, medusa_utils.py:14-18) is the knob (DESIGN.md section 8):
    realistic (DEFAULT, headline)  alpha = 100   accept lengths 1 and 4 mixed, mean ~3   (3-5 tokens / iteration)
    mixed0                          alpha = 260   accept-0 iterations (two sweeps) interleaved with accepting ones
    best                            alpha = 0.3   every candidate accepted: K+1 tokens / iteration (upper bound)
    zero                            alpha = 1e6   nothing accepted: 2 tokens / iteration, two sweeps (lower bound)
The headline `value` / `e2e` / `roofline` are the realistic regime; `regimes` carries one short run of each of the
others and `k_sweep` BASELINE configs[4] (K in {2, 4, 6, 10} at the realistic regime).

Printed keys (one JSON line, rank 0):
  value       tokens/s of the decode loop with the encoder output resident in HBM (device time,
              CUDA events on the engine stream) -- whole job: sum of tokens over ranks / max time
  e2e         same metric through WhisperMedusaModel.generate_from_pcm with HOST buffers: pinned
              PCM in, token ids out, H2D/D2H inside the timed region, wall clock max over ranks
  roofline    decode iteration vs the HBM roofline: algorithmic bytes of SURVEY.md 8(d)
  cpu_baseline the CPU oracle timed on this box's host cores on a bounded sample
The run checks the tokens of stream 0 against the committed golden fixture of the same workload
(tests/golden/large_linear_k10_mixed.npz) and fails loudly on a mismatch.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

METRIC = "effective decoded tokens/sec (post-verify) Whisper-large-v2+Medusa"
REGIMES = {"realistic": 100.0, "mixed0": 260.0, "best": 0.3, "zero": 1.0e6}
PENALTY = (140, 1.01)          # eval_whisper_medusa.py:61-65 defaults (--regulation-start / --regulation-factor)


def algorithmic_bytes(cfg, iterations: int, sweeps_a: int, n_mean: float):
    """fp16 bytes the decode loop must move, from the unit figures of SURVEY.md 8(d)
    (DESIGN.md section 4).  Returns (bytes of THIS engine's schedule, bytes of the reference schedule).

    reference schedule: two decoder sweeps per iteration (pass A + pass B), K+1 head matrices + the
    base head again, two vocabulary projections.  Engine schedule (sweep elision): one sweep per
    iteration plus one extra sweep per accept-0 iteration and for the prompt (`sweeps_a`)."""
    d, f, V, K, S = cfg.d_model, cfg.decoder_ffn_dim, cfg.vocab_size, cfg.medusa_num_heads, cfg.max_source_positions
    layer = (6 * d * d + 2 * d * f) * 2 + 2 * S * d * 2          # weights + cross K/V of one layer
    proj = V * d * 2
    head = (d * d + d) * 2
    n_l = cfg.decoder_layers + (1 if cfg.is_block else 0)
    kv_sweep = 2 * d * 2 * n_l * n_mean                            # self-K/V rows read by one sweep
    sweep = n_l * layer + kv_sweep
    heads_iter = (K * head) if cfg.is_block else ((K + 1) * head + head)
    fixed = 2 * proj + heads_iter
    ref = iterations * (2 * sweep + fixed)
    eng = iterations * (sweep + fixed) + sweeps_a * sweep
    if cfg.is_block:                                               # tail re-runs the block layer on one row
        eng += iterations * (layer + kv_sweep / n_l)
    return float(eng), float(ref)


class ClockSampler:
    """nvidia-smi clocks / throttle reasons sampled DURING the timed region."""

    Q = ("clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,"
         "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
         "clocks_event_reasons.sw_power_cap")

    def __init__(self, index: int):
        self.index, self.rows, self._stop, self._t = index, [], threading.Event(), None

    def _run(self):
        while not self._stop.is_set():
            try:
                out = subprocess.run(["nvidia-smi", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits",
                                      "-i", str(self.index)], capture_output=True, text=True, timeout=5).stdout.strip()
                if out:
                    self.rows.append([c.strip() for c in out.split(",")])
            except Exception:  # noqa: BLE001
                pass
            self._stop.wait(0.2)

    def __enter__(self):
        self._t = threading.Thread(target=self._run, daemon=True)
        self._t.start()
        return self

    def __exit__(self, *a):
        self._stop.set()
        self._t.join(timeout=6)

    def summary(self):
        sm = [float(r[0]) for r in self.rows if r and r[0].replace(".", "").isdigit()]
        mx = [float(r[1]) for r in self.rows if len(r) > 1 and r[1].replace(".", "").isdigit()]
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        reasons = sorted({names[i] for r in self.rows if len(r) >= 7 for i in range(4) if r[3 + i].lower().startswith("active")})
        return {"sm_mhz": statistics.median(sm) if sm else None, "sm_max_mhz": max(mx) if mx else None,
                "reasons": reasons, "samples": len(self.rows)}


def measured_peak_gbs():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.isfile(p):
        try:
            return float(json.load(open(p))["hbm_gbs"]), "measured (MEASURED_PEAKS.json hbm_gbs)"
        except Exception:  # noqa: BLE001
            pass
    return 3350.0, "data sheet (H100 SXM HBM3 3.35 TB/s, not measured)"


def cpu_threads() -> int:
    """Threads of the CPU arm: fixed rule (every hardware thread up to 32 -- PyTorch eager on more threads of a large
    host is slower for this DRAM-bound batch-1 loop), so the number is reproducible from box to box."""
    return max(1, min(32, os.cpu_count() or 1))


class CpuReference:
    """The CPU oracle (PyTorch eager fp32 restatement of the reference loop: one proj_out per head, two passes per
    iteration, KV concatenation) on the same workload.  The encoder output of the clip is computed once (timed,
    reported); a step is the first `max_iters` speculative iterations of the decode loop from that state."""

    def __init__(self, cfg, sd, pcm, threads: int, alpha: float):
        from oracle import medusa_ref as M
        from oracle import whisper_ref as W

        torch.set_num_threads(threads)
        self.M, self.W, self.cfg = M, W, cfg
        self.w = W.RefWeights(sd)
        t0 = time.perf_counter()
        mel = torch.from_numpy(W.log_mel_spectrogram(pcm))
        t1 = time.perf_counter()
        with torch.inference_mode():
            self.enc = W.encoder_forward(self.w, cfg, mel, "fp32")
        t2 = time.perf_counter()
        self.s_mel, self.s_encoder = t1 - t0, t2 - t1
        self.prompt = M.init_tokens(cfg, "en" if cfg.is_multilingual else None)
        self.gp = M.gen_params(cfg, self.prompt, PENALTY, 448, posterior_alpha=alpha)

    def step(self, max_iters: int):
        t0 = time.perf_counter()
        with torch.inference_mode():
            tr = self.M.medusa_greedy_search(self.w, self.cfg, self.enc, self.prompt, self.gp, "fp32", max_iters=max_iters)
        dt = time.perf_counter() - t0
        return len(tr.sequences) - len(self.prompt), tr.iters, dt


def golden_tokens(args, regime: str):
    """Token ids of stream 0 from the committed fixture of exactly this workload (None when there is none)."""
    if not (args.preset == "large-v2" and args.heads_type == "base_head" and args.seconds == 30.0):
        return None
    name = {("realistic", 10): "large_linear_k10_mixed"}.get((regime, args.heads))
    if name is None:
        return None
    path = os.path.join(ROOT, "tests", "golden", name + ".npz")
    if not os.path.isfile(path):
        return None
    return np.load(path)["tokens"].tolist()


def run_streams(model, clips, idx, language, alpha, max_iters=0):
    """Run clips[idx] through generate_from_pcm; returns per-call traces and the wall time."""
    traces, outs = [], []
    t0 = time.perf_counter()
    for i in idx:
        out = model.generate_from_pcm(clips[i], language=language, exponential_decay_length_penalty=PENALTY,
                                      posterior_alpha=alpha, max_iters=max_iters)      # H2D of PCM + D2H of ids inside
        outs.append(out.cpu()[0].tolist())
        traces.append(model.last_trace)
    return traces, outs, time.perf_counter() - t0


def dump_outputs(path, model, tokens, trace):
    """The last timed step's results, as a caller of generate_from_pcm receives them: the token ids, the full sequence
    and accept lengths of the trace, plus the state they were computed from -- the encoder output and the raw logits of
    the last verify pass (both fp32, a few MB at large-v2).  Token ids are exact in float64."""
    os.makedirs(path, exist_ok=True)
    arrays = {"tokens": np.asarray(tokens, np.float64), "sequences": np.asarray(trace.sequences, np.float64),
              "accept_lengths": np.asarray(trace.accept_lengths, np.float64),
              "encoder_output": model.encoder_output().numpy().astype(np.float32),
              "last_logits_verify": model.last_logits(1).numpy().astype(np.float32)}
    for name, a in arrays.items():
        np.save(os.path.join(path, name + ".npy"), a)


def summarize(cfg, traces, peak):
    toks = sum(t.n_new_tokens for t in traces)
    iters = sum(t.iterations for t in traces)
    dec_ms = sum(t.ms_decode for t in traces)
    n_sum = sum(0.5 * len(t.sequences) * t.iterations for t in traces)
    sweeps_a = sum(1 + sum(1 for a in t.accept_lengths[:-1] if a == 0) for t in traces)
    hist = np.bincount(np.concatenate([np.array(t.accept_lengths, dtype=np.int64) for t in traces]),
                       minlength=cfg.medusa_num_heads + 1).tolist()
    b_eng, b_ref = algorithmic_bytes(cfg, iters, sweeps_a, n_sum / max(1, iters))
    achieved = b_eng / (dec_ms / 1e3) / 1e9
    return {"tokens": toks, "iterations": iters, "ms_decode": dec_ms, "tokens_per_s": toks / (dec_ms / 1e3),
            "ms_per_iteration": dec_ms / max(1, iters), "tokens_per_iteration": toks / max(1, iters),
            "mean_accept": float(np.dot(hist, np.arange(len(hist))) / max(1, sum(hist))), "accept_hist": hist,
            "two_sweep_iterations": sweeps_a - len(traces), "achieved_gbs": achieved, "frac": achieved / peak,
            "bytes_eng": b_eng, "bytes_ref": b_ref, "n_sum": n_sum, "sweeps_a": sweeps_a}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="engine", choices=["engine", "reference"])
    ap.add_argument("--mode", default=os.environ.get("WM_DECODE_MODE", "persistent"), choices=["graph", "persistent_simple", "persistent"])
    ap.add_argument("--preset", default="large-v2")
    ap.add_argument("--heads", type=int, default=10)
    ap.add_argument("--heads-type", default="base_head", choices=["base_head", "medusa_block"])
    ap.add_argument("--seconds", type=float, default=30.0)
    ap.add_argument("--regime", default="realistic", choices=sorted(REGIMES))
    ap.add_argument("--cpu-iters", type=int, default=6, help="speculative iterations per step of the CPU arm / baseline sample")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-extras", action="store_true", help="skip the other regimes and the K sweep")
    ap.add_argument("--streams", type=int, default=4,
                    help="concurrent streams per GPU of the multi-stream measurement (detail.multi_stream; BASELINE configs[3])")
    ap.add_argument("--dump-tokens", default=None, help="write this rank's token lists (JSON) to PATH.rank<r>")
    ap.add_argument("--dump-outputs", default=None, metavar="DIR",
                    help="write what the last timed step returned (rank 0) as DIR/<name>.npy, for output-by-output "
                         "comparison of two builds")
    args = ap.parse_args()

    from whisper_medusa_b200.synthetic import preset_config, synthetic_audio, synthetic_state_dict

    rank = int(os.environ.get("RANK", "0"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    cfg = preset_config(args.preset, heads=args.heads, heads_type=args.heads_type)
    alpha = REGIMES[args.regime]
    workload = (f"whisper-{args.preset} + {args.heads} Medusa-{'Block' if cfg.is_block else 'Linear'} heads, batch 1, "
                f"{args.seconds:g} s synthetic 16 kHz audio per stream, typical acceptance, language=en, "
                f"exponential_decay_length_penalty={PENALTY}, max_length 448")
    # identical in both arms (the driver compares the two `config` objects)
    config = {"workload": workload, "acceptance_regime": f"{args.regime} (posterior_alpha={alpha:g})",
              "streams_per_step": world, "parallelism": f"replicas x{world} (independent streams)",
              "weights": "seeded synthetic fp16 (seed 0)",
              "l2": "weights (3.1 GB) >> L2 (50 MB): every iteration re-streams them from HBM"}
    threads = cpu_threads()

    # ------------------------------------------------------------------ reference arm (CPU oracle)
    if args.impl == "reference":
        if rank != 0:
            return
        sd = synthetic_state_dict(cfg, seed=0)
        ref = CpuReference(cfg, sd, synthetic_audio(args.seconds, stream_id=0), threads, alpha)
        tok = iters = 0
        per_step = []
        for i in range(args.warmup + args.steps):
            n, it, dt = ref.step(args.cpu_iters)
            if i >= args.warmup:
                tok += n
                iters += it
                per_step.append(dt)
        value = tok / sum(per_step)
        sample = (f"per step: the first {args.cpu_iters} speculative iterations ({tok // max(1, args.steps)} tokens) of stream 0 of "
                  f"the same workload, decode loop only, encoder output resident in RAM (log-mel {ref.s_mel:.2f} s + "
                  f"encoder {ref.s_encoder:.2f} s measured once, NOT included: the ratio against it is conservative)")
        print(json.dumps({
            "impl": "reference", "metric": METRIC, "value": value, "unit": "tokens/s", "n_gpus": args.gpus,
            "steps": args.steps, "warmup": args.warmup, "ms_per_step": 1e3 * sum(per_step) / len(per_step),
            "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "fp32", "data": "synthetic",
            "config": config,
            "cpu_baseline": {"value": value, "unit": "tokens/s", "cores": threads, "kind": "port", "sample": sample},
            "e2e": {"value": value, "unit": "tokens/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
            "detail": {"tokens_per_iteration": tok / max(1, iters), "s_mel": ref.s_mel, "s_encoder": ref.s_encoder},
        }))
        return

    # ------------------------------------------------------------------ engine arm
    from whisper_medusa_b200 import WhisperMedusaModel

    dist = None
    if world > 1:
        import torch.distributed as dist

        torch.cuda.set_device(local_rank)
        dist.init_process_group("nccl", device_id=torch.device("cuda", local_rank))
    device = torch.device("cuda", local_rank)
    sd = synthetic_state_dict(cfg, seed=0) if (rank == 0 or world == 1) else None
    model = WhisperMedusaModel(cfg, sd)
    model.to(device, broadcast_src=0 if world > 1 else None)   # NCCL broadcast of the packed blob (N > 1)
    if args.mode != "persistent":
        model.set_decode_mode(args.mode)                       # (persistent is the engine's default)

    def clip(i):
        return torch.from_numpy(synthetic_audio(args.seconds, stream_id=rank + world * i)).pin_memory()

    # timed clips first (stream ids rank + world*i, i < steps), warm-up clips after them: stream 0 is always timed
    clips = [clip(i) for i in range(args.steps + args.warmup)]
    language = "en" if cfg.is_multilingual else None
    peak, peak_src = measured_peak_gbs()

    def barrier():
        torch.cuda.synchronize(device)
        if dist is not None:
            dist.barrier()
        torch.cuda.synchronize(device)

    run_streams(model, clips, range(args.steps, args.steps + args.warmup), language, alpha)
    barrier()
    with ClockSampler(local_rank) as cs:
        traces, outs, _ = run_streams(model, clips, range(args.steps), language, alpha)
        barrier_t0 = time.perf_counter()
        barrier()
        wall = _ + (time.perf_counter() - barrier_t0)
    clocks = cs.summary()
    sm = summarize(cfg, traces, peak)
    launches = sum(t.launches_encode + t.launches_decode for t in traces)
    enc_ms = sum(t.ms_encoder for t in traces)
    mel_ms = sum(t.ms_mel for t in traces)

    # output validation: stream 0 (rank 0, first timed clip) against the committed golden of this workload
    gold = golden_tokens(args, args.regime) if rank == 0 else None
    validated = None
    if gold is not None:
        if outs[0] != gold:
            raise SystemExit(f"bench: tokens of stream 0 differ from tests/golden (len {len(outs[0])} vs {len(gold)})")
        validated = "stream 0 == tests/golden/large_linear_k10_mixed.npz (%d tokens)" % len(gold)
    if args.dump_tokens:
        with open(f"{args.dump_tokens}.rank{rank}", "w") as f:
            json.dump({"stream_ids": [rank + world * i for i in range(args.steps)], "tokens": outs}, f)
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, model, outs[-1], traces[-1])

    stats = torch.tensor([sm["tokens"], sm["iterations"], sm["ms_decode"], wall, enc_ms, mel_ms, launches], dtype=torch.float64, device=device)
    if dist is not None:
        allv = [torch.zeros_like(stats) for _ in range(world)]
        dist.all_gather(allv, stats)
        allv = torch.stack(allv).cpu()
    else:
        allv = stats.cpu()[None]

    # ---- extras (rank 0, after the headline measurement): other regimes, K sweep --------------------------------------
    regimes, k_sweep = {}, {}
    if rank == 0 and not args.no_extras:
        for name, a in REGIMES.items():
            if name == args.regime:
                continue
            run_streams(model, clips, [args.steps], language, a, max_iters=4)            # warm the regime's path
            tr2, _, _ = run_streams(model, clips, range(min(2, args.steps)), language, a)
            s2 = summarize(cfg, tr2, peak)
            regimes[name] = {k: s2[k] for k in ("tokens_per_s", "ms_per_iteration", "tokens_per_iteration", "mean_accept",
                                                "accept_hist", "two_sweep_iterations", "frac")}
            regimes[name]["posterior_alpha"] = a
        if sd is not None and not cfg.is_block and args.preset == "large-v2":
            k_sweep[str(args.heads)] = {k: sm[k] for k in ("tokens_per_s", "ms_per_iteration", "tokens_per_iteration", "mean_accept")}
            for K in (2, 4, 6):
                if K >= args.heads:
                    continue
                # heads are drawn last and in order: the K-head checkpoint of this seed is a prefix of the K=10 one
                cK = preset_config(args.preset, heads=K, heads_type=args.heads_type)
                sdK = {k: v for k, v in sd.items() if not k.startswith("medusa_heads.") or int(k.split(".")[1]) <= K}
                mK = WhisperMedusaModel(cK, sdK).to(device)
                run_streams(mK, clips, [args.steps], language, alpha, max_iters=4)
                trK, _, _ = run_streams(mK, clips, range(min(2, args.steps)), language, alpha)
                sK = summarize(cK, trK, peak)
                k_sweep[str(K)] = {k: sK[k] for k in ("tokens_per_s", "ms_per_iteration", "tokens_per_iteration", "mean_accept", "frac")}
                mK.close()
    # ---- BASELINE configs[3]: concurrent streams per GPU (SURVEY 8(f) rank 3).  S engines share the weight blob and
    # decode on n_sm / S CTAs each; 2 S clips per GPU (two waves).  Rank 0 measures; every stream's tokens are checked
    # against the batch-1 run of the same clip.
    multi = None
    if rank == 0 and not args.no_extras and args.streams > 1:
        from whisper_medusa_b200 import StreamGroup

        try:
            n_clips = 2 * args.streams
            mclips = [clips[i % len(clips)] for i in range(n_clips)]
            want = [outs[i % len(clips)] if (i % len(clips)) < args.steps else None for i in range(n_clips)]
            grp = StreamGroup(cfg, None, device, n_streams=args.streams, weights_from=model)
            gkw = dict(language=language, exponential_decay_length_penalty=PENALTY, posterior_alpha=alpha)
            grp.generate_from_pcm(mclips[: args.streams], **dict(gkw, max_iters=4))
            torch.cuda.synchronize(device)
            got = [o[0].tolist() for o in grp.generate_from_pcm(mclips, **gkw)]
            bad = [i for i, (g_, w_) in enumerate(zip(got, want)) if w_ is not None and g_ != w_]
            if bad:
                raise SystemExit(f"bench: concurrent streams {bad} differ from their batch-1 runs")
            sM = summarize(cfg, grp.last_traces, peak)
            enc_s = sum(t.ms_encoder + t.ms_mel for t in grp.last_traces) / 1e3
            # decode phase = the busiest engine's summed decode-loop device times (CUDA events on its own stream; the
            # engines decode concurrently, a queued clip's encoder runs on the SMs its own engine leaves free)
            dec_s = max(1e-9, grp.last_decode_phase_s)
            multi = {"streams": args.streams, "ctas_per_stream": grp.ctas_per_stream, "clips": n_clips,
                     "tokens_per_s_e2e": sM["tokens"] / grp.last_wall_s, "tokens_per_s_decode_phase": sM["tokens"] / dec_s,
                     "ms_per_iteration_per_stream": sM["ms_per_iteration"], "achieved_gbs": sM["bytes_eng"] / dec_s / 1e9,
                     "frac": sM["bytes_eng"] / dec_s / 1e9 / peak, "vs_batch1_decode": (sM["tokens"] / dec_s) / sm["tokens_per_s"],
                     # steady state (all S engines decoding): S iterations every ms_per_iteration_per_stream
                     "steady_state_iteration_rate_vs_batch1": args.streams * sm["ms_per_iteration"] / sM["ms_per_iteration"],
                     "steady_state_frac": args.streams * (sM["bytes_eng"] / max(1, sM["iterations"])) / (sM["ms_per_iteration"] / 1e3) / 1e9 / peak,
                     "validated": "every stream == its batch-1 tokens", "wall_s": grp.last_wall_s, "encoder_s": enc_s}
            grp.close()
        except SystemExit:
            raise
        except Exception as e:  # noqa: BLE001
            multi = {"streams": args.streams, "error": f"{type(e).__name__}: {e}"}
    if rank != 0:
        if dist is not None:
            dist.barrier()
            dist.destroy_process_group()
        return
    tot_tok = float(allv[:, 0].sum())
    tot_iter = float(allv[:, 1].sum())
    max_dec_ms = float(allv[:, 2].max())
    max_wall = float(allv[:, 3].max())
    value = tot_tok / (max_dec_ms / 1e3)
    e2e_value = tot_tok / max_wall
    tok_iter = tot_tok / max(1.0, tot_iter)
    ref_roofline_tok_s = peak * 1e9 / (sm["bytes_ref"] / max(1, sm["iterations"])) * tok_iter   # per GPU
    result = {
        "metric": METRIC, "value": value, "unit": "tokens/s", "n_gpus": world, "steps": args.steps, "warmup": args.warmup,
        "ms_per_step": 1e3 * max_wall / args.steps, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
        "dtype": "fp16 weights+KV / fp32 accumulate", "data": "synthetic", "config": config,
        "e2e": {"value": e2e_value, "unit": "tokens/s", "h2d_bytes_per_step": 480000 * 4,
                "d2h_bytes_per_step": int(4 * tot_tok / max(1, world * args.steps)) + 16 * 4},
        "gpu_launches": int(allv[:, 6].sum()),
        "clocks": clocks,
        "roofline": {"bound": "hbm", "achieved": sm["achieved_gbs"], "peak": peak, "unit": "GB/s", "frac": sm["frac"],
                     "peak_source": peak_src,
                     "kernel": "dec_iteration_ring_kernel (one launch = one speculative iteration)"
                     if args.mode == "persistent" else f"decode iteration ({args.mode})",
                     "algorithmic_bytes_per_iteration": sm["bytes_eng"] / max(1, sm["iterations"]),
                     "ms_per_iteration": sm["ms_per_iteration"],
                     "reference_schedule_bytes_per_iteration": sm["bytes_ref"] / max(1, sm["iterations"]),
                     "frac_of_reference_schedule_roofline": (value / world) / ref_roofline_tok_s},
        "detail": {"decode_mode": args.mode, "tokens_per_step": tot_tok / (world * args.steps),
                   "iterations_per_step": tot_iter / (world * args.steps), "tokens_per_iteration": tok_iter,
                   "mean_accept": sm["mean_accept"], "accept_hist": sm["accept_hist"],
                   "two_sweep_iterations": sm["two_sweep_iterations"],
                   "ms_mel": float(allv[0, 5]) / args.steps, "ms_encoder": float(allv[0, 4]) / args.steps,
                   "ms_decode": float(allv[0, 2]) / args.steps, "validated": validated,
                   "regimes": regimes, "k_sweep": k_sweep, "multi_stream": multi},
    }
    if not args.no_cpu_baseline:
        try:
            if sd is None:
                sd = synthetic_state_dict(cfg, seed=0)
            ref = CpuReference(cfg, sd, clips[0].numpy(), threads, alpha)
            n, it, dt = ref.step(args.cpu_iters)
            result["cpu_baseline"] = {
                "value": n / dt, "unit": "tokens/s", "cores": threads, "kind": "port",
                "sample": (f"stream 0: first {it} speculative iterations ({n} tokens) of the decode loop in {dt:.2f} s, encoder "
                           f"output resident (log-mel {ref.s_mel:.2f} s + encoder {ref.s_encoder:.2f} s, not included)")}
        except Exception as e:  # noqa: BLE001
            result["cpu_baseline"] = {"value": None, "unit": "tokens/s", "cores": threads, "kind": "port", "sample": f"failed: {e}"}
    print(json.dumps(result))
    if dist is not None:
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
