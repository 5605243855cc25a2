"""Several audio streams decoded CONCURRENTLY on one GPU (SURVEY.md 8(f) rank 3; the reference asserts batch 1,
``whisper_medusa/models/model.py:1451``, and decodes streams back to back).

One speculative iteration is a chain of ~260 dependent stages, each bounded by on-chip latencies, not by HBM: a
single stream on all SMs leaves most of the memory bandwidth unused.  A ``StreamGroup`` therefore partitions the SMs:
S engine handles share ONE copy of the packed weights (``wm_weights_device_ptr`` -> ``wm_adopt_weights``), each runs its
persistent decode kernel on ``n_sm / S`` CTAs (option ``decode_ctas``) and on its own CUDA stream, so S cooperative
kernels are co-resident and S weight streams are in flight at once.  Every stream computes exactly what it computes
alone (same kernels, same per-stream state): token ids are bit-identical to the batch-1 run.
"""
from __future__ import annotations

import queue
import threading
from typing import Dict, List, Optional, Sequence, Union

import numpy as np
import torch

from .config import MedusaConfig
from .model import EngineError, GenerateTrace, WhisperMedusaModel


class StreamGroup:
    """``n_streams`` engines on one device sharing one weight blob; ``generate_*`` take a list of clips and run up to
    ``n_streams`` of them at a time (further clips queue: 8 streams per GPU on a 4-way group = two waves)."""

    def __init__(self, config: MedusaConfig, state_dict: Optional[Dict[str, torch.Tensor]], device: Union[str, torch.device],
                 n_streams: int = 4, ctas_per_stream: Optional[int] = None, broadcast_src: Optional[int] = None,
                 weights_from: Optional[WhisperMedusaModel] = None):
        device = torch.device(device)
        if device.type != "cuda":
            raise EngineError("StreamGroup runs on CUDA devices only")
        index = device.index if device.index is not None else torch.cuda.current_device()
        n_sm = torch.cuda.get_device_properties(index).multi_processor_count
        if n_streams < 1 or n_streams > 8:
            raise ValueError("n_streams must be in 1..8")
        self.n_streams = int(n_streams)
        self.ctas_per_stream = int(ctas_per_stream) if ctas_per_stream else n_sm // self.n_streams
        if self.ctas_per_stream * self.n_streams > n_sm:
            raise ValueError(f"{self.n_streams} x {self.ctas_per_stream} CTAs do not fit {n_sm} SMs (the kernels must be co-resident)")
        if weights_from is not None:     # an engine of the same shape already on this GPU: adopt its blob (no second upload)
            first = WhisperMedusaModel(config, None).to(torch.device("cuda", index), weights_from=weights_from)
            first.generation_config = weights_from.generation_config
        else:
            first = WhisperMedusaModel(config, state_dict).to(torch.device("cuda", index), broadcast_src=broadcast_src)
        self.models: List[WhisperMedusaModel] = [first]
        for _ in range(1, self.n_streams):
            self.models.append(WhisperMedusaModel(config, None).to(torch.device("cuda", index), weights_from=first))
        for m in self.models:
            m.generation_config = first.generation_config
            if self.n_streams > 1:
                m.set_option("decode_ctas", self.ctas_per_stream)
        self.config = config
        self.device = torch.device("cuda", index)
        self.last_traces: List[GenerateTrace] = []
        self.last_windows: List[list] = []
        self.last_wall_s = 0.0
        self.last_decode_phase_s = 0.0

    def close(self) -> None:
        for m in reversed(self.models):
            m.close()

    # ------------------------------------------------------------------------------------------------
    def _run(self, clips: Sequence, call, kwargs) -> List[torch.Tensor]:
        import time

        n = len(clips)
        outs: List[Optional[torch.Tensor]] = [None] * n
        traces: List[Optional[GenerateTrace]] = [None] * n
        errors: List[BaseException] = []
        work: "queue.Queue[int]" = queue.Queue()
        for i in range(n):
            work.put(i)

        def worker(model: WhisperMedusaModel, widx: int):
            # one host thread per engine: ctypes releases the GIL inside the C ABI calls, so the S loops enqueue and
            # wait concurrently; each engine owns its CUDA stream
            while True:
                try:
                    i = work.get_nowait()
                except queue.Empty:
                    return
                try:
                    outs[i] = call(model, clips[i], kwargs)
                    traces[i] = model.last_trace
                    traces[i].engine_index = widx
                except BaseException as e:  # noqa: BLE001
                    errors.append(e)
                    return

        t0 = time.perf_counter()
        threads = [threading.Thread(target=worker, args=(m, k)) for k, m in enumerate(self.models[: max(1, min(self.n_streams, n))])]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
        self.last_wall_s = time.perf_counter() - t0
        if errors:
            raise errors[0]
        self.last_traces = traces  # type: ignore[assignment]
        # length of the decode phase: the engines decode concurrently, each for the sum of its own loops' device times
        busy: Dict[int, float] = {}
        for t in traces:
            busy[t.engine_index] = busy.get(t.engine_index, 0.0) + t.ms_decode  # type: ignore[union-attr]
        self.last_decode_phase_s = max(busy.values()) / 1e3 if busy else 0.0
        return outs  # type: ignore[return-value]

    def generate_from_pcm(self, clips: Sequence[Union[np.ndarray, torch.Tensor]], **kwargs) -> List[torch.Tensor]:
        """16 kHz mono PCM clips (each <= 30 s) -> one ``LongTensor[1, n_i]`` per clip (arguments of
        ``WhisperMedusaModel.generate_from_pcm``)."""
        return self._run(clips, lambda m, x, kw: m.generate_from_pcm(x, **kw), kwargs)

    def transcribe(self, recordings, sampling_rate: Union[int, Sequence[int]] = 16000, chunk_length_s: float = 30.0,
                   stride_length_s=None, **kwargs) -> List[torch.Tensor]:
        """Long-form ``WhisperMedusaModel.transcribe`` of one recording or a list of them (``sampling_rate``: one rate
        for all, or one per recording) -> one ``LongTensor[1, n_i]`` per recording.

        Each recording is uploaded and resampled once into a device buffer that every engine reads; the windows of all
        recordings go into one work queue, so they decode concurrently on the S engines, and each recording's windows
        are merged in order.  The results equal ``model.transcribe`` of each recording, with the same
        ``no_speech_threshold`` / ``logprob_threshold`` rule and ``return_token_timestamps`` / ``time_precision`` (then
        one ``MedusaGenerateOutput`` per recording).  Per-window results: ``self.last_windows[i]`` for recording i."""
        from .longform import plan_windows, window_params
        from .model import _check_recording

        recs = [recordings] if isinstance(recordings, (np.ndarray, torch.Tensor)) else list(recordings)
        rates = list(sampling_rate) if isinstance(sampling_rate, (list, tuple)) else [sampling_rate] * len(recs)
        if len(rates) != len(recs):
            raise ValueError(f"{len(rates)} sampling rates for {len(recs)} recordings")
        params = window_params(chunk_length_s, stride_length_s)
        for r, sr in zip(recs, rates):
            _check_recording(r, sr)
        lead = self.models[0]
        # (same rules and arguments as model.transcribe)
        fallback, no_speech, temperature = lead._fallback_request(
            kwargs.get("temperature"), kwargs.pop("compression_ratio_threshold", None),
            kwargs.pop("logprob_threshold", None), kwargs.pop("no_speech_threshold", None), kwargs.pop("top_k", None))
        if no_speech is not None:
            kwargs["no_speech"] = no_speech
        if fallback is not None:
            kwargs["fallback"] = fallback
        kwargs["temperature"] = temperature
        timed = bool(kwargs.pop("return_token_timestamps", None))
        time_precision = kwargs.pop("time_precision", 0.02)
        lead._check_unsupported(temperature, None, {k: v for k, v in kwargs.items()
                                                    if k not in ("language", "task", "temperature", "no_speech", "fallback")})
        lead._logits_processors(kwargs)
        if timed:
            lead._timestamp_request(None, kwargs.get("task"), None, time_precision)
            kwargs["time_precision"] = float(time_precision)
        # one seed per recording, drawn in recording order: the same draws as model.transcribe of each in turn
        seeds = [lead._recording_seed() for _ in recs] if fallback is not None else None
        x16 = [lead._upload_16k(r, sr) for r, sr in zip(recs, rates)]
        stream = torch.cuda.current_stream(self.device).cuda_stream     # every window's encode is ordered after it
        items = [(i, k, w) for i, x in enumerate(x16) for k, w in enumerate(plan_windows(x.numel(), *params))]

        def window(m, it, kw):
            seed = {"seed": (seeds[it[0]], it[1])} if seeds is not None else {}
            return m._transcribe_window(x16[it[0]], it[2], stream, **seed, **kw)

        results = self._run(items, window, kwargs)
        self.last_windows = [[res for (i, _, _), res in zip(items, results) if i == k] for k in range(len(recs))]
        return [lead._merge_results(ws, timed) for ws in self.last_windows]

    def generate(self, input_features: torch.Tensor, **kwargs) -> List[torch.Tensor]:
        """``input_features [B, 80, 3000]`` with any B (the batch dimension the reference refuses, model.py:1451):
        one result per row.  ``attention_mask [B, 3000]`` (the feature extractor's): row i goes with clip i."""
        B = input_features.shape[0]
        mask = kwargs.pop("attention_mask", None)
        if mask is not None:
            mask = torch.as_tensor(mask)
            if mask.dim() == 1:
                mask = mask[None]
            if mask.dim() != 2 or mask.shape[0] != B:
                raise ValueError(f"attention_mask must have one row per clip, [{B}, 3000], got shape {tuple(mask.shape)}")
        rows = [(input_features[i : i + 1], None if mask is None else mask[i : i + 1]) for i in range(B)]
        return self._run(rows, lambda m, x, kw: m.generate(x[0], **kw) if x[1] is None else
                         m.generate(x[0], attention_mask=x[1], **kw), kwargs)
