"""Drop-in host for the reference's decode path: ``WhisperMedusaModel.from_pretrained / .to /
.generate`` (reference ``whisper_medusa/models/model.py:213``, re-exported at
``whisper_medusa/__init__.py:1``) over the C ABI in ``include/whisper_medusa_b200.h``.

Same names, argument meaning and error behaviour as the reference for this path:

* ``generate`` asserts batch size 1 (``model.py:1451``);
* ``return_timestamps`` -> ``NotImplementedError`` (``:1171-1174``); ``no_speech_threshold`` ->
  ``NotImplementedError`` (``:1201-1204``); more than 3000 feature frames (long-form) ->
  ``NotImplementedError`` (``:1213-1214``); beam search -> ``Exception`` (``:1153-1156``);
* the returned ``LongTensor[1, n]`` has the prompt and the trailing EOS stripped (``:1929-1973``).

Beyond the reference (which takes 16 kHz clips of at most 30 s): ``transcribe`` takes a recording of any length at any
integer sampling rate, with the semantics of HF's chunked ASR pipeline (``longform.py``); ``generate_from_pcm`` takes
``sampling_rate``.  Both resample on the GPU (``csrc/resample.cu``).

There is no PyTorch / CPU fallback: every tensor op of the path runs in the CUDA engine, and the
constructor raises if the engine library is missing.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Dict, List, Optional, Sequence, Tuple, Union

import numpy as np
import torch

from . import _lib
from .config import MedusaConfig, MedusaGenerationConfig
from .longform import (MAX_WINDOW_SAMPLES, SAMPLE_RATE, Window, WindowResult, merge_windows, plan_windows,
                       resampled_length, text_ids, window_params)
from .weights import pack_blob

N_FRAMES = 3000


def _rate(sampling_rate) -> int:
    """A sampling rate as a positive integer (the resampler supports integer rates only)."""
    if isinstance(sampling_rate, bool) or int(sampling_rate) != sampling_rate or int(sampling_rate) <= 0:
        raise ValueError(f"sampling_rate must be a positive integer number of Hz, got {sampling_rate!r}")
    return int(sampling_rate)


def _check_recording(audio, sampling_rate) -> None:
    _rate(sampling_rate)
    ndim = audio.dim() if isinstance(audio, torch.Tensor) else np.ndim(audio)
    if ndim != 1:
        raise ValueError(f"audio must be a 1-D mono recording, got {ndim} dimensions (downmix multi-channel audio first)")


class EngineError(RuntimeError):
    pass


def _check(lib, handle, rc: int, what: str) -> None:
    if rc != 0:
        msg = lib.wm_last_error(handle).decode() if handle else ""
        raise EngineError(f"{what}: {lib.wm_strerror(rc).decode()} ({rc}) {msg}")


def _load_state_dict(path: str) -> Dict[str, torch.Tensor]:
    """Weights of an HF checkpoint directory, whichever way `save_pretrained` wrote them: one
    ``model.safetensors``, shards listed in ``model.safetensors.index.json`` (what HF writes above its
    shard size -- whisper-large-v2 in fp32 is 6.2 GB), or the legacy ``pytorch_model.bin`` (+ index).
    Any floating dtype is accepted: the packer casts matrices to fp16 and vectors to fp32 (weights.py)."""
    import json

    def shards(index_file: str) -> List[str]:
        with open(os.path.join(path, index_file)) as f:
            return sorted(set(json.load(f)["weight_map"].values()))

    sd: Dict[str, torch.Tensor] = {}
    if os.path.isfile(os.path.join(path, "model.safetensors")) or os.path.isfile(os.path.join(path, "model.safetensors.index.json")):
        from safetensors.torch import load_file

        files = ["model.safetensors"] if os.path.isfile(os.path.join(path, "model.safetensors")) else shards("model.safetensors.index.json")
        for fn in files:
            sd.update(load_file(os.path.join(path, fn)))
    elif os.path.isfile(os.path.join(path, "pytorch_model.bin")) or os.path.isfile(os.path.join(path, "pytorch_model.bin.index.json")):
        files = ["pytorch_model.bin"] if os.path.isfile(os.path.join(path, "pytorch_model.bin")) else shards("pytorch_model.bin.index.json")
        for fn in files:
            sd.update(torch.load(os.path.join(path, fn), map_location="cpu", weights_only=True))
    else:
        raise OSError(f"no model.safetensors / pytorch_model.bin (or their shard indices) in {path}")
    return sd


class ForwardOutput:
    """What ``forward`` returns: the fields of the reference's ``Seq2SeqLMOutput`` that an inference engine can fill
    (reference ``model.py:1335-1347``)."""

    def __init__(self, logits: torch.Tensor):
        self.logits = logits     # [K+1, 1, T, V] stacked head logits (``[1, 1, T, V]`` with disable_medusa)
        self.loss = None

    def __getitem__(self, i):    # outputs[0] / outputs["logits"] as HF ModelOutput allows
        if i in (0, "logits"):
            return self.logits
        raise KeyError(i)


class GenerateTrace:
    """Per-call measurements (the reference collects ``accept_length_list`` but drops it,
    ``model.py:633,705``)."""

    def __init__(self):
        self.accept_lengths: List[int] = []
        self.iterations = 0
        self.sequences: List[int] = []       # prompt + generated, after the post-EOS fill
        self.n_new_tokens = 0                 # effective decoded tokens (up to and incl. first EOS)
        self.ms_mel = self.ms_encoder = self.ms_decode = 0.0
        self.launches_encode = self.launches_decode = 0
        self.cluster_decode = 1                # CTAs per cluster of the persistent ring kernel


class WhisperMedusaModel:
    """Whisper + Medusa heads, inference only, CUDA engine behind the reference's API."""

    def __init__(self, config: MedusaConfig, state_dict: Optional[Dict[str, torch.Tensor]] = None):
        _lib.load()  # fail loudly here, not at first generate
        self.config = config
        self.generation_config = MedusaGenerationConfig.from_model_config(config)   # model.py:258-263
        self.generation_config.update(**{k: v for k, v in config.to_dict().items()
                                         if k in ("posterior_threshold", "posterior_alpha")})
        self._state_dict = state_dict
        self._handle = None
        self._device: Optional[torch.device] = None
        self._wblob_dev: Optional[torch.Tensor] = None
        self.last_trace = GenerateTrace()
        self.last_windows: List[WindowResult] = []    # per-window results of the last transcribe()
        if len(config.medusa_choices) != config.medusa_num_heads + 1:
            raise ValueError("len(medusa_choices) must be medusa_num_heads + 1")

    # ------------------------------------------------------------------ construction
    @classmethod
    def from_pretrained(cls, pretrained_model_name_or_path: str, *args, **kwargs) -> "WhisperMedusaModel":
        """Reference ``model.py:265-291``: config.json (+ generation_config.json) + model.safetensors."""
        path = pretrained_model_name_or_path
        if not os.path.isdir(path):
            raise OSError(f"{path} is not a local directory (hub access is not available)")
        config = MedusaConfig.from_pretrained(path)
        sd = _load_state_dict(path)
        if "whisper_model.proj_out.weight" not in sd:  # tied weight is not serialised by safetensors
            sd["whisper_model.proj_out.weight"] = sd["whisper_model.model.decoder.embed_tokens.weight"]
        model = cls(config, sd)
        try:
            model.generation_config = MedusaGenerationConfig.from_pretrained(path)
        except OSError:
            pass  # reference model.py:286-290
        return model

    def save_pretrained(self, path: str) -> None:
        from safetensors.torch import save_file

        if self._state_dict is None:
            raise RuntimeError("state dict was released")
        os.makedirs(path, exist_ok=True)
        self.config.save_pretrained(path)
        self.generation_config.save_pretrained(path)
        sd = {k: v.contiguous() for k, v in self._state_dict.items() if k != "whisper_model.proj_out.weight"}
        save_file(sd, os.path.join(path, "model.safetensors"))

    def get_medusa_choice(self):
        return self.config.medusa_choices

    @property
    def device(self) -> torch.device:
        return self._device if self._device is not None else torch.device("cpu")

    # ------------------------------------------------------------------ engine
    def _wm_config(self) -> _lib.WmConfig:
        c = self.config
        if c.encoder_attention_heads != c.decoder_attention_heads or c.encoder_ffn_dim != c.decoder_ffn_dim:
            raise NotImplementedError("encoder and decoder must share heads / ffn width (true for every Whisper size)")
        return _lib.WmConfig(
            vocab_size=c.vocab_size, d_model=c.d_model, n_heads=c.decoder_attention_heads, ffn_dim=c.decoder_ffn_dim,
            enc_layers=c.encoder_layers, dec_layers=c.decoder_layers, n_mels=c.num_mel_bins,
            max_source_positions=c.max_source_positions, max_target_positions=c.max_target_positions,
            medusa_num_heads=c.medusa_num_heads, medusa_block=1 if c.is_block else 0)

    def to(self, device: Union[str, torch.device], broadcast_src: Optional[int] = None,
           weights_from: Optional["WhisperMedusaModel"] = None) -> "WhisperMedusaModel":
        """Create the engine on ``device`` and upload the packed weights.

        ``weights_from`` = another model of the same shape already on this GPU: its device blob is adopted instead
        of a second upload (every concurrent stream of a ``StreamGroup`` reads the same 3.1 GB).

        With ``broadcast_src`` (inside an initialised ``torch.distributed`` NCCL group) only that rank
        packs the checkpoint; the blob reaches the other GPUs with one NCCL broadcast over NVLink and
        the engine adopts the device buffer (``wm_adopt_weights``) -- the only collective of the path.
        """
        device = torch.device(device)
        if device.type != "cuda":
            raise EngineError("WhisperMedusaModel (H100 engine) runs on CUDA devices only; there is no CPU path")
        index = device.index if device.index is not None else torch.cuda.current_device()
        lib = _lib.load()
        if self._handle is not None:
            if self._device == torch.device("cuda", index):
                return self
            self.close()
        handle = C.c_void_p()
        cfg = self._wm_config()
        rc = lib.wm_create(C.byref(cfg), index, C.byref(handle))
        if rc != 0:
            msg = lib.wm_last_error(handle).decode() if handle else ""
            if handle:
                lib.wm_destroy(handle)
            raise EngineError(f"wm_create: {lib.wm_strerror(rc).decode()} {msg}")
        self._handle = handle
        self._device = torch.device("cuda", index)
        nbytes = lib.wm_weights_nbytes(handle)
        if weights_from is not None:
            weights_from._require_engine()
            if weights_from._device != self._device or lib.wm_weights_nbytes(weights_from._handle) != nbytes:
                raise EngineError("weights_from must be a model of the same shape on the same device")
            ptr = lib.wm_weights_device_ptr(weights_from._handle)
            if not ptr:
                raise EngineError("weights_from has no weights loaded")
            self._weights_owner = weights_from     # keep the owning engine alive
            _check(lib, handle, lib.wm_adopt_weights(handle, C.c_void_p(ptr), nbytes), "wm_adopt_weights")
        elif broadcast_src is None:
            if self._state_dict is None:
                raise RuntimeError("no state dict to upload")
            blob = pack_blob(handle, self.config, self._state_dict)
            _check(lib, handle, lib.wm_load_weights(handle, C.c_void_p(blob.data_ptr()), nbytes), "wm_load_weights")
        else:
            import torch.distributed as dist

            from .parallel import broadcast_packed_weights

            with torch.cuda.device(index):
                blob = pack_blob(handle, self.config, self._state_dict) if dist.get_rank() == broadcast_src else None
                dev_blob = broadcast_packed_weights(nbytes, broadcast_src, blob, self._device)
                torch.cuda.synchronize(index)
            self._wblob_dev = dev_blob  # keep alive: the engine does not own it
            _check(lib, handle, lib.wm_adopt_weights(handle, C.c_void_p(dev_blob.data_ptr()), nbytes), "wm_adopt_weights")
        self._push_suppress()
        # candidate tree (all ones = the top-1 chain the reference ships, README.md:181; branching choices: per-head
        # top-k + tree verify, medusa_utils.py:305-458 -- the engine holds trees of <= 16 nodes / 32 paths / k <= 4)
        ch = [int(c) for c in self.config.medusa_choices]
        arr = (C.c_int32 * len(ch))(*ch)
        rc = lib.wm_set_medusa_choices(handle, arr, len(ch))
        if rc == -4:
            raise NotImplementedError(f"medusa_choices {ch}: {lib.wm_last_error(handle).decode()}")
        _check(lib, handle, rc, "wm_set_medusa_choices")
        return self

    def cuda(self, index: int = 0) -> "WhisperMedusaModel":
        return self.to(torch.device("cuda", index))

    def eval(self) -> "WhisperMedusaModel":
        return self

    def release_state_dict(self) -> None:
        """Drop the host copy of the checkpoint once it is on the device."""
        self._state_dict = None

    def close(self) -> None:
        if self._handle is not None:
            _lib.load().wm_destroy(self._handle)
            self._handle = None
            self._wblob_dev = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_decode_mode(self, mode: str) -> None:
        """``"graph"``: CUDA graphs of stage kernels (debug / per-stage profiling); ``"persistent"``: one
        cooperative kernel per speculative iteration with the weight ring (product path);
        ``"persistent_simple"``: the same without the ring (grid barriers only).  A mode the engine cannot run here
        (``"persistent"`` at a decoder width without a ring-kernel instantiation) raises ``EngineError``."""
        self._require_engine()
        lib = _lib.load()
        rc = lib.wm_set_decode_mode(self._handle, {"graph": 0, "persistent_simple": 1, "persistent": 2}[mode])
        if rc < 0:
            _check(lib, self._handle, rc, f"set_decode_mode({mode!r})")

    def set_option(self, key: str, value: int) -> None:
        """Engine options (``wm_set_option``): ``enc_gemm`` 0 = mma.sync, 1 = wgmma/TMA encoder GEMM."""
        self._require_engine()
        lib = _lib.load()
        _check(lib, self._handle, lib.wm_set_option(self._handle, key.encode(), int(value)), f"wm_set_option({key})")

    def _require_engine(self):
        if self._handle is None:
            raise EngineError("call .to('cuda') first: the model has no CPU execution path")

    def _push_suppress(self):
        lib = _lib.load()
        g = self.generation_config
        sup = list(g.suppress_tokens or [])
        beg = list(g.begin_suppress_tokens or [])
        a = (C.c_int32 * max(1, len(sup)))(*sup)
        b = (C.c_int32 * max(1, len(beg)))(*beg)
        _check(lib, self._handle, lib.wm_set_suppress(self._handle, a, len(sup), b, len(beg)), "wm_set_suppress")
        self._pushed = (tuple(sup), tuple(beg))

    # ------------------------------------------------------------------ generate
    def _init_tokens(self, language: Optional[str], task: Optional[str], g=None) -> List[int]:
        """Prompt ids for the supported cases of HF ``generation_whisper.py:1455-1608``."""
        g = g if g is not None else self.generation_config
        toks = [int(g.decoder_start_token_id)]
        if g.is_multilingual:
            if language is None:
                lang_id = self._detect_language(g)
            else:
                from .config import language_token

                key = language_token(language)
                if key not in g.lang_to_id:
                    raise ValueError(f"Unsupported language: {language}. Language should be one of: {sorted(g.lang_to_id)}.")
                lang_id = int(g.lang_to_id[key])
            toks.append(lang_id)
            toks.append(int(g.task_to_id[task or "transcribe"]))
        elif language is not None or task is not None:
            raise ValueError("Cannot specify `task` or `language` for an English-only model")
        toks.append(int(g.no_timestamps_token_id))
        return toks

    def _detect_language(self, g=None) -> int:
        """HF ``generation_whisper.py:1559-1566`` / ``detect_language``: one decoder step on ``<|startoftranscript|>``;
        the language token with the largest base logit wins (all non-language ids masked)."""
        g = g if g is not None else self.generation_config
        lang_ids = sorted(int(v) for v in g.lang_to_id.values())
        if not lang_ids:
            raise ValueError("generation_config.lang_to_id is empty: cannot detect the language")
        logits = self.forward(decoder_input_ids=torch.tensor([[int(g.decoder_start_token_id)]]), disable_medusa=True).logits
        row = logits[0, 0, -1]
        return lang_ids[int(torch.argmax(row[torch.tensor(lang_ids)]))]

    def _gen_params(self, prompt_len: int, exponential_decay_length_penalty, max_length, temperature,
                    max_iters, g=None) -> _lib.WmGenParams:
        g = g if g is not None else self.generation_config
        pen = exponential_decay_length_penalty if exponential_decay_length_penalty is not None \
            else g.exponential_decay_length_penalty
        return _lib.WmGenParams(
            max_length=int(max_length if max_length is not None else g.max_length),
            eos_token_id=int(g.eos_token_id), pad_token_id=int(g.pad_token_id), begin_index=prompt_len,
            temperature=float(temperature), posterior_threshold=float(g.posterior_threshold),
            posterior_alpha=float(g.posterior_alpha),
            penalty_start=int(pen[0]) if pen is not None else -1,
            penalty_factor=float(pen[1]) if pen is not None else 1.0,
            max_iters=int(max_iters or 0), tree_attention=0)

    def _run_loop(self, prompt: Sequence[int], gp: _lib.WmGenParams) -> GenerateTrace:
        lib = _lib.load()
        cap = int(gp.max_length) + self.config.medusa_num_heads + 8
        out = (C.c_int32 * cap)()
        acc = (C.c_int32 * cap)()
        n_out, n_iter = C.c_int32(0), C.c_int32(0)
        p = (C.c_int32 * len(prompt))(*prompt)
        _check(lib, self._handle,
               lib.wm_generate(self._handle, p, len(prompt), C.byref(gp), out, C.byref(n_out), acc, C.byref(n_iter)),
               "wm_generate")
        tr = GenerateTrace()
        tr.sequences = list(out[: n_out.value])
        tr.accept_lengths = list(acc[: n_iter.value])
        tr.iterations = n_iter.value
        gen = tr.sequences[len(prompt):]
        eos = int(gp.eos_token_id)
        tr.n_new_tokens = gen.index(eos) + 1 if eos in gen else len(gen)
        tr.ms_mel, tr.ms_encoder, tr.ms_decode = (lib.wm_last_ms(self._handle, i) for i in range(3))
        tr.launches_encode = lib.wm_last_launches(self._handle, 1)
        tr.launches_decode = lib.wm_last_launches(self._handle, 2)
        tr.cluster_decode = lib.wm_decode_cluster(self._handle)
        return tr

    @staticmethod
    def _strip(sequences: Sequence[int], prompt_len: int, pad: int, eos: int) -> List[int]:
        """Reference ``model.py:1929`` (drop prompt) + ``:1950-1973`` (drop trailing pad / EOS)."""
        seq = list(sequences[prompt_len:])
        if seq and seq[-1] == pad:
            n_pad = sum(1 for t in seq if t == pad)
            if pad == eos:
                n_pad -= 1
            if n_pad != 0:
                seq = seq[:-n_pad]
        if seq and seq[-1] == eos:
            seq = seq[:-1]
        return seq

    def generate(self, input_features: Optional[torch.Tensor] = None, generation_config=None, logits_processor=None,
                 stopping_criteria=None, prefix_allowed_tokens_fn=None, synced_gpus: bool = False,
                 return_timestamps: Optional[bool] = None, task: Optional[str] = None, language: Optional[str] = None,
                 is_multilingual: Optional[bool] = None, prompt_ids=None, prompt_condition_type=None,
                 condition_on_prev_tokens=None, temperature=None, compression_ratio_threshold=None,
                 logprob_threshold=None, no_speech_threshold=None, num_segment_frames=None, attention_mask=None,
                 time_precision: float = 0.02, return_token_timestamps=None, return_segments: bool = False,
                 return_dict_in_generate=None, **kwargs) -> torch.Tensor:
        """Transcribe one <= 30 s clip given its log-mel features ``[1, 80, 3000]``
        (reference ``model.py:1419-1779``); returns ``LongTensor[1, n]``."""
        self._require_engine()
        if input_features is None:
            raise ValueError("input_features is required")
        assert input_features.shape[0] == 1, "Batch size should be 1 for medusa generation"   # model.py:1451
        if return_timestamps is True or getattr(self.generation_config, "return_timestamps", False) is True:
            raise NotImplementedError("return_timestamps is not supported with medusa for now")       # :1171
        nst = no_speech_threshold if no_speech_threshold is not None else self.generation_config.no_speech_threshold
        if nst is not None:
            raise NotImplementedError("no_speech_detection is not supported with medusa for now")     # :1201
        if input_features.shape[-1] > N_FRAMES:
            raise NotImplementedError("Longform generation is not supported yet")                     # :1213
        if kwargs.get("num_beams", 1) not in (None, 1):
            raise Exception("Only greedy search is supported with medusa (beam modes raise in the reference, model.py:1153-1156)")
        for unsupported in (logits_processor, stopping_criteria, prefix_allowed_tokens_fn, prompt_ids):
            if unsupported:
                raise NotImplementedError("custom logits processors / stopping criteria / prompt_ids are not implemented")
        if input_features.shape[-1] != N_FRAMES or input_features.shape[-2] != self.config.num_mel_bins:
            raise ValueError(f"input_features must be [1, {self.config.num_mel_bins}, {N_FRAMES}] (WhisperProcessor output)")
        self._check_unsupported(temperature, attention_mask, kwargs)
        self._encode_features(input_features)
        return self._decode(language, task, kwargs, temperature, generation_config)

    def _encode_features(self, input_features: torch.Tensor) -> None:
        lib = _lib.load()
        if input_features.is_cuda:
            # device-resident features (the reference's callers do input_features.to(device) first): one
            # device-to-device copy ordered after the producing stream, no host round trip
            if input_features.device != self._device:
                raise EngineError(f"input_features are on {input_features.device}, the engine on {self._device}")
            mel = input_features.detach().to(torch.float32).contiguous()
            stream = torch.cuda.current_stream(self._device).cuda_stream
            _check(lib, self._handle, lib.wm_encode_mel_device(self._handle, C.c_void_p(mel.data_ptr()), C.c_void_p(stream)),
                   "wm_encode_mel_device")
        else:
            mel = input_features.detach().to(torch.float32).contiguous()
            _check(lib, self._handle, lib.wm_encode_mel(self._handle, C.cast(mel.data_ptr(), C.POINTER(C.c_float))),
                   "wm_encode_mel")

    @staticmethod
    def _check_unsupported(temperature, attention_mask, kwargs) -> None:
        """Options the reference accepts but cannot honour on this path fail loudly instead of being dropped."""
        temps = temperature if isinstance(temperature, (tuple, list)) else (temperature,)
        if any(t not in (None, 0, 0.0) for t in temps) or kwargs.get("do_sample"):
            # generate_with_fallback turns temperature > 0 into do_sample=True (model.py:1878-1881), and
            # _multi_heads_generate has no sampling branch (model.py:1130-1156)
            raise NotImplementedError("sampling (temperature > 0 / do_sample) is not supported with medusa: greedy search only")
        known = {"exponential_decay_length_penalty", "max_length", "max_new_tokens", "max_iters", "medusa_temperature",
                 "posterior_threshold", "posterior_alpha", "num_beams", "do_sample", "use_cache", "tree_attention",
                 "decoder_input_ids"}
        unknown = sorted(set(kwargs) - known)
        if unknown:
            raise NotImplementedError(f"generate() options not implemented by the H100 engine: {unknown}")

    def generate_from_pcm(self, pcm: Union[np.ndarray, torch.Tensor], language: Optional[str] = None,
                          task: Optional[str] = None, temperature=None, sampling_rate: int = SAMPLE_RATE,
                          **kwargs) -> torch.Tensor:
        """Same as ``generate`` but takes mono f32 PCM and runs the log-mel frontend on the GPU
        (what ``WhisperProcessor`` does on the CPU in the reference's caller, eval_whisper_medusa.py:46-51).
        ``sampling_rate`` other than 16000 (any positive integer rate): the clip is uploaded and resampled to 16 kHz on
        the GPU first (``torchaudio.functional.resample`` with its defaults); the 30 s limit applies after resampling."""
        self._require_engine()
        if _rate(sampling_rate) != SAMPLE_RATE:
            x = torch.as_tensor(pcm).detach().to(torch.float32).reshape(-1)
            if resampled_length(x.numel(), _rate(sampling_rate), SAMPLE_RATE) > MAX_WINDOW_SAMPLES:
                raise NotImplementedError("Longform generation is not supported yet")
            self._check_unsupported(temperature, None, kwargs)
            x16 = self._upload_16k(x, sampling_rate)
            self._encode_window(x16, Window(0, x16.numel(), 0, 0), torch.cuda.current_stream(self._device).cuda_stream)
            return self._decode(language, task, kwargs, temperature)
        x = torch.as_tensor(pcm).detach().to("cpu", torch.float32).contiguous().reshape(-1)
        if x.numel() > 480000:
            raise NotImplementedError("Longform generation is not supported yet")
        lib = _lib.load()
        _check(lib, self._handle,
               lib.wm_encode_pcm(self._handle, C.cast(x.data_ptr(), C.POINTER(C.c_float)), int(x.numel())),
               "wm_encode_pcm")
        self._check_unsupported(temperature, None, kwargs)
        return self._decode(language, task, kwargs, temperature)

    # ------------------------------------------------------------------ long-form (HF chunked ASR pipeline)
    def transcribe(self, audio: Union[np.ndarray, torch.Tensor], sampling_rate: int = SAMPLE_RATE,
                   chunk_length_s: float = 30.0, stride_length_s: Optional[Union[float, Sequence[float]]] = None,
                   language: Optional[str] = None, task: Optional[str] = None, temperature=None,
                   **generate_kwargs) -> torch.Tensor:
        """Transcribe a mono recording of any length at any integer sampling rate; returns ``LongTensor[1, n]``.

        The semantics of HF's ``pipeline("automatic-speech-recognition", chunk_length_s=30)`` without timestamps
        (``longform.py``): the recording is cut into windows of ``chunk_length_s`` (at most 30 s) overlapping by
        ``stride_length_s`` on each side (default ``chunk_length_s / 6``), each window is transcribed like a short clip
        with the same options as ``generate`` (``language=None`` on a multilingual model: each window detects its own
        language), and the windows' text ids (special ids, all ``>= eos_token_id``, dropped) are merged by the
        longest-common-sequence rule.

        ``audio``: 1-D f32 samples as a numpy array, a CPU tensor, or a CUDA tensor on the engine's device (used in place,
        ordered after the current stream).  The recording is uploaded once and, if ``sampling_rate != 16000``, resampled
        once on the GPU.  Every window's log-mel is computed from the device-resident samples.  Per-window results go
        to ``self.last_windows``.  An empty recording has no windows and gives ``[1, 0]``."""
        self._require_engine()
        params = window_params(chunk_length_s, stride_length_s)
        _check_recording(audio, sampling_rate)
        self._check_unsupported(temperature, None, generate_kwargs)
        x16 = self._upload_16k(audio, sampling_rate)
        stream = torch.cuda.current_stream(self._device).cuda_stream
        results = [self._transcribe_window(x16, w, stream, language=language, task=task, temperature=temperature,
                                           **generate_kwargs)
                   for w in plan_windows(x16.numel(), *params)]
        self.last_windows = results
        merged = merge_windows([text_ids(r.ids, int(self.generation_config.eos_token_id)) for r in results])
        return torch.tensor([merged], dtype=torch.long, device=self._device)

    def _upload_16k(self, audio, sampling_rate) -> torch.Tensor:
        """The recording as contiguous f32 16 kHz samples on the engine's device: one upload (none for a CUDA tensor on
        this device) and, at another rate, one resampling kernel on the current stream."""
        lib = _lib.load()
        if isinstance(audio, torch.Tensor) and audio.is_cuda:
            if audio.device != self._device:
                raise EngineError(f"audio is on {audio.device}, the engine on {self._device}")
            x = audio.detach().to(torch.float32).reshape(-1).contiguous()
        else:
            x = torch.as_tensor(audio).detach().to(torch.float32).reshape(-1).contiguous().to(self._device)
        sr = _rate(sampling_rate)
        if sr == SAMPLE_RATE or x.numel() == 0:
            return x
        n_out = resampled_length(x.numel(), sr, SAMPLE_RATE)
        y = torch.empty(n_out, dtype=torch.float32, device=self._device)
        got = C.c_int64(0)
        stream = torch.cuda.current_stream(self._device).cuda_stream
        _check(lib, self._handle,
               lib.wm_resample(self._handle, C.c_void_p(x.data_ptr()), x.numel(), sr, SAMPLE_RATE, C.c_void_p(y.data_ptr()),
                               n_out, C.byref(got), C.c_void_p(stream)), "wm_resample")
        if got.value != n_out:
            raise EngineError(f"wm_resample produced {got.value} samples, expected {n_out}")
        return y

    def _encode_window(self, x16: torch.Tensor, w: Window, producer_stream: int) -> None:
        """Log-mel + encoder of samples ``w.start:w.end`` of a device-resident 16 kHz recording."""
        lib = _lib.load()
        ptr = x16.data_ptr() + w.start * x16.element_size()
        _check(lib, self._handle,
               lib.wm_encode_pcm_device(self._handle, C.c_void_p(ptr), int(w.end - w.start), C.c_void_p(producer_stream)),
               "wm_encode_pcm_device")

    def _transcribe_window(self, x16: torch.Tensor, w: Window, producer_stream: int, language=None, task=None,
                           temperature=None, **kwargs) -> WindowResult:
        self._encode_window(x16, w, producer_stream)
        ids = self._decode(language, task, kwargs, temperature)[0].tolist()
        return WindowResult(w, ids, self.last_trace)

    def _decode(self, language, task, kwargs, temperature, generation_config=None) -> torch.Tensor:
        g = generation_config if generation_config is not None else self.generation_config
        cur = (tuple(g.suppress_tokens or []), tuple(g.begin_suppress_tokens or []))
        if cur != getattr(self, "_pushed", None):
            self._push_suppress()
        explicit = kwargs.pop("decoder_input_ids", None)
        if explicit is not None:
            # an explicit decoder prompt (HF generate(decoder_input_ids=...)); any length up to max_length - K - 2: tokens
            # beyond the 16 rows of a stage tile are cached by prefill launches
            prompt = [int(t) for t in torch.as_tensor(explicit).reshape(-1).tolist()]
        else:
            prompt = self._init_tokens(language, task, g)
        # generate() always runs the loop with temperature 1.0 => typical acceptance (model.py:1878-1881);
        # `medusa_temperature=0` selects the exact-match branch reachable through _medusa_greedy_search.
        t = kwargs.pop("medusa_temperature", 1.0)
        max_length = kwargs.pop("max_length", None)
        if kwargs.get("max_new_tokens") is not None:         # HF: max_length = prompt + max_new_tokens
            max_length = len(prompt) + int(kwargs.pop("max_new_tokens"))
        gp = self._gen_params(len(prompt), kwargs.pop("exponential_decay_length_penalty", None),
                              max_length, t, kwargs.pop("max_iters", 0), g)
        # per-call overrides of the acceptance constants (HF generate(**kwargs) updates the generation config)
        if kwargs.get("posterior_threshold") is not None:
            gp.posterior_threshold = float(kwargs.pop("posterior_threshold"))
        if kwargs.get("posterior_alpha") is not None:
            gp.posterior_alpha = float(kwargs.pop("posterior_alpha"))
        # branching medusa_choices: False (default) = the reference's behaviour (its medusa_attn_mask is built but never
        # applied: verify rows attend causally over cache order); True = every node attends to its ancestors only
        gp.tree_attention = 1 if kwargs.pop("tree_attention", False) else 0
        tr = self._run_loop(prompt, gp)
        self.last_trace = tr
        out = self._strip(tr.sequences, len(prompt), int(gp.pad_token_id), int(gp.eos_token_id))
        return torch.tensor([out], dtype=torch.long, device=self._device)

    # ------------------------------------------------------------------ forward (reference model.py:1223-1347)
    def forward(self, input_features: Optional[torch.Tensor] = None, attention_mask=None,
                decoder_input_ids: Optional[torch.Tensor] = None, decoder_attention_mask=None, head_mask=None,
                decoder_head_mask=None, cross_attn_head_mask=None, encoder_outputs=None, past_key_values=None,
                decoder_inputs_embeds=None, decoder_position_ids=None, labels=None, use_cache=None,
                output_attentions=None, output_hidden_states=None, return_dict=None, disable_medusa: bool = False,
                **kwargs):
        """Teacher-forced pass: ``.logits`` = stacked head logits ``[K+1, 1, T, V]`` (``disable_medusa`` -> ``[1, 1, T,
        V]``), T <= 16 decoder ids from an empty cache.  ``input_features`` (host or device) are encoded first; without
        them the encoder states of the previous ``generate`` / ``forward`` call are reused (the reference's
        ``encoder_outputs`` argument; tensors cannot be injected into the engine)."""
        self._require_engine()
        for name, v in (("labels", labels), ("past_key_values", past_key_values), ("decoder_inputs_embeds", decoder_inputs_embeds),
                        ("decoder_position_ids", decoder_position_ids), ("decoder_attention_mask", decoder_attention_mask)):
            if v is not None:
                raise NotImplementedError(f"forward({name}=...) is not implemented by the inference engine")
        if decoder_input_ids is None:
            raise ValueError("decoder_input_ids is required")
        ids = torch.as_tensor(decoder_input_ids).detach().to("cpu", torch.int32).contiguous()
        assert ids.dim() == 2 and ids.shape[0] == 1, "Batch size should be 1"
        if input_features is not None:
            assert input_features.shape[0] == 1, "Batch size should be 1"
            self._encode_features(input_features)
        n = int(ids.shape[1])
        K1, V = self.config.medusa_num_heads + 1, self.config.vocab_size
        out = torch.empty(K1, 1, n, V, dtype=torch.float32)
        lib = _lib.load()
        _check(lib, self._handle,
               lib.wm_forward(self._handle, C.cast(ids.data_ptr(), C.POINTER(C.c_int32)), n,
                              C.cast(out.data_ptr(), C.POINTER(C.c_float))), "wm_forward")

        return ForwardOutput((out[:1] if disable_medusa else out).to(self._device))

    __call__ = forward

    def state_dict(self) -> Dict[str, torch.Tensor]:
        if self._state_dict is None:
            raise RuntimeError("state dict was released")
        return dict(self._state_dict)

    def parameters(self):
        return iter(self.state_dict().values())

    # ------------------------------------------------------------------ parity taps
    def last_logits(self, which: int) -> torch.Tensor:
        self._require_engine()
        n = (self.config.medusa_num_heads + 1, self.config.vocab_size)
        out = torch.empty(n, dtype=torch.float32)
        lib = _lib.load()
        _check(lib, self._handle, lib.wm_last_logits(self._handle, which, C.cast(out.data_ptr(), C.POINTER(C.c_float))),
               "wm_last_logits")
        return out

    def encoder_output(self) -> torch.Tensor:
        self._require_engine()
        out = torch.empty(self.config.max_source_positions, self.config.d_model, dtype=torch.float32)
        lib = _lib.load()
        _check(lib, self._handle, lib.wm_get_encoder_out(self._handle, C.cast(out.data_ptr(), C.POINTER(C.c_float))),
               "wm_get_encoder_out")
        return out

    def mel(self) -> torch.Tensor:
        self._require_engine()
        out = torch.empty(self.config.num_mel_bins, N_FRAMES, dtype=torch.float32)
        lib = _lib.load()
        _check(lib, self._handle, lib.wm_get_mel(self._handle, C.cast(out.data_ptr(), C.POINTER(C.c_float))), "wm_get_mel")
        return out
