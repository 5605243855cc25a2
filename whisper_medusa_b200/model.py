"""Drop-in host for the reference's decode path: ``WhisperMedusaModel.from_pretrained / .to /
.generate`` (reference ``whisper_medusa/models/model.py:213``, re-exported at
``whisper_medusa/__init__.py:1``) over the C ABI in ``include/whisper_medusa_b200.h``.

Same names, argument meaning and error behaviour as the reference for this path:

* ``generate`` asserts batch size 1 (``model.py:1451``);
* ``return_timestamps`` -> ``NotImplementedError`` (``:1171-1174``); ``no_speech_threshold`` ->
  ``NotImplementedError`` (``:1201-1204``); more than 3000 feature frames (long-form) ->
  ``NotImplementedError`` (``:1213-1214``); beam search -> ``Exception`` (``:1153-1156``);
* the returned ``LongTensor[1, n]`` has the prompt and the trailing EOS stripped (``:1929-1973``);
* ``return_dict_in_generate=True`` with ``output_scores`` / ``output_logits`` returns the per-iteration processed rows the
  reference collects (``:737-742``) in a ``MedusaGenerateOutput``, with per-token log-probabilities added (computed on the
  GPU, ``csrc/scores.cu``).

Beyond the reference (which takes 16 kHz clips of at most 30 s): ``transcribe`` takes a recording of any length at any
integer sampling rate, with the semantics of HF's chunked ASR pipeline (``longform.py``); ``generate_from_pcm`` takes
``sampling_rate``.  Both resample on the GPU (``csrc/resample.cu``).

There is no PyTorch / CPU fallback: every tensor op of the path runs in the CUDA engine, and the
constructor raises if the engine library is missing.
"""
from __future__ import annotations

import ctypes as C
import os
import warnings
from typing import Dict, List, Optional, Sequence, Tuple, Union

import numpy as np
import torch

from . import _lib
from .config import MedusaConfig, MedusaGenerationConfig
from .longform import (MAX_WINDOW_SAMPLES, SAMPLE_RATE, Fallback, Window, WindowResult, compression_ratio,
                       fallback_rule, merge_timed, merge_windows, needs_fallback, no_speech_rule, plan_windows,
                       resampled_length, skip_window, window_params)
from . import processors as _processors
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


class MedusaGenerateOutput:
    """What ``generate(..., return_dict_in_generate=True)`` returns (the reference returns a
    ``GenerateEncoderDecoderOutput``, ``model.py:812-824``).

    * ``sequences``: ``LongTensor[1, n]``, exactly what the call returns without ``return_dict_in_generate``;
    * ``scores`` (``output_scores=True``, else ``None``): one ``FloatTensor[1, V]`` per speculative iteration, the
      processed verify row of the accepted path's last node (the reference's ``next_token_logits``, whose own shape is
      ``[1, 1, V]``); suppressed ids are ``-inf``;
    * ``logits`` (``output_logits=True``, else ``None``): the same rows (the reference appends the same processed tensor
      to both tuples, ``model.py:739-742``);
    * ``token_logprobs``: ``FloatTensor[1, n_new_tokens]``, the log-probability (log_softmax at temperature 1 of the
      processed row) of every generated token up to and including the first EOS, under the row it was chosen from;
    * ``avg_logprob``: their mean (a float);
    * ``accept_lengths``: the accept length of every iteration;
    * ``no_speech_prob`` (``output_no_speech_prob=True``, else ``None``): the probability of ``<|nospeech|>``
      (``no_timestamps_token_id - 1``) in the softmax of the raw base-head logits at the start-of-transcript position
      (HF ``WhisperNoSpeechDetection``), computed on the GPU (``csrc/no_speech.cu``); a float;
    * ``token_timestamps`` (``return_token_timestamps=True``, else ``None``): ``FloatTensor[1, n]``, the time in seconds
      of every id of ``sequences[0]`` (HF ``_extract_token_timestamps``: DTW over the alignment heads' cross-attention),
      computed on the GPU (``csrc/timestamps.cu``).  Without ``return_dict_in_generate`` it is the only field besides
      ``sequences``.  From ``transcribe(..., return_token_timestamps=True)`` it is ``FloatTensor[1, n, 2]``, the
      ``(start, end)`` of every id in seconds of the recording, and the only field besides ``sequences``.

    Fields are attributes and keys (``out.scores`` / ``out["scores"]``); an integer indexes the fields that are not
    ``None``, in the order above, as HF ``ModelOutput`` does."""

    FIELDS = ("sequences", "scores", "logits", "token_logprobs", "avg_logprob", "accept_lengths", "no_speech_prob",
              "token_timestamps")

    def __init__(self, sequences, scores, logits, token_logprobs, avg_logprob, accept_lengths, no_speech_prob=None,
                 token_timestamps=None):
        self.sequences = sequences
        self.scores = scores
        self.logits = logits
        self.token_logprobs = token_logprobs
        self.avg_logprob = avg_logprob
        self.accept_lengths = accept_lengths
        self.no_speech_prob = no_speech_prob
        self.token_timestamps = token_timestamps

    def keys(self) -> List[str]:
        return [k for k in self.FIELDS if getattr(self, k) is not None]

    def to_tuple(self) -> tuple:
        return tuple(getattr(self, k) for k in self.keys())

    def __getitem__(self, i):
        if isinstance(i, str):
            if i not in self.FIELDS:
                raise KeyError(i)
            return getattr(self, i)
        return self.to_tuple()[i]


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
            medusa_num_heads=c.medusa_num_heads, medusa_block=1 if c.is_block else 0,
            medusa_num_layers=c.medusa_num_layers)

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
                 return_dict_in_generate=None, **kwargs) -> Union[torch.Tensor, MedusaGenerateOutput]:
        """Transcribe one <= 30 s clip given its log-mel features ``[1, 80, 3000]``
        (reference ``model.py:1419-1779``); returns ``LongTensor[1, n]``, or with ``return_dict_in_generate=True`` a
        ``MedusaGenerateOutput`` (``output_scores`` / ``output_logits`` / ``output_no_speech_prob`` select its
        ``scores`` / ``logits`` / ``no_speech_prob``; without ``return_dict_in_generate`` they have no effect, as in HF
        and the reference).  ``no_speech_threshold`` raises as in the reference: the skip rule is ``transcribe``'s.

        ``return_token_timestamps=True``: token-level timestamps as HF computes them (``_extract_token_timestamps`` with
        the generation config's ``alignment_heads``, ``config.median_filter_width`` and ``time_precision``), in
        ``token_timestamps`` of a ``MedusaGenerateOutput`` (the only other field is ``sequences`` unless
        ``return_dict_in_generate``).  ``attention_mask`` (the feature extractor's, ``[1, 3000]``) crops the alignment to
        the clip's frames.  Chains of ``medusa_choices`` only."""
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
        self._logits_processors(kwargs, generation_config)
        num_frames = self._mask_frames(attention_mask) if attention_mask is not None else None
        ts = self._timestamp_request(generation_config, task, num_frames, time_precision) if return_token_timestamps else None
        self._encode_features(input_features)
        return self._decode(language, task, kwargs, temperature, generation_config, return_dict_in_generate,
                            **({"token_timestamps": ts} if ts else {}))

    @staticmethod
    def _mask_frames(attention_mask) -> int:
        """Frame count of the clip (HF ``attention_mask.sum(-1)``) from a one-row feature-extractor mask, ``[1, 3000]``
        or ``[3000]``.  A mask of several rows belongs to a batch: ``generate`` takes one clip, so it raises rather than
        crop this clip by another row (``StreamGroup.generate`` hands each row its own mask)."""
        mask = torch.as_tensor(attention_mask)
        if mask.dim() == 2 and mask.shape[0] == 1:
            mask = mask[0]
        if mask.dim() != 1 or mask.shape[0] != N_FRAMES:
            raise ValueError(f"attention_mask must be one clip's mask, [1, {N_FRAMES}] or [{N_FRAMES}], got shape "
                             f"{tuple(torch.as_tensor(attention_mask).shape)} (for a batch, use StreamGroup.generate)")
        return int(mask.sum())

    @staticmethod
    def pcm_num_frames(n_samples: int) -> int:
        """Feature frames of a clip of ``n_samples`` 16 kHz samples: the ``attention_mask.sum(-1)`` of
        ``WhisperFeatureExtractor(..., return_attention_mask=True)`` (one frame per started hop of 160 samples)."""
        return min(N_FRAMES, (int(n_samples) + 159) // 160)

    def _timestamp_request(self, generation_config, task, num_frames: Optional[int],
                           time_precision: float) -> Tuple[Optional[int], float]:
        """Checks of ``return_token_timestamps=True`` before any GPU work (HF ``_set_num_frames`` / ``_median_filter``);
        returns ``(num_frames, time_precision)`` for ``_decode``."""
        g = generation_config if generation_config is not None else self.generation_config
        if (task or getattr(g, "task", None)) == "translate":
            warnings.warn("Token-level timestamps may not be reliable for task 'translate'.")
        heads = getattr(g, "alignment_heads", None)
        if heads is None:
            raise ValueError(
                "Model generation config has no `alignment_heads`, token-level timestamps not available. "
                "See https://gist.github.com/hollance/42e32852f24243b748ae6bc1f985b13a on how to add this property to the generation config.")
        for pair in heads:
            l, h = (int(v) for v in pair)
            if not (0 <= l < self.config.decoder_layers and 0 <= h < self.config.decoder_attention_heads):
                raise ValueError(f"alignment head {[l, h]} is out of range: {self.config.decoder_layers} decoder layers of "
                                 f"{self.config.decoder_attention_heads} heads")
        width = int(getattr(self.config, "median_filter_width", 7))
        if width <= 0 or width % 2 != 1:
            raise ValueError("`filter_width` should be an odd number")
        if any(int(c) != 1 for c in self.config.medusa_choices):
            raise NotImplementedError("return_token_timestamps needs a chain of medusa_choices (all 1): the verify rows of "
                                      "a branching tree are not the rows of one decoded sequence")
        return num_frames, float(time_precision)

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
                 "decoder_input_ids", "output_scores", "output_logits", "output_no_speech_prob", *_processors.KEYS}
        unknown = sorted(set(kwargs) - known)
        if unknown:
            raise NotImplementedError(f"generate() options not implemented by the H100 engine: {unknown}")

    def _logits_processors(self, kwargs, generation_config=None,
                           prompt: Optional[Sequence[int]] = None) -> Optional[_processors.Processors]:
        """The call's ``sequence_bias`` / ``bad_words_ids`` / ``no_repeat_ngram_size`` / ``min_length`` /
        ``min_new_tokens`` (kwargs, else the generation config's attributes), checked, as engine tables; None = off.
        Without ``prompt`` (checks before any GPU work) the prompt length is the one ``_decode`` will use."""
        g = generation_config if generation_config is not None else self.generation_config
        if prompt is not None:
            n_prompt = len(prompt)
        elif kwargs.get("decoder_input_ids") is not None:
            n_prompt = int(torch.as_tensor(kwargs["decoder_input_ids"]).numel())
        else:
            n_prompt = 4 if g.is_multilingual else 2      # _init_tokens
        max_length = kwargs.get("max_length") if kwargs.get("max_length") is not None else g.max_length
        if kwargs.get("max_new_tokens") is not None:
            max_length = n_prompt + int(kwargs["max_new_tokens"])
        pen = kwargs.get("exponential_decay_length_penalty")
        pen = pen if pen is not None else g.exponential_decay_length_penalty
        return _processors.build(_processors.options(kwargs, g), int(g.eos_token_id), int(self.config.vocab_size),
                                 n_prompt, int(max_length), pen)

    def _push_logits_processors(self, procs: Optional[_processors.Processors]) -> None:
        """Sent on every call that has processors, and switched off again on the engine that last had them, so a call
        without processors launches nothing extra."""
        if procs is None and getattr(self, "_lp_engine", None) != self._handle.value:
            return
        lib = _lib.load()
        seqs = procs.seqs if procs is not None else []
        toks = [t for ids, _ in seqs for t in ids]
        offs = [0]
        for ids, _ in seqs:
            offs.append(offs[-1] + len(ids))
        _check(lib, self._handle,
               lib.wm_set_logits_processors(self._handle, (C.c_int32 * max(1, len(toks)))(*toks),
                                            (C.c_int32 * len(offs))(*offs),
                                            (C.c_float * max(1, len(seqs)))(*[v for _, v in seqs]), len(seqs),
                                            procs.ngram if procs is not None else 0,
                                            procs.eos_min_length if procs is not None else 0),
               "wm_set_logits_processors")
        self._lp_engine = self._handle.value if procs is not None else None

    def generate_from_pcm(self, pcm: Union[np.ndarray, torch.Tensor], language: Optional[str] = None,
                          task: Optional[str] = None, temperature=None, sampling_rate: int = SAMPLE_RATE,
                          return_dict_in_generate=None, return_token_timestamps=None, time_precision: float = 0.02,
                          **kwargs) -> Union[torch.Tensor, MedusaGenerateOutput]:
        """Same as ``generate`` but takes mono f32 PCM and runs the log-mel frontend on the GPU
        (what ``WhisperProcessor`` does on the CPU in the reference's caller, eval_whisper_medusa.py:46-51).
        ``sampling_rate`` other than 16000 (any positive integer rate): the clip is uploaded and resampled to 16 kHz on
        the GPU first (``torchaudio.functional.resample`` with its defaults); the 30 s limit applies after resampling.
        ``return_token_timestamps`` as in ``generate``, with the clip's frame count (after resampling) as the attention
        mask's."""
        self._require_engine()
        self._logits_processors(kwargs)
        n16 = (int(torch.as_tensor(pcm).numel()) if _rate(sampling_rate) == SAMPLE_RATE
               else resampled_length(int(torch.as_tensor(pcm).numel()), _rate(sampling_rate), SAMPLE_RATE))
        ts = (self._timestamp_request(None, task, self.pcm_num_frames(n16), time_precision)
              if return_token_timestamps else None)
        if _rate(sampling_rate) != SAMPLE_RATE:
            x = torch.as_tensor(pcm).detach().to(torch.float32).reshape(-1)
            if resampled_length(x.numel(), _rate(sampling_rate), SAMPLE_RATE) > MAX_WINDOW_SAMPLES:
                raise NotImplementedError("Longform generation is not supported yet")
            self._check_unsupported(temperature, None, kwargs)
            x16 = self._upload_16k(x, sampling_rate)
            self._encode_window(x16, Window(0, x16.numel(), 0, 0), torch.cuda.current_stream(self._device).cuda_stream)
            return self._decode(language, task, kwargs, temperature, return_dict_in_generate=return_dict_in_generate,
                                **({"token_timestamps": ts} if ts else {}))
        x = torch.as_tensor(pcm).detach().to("cpu", torch.float32).contiguous().reshape(-1)
        if x.numel() > 480000:
            raise NotImplementedError("Longform generation is not supported yet")
        lib = _lib.load()
        _check(lib, self._handle,
               lib.wm_encode_pcm(self._handle, C.cast(x.data_ptr(), C.POINTER(C.c_float)), int(x.numel())),
               "wm_encode_pcm")
        self._check_unsupported(temperature, None, kwargs)
        return self._decode(language, task, kwargs, temperature, return_dict_in_generate=return_dict_in_generate,
                            **({"token_timestamps": ts} if ts else {}))

    # ------------------------------------------------------------------ long-form (HF chunked ASR pipeline)
    def transcribe(self, audio: Union[np.ndarray, torch.Tensor], sampling_rate: int = SAMPLE_RATE,
                   chunk_length_s: float = 30.0, stride_length_s: Optional[Union[float, Sequence[float]]] = None,
                   language: Optional[str] = None, task: Optional[str] = None, temperature=None,
                   no_speech_threshold: Optional[float] = None, logprob_threshold: Optional[float] = None,
                   return_token_timestamps: Optional[bool] = None, time_precision: float = 0.02,
                   compression_ratio_threshold: Optional[float] = None, top_k: Optional[int] = None,
                   **generate_kwargs) -> Union[torch.Tensor, MedusaGenerateOutput]:
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
        to ``self.last_windows``.  An empty recording has no windows and gives ``[1, 0]``.

        ``no_speech_threshold`` with ``logprob_threshold``: HF's no-speech rule.  A window is skipped -- it adds no ids to
        the merge -- when the probability of ``<|nospeech|>`` at its start-of-transcript position is above
        ``no_speech_threshold`` and the average log-probability of its tokens is below ``logprob_threshold``.  Each
        window is still decoded in full (the rule needs its average log-probability).  ``no_speech_threshold`` alone
        raises ``ValueError``; ``logprob_threshold`` alone without a temperature schedule ``NotImplementedError``.

        ``return_token_timestamps=True``: a ``MedusaGenerateOutput`` whose ``sequences`` (``LongTensor[1, n]``) and
        ``token_timestamps`` (``FloatTensor[1, n, 2]``, the ``(start, end)`` of every id in seconds of the recording) are
        what HF's pipeline gives with ``return_timestamps="word"`` for windows without timestamp tokens
        (``_decode_asr``).  Each window is decoded as ``generate_from_pcm(window, return_token_timestamps=True,
        time_precision=...)`` would decode it, cropped to its own frames; its times are moved by the window's offset and
        the windows are merged by HF's timed rule, which matches overlapping ids only when their times are in order.
        The merged ids can therefore differ from those of the call without timestamps.  ``last_windows[i]`` holds each
        window's ``token_timestamps`` (relative to the window) and ``num_frames``.  The checks of ``generate``'s flag
        (``alignment_heads``, filter width, a chain of ``medusa_choices``) run before anything is uploaded.

        Temperature fallback (HF ``generate_with_fallback``): ``temperature`` a schedule such as ``(0.0, 0.2, 0.4, 0.6,
        0.8, 1.0)`` whose first entry is 0.0, with ``compression_ratio_threshold`` and / or ``logprob_threshold``.  Each
        window is first decoded as without the schedule; while its result has a compression ratio (HF's, over the
        generated ids and the EOS) above ``compression_ratio_threshold`` or an average log-probability below
        ``logprob_threshold``, it is decoded again from the same encoder output and prompt by sampling at the next
        temperature, from the processed rows' top ``top_k`` entries (default: the generation config's, else 50; 0 = all;
        at most 64).  The first attempt that passes is kept, else the last.  With ``no_speech_threshold`` the no-speech
        rule skips a window instead and ends its attempts.  Sampling is reproducible under ``torch.manual_seed``: one
        64-bit seed per recording is drawn from torch's default generator when a fallback is possible, and each
        attempt's noise depends on (seed, window, attempt) only.  ``last_windows[i]`` records ``temperature``,
        ``compression_ratio``, ``avg_logprob`` and ``attempts``.  Chains of ``medusa_choices`` only.  A one-entry schedule
        takes the thresholds and never falls back (HF); ``top_k`` without a fallback raises ``NotImplementedError``."""
        self._require_engine()
        params = window_params(chunk_length_s, stride_length_s)
        _check_recording(audio, sampling_rate)
        fallback, no_speech, temperature = self._fallback_request(temperature, compression_ratio_threshold,
                                                                  logprob_threshold, no_speech_threshold, top_k)
        self._check_unsupported(temperature, None, generate_kwargs)
        self._logits_processors(generate_kwargs)
        if return_token_timestamps:
            self._timestamp_request(None, task, None, time_precision)
            generate_kwargs["time_precision"] = float(time_precision)
        seed = self._recording_seed() if fallback is not None else None
        x16 = self._upload_16k(audio, sampling_rate)
        stream = torch.cuda.current_stream(self._device).cuda_stream
        fb = {} if fallback is None else {"fallback": fallback}
        results = [self._transcribe_window(x16, w, stream, language=language, task=task, temperature=temperature,
                                           no_speech=no_speech, **({"seed": (seed, i)} if fb else {}), **fb,
                                           **generate_kwargs)
                   for i, w in enumerate(plan_windows(x16.numel(), *params))]
        self.last_windows = results
        return self._merge_results(results, bool(return_token_timestamps))

    def _fallback_request(self, temperature, compression_ratio_threshold, logprob_threshold, no_speech_threshold, top_k):
        """Checks of ``transcribe``'s temperature-fallback and no-speech arguments before any GPU work: ``(fallback or
        None, (no_speech_threshold, logprob_threshold) or None, the temperature left for the sampling refusal)``."""
        fallback = fallback_rule(temperature, compression_ratio_threshold, logprob_threshold, top_k,
                                 int(self.config.vocab_size), getattr(self.generation_config, "top_k", None))
        if fallback is not None and any(int(c) != 1 for c in self.config.medusa_choices):
            raise NotImplementedError("temperature fallback needs a chain of medusa_choices (all 1): sampled attempts "
                                      "do not run on a branching tree")
        # with a schedule, logprob_threshold without no_speech_threshold is a fallback threshold (a one-entry schedule
        # has nothing to fall back to, as in HF); without one the rule refuses it as before
        schedule = isinstance(temperature, (tuple, list))
        lpt_rule = None if (schedule and no_speech_threshold is None) else logprob_threshold
        no_speech = ((float(no_speech_threshold), float(logprob_threshold))
                     if no_speech_rule(no_speech_threshold, lpt_rule) else None)
        return fallback, no_speech, (None if isinstance(temperature, (tuple, list)) else temperature)

    @staticmethod
    def _recording_seed() -> Tuple[int, int]:
        """One 64-bit seed of a recording's sampled attempts, as two 32-bit words, from torch's default generator."""
        w = torch.randint(0, 2 ** 32, (2,), dtype=torch.int64)
        return int(w[0]), int(w[1])

    def _merge_results(self, results: List[WindowResult], timed: bool) -> Union[torch.Tensor, MedusaGenerateOutput]:
        """The windows' merge: ``LongTensor[1, n]``, or with token timestamps the output of ``transcribe``."""
        eos = int(self.generation_config.eos_token_id)
        if not timed:
            merged = merge_windows([r.merge_ids(eos) for r in results])
            return torch.tensor([merged], dtype=torch.long, device=self._device)
        ids, pairs = merge_timed(results, eos)
        return MedusaGenerateOutput(torch.tensor([ids], dtype=torch.long, device=self._device), None, None, None, None,
                                    None, token_timestamps=torch.tensor(pairs, dtype=torch.float32).reshape(1, -1, 2)
                                    .to(self._device))

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
                           temperature=None, no_speech: Optional[Tuple[float, float]] = None,
                           time_precision: Optional[float] = None, fallback: Optional[Fallback] = None,
                           seed: Optional[Tuple[Tuple[int, int], int]] = None, **kwargs) -> WindowResult:
        """One window; ``no_speech`` = (no_speech_threshold, logprob_threshold) or None (the rule off);
        ``time_precision`` = token timestamps with that precision, cropped to the window's frames, or None (off);
        ``fallback`` with ``seed`` = ((seed words of the recording), window index): temperature fallback, or None."""
        self._encode_window(x16, w, producer_stream)
        num_frames = None if time_precision is None else self.pcm_num_frames(w.end - w.start)
        ts = {} if time_precision is None else {"token_timestamps": (num_frames, float(time_precision))}
        if fallback is not None:
            return self._fallback_window(w, language, task, kwargs, no_speech, ts, num_frames, fallback, *seed)
        if no_speech is None:
            out = self._decode(language, task, kwargs, temperature, **ts)
            if not ts:
                return WindowResult(w, out[0].tolist(), self.last_trace)
            return WindowResult(w, out.sequences[0].tolist(), self.last_trace, token_timestamps=out.token_timestamps,
                                num_frames=num_frames)
        out = self._decode(language, task, dict(kwargs, output_no_speech_prob=True), temperature,
                           return_dict_in_generate=True, **ts)
        return WindowResult(w, out.sequences[0].tolist(), self.last_trace, no_speech_prob=out.no_speech_prob,
                            avg_logprob=out.avg_logprob,
                            skipped=skip_window(out.no_speech_prob, out.avg_logprob, *no_speech),
                            token_timestamps=out.token_timestamps, num_frames=num_frames)

    def _fallback_window(self, w: Window, language, task, kwargs, no_speech, ts, num_frames, fb: Fallback,
                         seed: Tuple[int, int], window_index: int) -> WindowResult:
        """HF ``generate_with_fallback`` for one window whose encoder output is in place: attempts in schedule order
        from the same prompt (the first one's: language detection runs once), until one does not need fallback or the
        no-speech rule skips the window; the last attempt is kept when every one needs fallback."""
        explicit = kwargs.pop("decoder_input_ids", None)
        prompt = ([int(v) for v in torch.as_tensor(explicit).reshape(-1).tolist()] if explicit is not None
                  else self._init_tokens(language, task))
        attempts: List[Tuple[float, float, float]] = []
        for a, t in enumerate(fb.temperatures):
            kw = dict(kwargs, output_no_speech_prob=no_speech is not None, decoder_input_ids=prompt)
            sampling = (t, fb.top_k, seed[0], seed[1], window_index, a) if t > 0 else None
            if sampling is not None:
                kw["medusa_temperature"] = 0.0       # exact-match acceptance against the sampled choices
            out = self._decode(language, task, kw, None, return_dict_in_generate=True, sampling=sampling, **ts)
            tr = self.last_trace
            # HF's seek_sequence: the generated ids, up to and including the first EOS
            ratio = compression_ratio(tr.sequences[len(prompt):len(prompt) + tr.n_new_tokens], int(self.config.vocab_size))
            attempts.append((float(t), ratio, float(out.avg_logprob)))
            skipped = no_speech is not None and skip_window(out.no_speech_prob, out.avg_logprob, *no_speech)
            if skipped or not needs_fallback(ratio, out.avg_logprob, fb):
                break
        return WindowResult(w, out.sequences[0].tolist(), tr, no_speech_prob=out.no_speech_prob,
                            avg_logprob=out.avg_logprob, skipped=skipped if no_speech is not None else None,
                            token_timestamps=out.token_timestamps, num_frames=num_frames, temperature=float(t),
                            compression_ratio=ratio, attempts=attempts)

    def _push_sampling(self, sampling: Optional[Tuple[float, int, int, int, int, int]]) -> None:
        """A sampled attempt's ``(temperature, top_k, seed_lo, seed_hi, window, attempt)``: sent on every sampled call
        and switched off again on the engine that last had it, so other calls launch and draw nothing extra."""
        if sampling is None and getattr(self, "_smp_engine", None) != self._handle.value:
            return
        lib = _lib.load()
        t, k, lo, hi, win, att = sampling if sampling is not None else (0.0, 0, 0, 0, 0, 0)
        _check(lib, self._handle, lib.wm_set_sampling(self._handle, float(t), int(k), lo, hi, win, att), "wm_set_sampling")
        self._smp_engine = self._handle.value if sampling is not None else None

    def _decode(self, language, task, kwargs, temperature, generation_config=None, return_dict_in_generate=None,
                token_timestamps: Optional[Tuple[Optional[int], float]] = None,
                sampling: Optional[Tuple[float, int, int, int, int, int]] = None) -> Union[torch.Tensor, MedusaGenerateOutput]:
        """``token_timestamps``: ``(num_frames or None, time_precision)`` from ``_timestamp_request``, or None;
        ``sampling``: a sampled attempt of temperature fallback (``_push_sampling``), or None."""
        g = generation_config if generation_config is not None else self.generation_config
        output_scores = bool(kwargs.pop("output_scores", False))
        output_logits = bool(kwargs.pop("output_logits", False))
        as_dict = bool(return_dict_in_generate)
        want_ns = as_dict and bool(kwargs.pop("output_no_speech_prob", False))
        kwargs.pop("output_no_speech_prob", None)
        # engine option "scores" for this call: bit 0 = per-token log-probabilities (every dict result), bit 1 = the
        # scores rows.  0 without return_dict_in_generate: the loop then launches nothing extra.
        score_bits = (1 | (2 if output_scores or output_logits else 0)) if as_dict else 0
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
        procs = self._logits_processors(kwargs, g, prompt)
        for k in _processors.KEYS:
            kwargs.pop(k, None)
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
        lib = _lib.load()
        _check(lib, self._handle, lib.wm_set_option(self._handle, b"scores", score_bits), "wm_set_option(scores)")
        # engine option "no_speech_row" for this call (set on every call, like "scores": a host-side store, and a new
        # engine after to() / close() starts with it off)
        ns_row = self._no_speech_row(prompt, g) if want_ns else -1
        _check(lib, self._handle, lib.wm_set_option(self._handle, b"no_speech_row", ns_row), "wm_set_option(no_speech_row)")
        # alignment heads captured by this call's loop: sent on every call that asks for timestamps (a new engine after
        # to() / close() starts with capture off), and switched off again on the engine that last had them
        if token_timestamps is not None or getattr(self, "_ts_engine", None) == self._handle.value:
            pairs = [int(v) for p in g.alignment_heads for v in p] if token_timestamps is not None else []
            arr = (C.c_int32 * max(1, len(pairs)))(*pairs)
            _check(lib, self._handle, lib.wm_set_alignment_heads(self._handle, arr, len(pairs) // 2),
                   "wm_set_alignment_heads")
            self._ts_engine = self._handle.value if pairs else None
        self._push_logits_processors(procs)
        self._push_sampling(sampling)
        tr = self._run_loop(prompt, gp)
        self.last_trace = tr
        self._last_medusa_temperature = float(gp.temperature)
        out = self._strip(tr.sequences, len(prompt), int(gp.pad_token_id), int(gp.eos_token_id))
        sequences = torch.tensor([out], dtype=torch.long, device=self._device)
        stamps = self._token_timestamps(tr, len(prompt), len(out), *token_timestamps) if token_timestamps else None
        if not as_dict:
            if stamps is not None:     # the reference's {"sequences", "token_timestamps"} (model.py:1764-1769)
                return MedusaGenerateOutput(sequences, None, None, None, None, None, token_timestamps=stamps)
            return sequences
        out = self._generate_output(sequences, tr, output_scores, output_logits)
        out.token_timestamps = stamps
        if want_ns:
            prob = C.c_float(0.0)
            token = int(g.no_timestamps_token_id) - 1      # HF's choice (generation_whisper.py _setup_no_speech_detection)
            _check(lib, self._handle, lib.wm_last_no_speech(self._handle, token, C.byref(prob), None), "wm_last_no_speech")
            out.no_speech_prob = float(prob.value)
        return out

    def _token_timestamps(self, tr: GenerateTrace, n_prompt: int, n_ids: int, num_frames: Optional[int],
                          time_precision: float) -> torch.Tensor:
        """HF's timestamps of the sequence up to and including its first EOS (``wm_token_timestamps``), cut to the
        ``n_ids`` ids ``generate`` returns (the prompt and the trailing EOS stripped)."""
        lib = _lib.load()
        n_total = n_prompt + tr.n_new_tokens
        buf = torch.zeros(max(1, n_total), dtype=torch.float32)
        _check(lib, self._handle,
               lib.wm_token_timestamps(self._handle, n_prompt, n_total, -1 if num_frames is None else int(num_frames),
                                       int(getattr(self.config, "median_filter_width", 7)), float(time_precision),
                                       C.cast(buf.data_ptr(), C.POINTER(C.c_float)), None, None), "wm_token_timestamps")
        if n_ids > tr.n_new_tokens:
            raise EngineError(f"{n_ids} ids returned for {tr.n_new_tokens} decoded tokens")
        return buf[n_prompt : n_prompt + n_ids][None].to(self._device)

    def last_alignment_probs(self, row0: int, n_rows: int) -> torch.Tensor:
        """Cross-attention probabilities the last ``generate(..., return_token_timestamps=True)`` captured at positions
        ``row0 .. row0 + n_rows - 1``: ``[alignment pairs, n_rows, 1500]`` (``wm_last_alignment_probs``)."""
        self._require_engine()
        lib = _lib.load()
        n_pairs = C.c_int32(0)     # the pairs the engine captured with (the config may have changed since)
        _check(lib, self._handle, lib.wm_last_alignment_probs(self._handle, 0, 0, None, 0, C.byref(n_pairs)),
               "wm_last_alignment_probs")
        out = torch.empty(n_pairs.value, int(n_rows), self.config.max_source_positions, dtype=torch.float32)
        _check(lib, self._handle, lib.wm_last_alignment_probs(self._handle, int(row0), int(n_rows),
                                                              C.cast(out.data_ptr(), C.POINTER(C.c_float)), out.numel(),
                                                              None), "wm_last_alignment_probs")
        return out

    def timestamps_from_probs(self, probs: torch.Tensor, n_prompt: int, num_frames: Optional[int] = None,
                              time_precision: float = 0.02, filter_width: Optional[int] = None):
        """The extraction kernels on given probability rows ``probs [heads, N, W]`` (``wm_token_timestamps_from_probs``):
        returns ``(timestamps [n_prompt + N + 1], matrix [N, F], jumps [N])``."""
        self._require_engine()
        lib = _lib.load()
        p = torch.as_tensor(probs, dtype=torch.float32).detach().cpu().contiguous()
        nh, n, w = (int(v) for v in p.shape)
        f = w if num_frames is None else min(w, int(num_frames) // 2)
        ts = torch.zeros(n_prompt + n + 1, dtype=torch.float32)
        mat = torch.zeros(max(1, n * f), dtype=torch.float32)
        jumps = torch.zeros(max(1, n), dtype=torch.int32)
        width = int(filter_width if filter_width is not None else getattr(self.config, "median_filter_width", 7))
        _check(lib, self._handle,
               lib.wm_token_timestamps_from_probs(self._handle, C.cast(p.data_ptr(), C.POINTER(C.c_float)), nh, n, w,
                                                  int(n_prompt), -1 if num_frames is None else int(num_frames), width,
                                                  float(time_precision), C.cast(ts.data_ptr(), C.POINTER(C.c_float)),
                                                  C.cast(mat.data_ptr(), C.POINTER(C.c_float)),
                                                  C.cast(jumps.data_ptr(), C.POINTER(C.c_int32))),
               "wm_token_timestamps_from_probs")
        return ts, mat[: n * f].reshape(n, f), jumps[:n]

    def last_timestamp_matrix(self, n_prompt: int, n_total: int, num_frames: Optional[int] = None,
                              time_precision: float = 0.02):
        """``(timestamps [n_total], matrix [N, F], jumps [N])`` of the last captured ``generate`` for its first
        ``n_total`` ids (``wm_token_timestamps``), N = n_total - 1 - n_prompt."""
        self._require_engine()
        lib = _lib.load()
        n = max(0, n_total - 1 - n_prompt)
        f = self.config.max_source_positions if num_frames is None else min(self.config.max_source_positions,
                                                                             int(num_frames) // 2)
        ts = torch.zeros(max(1, n_total), dtype=torch.float32)
        mat = torch.zeros(max(1, n * f), dtype=torch.float32)
        jumps = torch.zeros(max(1, n), dtype=torch.int32)
        _check(lib, self._handle,
               lib.wm_token_timestamps(self._handle, int(n_prompt), int(n_total), -1 if num_frames is None else int(num_frames),
                                       int(getattr(self.config, "median_filter_width", 7)), float(time_precision),
                                       C.cast(ts.data_ptr(), C.POINTER(C.c_float)), C.cast(mat.data_ptr(), C.POINTER(C.c_float)),
                                       C.cast(jumps.data_ptr(), C.POINTER(C.c_int32))), "wm_token_timestamps")
        return ts[:n_total], mat[: n * f].reshape(n, f), jumps[:n]

    def _no_speech_row(self, prompt: Sequence[int], g) -> int:
        """Index in the prompt of the start-of-transcript token, whose raw base-head row gives the no-speech
        probability.  It must be among the rows the first iteration computes: the last ((n - 1) % 16) + 1 rows of a
        prompt of n tokens (the leading 16-token chunks of a longer prompt are cached by prefill launches)."""
        sot = int(g.decoder_start_token_id)
        if getattr(g, "no_timestamps_token_id", None) is None:
            raise ValueError("output_no_speech_prob needs the generation config's no_timestamps_token_id")
        if sot not in prompt:
            raise ValueError(f"output_no_speech_prob: the prompt has no start-of-transcript token ({sot})")
        row = list(prompt).index(sot)
        if row < (len(prompt) - 1) // 16 * 16:
            raise NotImplementedError("output_no_speech_prob: the start-of-transcript token of a prompt longer than 16 "
                                      "tokens must be among its last ((len - 1) % 16) + 1 tokens")
        return row

    def _generate_output(self, sequences: torch.Tensor, tr: GenerateTrace, output_scores: bool,
                         output_logits: bool) -> MedusaGenerateOutput:
        """Read back what the scoring kernel recorded during the last loop (``wm_last_scores``)."""
        lib = _lib.load()
        n_tok, n_rows = C.c_int32(0), C.c_int32(0)
        cap = max(1, len(tr.sequences))
        lp = torch.empty(cap, dtype=torch.float32)
        want_rows = output_scores or output_logits
        V = self.config.vocab_size
        rows = torch.empty((max(1, tr.iterations) if want_rows else 1), V, dtype=torch.float32)
        _check(lib, self._handle,
               lib.wm_last_scores(self._handle, C.cast(lp.data_ptr(), C.POINTER(C.c_float)), cap, C.byref(n_tok),
                                  C.cast(rows.data_ptr(), C.POINTER(C.c_float)) if want_rows else None,
                                  rows.shape[0], C.byref(n_rows) if want_rows else None), "wm_last_scores")
        if n_tok.value < tr.n_new_tokens:
            raise EngineError(f"wm_last_scores returned {n_tok.value} log-probabilities for {tr.n_new_tokens} tokens")
        token_logprobs = lp[: tr.n_new_tokens]
        avg = float(token_logprobs.double().mean())
        rows_t = None
        if want_rows:
            if n_rows.value != tr.iterations:
                raise EngineError(f"wm_last_scores returned {n_rows.value} rows for {tr.iterations} iterations")
            dev = rows[: tr.iterations].to(self._device)
            rows_t = tuple(dev[i : i + 1] for i in range(tr.iterations))
        return MedusaGenerateOutput(sequences=sequences, scores=rows_t if output_scores else None,
                                    logits=rows_t if output_logits else None,
                                    token_logprobs=token_logprobs[None].to(self._device), avg_logprob=avg,
                                    accept_lengths=list(tr.accept_lengths))

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
        """Raw logits of the last iteration: 0 = pass A ``[K+1, V]`` (every head at the newest position), 1 = the first
        K+1 verify rows ``[K+1, V]``, 2 = every verify row ``[n_tree, V]`` (tree nodes level by level)."""
        self._require_engine()
        rows = self.config.medusa_num_heads + 1
        if which == 2:
            rows = 0
            level = 1
            for c in self.config.medusa_choices:
                level *= int(c)
                rows += level
        n = (rows, self.config.vocab_size)
        out = torch.empty(n, dtype=torch.float32)
        lib = _lib.load()
        _check(lib, self._handle, lib.wm_last_logits(self._handle, which, C.cast(out.data_ptr(), C.POINTER(C.c_float))),
               "wm_last_logits")
        return out

    def last_no_speech(self, token: Optional[int] = None) -> Tuple[float, torch.Tensor]:
        """What the last ``generate(..., output_no_speech_prob=True)`` computed: ``p[token]`` (default: HF's no-speech
        token, ``no_timestamps_token_id - 1``) and the raw base-head logits ``FloatTensor[V]`` of the SOT row."""
        lib = _lib.load()
        token = int(self.generation_config.no_timestamps_token_id) - 1 if token is None else int(token)
        row = torch.empty(self.config.vocab_size, dtype=torch.float32)
        prob = C.c_float(0.0)
        _check(lib, self._handle, lib.wm_last_no_speech(self._handle, token, C.byref(prob),
                                                        C.cast(row.data_ptr(), C.POINTER(C.c_float))), "wm_last_no_speech")
        return float(prob.value), row

    def last_accept(self) -> Dict[str, Optional[Union[torch.Tensor, int]]]:
        """What the accept step of the last ``generate`` iteration compared (``wm_last_accept``), one entry per verify row
        / tree node (``n_tree`` = K+1 for a chain): ``cand`` the node tokens, ``row_argmax`` the argmax of every processed
        verify row, ``row_pc[n]`` (n >= 1) the probability of node n's token under its parent row's posterior,
        ``row_thr[r]`` the acceptance threshold ``min(posterior_threshold, posterior_alpha * exp(-entropy))`` of row r,
        ``path_node`` (trees only, else None) the node at depth ``accept`` of the best path.  ``row_pc`` and ``row_thr``
        are None at ``medusa_temperature=0`` (exact-match acceptance computes neither); entries of rows that have no
        child (chain: ``row_thr[K]``; ``row_pc[0]``) are not part of the decision."""
        self._require_engine()
        nt = self.config.medusa_num_heads + 1
        tree = any(int(c) != 1 for c in self.config.medusa_choices)
        if tree:
            nt, level = 0, 1
            for c in self.config.medusa_choices:
                level *= int(c)
                nt += level
        cand = torch.empty(16, dtype=torch.int32)
        arg = torch.empty(16, dtype=torch.int32)
        pc = torch.empty(16, dtype=torch.float32)
        thr = torch.empty(16, dtype=torch.float32)
        node = C.c_int32(0)
        lib = _lib.load()
        _check(lib, self._handle,
               lib.wm_last_accept(self._handle, C.cast(cand.data_ptr(), C.POINTER(C.c_int32)),
                                  C.cast(arg.data_ptr(), C.POINTER(C.c_int32)), C.cast(pc.data_ptr(), C.POINTER(C.c_float)),
                                  C.cast(thr.data_ptr(), C.POINTER(C.c_float)), C.byref(node)), "wm_last_accept")
        typical = getattr(self, "_last_medusa_temperature", 1.0) != 0.0
        return {"cand": cand[:nt], "row_argmax": arg[:nt], "row_pc": pc[:nt] if typical else None,
                "row_thr": thr[:nt] if typical else None, "path_node": int(node.value) if tree else None}

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
