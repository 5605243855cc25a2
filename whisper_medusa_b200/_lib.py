"""ctypes binding of the C ABI declared in ``include/whisper_medusa_b200.h``.

The product path has no fallback: if the shared library is missing or a symbol is absent the
import of the engine fails loudly (``EngineUnavailable``).
"""
from __future__ import annotations

import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "_lib", "libwm_b200.so")


class EngineUnavailable(RuntimeError):
    pass


class WmConfig(C.Structure):
    _fields_ = [(n, C.c_int32) for n in (
        "vocab_size", "d_model", "n_heads", "ffn_dim", "enc_layers", "dec_layers", "n_mels",
        "max_source_positions", "max_target_positions", "medusa_num_heads", "medusa_block", "medusa_num_layers")]

WM_MAX_HEAD_LAYERS = 4   # include/whisper_medusa_b200.h


class WmGenParams(C.Structure):
    _fields_ = [
        ("max_length", C.c_int32), ("eos_token_id", C.c_int32), ("pad_token_id", C.c_int32),
        ("begin_index", C.c_int32), ("temperature", C.c_float), ("posterior_threshold", C.c_float),
        ("posterior_alpha", C.c_float), ("penalty_start", C.c_int32), ("penalty_factor", C.c_float),
        ("max_iters", C.c_int32), ("tree_attention", C.c_int32),
    ]


# name -> (restype, argtypes); must list every symbol of include/whisper_medusa_b200.h
_P = C.POINTER
SYMBOLS = {
    "wm_create": (C.c_int, [_P(WmConfig), C.c_int, _P(C.c_void_p)]),
    "wm_destroy": (C.c_int, [C.c_void_p]),
    "wm_strerror": (C.c_char_p, [C.c_int]),
    "wm_last_error": (C.c_char_p, [C.c_void_p]),
    "wm_tensor_count": (C.c_int, [C.c_void_p]),
    "wm_tensor_name": (C.c_char_p, [C.c_void_p, C.c_int]),
    "wm_tensor_info": (C.c_int, [C.c_void_p, C.c_char_p, _P(C.c_size_t), _P(C.c_size_t), _P(C.c_int32)]),
    "wm_weights_nbytes": (C.c_size_t, [C.c_void_p]),
    "wm_load_weights": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t]),
    "wm_adopt_weights": (C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t]),
    "wm_set_medusa_choices": (C.c_int, [C.c_void_p, _P(C.c_int32), C.c_int32]),
    "wm_set_suppress": (C.c_int, [C.c_void_p, _P(C.c_int32), C.c_int32, _P(C.c_int32), C.c_int32]),
    "wm_encode_pcm": (C.c_int, [C.c_void_p, _P(C.c_float), C.c_int32]),
    "wm_encode_mel": (C.c_int, [C.c_void_p, _P(C.c_float)]),
    "wm_encode_mel_device": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
    "wm_encode_pcm_device": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p]),
    "wm_resample": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_void_p, C.c_int64,
                              _P(C.c_int64), C.c_void_p]),
    "wm_resample_taps": (C.c_int, [C.c_int32, C.c_int32, _P(C.c_float), _P(C.c_int32), _P(C.c_int32), C.c_int64,
                                   _P(C.c_int32)]),
    "wm_generate": (C.c_int, [C.c_void_p, _P(C.c_int32), C.c_int32, _P(WmGenParams), _P(C.c_int32),
                              _P(C.c_int32), _P(C.c_int32), _P(C.c_int32)]),
    "wm_last_scores": (C.c_int, [C.c_void_p, _P(C.c_float), C.c_int32, _P(C.c_int32), _P(C.c_float), C.c_int32,
                                 _P(C.c_int32)]),
    "wm_last_no_speech": (C.c_int, [C.c_void_p, C.c_int32, _P(C.c_float), _P(C.c_float)]),
    "wm_set_alignment_heads": (C.c_int, [C.c_void_p, _P(C.c_int32), C.c_int32]),
    "wm_set_logits_processors": (C.c_int, [C.c_void_p, _P(C.c_int32), _P(C.c_int32), _P(C.c_float), C.c_int32,
                                           C.c_int32, C.c_int32]),
    "wm_set_sampling": (C.c_int, [C.c_void_p, C.c_float, C.c_int32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32]),
    "wm_sample_noise": (C.c_int, [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_int32, C.c_int32,
                                  C.c_int32, _P(C.c_float)]),
    "wm_token_timestamps": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_double, _P(C.c_float),
                                      _P(C.c_float), _P(C.c_int32)]),
    "wm_token_timestamps_from_probs": (C.c_int, [C.c_void_p, _P(C.c_float), C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                                 C.c_int32, C.c_int32, C.c_double, _P(C.c_float), _P(C.c_float),
                                                 _P(C.c_int32)]),
    "wm_last_alignment_probs": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, _P(C.c_float), C.c_int64, _P(C.c_int32)]),
    "wm_forward": (C.c_int, [C.c_void_p, _P(C.c_int32), C.c_int32, _P(C.c_float)]),
    "wm_get_mel": (C.c_int, [C.c_void_p, _P(C.c_float)]),
    "wm_get_encoder_out": (C.c_int, [C.c_void_p, _P(C.c_float)]),
    "wm_last_logits": (C.c_int, [C.c_void_p, C.c_int32, _P(C.c_float)]),
    "wm_last_accept": (C.c_int, [C.c_void_p, _P(C.c_int32), _P(C.c_int32), _P(C.c_float), _P(C.c_float),
                                 _P(C.c_int32)]),
    "wm_last_ms": (C.c_double, [C.c_void_p, C.c_int32]),
    "wm_last_launches": (C.c_int64, [C.c_void_p, C.c_int32]),
    "wm_decode_cluster": (C.c_int, [C.c_void_p]),
    "wm_set_decode_mode": (C.c_int, [C.c_void_p, C.c_int32]),
    "wm_weights_device_ptr": (C.c_void_p, [C.c_void_p]),
    "wm_enc_gemm_tile": (C.c_int, [C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, _P(C.c_int32)]),
    "wm_ring_schedule_check": (C.c_int, [C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                         _P(C.c_int32), _P(C.c_int32)]),
    "wm_ring_prefetch_check": (C.c_int, [C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                         _P(C.c_int32), _P(C.c_int32)]),
    "wm_ring_schedule_check_head_layers": (C.c_int, [C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                                     C.c_int32, _P(C.c_int32), _P(C.c_int32)]),
    "wm_set_option": (C.c_int, [C.c_void_p, C.c_char_p, C.c_int32]),
    "wm_get_stage_profile": (C.c_int, [C.c_void_p, _P(C.c_int64), C.c_int32, _P(C.c_int32)]),
}

_lib = None


def load():
    """Load the engine library (no GPU needed to load; needed to call)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.isfile(LIB_PATH):
        raise EngineUnavailable(
            f"{LIB_PATH} is missing: build it with `python -m whisper_medusa_b200.build` "
            "(there is no CPU / PyTorch fallback for this path)")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SYMBOLS.items():
        try:
            fn = getattr(lib, name)
        except AttributeError as e:
            raise EngineUnavailable(f"{LIB_PATH} does not export {name}") from e
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib
