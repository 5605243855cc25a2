"""Configuration types of the decode path.

Mirrors the two config classes the reference's hot path reads:

* ``MedusaConfig``            -- reference ``whisper_medusa/utils/config_and_args.py:17-62``
  (``WhisperConfig`` + ``medusa_*`` fields).  The reference's constructor calls
  ``AutoConfig.from_pretrained(whisper_model_name)`` (``config_and_args.py:49``), i.e. it
  needs the hub.  This engine is used offline, so the Whisper dimensions come either from
  the checkpoint's own ``config.json`` (which ``save_pretrained`` writes with the merged
  Whisper fields, ``config_and_args.py:60-62``) or from the built-in presets below.
* ``MedusaGenerationConfig``  -- reference ``whisper_medusa/models/medusa_utils.py:14-18``
  (``GenerationConfig`` + ``posterior_threshold=0.09`` / ``posterior_alpha=0.3``).

Only the fields the decode path reads are kept (SURVEY.md section 5, "Config / flags").
"""
from __future__ import annotations

import copy
import json
import os
from typing import Any, Dict, List, Optional

# Token-suppression lists of the public openai/whisper-* generation configs.  They are
# data, not code; reproduced from memory because the hub is unreachable here -- a real
# checkpoint directory brings its own ``generation_config.json`` which takes precedence.
_SUPPRESS_MULTILINGUAL = [
    1, 2, 7, 8, 9, 10, 14, 25, 26, 27, 28, 29, 31, 58, 59, 60, 61, 62, 63, 90, 91, 92, 93,
    359, 503, 522, 542, 873, 893, 902, 918, 922, 931, 1350, 1853, 1982, 2460, 2627, 3246,
    3253, 3268, 3536, 3846, 3961, 4183, 4667, 6585, 6647, 7273, 9061, 9383, 10428, 10929,
    11938, 12033, 12331, 12562, 13793, 14157, 14635, 15265, 15618, 16553, 16604, 18362,
    18956, 20075, 21675, 22520, 26130, 26161, 26435, 28279, 29464, 31650, 32302, 32470,
    36865, 42863, 47425, 49870, 50254, 50258, 50358, 50359, 50360, 50361, 50362,
]
_SUPPRESS_EN = [
    1, 2, 7, 8, 9, 10, 14, 25, 26, 27, 28, 29, 31, 58, 59, 60, 61, 62, 63, 90, 91, 92, 93,
    357, 366, 438, 532, 685, 705, 796, 930, 1058, 1220, 1267, 1279, 1303, 1343, 1377, 1391,
    1635, 1782, 1875, 2162, 2361, 2488, 3467, 4008, 4211, 4600, 4808, 5299, 5855, 6329,
    7203, 9609, 9959, 10563, 10786, 11420, 11709, 11907, 13163, 13697, 13700, 14808, 15306,
    16410, 16791, 17992, 19203, 19510, 20724, 22305, 22935, 27007, 30109, 30420, 33409,
    34949, 40283, 40493, 40549, 47282, 49146, 50257, 50357, 50358, 50359, 50360, 50361,
]

#: Whisper's language codes in token order (openai/whisper ``tokenizer.py`` LANGUAGES; multilingual checkpoints up to
#: large-v2 number them 50259 + index) and the spoken names HF's ``generate(language=...)`` also accepts
#: (``tokenization_whisper.py`` TO_LANGUAGE_CODE).  tests/test_cabi_and_host.py compares both with the installed
#: transformers tables.
WHISPER_LANGUAGE_CODES = (
    "en zh de es ru ko fr ja pt tr pl ca nl ar sv it id hi fi vi he uk el ms cs ro da hu ta no th ur hr bg lt la mi ml cy "
    "sk te fa lv bn sr az sl kn et mk br eu is hy ne mn bs kk sq sw gl mr pa si km sn yo so af oc ka be tg sd gu am yi lo "
    "uz fo ht ps tk nn mt sa lb my bo tl mg as tt haw ln ha ba jw su").split()
WHISPER_LANGUAGE_NAMES = {
    "english": "en", "chinese": "zh", "german": "de", "spanish": "es", "russian": "ru", "korean": "ko", "french": "fr",
    "japanese": "ja", "portuguese": "pt", "turkish": "tr", "polish": "pl", "catalan": "ca", "dutch": "nl", "arabic": "ar",
    "swedish": "sv", "italian": "it", "indonesian": "id", "hindi": "hi", "finnish": "fi", "vietnamese": "vi",
    "hebrew": "he", "ukrainian": "uk", "greek": "el", "malay": "ms", "czech": "cs", "romanian": "ro", "danish": "da",
    "hungarian": "hu", "tamil": "ta", "norwegian": "no", "thai": "th", "urdu": "ur", "croatian": "hr", "bulgarian": "bg",
    "lithuanian": "lt", "latin": "la", "maori": "mi", "malayalam": "ml", "welsh": "cy", "slovak": "sk", "telugu": "te",
    "persian": "fa", "latvian": "lv", "bengali": "bn", "serbian": "sr", "azerbaijani": "az", "slovenian": "sl",
    "kannada": "kn", "estonian": "et", "macedonian": "mk", "breton": "br", "basque": "eu", "icelandic": "is",
    "armenian": "hy", "nepali": "ne", "mongolian": "mn", "bosnian": "bs", "kazakh": "kk", "albanian": "sq",
    "swahili": "sw", "galician": "gl", "marathi": "mr", "punjabi": "pa", "sinhala": "si", "khmer": "km", "shona": "sn",
    "yoruba": "yo", "somali": "so", "afrikaans": "af", "occitan": "oc", "georgian": "ka", "belarusian": "be",
    "tajik": "tg", "sindhi": "sd", "gujarati": "gu", "amharic": "am", "yiddish": "yi", "lao": "lo", "uzbek": "uz",
    "faroese": "fo", "haitian creole": "ht", "pashto": "ps", "turkmen": "tk", "nynorsk": "nn", "maltese": "mt",
    "sanskrit": "sa", "luxembourgish": "lb", "myanmar": "my", "tibetan": "bo", "tagalog": "tl", "malagasy": "mg",
    "assamese": "as", "tatar": "tt", "hawaiian": "haw", "lingala": "ln", "hausa": "ha", "bashkir": "ba",
    "javanese": "jw", "sundanese": "su", "burmese": "my", "valencian": "ca", "flemish": "nl", "haitian": "ht",
    "letzeburgesch": "lb", "pushto": "ps", "panjabi": "pa", "moldavian": "ro", "moldovan": "ro", "sinhalese": "si",
    "castilian": "es", "mandarin": "zh", "cantonese": "yue",
}


def language_token(language: str) -> str:
    """``"en"`` / ``"english"`` / ``"<|en|>"`` -> ``"<|en|>"`` (HF ``generation_whisper.py:1490-1520``)."""
    lang = language.lower()
    if lang.startswith("<|") and lang.endswith("|>"):
        return lang
    lang = WHISPER_LANGUAGE_NAMES.get(lang, lang)
    return f"<|{lang}|>"


_LANG_TO_ID_V2 = {f"<|{c}|>": 50259 + i for i, c in enumerate(WHISPER_LANGUAGE_CODES)}

#: Whisper dimensions per base model name (SURVEY.md section 2.1).  ``micro`` is a
#: test-only shape small enough for pure-Python oracle loops.
WHISPER_PRESETS: Dict[str, Dict[str, Any]] = {
    "openai/whisper-large-v2": dict(
        vocab_size=51865, num_mel_bins=80, d_model=1280,
        encoder_layers=32, encoder_attention_heads=20, encoder_ffn_dim=5120,
        decoder_layers=32, decoder_attention_heads=20, decoder_ffn_dim=5120,
        max_source_positions=1500, max_target_positions=448,
        pad_token_id=50257, bos_token_id=50257, eos_token_id=50257,
        decoder_start_token_id=50258, is_multilingual=True,
        suppress_tokens=_SUPPRESS_MULTILINGUAL, begin_suppress_tokens=[220, 50257],
        # <|startoftranscript|> <|en|> <|transcribe|> <|notimestamps|>  (SURVEY.md 3.2 step 4)
        lang_to_id=_LANG_TO_ID_V2, task_to_id={"transcribe": 50359, "translate": 50358},
        no_timestamps_token_id=50363, max_length=448,
    ),
    "openai/whisper-tiny.en": dict(
        vocab_size=51864, num_mel_bins=80, d_model=384,
        encoder_layers=4, encoder_attention_heads=6, encoder_ffn_dim=1536,
        decoder_layers=4, decoder_attention_heads=6, decoder_ffn_dim=1536,
        max_source_positions=1500, max_target_positions=448,
        pad_token_id=50256, bos_token_id=50256, eos_token_id=50256,
        decoder_start_token_id=50257, is_multilingual=False,
        suppress_tokens=_SUPPRESS_EN, begin_suppress_tokens=[220, 50256],
        lang_to_id={}, task_to_id={}, no_timestamps_token_id=50362, max_length=448,
    ),
    "synthetic/whisper-micro": dict(
        vocab_size=512, num_mel_bins=80, d_model=128,
        encoder_layers=2, encoder_attention_heads=2, encoder_ffn_dim=256,
        decoder_layers=2, decoder_attention_heads=2, decoder_ffn_dim=256,
        max_source_positions=1500, max_target_positions=448,
        pad_token_id=500, bos_token_id=500, eos_token_id=500,
        decoder_start_token_id=501, is_multilingual=False,
        suppress_tokens=[1, 2, 7, 8, 9, 10, 14, 25, 501, 503], begin_suppress_tokens=[220, 500],
        lang_to_id={}, task_to_id={}, no_timestamps_token_id=502, max_length=448,
    ),
}
# The multilingual sizes between tiny and large (OpenAI's published dimensions: d_model, heads, encoder = decoder
# layers, FFN width) share large-v2's vocabulary, special tokens and suppress lists.
for _name, (_d, _h, _l, _f) in {"openai/whisper-base": (512, 8, 6, 2048), "openai/whisper-small": (768, 12, 12, 3072),
                                "openai/whisper-medium": (1024, 16, 24, 4096)}.items():
    WHISPER_PRESETS[_name] = dict(copy.deepcopy(WHISPER_PRESETS["openai/whisper-large-v2"]), d_model=_d,
                                  encoder_layers=_l, encoder_attention_heads=_h, encoder_ffn_dim=_f,
                                  decoder_layers=_l, decoder_attention_heads=_h, decoder_ffn_dim=_f)

_GENERATION_KEYS = (
    "suppress_tokens", "begin_suppress_tokens", "lang_to_id", "task_to_id",
    "no_timestamps_token_id", "max_length", "is_multilingual",
    "pad_token_id", "bos_token_id", "eos_token_id", "decoder_start_token_id",
)


class MedusaConfig:
    """Whisper dimensions + Medusa fields (reference ``config_and_args.py:17-62``)."""

    model_type = "whisper"

    def __init__(
        self,
        medusa_num_heads: int = 4,
        medusa_num_layers: int = 1,
        medusa_hidden_size: int = 1280,
        whisper_model_name: str = "openai/whisper-large-v2",
        medusa_choices: Optional[List[int]] = None,
        medusa_heads_type: str = "base_head",
        medusa_loss_on_original: bool = False,
        medusa_kl_loss: bool = False,
        medusa_kl_weight: float = 0,
        output_whisper_original: bool = False,
        **kwargs: Any,
    ) -> None:
        self.medusa_num_heads = int(medusa_num_heads)
        self.medusa_num_layers = int(medusa_num_layers)
        self.medusa_hidden_size = int(medusa_hidden_size)
        self.whisper_model_name = whisper_model_name
        self.medusa_choices = list(medusa_choices) if medusa_choices is not None else [1] * (self.medusa_num_heads + 1)
        self.medusa_heads_type = medusa_heads_type
        self.medusa_loss_on_original = medusa_loss_on_original
        self.medusa_kl_loss = medusa_kl_loss
        self.medusa_kl_weight = medusa_kl_weight
        self.output_whisper_original = output_whisper_original
        # Whisper fields: checkpoint values (kwargs) win over the preset, exactly like the
        # reference where config.json overlays the AutoConfig dict (config_and_args.py:60-62).
        base = copy.deepcopy(WHISPER_PRESETS.get(whisper_model_name, {}))
        base.update(kwargs)
        required = ("vocab_size", "d_model", "encoder_layers", "decoder_layers",
                    "encoder_attention_heads", "decoder_attention_heads",
                    "encoder_ffn_dim", "decoder_ffn_dim")
        missing = [k for k in required if k not in base]
        if missing:
            raise ValueError(
                f"unknown whisper_model_name {whisper_model_name!r} and the Whisper fields "
                f"{missing} were not supplied (no hub access: presets are {sorted(WHISPER_PRESETS)})")
        base.setdefault("num_mel_bins", 80)
        base.setdefault("max_source_positions", 1500)
        base.setdefault("max_target_positions", 448)
        base.setdefault("activation_function", "gelu")
        base.setdefault("scale_embedding", False)
        # width of the median filter applied to the alignment heads' weights for token timestamps (HF WhisperConfig)
        base.setdefault("median_filter_width", 7)
        for k, v in base.items():
            setattr(self, k, v)
        if self.medusa_heads_type not in ("base_head", "medusa_block"):
            # reference model.py:224-228
            raise ValueError(
                f"medusa_heads_type {self.medusa_heads_type} is not supported, "
                "select from ['base_head', 'medusa_block']")

    # -- HF-like surface -------------------------------------------------------------
    def to_dict(self) -> Dict[str, Any]:
        return {k: copy.deepcopy(v) for k, v in self.__dict__.items() if not k.startswith("_")}

    def save_pretrained(self, path: str) -> None:
        os.makedirs(path, exist_ok=True)
        with open(os.path.join(path, "config.json"), "w") as f:
            json.dump(self.to_dict(), f, indent=1)

    @classmethod
    def from_pretrained(cls, path: str, **kwargs: Any) -> "MedusaConfig":
        cfg_file = os.path.join(path, "config.json")
        if not os.path.isfile(cfg_file):
            raise OSError(f"{cfg_file} not found (hub download is not available; pass a local checkpoint directory)")
        with open(cfg_file) as f:
            d = json.load(f)
        d.update(kwargs)
        for k in ("model_type", "architectures", "transformers_version", "torch_dtype", "dtype", "_name_or_path"):
            d.pop(k, None)
        return cls(**d)

    # convenience
    @property
    def head_dim(self) -> int:
        return self.d_model // self.decoder_attention_heads

    @property
    def is_block(self) -> bool:
        return self.medusa_heads_type == "medusa_block"


class MedusaGenerationConfig:
    """Generation config + Medusa acceptance fields (reference ``medusa_utils.py:14-18``)."""

    def __init__(self, **kwargs: Any) -> None:
        self.posterior_threshold = kwargs.pop("posterior_threshold", 0.09)
        self.posterior_alpha = kwargs.pop("posterior_alpha", 0.3)
        self.max_length = kwargs.pop("max_length", 448)
        self.suppress_tokens = kwargs.pop("suppress_tokens", None)
        self.begin_suppress_tokens = kwargs.pop("begin_suppress_tokens", None)
        self.eos_token_id = kwargs.pop("eos_token_id", None)
        self.pad_token_id = kwargs.pop("pad_token_id", None)
        self.bos_token_id = kwargs.pop("bos_token_id", None)
        self.decoder_start_token_id = kwargs.pop("decoder_start_token_id", None)
        self.is_multilingual = kwargs.pop("is_multilingual", False)
        self.lang_to_id = kwargs.pop("lang_to_id", {})
        self.task_to_id = kwargs.pop("task_to_id", {})
        self.no_timestamps_token_id = kwargs.pop("no_timestamps_token_id", None)
        self.return_timestamps = kwargs.pop("return_timestamps", False)
        self.no_speech_threshold = kwargs.pop("no_speech_threshold", None)
        self.exponential_decay_length_penalty = kwargs.pop("exponential_decay_length_penalty", None)
        self.temperature = kwargs.pop("temperature", 1.0)
        self.num_beams = kwargs.pop("num_beams", 1)
        self.do_sample = kwargs.pop("do_sample", False)
        # [[layer, head], ...] cross-attention heads whose weights align tokens with audio frames (token timestamps); a
        # checkpoint brings them in its generation_config.json.  None: not available (saved only when set).
        self.alignment_heads = kwargs.pop("alignment_heads", None)
        self._extra = kwargs

    def update(self, **kwargs: Any) -> None:
        for k, v in kwargs.items():
            if hasattr(self, k):
                setattr(self, k, v)

    def to_dict(self) -> Dict[str, Any]:
        d = {k: copy.deepcopy(v) for k, v in self.__dict__.items() if not k.startswith("_")}
        if d.get("alignment_heads") is None:
            d.pop("alignment_heads", None)
        return d

    def save_pretrained(self, path: str) -> None:
        os.makedirs(path, exist_ok=True)
        with open(os.path.join(path, "generation_config.json"), "w") as f:
            json.dump(self.to_dict(), f, indent=1)

    @classmethod
    def from_pretrained(cls, path: str) -> "MedusaGenerationConfig":
        f = os.path.join(path, "generation_config.json")
        if not os.path.isfile(f):
            raise OSError(f"{f} not found")
        with open(f) as fh:
            d = json.load(fh)
        d.pop("transformers_version", None)
        return cls(**d)

    @classmethod
    def from_model_config(cls, config: MedusaConfig) -> "MedusaGenerationConfig":
        """Reference ``model.py:258-263``: Whisper generation config, then ``update(**config)``."""
        d = {k: copy.deepcopy(getattr(config, k)) for k in _GENERATION_KEYS if hasattr(config, k)}
        return cls(**d)
