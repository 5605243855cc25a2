"""H100-native Whisper-Medusa decode path behind the reference's Python API.

``from whisper_medusa_b200 import WhisperMedusaModel`` mirrors
``from whisper_medusa import WhisperMedusaModel`` (reference ``whisper_medusa/__init__.py:1``).
"""
from .config import MedusaConfig, MedusaGenerationConfig  # noqa: F401
from .model import EngineError, MedusaGenerateOutput, WhisperMedusaModel  # noqa: F401
from .streams import StreamGroup  # noqa: F401

__all__ = ["WhisperMedusaModel", "StreamGroup", "MedusaConfig", "MedusaGenerationConfig", "EngineError",
           "MedusaGenerateOutput"]
