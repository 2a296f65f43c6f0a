"""Hopper (H100) Whisper engine with faster-whisper's public API (reference ``faster_whisper/__init__.py:1-14``)."""

from .audio import decode_audio
from .transcribe import BatchedInferencePipeline, WhisperModel
from .utils import available_models, download_model, format_timestamp
from .version import __version__

__all__ = [
    "available_models",
    "decode_audio",
    "WhisperModel",
    "BatchedInferencePipeline",
    "download_model",
    "format_timestamp",
    "__version__",
]
