"""Version of the H100 engine; ``reference_version`` is the faster-whisper release whose API it mirrors."""

__version__ = "0.1.0"
reference_version = "1.2.1"
