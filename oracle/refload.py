"""Import the UNMODIFIED reference package from a faster-whisper source tree with its absent native deps stubbed.

TEST INFRASTRUCTURE ONLY (see oracle/whisper_oracle.py).  ``av``, ``ctranslate2`` and ``onnxruntime`` are
not installed in this image (SURVEY.md §8c); the reference's pure-Python host layer imports fine once
empty modules of those names exist.  ``ctranslate2`` can instead be bound to a shim backed by an engine
(``oracle/ct2_shim.py``) so the reference's own ``transcribe.py`` drives our engine or the oracle.
The tree is looked for at $B2W_REFERENCE_ROOT.  Tests do not need it: what they compare against is
stored under tests/golden/ (``RecordedReference``, gzip-compressed JSON); with the tree present and B2W_RECORD_REFERENCE=1 it is recorded again.
"""
import gzip
import importlib
import importlib.machinery
import json
import os
import sys
import types

REFERENCE_ROOT = os.environ.get("B2W_REFERENCE_ROOT", "")


def reference_available() -> bool:
    return bool(REFERENCE_ROOT) and os.path.isdir(os.path.join(REFERENCE_ROOT, "faster_whisper"))


def load_reference(ct2_module=None):
    """Returns the imported ``faster_whisper`` reference package (fresh import)."""
    if not reference_available():
        raise RuntimeError("reference tree not present")
    for name in list(sys.modules):
        if name == "faster_whisper" or name.startswith("faster_whisper."):
            del sys.modules[name]
    for name in ("av", "av.audio", "av.audio.fifo", "av.audio.resampler", "onnxruntime"):
        if name not in sys.modules:
            stub = types.ModuleType(name)
            # a real spec: importlib.util.find_spec (used by transformers' availability probes) raises on modules whose __spec__ is None
            stub.__spec__ = importlib.machinery.ModuleSpec(name, None)
            sys.modules[name] = stub
    if ct2_module is None:
        ct2_module = types.ModuleType("ctranslate2")
        ct2_module.models = types.ModuleType("ctranslate2.models")
        ct2_module.StorageView = type("StorageView", (), {})
        ct2_module.models.Whisper = type("Whisper", (), {})
        ct2_module.models.WhisperGenerationResult = type("WhisperGenerationResult", (), {})
    sys.modules["ctranslate2"] = ct2_module
    sys.modules["ctranslate2.models"] = ct2_module.models
    if REFERENCE_ROOT not in sys.path:
        sys.path.insert(0, REFERENCE_ROOT)
    try:
        return importlib.import_module("faster_whisper")
    finally:
        sys.path.remove(REFERENCE_ROOT)


def canon(x):
    """The JSON form of a value (tuples -> lists, NumPy scalars -> Python numbers)."""
    return json.loads(json.dumps(x, default=lambda o: o.item() if hasattr(o, "item") else o.tolist()))


class RecordedReference:
    """Values computed by the reference, stored as gzip-compressed JSON: ``get(key, fn)`` runs ``fn`` (on the reference) and stores
    its result when recording (B2W_RECORD_REFERENCE=1, reference tree at $B2W_REFERENCE_ROOT), and reads the stored result otherwise."""

    def __init__(self, path: str):
        self.path = path
        self.record = os.environ.get("B2W_RECORD_REFERENCE") == "1"
        if self.record and not reference_available():
            raise RuntimeError("B2W_RECORD_REFERENCE=1 needs the reference tree at $B2W_REFERENCE_ROOT")
        self.store = {}
        if os.path.exists(path):
            with gzip.open(path, "rt") as f:
                self.store = json.load(f)

    def get(self, key, fn):
        if self.record:
            self.store[key] = canon(fn())
            data = json.dumps(self.store, sort_keys=True, separators=(",", ":")).encode()
            with open(self.path, "wb") as f, gzip.GzipFile(fileobj=f, mode="wb", mtime=0) as z:  # mtime 0: same bytes for the same values
                z.write(data)
        return self.store[key]
