"""Test assets of the Silero VAD tests, copied from a faster-whisper source tree into oracle/_ref/ (kept out of git).

TEST INFRASTRUCTURE ONLY.  ``fetch()`` (run by ``__graft_entry__.build()``) copies the reference's ONNX asset
``faster_whisper/assets/silero_vad_v6.onnx`` and its speech recording ``tests/data/physicsworks.wav`` (203 s, 16 kHz mono
PCM16).  The tree is looked for at $B2W_REFERENCE_ROOT, else in a directory ``reference`` beside this repository or in the
home directory, else where an installed ``faster_whisper`` package lives.  ``fetch()`` says on stderr what it copied and
which files it could not find; the tests that need a missing file skip (the reader, parity and pipeline tests also run on a
Silero-shaped graph written from seeded weights, which needs neither file).  Tests read only oracle/_ref/.
"""
import importlib.util
import os
import shutil
import sys
import wave

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_DIR = os.path.join(ROOT, "oracle", "_ref")
FILES = {"silero_vad_v6.onnx": ("faster_whisper", "assets", "silero_vad_v6.onnx"),
         "physicsworks.wav": ("tests", "data", "physicsworks.wav")}


def reference_roots():
    """Candidate faster-whisper trees, most specific first."""
    cands = [os.environ.get("B2W_REFERENCE_ROOT", ""), os.path.join(os.path.dirname(ROOT), "reference"),
             os.path.join(os.path.expanduser("~"), "reference")]
    try:
        spec = importlib.util.find_spec("faster_whisper")
    except (ImportError, ValueError):
        spec = None
    if spec is not None and spec.origin:
        cands.append(os.path.dirname(os.path.dirname(spec.origin)))
    return [c for c in cands if c and os.path.isdir(os.path.join(c, "faster_whisper"))]


def fetch() -> None:
    roots = reference_roots()
    for name, rel in FILES.items():
        dst = os.path.join(REF_DIR, name)
        src = next((os.path.join(r, *rel) for r in roots if os.path.isfile(os.path.join(r, *rel))), "")
        if not src:
            if not os.path.isfile(dst):
                sys.stderr.write(f"silero_assets: {'/'.join(rel)} not found in a faster-whisper tree "
                                 f"(set B2W_REFERENCE_ROOT); tests that need oracle/_ref/{name} will skip\n")
            continue
        if os.path.isfile(dst) and os.path.getsize(dst) == os.path.getsize(src):
            continue
        os.makedirs(REF_DIR, exist_ok=True)
        tmp = dst + ".tmp%d" % os.getpid()
        shutil.copyfile(src, tmp)
        os.replace(tmp, dst)
        sys.stderr.write(f"silero_assets: copied {src} to oracle/_ref/{name}\n")


def path(name: str) -> str:
    """Path of a fetched asset, or "" when it is absent."""
    p = os.path.join(REF_DIR, name)
    return p if os.path.isfile(p) else ""


def physicsworks() -> np.ndarray:
    """The recording as float32 in [-1, 1)."""
    with wave.open(path("physicsworks.wav"), "rb") as w:
        assert w.getnchannels() == 1 and w.getsampwidth() == 2 and w.getframerate() == 16000
        return np.frombuffer(w.readframes(w.getnframes()), "<i2").astype(np.float32) / 32768.0
