"""In-tree build of libb200whisper.so (nvcc, sm_90a only).

``python -m faster_whisper_b200.build`` or ``__graft_entry__.build()``.  Objects go to ``build/`` (ignored),
the shared library lands next to this file so the package is importable from the source tree.
"""

from __future__ import annotations

import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libb200whisper.so")
SOURCES = ["mel.cu", "gemm.cu", "attention.cu", "encoder_misc.cu", "decode.cu", "dstep.cu", "bstep.cu", "search.cu", "align.cu", "vad.cu", "engine.cu"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC,-O3,-Wall,-Wno-unused-function", "--expt-relaxed-constexpr",
]


def source_fingerprint(path: str) -> str:
    """sha256 (16 hex digits) of a source file's CODE: blank lines and lines that are entirely a ``//`` comment do not count, so a
    profile keyed by it (tools/make_profiles.py) survives comment edits."""
    import hashlib

    h = hashlib.sha256()
    with open(path, "rb") as f:
        for line in f:
            t = line.strip()
            if t and not t.startswith(b"//"):
                h.update(t + b"\n")
    return h.hexdigest()[:16]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found; libb200whisper has no prebuilt or CPU fallback")


def _stale(target: str, deps) -> bool:
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False, ticks: bool = False) -> str:
    """``ticks=True`` builds libb200whisper_ticks.so with the cycle counters of the persistent step kernels compiled in
    (-DB2W_STEP_TICKS); point B2W_LIBRARY at it for a B2W_DSTEP_PROF=1 profile run."""
    from faster_whisper_b200.gen_wgmma import header

    nvcc = _nvcc()
    obj_dir = os.path.join(ROOT, "build", "obj_ticks" if ticks else "obj")
    gen_dir = os.path.join(ROOT, "build", "gen")
    lib = LIB.replace(".so", "_ticks.so") if ticks else LIB
    flags = NVCC_FLAGS + ["-I", gen_dir] + (["-DB2W_STEP_TICKS"] if ticks else [])
    os.makedirs(obj_dir, exist_ok=True)
    os.makedirs(gen_dir, exist_ok=True)
    gen = os.path.join(gen_dir, "wgmma.cuh")  # generated wgmma wrappers, rewritten only when their text changes
    text = header()
    if not os.path.exists(gen) or open(gen).read() != text:
        with open(gen, "w") as f:
            f.write(text)
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".h", ".cuh"))] + [gen]
    headers.append(os.path.join(ROOT, "include", "b200whisper.h"))
    jobs = []
    objs = []
    for src in SOURCES:
        s = os.path.join(CSRC, src)
        o = os.path.join(obj_dir, src.replace(".cu", ".o"))
        objs.append(o)
        if force or _stale(o, [s] + headers):
            cmd = [nvcc] + flags + (["-Xptxas", "-v"] if verbose else []) + ["-c", s, "-o", o]
            jobs.append(cmd)

    def run(cmd):
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed: %s\n%s\n%s" % (" ".join(cmd), r.stdout, r.stderr))
        if verbose:
            sys.stderr.write(r.stderr)
        return r

    if jobs:
        with ThreadPoolExecutor(max_workers=min(8, len(jobs))) as pool:
            list(pool.map(run, jobs))
    if jobs or force or _stale(lib, objs):
        # link to a temporary name and rename: a concurrent reader (another process) never sees a half-written library
        tmp = lib + ".tmp%d" % os.getpid()
        run([nvcc, "-shared", "-o", tmp] + objs + ["-gencode", "arch=compute_90a,code=sm_90a", "-cudart", "static", "-Xcompiler", "-fPIC"])
        os.replace(tmp, lib)
    return lib


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv, ticks="--ticks" in sys.argv))
