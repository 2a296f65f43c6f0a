"""compute_type float16 against float8_float16 in one process, arms alternating after warm-up.

Reports, per arm: the encoder stage's device time per chunk (the engine's ``encoder`` stage events) at large-v3 with 16 chunks
per call, the achieved TFLOP/s against the H100 SXM data-sheet dense peaks (989 fp16, 1 979 fp8), encode + generate audio-s/s
at large-v3 and turbo geometry (synthetic weights, beam 5, end-of-text suppressed so every chunk decodes the same tokens), and
the fp8 arm's encoder-output error against the float16 arm.  The card's name and power limit are read in the same run.

    python tools/fp8_encoder_bench.py [--reps 5] [--tokens 64] [--out fp8_encoder_bench.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from faster_whisper_b200 import engine  # noqa: E402
from faster_whisper_b200.config import MODEL_DIMS, special_tokens  # noqa: E402
from faster_whisper_b200.synthetic import make_weights, synthetic_audio  # noqa: E402
from oracle.whisper_oracle import log_mel, pad_or_trim  # noqa: E402

ARMS = ("float16", "float8_float16")


def encoder_flops(dims) -> float:
    """Per chunk: conv stem, the four linear layers of each block, and attention (QK^T and PV)."""
    d, T = dims.n_audio_state, 1500
    conv = 2 * 3000 * d * 3 * dims.n_mels + 2 * T * d * 3 * d
    linear = dims.n_audio_layer * 2 * T * 12 * d * d
    attn = dims.n_audio_layer * 2 * 2 * T * T * d
    return float(conv + linear + attn), float(linear)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--chunks", type=int, default=16)
    ap.add_argument("--tokens", type=int, default=64)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    result = {"card": card()}
    for name in ("large-v3", "large-v3-turbo"):
        dims = MODEL_DIMS[name]
        st = special_tokens(dims.n_vocab)
        w = make_weights(dims, seed=0)
        engines = {ct: engine.Whisper(dims=dims, weights=w, tokens=st, device="cuda", compute_type=ct) for ct in ARMS}
        del w
        feats = np.stack([pad_or_trim(log_mel(synthetic_audio(i, 30.0), dims.n_mels)[:, :-1]) for i in range(args.chunks)])
        prompt = [[st.sot, st.lang_begin, st.transcribe, st.no_timestamps]] * args.chunks
        kw = dict(beam_size=5, max_length=len(prompt[0]) + args.tokens, suppress_tokens=[st.eot])
        total, linear = encoder_flops(dims)
        enc_ms = {ct: [] for ct in ARMS}
        e2e = {ct: [] for ct in ARMS}
        outs = {}
        for rep in range(args.reps + 1):  # rep 0 warms every shape up
            for ct in ARMS:
                e = engines[ct]
                e.timing(enable=True, reset=True)
                enc = e.encode(feats)
                ms = e.timing()["encoder_ms"]
                if name == "large-v3":
                    outs[ct] = enc.numpy()
                t0 = time.perf_counter()
                e.generate(e.encode(feats), prompt, **kw)
                dt = time.perf_counter() - t0
                if rep > 0:
                    enc_ms[ct].append(ms / args.chunks)
                    e2e[ct].append(args.chunks * 30.0 / dt)
        r = {}
        for ct in ARMS:
            m = float(np.median(enc_ms[ct]))
            r[ct] = dict(encoder_ms_per_chunk=m, encoder_ms_per_chunk_all=enc_ms[ct], encoder_tflops=total / m / 1e9,
                         share_of_fp16_peak=total / m / 1e9 / 989.0, share_of_fp8_peak=total / m / 1e9 / 1979.0,
                         audio_s_per_s=float(np.median(e2e[ct])), audio_s_per_s_all=e2e[ct])
        sp = [a / b for a, b in zip(enc_ms["float16"], enc_ms["float8_float16"])]
        r["encoder_speedup_per_rep"] = sp
        r["gflop_per_chunk"] = total / 1e9
        r["linear_share"] = linear / total
        if name == "large-v3":
            a, b = outs["float8_float16"], outs["float16"]
            r["fp8_vs_fp16_encoder_output"] = dict(max_abs=float(np.abs(a - b).max()),
                                                   rel_frobenius=float(np.linalg.norm(a - b) / np.linalg.norm(b)))
        result[name] = r
        print(name, json.dumps(r, indent=1), flush=True)
        del engines
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)
    print(json.dumps({k: (v if isinstance(v, str) else {ct: v[ct]["encoder_ms_per_chunk"] for ct in ARMS}) for k, v in result.items()}))


if __name__ == "__main__":
    main()
