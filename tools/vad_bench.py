"""Times the Silero VAD network on the GPU (vad.SileroGpuVAD, csrc/vad.cu) over one hour of audio.

    python tools/vad_bench.py [--hours 1] [--repeats 5] [--model PATH]

Device time per kernel comes from CUDA events the library records around each launch (b2w_vad_timing); the end-to-end rate
is host wall time of the whole call (PCM upload, kernels, probabilities back).  The audio is seeded synthetic speech-like
signal (the network's cost does not depend on the signal).  Weights: the ONNX asset when given or present in oracle/_ref/,
else seeded Silero-shaped weights.  Prints one JSON line with the card's name and power limit read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from faster_whisper_b200 import engine, silero  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = (s.strip() for s in out.split(","))
        return name, power
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})", "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--hours", type=float, default=1.0)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--model", default="")
    args = ap.parse_args()
    if engine.device_count() == 0:
        raise SystemExit("no CUDA device: nothing is measured")
    path = args.model or os.path.join(ROOT, "oracle", "_ref", "silero_vad_v6.onnx")
    if os.path.isfile(path):
        weights, source = silero.load_weights(path), os.path.basename(path)
    else:
        from oracle.silero_oracle import synthetic_weights

        weights, source = synthetic_weights(0), "synthetic"
    n = int(args.hours * 3600 * 16000) // 512
    rng = np.random.default_rng(0)
    audio = (0.05 * rng.standard_normal(n * 512) * np.repeat(rng.random(n // 64 + 1) < 0.6, 64 * 512)[: n * 512]).astype(np.float32)
    model = engine.SileroVad(weights)
    for _ in range(args.warmup):
        model.probs(audio)
    walls, dev = [], []
    for _ in range(args.repeats):
        t0 = time.perf_counter()
        model.probs(audio)
        walls.append(time.perf_counter() - t0)
        dev.append(model.timing())
    name, power = card()
    med = lambda xs: float(np.median(xs))  # noqa: E731
    win, rec, dec = (med([d[k] for d in dev]) for k in ("window", "recurrence", "decoder"))
    per_hour = 3600.0 / (n * 512 / 16000.0)
    print(json.dumps({
        "gpu": name, "power_limit": power, "weights": source, "windows": n, "repeats": args.repeats,
        "audio_s_per_s_wall": round(n * 512 / 16000.0 / med(walls), 1),
        "audio_s_per_s_device": round(n * 512 / 16000.0 / ((win + rec + dec) / 1e3), 1),
        "ms_per_audio_hour": {"window_kernel": round(win * per_hour, 3), "recurrence": round(rec * per_hour, 3),
                              "decoder": round(dec * per_hour, 3), "wall": round(med(walls) * 1e3 * per_hour, 3)},
        "us_per_recurrence_step": round(rec * 1e3 / n, 4),
        "recurrence_ms_spread": [round(min(d["recurrence"] for d in dev), 3), round(max(d["recurrence"] for d in dev), 3)],
    }))


if __name__ == "__main__":
    main()
