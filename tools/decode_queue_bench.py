"""Group-at-a-time decoding against continuous batching on chunks of unequal length.

    python tools/decode_queue_bench.py [--chunks 128] [--repeats 3] [--dist uniform|bimodal|both]

large-v3 geometry with seeded weights (``synthetic_seed``), fp16, beam 5, seeded synthetic 30 s chunks encoded once.  Every chunk
gets its own new-token cap from a seeded distribution (uniform 16-128, or bimodal: 16-32 for 70 % of the chunks and 112-128 for
the rest) and <|endoftext|> is suppressed, so a chunk decodes exactly its cap and the work does not depend on the weights.  Two
arms run in the same process, alternating after a warm-up of both:
  (a) ``generate`` per group of 16 chunks with the group's largest cap: what group-at-a-time decoding costs;
  (b) one ``decode_queue`` over all chunks with per-item caps: a finished chunk's slot takes the next queued chunk.
Decode time is CUDA-event time on the model's stream (span_begin / span_end) around the whole arm; audio-s/s is the chunks' 30 s
each over that time (median over the repeats).  Also printed: decode steps of each arm, the queue's mean occupied rows per step,
and the step ratio the caps predict, computed from the caps alone (sum of group maxima over the queue's steps when every slot is
refilled the moment it frees, simulated on the CPU).  One JSON line per distribution, with the card's name and power limit read
in the same run."""
import argparse
import heapq
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from faster_whisper_b200 import engine  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = (s.strip() for s in out.split(","))
        return name, power
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})", "unknown"


def caps_for(dist, n, seed):
    rng = np.random.default_rng(seed)
    if dist == "uniform":
        return rng.integers(16, 129, n)
    short = rng.random(n) < 0.7
    return np.where(short, rng.integers(16, 33, n), rng.integers(112, 129, n))


def predicted_steps(caps, group):
    """(group-at-a-time steps, queue steps) from the caps alone: groups cost their largest cap; the queue hands each item in push
    order to the slot that frees first, and runs until the last slot finishes."""
    grouped = sum(int(caps[i : i + group].max()) for i in range(0, len(caps), group))
    slots = [0] * min(group, len(caps))
    for c in caps:
        t = heapq.heappop(slots)
        heapq.heappush(slots, t + int(c))
    return grouped, max(slots)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--chunks", type=int, default=128)
    ap.add_argument("--model", default="large-v3")
    ap.add_argument("--beam-size", type=int, default=5)
    ap.add_argument("--group", type=int, default=16)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--dist", choices=["uniform", "bimodal", "both"], default="both")
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()
    if engine.device_count() == 0:
        raise SystemExit("no CUDA device: nothing is measured")

    from faster_whisper_b200 import WhisperModel
    from faster_whisper_b200.config import MODEL_DIMS, special_tokens
    from faster_whisper_b200.synthetic import synthetic_audio

    st = special_tokens(MODEL_DIMS[args.model].n_vocab)
    model = WhisperModel(args.model, device="cuda", compute_type="float16", synthetic_seed=args.seed)
    w = model.model
    prompt = [st.sot, st.lang_begin, st.transcribe, st.no_timestamps]
    P = len(prompt)
    G = args.group
    encs = [w.encode_audio([synthetic_audio(args.seed * 1000 + i, 30.0) for i in range(g0, min(args.chunks, g0 + G))])
            for g0 in range(0, args.chunks, G)]
    kw = dict(beam_size=args.beam_size, suppress_tokens=[-1, st.eot])
    name, power = card()

    def grouped(caps):
        out = []
        for gi, enc in enumerate(encs):
            c = caps[gi * G : gi * G + enc.shape[0]]
            out += w.generate(enc, [prompt] * enc.shape[0], max_length=P + int(c.max()), **kw)
        return out

    def queued(caps):
        q = w.decode_queue(max_length=P + int(caps.max()), slots=G, **kw)
        for gi, enc in enumerate(encs):
            c = caps[gi * G : gi * G + enc.shape[0]]
            q.push(enc, [prompt] * enc.shape[0], [P + int(x) for x in c])
        res = dict(q)
        steps, rows = q.counters()
        q.close()
        return [res[i] for i in range(len(caps))], steps, rows

    def timed(f):
        w.sync()
        w.span_begin()
        r = f()
        return r, w.span_end()

    for dist in (["uniform", "bimodal"] if args.dist == "both" else [args.dist]):
        caps = caps_for(dist, args.chunks, args.seed + (0 if dist == "uniform" else 1))
        timed(lambda: grouped(caps))
        timed(lambda: queued(caps))
        ms_a, ms_b = [], []
        steps_a = steps_b = rows_b = 0
        for _ in range(args.repeats):
            before = w.timing().get("decode_steps", 0)
            res_a, t = timed(lambda: grouped(caps))
            steps_a = int(w.timing().get("decode_steps", 0) - before)
            ms_a.append(t)
            (res_b, steps_b, rows_b), t = timed(lambda: queued(caps))
            ms_b.append(t)
        lens_ok = all(len(r.sequences_ids[0]) == int(c) for r, c in zip(res_b, caps))
        same = sum(a.sequences_ids[0][: int(c)] == b.sequences_ids[0] for a, b, c in zip(res_a, res_b, caps))
        pred_a, pred_b = predicted_steps(caps, G)
        audio = 30.0 * args.chunks
        print(json.dumps({
            "gpu": name, "power_limit": power, "model": args.model, "dtype": "f16", "beam": args.beam_size, "chunks": args.chunks,
            "dist": dist, "caps_mean": float(caps.mean()),
            "grouped_audio_s_per_s": audio / (float(np.median(ms_a)) / 1e3), "queue_audio_s_per_s": audio / (float(np.median(ms_b)) / 1e3),
            "grouped_ms": [round(x, 1) for x in ms_a], "queue_ms": [round(x, 1) for x in ms_b],
            "grouped_steps": steps_a, "queue_steps": steps_b, "queue_mean_live_rows": rows_b / max(1, steps_b),
            "predicted_steps": [pred_a, pred_b], "predicted_step_ratio": pred_a / pred_b,
            "queue_items_decode_their_cap": lens_ok, "items_with_equal_prefix": same,
        }), flush=True)


if __name__ == "__main__":
    main()
