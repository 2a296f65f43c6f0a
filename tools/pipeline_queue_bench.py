"""``BatchedInferencePipeline.transcribe_many`` decoded group by group (``generate``) against one decode queue per call
(``continuous_batching=True``).

    python tools/pipeline_queue_bench.py [--files 16] [--eot-scale 3.6] [--repeats 2]

The workload is N seeded synthetic recordings of 30-120 s cut into 30 s clips, on the large-v3 geometry with seeded weights,
batch_size 16 and beam 5, <|endoftext|> allowed and no cap below the model's 448 tokens.  Seeded weights almost never rank
<|endoftext|> first, so every chunk would run to the cap and both arms would do the same work.  This script (only this script)
therefore scales the <|endoftext|> row of the checkpoint's tied token embedding by ``--eot-scale``: chunks then end at seeded,
varied steps, as real speech ends chunks after a few tokens or after hundreds.  ``--scan`` instead prints the new-token histogram
of one continuous pass for each scale it is given, to choose the scale.  With seed 0 the change is abrupt: up to 3.4 every chunk
runs past 256 tokens, from 3.6 most end within 8 tokens and a few run past 256 (the default, 3.6, gives 43 and 6 of 49).

After a warm-up of both arms they run alternately, ``--repeats`` times each; audio-s/s is total audio over host wall time of one
whole pass (median).  Prints one JSON line: the card's name and power limit read in the same run, the histogram of new-token
counts, the predicted step ratio (the sum over the group path's groups of the group's longest chunk, over the sum of lengths divided
by the slots), per arm its decode steps, audio-s/s and peak encoder-output bytes (``Whisper.memory``, sampled after every engine
call that can raise it, so the continuous arm's peak includes a batch's own output while it is being split), and the chunks whose tokens differ between the arms with both arms' avg_logprob: a different batch
composition changes the order of floating-point sums, which can flip a near-tie."""
import argparse
import json
import os
import subprocess
import sys
import time

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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--files", type=int, default=16)
    ap.add_argument("--min-s", type=float, default=30.0)
    ap.add_argument("--max-s", type=float, default=120.0)
    ap.add_argument("--model", default="large-v3")
    ap.add_argument("--batch-size", type=int, default=16)
    ap.add_argument("--beam-size", type=int, default=5)
    ap.add_argument("--eot-scale", type=float, default=3.6)
    ap.add_argument("--scan", type=float, nargs="*", help="print the token-count histogram of each of these scales and stop")
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()
    if engine.device_count() == 0:
        raise SystemExit("no CUDA device: nothing is measured")

    from faster_whisper_b200 import BatchedInferencePipeline, WhisperModel
    from faster_whisper_b200.config import MODEL_DIMS, special_tokens
    from faster_whisper_b200.synthetic import make_weights, synthetic_audio

    dims = MODEL_DIMS[args.model]
    st = special_tokens(dims.n_vocab)
    rng = np.random.default_rng(args.seed)
    seconds = np.round(rng.uniform(args.min_s, args.max_s, args.files), 2)
    audios = [synthetic_audio(args.seed * 10000 + i, float(s)) for i, s in enumerate(seconds)]
    clips = [[{"start": lo, "end": min(lo + 30.0, float(s))} for lo in np.arange(0.0, float(s), 30.0)] for s in seconds]
    total_audio = float(seconds.sum())
    kw = dict(language="en", batch_size=args.batch_size, beam_size=args.beam_size, without_timestamps=True, vad_filter=False)
    base = make_weights(dims, seed=args.seed)
    emb = base["decoder.token_embedding.weight"]

    def model_at(scale):
        w = dict(base)
        w["decoder.token_embedding.weight"] = emb.copy()
        w["decoder.token_embedding.weight"][st.eot] *= scale
        return WhisperModel(args.model, device="cuda", weights=w, dims=dims)

    def lengths(res):
        return [len(s.tokens) for segs, _ in res for s in segs]

    def histogram(n):
        edges = [0, 8, 16, 32, 64, 128, 256, 447, 448]
        h, _ = np.histogram(n, bins=edges + [449])
        return {f"{lo}-{hi - 1}": int(c) for lo, hi, c in zip(edges, edges[1:] + [449], h)}

    if args.scan:
        for scale in args.scan:
            model = model_at(scale)
            n = lengths(BatchedInferencePipeline(model, continuous_batching=True).transcribe_many(audios, clip_timestamps=clips, **kw))
            print(json.dumps({"eot_scale": scale, "chunks": len(n), "histogram": histogram(n)}))
            model.model.unload_model()
            del model
        return

    model = model_at(args.eot_scale)
    inner = model.model
    peak = [0]
    for name in ("generate", "split_encoded", "encode_audio", "encode"):
        real = getattr(inner, name)

        def sampled(*a, _real=real, **k):
            out = _real(*a, **k)
            peak[0] = max(peak[0], inner.memory()["encoded_bytes"])
            return out

        setattr(inner, name, sampled)
    push = engine.DecodeQueue.push

    def sampled_push(self, *a, **k):
        ids = push(self, *a, **k)
        peak[0] = max(peak[0], inner.memory()["encoded_bytes"])
        return ids

    engine.DecodeQueue.push = sampled_push
    arms = {"group": BatchedInferencePipeline(model), "continuous": BatchedInferencePipeline(model, continuous_batching=True)}

    def timed(name):
        peak[0] = 0
        inner.sync()
        steps = inner.timing()["decode_steps"]
        t0 = time.perf_counter()
        res = arms[name].transcribe_many(audios, clip_timestamps=clips, **kw)
        inner.sync()
        wall = time.perf_counter() - t0
        toks = [(list(s.tokens), s.avg_logprob) for segs, _ in res for s in segs]
        return wall, toks, inner.timing()["decode_steps"] - steps, peak[0]

    for name in arms:  # warm-up
        timed(name)
    runs = {name: [] for name in arms}
    for _ in range(args.repeats):
        for name in arms:
            runs[name].append(timed(name))
    gpu, power = card()
    n = [len(t) for t, _ in runs["group"][-1][1]]
    slots = min(args.batch_size, 80 // args.beam_size)
    longest = sum(max(n[lo : lo + args.batch_size]) for lo in range(0, len(n), args.batch_size))
    med = lambda xs: float(np.median(xs))  # noqa: E731
    differ = []
    for c, (a, b) in enumerate(zip(runs["group"][-1][1], runs["continuous"][-1][1])):
        if a[0] != b[0]:
            pos = next((i for i, (p, q) in enumerate(zip(a[0], b[0])) if p != q), min(len(a[0]), len(b[0])))
            differ.append({"chunk": c, "token": pos, "avg_logprob": [round(a[1], 5), round(b[1], 5)]})
    per_chunk = 1500 * 2 * (dims.n_audio_state + 2 * dims.n_text_layer * dims.n_text_state)
    out = {"gpu": gpu, "power_limit": power, "model": args.model, "files": args.files, "chunks": len(n), "audio_s": round(total_audio, 1),
           "batch_size": args.batch_size, "beam_size": args.beam_size, "slots": slots, "eot_scale": args.eot_scale,
           "new_tokens_histogram": histogram(n), "predicted_step_ratio": round(longest / (sum(n) / slots), 3)}
    for name, rs in runs.items():
        out[name] = {"audio_s_per_s": round(total_audio / med([r[0] for r in rs]), 1), "wall_s": [round(r[0], 3) for r in rs],
                     "decode_steps": int(rs[-1][2]), "peak_encoded_bytes": int(max(r[3] for r in rs)),
                     "peak_encoded_chunks": round(max(r[3] for r in rs) / per_chunk, 2)}
    out["speedup"] = round(out["continuous"]["audio_s_per_s"] / out["group"]["audio_s_per_s"], 3)
    out["chunks_with_different_tokens"] = len(differ)
    out["different_tokens"] = differ
    print(json.dumps(out))


if __name__ == "__main__":
    main()
