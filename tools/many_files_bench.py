"""Many short recordings: one ``BatchedInferencePipeline.transcribe`` call per file against one ``transcribe_many`` call.

    python tools/many_files_bench.py [--files 64] [--min-s 8] [--max-s 75] [--repeats 3] [--vad]

The workload is N seeded synthetic recordings of mixed lengths on the large-v3 geometry with seeded weights
(``synthetic_seed``).  Both modes use the same options: batch_size 16, beam 5 and ``max_new_tokens`` with <|endoftext|>
suppressed, so every chunk decodes exactly that many tokens and the work does not depend on the weights.  Without ``--vad`` a
file is cut into clips of at most 30 s (the whole file when it is shorter); with ``--vad`` the chunks come from the Silero VAD
on the GPU, with the ONNX asset when oracle/_ref/ holds it, else seeded Silero-shaped weights written as an ONNX file.

After a warm-up of both modes they run alternately, ``--repeats`` times each; audio-s/s is total audio over host wall time of
one whole pass (median).  Prints one JSON line with the card's name and power limit read in the same run, the VAD device
milliseconds of each mode (b2w_vad_timing, summed over the mode's VAD calls), the generate calls and chunks per call, and the
files whose tokens differ between the modes.  A different batch composition changes the order of floating-point sums, which can
flip a near-tie; for each such file the line gives its first differing chunk, the token where the two decodes part, and both
modes' avg_logprob of that chunk: two hypotheses of nearly equal score are what a near-tie looks like."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
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
    ap.add_argument("--files", type=int, default=64)
    ap.add_argument("--min-s", type=float, default=8.0)
    ap.add_argument("--max-s", type=float, default=75.0)
    ap.add_argument("--model", default="large-v3")
    ap.add_argument("--max-new-tokens", type=int, default=128)
    ap.add_argument("--batch-size", type=int, default=16)
    ap.add_argument("--beam-size", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--vad", action="store_true")
    args = ap.parse_args()
    if engine.device_count() == 0:
        raise SystemExit("no CUDA device: nothing is measured")

    from faster_whisper_b200 import BatchedInferencePipeline, WhisperModel, vad
    from faster_whisper_b200.config import MODEL_DIMS, special_tokens
    from faster_whisper_b200.synthetic import synthetic_audio

    tmp = tempfile.mkdtemp(prefix="many_files_bench_")
    if args.vad:
        asset = os.path.join(ROOT, "oracle", "_ref", "silero_vad_v6.onnx")
        if os.path.isfile(asset):
            path, vad_weights = asset, "silero_vad_v6.onnx"
        else:
            from oracle.silero_oracle import synthetic_weights, write_onnx

            path, vad_weights = os.path.join(tmp, "silero_synthetic.onnx"), "synthetic"
            write_onnx(synthetic_weights(3), path)
        sys.modules["onnxruntime"] = None  # the GPU network, not onnxruntime on the CPU
        os.environ["B2W_SILERO_VAD"] = path
        vad.set_vad_model(None)

    rng = np.random.default_rng(args.seed)
    seconds = np.round(rng.uniform(args.min_s, args.max_s, args.files), 2)
    audios = [synthetic_audio(args.seed * 10000 + i, float(s)) for i, s in enumerate(seconds)]
    clips = None if args.vad else [[{"start": lo, "end": min(lo + 30.0, float(s))} for lo in np.arange(0.0, float(s), 30.0)]
                                   for s in seconds]
    total_audio = float(seconds.sum())

    st = special_tokens(MODEL_DIMS[args.model].n_vocab)
    model = WhisperModel(args.model, device="cuda", synthetic_seed=args.seed)
    pipe = BatchedInferencePipeline(model)
    kw = dict(language="en", batch_size=args.batch_size, beam_size=args.beam_size, max_new_tokens=args.max_new_tokens,
              suppress_tokens=[-1, st.eot], without_timestamps=True, vad_filter=args.vad)

    gen_sizes = []
    real_generate = model.model.generate

    def counting_generate(features, prompts, **k):
        gen_sizes.append(len(prompts))
        return real_generate(features, prompts, **k)

    model.model.generate = counting_generate

    def vad_ms():
        return sum(vad.get_vad_model(model.model.device_index[0]).model.timing().values()) if args.vad else 0.0

    def per_file():
        out, ms = [], 0.0
        for i, a in enumerate(audios):
            segs, _ = pipe.transcribe(a, clip_timestamps=clips[i] if clips else None, **kw)
            out.append([(list(s.tokens), s.avg_logprob) for s in segs])
            ms += vad_ms()
        return out, ms

    def many():
        res = pipe.transcribe_many(audios, clip_timestamps=clips, **kw)
        return [[(list(s.tokens), s.avg_logprob) for s in segs] for segs, _ in res], vad_ms()

    def timed(fn):
        gen_sizes.clear()
        model.model.sync()
        t0 = time.perf_counter()
        toks, ms = fn()
        model.model.sync()
        return time.perf_counter() - t0, toks, ms, list(gen_sizes)

    timed(per_file)  # warm-up of both modes
    timed(many)
    runs = {"per_file": [], "many": []}
    for _ in range(args.repeats):
        for name, fn in (("per_file", per_file), ("many", many)):
            runs[name].append(timed(fn))
    name, power = card()
    med = lambda xs: float(np.median(xs))  # noqa: E731
    a, b = runs["per_file"][-1], runs["many"][-1]
    differ = []  # per file whose tokens differ: its first differing chunk, where the tokens part, both modes' avg_logprob
    for f, (x, y) in enumerate(zip(a[1], b[1])):
        if [t for t, _ in x] == [t for t, _ in y]:
            continue
        c = next(i for i, (u, v) in enumerate(zip(x, y)) if u[0] != v[0])
        pos = next((i for i, (p, q) in enumerate(zip(x[c][0], y[c][0])) if p != q), min(len(x[c][0]), len(y[c][0])))
        differ.append({"file": f, "chunk": c, "token": pos, "avg_logprob": [round(x[c][1], 5), round(y[c][1], 5)]})
    out = {"gpu": name, "power_limit": power, "model": args.model, "files": args.files,
           "seconds": [args.min_s, args.max_s], "audio_s": round(total_audio, 1), "vad": args.vad,
           "batch_size": args.batch_size, "beam_size": args.beam_size, "max_new_tokens": args.max_new_tokens}
    if args.vad:
        out["vad_weights"] = vad_weights
    for key, rs in runs.items():
        sizes = rs[-1][3]
        out[key] = {"audio_s_per_s": round(total_audio / med([r[0] for r in rs]), 1),
                    "wall_s": [round(r[0], 3) for r in rs], "vad_ms": round(med([r[2] for r in rs]), 3),
                    "generate_calls": len(sizes), "chunks_per_call": round(sum(sizes) / max(1, len(sizes)), 2)}
    out["files_with_different_tokens"] = len(differ)
    out["different_tokens"] = differ
    if differ:
        out["max_abs_d_avg_logprob"] = round(max(abs(d["avg_logprob"][0] - d["avg_logprob"][1]) for d in differ), 5)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
