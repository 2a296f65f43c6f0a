"""Word-timestamp alignment at large-v3: per-item b2w_align loop vs one b2w_align_batch call, and the batched pipeline with
word_timestamps on vs off.

Synthetic large-v3 (synthetic_seed=0), 16 chunks of synthetic audio, seeded text of --tokens tokens per chunk, num_frames 3000
(the last chunk 1700), with the default alignment heads (every head of the last 16 decoder layers: 320) and with a 10-pair list.
Times are host clocks around calls that end in a stream synchronise, after one warm-up call of each shape.

    python tools/align_bench.py [--dump align.json]

--per-item times only the b2w_align loop, so the script also runs from a checkout whose library has no b2w_align_batch: copy it
into that checkout's tools/ and compare the two --dump files output for output.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402

TEN_HEADS = [(16 + i, (3 * i) % 20) for i in range(10)]


def card() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def align_one(eng, enc, b, start, text, frames):
    from faster_whisper_b200 import engine

    rep = eng._replica_for(enc)
    s = np.ascontiguousarray(start, np.int32)
    t = np.ascontiguousarray(text, np.int32)
    cap = len(text) + frames // 2 + 2
    pairs = np.zeros((cap, 2), np.int32)
    probs = np.zeros(max(1, len(text)), np.float32)
    n = C.c_int32(0)
    engine._check(rep._lib.b2w_align(rep.handle, enc._handle, b, engine._ptr(s), len(s), engine._ptr(t), len(text), frames, 7,
                                     engine._ptr(pairs), cap, C.byref(n), engine._ptr(probs)))
    return pairs[: n.value].tolist(), probs[: len(text)].tolist()


def timed(fn, reps):
    fn()  # warm-up
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        out = fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return out, ts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--chunks", type=int, default=16)
    ap.add_argument("--tokens", type=int, default=150)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--per-item", action="store_true", help="time only the b2w_align loop")
    ap.add_argument("--no-transcribe", action="store_true")
    # synthetic weights decode to the length limit; a text that long leaves no room for the forced sequence of align
    ap.add_argument("--max-new-tokens", type=int, default=128)
    ap.add_argument("--dump", default=None, help="write every alignment and probability here (JSON)")
    args = ap.parse_args()

    from faster_whisper_b200 import BatchedInferencePipeline, WhisperModel
    from faster_whisper_b200.synthetic import synthetic_audio
    from oracle import whisper_oracle as orc

    print(json.dumps({"card": card()}), flush=True)
    model = WhisperModel("large-v3", device="cuda", synthetic_seed=0)
    eng = model.model
    n_mels = eng.dims.n_mels
    B = args.chunks
    feats = np.stack([orc.pad_or_trim(orc.log_mel(synthetic_audio(i, 30.0), n_mels)[:, :-1]) for i in range(B)])
    enc = eng.encode(feats)
    tok = eng.tokens
    start = [tok.sot, tok.lang_begin, tok.transcribe]
    rng = np.random.default_rng(0)
    texts = [rng.integers(100, 20000, args.tokens).tolist() for _ in range(B)]
    frames = [3000] * (B - 1) + [1700]
    dump = {}
    for name, heads in (("default_heads", None), ("ten_heads", TEN_HEADS)):
        eng.set_alignment_heads(heads)
        loop = lambda: [align_one(eng, enc, b, start, texts[b], frames[b]) for b in range(B)]  # noqa: E731
        per_item, t_loop = timed(loop, args.reps)
        line = {"heads": name, "chunks": B, "tokens": args.tokens, "per_item_ms": [round(t, 2) for t in t_loop]}
        if not args.per_item:
            batch = lambda: eng.align(enc, start, texts, frames)  # noqa: E731
            got, t_batch = timed(batch, args.reps)
            line["batched_ms"] = [round(t, 2) for t in t_batch]
            line["speedup"] = round(statistics.median(t_loop) / statistics.median(t_batch), 2)
            line["batched_pairs_equal_per_item"] = sum(g.alignments == [tuple(p) for p in pi[0]] for g, pi in zip(got, per_item))
        print(json.dumps(line), flush=True)
        dump[name] = per_item
    eng.set_alignment_heads(None)
    if args.dump:
        with open(args.dump, "w") as f:
            json.dump(dump, f)
    if args.per_item or args.no_transcribe:
        return
    audio = np.concatenate([synthetic_audio(i, 30.0) for i in range(B)])
    clips = [{"start": 30.0 * i, "end": 30.0 * (i + 1)} for i in range(B)]
    pipe = BatchedInferencePipeline(model)
    for wt in (False, True):
        run = lambda: list(pipe.transcribe(audio, batch_size=16, vad_filter=False, clip_timestamps=clips, language="en",  # noqa: E731
                                           max_new_tokens=args.max_new_tokens, word_timestamps=wt)[0])
        segs, ts = timed(run, args.reps)
        n_words = sum(len(s.words or []) for s in segs)
        print(json.dumps({"transcribe_word_timestamps": wt, "clips": B, "ms": [round(t, 1) for t in ts], "segments": len(segs),
                          "words": n_words}), flush=True)


if __name__ == "__main__":
    main()
