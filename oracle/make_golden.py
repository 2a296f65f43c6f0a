"""Generates tests/golden/*.npz|json by RUNNING THE REFERENCE (imported from the reference tree with stubs, oracle/refload.py).

TEST INFRASTRUCTURE ONLY.  Run where the reference tree exists ($B2W_REFERENCE_ROOT):

    python oracle/make_golden.py

Fixtures:
  mel_golden.npz       reference FeatureExtractor outputs: seeded synthetic clips (80/128 mels, several lengths) in full,
                       and the first 30 s of tests/data/physicsworks.wav subsampled (every 7th frame) + its global stats.
  host_golden.json     reference host-logic outputs: _split_segments_by_timestamps, get_prompt, get_suppressed_tokens,
                       collect_chunks, SpeechTimestampsMap, format_timestamp, merge_punctuations on fixed inputs.
"""
import json
import os
import sys
import wave

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from faster_whisper_b200.synthetic import make_tokenizer, synthetic_audio  # noqa: E402
from oracle.refload import REFERENCE_ROOT, load_reference  # noqa: E402


def read_wav(path, seconds):
    with wave.open(path, "rb") as w:
        n = min(w.getnframes(), int(seconds * w.getframerate()))
        x = np.frombuffer(w.readframes(n), dtype="<i2").astype(np.float32) / 32768.0
    return x


def main():
    if not REFERENCE_ROOT:
        raise SystemExit("make_golden.py runs the reference: set B2W_REFERENCE_ROOT to the faster-whisper source tree")
    fw = load_reference()
    out = {}
    for nm in (80, 128):
        fe = fw.feature_extractor.FeatureExtractor(feature_size=nm)
        for n in (0, 159, 160, 4000, 48000):
            out[f"synth_{nm}_{n}"] = fe(synthetic_audio(5, n / 16000.0))
    speech = read_wav(os.path.join(REFERENCE_ROOT, "tests", "data", "physicsworks.wav"), 30.0)
    out["speech_pcm_head"] = speech[:48000]
    for nm in (80, 128):
        fe = fw.feature_extractor.FeatureExtractor(feature_size=nm)
        full = fe(speech)
        out[f"speech_{nm}_sub7"] = full[:, ::7]
        out[f"speech_{nm}_stats"] = np.array([full.mean(), full.std(), full.max(), full.min()], np.float64)
        out[f"speech_head_{nm}"] = fe(speech[:48000])
    np.savez_compressed(os.path.join(ROOT, "tests/golden/mel_golden.npz"), **out)

    # ---- host logic --------------------------------------------------------------------------------------
    T = fw.transcribe
    tok_hf = make_tokenizer(51865)
    tok = fw.tokenizer.Tokenizer(tok_hf, True, task="transcribe", language="en")
    model = T.WhisperModel.__new__(T.WhisperModel)
    model.time_precision, model.input_stride, model.max_length = 0.02, 2, 448
    ts0 = tok.timestamp_begin
    rng = np.random.default_rng(0)
    split_cases = []
    fixed = [
        [ts0, 100, 101, ts0 + 50, ts0 + 50, 200, ts0 + 120, ts0 + 120, 300, 301],
        [ts0, 100, ts0 + 40],
        [100, 101, 102],
        [ts0 + 5, 100, ts0 + 30, ts0 + 30, 7, 8, ts0 + 99],
        [],
        [ts0, ts0],
        [ts0, 5, ts0 + 10, ts0 + 10],
    ]
    for _ in range(40):
        n = int(rng.integers(1, 30))
        seq, t = [], 0
        for _ in range(n):
            if rng.random() < 0.4:
                t += int(rng.integers(0, 60))
                seq.append(ts0 + min(t, 1500))
                if rng.random() < 0.5:
                    seq.append(ts0 + min(t, 1500))
            else:
                seq.append(int(rng.integers(0, 50000)))
        fixed.append(seq)
    for seq in fixed:
        segs, seek, single = model._split_segments_by_timestamps(tok, list(seq), 12.5, 2800, 28.0, 100)
        split_cases.append(dict(tokens=list(map(int, seq)), segments=segs, seek=int(seek), single=bool(single)))
    prompts = []
    for kw in [dict(previous_tokens=[], without_timestamps=False), dict(previous_tokens=[1, 2, 3], without_timestamps=True),
               dict(previous_tokens=list(range(400)), without_timestamps=False, prefix="hello world"),
               dict(previous_tokens=[], without_timestamps=True, hotwords="ab cd"),
               dict(previous_tokens=[9], without_timestamps=False, hotwords="ab cd", prefix="zz")]:
        prompts.append(dict(kwargs=kw, prompt=model.get_prompt(tok, **kw)))
    sup = [dict(arg=a, out=list(T.get_suppressed_tokens(tok, list(a)))) for a in ([-1], [13], [-1, 5, 6], [])]
    audio = np.arange(16000 * 100, dtype=np.float32)
    spans = [{"start": 1000, "end": 200000}, {"start": 300000, "end": 700000}, {"start": 800000, "end": 900000},
             {"start": 1000000, "end": 1500000}]
    chunks, metas = fw.vad.collect_chunks(audio, spans, max_duration=30)
    tsm = fw.vad.SpeechTimestampsMap(spans, 16000)
    vad = dict(spans=spans, chunk_lens=[int(c.shape[0]) for c in chunks], chunk_first=[float(c[0]) if c.size else None for c in chunks],
               metas=metas, orig=[tsm.get_original_time(t) for t in (0.0, 5.0, 12.4, 30.0, 60.0)],
               orig_end=[tsm.get_original_time(t, is_end=True) for t in (12.4375, 37.4375)])
    fmt = [[s, fw.utils.format_timestamp(s), fw.utils.format_timestamp(s, True, ",")] for s in (0, 1.2345, 59.9996, 3661.5)]
    al = [dict(word=" (", tokens=[1]), dict(word=" hello", tokens=[2, 3]), dict(word=",", tokens=[4]), dict(word=" world", tokens=[5]),
          dict(word=".", tokens=[6]), dict(word=" \"", tokens=[7]), dict(word=" yes", tokens=[8])]
    T.merge_punctuations(al, "\"'“¿([{-", "\"'.。,，!！?？:：”)]}、")
    host = dict(split=split_cases, prompts=prompts, suppressed=sup, vad=vad, format_timestamp=fmt, merged=al,
                special=dict(sot=tok.sot, eot=tok.eot, ts0=ts0, no_speech=tok.no_speech, sot_sequence=tok.sot_sequence),
                compression=[[s, T.get_compression_ratio(s)] for s in ("hello hello hello hello", "abc")])
    with open(os.path.join(ROOT, "tests/golden/host_golden.json"), "w") as f:
        json.dump(host, f)
    print("wrote goldens:", {k: v.shape for k, v in list(out.items())[:4]}, len(split_cases))


if __name__ == "__main__":
    main()
