"""CPU: our WhisperModel / BatchedInferencePipeline and the UNMODIFIED reference host code, both driven over the same
oracle-backed ``ctranslate2`` shim on the same audio, must produce the same segments and info (drop-in check of the host
layer: prompt building, windowing/seek loop, fallback, batching, timestamp splitting).

The reference side of every comparison is stored in tests/golden/dropin_golden.json.gz, so the tests need nothing outside the
repository; oracle/refload.py records it again from the reference tree (B2W_RECORD_REFERENCE=1)."""
import dataclasses
import json
import os

import numpy as np
import pytest

from faster_whisper_b200 import engine as our_engine
from faster_whisper_b200 import transcribe as T
from faster_whisper_b200.synthetic import make_tokenizer, synthetic_audio
from oracle import ct2_shim
from oracle import whisper_oracle as orc
from oracle.refload import RecordedReference, canon, load_reference

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "dropin_golden.json.gz")


@pytest.fixture(scope="module")
def both(micro_ml):
    dims, weights = micro_ml["dims"], micro_ml["weights"]
    calls_ref, calls_our = [], []
    hf = make_tokenizer(dims.n_vocab)
    files = {"tokenizer.json": hf.to_str().encode(), "preprocessor_config.json": json.dumps({"feature_size": dims.n_mels}).encode()}
    ref = RecordedReference(GOLDEN)
    ref.fw = ref.model = None  # the reference package and its model, when recording
    if ref.record:
        mod, _ = ct2_shim.make_module(dims, weights, calls_ref)
        ref.fw = load_reference(ct2_module=mod)
        ref.model = ref.fw.WhisperModel("synthetic", device="cpu", files=dict(files))
    # ours: same shim class in place of the CUDA engine, oracle log-mel in place of the CUDA kernel
    whisper_cls, _ = ct2_shim.make_whisper_class(dims, weights, calls_our)
    mp = pytest.MonkeyPatch()
    mp.setattr(our_engine, "Whisper", lambda *a, **k: whisper_cls())
    mp.setattr(our_engine, "log_mel", lambda x, n_mels, padding=160, device=0: orc.log_mel(x, n_mels, padding))
    mp.setattr(our_engine, "StorageView", ct2_shim.StorageView)
    our_model = T.WhisperModel("synthetic", device="cuda", files=dict(files), dims=dims, weights=weights)
    yield ref, our_model, calls_ref, calls_our
    mp.undo()


def seg_tuple(s):
    return (s.id, s.seek, round(s.start, 3), round(s.end, 3), s.text, tuple(s.tokens), round(s.avg_logprob, 4),
            round(s.compression_ratio, 4), round(s.no_speech_prob, 5), s.temperature)


def strip(calls):
    out = []
    for c in calls:
        if c[0] == "generate":
            kw = {k: (round(v, 6) if isinstance(v, float) else v) for k, v in c[2].items()}
            out.append(("generate", c[1], kw))
        else:
            out.append(c)
    return out


COMMON = dict(no_speech_threshold=None, log_prob_threshold=None, compression_ratio_threshold=None)


def transcribe_record(model, calls, audio, kw):
    """Segments, engine traffic and info of one sequential transcribe() call, in the form the golden file stores."""
    calls.clear()
    segs, info = model.transcribe(audio.copy(), **kw)
    segs = [seg_tuple(s) for s in segs]
    return canon(dict(segs=segs, calls=strip(calls), info=[info.language, info.duration, info.duration_after_vad],
                      language_probability=info.language_probability, options=dataclasses.asdict(info.transcription_options)))


@pytest.mark.parametrize("kw", [
    dict(language="en", beam_size=2, max_new_tokens=12, **COMMON),
    dict(language="fr", task="translate", beam_size=1, without_timestamps=True, max_new_tokens=8, initial_prompt="hello there", **COMMON),
    dict(beam_size=2, max_new_tokens=6, temperature=[0.0, 0.4], log_prob_threshold=-0.5, no_speech_threshold=None,
         compression_ratio_threshold=2.4, best_of=2),
    dict(language="de", beam_size=1, max_new_tokens=10, clip_timestamps="3,20,31,40", hotwords="ab cd", condition_on_previous_text=False, **COMMON),
])
def test_sequential_transcribe_matches_reference(both, kw, request):
    ref, our_model, calls_ref, calls_our = both
    audio = np.concatenate([synthetic_audio(60, 30.0), synthetic_audio(61, 14.0)])
    want = ref.get(request.node.name, lambda: transcribe_record(ref.model, calls_ref, audio, kw))
    got = transcribe_record(our_model, calls_our, audio, kw)
    assert got["segs"] == want["segs"]
    assert len(want["segs"]) > 0
    assert got["calls"] == want["calls"]  # identical engine traffic: same prompts, same keyword arguments
    assert got["info"] == want["info"]
    assert got["language_probability"] == pytest.approx(want["language_probability"])
    assert got["options"] == want["options"]


@pytest.mark.parametrize("kw", [
    dict(language="en", beam_size=2, batch_size=2, max_new_tokens=8),
    dict(beam_size=1, batch_size=3, max_new_tokens=6, without_timestamps=False, multilingual=True),
    # prompt and hotwords, search options, a temperature list (the batched path takes its first entry), one chunk per call
    dict(language="fr", task="translate", beam_size=3, batch_size=1, max_new_tokens=7, initial_prompt="bonjour", hotwords="alpha beta", patience=2.0,
         length_penalty=0.7, repetition_penalty=1.1, no_repeat_ngram_size=3, temperature=[0.2, 0.8], suppress_tokens=[-1, 50]),
    # more chunks per call than there are chunks; thresholds that drop segments; timestamps on
    dict(language="en", beam_size=2, batch_size=8, max_new_tokens=9, without_timestamps=False, log_prob_threshold=-0.2, no_speech_threshold=0.3,
         compression_ratio_threshold=1.2),
])
def test_batched_transcribe_matches_reference(both, kw, request):
    ref, our_model, calls_ref, calls_our = both
    audio = np.concatenate([synthetic_audio(70 + i, 30.0) for i in range(3)] + [synthetic_audio(75, 7.5)])
    clips = [{"start": 0.0, "end": 30.0}, {"start": 30.0, "end": 60.0}, {"start": 60.0, "end": 90.0}, {"start": 90.0, "end": 97.5}]

    def run(pipe):
        segs, info = pipe.transcribe(audio.copy(), vad_filter=False, clip_timestamps=clips, **kw)
        return canon(dict(segs=[seg_tuple(s) for s in segs], info=[info.language, info.duration, info.duration_after_vad]))

    want = ref.get(request.node.name, lambda: run(ref.fw.BatchedInferencePipeline(ref.model)))
    got = run(T.BatchedInferencePipeline(our_model))
    assert got["segs"] == want["segs"] and (len(want["segs"]) >= 4 or "log_prob_threshold" in kw)
    assert got["info"] == want["info"]


def test_batched_errors_match_reference(both, request):
    ref, our_model, _, _ = both
    audio = synthetic_audio(1, 40.0)

    def errors(pipe):
        out = []
        with pytest.raises(RuntimeError, match="No clip timestamps found") as e1:
            pipe.transcribe(audio, vad_filter=False)
        out.append(["RuntimeError", str(e1.value)])
        with pytest.raises(ValueError, match="max_new_tokens") as e2:
            segs, _ = pipe.transcribe(audio[: 16000 * 10], vad_filter=False, language="en", max_new_tokens=500)
            list(segs)
        out.append(["ValueError", str(e2.value)])
        return out

    want = ref.get(request.node.name, lambda: errors(ref.fw.BatchedInferencePipeline(ref.model)))
    assert canon(errors(T.BatchedInferencePipeline(our_model))) == want


def test_detect_language_matches_reference(both, request):
    ref, our_model, _, _ = both
    audio = synthetic_audio(5, 45.0)
    a = ref.get(request.node.name, lambda: ref.model.detect_language(audio=audio, language_detection_segments=2, language_detection_threshold=0.99))
    b = our_model.detect_language(audio=audio, language_detection_segments=2, language_detection_threshold=0.99)
    assert a[0] == b[0] and a[1] == pytest.approx(b[1]) and [x[0] for x in a[2]] == [x[0] for x in b[2]]


def word_tuple(w):
    return (round(float(w.start), 3), round(float(w.end), 3), w.word, round(float(w.probability), 5))


def words_record(model, calls, audio, kw):
    """Segments with their words, engine traffic and info of one sequential transcribe() call (golden form)."""
    calls.clear()
    segs, info = model.transcribe(audio.copy(), **kw)
    segs = [(seg_tuple(s), [word_tuple(w) for w in (s.words or [])]) for s in segs]
    return canon(dict(segs=segs, calls=strip(calls), info=[info.language, info.duration], options=dataclasses.asdict(info.transcription_options)))


def test_word_timestamps_match_reference(both, request):
    """word_timestamps=True: both host layers call Whisper.align over the shim and post-process its alignments
    (merge punctuation, duration clamps, segment boundary fix-ups — transcribe.py:1567-1766)."""
    ref, our_model, calls_ref, calls_our = both
    audio = np.concatenate([synthetic_audio(80, 30.0), synthetic_audio(81, 9.0)])
    kw = dict(language="en", beam_size=2, max_new_tokens=10, word_timestamps=True, **COMMON)
    want = ref.get(request.node.name, lambda: words_record(ref.model, calls_ref, audio, kw))
    got = words_record(our_model, calls_our, audio, kw)
    assert got["segs"] == want["segs"]
    assert any(c[0] == "align" for c in want["calls"])
    assert got["calls"] == want["calls"]
    assert sum(len(w) for _, w in want["segs"]) > 0


@pytest.mark.parametrize("kw", [
    dict(language="en", beam_size=2, max_new_tokens=10, word_timestamps=True, hallucination_silence_threshold=0.5, **COMMON),
    dict(language="en", beam_size=1, max_new_tokens=9, prefix="hello", condition_on_previous_text=True, prompt_reset_on_temperature=0.3, **COMMON),
    dict(language="es", beam_size=2, max_new_tokens=8, without_timestamps=True, word_timestamps=True, prepend_punctuations="\"'“¿([{-",
         append_punctuations="\"'.。,，!！?？:：”)]}、", **COMMON),
    dict(beam_size=1, max_new_tokens=7, multilingual=True, language_detection_segments=2, language_detection_threshold=0.9, **COMMON),
    dict(language="en", beam_size=2, max_new_tokens=6, chunk_length=20, max_initial_timestamp=0.5, suppress_blank=False,
         suppress_tokens=[-1, 100, 200], length_penalty=0.8, patience=1.5, repetition_penalty=1.2, no_repeat_ngram_size=2, **COMMON),
    dict(language="en", beam_size=1, max_new_tokens=8, clip_timestamps=[2.0, 21.5], word_timestamps=True, **COMMON),
    # sampling fallback chain driven by the compression-ratio and log-prob tests; prompt given as token ids; empty suppress list
    dict(language="en", beam_size=2, best_of=3, max_new_tokens=8, temperature=[0.0, 0.5, 1.0], compression_ratio_threshold=0.1, log_prob_threshold=-0.01,
         no_speech_threshold=0.99, initial_prompt=[100, 200, 300], suppress_tokens=[]),
    # best_of sampling only, previous-text conditioning across windows, language detection on a later window
    dict(beam_size=1, best_of=2, temperature=0.7, max_new_tokens=6, condition_on_previous_text=True, language_detection_segments=2,
         language_detection_threshold=0.05, **COMMON),
    # hotwords without a prompt, timestamps on, vad parameters given although the filter is off, short chunk length
    dict(language="it", task="transcribe", beam_size=2, max_new_tokens=7, hotwords="uno due tre", chunk_length=15, vad_filter=False,
         vad_parameters=dict(threshold=0.4), **COMMON),
])
def test_more_sequential_options_match_reference(both, kw, request):
    ref, our_model, calls_ref, calls_our = both
    audio = np.concatenate([synthetic_audio(85, 30.0), synthetic_audio(86, 18.0)])
    want = ref.get(request.node.name, lambda: words_record(ref.model, calls_ref, audio, kw))
    got = words_record(our_model, calls_our, audio, kw)
    assert got["segs"] == want["segs"] and len(want["segs"]) > 0
    assert got["calls"] == want["calls"]
    assert got["info"] == want["info"]
    assert got["options"] == want["options"]


def batched_words(pipe, audio, kw):
    segs, info = pipe.transcribe(audio.copy(), **kw)
    return canon([(seg_tuple(s), [word_tuple(w) for w in (s.words or [])]) for s in segs])


def test_batched_word_timestamps_match_reference(both, request):
    ref, our_model, calls_ref, calls_our = both
    audio = np.concatenate([synthetic_audio(87 + i, 30.0) for i in range(2)] + [synthetic_audio(89, 11.0)])
    clips = [{"start": 0.0, "end": 30.0}, {"start": 30.0, "end": 60.0}, {"start": 60.0, "end": 71.0}]
    kw = dict(language="en", beam_size=2, batch_size=2, max_new_tokens=8, word_timestamps=True, vad_filter=False, clip_timestamps=clips)
    want = ref.get(request.node.name, lambda: batched_words(ref.fw.BatchedInferencePipeline(ref.model), audio, kw))
    got = batched_words(T.BatchedInferencePipeline(our_model), audio, kw)
    assert got == want and len(want) >= 3 and sum(len(w) for _, w in want) > 0


# ---- VAD segmentation logic vs the reference's, on the same per-window speech probabilities ----------------------------------
class _FakeVad:
    def __init__(self, seed, n_windows_hint=0):
        self.seed = seed

    def __call__(self, padded_audio, *a, **k):
        n = padded_audio.shape[0] // 512
        rng = np.random.default_rng(self.seed)
        # piecewise speech / silence with noisy probabilities so every branch of the hysteresis is visited
        p = np.zeros(n, np.float32)
        i = 0
        speech = bool(rng.integers(0, 2))
        while i < n:
            run = int(rng.integers(1, 120))
            lo, hi = (0.55, 1.0) if speech else (0.0, 0.45)
            p[i : i + run] = rng.uniform(lo, hi, min(run, n - i))
            i += run
            speech = not speech
        flip = rng.random(n) < 0.03
        p[flip] = 1.0 - p[flip]
        return p


@pytest.mark.parametrize("seed", range(12))
def test_vad_segmentation_matches_reference(both, seed, request):
    from faster_whisper_b200 import vad as our_vad

    ref = both[0]
    rng = np.random.default_rng(100 + seed)
    n = int(rng.integers(16000 * 5, 16000 * 120))
    audio = np.zeros(n, np.float32)
    opts = dict(threshold=float(rng.choice([0.5, 0.35, 0.6])), neg_threshold=[None, 0.2, 0.4][seed % 3],
                min_speech_duration_ms=int(rng.choice([0, 250, 1000])), max_speech_duration_s=float(rng.choice([float("inf"), 4.0, 12.0, 30.0])),
                min_silence_duration_ms=int(rng.choice([100, 500, 2000])), speech_pad_ms=int(rng.choice([0, 30, 400])))
    fake = _FakeVad(seed)
    times = (0.0, 1.234, 7.5, 33.3)

    def run(vad, mp=None):
        """Speech timestamps, the chunk packing and the timestamp map built on them (golden form)."""
        if mp is not None:
            mp.setattr(vad, "get_vad_model", lambda: fake)
        else:
            vad.set_vad_model(fake)
        ts = vad.get_speech_timestamps(audio, vad.VadOptions(**opts))
        out = dict(ts=ts, all_int=all(type(v) is int for s in ts for v in s.values()), chunks=[])
        for max_dur in (float("inf"), 30.0):
            chunks, meta = vad.collect_chunks(audio, ts, max_duration=max_dur)
            out["chunks"].append([[len(c) for c in chunks], meta])
        if ts:
            m = vad.SpeechTimestampsMap(ts, 16000)
            out["map"] = [[m.get_original_time(t), m.get_chunk_index(t)] for t in times]
        return canon(out)

    mp = pytest.MonkeyPatch()
    try:
        want = ref.get(request.node.name, lambda: run(ref.fw.vad, mp))
        got = run(our_vad)
        assert got["ts"] == want["ts"] and got["all_int"] == want["all_int"]
        # and the chunk packing / timestamp restoration built on top of it
        assert got["chunks"] == want["chunks"]
        assert got.get("map") == want.get("map")
    finally:
        mp.undo()
        our_vad.set_vad_model(None)


def test_transcribe_with_vad_filter_matches_reference(both, request):
    """vad_filter=True end to end (the batched pipeline's default): speech spans -> packed chunks -> engine -> restored times."""
    from faster_whisper_b200 import vad as our_vad

    ref, our_model, calls_ref, calls_our = both
    audio = np.concatenate([synthetic_audio(92, 30.0), synthetic_audio(93, 30.0), synthetic_audio(94, 12.0)])
    fake = _FakeVad(5)
    kw = dict(language="en", beam_size=1, max_new_tokens=8, vad_filter=True, vad_parameters=dict(min_silence_duration_ms=300), **COMMON)
    bkw = dict(language="en", beam_size=1, batch_size=2, max_new_tokens=6, word_timestamps=True)  # vad_filter defaults to True here

    def run(model, pipe):
        segs, info = model.transcribe(audio.copy(), **kw)
        out = dict(segs=[seg_tuple(s) for s in segs], after_vad=info.duration_after_vad, duration=info.duration)
        segs, info = pipe.transcribe(audio.copy(), **bkw)
        out["batched"] = [(seg_tuple(s), [word_tuple(w) for w in (s.words or [])]) for s in segs]
        out["batched_after_vad"] = info.duration_after_vad
        return canon(out)

    mp = pytest.MonkeyPatch()
    our_vad.set_vad_model(fake)
    try:
        def run_ref():
            mp.setattr(ref.fw.vad, "get_vad_model", lambda: fake)
            return run(ref.model, ref.fw.BatchedInferencePipeline(ref.model))

        want = ref.get(request.node.name, run_ref)
        got = run(our_model, T.BatchedInferencePipeline(our_model))
        assert got["segs"] == want["segs"] and len(want["segs"]) > 0
        assert got["after_vad"] == want["after_vad"] < want["duration"]
        assert got["batched"] == want["batched"] and len(want["batched"]) > 0
        assert got["batched_after_vad"] == want["batched_after_vad"]
    finally:
        mp.undo()
        our_vad.set_vad_model(None)


def test_batched_language_detection_window_spans_chunks(both, request):
    """A short first chunk: the reference's detection window continues into the NEXT chunk's frames (it concatenates all chunk features,
    transcribe.py:478-489); ours must pick the same language with the same probability and emit the same segments."""
    ref, our_model, calls_ref, calls_our = both
    audio = np.concatenate([synthetic_audio(80, 8.0), synthetic_audio(81, 30.0), synthetic_audio(82, 5.0)])
    clips = [{"start": 0.0, "end": 8.0}, {"start": 8.0, "end": 38.0}, {"start": 38.0, "end": 43.0}]
    kw = dict(beam_size=1, batch_size=2, max_new_tokens=5, vad_filter=False, clip_timestamps=clips, language_detection_segments=2)

    def run(pipe):
        segs, info = pipe.transcribe(audio.copy(), **kw)
        return canon(dict(segs=[seg_tuple(s) for s in segs], language=info.language, probability=info.language_probability,
                          top5=[x[0] for x in info.all_language_probs[:5]]))

    want = ref.get(request.node.name, lambda: run(ref.fw.BatchedInferencePipeline(ref.model)))
    got = run(T.BatchedInferencePipeline(our_model))
    assert got["language"] == want["language"] and got["probability"] == pytest.approx(want["probability"])
    assert got["top5"] == want["top5"]
    assert got["segs"] == want["segs"] and len(want["segs"]) >= 3


def test_batched_clip_longer_than_30s_matches_reference(both, request):
    """A user-supplied clip of more than 30 s: the reference computes the log-mel of the WHOLE clip (clamp maximum, last frames) and then trims
    the features to 3000 frames; so do we (the fused audio path is bypassed for such a block).  Also through language detection, whose
    window is cut out of the concatenated, untrimmed chunk features."""
    ref, our_model, calls_ref, calls_our = both
    loud_tail = np.concatenate([synthetic_audio(90, 30.0), 4.0 * synthetic_audio(91, 11.0)])  # the maximum sits beyond 30 s
    audio = np.concatenate([loud_tail, synthetic_audio(92, 20.0)])
    clips = [{"start": 0.0, "end": 41.0}, {"start": 41.0, "end": 61.0}]

    def run(pipe, calls, kw):
        calls.clear()
        segs, info = pipe.transcribe(audio.copy(), vad_filter=False, clip_timestamps=clips, **kw)
        segs = [seg_tuple(s) for s in segs]
        return canon(dict(segs=segs, encode=[c for c in calls if c[0] == "encode"],
                          info=[info.language, round(info.language_probability, 5), info.duration]))

    for i, kw in enumerate((dict(language="en", beam_size=2, batch_size=2, max_new_tokens=8), dict(beam_size=1, batch_size=1, max_new_tokens=6))):
        want = ref.get("%s/%d" % (request.node.name, i), lambda: run(ref.fw.BatchedInferencePipeline(ref.model), calls_ref, kw))
        got = run(T.BatchedInferencePipeline(our_model), calls_our, kw)
        assert got["segs"] == want["segs"] and len(want["segs"]) >= 2
        # the features that reached the encoder are the reference's, bit for bit (shape + checksum per engine call)
        assert got["encode"] == want["encode"]
        assert got["info"] == want["info"]


def test_empty_audio_matches_reference(both, request):
    """The reference's own test_empty_audio (tests/test_transcribe.py:91-97): an empty waveform gives no segments from either front end and
    language detection still answers; same results and same info from ours."""
    ref, our_model, calls_ref, calls_our = both
    audio = np.asarray([], dtype="float32")

    def run(model, pipe):
        out = {}
        segs, info = model.transcribe(audio.copy())
        out["sequential"] = [list(segs), [info.language, info.duration, info.duration_after_vad]]
        segs, info = pipe.transcribe(audio.copy(), vad_filter=False)
        out["batched"] = [list(segs), [info.language, info.duration, info.duration_after_vad]]
        out["detect"] = model.detect_language(audio.copy())
        return canon(out)

    want = ref.get(request.node.name, lambda: run(ref.model, ref.fw.BatchedInferencePipeline(ref.model)))
    got = run(our_model, T.BatchedInferencePipeline(our_model))
    for k in ("sequential", "batched"):
        assert want[k][0] == [] and got[k][0] == []
        assert got[k][1] == want[k][1]
    a, b = want["detect"], got["detect"]
    assert a[0] == b[0] and abs(a[1] - b[1]) < 1e-6 and [x for x, _ in a[2]] == [x for x, _ in b[2]]


def test_batched_clips_with_gaps_match_reference(both, request):
    """The reference's test_cliptimestamps_timings (tests/test_transcribe.py:295-310) shape: user clips of uneven length with gaps between
    them, with and without timestamps and word timestamps: segment times (and word times) are restored per clip exactly like the reference's."""
    ref, our_model, calls_ref, calls_our = both
    audio = np.concatenate([synthetic_audio(150, 20.0), synthetic_audio(151, 15.0)])
    clips = [{"start": 0.0, "end": 5.0}, {"start": 6.0, "end": 15.0}, {"start": 20.5, "end": 31.25}]
    for i, kw in enumerate((dict(language="en", beam_size=1, batch_size=2, max_new_tokens=8), dict(language="en", beam_size=2, batch_size=3, max_new_tokens=8,
                                                                                                 without_timestamps=False, word_timestamps=True))):
        kw = dict(kw, vad_filter=False, clip_timestamps=clips)
        want = ref.get("%s/%d" % (request.node.name, i), lambda: batched_words(ref.fw.BatchedInferencePipeline(ref.model), audio, kw))
        got = batched_words(T.BatchedInferencePipeline(our_model), audio, kw)
        assert got == want and len(want) >= 3
        if kw.get("without_timestamps", True):
            assert [[s[0][2], s[0][3]] for s in want] == [[c["start"], c["end"]] for c in clips]  # one segment per clip, at the clip's bounds
