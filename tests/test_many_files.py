"""CPU: ``BatchedInferencePipeline.transcribe_many`` against one ``transcribe`` per file, both over the oracle-backed engine shim.

The shim's engine calls are wrapped to compute batch item by batch item, so the oracle's results cannot depend on which
chunks share a call and ``transcribe_many(files)[i]`` must equal ``transcribe(files[i])`` exactly: segments, words and info.
The recorded traffic shows how the chunks of all files were packed into ``generate`` calls."""
import json
from math import ceil

import numpy as np
import pytest
import torch

from faster_whisper_b200 import engine as our_engine
from faster_whisper_b200 import transcribe as T
from faster_whisper_b200 import vad
from faster_whisper_b200.synthetic import make_tokenizer, synthetic_audio
from oracle import ct2_shim, silero_oracle
from oracle import whisper_oracle as orc

COMMON = dict(beam_size=2, max_new_tokens=6, without_timestamps=False)


def _per_item_model(m, calls):
    """WhisperModel over the shim, every engine call computed one batch item at a time."""
    dims, weights = m["dims"], m["weights"]
    whisper_cls, oracle = ct2_shim.make_whisper_class(dims, weights)

    class PerItem(whisper_cls):
        def encode(self, features, to_cpu=False):
            arr = features.numpy() if hasattr(features, "numpy") else np.asarray(features)
            calls.append(("encode", arr.shape[0]))
            return ct2_shim.StorageView(tensor=torch.cat([oracle.encode(arr[i : i + 1]) for i in range(arr.shape[0])]))

        def generate(self, features, prompts, **kw):
            calls.append(("generate", [list(p) for p in prompts]))
            kw.pop("asynchronous", None)
            enc = features.tensor
            out = [oracle.generate(enc[i : i + 1], [p], **kw)[0] for i, p in enumerate(prompts)]
            return [ct2_shim.WhisperGenerationResult(r.sequences_ids, r.scores, r.no_speech_prob) for r in out]

        def detect_language(self, features):
            calls.append(("detect_language", features.tensor.shape[0]))
            enc = features.tensor
            return [whisper_cls.detect_language(self, ct2_shim.StorageView(tensor=enc[i : i + 1]))[0] for i in range(enc.shape[0])]

        def align(self, features, start_sequence, text_tokens, num_frames, median_filter_width=7):
            calls.append(("align", list(start_sequence), [len(t) for t in text_tokens]))
            enc = features.tensor
            frames = num_frames if isinstance(num_frames, (list, tuple)) else [num_frames] * enc.shape[0]
            return [oracle.align(enc[i : i + 1], start_sequence, [t], [frames[i]], median_filter_width)[0]
                    for i, t in enumerate(text_tokens)]

    files = {"tokenizer.json": make_tokenizer(dims.n_vocab).to_str().encode(),
             "preprocessor_config.json": json.dumps({"feature_size": dims.n_mels}).encode()}
    mp = pytest.MonkeyPatch()
    mp.setattr(our_engine, "Whisper", lambda *a, **k: PerItem())
    mp.setattr(our_engine, "log_mel", lambda x, n_mels, padding=160, device=0: orc.log_mel(x, n_mels, padding))
    mp.setattr(our_engine, "StorageView", ct2_shim.StorageView)
    return T.WhisperModel("synthetic", device="cuda", files=files, dims=dims, weights=weights), mp


@pytest.fixture(scope="module")
def en(micro):
    calls = []
    model, mp = _per_item_model(micro, calls)
    yield model, calls
    mp.undo()


@pytest.fixture(scope="module")
def ml(micro_ml):
    calls = []
    model, mp = _per_item_model(micro_ml, calls)
    yield model, calls
    mp.undo()


def _files(seconds, seed):
    return [synthetic_audio(seed + i, s) if s else np.zeros(0, np.float32) for i, s in enumerate(seconds)]


def _check_against_single(model, calls, audios, kw, clips=None):
    """transcribe_many equals transcribe per file; returns the generate calls of transcribe_many."""
    pipe = T.BatchedInferencePipeline(model)
    calls.clear()
    got = pipe.transcribe_many([a.copy() for a in audios], clip_timestamps=clips, **kw)
    many_calls = list(calls)
    assert pipe.last_speech_timestamp == 0.0
    assert len(got) == len(audios)
    for i, a in enumerate(audios):
        segs, info = pipe.transcribe(a.copy(), clip_timestamps=clips[i] if clips else None, **kw)
        want = (list(segs), info)
        assert got[i][0] == want[0], f"file {i}: segments differ"
        assert got[i][1] == want[1], f"file {i}: info differs"
    return [c for c in many_calls if c[0] == "generate"]


def _n_chunks(model, audios, clips, kw):
    pipe = T.BatchedInferencePipeline(model)
    params = {k: p.default for k, p in T.signature(pipe.transcribe).parameters.items() if k not in ("audio", "clip_timestamps")}
    params.update(kw)
    return sum(len(p.chunks) for p in pipe._prepare([a.copy() for a in audios], clips or [None] * len(audios), params))


@pytest.mark.parametrize("batch_size", [2, 64])
def test_clips_and_whole_files(en, batch_size):
    """Files of 0 s, 3 s and 29 s transcribed whole, a 95 s file through user clips (one of them 41 s long)."""
    model, calls = en
    audios = _files([0, 3.0, 29.0, 95.0], seed=300)
    clips = [None, None, None, [{"start": 0.0, "end": 41.0}, {"start": 41.0, "end": 70.0}, {"start": 75.0, "end": 95.0}]]
    kw = dict(COMMON, language="en", vad_filter=False, batch_size=batch_size)
    gen = _check_against_single(model, calls, audios, kw, clips)
    n = _n_chunks(model, audios, clips, kw)
    assert n == 5
    assert len(gen) == ceil(n / batch_size)
    assert [len(c[1]) for c in gen] == [min(batch_size, n - lo) for lo in range(0, n, batch_size)]
    got = T.BatchedInferencePipeline(model).transcribe_many(audios, clip_timestamps=clips, **kw)
    assert got[0][0] == [] and got[0][1].duration == 0
    assert all(len(segs) > 0 for segs, _ in got[1:])


@pytest.fixture
def seeded_vad():
    w = silero_oracle.synthetic_weights(3)
    vad.set_vad_model(lambda a: silero_oracle.probs(w, a))
    yield
    vad.set_vad_model(None)


def test_vad_files(en, seeded_vad):
    """VAD through set_vad_model (the float64 Silero restatement on seeded weights) on files of 0, 3, 29 and 95 s."""
    model, calls = en
    audios = _files([0, 3.0, 29.0, 95.0], seed=310)
    kw = dict(COMMON, language="en", batch_size=3)
    gen = _check_against_single(model, calls, audios, kw)
    n = _n_chunks(model, audios, None, kw)
    assert n >= 4 and len(gen) == ceil(n / 3)
    infos = [info for _, info in T.BatchedInferencePipeline(model).transcribe_many(audios, **kw)]
    assert any(0 < i.duration_after_vad < i.duration for i in infos)


def test_word_timestamps(en):
    model, calls = en
    audios = _files([3.0, 29.0, 12.0], seed=320)
    kw = dict(COMMON, language="en", vad_filter=False, batch_size=2, word_timestamps=True, max_new_tokens=10)
    _check_against_single(model, calls, audios, kw)
    got = T.BatchedInferencePipeline(model).transcribe_many(audios, **kw)
    assert any(seg.words for segs, _ in got for seg in segs)


def test_multilingual(ml):
    model, calls = ml
    audios = _files([3.0, 29.0, 12.0, 20.0], seed=330)
    _check_against_single(model, calls, audios, dict(COMMON, language="en", vad_filter=False, batch_size=3, multilingual=True))


def _detect_files():
    """Two 9 s files the micro multilingual model puts in different languages (the quiet copy of a signal goes to another
    language), and a 35 s file in two clips whose features fill two detection windows."""
    audios = [synthetic_audio(0, 9.0), 0.01 * synthetic_audio(0, 9.0), synthetic_audio(1, 35.0)]
    clips = [None, None, [{"start": 0.0, "end": 20.0}, {"start": 20.0, "end": 35.0}]]
    return audios, clips


@pytest.mark.parametrize("word_timestamps", [False, True])
def test_detected_languages_share_a_generate_call(ml, word_timestamps):
    model, calls = ml
    audios, clips = _detect_files()
    kw = dict(COMMON, vad_filter=False, batch_size=8, word_timestamps=word_timestamps, language_detection_segments=2)
    gen = _check_against_single(model, calls, audios, kw, clips)
    got = T.BatchedInferencePipeline(model).transcribe_many(audios, clip_timestamps=clips, **kw)
    langs = [info.language for _, info in got]
    assert langs[0] != langs[1], langs
    assert len(gen) == 1 and len(gen[0][1]) == 4
    lang_ids = {model.hf_tokenizer.token_to_id(f"<|{lang}|>") for lang in langs}
    in_prompts = {t for p in gen[0][1] for t in p if t in lang_ids}
    assert len(in_prompts) >= 2, "one generate call carries two language tokens"
    if word_timestamps:
        assert len([c for c in calls if c[0] == "align"]) >= 2  # one align call per distinct start sequence


def test_language_detection_is_batched(ml):
    """Round 1 detects the first window of all three files in one encode + detect_language, round 2 the 35 s file's second
    window (its first was below the threshold); a round holds at most batch_size windows per call."""
    model, calls = ml
    audios, clips = _detect_files()
    calls.clear()
    T.BatchedInferencePipeline(model).transcribe_many(audios, clip_timestamps=clips, language_detection_segments=2,
                                                      **dict(COMMON, vad_filter=False))
    detect = [c for c in calls if c[0] in ("encode", "detect_language")][:4]
    assert detect == [("encode", 3), ("detect_language", 3), ("encode", 1), ("detect_language", 1)]
    # at most batch_size windows per encode: round 1 splits into 2 + 1
    calls.clear()
    T.BatchedInferencePipeline(model).transcribe_many(audios, clip_timestamps=clips, language_detection_segments=2,
                                                      batch_size=2, **dict(COMMON, vad_filter=False))
    detect = [c for c in calls if c[0] in ("encode", "detect_language")][:6]
    assert detect == [("encode", 2), ("detect_language", 2), ("encode", 1), ("detect_language", 1), ("encode", 1),
                      ("detect_language", 1)]


def test_speech_timestamps_many_without_a_multi_stream_model():
    w = silero_oracle.synthetic_weights(3)
    seen = []

    def model(a):
        seen.append(a.shape[0])
        return silero_oracle.probs(w, a)

    audios = _files([0, 3.0, 20.0], seed=340)
    opts = vad.VadOptions(min_silence_duration_ms=160)
    vad.set_vad_model(model)
    try:
        got = vad.get_speech_timestamps_many(audios, opts)
        want = [vad.get_speech_timestamps(a, opts) for a in audios]
    finally:
        vad.set_vad_model(None)
    assert got == want and len(seen) == 6


def test_rejects_unknown_arguments_and_mismatched_clips(en):
    model, _ = en
    pipe = T.BatchedInferencePipeline(model)
    with pytest.raises(TypeError, match="no_such_option"):
        pipe.transcribe_many([np.zeros(16000, np.float32)], no_such_option=1)
    with pytest.raises(ValueError, match="one entry"):
        pipe.transcribe_many([np.zeros(16000, np.float32)], clip_timestamps=[None, None])
    assert pipe.transcribe_many([]) == []
