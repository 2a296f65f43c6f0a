"""CPU: ``BatchedInferencePipeline(model, continuous_batching=True)`` against the group path, both over the oracle-backed engine shim.

The shim computes every engine call batch item by batch item (``test_many_files._per_item_model``), so results cannot depend on
which chunks share a call.  A fake decode queue, defined here, returns finished items in a seeded scrambled order and a seeded number
at a time, holds a finished item's encoding until the next ``run`` (as a session slot does until it is rebound), and counts the
per-chunk encodings alive.  Continuous output must equal the group path's exactly: every Segment field, words and info."""
import weakref

import numpy as np
import pytest

from faster_whisper_b200 import transcribe as T
from faster_whisper_b200 import vad
from oracle import ct2_shim, silero_oracle
from oracle import whisper_oracle as orc
from test_many_files import _files, _per_item_model

COMMON = dict(beam_size=2, max_new_tokens=6, without_timestamps=False)


class Tracker:
    """Sessions opened and closed, per-chunk encodings alive (and their peak), encode calls, and an optional failing run."""

    def __init__(self):
        self.reset()

    def reset(self, fail_after=None):
        self.sessions, self.live, self.peak, self.encodes, self.fail_after, self.slots = [], 0, 0, 0, fail_after, []

    def born(self, sv):
        self.live += 1
        self.peak = max(self.peak, self.live)
        weakref.finalize(sv, self._died)

    def _died(self):
        self.live -= 1


class FakeQueue:
    """``DecodeQueue``'s contract over the oracle: slots as the session sets them (at most 80 // rows per chunk), FIFO refill, and
    only encoder outputs of its own replica."""

    def __init__(self, oracle, tracker, slots, seed, replica, **kw):
        self.oracle, self.tracker, self.kw, self.replica = oracle, tracker, kw, replica
        self.slots = min(slots, max(1, 80 // kw["beam_size"]))
        self.rng = np.random.default_rng(seed)
        self.items, self.held, self.next_id, self.closed, self.runs = [], [], 0, False, 0
        tracker.sessions.append(self)
        tracker.slots.append(self.slots)

    def push(self, sv, prompts, max_lengths):
        assert not self.closed and sv.shape[0] == len(prompts) == len(max_lengths) == 1
        if sv.replica != self.replica:
            raise ValueError("the encoder output belongs to another replica")
        self.items.append((self.next_id, sv, list(prompts[0]), int(max_lengths[0])))
        self.next_id += 1
        return [self.next_id - 1]

    def pending(self):
        return len(self.items)

    def run(self):
        assert not self.closed
        self.runs += 1
        if self.tracker.fail_after is not None and self.runs > self.tracker.fail_after:
            raise RuntimeError("injected run failure")
        if len(self.items) >= self.slots:  # idle slots are rebound, dropping the finished items they held
            self.held = []
        if not self.items:
            return []
        decoding = self.items[: self.slots]
        k = int(self.rng.integers(1, len(decoding) + 1))
        pick = sorted(self.rng.choice(len(decoding), k, replace=False).tolist())
        done = [decoding[j] for j in pick]
        self.items = [it for j, it in enumerate(self.items) if j not in pick]
        self.held = [sv for _, sv, _, _ in done]
        out = []
        for item, sv, prompt, ml in done:
            kw = dict(self.kw, max_length=ml)
            r = self.oracle.generate(sv.tensor, [prompt], **kw)[0]
            out.append((item, ct2_shim.WhisperGenerationResult(r.sequences_ids, r.scores, r.no_speech_prob)))
        return [out[j] for j in self.rng.permutation(len(out))]

    def close(self):
        self.closed, self.items, self.held = True, [], []


def _continuous_model(m, tracker, n_replicas=1):
    """The per-item shim with split_encoded, align_items and a fake decode_queue, and `n_replicas` engine replicas: an encoder
    output remembers the replica that made it, chosen round-robin unless the call names one, as ``engine.Whisper`` does."""
    calls = []
    model, mp = _per_item_model(m, calls)
    oracle = m["oracle"]
    engine = model.model
    base_encode = engine.encode
    seeds = iter(range(10**6))
    turn = iter(range(10**6))

    def pick(replica):
        return next(turn) % n_replicas if replica is None else replica

    def encode(features, to_cpu=False, replica=None):
        tracker.encodes += 1
        sv = base_encode(features, to_cpu)
        sv.replica = pick(replica)
        return sv

    def encode_audio(chunks, return_features=False, replica=None):
        feats = np.stack([orc.pad_or_trim(orc.log_mel(c, m["dims"].n_mels)[:, :-1]) for c in chunks])
        sv = encode(ct2_shim.StorageView.from_array(np.ascontiguousarray(feats)), replica=replica)
        return (sv, feats) if return_features else sv

    def split_encoded(sv):
        parts = [ct2_shim.StorageView(tensor=sv.tensor[i : i + 1].clone()) for i in range(sv.shape[0])]
        for p in parts:
            p.replica = sv.replica
            tracker.born(p)
        return parts

    def align_items(pairs, start_sequence, text_tokens, num_frames, median_filter_width=7):
        calls.append(("align_items", list(start_sequence), len(pairs)))
        return [oracle.align(sv.tensor[i : i + 1], start_sequence, [t], [nf], median_filter_width)[0]
                for (sv, i), t, nf in zip(pairs, text_tokens, num_frames)]

    def decode_queue(slots=0, replica=0, **kw):
        return FakeQueue(oracle, tracker, slots, next(seeds), pick(replica), **kw)

    engine.encode = encode
    engine.encode_audio = encode_audio
    engine.split_encoded = split_encoded
    engine.align_items = align_items
    engine.decode_queue = decode_queue
    return model, mp, calls


@pytest.fixture(scope="module")
def en(micro):
    tracker = Tracker()
    model, mp, calls = _continuous_model(micro, tracker)
    yield model, tracker, calls
    mp.undo()


@pytest.fixture(scope="module")
def en_two_replicas(micro):
    tracker = Tracker()
    model, mp, calls = _continuous_model(micro, tracker, n_replicas=2)
    yield model, tracker, calls
    mp.undo()


@pytest.fixture(scope="module")
def ml(micro_ml):
    tracker = Tracker()
    model, mp, calls = _continuous_model(micro_ml, tracker)
    yield model, tracker, calls
    mp.undo()


def _check(model, tracker, audios, kw, clips=None):
    """Continuous equals the group path for transcribe_many and for transcribe of each file; every session is closed and the
    per-chunk encodings alive stay below 3 x slots."""
    group, cont = T.BatchedInferencePipeline(model), T.BatchedInferencePipeline(model, continuous_batching=True)
    tracker.reset()
    got = cont.transcribe_many([a.copy() for a in audios], clip_timestamps=clips, **kw)
    want = group.transcribe_many([a.copy() for a in audios], clip_timestamps=clips, **kw)
    assert got == want
    assert cont.last_speech_timestamp == 0.0
    for i, a in enumerate(audios):
        segs, info = cont.transcribe(a.copy(), clip_timestamps=clips[i] if clips else None, **kw)
        wsegs, winfo = group.transcribe(a.copy(), clip_timestamps=clips[i] if clips else None, **kw)
        assert (list(segs), info) == (list(wsegs), winfo), f"file {i}"
    assert all(q.closed for q in tracker.sessions)
    assert tracker.live == 0
    if tracker.slots:
        assert tracker.peak < 3 * min(tracker.slots), (tracker.peak, tracker.slots)
    return got


@pytest.mark.parametrize("batch_size", [1, 2, 40, 64])
def test_clips_and_whole_files(en, batch_size):
    """Files of 0 s, 3 s and 29 s transcribed whole, a 95 s file through user clips (one of them 41 s long).  With beam 2 a
    session has 40 slots: batch sizes below, at and above it."""
    model, tracker, _ = en
    audios = _files([0, 3.0, 29.0, 95.0], seed=300)
    clips = [None, None, None, [{"start": 0.0, "end": 41.0}, {"start": 41.0, "end": 70.0}, {"start": 75.0, "end": 95.0}]]
    got = _check(model, tracker, audios, dict(COMMON, language="en", vad_filter=False, batch_size=batch_size), clips)
    assert got[0][0] == [] and all(len(segs) > 0 for segs, _ in got[1:])


def test_fewer_slots_than_batch_size(en):
    """Beam 16: 5 slots, so batches of 5 chunks are encoded although batch_size is 8; 14 chunks pass through them."""
    model, tracker, _ = en
    audios = [_files([60.0], seed=305)[0]]
    clips = [[{"start": 4.0 * i, "end": 4.0 * i + 3.5} for i in range(14)]]
    _check(model, tracker, audios, dict(COMMON, beam_size=16, language="en", batch_size=8, max_new_tokens=3), clips)
    assert tracker.slots and set(tracker.slots) == {5}


@pytest.fixture
def seeded_vad():
    w = silero_oracle.synthetic_weights(3)
    vad.set_vad_model(lambda a: silero_oracle.probs(w, a))
    yield
    vad.set_vad_model(None)


def test_vad_files(en, seeded_vad):
    model, tracker, _ = en
    _check(model, tracker, _files([0, 3.0, 29.0, 95.0], seed=310), dict(COMMON, language="en", batch_size=3))


def test_word_timestamps(en):
    model, tracker, calls = en
    audios = _files([3.0, 29.0, 12.0, 20.0], seed=320)
    calls.clear()
    got = _check(model, tracker, audios, dict(COMMON, language="en", vad_filter=False, batch_size=2, word_timestamps=True,
                                              max_new_tokens=10))
    assert any(seg.words for segs, _ in got for seg in segs)
    assert any(c[0] == "align_items" for c in calls)


@pytest.mark.parametrize("word_timestamps", [False, True])
def test_multilingual_with_detected_languages(ml, word_timestamps):
    """Two 9 s files the micro multilingual model puts in different languages, a 35 s file in two clips; multilingual=True also
    detects the language of every chunk."""
    model, tracker, _ = ml
    audios = [_files([9.0], seed=0)[0], 0.01 * _files([9.0], seed=0)[0], _files([35.0], seed=1)[0]]
    clips = [None, None, [{"start": 0.0, "end": 20.0}, {"start": 20.0, "end": 35.0}]]
    kw = dict(COMMON, vad_filter=False, batch_size=3, word_timestamps=word_timestamps, language_detection_segments=2)
    got = _check(model, tracker, audios, kw, clips)
    assert got[0][1].language != got[1][1].language
    _check(model, tracker, audios, dict(kw, language="en", multilingual=True), clips)


def test_max_new_tokens(en):
    model, tracker, _ = en
    _check(model, tracker, _files([3.0, 29.0, 12.0], seed=340), dict(COMMON, language="en", vad_filter=False, batch_size=2,
                                                                        max_new_tokens=2))


def test_no_speech_creates_no_session(en):
    model, tracker, _ = en
    tracker.reset()
    pipe = T.BatchedInferencePipeline(model, continuous_batching=True)
    segs, info = pipe.transcribe(np.zeros(0, np.float32), language="en", vad_filter=False)
    assert list(segs) == [] and info.duration == 0
    assert pipe.transcribe_many([np.zeros(0, np.float32)] * 2, language="en", vad_filter=False)[0][0] == []
    assert tracker.sessions == [] and tracker.encodes == 0


def _many_clips():
    audio = _files([70.0], seed=350)[0]
    return audio, [{"start": 5.0 * i, "end": 5.0 * i + 4.0} for i in range(12)]


def test_transcribe_is_lazy(en):
    """The first segment comes before the last batch is encoded: 12 clips in batches of 2 chunks."""
    model, tracker, _ = en
    audio, clips = _many_clips()
    tracker.reset()
    segs, _ = T.BatchedInferencePipeline(model, continuous_batching=True).transcribe(
        audio, clip_timestamps=clips, language="en", batch_size=2, **COMMON)
    assert tracker.sessions == []
    first = next(iter(segs))
    assert first.id == 1 and len(tracker.sessions) == 1
    assert tracker.encodes < 6
    rest = list(segs)
    assert tracker.encodes == 6 and tracker.sessions[0].closed and rest


def test_sessions_close_on_close_and_on_error(en):
    model, tracker, _ = en
    audio, clips = _many_clips()
    pipe = T.BatchedInferencePipeline(model, continuous_batching=True)
    tracker.reset()
    segs, _ = pipe.transcribe(audio, clip_timestamps=clips, language="en", batch_size=2, **COMMON)
    next(segs)
    assert not tracker.sessions[0].closed
    segs.close()
    assert tracker.sessions[0].closed and pipe.last_speech_timestamp == 0.0
    assert tracker.live == 0
    tracker.reset(fail_after=2)
    segs, _ = pipe.transcribe(audio, clip_timestamps=clips, language="en", batch_size=2, **COMMON)
    with pytest.raises(RuntimeError, match="injected"):
        list(segs)
    assert tracker.sessions[0].closed
    tracker.reset(fail_after=1)
    with pytest.raises(RuntimeError, match="injected"):
        pipe.transcribe_many([audio], clip_timestamps=[clips], language="en", batch_size=2, **COMMON)
    assert tracker.sessions[0].closed


@pytest.mark.parametrize("long_clip", [False, True])
def test_two_replicas(en_two_replicas, long_clip):
    """A model with two replicas (several GPUs, or num_workers=2): each call decodes on one replica, and every batch it encodes,
    through the fused path or the features of a clip longer than 30 s, lands on that replica (a queue takes only its own
    replica's encoder outputs).  Calls take the replicas in turn."""
    model, tracker, _ = en_two_replicas
    audio, clips = _many_clips()
    if long_clip:
        clips = [{"start": 0.0, "end": 41.0}] + clips[9:]
    kw = dict(COMMON, language="en", batch_size=2)
    tracker.reset()
    got = list(T.BatchedInferencePipeline(model, continuous_batching=True).transcribe(audio, clip_timestamps=clips, **kw)[0])
    got2 = list(T.BatchedInferencePipeline(model, continuous_batching=True).transcribe(audio, clip_timestamps=clips, **kw)[0])
    want = list(T.BatchedInferencePipeline(model).transcribe(audio, clip_timestamps=clips, **kw)[0])
    assert got == want == got2
    assert sorted(q.replica for q in tracker.sessions) == [0, 1]
