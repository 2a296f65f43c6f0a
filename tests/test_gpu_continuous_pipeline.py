"""-m gpu: per-chunk encoder outputs (``Whisper.split_encoded``), alignment over items of several encoder outputs
(``Whisper.align_items``), the encoder-output memory counter, and ``BatchedInferencePipeline(continuous_batching=True)``.

Split items are bit-identical to their batch's items, and decode and align bit-identically at the same shape.  The pipeline is
checked against the same host code over the oracle shim with the criteria of tests/test_gpu_many_files.py (tokens, seeks and times
exact unless the oracle reports a near-tie, avg_logprob / no_speech within 5e-3), and at the large-v3 geometry against the group
path, with the live encoder outputs bounded by 3 x slots chunks."""
import gc
import json
import os

import numpy as np
import pytest

from faster_whisper_b200 import engine
from faster_whisper_b200 import transcribe as T
from faster_whisper_b200.synthetic import make_tokenizer, synthetic_audio
from oracle import whisper_oracle as orc
from test_gpu_decode_queue import LOGIT_TOL, features_for, make_engine, prompts_for
from test_gpu_many_files import _compare, _models, _oracle_per_file

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def large_v3():
    import torch

    from faster_whisper_b200.config import MODEL_DIMS, special_tokens
    from faster_whisper_b200.synthetic import make_weights

    torch.set_num_threads(min(16, os.cpu_count() or 1))
    dims = MODEL_DIMS["large-v3"]
    st = special_tokens(dims.n_vocab)
    w = make_weights(dims, seed=0)
    return dict(dims=dims, weights=w, tokens=st)


def _geometry(request, which):
    return request.getfixturevalue(which)


def _xkv(eng, enc, prompt):
    """The cross-attention K/V of `enc` as the decoder reads it, [L][2][B][H][1500][64], after a one-step generate."""
    d = eng.dims
    B = enc.shape[0]
    eng.generate(enc, [prompt] * B, beam_size=1, max_length=len(prompt) + 1)
    n = d.n_text_layer * 2 * B * 1500 * d.n_text_state
    return eng.debug_fetch(11, n).reshape(d.n_text_layer, 2, B, d.n_text_head, 1500, 64)


@pytest.mark.parametrize("which", ["micro", "micro_ml", "large_v3"])
def test_split_items_are_bit_identical(request, which):
    m = _geometry(request, which)
    eng = make_engine(m)
    st = m["tokens"]
    B = 3
    d = m["dims"]
    enc = eng.encode(features_for(m, B, seed=7))
    prompt = [st.sot] + ([st.lang_begin, st.transcribe] if d.is_multilingual else []) + [st.no_timestamps]
    xkv = _xkv(eng, enc, prompt)  # the batch's cross-KV exists from here on
    mem0 = eng.memory()["encoded_bytes"]
    assert mem0 == B * 1500 * 2 * (d.n_audio_state + 2 * d.n_text_layer * d.n_text_state)
    parts = eng.split_encoded(enc)
    assert eng.memory()["encoded_bytes"] == 2 * mem0
    assert len(parts) == B and all(p.shape == [1, 1500, d.n_audio_state] for p in parts)
    host = enc.numpy()
    for b, p in enumerate(parts):
        assert np.array_equal(p.numpy().view(np.uint32), host[b : b + 1].view(np.uint32))
        assert np.array_equal(_xkv(eng, p, prompt).view(np.uint32), xkv[:, :, b : b + 1].view(np.uint32))
    # the same decode at the same shape: a queue over the batch's items and one over the split items
    prompts = prompts_for(m, B, timestamps=True, seed=3)
    caps = [len(p) + 12 for p in prompts]
    kw = dict(beam_size=5, return_scores=True, return_no_speech_prob=True, max_length=max(caps))
    q = eng.decode_queue(**kw)
    q.push(enc, prompts, caps)
    want = dict(q)
    q.close()
    q = eng.decode_queue(**kw)
    for p, pr, c in zip(parts, prompts, caps):
        q.push(p, [pr], [c])
    got = dict(q)
    q.close()
    for i in range(B):
        assert got[i].sequences_ids == want[i].sequences_ids and got[i].scores == want[i].scores
        assert got[i].no_speech_prob == want[i].no_speech_prob
    del parts, p, q
    gc.collect()
    assert eng.memory()["encoded_bytes"] == mem0
    # generate on a split item and on its batch at the same shape (one chunk).  Two generate calls on the same input need not
    # give the same last bits of their scores (the batch is decoded twice to show the size of that), so scores are compared
    # within 5e-3, the pipeline tests' tolerance; tokens exactly
    one = eng.encode(features_for(m, 1, seed=9))
    (part,) = eng.split_encoded(one)
    gkw = dict(beam_size=5, max_length=len(prompts[0]) + 12, return_scores=True, return_no_speech_prob=True)
    (w1,), (g1,), (w2,) = (eng.generate(x, prompts[:1], **gkw) for x in (one, part, one))
    print("%s: split item score %.7f, batch item %.7f and %.7f" % (which, g1.scores[0], w1.scores[0], w2.scores[0]))
    assert g1.sequences_ids == w1.sequences_ids == w2.sequences_ids
    assert abs(g1.scores[0] - w1.scores[0]) < 5e-3 and abs(g1.no_speech_prob - w1.no_speech_prob) < 5e-3
    del one, part
    gc.collect()
    del enc
    gc.collect()
    assert eng.memory()["encoded_bytes"] == 0


def _texts(m, n, seed):
    rng = np.random.default_rng(seed)
    return [rng.integers(100, 5000, int(k)).tolist() for k in rng.integers(0, 40, n)]


def test_align_items_over_split_items_is_bit_identical(micro_ml):
    eng = make_engine(micro_ml)
    st = micro_ml["tokens"]
    enc = eng.encode(features_for(micro_ml, 5, seed=20))
    parts = eng.split_encoded(enc)
    start = [st.sot, st.lang_begin, st.transcribe]
    text = _texts(micro_ml, 5, seed=1)
    text[0] = text[0] or [500, 600]
    frames = [3000, 2000, 3000, 900, 2500]
    want = eng.align(enc, start, text, frames)
    got = eng.align_items([(p, 0) for p in parts], start, text, frames)
    assert [(g.alignments, g.text_token_probs) for g in got] == [(w.alignments, w.text_token_probs) for w in want]


def test_align_items_over_three_encodings(micro_ml):
    """Items drawn from encodings of 1, 2 and 3 chunks, interleaved: each matches align on its own encoding (its group differs, so
    boundaries within 2 frames and probabilities within 1 %, as tests/test_gpu_align.py compares them)."""
    from test_gpu_align import _close_boundaries

    eng = make_engine(micro_ml)
    st = micro_ml["tokens"]
    encs = [eng.encode(features_for(micro_ml, n, seed=30 + 10 * n)) for n in (1, 2, 3)]
    pairs = [(2, 1), (0, 0), (1, 1), (2, 0), (1, 0), (2, 2)]
    start = [st.sot, st.lang_begin, st.transcribe]
    text = [t or [700] for t in _texts(micro_ml, len(pairs), seed=2)]
    frames = [3000 - 300 * j for j in range(len(pairs))]
    got = eng.align_items([(encs[k], i) for k, i in pairs], start, text, frames)
    for j, (k, i) in enumerate(pairs):
        mine = [jj for jj, (kk, _) in enumerate(pairs) if kk == k]
        order = {pairs[jj][1]: jj for jj in mine}
        own = eng.align(encs[k], start, [text[order[b]] for b in range(encs[k].shape[0])],
                        [frames[order[b]] for b in range(encs[k].shape[0])])[i]
        assert _close_boundaries(got[j].alignments, own.alignments, len(text[j]) + 1), j
        assert np.allclose(got[j].text_token_probs, own.text_token_probs, rtol=1e-2, atol=1e-6)


# ---- the pipeline ----------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def tiny_en():
    from faster_whisper_b200.config import MODEL_DIMS
    from faster_whisper_b200.synthetic import make_weights

    dims = MODEL_DIMS["tiny.en"]
    return _models(dims, make_weights(dims, seed=5))


def test_transcribe_more_clips_than_three_times_the_slots(tiny_en):
    """11 clips through 2 slots, with timestamps, suppress_tokens=[-1] and room to reach <|endoftext|>."""
    gpu, cpu, mp, margins = tiny_en
    audio = np.concatenate([synthetic_audio(600 + i, 6.0) for i in range(11)])
    clips = [[{"start": 6.0 * i, "end": 6.0 * i + 6.0} for i in range(11)]]
    kw = dict(beam_size=1, batch_size=2, vad_filter=False, language="en", without_timestamps=False, suppress_tokens=[-1],
              max_new_tokens=64, repetition_penalty=1.2, no_repeat_ngram_size=3)
    segs, info = T.BatchedInferencePipeline(gpu, continuous_batching=True).transcribe(audio.copy(), clip_timestamps=clips[0], **kw)
    got = [(list(segs), info)]
    want, file_margins = _oracle_per_file(cpu, mp, margins, [audio], clips, kw)
    assert len({s.seek for s in want[0][0]}) == 11
    _compare(got, want, file_margins)


def test_two_replicas_on_one_gpu(tiny_en):
    """num_workers=2 gives two replicas, which encode in turn: each call's batches are encoded on its queue's replica, and the
    segments are those of a one-replica model (tokens and times exact, avg_logprob within 5e-3)."""
    from faster_whisper_b200.config import MODEL_DIMS
    from faster_whisper_b200.synthetic import make_weights

    gpu = tiny_en[0]
    dims = MODEL_DIMS["tiny.en"]
    files = {"tokenizer.json": make_tokenizer(dims.n_vocab).to_str().encode(),
             "preprocessor_config.json": json.dumps({"feature_size": dims.n_mels}).encode()}
    two = T.WhisperModel("synthetic", device="cuda", files=files, dims=dims, weights=make_weights(dims, seed=5), num_workers=2)
    assert len(two.model._replicas) == 2
    audio = np.concatenate([synthetic_audio(650 + i, 6.0) for i in range(7)])
    clips = [{"start": 6.0 * i, "end": 6.0 * i + 6.0} for i in range(7)]
    kw = dict(beam_size=1, batch_size=2, vad_filter=False, language="en", clip_timestamps=clips, max_new_tokens=24)
    want = list(T.BatchedInferencePipeline(gpu, continuous_batching=True).transcribe(audio.copy(), **kw)[0])
    for _ in range(2):  # the second call takes the other replica
        got = list(T.BatchedInferencePipeline(two, continuous_batching=True).transcribe(audio.copy(), **kw)[0])
        assert [(s.tokens, s.start, s.end) for s in got] == [(s.tokens, s.start, s.end) for s in want]
        assert all(abs(g.avg_logprob - w.avg_logprob) < 5e-3 for g, w in zip(got, want))


@pytest.mark.parametrize("beam", [1, 5])
def test_transcribe_many(tiny_en, beam):
    gpu, cpu, mp, margins = tiny_en
    audios = [synthetic_audio(400 + i, s) for i, s in enumerate([3.0, 29.0, 12.0, 45.0, 20.0, 58.0])]
    clips = [None, None, None, [{"start": 0.0, "end": 30.0}, {"start": 30.0, "end": 45.0}], None,
             [{"start": 0.0, "end": 29.0}, {"start": 29.0, "end": 58.0}]]
    kw = dict(beam_size=beam, batch_size=3, vad_filter=False, language="en", max_new_tokens=24, repetition_penalty=1.2,
              no_repeat_ngram_size=3)
    got = T.BatchedInferencePipeline(gpu, continuous_batching=True).transcribe_many(audios, clip_timestamps=clips, **kw)
    want, file_margins = _oracle_per_file(cpu, mp, margins, audios, clips, kw)
    _compare(got, want, file_margins)


def test_word_timestamps_match_the_group_path(micro_ml):
    """The same words as the group path (within 40 ms, all but one per segment), as tests/test_gpu_align.py compares them."""
    dims = micro_ml["dims"]
    files = {"tokenizer.json": make_tokenizer(dims.n_vocab).to_str().encode(),
             "preprocessor_config.json": json.dumps({"feature_size": dims.n_mels}).encode()}
    model = T.WhisperModel("synthetic", device="cuda", files=files, dims=dims, weights=micro_ml["weights"])
    lens = [30.0, 20.0, 30.0, 12.0, 25.0]
    audio = np.concatenate([synthetic_audio(100 + i, n) for i, n in enumerate(lens)])
    edges = np.concatenate([[0.0], np.cumsum(lens)])
    clips = [{"start": float(a), "end": float(b)} for a, b in zip(edges[:-1], edges[1:])]
    kw = dict(batch_size=2, vad_filter=False, clip_timestamps=clips, language="en", beam_size=2, max_new_tokens=12,
              word_timestamps=True)
    segs = list(T.BatchedInferencePipeline(model, continuous_batching=True).transcribe(audio, **kw)[0])
    ref = list(T.BatchedInferencePipeline(model).transcribe(audio, **kw)[0])
    assert sum(len(s.words or []) for s in segs) > 0
    assert [s.text for s in segs] == [s.text for s in ref]
    for s, r in zip(segs, ref):
        ws, wr = s.words or [], r.words or []
        assert [w.word for w in ws] == [w.word for w in wr]
        off = sum(abs(a.start - b.start) > 0.04 or abs(a.end - b.end) > 0.04 for a, b in zip(ws, wr))
        assert off <= 1, [(a.start, a.end, b.start, b.end) for a, b in zip(ws, wr)]


def test_large_v3_geometry_pipeline(large_v3):
    """16 slots x beam 5 over 44 chunks: tokens as the group path's, exact unless the oracle reports a near-tie on a differing chunk;
    live encoder outputs (sampled after every push, when the batch's own output is already freed) at most 3 x 16 chunks."""
    dims, w, st = large_v3["dims"], large_v3["weights"], large_v3["tokens"]
    files = {"tokenizer.json": make_tokenizer(dims.n_vocab).to_str().encode(),
             "preprocessor_config.json": json.dumps({"feature_size": dims.n_mels}).encode()}
    model = T.WhisperModel("synthetic", device="cuda", files=files, dims=dims, weights=w)
    inner = model.model
    n = 44
    audio = np.concatenate([synthetic_audio(700 + i, 10.0) for i in range(n)])
    clips = [{"start": 10.0 * i, "end": 10.0 * i + 10.0} for i in range(n)]
    kw = dict(batch_size=16, beam_size=5, vad_filter=False, language="en", clip_timestamps=clips, without_timestamps=True,
              max_new_tokens=8, repetition_penalty=1.3, no_repeat_ngram_size=2)
    peak = [0]
    push = engine.DecodeQueue.push

    def recording_push(self, *a, **k):
        ids = push(self, *a, **k)
        peak[0] = max(peak[0], inner.memory()["encoded_bytes"])
        return ids

    engine.DecodeQueue.push = recording_push
    try:
        got = list(T.BatchedInferencePipeline(model, continuous_batching=True).transcribe(audio.copy(), **kw)[0])
    finally:
        engine.DecodeQueue.push = push
    want = list(T.BatchedInferencePipeline(model).transcribe(audio.copy(), **kw)[0])
    per_chunk = 1500 * 2 * (dims.n_audio_state + 2 * dims.n_text_layer * dims.n_text_state)
    print("peak encoded bytes %d = %.1f chunks" % (peak[0], peak[0] / per_chunk))
    assert 0 < peak[0] <= 3 * 16 * per_chunk
    assert len(got) == len(want) == n
    differ = [i for i in range(n) if got[i].tokens != want[i].tokens]
    print("chunks whose tokens differ:", differ)
    assert len(differ) <= 6
    if differ:
        o = orc.WhisperOracle(dims.to_dict(), w, st.to_dict())
        prompt = [st.sot, st.no_timestamps] if not dims.is_multilingual else [st.sot, st.lang_begin, st.transcribe, st.no_timestamps]
        sup = T.get_suppressed_tokens(T.Tokenizer(model.hf_tokenizer, True, task="transcribe", language="en"), [-1])
        for i in differ:
            chunk = audio[int(clips[i]["start"] * 16000) : int(clips[i]["end"] * 16000)]
            enc = o.encode(orc.pad_or_trim(orc.log_mel(chunk, dims.n_mels)[:, :-1])[None])
            r = o.generate(enc, [prompt], beam_size=5, max_length=len(prompt) + 8, suppress_tokens=list(sup), repetition_penalty=1.3,
                           no_repeat_ngram_size=2, return_scores=True)[0]
            assert r.min_margin < 2 * LOGIT_TOL, (i, r.min_margin)
    assert inner.memory()["encoded_bytes"] == 0
