"""Whisper.align on the device: the cost-matrix and DTW kernels against float64 restatements (bit for bit), the batched entry point
against the oracle and against per-item b2w_align, and word timestamps of the batched pipeline.  The argument checks run without
a GPU."""
import ctypes as C

import numpy as np
import pytest

from faster_whisper_b200 import engine
from oracle import whisper_oracle as orc
from test_gpu_engine import _check_align, features_for, make_engine


# ---- float64 restatement of the cost matrix: sums in the order of sequential loops (np.mean's pairwise sums differ) ---------
def cost_reference(cap: np.ndarray, n_start: int, n_text: int, width: int) -> np.ndarray:
    n_heads, n_tok, nf = cap.shape
    acc = np.zeros((n_text + 1, nf))
    for h in range(n_heads):
        a = cap[h].astype(np.float64)
        mu = np.zeros(nf)
        for t in range(n_tok):
            mu = mu + a[t]
        mu = mu / n_tok
        var = np.zeros(nf)
        for t in range(n_tok):
            d = a[t] - mu
            var = var + d * d
        sd = np.sqrt(var / n_tok)
        w = (a[n_start : n_start + n_text + 1] - mu) / sd
        acc = acc + orc.median_filter(w, width)  # a selection: np.sort of each window
    return -acc / n_heads


def random_capture(rng, n_heads, n_tok, nf):
    """Softmax-like rows over the frames; every (head, frame) column varies over the tokens (a single frame is not normalised:
    it would be 1 for every token)."""
    x = np.exp(rng.standard_normal((n_heads, n_tok, nf)).astype(np.float32) * 2)
    return (x / (x.sum(axis=-1, keepdims=True) if nf > 1 else x.max())).astype(np.float32)


@pytest.mark.gpu
@pytest.mark.parametrize("n_heads,n_tok,nf,width", [
    (1, 448, 1500, 7), (6, 40, 1, 7), (6, 40, 3, 7), (6, 40, 4, 7), (6, 40, 4, 3), (6, 100, 750, 3), (6, 60, 750, 1),
    (6, 20, 1, 1), (320, 160, 1500, 7), (320, 24, 3, 3)])
def test_cost_kernel_matches_float64_restatement_bit_for_bit(n_heads, n_tok, nf, width):
    rng = np.random.default_rng(n_heads * 7 + n_tok + nf + width)
    cap = random_capture(rng, n_heads, n_tok, nf)
    n_start = 3
    n_text = n_tok - n_start - 2
    got = engine.debug_align_cost(cap, n_start, n_text, width)
    want = cost_reference(cap, n_start, n_text, width)
    assert got.shape == want.shape
    assert np.array_equal(got.view(np.int64), want.view(np.int64)), np.abs(got - want).max()


@pytest.mark.gpu
@pytest.mark.parametrize("N,M,kind", [(1, 1, "rand"), (1, 40, "rand"), (40, 1, "rand"), (60, 20, "rand"), (60, 20, "ties"),
                                      (20, 300, "ties"), (7, 9, "zeros"), (449, 1500, "rand"), (449, 1500, "ties")])
def test_dtw_kernel_matches_reference_path(N, M, kind):
    rng = np.random.default_rng(N * 1000 + M)
    if kind == "rand":
        cost = rng.standard_normal((N, M))
    elif kind == "ties":  # small integers: equal accumulated costs everywhere, so every branch of the tie rule is taken
        cost = rng.integers(0, 3, (N, M)).astype(np.float64)
    else:
        cost = np.zeros((N, M))
    ti, fi = orc.dtw(cost)
    assert engine.debug_dtw(cost) == list(zip(ti.tolist(), fi.tolist()))


# ---- the entry points ------------------------------------------------------------------------------------------------------
def _align_batch_raw(eng, enc, start, texts, frames, capacity=None, width=7):
    """b2w_align_batch with the caller's own buffers (capacity in pairs); returns per-item (pairs, probs)."""
    rep = eng._replica_for(enc)
    B = len(texts)
    offsets = np.zeros(B + 1, np.int32)
    offsets[1:] = np.cumsum([len(t) for t in texts])
    toks = np.ascontiguousarray(np.concatenate([np.asarray(t, np.int32) for t in texts] + [np.zeros(1, np.int32)]), np.int32)
    frames = np.ascontiguousarray(frames, np.int32)
    need = sum(len(t) + 1 + max(1, min(1500, f // 2)) for t, f in zip(texts, frames) if len(t))
    cap = need if capacity is None else capacity
    pairs = np.zeros((max(1, cap), 2), np.int32)
    poff = np.zeros(B + 1, np.int32)
    probs = np.zeros(max(1, int(offsets[-1])), np.float32)
    start = np.ascontiguousarray(start, np.int32)
    engine._check(rep._lib.b2w_align_batch(rep.handle, enc._handle, engine._ptr(start), len(start), engine._ptr(toks), engine._ptr(offsets),
                                           engine._ptr(frames), width, engine._ptr(pairs), cap, engine._ptr(poff), engine._ptr(probs)))
    return [(pairs[poff[b]:poff[b + 1]].tolist(), probs[offsets[b]:offsets[b + 1]].tolist()) for b in range(B)]


def _align_one(eng, enc, b, start, text, frames, width=7):
    rep = eng._replica_for(enc)
    start = np.ascontiguousarray(start, np.int32)
    toks = np.ascontiguousarray(text, np.int32)
    cap = len(text) + frames // 2 + 2
    pairs = np.zeros((cap, 2), np.int32)
    probs = np.zeros(max(1, len(text)), np.float32)
    n = C.c_int32(0)
    engine._check(rep._lib.b2w_align(rep.handle, enc._handle, b, engine._ptr(start), len(start), engine._ptr(toks), len(text), frames, width,
                                     engine._ptr(pairs), cap, C.byref(n), engine._ptr(probs)))
    return pairs[: n.value].tolist(), probs[: len(text)].tolist()


@pytest.fixture(scope="module")
def eng_ml(micro_ml):
    return make_engine(micro_ml)


def _close_boundaries(a, b, n_rows):
    from test_gpu_engine import _jump_frames

    ja, jb = _jump_frames(a, n_rows), _jump_frames(b, n_rows)
    return sum(abs(x - y) <= 2 for x, y in zip(ja, jb)) >= n_rows - 1


@pytest.mark.gpu
def test_single_item_batch_equals_b2w_align(micro_ml, eng_ml):
    """One item through b2w_align_batch runs the same passes as b2w_align: identical pairs and probabilities."""
    st = micro_ml["tokens"]
    start = [st.sot, st.lang_begin, st.transcribe]
    rng = np.random.default_rng(11)
    for b, (n_text, frames) in enumerate([(14, 3000), (120, 2400), (1, 7)]):
        enc = eng_ml.encode(features_for(micro_ml, 1, seed=70 + b))
        text = rng.integers(100, 5000, n_text).tolist()
        (batch,) = _align_batch_raw(eng_ml, enc, start, [text], [frames])
        assert batch == _align_one(eng_ml, enc, 0, start, text, frames)


@pytest.mark.gpu
@pytest.mark.parametrize("heads", [None, [(1, 0), (1, 1), (0, 1)]])
def test_batched_align_matches_oracle_and_per_item(micro_ml, eng_ml, heads):
    """Items of different text lengths and frame counts, one with no text and one of 125 positions (longer than a pass)."""
    st = micro_ml["tokens"]
    feats = features_for(micro_ml, 5, seed=80)
    rng = np.random.default_rng(5)
    text = [rng.integers(100, 5000, n).tolist() for n in (14, 0, 120, 3, 40)]
    frames = [3000, 2000, 3000, 900, 2500]
    start = [st.sot, st.lang_begin, st.transcribe]
    keep = [b for b in range(5) if text[b]]
    _check_align(eng_ml, micro_ml, feats[keep], start, [text[b] for b in keep], [frames[b] for b in keep], heads)
    eng_ml.set_alignment_heads(heads)
    try:
        enc = eng_ml.encode(feats)
        got = eng_ml.align(enc, start, text, frames)
        assert got[1].alignments == [] and got[1].text_token_probs == []
        for b in keep:
            pairs, probs = _align_one(eng_ml, enc, b, start, text[b], frames[b])
            assert _close_boundaries(got[b].alignments, pairs, len(text[b]) + 1)
            assert np.allclose(got[b].text_token_probs, probs, rtol=1e-2, atol=1e-6)
    finally:
        eng_ml.set_alignment_heads(None)


@pytest.mark.gpu
def test_batched_align_over_several_groups(micro_ml, eng_ml):
    """83 items of short text: several forced-decoding groups, the first of them holding many chunks."""
    st = micro_ml["tokens"]
    base = features_for(micro_ml, 4, seed=90)
    feats = base[np.arange(83) % 4]
    rng = np.random.default_rng(9)
    text = [rng.integers(100, 5000, 2 + (b * 7) % 30).tolist() for b in range(83)]
    frames = [3000 - 20 * (b % 50) for b in range(83)]
    start = [st.sot, st.lang_begin, st.transcribe]
    enc = eng_ml.encode(feats)
    got = eng_ml.align(enc, start, text, frames)
    o = micro_ml["oracle"]
    pick = [0, 1, 2, 3, 40, 79, 80, 81, 82]
    want = o.align(o.encode(base[[b % 4 for b in pick]]), start, [text[b] for b in pick], [frames[b] for b in pick])
    for k, b in enumerate(pick):
        assert _close_boundaries(got[b].alignments, want[k].alignments, len(text[b]) + 1), b
        gi = np.array(got[b].alignments)
        assert gi[0].tolist() == [0, 0] and gi[-1].tolist() == [len(text[b]), frames[b] // 2 - 1]
        pairs, _ = _align_one(eng_ml, enc, b, start, text[b], frames[b])
        assert _close_boundaries(got[b].alignments, pairs, len(text[b]) + 1), b


@pytest.mark.gpu
def test_batched_align_rejects_bad_arguments(micro_ml, eng_ml):
    st = micro_ml["tokens"]
    enc = eng_ml.encode(features_for(micro_ml, 2, seed=95))
    start = [st.sot, st.lang_begin, st.transcribe]
    text = [[500, 600, 700], [800]]
    with pytest.raises(ValueError, match="odd"):
        _align_batch_raw(eng_ml, enc, start, text, [3000, 3000], width=4)
    with pytest.raises(ValueError, match="odd"):
        _align_batch_raw(eng_ml, enc, start, text, [3000, 3000], width=0)
    with pytest.raises(ValueError, match="too small"):
        _align_batch_raw(eng_ml, enc, start, text, [3000, 3000], capacity=100)
    with pytest.raises(ValueError, match="token id out of range"):
        _align_batch_raw(eng_ml, enc, start, [[500, micro_ml["dims"].n_vocab], [800]], [3000, 3000])
    with pytest.raises(ValueError, match="decoder context"):
        _align_batch_raw(eng_ml, enc, start, [[500] * 446, [800]], [3000, 3000])
    rep = eng_ml._replica_for(enc)
    offs = np.array([0, 3, 2], np.int32)  # decreasing
    toks = np.array([500, 600, 700], np.int32)
    s = np.array(start, np.int32)
    buf = np.zeros((4000, 2), np.int32)
    with pytest.raises(ValueError, match="text_offsets"):
        engine._check(rep._lib.b2w_align_batch(rep.handle, enc._handle, engine._ptr(s), 3, engine._ptr(toks), engine._ptr(offs),
                                               engine._ptr(np.array([3000, 3000], np.int32)), 7, engine._ptr(buf), 4000,
                                               engine._ptr(np.zeros(3, np.int32)), engine._ptr(np.zeros(3, np.float32))))


@pytest.mark.gpu
def test_large_v3_geometry_batched_align_matches_oracle():
    """Synthetic large-v3 (32 decoder layers x 20 heads: 320 default alignment heads), two chunks aligned in one call."""
    import os

    import torch

    from faster_whisper_b200.config import MODEL_DIMS, special_tokens
    from faster_whisper_b200.synthetic import make_weights, synthetic_audio

    torch.set_num_threads(min(16, os.cpu_count() or 1))
    dims = MODEL_DIMS["large-v3"]
    st = special_tokens(dims.n_vocab)
    w = make_weights(dims, seed=0)
    m = dict(dims=dims, weights=w, tokens=st, oracle=orc.WhisperOracle(dims.to_dict(), w, st.to_dict()))
    e = engine.Whisper(dims=dims, weights=w, tokens=st, device="cuda")
    feats = np.stack([orc.pad_or_trim(orc.log_mel(synthetic_audio(i, 30.0), dims.n_mels)[:, :-1]) for i in range(2)])
    rng = np.random.default_rng(21)
    text = [rng.integers(100, 20000, 30).tolist(), rng.integers(100, 20000, 12).tolist()]
    _check_align(e, m, feats, [st.sot, st.lang_begin, st.transcribe], text, [3000, 2200])


@pytest.mark.gpu
def test_batched_pipeline_word_timestamps_match_per_item_align(micro_ml):
    """BatchedInferencePipeline(word_timestamps=True), 4 clips: words within their clips, and the same words (within 40 ms, all but
    one per segment) as a run whose model.align is a per-item loop of b2w_align."""
    import json

    from faster_whisper_b200 import BatchedInferencePipeline, WhisperModel
    from faster_whisper_b200.synthetic import make_tokenizer, synthetic_audio

    dims = micro_ml["dims"]
    files = {"tokenizer.json": make_tokenizer(dims.n_vocab).to_str().encode(),
             "preprocessor_config.json": json.dumps({"feature_size": dims.n_mels}).encode()}
    model = WhisperModel("synthetic", device="cuda", files=files, dims=dims, weights=micro_ml["weights"])
    lens = [30.0, 20.0, 30.0, 12.0]
    audio = np.concatenate([synthetic_audio(100 + i, n) for i, n in enumerate(lens)])
    edges = np.concatenate([[0.0], np.cumsum(lens)])
    clips = [{"start": float(a), "end": float(b)} for a, b in zip(edges[:-1], edges[1:])]
    kw = dict(batch_size=4, vad_filter=False, clip_timestamps=clips, language="en", beam_size=2, max_new_tokens=12, word_timestamps=True)

    def run():
        segs, _ = BatchedInferencePipeline(model).transcribe(audio, **kw)
        return list(segs)

    segs = run()
    words = [w for s in segs for w in (s.words or [])]
    assert len(words) > 0
    for w in words:
        assert w.start <= w.end and any(c["start"] - 1e-6 <= w.start and w.end <= c["end"] + 1e-6 for c in clips), (w.start, w.end)

    inner = model.model
    batched = inner.align

    def per_item(features, start_sequence, text_tokens, num_frames, median_filter_width=7):
        enc = inner._as_encoded(features)
        out = []
        for b, toks in enumerate(text_tokens):
            nf = int(num_frames[b] if isinstance(num_frames, (list, tuple)) else num_frames)
            pairs, probs = _align_one(inner, enc, b, list(start_sequence), list(toks), nf, median_filter_width)
            out.append(engine.WhisperAlignmentResult([tuple(p) for p in pairs], probs))
        return out

    inner.align = per_item
    try:
        ref = run()
    finally:
        inner.align = batched
    assert [s.text for s in segs] == [s.text for s in ref]
    for s, r in zip(segs, ref):
        ws, wr = s.words or [], r.words or []
        assert [w.word for w in ws] == [w.word for w in wr]
        off = sum(abs(a.start - b.start) > 0.04 or abs(a.end - b.end) > 0.04 for a, b in zip(ws, wr))
        assert off <= 1, [(a.start, a.end, b.start, b.end) for a, b in zip(ws, wr)]


# ---- argument checks: no device is touched, so these run anywhere --------------------------------------------------------------
def test_align_hooks_reject_bad_arguments():
    cap = np.full((2, 10, 8), 0.125, np.float32)
    for width in (0, -1, 2, 8):
        with pytest.raises(ValueError, match="odd"):
            engine.debug_align_cost(cap, 3, 5, width)
    with pytest.raises(ValueError, match="kept rows"):
        engine.debug_align_cost(cap, 3, 7, 7)  # rows 3..10 of 10 tokens
    with pytest.raises(ValueError, match="nf must be"):
        engine.debug_align_cost(np.zeros((1, 4, 1501), np.float32), 0, 1, 7)
    with pytest.raises(ValueError, match="too small"):
        engine.debug_dtw(np.zeros((4, 5)), capacity=8)
    with pytest.raises(ValueError, match="rows x"):
        engine.debug_dtw(np.zeros((450, 5)))
    with pytest.raises(ValueError, match="rows x"):
        engine.debug_dtw(np.zeros((4, 1501)))
