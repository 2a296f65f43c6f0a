"""-m gpu: the continuous-batching decode session (Whisper.decode_queue) against the oracle's generate.

Every item is compared with the oracle decoding that item alone (its own prompt and max_length): tokens exact unless the oracle
itself reports a near-tie (margin below twice the teacher-forced logit tolerance) at the first divergence, scores within 0.05,
no-speech probabilities within the tolerance of tests/test_gpu_engine.py.  Sampled items are compared with the oracle decoding all
of them as one batch: an item's noise is keyed by its id (push order) and its row, as a generate call keys it by the chunk index.
"""
import os

import numpy as np
import pytest

from faster_whisper_b200 import engine
from faster_whisper_b200.synthetic import synthetic_audio
from oracle import whisper_oracle as orc

pytestmark = pytest.mark.gpu

LOGIT_TOL = 0.05


def make_engine(m, **env):
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        return engine.Whisper(dims=m["dims"], weights=m["weights"], tokens=m["tokens"], device="cuda")
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def features_for(m, n_chunks, seed=0):
    return np.stack([orc.pad_or_trim(orc.log_mel(synthetic_audio(seed + i, 30.0), m["dims"].n_mels)[:, :-1]) for i in range(n_chunks)])


def prompts_for(m, n, timestamps, seed):
    """Per-item prompts of different lengths: optional previous text, the SOT sequence, and <|notimestamps|> when asked."""
    st = m["tokens"]
    rng = np.random.default_rng(seed)
    sot_seq = [st.sot] if not m["dims"].is_multilingual else [st.sot, st.lang_begin + int(rng.integers(0, 5)), st.transcribe]
    out = []
    for i in range(n):
        prev = [] if i % 3 == 0 else [st.sot_prev] + rng.integers(300, 3000, int(rng.integers(1, 9))).tolist()
        out.append(prev + sot_seq + ([] if timestamps else [st.no_timestamps]))
    return out


def run_queue(eng, enc, prompts, max_lengths, slots=0, **kw):
    q = eng.decode_queue(return_scores=True, return_no_speech_prob=True, slots=slots, **kw)
    ids = q.push(enc, prompts, max_lengths)
    assert ids == list(range(len(prompts)))
    assert q.pending() == len(prompts)
    got = dict(q)
    assert sorted(got) == ids and q.pending() == 0
    steps, live = q.counters()
    assert steps > 0 and live > 0
    q.close()
    return [got[i] for i in ids], q.slots


def compare(want, got):
    for w, g in zip(want, got):
        assert abs(g.no_speech_prob - w.no_speech_prob) < 5e-3 * max(1.0, w.no_speech_prob) + 1e-6
        if g.sequences_ids[0] == w.sequences_ids[0]:
            assert abs(g.scores[0] - w.scores[0]) < 0.05, (g.scores[0], w.scores[0])
        else:
            assert w.min_margin < 2 * LOGIT_TOL, (w.min_margin, g.sequences_ids[0][:12], w.sequences_ids[0][:12])


def oracle_per_item(m, feats, prompts, max_lengths, **kw):
    o = m["oracle"]
    enc = o.encode(feats)
    return [o.generate(enc[i : i + 1], [p], max_length=ml, return_scores=True, return_no_speech_prob=True, **kw)[0]
            for i, (p, ml) in enumerate(zip(prompts, max_lengths))]


# (model, step path, slots, beam, timestamps): 1 slot x 5 rows runs the <= 8-row kernel, 16 x 5 the many-row kernel, beam 9 and
# B2W_STEP=layers the layered step
CASES = [
    ("micro", None, 1, 5, False),
    ("micro", None, 4, 1, True),
    ("micro", None, 0, 5, True),
    ("micro_ml", None, 0, 5, False),
    ("micro_ml", None, 2, 1, False),
    ("micro_ml", None, 0, 9, True),
    ("micro_ml", "layers", 3, 5, False),
]


@pytest.mark.parametrize("model,path,slots,beam,timestamps", CASES)
def test_queue_matches_oracle(request, model, path, slots, beam, timestamps):
    m = request.getfixturevalue(model)
    eng = make_engine(m, **({"B2W_STEP": path} if path else {}))
    S = slots or 80 // beam
    n = max(3 * S, 6)  # every slot refilled at least twice
    feats = features_for(m, n, seed=100 + 7 * len(CASES) + beam)
    prompts = prompts_for(m, n, timestamps, seed=slots + beam)
    rng = np.random.default_rng(beam)
    # per-item caps: some a single generated token (max_length = P + 1), the rest 4 .. 40 new tokens
    max_lengths = [len(p) + (1 if i % 5 == 2 else int(rng.integers(4, 41))) for i, p in enumerate(prompts)]
    got, S_got = run_queue(eng, eng.encode(feats), prompts, max_lengths, slots=slots, beam_size=beam)
    assert S_got == S
    for g, p, ml in zip(got, prompts, max_lengths):
        assert len(g.sequences_ids[0]) <= ml - len(p)
    compare(oracle_per_item(m, feats, prompts, max_lengths, beam_size=beam), got)


def test_sampling_matches_oracle_and_is_slot_independent(micro):
    """best_of 5 sampling: 12 items through 2 slots, so most items land in whichever slot frees first; their draws must still be
    the oracle's for their id."""
    st = micro["tokens"]
    eng = make_engine(micro)
    n = 12
    feats = features_for(micro, n, seed=300)
    prompts = [[st.sot_prev, 500 + i, st.sot, st.no_timestamps] for i in range(n)]
    kw = dict(beam_size=1, num_hypotheses=5, sampling_topk=0, sampling_temperature=0.7, seed=99)
    got, _ = run_queue(eng, eng.encode(feats), prompts, [30] * n, slots=2, **kw)
    o = micro["oracle"]
    want = o.generate(o.encode(feats), prompts, max_length=30, return_scores=True, return_no_speech_prob=True, **kw)
    for w, g in zip(want, got):
        assert abs(g.no_speech_prob - w.no_speech_prob) < 5e-3 * max(1.0, w.no_speech_prob) + 1e-6
        same = [gs == ws for gs, ws in zip(g.sequences_ids, w.sequences_ids)]
        assert sum(same) >= 4 or w.min_margin < 2 * LOGIT_TOL, (same, w.min_margin)


def test_slot_hygiene_long_then_short(micro_ml):
    """One slot: a 60-token occupant, then a 3-token one, then a 20-token one in the same slot.  A stale self-KV entry, ancestry
    byte or history token from the previous occupant would change the next one's tokens."""
    m = micro_ml
    st = m["tokens"]
    eng = make_engine(m)
    feats = features_for(m, 3, seed=400)
    prompts = [[st.sot_prev, 900, 901, 902, 903, st.sot, st.lang_begin, st.transcribe, st.no_timestamps],
               [st.sot, st.lang_begin + 1, st.transcribe],
               [st.sot_prev, 77, st.sot, st.lang_begin + 2, st.transcribe]]
    max_lengths = [len(prompts[0]) + 60, len(prompts[1]) + 3, len(prompts[2]) + 20]
    got, _ = run_queue(eng, eng.encode(feats), prompts, max_lengths, slots=1, beam_size=5, suppress_tokens=[-1, st.eot])
    compare(oracle_per_item(m, feats, prompts, max_lengths, beam_size=5, suppress_tokens=[-1, st.eot]), got)


def test_queue_is_deterministic_and_interleaves_with_generate(micro):
    """The same pushes twice give bit-identical tokens and scores, also with a generate call on the same model between two runs
    of the session (the session's workspace is its own)."""
    st = micro["tokens"]
    eng = make_engine(micro)
    n = 20
    feats = features_for(micro, n, seed=500)
    prompts = prompts_for(micro, n, True, seed=5)
    max_lengths = [len(p) + 10 + (i % 7) * 5 for i, p in enumerate(prompts)]
    enc = eng.encode(feats)
    a, _ = run_queue(eng, enc, prompts, max_lengths, slots=3, beam_size=5)
    q = eng.decode_queue(return_scores=True, return_no_speech_prob=True, slots=3, beam_size=5)
    q.push(enc, prompts, max_lengths)
    del enc  # the session keeps the encoder output alive
    b = {}
    first = True
    for i, r in q:
        b[i] = r
        if first:
            eng.generate(eng.encode(features_for(micro, 2, seed=600)), [[st.sot]] * 2, beam_size=2, max_length=12)
            first = False
    q.close()
    for x, i in zip(a, range(n)):
        assert x.sequences_ids == b[i].sequences_ids and x.scores == b[i].scores and x.no_speech_prob == b[i].no_speech_prob


def test_queue_arguments(micro):
    st = micro["tokens"]
    eng = make_engine(micro)
    enc = eng.encode(features_for(micro, 1))
    q = eng.decode_queue(max_length=20)
    with pytest.raises(ValueError, match="startoftranscript"):
        q.push(enc, [[5, 6]])
    with pytest.raises(ValueError, match="max_length"):
        q.push(enc, [[st.sot]], [21])
    with pytest.raises(ValueError, match="max_length"):
        q.push(enc, [[st.sot, st.no_timestamps]], [2])
    with pytest.raises(ValueError):
        q.push(enc, [[st.sot], [st.sot]])
    assert q.run() == [] and q.pending() == 0
    q.close()


@pytest.mark.parametrize("slots", [1, 0])  # 1 slot x 5 rows: the <= 8-row kernel; 16 x 5: the many-row kernel
def test_slots_bound_to_different_encoder_outputs(micro_ml, slots):
    """Items from three encoder outputs of batch sizes 2, 5 and 1 share one queue, so a step's slots read different cross-KV
    buffers with different batch strides: each item must match the oracle on its own encoder output."""
    m = micro_ml
    eng = make_engine(m)
    sizes = [2, 5, 1]
    feats = [features_for(m, b, seed=700 + 10 * i) for i, b in enumerate(sizes)]
    q = eng.decode_queue(return_scores=True, return_no_speech_prob=True, slots=slots, beam_size=5)
    S = q.slots
    rounds = max(1, -(-3 * S // sum(sizes)))  # at least 3x the slots
    rng = np.random.default_rng(slots)
    pushed = []  # (feats index, item, prompt, max_length) in id order
    for r in range(rounds):
        for i, f in enumerate(feats):
            prompts = prompts_for(m, f.shape[0], bool(r % 2), seed=100 * r + i)
            mls = [len(p) + int(rng.integers(2, 30)) for p in prompts]
            q.push(eng.encode(f), prompts, mls)  # the session keeps each encoder output alive
            pushed += [(i, j, p, ml) for j, (p, ml) in enumerate(zip(prompts, mls))]
    got = dict(q)
    q.close()
    assert sorted(got) == list(range(len(pushed)))
    o = m["oracle"]
    encs = [o.encode(f) for f in feats]
    want = [o.generate(encs[i][j : j + 1], [p], max_length=ml, beam_size=5, return_scores=True, return_no_speech_prob=True)[0]
            for i, j, p, ml in pushed]
    compare(want, [got[k] for k in range(len(pushed))])


def test_refilled_slot_teacher_forced_logits(micro_ml):
    """Greedy, 2 slots: every step's logits of every item, including items that reuse a slot after a long occupant, against the
    oracle teacher-forced on the item's own prompt and tokens: <= 0.05 absolute at every step, no near-tie escape.  A stale
    self-KV entry or ancestry byte of the previous occupant shows here even when it would not flip a token."""
    import torch

    m = micro_ml
    st = m["tokens"]
    eng = make_engine(m)
    n = 8
    feats = features_for(m, n, seed=800)
    prompts = prompts_for(m, n, False, seed=8)
    max_lengths = [len(p) + (60 if i < 2 else 5 + 3 * i) for i, p in enumerate(prompts)]  # long first occupants, then shorter ones
    sup = [-1, st.eot]
    q = eng.decode_queue(slots=2, beam_size=1, suppress_tokens=sup)
    q.debug_record()
    q.push(eng.encode(feats), prompts, max_lengths)
    got = dict(q)
    o = m["oracle"]
    xkv = o.cross_kv(o.encode(feats))
    worst = 0.0
    for i in range(n):
        toks = got[i].sequences_ids[0]
        assert len(toks) == max_lengths[i] - len(prompts[i])  # <|endoftext|> suppressed: every item runs to its cap
        rec = q.debug_logits(i)
        assert rec.shape[0] >= len(toks)
        seq = np.asarray([prompts[i] + toks], np.int64)
        cache = [None] * m["dims"].n_text_layer
        want = o.decoder_forward(torch.from_numpy(seq), 0, cache, xkv, torch.tensor([i])).numpy()[0]
        P = len(prompts[i])
        err = np.abs(rec[: len(toks)] - want[P - 1 : P - 1 + len(toks)]).max()
        worst = max(worst, float(err))
        assert err <= LOGIT_TOL, (i, err)
    q.close()
    print("refilled-slot teacher-forced logits: worst abs error %.4g" % worst)


def test_large_v3_geometry_queue():
    """The bench's shape, 16 slots x beam 5, on large-v3 weights: 20 items (four chunks pushed five times, two caps), so four slots
    are refilled; tokens against the fp32 oracle, exact unless near-tie."""
    import torch

    from faster_whisper_b200.config import MODEL_DIMS, special_tokens
    from faster_whisper_b200.synthetic import make_weights

    torch.set_num_threads(min(16, os.cpu_count() or 1))
    dims = MODEL_DIMS["large-v3"]
    st = special_tokens(dims.n_vocab)
    w = make_weights(dims, seed=0)
    o = orc.WhisperOracle(dims.to_dict(), w, st.to_dict())
    e = engine.Whisper(dims=dims, weights=w, tokens=st, device="cuda")
    feats = np.stack([orc.pad_or_trim(orc.log_mel(synthetic_audio(40 + i, 30.0), dims.n_mels)[:, :-1]) for i in range(4)])
    prompt = [st.sot, st.lang_begin, st.transcribe, st.no_timestamps]
    sup = [st.eot, st.sot, st.transcribe, st.translate, st.sot_prev, st.sot_lm, st.no_speech]
    caps = [len(prompt) + 6, len(prompt) + 10]
    kw = dict(beam_size=5, suppress_tokens=sup, repetition_penalty=1.3, no_repeat_ngram_size=2)
    q = e.decode_queue(return_scores=True, return_no_speech_prob=True, **kw)
    assert q.slots == 16
    enc = e.encode(feats)
    pushed = []
    for r in range(5):
        q.push(enc, [prompt] * 4, [caps[r % 2]] * 4)
        pushed += [(j, caps[r % 2]) for j in range(4)]
    got = dict(q)
    q.close()
    enc_o = o.encode(feats)
    want = {(j, ml): o.generate(enc_o[j : j + 1], [prompt], max_length=ml, return_scores=True, return_no_speech_prob=True, **kw)[0]
            for j, ml in set(pushed)}
    compare([want[k] for k in pushed], [got[i] for i in range(len(pushed))])
