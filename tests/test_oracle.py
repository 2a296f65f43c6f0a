"""CPU: the oracle against the reference's own outputs (golden fixtures made by oracle/make_golden.py and recorded through
oracle/refload.py), plus internal consistency of its search code."""
import hashlib
import os

import numpy as np
import pytest

from conftest import fake_logits_numpy
from faster_whisper_b200.synthetic import synthetic_audio
from oracle import whisper_oracle as orc

GOLD = os.path.join(os.path.dirname(__file__), "golden")


@pytest.fixture(scope="module")
def mel_gold():
    return np.load(os.path.join(GOLD, "mel_golden.npz"))


@pytest.mark.parametrize("n_mels", [80, 128])
def test_log_mel_matches_reference_goldens(mel_gold, n_mels):
    for n in (0, 159, 160, 4000, 48000):
        want = mel_gold[f"synth_{n_mels}_{n}"]
        got = orc.log_mel(synthetic_audio(5, n / 16000.0), n_mels)
        assert got.shape == want.shape and got.dtype == np.float32
        # bit-identical on the NumPy the fixtures were made with (2.3); 1e-6 leaves room for another pocketfft build
        assert np.abs(got - want).max() <= 1e-6
    got = orc.log_mel(mel_gold["speech_pcm_head"], n_mels)
    assert np.abs(got - mel_gold[f"speech_head_{n_mels}"]).max() <= 1e-6


def _digest(a):
    a = np.ascontiguousarray(a)
    return [str(a.dtype), list(a.shape), hashlib.sha256(a.tobytes()).hexdigest()]


def test_log_mel_matches_reference_live():
    """The reference's FeatureExtractor (mel filters and log-mel of four clip lengths) against the oracle, bit for bit: dtype, shape
    and SHA-256 of the reference's arrays are stored in tests/golden/reference_golden.json.gz (oracle/refload.py records them).  The
    digests pin the NumPy the goldens were recorded with (stored beside them): under another NumPy a changed FFT or rounding shows
    here even if the oracle is still right — re-record against the reference tree then."""
    from oracle.refload import RecordedReference, load_reference

    rec = RecordedReference(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_golden.json.gz"))
    fw = load_reference() if rec.record else None
    note = "goldens recorded under NumPy %s, running %s" % (rec.get("log_mel/numpy_version", lambda: np.__version__), np.__version__)
    for nm in (80, 128):
        fe = fw.feature_extractor.FeatureExtractor(feature_size=nm) if fw else None
        assert _digest(orc.mel_filters(n_mels=nm)) == rec.get(f"log_mel/filters_{nm}", lambda: _digest(fe.mel_filters)), note
        for n in (1, 161, 30000, 480000):
            x = synthetic_audio(9, n / 16000.0)
            assert _digest(orc.log_mel(x, nm)) == rec.get(f"log_mel/{nm}_{n}", lambda: _digest(fe(x))), note


def test_pad_or_trim():
    a = np.ones((3, 10), np.float32)
    assert orc.pad_or_trim(a, 12).shape == (3, 12) and orc.pad_or_trim(a, 12)[:, 10:].sum() == 0
    assert orc.pad_or_trim(a, 4).shape == (3, 4)


def _oracle(micro):
    return micro["oracle"], micro["tokens"]


def test_beam1_equals_greedy_on_fake_logits(micro):
    o, st = _oracle(micro)
    fl = fake_logits_numpy(micro["dims"].n_vocab, st.timestamp_begin, st.eot)
    prompts = [[st.sot, st.no_timestamps, 5]]
    g = o.generate(None, prompts, fake_logits=fl, beam_size=1, max_length=40)[0]
    assert 0 < len(g.sequences_ids[0]) <= 37
    # score is cumulative log-prob / len (EOS excluded from len) when length_penalty = 1
    g0 = o.generate(None, prompts, fake_logits=fl, beam_size=1, max_length=40, length_penalty=0.0)[0]
    assert g0.sequences_ids == g.sequences_ids
    assert abs(g0.scores[0] / len(g.sequences_ids[0]) - g.scores[0]) < 1e-5


def test_timestamp_rules_hold(micro):
    o, st = _oracle(micro)
    fl = fake_logits_numpy(micro["dims"].n_vocab, st.timestamp_begin, st.eot)
    for beam in (1, 5):
        specials = list(range(st.eot + 1, st.timestamp_begin))  # language/task tokens are not covered by the rules themselves
        for r in o.generate(None, [[st.sot, 11], [st.sot, 12]], fake_logits=fl, beam_size=beam, max_length=80,
                            max_initial_timestamp_index=25, suppress_tokens=specials):
            toks = r.sequences_ids[0]
            ts0 = st.timestamp_begin
            assert ts0 <= toks[0] <= ts0 + 25  # first sampled token is a timestamp within the initial window
            stamps = [t for t in toks if t >= ts0]
            assert stamps == sorted(stamps)  # never decreasing
            assert st.no_timestamps not in toks
            for i in range(1, len(toks) - 1):  # a lone timestamp is followed by a timestamp (pairs)
                if toks[i] >= ts0 and toks[i - 1] < ts0:
                    assert toks[i + 1] >= ts0


def test_suppress_and_ngram_and_repetition(micro):
    o, st = _oracle(micro)
    fl = fake_logits_numpy(micro["dims"].n_vocab, st.timestamp_begin, st.eot)
    base = o.generate(None, [[st.sot, st.no_timestamps, 3]], fake_logits=fl, beam_size=1, max_length=30)[0].sequences_ids[0]
    banned = base[:3]
    r = o.generate(None, [[st.sot, st.no_timestamps, 3]], fake_logits=fl, beam_size=1, max_length=30, suppress_tokens=banned)[0]
    assert not set(banned) & set(r.sequences_ids[0])
    r = o.generate(None, [[st.sot, st.no_timestamps, 3]], fake_logits=fl, beam_size=3, max_length=60, no_repeat_ngram_size=1)[0]
    assert len(set(r.sequences_ids[0])) == len(r.sequences_ids[0])


def test_sampling_is_seeded(micro):
    o, st = _oracle(micro)
    fl = fake_logits_numpy(micro["dims"].n_vocab, st.timestamp_begin, st.eot)
    kw = dict(fake_logits=fl, beam_size=1, num_hypotheses=3, sampling_topk=0, sampling_temperature=0.8, max_length=20)
    a = o.generate(None, [[st.sot, st.no_timestamps]], seed=7, **kw)[0]
    b = o.generate(None, [[st.sot, st.no_timestamps]], seed=7, **kw)[0]
    c = o.generate(None, [[st.sot, st.no_timestamps]], seed=8, **kw)[0]
    assert a.sequences_ids == b.sequences_ids and a.sequences_ids != c.sequences_ids
    assert a.scores == sorted(a.scores, reverse=True) and len(a.sequences_ids) == 3


# ---- Whisper.align helpers ---------------------------------------------------------------------------------------------------
def test_median_filter_matches_scipy_mirror():
    from scipy.ndimage import median_filter as sp_median

    rng = np.random.default_rng(0)
    x = rng.standard_normal((3, 5, 40))
    for w in (3, 7):
        assert np.array_equal(orc.median_filter(x, w), sp_median(x, size=(1, 1, w), mode="mirror"))
    assert np.array_equal(orc.median_filter(x[..., :3], 7), x[..., :3])  # shorter than the padding: unchanged


def test_dtw_is_optimal_and_monotone():
    import itertools

    rng = np.random.default_rng(1)
    for n, m in ((2, 3), (3, 4), (4, 4)):
        cost = rng.standard_normal((n, m))
        ti, fi = orc.dtw(cost)
        assert (ti[0], fi[0]) == (0, 0) and (ti[-1], fi[-1]) == (n - 1, m - 1)
        steps = set(zip(np.diff(ti).tolist(), np.diff(fi).tolist()))
        assert steps <= {(1, 1), (1, 0), (0, 1)}
        got = cost[ti, fi].sum()
        # brute force over all monotone paths
        best = np.inf
        moves = [(1, 1), (1, 0), (0, 1)]
        for length in range(max(n, m) - 1, n + m - 1):
            for seq in itertools.product(moves, repeat=length):
                i = j = 0
                tot = cost[0, 0]
                ok = True
                for di, dj in seq:
                    i, j = i + di, j + dj
                    if i >= n or j >= m:
                        ok = False
                        break
                    tot += cost[i, j]
                if ok and (i, j) == (n - 1, m - 1):
                    best = min(best, tot)
        assert abs(got - best) < 1e-9


def test_align_shapes_and_probabilities(micro):
    o, st = micro["oracle"], micro["tokens"]
    feats = np.stack([orc.pad_or_trim(orc.log_mel(synthetic_audio(3, 30.0), micro["dims"].n_mels)[:, :-1])])
    text = [[1000, 1001, 1002, 1003, 1004]]
    res = o.align(o.encode(feats), [st.sot], text, 3000, 7)[0]
    ti = np.array([p[0] for p in res.alignments])
    fi = np.array([p[1] for p in res.alignments])
    assert ti[0] == 0 and ti[-1] == len(text[0]) and fi[0] == 0 and fi[-1] == 1499  # rows predict text + eot
    assert (np.diff(ti) >= 0).all() and (np.diff(fi) >= 0).all()
    assert len(res.text_token_probs) == len(text[0]) and all(0.0 <= p <= 1.0 for p in res.text_token_probs)


def test_greedy_rows_report_the_margin_of_every_step(micro):
    """The GPU parity tests accept a divergence only where the oracle's own top-1 / top-2 gap AT THAT STEP is a near-tie: greedy rows
    carry one gap per generated token, their minimum is min_margin; beam search has no per-step list."""
    o, st = micro["oracle"], micro["tokens"]
    rng = np.random.default_rng(5)
    feats = rng.standard_normal((2, micro["dims"].n_mels, 3000)).astype(np.float32) * 0.1
    enc = o.encode(feats)
    res = o.generate(enc, [[st.sot, st.no_timestamps]] * 2, beam_size=1, max_length=14, suppress_tokens=[st.eot])
    for r in res:
        assert r.step_margins is not None and len(r.step_margins) == len(r.sequences_ids[0]) == r.steps
        assert all(m >= 0 for m in r.step_margins) and abs(min(r.step_margins) - r.min_margin) < 1e-12
    res = o.generate(enc, [[st.sot, st.no_timestamps]] * 2, beam_size=3, max_length=10)
    assert all(r.step_margins is None for r in res)
