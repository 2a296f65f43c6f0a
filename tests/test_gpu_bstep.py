"""-m gpu: the many-row persistent decode step (csrc/bstep.cu) as a decode LOOP against the CPU oracle, through the C ABI.

BatchedInferencePipeline's shape (reference faster_whisper/transcribe.py:222-236 driven by :580-617): one generate() call for
many chunks, R = chunks x beam rows per step.  Tokens must be identical to the oracle's unless the oracle itself reports a
near-tie (top-1/top-2 margin below twice the logit tolerance) — the margin is printed; scores within 0.05.
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


def compare(eng, m, feats, prompts, **kw):
    o = m["oracle"]
    want = o.generate(o.encode(feats), prompts, return_scores=True, return_no_speech_prob=True, **kw)
    got = eng.generate(eng.encode(feats), prompts, return_scores=True, return_no_speech_prob=True, **kw)
    exact = 0
    compare.first_divergence = []
    for i, (w, g) in enumerate(zip(want, got)):
        assert abs(g.no_speech_prob - w.no_speech_prob) < 5e-3 * max(1.0, w.no_speech_prob) + 1e-6
        if g.sequences_ids[0] == w.sequences_ids[0]:
            exact += 1
            assert abs(g.scores[0] - w.scores[0]) < 0.05, (i, g.scores[0], w.scores[0])
        else:
            first = next((j for j, (x, y) in enumerate(zip(g.sequences_ids[0], w.sequences_ids[0])) if x != y), -1)
            compare.first_divergence.append(first)
            if w.step_margins is not None and 0 <= first < len(w.step_margins):
                # greedy rows: the oracle's own top-1 / top-2 gap AT the step where the sequences part must be a near-tie
                print("chunk %d diverges at token %d, oracle margin at that step %.4f" % (i, first, w.step_margins[first]))
                assert w.step_margins[first] < 2 * LOGIT_TOL, (i, first, w.step_margins[first], g.sequences_ids[0][:12], w.sequences_ids[0][:12])
            else:
                print("chunk %d diverges at token %d, oracle min margin %.4f" % (i, first, w.min_margin))
                assert w.min_margin < 2 * LOGIT_TOL, (i, first, w.min_margin, g.sequences_ids[0][:12], w.sequences_ids[0][:12])
    return exact, len(want)


@pytest.mark.parametrize("n_chunks,beam", [(16, 5), (4, 5), (9, 2), (11, 1)])
def test_batched_decode_loop_matches_oracle(micro, n_chunks, beam):
    """R = 80 / 20 / 18 / 11 rows, >= 40 steps, repetition penalty + n-gram blocking so that tokens vary from step to step."""
    st = micro["tokens"]
    eng = make_engine(micro)
    feats = features_for(micro, n_chunks, seed=200)
    prompts = [[st.sot, st.no_timestamps]] * n_chunks
    exact, n = compare(eng, micro, feats, prompts, beam_size=beam, max_length=46, repetition_penalty=1.3, no_repeat_ngram_size=3,
                       suppress_tokens=[st.eot, st.sot, st.no_speech])
    # every divergence has already been checked to sit at a near-tie of the oracle (compare prints the margin); most chunks are exact
    assert 2 * exact >= n, (exact, n)


def test_batched_decode_multilingual_geometry(micro_ml):
    """d = 192 (the second 128-channel n-block is half empty), 3 heads, 3 layers, timestamps on, 16 x 5 rows."""
    st = micro_ml["tokens"]
    eng = make_engine(micro_ml)
    feats = features_for(micro_ml, 16, seed=300)
    prompts = [[st.sot, st.lang_begin + 1, st.transcribe]] * 16
    exact, n = compare(eng, micro_ml, feats, prompts, beam_size=5, max_length=44, repetition_penalty=1.2, no_repeat_ngram_size=2)
    assert 2 * exact >= n, (exact, n)


@pytest.mark.parametrize("n_chunks,beam", [(1, 5), (3, 1), (1, 1)])
def test_many_row_kernel_on_few_rows(micro_ml, n_chunks, beam):
    """B2W_STEP=bstep routes R <= 8 through the many-row kernel too (wgmma N = 16): same tokens as the oracle."""
    st = micro_ml["tokens"]
    eng = make_engine(micro_ml, B2W_STEP="bstep")
    feats = features_for(micro_ml, n_chunks, seed=310)
    prompts = [[st.sot_prev, 700, 701, st.sot, st.lang_begin, st.transcribe]] * n_chunks
    exact, n = compare(eng, micro_ml, feats, prompts, beam_size=beam, max_length=40, repetition_penalty=1.2, no_repeat_ngram_size=3)
    assert exact == n or n > 1


def test_many_row_kernel_matches_multikernel_path(micro):
    """Same call through the persistent kernel and through the layered multi-kernel step (B2W_STEP=layers)."""
    st = micro["tokens"]
    feats = features_for(micro, 6, seed=320)
    prompts = [[st.sot, st.no_timestamps]] * 6
    kw = dict(beam_size=5, max_length=30, return_scores=True, repetition_penalty=1.25, no_repeat_ngram_size=3, suppress_tokens=[st.eot])
    a = make_engine(micro, B2W_STEP="bstep")
    b = make_engine(micro, B2W_STEP="layers")
    ra = a.generate(a.encode(feats), prompts, **kw)
    rb = b.generate(b.encode(feats), prompts, **kw)
    same = sum(x.sequences_ids[0] == y.sequences_ids[0] for x, y in zip(ra, rb))
    assert same >= 5
    for x, y in zip(ra, rb):
        if x.sequences_ids[0] == y.sequences_ids[0]:
            assert abs(x.scores[0] - y.scores[0]) < 5e-3


@pytest.mark.parametrize("n_chunks,beam,late", [(2, 5, 64), (6, 1, 0)])
def test_many_row_kernel_long_context(micro_ml, n_chunks, beam, late):
    """236 steps: up to 15 sixteen-key blocks per self-attention task, double-buffer wrap-around, slot bytes of all eight 32-key
    groups; tokens vs the oracle.  Beam 5 on the micro model produces duplicate beams, i.e. exact ties (margin 0) whose resolution
    depends on the fp32 summation order of the split-K reductions, so there a divergence is only required to come late.  The six
    greedy rows are checked exactly: a row may part from the oracle only at a step where the oracle's own top-1 / top-2 gap is below
    twice the logit tolerance (compare() looks the gap up at that very step), and most rows must run the whole length identical."""
    st = micro_ml["tokens"]
    eng = make_engine(micro_ml, B2W_STEP="bstep")
    feats = features_for(micro_ml, n_chunks, seed=330)
    prompts = [[st.sot, st.lang_begin, st.transcribe, st.no_timestamps]] * n_chunks
    exact, n = compare(eng, micro_ml, feats, prompts, beam_size=beam, max_length=240, suppress_tokens=[st.eot], repetition_penalty=1.3, no_repeat_ngram_size=3)
    # a divergence (only ever at a near-tie of the oracle, checked in compare) must come late
    assert all(f >= late for f in compare.first_divergence), compare.first_divergence
    if beam == 1:
        assert 2 * exact >= n, (exact, n)


@pytest.mark.parametrize("n_chunks,beam,extra", [(2, 8, {}), (7, 5, dict(patience=2.0, length_penalty=0.6)), (5, 3, dict(num_hypotheses=2))])
def test_many_row_kernel_other_beam_shapes(micro, n_chunks, beam, extra):
    """8 rows per chunk (the cross-attention task's maximum), an odd number of chunks with patience / length penalty, several hypotheses."""
    st = micro["tokens"]
    eng = make_engine(micro)
    feats = features_for(micro, n_chunks, seed=340)
    prompts = [[st.sot_prev, 900, 901, st.sot]] * n_chunks  # timestamps on
    exact, n = compare(eng, micro, feats, prompts, beam_size=beam, max_length=40, repetition_penalty=1.2, no_repeat_ngram_size=3, **extra)
    assert 2 * exact >= n, (exact, n)


def test_repeated_batched_steps_are_bit_identical(micro_ml):
    """16 chunks x beam 5 = 80 rows through the many-row kernel, twice on the same inputs.  The split-K sums, the LayerNorm statistics
    and the prefill's residual GEMMs are reduced in a fixed order, so tokens, scores and the last step's residual stream, statistics and
    logits are the same bits every run (fp32 atomics let near-tied beams flip between runs of the benchmark)."""
    st, dims = micro_ml["tokens"], micro_ml["dims"]
    eng = make_engine(micro_ml)
    feats = features_for(micro_ml, 16, seed=60)
    prompts = [[st.sot, st.lang_begin, st.transcribe, st.no_timestamps]] * 16
    R, L = 16 * 5, dims.n_text_layer
    runs = []
    for _ in range(2):
        res = eng.generate(eng.encode(feats), prompts, beam_size=5, max_length=40, suppress_tokens=[st.eot], return_scores=True)
        bufs = [eng.debug_fetch(which, n) for which, n in ((0, R * dims.n_text_state), (7, 3 * L * R * 2), (8, R * dims.n_vocab))]
        runs.append(([r.sequences_ids[0] for r in res], [r.scores[0] for r in res], bufs))
    (t0, s0, b0), (t1, s1, b1) = runs
    assert t0 == t1 and s0 == s1
    for name, x, y in zip(("residual stream", "LayerNorm statistics", "logits"), b0, b1):
        assert np.array_equal(x, y), (name, np.abs(x - y).max())


def test_forced_step_runs_the_path_it_names(micro_ml, capfd):
    """B2W_STEP forces one decode-step path.  A shape the forced kernel cannot take is a ValueError, not a fallback.  Each setting
    runs what it names: with a prompt of [sot] there is no prefill, and a second generate() over the same encoder output computes
    no cross-attention K/V, so the launches counted per step are those of one step graph — O(L) kernels for the layered step, the
    same constant number for both persistent kernels, which tell themselves apart by the profile they print (B2W_DSTEP_PROF)."""
    st, L = micro_ml["tokens"], micro_ml["dims"].n_text_layer
    feats = features_for(micro_ml, 2, seed=350)
    kw = dict(beam_size=2, max_length=12, suppress_tokens=[st.eot])
    per_step = {}
    for path in ("dstep", "bstep", "layers"):
        eng = make_engine(micro_ml, B2W_STEP=path, B2W_DSTEP_PROF="1")
        if path == "dstep":
            with pytest.raises(ValueError):
                eng.generate(eng.encode(feats), [[st.sot]] * 2, beam_size=5, max_length=8)  # 2 chunks x beam 5 = 10 rows
        if path == "bstep":
            with pytest.raises(ValueError):
                eng.generate(eng.encode(feats), [[st.sot]] * 2, beam_size=9, max_length=8)  # 9 rows per chunk
        enc = eng.encode(feats[:1])
        eng.generate(enc, [[st.sot]], **kw)
        capfd.readouterr()
        eng.timing(reset=True)
        eng.generate(enc, [[st.sot]], **kw)
        t, err = eng.timing(), capfd.readouterr().err
        assert t["decode_steps"] > 0 and t["launches"] % t["decode_steps"] == 0, t
        per_step[path] = t["launches"] // t["decode_steps"]
        assert ("[dstep prof]" in err) == (path == "dstep") and ("[bstep prof]" in err) == (path == "bstep"), (path, err[:300])
    assert per_step["dstep"] == per_step["bstep"], per_step
    assert per_step["layers"] >= per_step["dstep"] + 8 * L, per_step  # per layer: 4 projections, 2 attentions, 2 FFN GEMMs
