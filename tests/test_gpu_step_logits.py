"""The decode-step kernels' logits at every step against the fp32 oracle, teacher-forced through Whisper.debug_step_logits.

The token-level tests accept a divergence wherever the oracle reports a near-tie, and random micro models have many, so they cannot
see a kernel whose logits are off by a few tenths on some rows.  Here every step of every row is compared, with no such escape.
debug_step_logits runs the step path generate() takes for the shape (B2W_STEP forces dstep_kernel, bstep_kernel or the layered
step) on forced tokens and a forced beam ancestry: at step t row (chunk b, slot k) feeds tokens[t, b, k] and continues the history
of slot parents[t, b, k] of its chunk.  The reference runs the oracle's decoder one position at a time over the engine's own encoder
output (only the decoder step is compared), reordering each chunk's self-attention cache by the same parents, as the oracle's beam
search does.  test_reference_matches_full_sequences checks that reference against single decoder_forward calls over every row's
full token sequence.

Bounds, for every step and row: max |logit - oracle| <= LOGIT_TOL (the suite's teacher-forced contract) and per step
||logits - oracle||_F / ||oracle||_F <= REL_FRO.  Different paths on the same inputs agree to within CROSS_TOL.  The oracle runs on
the fp32 weights.  Largest values measured on an H100 80GB HBM3 (700 W power limit), max |d| / relative Frobenius:

    micro     dstep 0.0131 / 6.2e-4   bstep 0.0148 / 6.1e-4   layers 0.0149 / 6.1e-4
    micro_ml  dstep 0.0134 / 6.6e-4   bstep 0.0132 / 6.4e-4   layers 0.0130 / 6.3e-4   (448-step and identity-parent cases included)
    wide      dstep 0.0120 / 6.2e-4   bstep 0.0134 / 6.3e-4
    int8      micro_ml dstep 0.0137 / 6.7e-4, bstep 0.0153 / 6.9e-4;  wide dstep 0.0178 / 9.1e-4, bstep 0.0197 / 9.1e-4
    path vs path: 0.0122 (micro, bstep vs layers); dstep vs bstep 0.0103
"""
import os

import numpy as np
import pytest
import torch

from faster_whisper_b200 import engine
from faster_whisper_b200.config import special_tokens
from faster_whisper_b200.synthetic import custom_dims, make_weights, synthetic_audio
from oracle import whisper_oracle as orc
from test_gpu_int8 import quantised_weights

LOGIT_TOL = 0.05
REL_FRO = 2e-3
CROSS_TOL = 0.02
STEPS = 24


def make_engine(m, compute_type="default", **env):
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        return engine.Whisper(dims=m["dims"], weights=m["weights"], tokens=m["tokens"], device="cuda", compute_type=compute_type)
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def features_for(m, n_chunks, seed=0):
    return np.stack([orc.pad_or_trim(orc.log_mel(synthetic_audio(seed + i, 30.0), m["dims"].n_mels)[:, :-1]) for i in range(n_chunks)])


def row_sequences(prompts, tokens, parents):
    """seqs[t, b, k, :P+t]: the tokens row (b, k) has seen at step t, i.e. prompt[:P-1] and then the forced token of each of its
    ancestors at steps 0..t (its own at t).  Later entries are -1.  parents None: every slot continues itself."""
    n_steps, n, K = tokens.shape
    P = prompts.shape[1]
    seqs = np.full((n_steps, n, K, P - 1 + n_steps), -1, np.int64)
    seqs[:, :, :, : P - 1] = prompts[None, :, None, : P - 1]
    for t in range(n_steps):
        if t:
            par = parents[t] if parents is not None else np.broadcast_to(np.arange(K), (n, K))
            seqs[t, :, :, P - 1 : P - 1 + t] = np.take_along_axis(seqs[t - 1, :, :, P - 1 : P - 1 + t], par[:, :, None], axis=1)
        seqs[t, :, :, P - 1 + t] = tokens[t]
    return seqs


@torch.no_grad()
def oracle_step_logits(o, enc, prompts, tokens, parents):
    """[n_steps, n, K, n_vocab] fp32 logits of the forced decode, one chunk at a time (its cross-attention K/V broadcast to its rows)."""
    n_steps, n, K = tokens.shape
    P = prompts.shape[1]
    out = np.empty((n_steps, n, K, o.n_vocab), np.float32)
    r2c = torch.zeros(K, dtype=torch.long)
    for b in range(n):
        xkv = o.cross_kv(torch.from_numpy(np.ascontiguousarray(enc[b : b + 1])).float())
        cache = [None] * o.dims["n_text_layer"]
        if P > 1:
            o.decoder_forward(torch.from_numpy(prompts[b : b + 1, : P - 1]).long(), 0, cache, xkv, r2c[:1])
            cache = [(k.expand(K, -1, -1), v.expand(K, -1, -1)) for k, v in cache]
        for t in range(n_steps):
            if t and parents is not None:
                idx = torch.from_numpy(parents[t, b]).long()
                cache = [(k[idx], v[idx]) for k, v in cache]
            lg = o.decoder_forward(torch.from_numpy(tokens[t, b][:, None]).long(), P - 1 + t, cache, xkv, r2c)
            out[t, b] = lg[:, 0].numpy()
    return out


def forced_inputs(st, n, K, n_steps, seed, prompt, random_parents=True):
    """Tokens from the whole vocabulary (every fourth one a timestamp), different in every row; random or identity parents."""
    rng = np.random.default_rng(seed)
    prompts = np.array([prompt] * n, np.int32)
    tokens = rng.integers(0, st.n_vocab, (n_steps, n, K)).astype(np.int32)
    ts = rng.random((n_steps, n, K)) < 0.25
    tokens[ts] = rng.integers(st.timestamp_begin, st.n_vocab, int(ts.sum()))
    parents = rng.integers(0, K, (n_steps, n, K)).astype(np.int32) if random_parents else None
    return prompts, tokens, parents


def prefix_prompt(st):
    return [st.sot_prev, 700, 701, st.sot, st.lang_begin, st.transcribe]


def check_against_oracle(got, want, label):
    """got, want [n_steps, rows, n_vocab]."""
    err = np.abs(got - want)
    rel = np.array([np.linalg.norm(got[t] - want[t]) / np.linalg.norm(want[t]) for t in range(got.shape[0])])
    worst = tuple(int(i) for i in np.unravel_index(err.argmax(), err.shape))
    max_err, max_rel = float(err.max()), float(rel.max())
    print("[step logits] %s max|d| %.5f at (step, row, token) %s, max rel_fro %.2e" % (label, max_err, worst, max_rel))
    assert max_err <= LOGIT_TOL, (label, "max |dlogit|", max_err, "at (step, row, token)", worst)
    assert max_rel <= REL_FRO, (label, "relative Frobenius", max_rel, "at step", int(rel.argmax()))


@pytest.fixture(scope="module")
def wide():
    """The large-v3 decoder layer (d = 1280, 20 heads, 51866 tokens) with 4 decoder layers: the kernels' shape-dependent code
    depends on d, heads, chunks, rows and vocabulary, not on the number of layers."""
    dims = custom_dims(name="wide", n_mels=128, d=1280, heads=20, enc_layers=1, dec_layers=4, n_vocab=51866)
    w = make_weights(dims, seed=13)
    st = special_tokens(dims.n_vocab)
    return dict(dims=dims, weights=w, tokens=st, oracle=orc.WhisperOracle(dims.to_dict(), w, st.to_dict()))


class Runs:
    """Engines per (model, path, compute type), features per (model, chunks) and oracles per (model, compute type), built once."""

    def __init__(self, request):
        self.request = request
        self.engines, self.feats, self.oracles = {}, {}, {}

    def model(self, name):
        return self.request.getfixturevalue(name)

    def engine(self, name, path, ct):
        key = (name, path, ct)
        if key not in self.engines:
            self.engines[key] = make_engine(self.model(name), compute_type=ct, B2W_STEP=path)
        return self.engines[key]

    def inputs(self, name, n, K, n_steps, long_context=False, random_parents=True):
        st = self.model(name)["tokens"]
        prompt = [st.sot] if long_context else prefix_prompt(st)
        return forced_inputs(st, n, K, n_steps, seed=1000 * n + 10 * K + random_parents, prompt=prompt, random_parents=random_parents)

    def run(self, name, path, n, K, n_steps=STEPS, ct="default", **kw):
        """(logits [n_steps, n, K, n_vocab], the engine's encoder output, (prompts, tokens, parents)) of one forced decode."""
        if (name, n) not in self.feats:
            self.feats[(name, n)] = features_for(self.model(name), n, seed=500 + n)
        eng = self.engine(name, path, ct)
        enc = eng.encode(self.feats[(name, n)])
        prompts, tokens, parents = self.inputs(name, n, K, n_steps, **kw)
        return eng.debug_step_logits(enc, prompts, tokens, parents), enc.numpy(), (prompts, tokens, parents)

    def oracle(self, name, ct):
        if (name, ct) not in self.oracles:
            m = self.model(name)
            self.oracles[(name, ct)] = m["oracle"] if ct == "default" else orc.WhisperOracle(
                m["dims"].to_dict(), quantised_weights(m["dims"], m["weights"]), m["tokens"].to_dict())
        return self.oracles[(name, ct)]


@pytest.fixture(scope="module")
def runs(request):
    return Runs(request)


def compare_with_oracle(runs, name, path, n, K, n_steps=STEPS, ct="default", **kw):
    got, enc, (prompts, tokens, parents) = runs.run(name, path, n, K, n_steps, ct, **kw)
    want = oracle_step_logits(runs.oracle(name, ct), enc, prompts, tokens, parents)
    assert got.shape == want.shape
    check_against_oracle(got.reshape(n_steps, n * K, -1), want.reshape(n_steps, n * K, -1), "%s %s %s n=%d K=%d %s" % (name, ct, path, n, K, kw))


DSTEP_SHAPES = [(1, 1), (1, 5), (1, 8), (2, 4), (8, 1), (3, 2)]
BSTEP_SHAPES = [(1, 1), (1, 5), (2, 5), (4, 4), (17, 1), (4, 8), (11, 3), (16, 4), (13, 5), (16, 5), (10, 8)]
LAYERS_SHAPES = [(16, 1), (17, 1), (6, 3), (5, 16), (16, 5), (1, 9)]
CASES = [("dstep",) + s for s in DSTEP_SHAPES] + [("bstep",) + s for s in BSTEP_SHAPES] + [("layers",) + s for s in LAYERS_SHAPES]


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["micro", "micro_ml"])
@pytest.mark.parametrize("path,n,K", CASES)
def test_step_logits_match_oracle(runs, name, path, n, K):
    """Rows 1-8 through dstep (K = 8 cross-attention queries), bstep's padded row counts on both sides of 16, 32, 64 and at 80
    with 1-8 rows per chunk, the layered step on both sides of its wgmma switch (17 rows) and with 9 and 16 rows per chunk (a second
    cross-attention query group of one row, two full groups)."""
    compare_with_oracle(runs, name, path, n, K)


@pytest.mark.gpu
@pytest.mark.parametrize("path,n,K", [("dstep", 1, 5), ("bstep", 4, 4), ("layers", 6, 3)])
def test_step_logits_identity_parents(runs, path, n, K):
    compare_with_oracle(runs, "micro_ml", path, n, K, random_parents=False)


@pytest.mark.gpu
@pytest.mark.parametrize("path,n,K", [("dstep", 1, 1), ("dstep", 1, 3), ("bstep", 2, 5), ("layers", 1, 2)])
def test_step_logits_long_context(runs, path, n, K):
    """Prompt [sot] and 448 steps: every position 0-447, i.e. dstep's third 192-key self-attention pass and bstep's 16-key
    blocks up to the 28th, over an ancestry table relinked at every step."""
    compare_with_oracle(runs, "micro_ml", path, n, K, n_steps=448, long_context=True)


@pytest.mark.gpu
@pytest.mark.parametrize("path,n,K", [("dstep", 1, 5), ("bstep", 2, 5), ("bstep", 16, 5)])
def test_step_logits_wide_geometry(runs, path, n, K):
    """d = 1280, 20 heads.  16 x 5 is the benchmark's shape: 2240 cross-attention tiles over 132 CTAs, whose runs of 17 tiles
    touch four (chunk, head) groups, the most the many-row kernel allows."""
    compare_with_oracle(runs, "wide", path, n, K, n_steps=6)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["micro_ml", "wide"])
@pytest.mark.parametrize("path,n,K", [("dstep", 1, 5), ("bstep", 16, 5)])
def test_int8_step_logits_match_quantised_oracle(runs, name, path, n, K):
    """compute_type int8_float16: the int8 weight atoms of both persistent kernels against the oracle on the de-quantised weights."""
    compare_with_oracle(runs, name, path, n, K, n_steps=STEPS if name != "wide" else 6, ct="int8_float16")


def paths_for(n, K):
    return [p for p, ok in (("dstep", n * K <= 8), ("bstep", K <= 8), ("layers", True)) if ok]


SHARED_SHAPES = sorted({(n, K) for _, n, K in CASES if len(paths_for(n, K)) > 1})


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["micro", "micro_ml"])
@pytest.mark.parametrize("n,K", SHARED_SHAPES)
def test_step_paths_agree(runs, name, n, K):
    """Every path that can take the shape, on the same inputs: closer to each other than to the oracle."""
    paths = paths_for(n, K)
    got = {p: runs.run(name, p, n, K)[0] for p in paths}
    for a, b in zip(paths, paths[1:]):
        d = float(np.abs(got[a] - got[b]).max())
        print("[step logits] %s n=%d K=%d %s vs %s max|d| %.5f" % (name, n, K, a, b, d))
        assert d <= CROSS_TOL, (name, n, K, a, b, d)


@pytest.mark.gpu
def test_step_hook_leaves_generate_unchanged(micro_ml):
    """generate() before and after the hook on the same engine, same shape (so the cached step graph is replayed): identical ids
    and scores.  bstep_kernel and the layered step reduce in a fixed order and must give the same bits.  dstep_kernel adds FFN2's
    K ranges with fp32 atomics, so its scores vary between any two runs (by up to 1.1e-4 here, measured on an H100)."""
    st = micro_ml["tokens"]
    for path in ("dstep", "bstep", "layers"):
        eng = make_engine(micro_ml, B2W_STEP=path)
        enc = eng.encode(features_for(micro_ml, 2, seed=610))
        kw = dict(beam_size=3, max_length=30, return_scores=True, suppress_tokens=[st.eot], repetition_penalty=1.2)
        prompts = [[st.sot, st.lang_begin, st.transcribe]] * 2
        before = eng.generate(enc, prompts, **kw)
        p, t, par = forced_inputs(st, 2, 3, 10, seed=611, prompt=prefix_prompt(st))
        eng.debug_step_logits(enc, p, t, par)
        after = eng.generate(enc, prompts, **kw)
        assert [r.sequences_ids for r in before] == [r.sequences_ids for r in after], path
        if path == "dstep":
            assert np.allclose([r.scores for r in before], [r.scores for r in after], rtol=0, atol=1e-3), path
        else:
            assert [r.scores for r in before] == [r.scores for r in after], path


@pytest.mark.gpu
def test_prefill_after_a_change_of_beam_size(micro_ml):
    """A prefill pass of >= 17 rows goes through the wgmma GEMM, whose QKV epilogue writes the K/V cache with the slot count,
    K cache and row table of its plan.  Plans were cached per (weights, activations, rows, mode) only, so after a call with 8 rows
    per chunk a 4-row call with the same prefill rows (4 chunks x 5 prompt positions) wrote its prompt keys 8 slots apart and the
    step kernels read them 4 apart.  The second call must give what a fresh engine gives."""
    st = micro_ml["tokens"]
    enc_feats = features_for(micro_ml, 4, seed=630)
    prompts = [prefix_prompt(st)] * 4
    kw = dict(max_length=24, return_scores=True, suppress_tokens=[st.eot])
    a = make_engine(micro_ml)
    a.generate(a.encode(enc_feats), prompts, beam_size=8, **kw)
    got = a.generate(a.encode(enc_feats), prompts, beam_size=4, **kw)
    b = make_engine(micro_ml)
    want = b.generate(b.encode(enc_feats), prompts, beam_size=4, **kw)
    assert [r.sequences_ids for r in got] == [r.sequences_ids for r in want]
    assert [r.scores for r in got] == [r.scores for r in want]


@pytest.mark.gpu
def test_step_hook_rejects_invalid_input(micro_ml):
    st, V, n_ctx = micro_ml["tokens"], micro_ml["dims"].n_vocab, micro_ml["dims"].n_text_ctx
    eng = make_engine(micro_ml)
    enc = eng.encode(features_for(micro_ml, 2, seed=620))
    p, t, par = forced_inputs(st, 2, 3, 4, seed=621, prompt=prefix_prompt(st))
    eng.debug_step_logits(enc, p, t, par)  # the valid call runs

    def bad(**kw):
        a = dict(enc=enc, prompts=p, tokens=t, parents=par)
        a.update(kw)
        with pytest.raises(ValueError):
            eng.debug_step_logits(**a)

    bad(enc=eng.encode(features_for(micro_ml, 1, seed=620)))  # e->B != n
    bad(prompts=p[:, :0])  # P = 0
    bad(tokens=np.zeros((4, 2, 0), np.int32), parents=None)  # K = 0
    bad(enc=eng.encode(features_for(micro_ml, 1, seed=620)), prompts=p[:1], tokens=np.zeros((2, 1, 17), np.int32), parents=None)  # K > 16
    bad(enc=eng.encode(features_for(micro_ml, 9, seed=620)), prompts=np.repeat(p[:1], 9, 0), tokens=np.zeros((2, 9, 9), np.int32), parents=None)  # 81 rows
    bad(tokens=np.zeros((n_ctx - p.shape[1] + 2, 2, 3), np.int32), parents=None)  # P - 1 + n_steps > n_text_ctx
    for arr, name, hi in ((p, "prompts", V), (t, "tokens", V), (par, "parents", 3)):
        for v in (-1, hi):
            x = arr.copy()
            x.flat[5] = v
            bad(**{name: x})
    forced = make_engine(micro_ml, B2W_STEP="dstep")
    with pytest.raises(ValueError):
        forced.debug_step_logits(forced.encode(features_for(micro_ml, 2, seed=620)), p, np.zeros((2, 2, 5), np.int32))  # 10 rows
    x = np.array([[st.sot, V]] * 2, np.int32)
    with pytest.raises(ValueError):
        eng.debug_logits(enc, x)


def test_row_sequences_three_step_beam():
    """Hand-worked: prompt [s0 s1 s2] (s2 is the prompt's last position, fed by step 0 instead), 2 slots, then the second chunk
    keeps identity ancestry."""
    prompts = np.array([[90, 91, 92], [80, 81, 82]], np.int32)
    tokens = np.array([[[10, 11], [40, 41]], [[20, 21], [50, 51]], [[30, 31], [60, 61]]], np.int32)
    parents = np.array([[[0, 0], [0, 1]], [[1, 0], [0, 1]], [[0, 0], [0, 1]]], np.int32)
    s = row_sequences(prompts, tokens, parents)
    assert s.shape == (3, 2, 2, 5)
    assert s[0, 0].tolist() == [[90, 91, 10, -1, -1], [90, 91, 11, -1, -1]]
    # step 1: slot 0 continues slot 1, slot 1 continues slot 0
    assert s[1, 0].tolist() == [[90, 91, 11, 20, -1], [90, 91, 10, 21, -1]]
    # step 2: both slots continue slot 0, whose history is [11, 20]
    assert s[2, 0].tolist() == [[90, 91, 11, 20, 30], [90, 91, 11, 20, 31]]
    assert s[2, 1].tolist() == [[80, 81, 40, 50, 60], [80, 81, 41, 51, 61]]
    assert np.array_equal(row_sequences(prompts, tokens, None)[:, 1], s[:, 1])


@pytest.mark.parametrize("P", [1, 4])
def test_reference_matches_full_sequences(P):
    """The incremental, cache-reordering reference equals one decoder_forward over every (step, row)'s full token sequence
    (row2chunk picking each chunk's encoder output; positions after a row's own are causally masked)."""
    dims = custom_dims(name="tiny", d=64, heads=1, enc_layers=1, dec_layers=2, n_vocab=51864)
    w = make_weights(dims, seed=5)
    st = special_tokens(dims.n_vocab)
    o = orc.WhisperOracle(dims.to_dict(), w, st.to_dict())
    enc = np.random.default_rng(6).standard_normal((2, 1500, 64)).astype(np.float32)
    prompts, tokens, parents = forced_inputs(st, 2, 3, 5, seed=7, prompt=prefix_prompt(st)[:P])
    got = oracle_step_logits(o, enc, prompts, tokens, parents)
    seqs = row_sequences(prompts, tokens, parents)
    n_steps, n, K, T = seqs.shape
    r2c = torch.from_numpy(np.broadcast_to(np.arange(n)[None, :, None], (n_steps, n, K)).reshape(-1).copy())
    with torch.no_grad():
        full = o.decoder_forward(torch.from_numpy(np.maximum(seqs, 0).reshape(-1, T)), 0, [None] * dims.n_text_layer,
                                 o.cross_kv(torch.from_numpy(enc)), r2c).numpy().reshape(n_steps, n, K, T, -1)
    want = np.stack([full[t, :, :, P - 1 + t] for t in range(n_steps)])
    assert np.abs(got - want).max() < 1e-3
