"""-m gpu: compute_type="float8_float16", the encoder's linear layers as e4m3 wgmma GEMMs.

a. the e4m3 GEMM against float64 on the same codes and scales, for each encoder epilogue, and the same bits for every CTA count;
b. the row quantisers against the rule of oracle/fp8_oracle.py: bit for bit from fp16, and from the LayerNorm's fp32 values
   except where the float64 value sits on a rounding boundary within fp32 error;
c. the encoder against the fp8 oracle (same rule at the same points), with the error against the fp32 oracle printed;
d. a chunk's encoder output does not depend on the batch it is encoded in;
e. generate (beam 5) against the oracle decoding the fp8 oracle's encoder output; the batched pipeline end to end, its continuous
   path giving the group path's tokens.
"""
import json
import os

import numpy as np
import pytest
import torch

from faster_whisper_b200 import engine
from faster_whisper_b200.synthetic import make_tokenizer, synthetic_audio
from oracle import fp8_oracle as f8
from oracle import whisper_oracle as orc

pytestmark = pytest.mark.gpu

LOGIT_TOL = 0.05
CT = "float8_float16"


def make_engine(m, **kw):
    return engine.Whisper(dims=m["dims"], weights=m["weights"], tokens=m["tokens"], device="cuda", compute_type=CT, **kw)


def features_for(m, n_chunks, seed=0):
    return np.stack([orc.pad_or_trim(orc.log_mel(synthetic_audio(seed + i, 30.0), m["dims"].n_mels)[:, :-1]) for i in range(n_chunks)])


def rel_fro(a, b):
    return float(np.linalg.norm(a - b) / np.linalg.norm(b))


def fp8_oracle(m):
    return f8.FP8EncoderOracle(m["dims"].to_dict(), m["weights"], m["tokens"].to_dict())


# ---- a. GEMM ------------------------------------------------------------------------------------------------------
def _codes(rng, rows, K, spread):
    x = rng.standard_normal((rows, K)).astype(np.float32) * np.exp(spread * rng.standard_normal((rows, 1))).astype(np.float32)
    q, s = f8.quantize_rows(torch.from_numpy(x))
    return f8.codes_to_bytes(q), s.numpy(), q


GEMM_CASES = [(K, N, batch) for K, d in ((192, 192), (384, 384), (1280, 1280), (5120, 1280)) for N in (d, 3 * d, 4 * d)
              for batch in (1, 3, 16)]


@pytest.mark.parametrize("K,N,batch", GEMM_CASES)
def test_fp8_gemm_against_float64(K, N, batch):
    rng = np.random.default_rng(K * 7 + N + batch)
    rows = 1500 * batch
    a, sa, qa = _codes(rng, rows, K, 1.0)
    w, sw, qw = _codes(rng, N, K, 0.5)
    bias = rng.standard_normal(N).astype(np.float32)
    dev = torch.device("cuda")
    qa64, qw64 = qa.to(dev).double(), qw.to(dev).double()
    sa64, sw64 = torch.from_numpy(sa).to(dev).double()[:, None], torch.from_numpy(sw).to(dev).double()[None]
    ref = (qa64 @ qw64.T) * sa64 * sw64 + torch.from_numpy(bias).to(dev).double()
    mag = (qa64.abs() @ qw64.abs().T) * sa64 * sw64  # sum of |products| times the scales
    del qa64, qw64
    epilogues = [engine.EPI_F16, engine.EPI_GELU_F16, engine.EPI_RESID_F32] if batch == 3 else [[engine.EPI_F16, engine.EPI_GELU_F16, engine.EPI_RESID_F32][(K + N) % 3]]
    for epi in epilogues:
        if epi == engine.EPI_RESID_F32:
            resid = rng.standard_normal((rows, N)).astype(np.float32)
            out = resid.copy()
            want = ref + torch.from_numpy(resid).to(dev).double()
        else:
            out = np.zeros((rows, N), np.float16)
            want = ref if epi == engine.EPI_F16 else torch.nn.functional.gelu(ref)
        engine.debug_gemm_fp8(a, sa, w, sw, out, epilogue=epi, bias=bias)
        got = torch.from_numpy(out.astype(np.float32)).to(dev).double()
        # the output's own rounding (fp16 half an ulp, float32 residual add), then the accumulation error relative to sum |products|
        own = want.abs() * (2.0 ** -11 if epi != engine.EPI_RESID_F32 else 2.0 ** -23) + (2.0 ** -24 if epi != engine.EPI_RESID_F32 else 0)
        ratio = float(((got - want).abs() - own).clamp(min=0).div(mag + 1e-30).max())
        print("fp8 GEMM K=%d N=%d rows=%d epi=%d: worst |err| beyond output rounding / sum|products| = %.3g" % (K, N, rows, epi, ratio))
        # the tensor cores sum each 128-wide K block with fewer bits than fp32 (measured worst 2.5e-4 of sum |products| at
        # K = 192 on an H100 SXM); the blocks are added in fp32, so the bound does not grow with K
        assert ratio < 2.0 ** -11, ratio
        if batch == 3 or K == 5120:  # several tiles per CTA: the same bits
            for ctas in (1, 7, 61):
                o2 = out.copy() if epi != engine.EPI_RESID_F32 else resid.copy()
                if epi != engine.EPI_RESID_F32:
                    o2[:] = 0
                engine.debug_gemm_fp8(a, sa, w, sw, o2, epilogue=epi, bias=bias, max_ctas=ctas)
                assert np.array_equal(o2.view(np.uint8), out.view(np.uint8)), ctas


def test_fp8_gemm_checks_arguments():
    a, s = np.zeros((64, 96), np.uint8), np.ones(64, np.float32)
    with pytest.raises(ValueError, match="multiple of 64"):
        engine.debug_gemm_fp8(a, s, np.zeros((64, 96), np.uint8), s, np.zeros((64, 64), np.float16), epilogue=engine.EPI_F16)
    with pytest.raises(ValueError, match="epilogue"):
        engine.debug_gemm_fp8(np.zeros((64, 64), np.uint8), s, np.zeros((64, 64), np.uint8), s, np.zeros((64, 64), np.float32),
                              epilogue=engine.EPI_F32)


# ---- b. quantisers ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("K", [192, 768, 1280, 5120])
def test_quantize_rows_bit_exact(K):
    rng = np.random.default_rng(K)
    x = np.clip(rng.standard_normal((300, K)) * np.exp(3 * rng.standard_normal((300, 1))), -65000, 65000).astype(np.float16)
    x[7] = 0
    x[8, :5] = [60000, -60000, 1e-7, -3e-8, 0]
    got_q, got_s = engine.debug_quantize_e4m3(x)
    q, s = f8.quantize_rows(torch.from_numpy(x.astype(np.float32)))
    assert np.array_equal(got_s.view(np.uint32), s.numpy().view(np.uint32))
    assert np.array_equal(got_q, f8.codes_to_bytes(q))


GRID = np.unique(torch.arange(256, dtype=torch.uint8).view(torch.float8_e4m3fn).float().numpy())
GRID = GRID[np.isfinite(GRID)].astype(np.float64)
MIDS = (GRID[1:] + GRID[:-1]) / 2


@pytest.mark.parametrize("d", [192, 384, 1280])
def test_layernorm_e4m3(d):
    rng = np.random.default_rng(d)
    x = (rng.standard_normal((1500, d)) * 3 + rng.standard_normal((1500, 1))).astype(np.float32)
    g = (1 + 0.3 * rng.standard_normal(d)).astype(np.float32)
    b = (0.2 * rng.standard_normal(d)).astype(np.float32)
    got_q, got_s = engine.debug_layernorm_e4m3(x, g, b)
    x64 = x.astype(np.float64)
    mu, var = x64.mean(1, keepdims=True), x64.var(1, keepdims=True)
    y = (x64 - mu) / np.sqrt(var + 1e-5) * g + b
    s64 = np.abs(y).max(1) / 448
    assert np.abs(got_s / s64 - 1).max() < 1e-5
    r = y / got_s[:, None]
    want = f8.codes_to_bytes(f8.round_e4m3(torch.from_numpy(r.astype(np.float32))))
    diff = got_q != want
    # a differing code is only allowed where the exact value lies within fp32 error of a rounding boundary
    # (fp32 LayerNorm values carry an error of a few ulp of the row's largest value: 448 * 2^-20 in code units)
    near = np.abs(r[diff][:, None] - MIDS[None]).min(1) <= 448 * 2.0 ** -20 + 1e-5 * np.abs(r[diff]) if diff.any() else np.zeros(0, bool)
    print("LayerNorm e4m3 d=%d: %d of %d codes differ from the float64 rule, all at rounding boundaries: %s" % (d, diff.sum(), diff.size, bool(near.all())))
    assert near.all()
    assert diff.sum() <= 1e-3 * diff.size


# ---- c. encoder --------------------------------------------------------------------------------------------------------
# Bounds from the measured values (H100 SXM): max abs 0.149 / 0.137 / 0.212 and relative Frobenius 0.022 / 0.021 / 0.037 against
# the fp8 oracle for micro / micro_ml / large-v3.  A code that lands on the other side of a rounding boundary (fp32 LayerNorm sums,
# fp16 attention, the tensor cores' block sums) moves its element by up to one e4m3 step, and the residual stream carries that on;
# against the fp32 oracle the same outputs differ by 0.053 / 0.049 / 0.084.
def _encoder_case(name, m, eng, n_chunks, seed, max_abs, fro):
    feats = features_for(m, n_chunks, seed=seed)
    got = eng.encode(feats).numpy()
    want = fp8_oracle(m).encode(feats).numpy()
    fp32 = m["oracle"].encode(feats).numpy() if "oracle" in m else orc.WhisperOracle(m["dims"].to_dict(), m["weights"], m["tokens"].to_dict()).encode(feats).numpy()
    err = np.abs(got - want)
    print("%s fp8 encoder vs fp8 oracle: max abs %.4g, rel Frobenius %.4g; vs fp32 oracle (the precision cost): max abs %.4g, rel Frobenius %.4g"
          % (name, err.max(), rel_fro(got, want), np.abs(got - fp32).max(), rel_fro(got, fp32)))
    assert err.max() < max_abs and rel_fro(got, want) < fro


def test_encoder_micro(micro):
    _encoder_case("micro", micro, make_engine(micro), 2, 0, 0.2, 0.03)


def test_encoder_micro_ml(micro_ml):
    _encoder_case("micro_ml", micro_ml, make_engine(micro_ml), 3, 4, 0.2, 0.03)


def test_encoder_large_v3_geometry():
    from faster_whisper_b200.config import MODEL_DIMS, special_tokens
    from faster_whisper_b200.synthetic import make_weights

    torch.set_num_threads(min(16, os.cpu_count() or 1))
    dims = MODEL_DIMS["large-v3"]
    m = dict(dims=dims, weights=make_weights(dims, seed=0), tokens=special_tokens(dims.n_vocab))
    _encoder_case("large-v3", m, make_engine(m), 1, 0, 0.3, 0.05)


def test_ref_gemm_is_refused(micro):
    os.environ["B2W_GEMM_IMPL"] = "ref"
    try:
        with pytest.raises(ValueError, match="no fp8 path"):
            make_engine(micro)
    finally:
        os.environ.pop("B2W_GEMM_IMPL")


# ---- d. batch invariance ------------------------------------------------------------------------------------------------
def test_batch_invariance(micro_ml):
    eng = make_engine(micro_ml)
    feats = features_for(micro_ml, 16, seed=70)
    alone = eng.encode(feats[5:6]).numpy()[0]
    in3 = eng.encode(feats[4:7]).numpy()[1]
    in16 = eng.encode(feats).numpy()[5]
    assert np.array_equal(alone.view(np.uint32), in3.view(np.uint32))
    assert np.array_equal(alone.view(np.uint32), in16.view(np.uint32))


# ---- e. end to end -------------------------------------------------------------------------------------------------------
def test_generate_beam5_against_fp8_oracle(micro_ml):
    eng = make_engine(micro_ml)
    assert eng.compute_type == CT
    st = micro_ml["tokens"]
    feats = features_for(micro_ml, 4, seed=80)
    prompts = [[st.sot, st.lang_begin, st.transcribe, st.no_timestamps]] * 4
    o = fp8_oracle(micro_ml)
    kw = dict(beam_size=5, max_length=28, return_scores=True, return_no_speech_prob=True)
    want = o.generate(o.encode(feats), prompts, **kw)
    got = eng.generate(eng.encode(feats), prompts, **kw)
    exact = 0
    for w, g in zip(want, got):
        if g.sequences_ids[0] == w.sequences_ids[0]:
            exact += 1
            assert abs(g.scores[0] - w.scores[0]) < 0.05
        else:
            assert w.min_margin < 2 * LOGIT_TOL, (w.min_margin, g.sequences_ids[0][:12], w.sequences_ids[0][:12])
    print("fp8 generate beam 5: %d of %d chunks token-exact against the fp8 oracle" % (exact, len(want)))
    # unload / load rebuilds the replicas with the same compute type
    enc = eng.encode(feats[:1])
    before = eng.generate(enc, prompts[:1], beam_size=5, max_length=28)[0].sequences_ids
    eng.unload_model()
    eng.load_model()
    assert eng.compute_type == CT
    assert eng.generate(eng.encode(feats[:1]), prompts[:1], beam_size=5, max_length=28)[0].sequences_ids == before


def test_batched_pipeline_end_to_end(micro_ml):
    from faster_whisper_b200 import transcribe as T

    dims = micro_ml["dims"]
    files = {"tokenizer.json": make_tokenizer(dims.n_vocab).to_str().encode(),
             "preprocessor_config.json": json.dumps({"feature_size": dims.n_mels}).encode()}
    model = T.WhisperModel("synthetic", device="cuda", files=files, dims=dims, weights=micro_ml["weights"], compute_type=CT)
    assert model.model.compute_type == CT
    lens = [30.0, 20.0, 30.0, 12.0]
    audio = np.concatenate([synthetic_audio(200 + i, n) for i, n in enumerate(lens)])
    edges = np.concatenate([[0.0], np.cumsum(lens)])
    clips = [{"start": float(a), "end": float(b)} for a, b in zip(edges[:-1], edges[1:])]
    kw = dict(batch_size=2, vad_filter=False, clip_timestamps=clips, language="en", beam_size=5, max_new_tokens=12,
              without_timestamps=True)
    segs = list(T.BatchedInferencePipeline(model, continuous_batching=True).transcribe(audio.copy(), **kw)[0])
    ref = list(T.BatchedInferencePipeline(model).transcribe(audio.copy(), **kw)[0])
    assert len(segs) == len(clips)
    assert [s.tokens for s in segs] == [s.tokens for s in ref]
