"""-m gpu: each CUDA kernel of the hot path against the CPU oracle / NumPy, through the C ABI.

Tolerances are stated per test.  Inputs are seeded; sizes are kept where the oracle finishes in seconds.
"""
import numpy as np
import pytest

from faster_whisper_b200 import engine
from faster_whisper_b200.synthetic import synthetic_audio
from oracle import whisper_oracle as orc

pytestmark = pytest.mark.gpu


def f16(x):
    return np.asarray(x, np.float32).astype(np.float16).astype(np.float32)


# ---- log-mel -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_mels", [80, 128])
@pytest.mark.parametrize("n", [0, 1, 159, 160, 161, 4000, 16000, 176000, 480000])
def test_logmel_matches_oracle(n_mels, n):
    x = synthetic_audio(5, n / 16000.0)
    want = orc.log_mel(x, n_mels)
    got = engine.log_mel(x, n_mels)
    assert got.shape == want.shape
    err = np.abs(got - want)
    # float32 DFT by direct summation vs pocketfft: agreement to ~1e-4 typical, 2e-3 at the clamp floor
    assert err.max() < 2e-3, (err.max(), err.mean())
    assert err.mean() < 1e-4, err.mean()


@pytest.mark.parametrize("n_mels", [80, 128])
def test_logmel_matches_reference_goldens(n_mels):
    """The CUDA front end against outputs of the REFERENCE's own FeatureExtractor (tests/golden/mel_golden.npz, made by
    oracle/make_golden.py from the first 3 s of tests/data/physicsworks.wav — real speech, not noise) and, beyond one chunk, against the
    oracle on a 47.3 s clip (the sequential path takes the log-mel of whole files with a whole-file clamp maximum)."""
    import os

    gold = np.load(os.path.join(os.path.dirname(__file__), "golden", "mel_golden.npz"))
    got = engine.log_mel(gold["speech_pcm_head"], n_mels)
    want = gold[f"speech_head_{n_mels}"]
    err = np.abs(got - want)
    assert got.shape == want.shape and err.max() < 2e-3 and err.mean() < 1e-4, (err.max(), err.mean())
    x = synthetic_audio(17, 47.3)
    got, want = engine.log_mel(x, n_mels), orc.log_mel(x, n_mels)
    err = np.abs(got - want)
    assert got.shape == want.shape == (n_mels, 1 + len(x) // 160) and err.max() < 2e-3 and err.mean() < 1e-4, (err.max(), err.mean())


def test_logmel_silence_and_impulse():
    z = np.zeros(16000, np.float32)
    got = engine.log_mel(z, 80)
    assert np.allclose(got, -1.5)
    imp = z.copy()
    imp[8000] = 1.0
    got, want = engine.log_mel(imp, 80), orc.log_mel(imp, 80)
    assert np.abs(got - want).max() < 2e-3


# ---- dense GEMM (wgmma) -------------------------------------------------------------------------------
@pytest.mark.parametrize("impl", [0, 1])
@pytest.mark.parametrize("shape", [(128, 128, 64), (300, 384, 128), (1500, 1280, 1280), (3001, 256, 192), (257, 5120, 320)])
def test_gemm_vs_numpy(impl, shape):
    M, N, K = shape
    rng = np.random.default_rng(M * 7 + N)
    a, w, b = rng.standard_normal((M, K), np.float32), rng.standard_normal((N, K), np.float32) / np.sqrt(K), rng.standard_normal(N).astype(np.float32)
    want = f16(a) @ f16(w).T + b
    got = engine.debug_gemm(a, w, b, impl=impl)
    assert np.abs(got - want).max() < 2e-3 * max(1.0, np.abs(want).max()), np.abs(got - want).max()


def test_gemm_gelu_epilogue():
    import math

    rng = np.random.default_rng(3)
    a, w, b = rng.standard_normal((200, 256), np.float32), rng.standard_normal((384, 256), np.float32) / 16, rng.standard_normal(384).astype(np.float32)
    y = f16(a) @ f16(w).T + b
    want = 0.5 * y * (1 + np.vectorize(math.erf)(y / math.sqrt(2)))
    got = engine.debug_gemm(a, w, b, impl=0, gelu=True)
    assert np.abs(got - want).max() < 4e-3


# ---- encoder attention (wgmma flash) ---------------------------------------------------------------------
@pytest.mark.parametrize("impl", [0, 1])
@pytest.mark.parametrize("T", [1500, 128, 77])
def test_attention_vs_numpy(impl, T):
    rng = np.random.default_rng(T)
    B, H = 2, 2
    qkv = rng.standard_normal((B, T, 3 * H * 64), np.float32)
    got = engine.debug_attention(qkv, H, impl=impl)
    x = f16(qkv).reshape(B, T, 3, H, 64)
    q, k, v = x[:, :, 0], x[:, :, 1], x[:, :, 2]
    s = np.einsum("bqhd,bkhd->bhqk", q, k) / 8.0
    p = np.exp(s - s.max(-1, keepdims=True))
    p /= p.sum(-1, keepdims=True)
    want = np.einsum("bhqk,bkhd->bqhd", p, v).reshape(B, T, H * 64)
    # fp16 probabilities and fp16 output rounding
    assert np.abs(got - want).max() < 6e-3, np.abs(got - want).max()


# ---- decode skinny GEMM (mma.sync, weights streamed once) ------------------------------------------------
@pytest.mark.parametrize("impl", [0, 1])
@pytest.mark.parametrize("R", [1, 5, 8, 17, 40, 80])
@pytest.mark.parametrize("NK", [(384, 384), (1280, 1280), (1000, 5120), (51864, 128)])
def test_skinny_gemm_vs_numpy(impl, R, NK):
    N, K = NK
    if impl == 1 and N * K * R > 3e8:
        pytest.skip("reference kernel is slow")
    rng = np.random.default_rng(R * 1000 + N)
    x, w, b = rng.standard_normal((R, K), np.float32), rng.standard_normal((N, K), np.float32) / np.sqrt(K), rng.standard_normal(N).astype(np.float32)
    want = f16(x) @ f16(w).T + b
    got = engine.debug_gemv(x, w, b, impl=impl)
    assert np.abs(got - want).max() < 2e-3 * max(1.0, np.abs(want).max())
