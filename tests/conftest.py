import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90)")


def _gpu_available() -> bool:
    try:
        from faster_whisper_b200 import engine

        return engine.device_count() > 0
    except Exception:  # noqa: BLE001
        return False


def pytest_collection_modifyitems(config, items):
    if _gpu_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def micro():
    """A 2+2-layer, d=128 model with the tiny.en vocabulary: weights, oracle, tokens."""
    from faster_whisper_b200.config import special_tokens
    from faster_whisper_b200.synthetic import custom_dims, make_weights
    from oracle.whisper_oracle import WhisperOracle

    dims = custom_dims(d=128, heads=2, enc_layers=2, dec_layers=2, n_vocab=51864)
    w = make_weights(dims, seed=11)
    st = special_tokens(dims.n_vocab)
    return dict(dims=dims, weights=w, tokens=st, oracle=WhisperOracle(dims.to_dict(), w, st.to_dict()))


@pytest.fixture(scope="session")
def micro_ml():
    """Multilingual (large-v3 vocabulary, 128 mels) micro model, d=192 / 3 heads / 2+3 layers."""
    from faster_whisper_b200.config import special_tokens
    from faster_whisper_b200.synthetic import custom_dims, make_weights
    from oracle.whisper_oracle import WhisperOracle

    dims = custom_dims(name="micro-ml", n_mels=128, d=192, heads=3, enc_layers=2, dec_layers=3, n_vocab=51866)
    w = make_weights(dims, seed=12)
    st = special_tokens(dims.n_vocab)
    return dict(dims=dims, weights=w, tokens=st, oracle=WhisperOracle(dims.to_dict(), w, st.to_dict()))


def fake_logits_numpy(n_vocab, timestamp_begin, eot):
    """NumPy mirror of csrc/search.cu:fake_logits_kernel (the decoder stand-in for search tests)."""

    def f(tokens_rows, step, hist):
        tok = np.asarray(tokens_rows, dtype=np.uint32)[:, None]
        v = np.arange(n_vocab, dtype=np.uint32)[None, :]
        h = (tok * np.uint32(0x9E3779B1)) ^ np.uint32((step * 0x85EBCA77) & 0xFFFFFFFF) ^ (v * np.uint32(0xC2B2AE3D))
        h ^= h >> np.uint32(16)
        h = h * np.uint32(0x7FEB352D)
        h ^= h >> np.uint32(15)
        h = h * np.uint32(0x846CA68B)
        h ^= h >> np.uint32(16)
        x = (h >> np.uint32(8)).astype(np.float32) * np.float32(9.5367431640625e-07) + np.float32(-8.0)
        x[:, timestamp_begin:] = x[:, timestamp_begin:] + np.float32(3.0)
        x[:, eot] = x[:, eot] + np.float32(0.25) * np.float32(step)
        return x.astype(np.float32)

    return f
