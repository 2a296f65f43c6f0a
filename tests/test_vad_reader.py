"""CPU: the Silero ONNX reader (faster_whisper_b200/silero.py), its structure check, the float64 restatement against a generic
executor of the stored graph, the VAD model selection, and the VAD C ABI's argument checks (no device is touched).

Every reader test runs on a v6-shaped ONNX file written from seeded weights (``silero_oracle.write_onnx``) and, when
oracle/_ref/ holds it, on the real asset."""
import ctypes
import sys

import numpy as np
import pytest

from faster_whisper_b200 import engine, silero, vad
from oracle import silero_assets, silero_oracle

ONNX = silero_assets.path("silero_vad_v6.onnx")
MODELS = ["synthetic", pytest.param("real", marks=pytest.mark.skipif(not ONNX, reason="oracle/_ref/silero_vad_v6.onnx absent"))]


@pytest.fixture(scope="module", params=MODELS)
def onnx_path(request, tmp_path_factory):
    if request.param == "real":
        return ONNX
    p = str(tmp_path_factory.mktemp("silero") / "synthetic.onnx")
    silero_oracle.write_onnx(silero_oracle.synthetic_weights(5), p)
    return p


@pytest.fixture(scope="module")
def onnx_bytes(onnx_path):
    with open(onnx_path, "rb") as f:
        return f.read()


def _load_bytes(tmp_path, data: bytes):
    p = tmp_path / "model.onnx"
    p.write_bytes(data)
    return silero.load_weights(str(p))


def test_reader_returns_the_weights(onnx_path):
    w = silero.load_weights(onnx_path)
    assert {k: v.shape for k, v in w.items()} == silero.WEIGHT_SHAPES
    assert all(v.dtype == np.float32 and np.isfinite(v).all() for v in w.values())
    g = silero.read_graph(onnx_path)
    assert len(g.nodes) == 25 and len({n.op for n in g.nodes}) == 13
    B = g.initializers["onnx::LSTM_211"]
    assert np.array_equal(w["lstm.bias"], B[0, :512] + B[0, 512:])
    assert "google.protobuf" not in sys.modules and "onnx" not in sys.modules


def test_reader_returns_the_weights_it_was_given(tmp_path):
    w = silero_oracle.synthetic_weights(6)
    silero_oracle.write_onnx(w, str(tmp_path / "m.onnx"))
    got = silero.load_weights(str(tmp_path / "m.onnx"))
    for k, v in w.items():
        if k == "lstm.bias":  # stored as two halves, summed in float32
            np.testing.assert_allclose(got[k], v, rtol=0, atol=1e-6)
        else:
            assert np.array_equal(got[k], v), k


@pytest.mark.parametrize("old,new,node", [
    # the first Conv attribute "strides = [2]" is conv_layers.1's
    (b"\x0a\x07strides\x40\x02\xa0\x01\x07", b"\x0a\x07strides\x40\x01\xa0\x01\x07", "conv_layers.1/Conv"),
    (b"reflect", b"REFLECT", "padding/Pad"),
])
def test_changed_attribute_is_refused_naming_the_node(tmp_path, onnx_bytes, old, new, node):
    assert onnx_bytes.count(old) >= 1
    with pytest.raises(ValueError, match=node):
        _load_bytes(tmp_path, onnx_bytes.replace(old, new, 1))


def test_missing_initializer_is_refused_naming_the_node(tmp_path, onnx_bytes):
    name = b"encoder.conv_layers.2.bias"
    i = onnx_bytes.rindex(name)  # the initializer's own name (node inputs come first)
    data = onnx_bytes[:i] + b"encoder.conv_layers.2.bia_" + onnx_bytes[i + len(name):]
    with pytest.raises(ValueError, match=r"conv_layers.2/Conv.*conv2 bias is not an initializer"):
        _load_bytes(tmp_path, data)


def test_changed_initializer_shape_is_refused(tmp_path, onnx_bytes):
    # conv0.weight dims (128, 129, 3) -> (128, 387, 1): same element count and file length, so the tensor itself parses and
    # only the structure check can refuse it
    old = b"\x08\x80\x01\x08\x81\x01\x08\x03\x10\x01\x42\x1cencoder.conv_layers.0.weight"
    new = b"\x08\x80\x01\x08\x83\x03\x08\x01\x10\x01\x42\x1cencoder.conv_layers.0.weight"
    assert onnx_bytes.count(old) == 1
    data = onnx_bytes.replace(old, new)
    p = tmp_path / "m.onnx"
    p.write_bytes(data)
    assert silero.read_graph(str(p)).initializers["encoder.conv_layers.0.weight"].shape == (128, 387, 1)
    with pytest.raises(ValueError, match=r"conv_layers.0/Conv.*conv0 weight has shape \(128, 387, 1\)"):
        silero.load_weights(str(p))


@pytest.mark.parametrize("cut", [0.5, 0.999])
def test_truncated_file_is_refused(tmp_path, onnx_bytes, cut):
    with pytest.raises(ValueError):
        _load_bytes(tmp_path, onnx_bytes[: int(len(onnx_bytes) * cut)])


@pytest.mark.parametrize("data", [b"", b"hello, world\n", bytes(range(256)) * 4])
def test_non_onnx_file_is_refused(tmp_path, data):
    with pytest.raises(ValueError):
        _load_bytes(tmp_path, data)


def _reference_windows(audio):
    """SileroVADModel.__call__'s input construction written out as the reference writes it (views, in-place zeroing, roll)."""
    batched = audio.reshape(-1, 512).copy()
    context = batched[..., -64:]
    context[-1] = 0
    context = np.roll(context, 1, 0)
    return np.concatenate([context, batched], 1)


@pytest.mark.parametrize("n", [1, 2, 5])
def test_window_inputs_match_the_reference_construction(n):
    a = np.random.default_rng(n).standard_normal(512 * n).astype(np.float32)
    x = silero_oracle.windows(a)
    assert np.array_equal(x, _reference_windows(a).astype(np.float64))
    assert not x[0, :64].any() and not x[-1, -64:].any()


def _graph_and_f64_weights(path):
    g = silero.read_graph(path)
    w = dict(silero.check_graph(g))
    B = g.initializers["onnx::LSTM_211"].astype(np.float64)
    w["lstm.bias"] = B[0, :512] + B[0, 512:]  # the executor adds the two bias halves in float64
    return g, w


@pytest.mark.parametrize("n", [1, 2, 37, 10001])
def test_restatement_equals_graph_executor_seeded(onnx_path, n):
    g, w = _graph_and_f64_weights(onnx_path)
    rng = np.random.default_rng(100 + n)
    a = (0.1 * rng.standard_normal(512 * n) * np.repeat(rng.random(n) < 0.5, 512)).astype(np.float32)
    a[-64:] = 0.3  # non-zero where the last window's tail is zeroed
    want = silero_oracle.graph_probs(g, a)
    got = silero_oracle.probs(w, a)
    assert got.shape == want.shape == (n,)
    assert np.abs(got - want).max() <= 1e-12


@pytest.mark.skipif(not (ONNX and silero_assets.path("physicsworks.wav")), reason="oracle/_ref assets absent")
def test_restatement_equals_graph_executor_on_speech():
    g, w = _graph_and_f64_weights(ONNX)
    a = silero_assets.physicsworks()
    a = np.pad(a, (0, 512 - a.shape[0] % 512))
    want = silero_oracle.graph_probs(g, a)
    got = silero_oracle.probs(w, a)
    assert np.abs(got - want).max() <= 1e-12
    assert (want > 0.5).any() and (want < 0.35).any()


class _Fake:
    def __init__(self, path, device=None):
        self.path, self.device = path, device


def test_vad_model_selection(monkeypatch, tmp_path):
    model = tmp_path / "silero.onnx"
    model.write_bytes(b"x")
    monkeypatch.setenv("B2W_SILERO_VAD", str(model))
    monkeypatch.setattr(vad, "_vad_model", None)
    monkeypatch.setattr(vad, "_silero", {})
    monkeypatch.setattr(vad, "SileroGpuVAD", type("Gpu", (_Fake,), {}))
    monkeypatch.setattr(vad, "SileroVADModel", type("Ort", (_Fake,), {}))
    monkeypatch.setitem(sys.modules, "onnxruntime", None)  # import fails
    m = vad.get_vad_model()
    assert type(m).__name__ == "Gpu" and m.path == str(model) and m.device == 0
    assert vad.get_vad_model() is m
    m1 = vad.get_vad_model(1)  # the transcription model's device
    assert type(m1).__name__ == "Gpu" and m1.device == 1 and m1 is not m
    monkeypatch.setitem(sys.modules, "onnxruntime", type(sys)("onnxruntime"))  # importable: unchanged
    assert type(vad.get_vad_model()).__name__ == "Ort" and type(vad.get_vad_model(1)).__name__ == "Ort"
    fake = lambda a: np.zeros(a.shape[0] // 512)  # noqa: E731
    vad.set_vad_model(fake)
    try:
        assert vad.get_vad_model(1) is fake
    finally:
        vad.set_vad_model(None)


def test_gpu_vad_reports_a_missing_model(monkeypatch, tmp_path):
    monkeypatch.setenv("B2W_SILERO_VAD", str(tmp_path / "absent.onnx"))
    monkeypatch.setattr(vad, "_vad_model", None)
    monkeypatch.setattr(vad, "_silero", {})
    monkeypatch.setitem(sys.modules, "onnxruntime", None)
    with pytest.raises(RuntimeError, match="Silero VAD model not found"):
        vad.get_vad_model()


def _probs_rc(n_samples, capacity, pcm_len=None):
    lib = engine.load_library()
    pcm = np.zeros(max(pcm_len if pcm_len is not None else n_samples, 1), np.float32)
    out = np.zeros(max(capacity, 1), np.float32)
    return engine._check(lib.b2w_vad_probs(None, pcm.ctypes.data_as(ctypes.c_void_p), n_samples, out.ctypes.data_as(ctypes.c_void_p), capacity))


@pytest.mark.parametrize("n_samples,capacity,match", [
    (1000, 10, "positive multiple of 512"),
    (512 * 3 + 1, 10, "positive multiple of 512"),
    (0, 10, "positive multiple of 512"),
    (-512, 10, "positive multiple of 512"),
    (512 * 4, 3, "output buffer too small"),
])
def test_vad_probs_checks_arguments_before_the_device(n_samples, capacity, match):
    with pytest.raises(ValueError, match=match):
        _probs_rc(n_samples, capacity, pcm_len=max(n_samples, 0))


def test_vad_create_checks_weights_before_the_device():
    w = silero_oracle.synthetic_weights(0)
    bad = dict(w, **{"conv1.weight": w["conv1.weight"][:, :, :2]})
    with pytest.raises(ValueError, match="conv1.weight has an unexpected shape"):
        engine.SileroVad(bad)
    bad = dict(w, **{"lstm.w_hh": w["lstm.w_hh"].T.copy()})
    with pytest.raises(ValueError, match="lstm.w_hh has an unexpected shape"):
        engine.SileroVad(bad)
    with pytest.raises(ValueError, match="missing weight tensor: decoder.bias"):
        engine.SileroVad({k: v for k, v in w.items() if k != "decoder.bias"})
