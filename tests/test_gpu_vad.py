"""-m gpu: the Silero VAD network on the GPU (csrc/vad.cu through vad.SileroGpuVAD / engine.SileroVad) against the float64
restatement (oracle/silero_oracle.py), on seeded Silero-shaped weights and on the real asset; block and run invariance; speech
spans and the batched pipeline's default (VAD on, onnxruntime absent) against the same host code driven by oracle probabilities.

Every check runs on seeded weights written as a Silero-shaped ONNX file and seeded speech-like audio; the same checks run on
the real asset and the physicsworks recording when oracle/_ref/ holds them."""
import json
import sys

import numpy as np
import pytest

from faster_whisper_b200 import engine, silero, vad
from oracle import silero_assets, silero_oracle

pytestmark = pytest.mark.gpu

BOUND = 1e-4  # max |p_gpu - p_oracle|
ONNX = silero_assets.path("silero_vad_v6.onnx")
WAV = silero_assets.path("physicsworks.wav")
needs_assets = pytest.mark.skipif(not (ONNX and WAV), reason="oracle/_ref assets absent (no reference tree at build time)")
HOUR = 112_500  # windows in one hour


def speechlike(n_windows: int, seed: int) -> np.ndarray:
    """Seeded bursts of band-limited noise and tones over quiet noise, n_windows * 512 samples."""
    rng = np.random.default_rng(seed)
    n = n_windows * 512
    t = np.arange(n) / 16000.0
    on = np.repeat(rng.random(n_windows // 20 + 1) < 0.5, 20 * 512)[:n]
    tone = np.sin(2 * np.pi * (150 + 100 * np.sin(2 * np.pi * 0.3 * t)) * t) * (1 + 0.5 * np.sin(2 * np.pi * 4 * t))
    x = 0.003 * rng.standard_normal(n) + on * (0.2 * tone + 0.05 * rng.standard_normal(n))
    x[-64:] = 0.25  # non-zero where the last window's tail counts as zero
    return x.astype(np.float32)


def physicsworks_padded() -> np.ndarray:
    a = silero_assets.physicsworks()
    return np.pad(a, (0, 512 - a.shape[0] % 512))


def one_hour() -> np.ndarray:
    """physicsworks tiled to one hour, seeded noise of a few seconds between copies."""
    rng = np.random.default_rng(7)
    a = silero_assets.physicsworks()
    parts, n = [], 0
    while n < HOUR * 512:
        gap = (0.01 * rng.standard_normal(int(rng.integers(16000, 80000)))).astype(np.float32)
        parts += [a, gap]
        n += a.shape[0] + gap.shape[0]
    return np.concatenate(parts)[: HOUR * 512]


@pytest.fixture(scope="module")
def synth():
    w = silero_oracle.synthetic_weights(3)
    return w, engine.SileroVad(w)


@pytest.fixture(scope="module")
def synth_onnx(tmp_path_factory):
    """(weights, path of the ONNX file written from them)"""
    w = silero_oracle.synthetic_weights(3)
    p = str(tmp_path_factory.mktemp("silero") / "synthetic.onnx")
    silero_oracle.write_onnx(w, p)
    return silero.load_weights(p), p


def _case(which, synth_onnx):
    """(weights, ONNX path, audio) of a case: the seeded graph on 200 s of speech-like audio, or the asset on physicsworks."""
    if which == "synthetic":
        w, p = synth_onnx
        return w, p, speechlike(6250, seed=11)
    if not (ONNX and WAV):
        pytest.skip("oracle/_ref assets absent (no reference tree at build time)")
    return silero.load_weights(ONNX), ONNX, silero_assets.physicsworks()


@pytest.fixture(scope="module")
def real():
    if not ONNX:
        pytest.skip("oracle/_ref/silero_vad_v6.onnx absent")
    w = silero.load_weights(ONNX)
    return w, vad.SileroGpuVAD(ONNX)


def _check(model, weights, audio, label):
    got = model.probs(audio) if isinstance(model, engine.SileroVad) else model(audio)
    want = silero_oracle.probs(weights, audio)
    assert got.shape == want.shape == (audio.shape[0] // 512,) and got.dtype == np.float32
    err = float(np.abs(got - want).max())
    print(f"VAD {label}: {want.shape[0]} windows, max |dp| = {err:.3g}, p in [{want.min():.3f}, {want.max():.3f}]")
    assert err <= BOUND, (label, err)
    return got, want


@pytest.mark.parametrize("n", [1, 2, 9_999, 10_000, 10_001])
@pytest.mark.parametrize("which", ["synthetic", "real"])
def test_probs_match_oracle(request, which, n):
    weights, model = request.getfixturevalue("synth" if which == "synthetic" else "real")
    got, want = _check(model, weights, speechlike(n, seed=n), f"{which} n={n}")
    if which == "synthetic" and n > 100:
        assert want.min() < 0.2 and want.max() > 0.6  # the probabilities are spread, not saturated


@needs_assets
@pytest.mark.parametrize("which", ["synthetic", "real"])
def test_probs_match_oracle_on_speech(request, which):
    weights, model = request.getfixturevalue("synth" if which == "synthetic" else "real")
    _check(model, weights, physicsworks_padded(), f"{which} physicsworks")


@pytest.mark.parametrize("which", ["synthetic", "real"])
def test_one_hour_matches_oracle_and_is_block_invariant(request, which):
    if which == "real" and not WAV:
        pytest.skip("oracle/_ref/physicsworks.wav absent")
    weights, model = request.getfixturevalue("synth" if which == "synthetic" else "real")
    # the seeded weights run on seeded speech-like audio, the asset on physicsworks tiled to an hour
    audio = np.concatenate([speechlike(HOUR // 10, seed=50 + k) for k in range(10)]) if which == "synthetic" else one_hour()
    got, _ = _check(model, weights, audio, f"{which} one hour")
    again = model.probs(audio) if isinstance(model, engine.SileroVad) else model(audio)
    assert np.array_equal(got.view(np.uint32), again.view(np.uint32)), "two runs differ"
    blocked = engine.SileroVad(weights, block_windows=7_777)  # 15 blocks, the last one short
    assert np.array_equal(got.view(np.uint32), blocked.probs(audio).view(np.uint32)), "blocks differ from one pass"
    t = blocked.timing()
    assert t["recurrence"] > 0 and t["window"] > 0 and t["decoder"] > 0


@pytest.mark.parametrize("block", [7, 1_000])
def test_blocks_match_one_pass(synth, block):
    """Several blocks in one call (context samples of the block before, the tail rule on the last block only, h and c carried
    between launches) give the bits of one pass."""
    weights, one_pass = synth
    audio = speechlike(3_001, seed=21)
    got, _ = _check(one_pass, weights, audio, "synthetic n=3001 one pass")
    blocked = engine.SileroVad(weights, block_windows=block)
    assert np.array_equal(got.view(np.uint32), blocked.probs(audio).view(np.uint32)), "blocks differ from one pass"
    # a block boundary exactly at the last window, and a last block of one window
    for n in (2 * block, 2 * block + 1):
        a = speechlike(n, seed=n)
        assert np.array_equal(one_pass.probs(a).view(np.uint32), blocked.probs(a).view(np.uint32)), n


def test_longer_than_the_default_block(synth):
    """70 001 windows: three blocks at the default block size, against the oracle and against a single block."""
    weights, model = synth
    audio = speechlike(70_001, seed=31)
    got, _ = _check(model, weights, audio, "synthetic n=70001 default blocks")
    single = engine.SileroVad(weights, block_windows=1 << 17)
    assert np.array_equal(got.view(np.uint32), single.probs(audio).view(np.uint32))
    assert np.array_equal(got.view(np.uint32), model.probs(audio).view(np.uint32)), "two runs differ"


def test_gpu_vad_reads_the_onnx_file(synth_onnx):
    weights, path = synth_onnx
    _check(vad.SileroGpuVAD(path), weights, speechlike(4_000, seed=41), "synthetic ONNX file")


def _spans_equal_unless_near_tie(got, want, p_oracle, opts):
    if got == want:
        return
    thr = opts.threshold
    neg = opts.neg_threshold if opts.neg_threshold is not None else max(thr - 0.15, 0.01)
    near = np.minimum(np.abs(p_oracle - thr), np.abs(p_oracle - neg))
    i = int(np.argmin(near))
    print(f"spans differ; closest oracle probability to a threshold: p[{i}] = {p_oracle[i]:.6f} ({near[i]:.2g} away)")
    assert near[i] <= BOUND, (got, want)


@pytest.mark.parametrize("kw", [{}, dict(min_silence_duration_ms=500, speech_pad_ms=200)])
@pytest.mark.parametrize("which", ["synthetic", "real"])
def test_speech_timestamps_match_oracle(synth_onnx, which, kw):
    weights, path, audio = _case(which, synth_onnx)
    model = vad.SileroGpuVAD(path)
    want_p = silero_oracle.probs(weights, np.pad(audio, (0, 512 - audio.shape[0] % 512)))
    opts = vad.VadOptions(**kw)
    try:
        vad.set_vad_model(model)
        got = vad.get_speech_timestamps(audio, opts)
        vad.set_vad_model(lambda a: want_p)
        want = vad.get_speech_timestamps(audio, opts)
    finally:
        vad.set_vad_model(None)
    assert len(want) >= 2, want  # speech and silence both occur
    assert sum(s["end"] - s["start"] for s in want) < audio.shape[0]
    _spans_equal_unless_near_tie(got, want, want_p, opts)


@pytest.mark.parametrize("which", ["synthetic", "real"])
def test_batched_pipeline_default_vad_without_onnxruntime(micro, monkeypatch, synth_onnx, which):
    from faster_whisper_b200 import transcribe as T
    from faster_whisper_b200.synthetic import make_tokenizer

    weights, path, audio = _case(which, synth_onnx)
    dims, w = micro["dims"], micro["weights"]
    files = {"tokenizer.json": make_tokenizer(dims.n_vocab).to_str().encode(),
             "preprocessor_config.json": json.dumps({"feature_size": dims.n_mels}).encode()}
    model = T.WhisperModel("synthetic", device="cuda", files=files, dims=dims, weights=w)
    want_p = silero_oracle.probs(weights, np.pad(audio, (0, 512 - audio.shape[0] % 512)))
    opts = vad.VadOptions(max_speech_duration_s=30, min_silence_duration_ms=160)  # the pipeline's default
    monkeypatch.setitem(sys.modules, "onnxruntime", None)
    monkeypatch.setenv("B2W_SILERO_VAD", path)
    vad.set_vad_model(None)
    try:
        segs, info = T.BatchedInferencePipeline(model).transcribe(audio.copy())
        got = list(segs)
        gpu_model = vad.get_vad_model()
        assert isinstance(gpu_model, vad.SileroGpuVAD)
        got_spans = vad.get_speech_timestamps(audio, opts)
        vad.set_vad_model(lambda a: want_p)
        want_spans = vad.get_speech_timestamps(audio, opts)
        want_segs, want_info = T.BatchedInferencePipeline(model).transcribe(audio.copy())
        want = list(want_segs)
    finally:
        vad.set_vad_model(None)
    assert len(want) >= 2 and 0 < want_info.duration_after_vad < want_info.duration
    if got_spans != want_spans:  # exact unless an oracle probability sits within the bound of a threshold
        _spans_equal_unless_near_tie(got_spans, want_spans, want_p, opts)
        return
    assert info.duration_after_vad == want_info.duration_after_vad
    key = lambda s: (list(s.tokens), round(s.start, 3), round(s.end, 3), s.text)  # noqa: E731
    assert [key(s) for s in got] == [key(s) for s in want]
