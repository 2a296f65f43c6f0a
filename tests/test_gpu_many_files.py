"""-m gpu: several recordings at once.  The multi-stream Silero VAD (b2w_vad_probs_multi) is bit-identical to one
b2w_vad_probs call per stream and within the bound of the float64 restatement; ``transcribe_many`` on the CUDA engine matches
per-file ``transcribe`` over the oracle shim (greedy and beam 5, tiny.en and multilingual micro geometry); VAD spans per file
equal the single-file spans."""
import json
import sys

import numpy as np
import pytest

from faster_whisper_b200 import engine as our_engine
from faster_whisper_b200 import silero, vad
from faster_whisper_b200 import transcribe as T
from faster_whisper_b200.config import MODEL_DIMS
from faster_whisper_b200.synthetic import make_tokenizer, make_weights, synthetic_audio
from oracle import ct2_shim, silero_assets, silero_oracle
from oracle import whisper_oracle as orc

pytestmark = pytest.mark.gpu

BOUND = 1e-4
LOGIT_TOL = 0.05
ONNX = silero_assets.path("silero_vad_v6.onnx")
WAV = silero_assets.path("physicsworks.wav")


def speechlike(n_windows: int, seed: int) -> np.ndarray:
    rng = np.random.default_rng(seed)
    n = n_windows * 512
    t = np.arange(n) / 16000.0
    on = np.repeat(rng.random(n_windows // 20 + 1) < 0.5, 20 * 512)[:n]
    x = 0.003 * rng.standard_normal(n) + on * (0.2 * np.sin(2 * np.pi * 180 * t) + 0.05 * rng.standard_normal(n))
    x[-64:] = 0.25  # non-zero where the last window's tail counts as zero
    return x.astype(np.float32)


LENGTHS = [1, 17, 6250]  # windows


def _calls(n_streams: int, seed: int):
    """The stream lists of the calls a case makes: one stream of each length, 3 streams of mixed lengths, or 100 streams
    (short ones, and one long stream among them)."""
    if n_streams == 1:
        return [[speechlike(n, seed=seed + n)] for n in LENGTHS]
    if n_streams == 3:
        return [[speechlike(n, seed=seed + i) for i, n in enumerate(LENGTHS)]]
    audios = [speechlike([1, 17][i % 2], seed=seed + i) for i in range(n_streams)]
    audios[50] = speechlike(6250, seed=7)
    return [audios]


@pytest.fixture(scope="module")
def seeded():
    return silero_oracle.synthetic_weights(3)


def _bits(x):
    return x.view(np.uint32)


@pytest.mark.parametrize("block", [1, 100, None])
@pytest.mark.parametrize("n_streams", [1, 3, 100])
def test_probs_many_bit_identical_to_one_stream(seeded, n_streams, block):
    model = our_engine.SileroVad(seeded, block_windows=block)
    for audios in _calls(n_streams, seed=n_streams):
        got = model.probs_many(audios)
        assert len(got) == len(audios)
        for a, g in zip(audios, got):
            assert np.array_equal(_bits(g), _bits(model.probs(a)))
        assert model.timing()["recurrence"] > 0
        if block is None:  # the oracle is slow: check the first three streams of the default block size
            for a, g in list(zip(audios, got))[:3]:
                err = float(np.abs(g - silero_oracle.probs(seeded, a)).max())
                assert err <= BOUND, err


def test_probs_many_on_the_asset():
    if not (ONNX and WAV):
        pytest.skip("oracle/_ref assets absent (no reference tree at build time)")
    weights = silero.load_weights(ONNX)
    a = silero_assets.physicsworks()
    a = np.pad(a, (0, 512 - a.shape[0] % 512))
    audios = [a, speechlike(17, 1), a[: 512 * 3000].copy()]
    model = our_engine.SileroVad(weights, block_windows=5000)
    got = model.probs_many(audios)
    for x, g in zip(audios, got):
        assert np.array_equal(_bits(g), _bits(model.probs(x)))
        assert float(np.abs(g - silero_oracle.probs(weights, x)).max()) <= BOUND


def test_vad_spans_per_file(seeded, tmp_path, monkeypatch):
    path = str(tmp_path / "synthetic.onnx")
    silero_oracle.write_onnx(seeded, path)
    monkeypatch.setitem(sys.modules, "onnxruntime", None)
    monkeypatch.setenv("B2W_SILERO_VAD", path)
    monkeypatch.setattr(vad, "_silero", {})
    vad.set_vad_model(None)
    audios = [speechlike(n, seed=60 + n) for n in (40, 900, 3000)]
    opts = vad.VadOptions(max_speech_duration_s=30, min_silence_duration_ms=160)
    got = vad.get_speech_timestamps_many(audios, opts)
    assert isinstance(vad.get_vad_model(), vad.SileroGpuVAD)
    assert got == [vad.get_speech_timestamps(a, opts) for a in audios]
    assert any(len(s) >= 2 for s in got)


# ---- the pipeline on the GPU against per-file transcribe over the oracle shim ----------------------------------------
def _models(dims, w):
    files = {"tokenizer.json": make_tokenizer(dims.n_vocab).to_str().encode(),
             "preprocessor_config.json": json.dumps({"feature_size": dims.n_mels}).encode()}
    gpu = T.WhisperModel("synthetic", device="cuda", files=dict(files), dims=dims, weights=w)
    whisper_cls, oracle = ct2_shim.make_whisper_class(dims, w)
    margins = []  # the oracle's smallest top-1/top-2 margin of every generated sequence

    class Recording(whisper_cls):
        def generate(self, features, prompts, **kw):
            kw.pop("asynchronous", None)
            res = oracle.generate(features.tensor, prompts, **kw)
            margins.extend(r.min_margin for r in res)
            return [ct2_shim.WhisperGenerationResult(r.sequences_ids, r.scores, r.no_speech_prob) for r in res]

    mp = pytest.MonkeyPatch()
    mp.setattr(our_engine, "Whisper", lambda *a, **k: Recording())
    mp.setattr(our_engine, "log_mel", lambda x, n_mels, padding=160, device=0: orc.log_mel(x, n_mels, padding))
    mp.setattr(our_engine, "StorageView", ct2_shim.StorageView)
    cpu = T.WhisperModel("synthetic", device="cuda", files=dict(files), dims=dims, weights=w)
    mp.undo()
    return gpu, cpu, mp, margins


@pytest.fixture(scope="module")
def tiny_en():
    dims = MODEL_DIMS["tiny.en"]
    return _models(dims, make_weights(dims, seed=5))


@pytest.fixture(scope="module")
def ml(micro_ml):
    return _models(micro_ml["dims"], micro_ml["weights"])


def _oracle_per_file(cpu, mp, margins, audios, clips, kw):
    """Per-file transcribe over the oracle shim: (segments, info) and the oracle's smallest margin of each file."""
    mp.setattr(our_engine, "log_mel", lambda x, n_mels, padding=160, device=0: orc.log_mel(x, n_mels, padding))
    mp.setattr(our_engine, "StorageView", ct2_shim.StorageView)
    try:
        out, file_margins = [], []
        for a, c in zip(audios, clips):
            margins.clear()
            segs, info = T.BatchedInferencePipeline(cpu).transcribe(a.copy(), clip_timestamps=c, **kw)
            out.append((list(segs), info))
            file_margins.append(min(margins, default=float("inf")))
        return out, file_margins
    finally:
        mp.undo()


def _compare(got, want, file_margins):
    """Tokens, seek and times exact and scores close, except in a file whose oracle decode has a near-tie (top-1/top-2
    margin below twice the logit tolerance), where the GPU may take the other branch."""
    print("oracle min margin per file:", ["%.4f" % m for m in file_margins])
    for (gs, gi), (ws, wi), margin in zip(got, want, file_margins):
        assert gi.language == wi.language and gi.duration == wi.duration
        if [list(s.tokens) for s in gs] != [list(s.tokens) for s in ws]:
            print("tokens differ at an oracle margin of %.4f" % margin)
            assert margin < 2 * LOGIT_TOL, margin
            continue
        for g, w in zip(gs, ws):
            assert (g.id, g.seek, round(g.start, 2), round(g.end, 2)) == (w.id, w.seek, round(w.start, 2), round(w.end, 2))
            assert abs(g.avg_logprob - w.avg_logprob) < 5e-3 and abs(g.no_speech_prob - w.no_speech_prob) < 5e-3


@pytest.mark.parametrize("which", ["tiny_en", "ml"])
def test_transcribe_many_greedy(request, which):
    gpu, cpu, mp, margins = request.getfixturevalue(which)
    audios = [synthetic_audio(400 + i, s) for i, s in enumerate([3.0, 29.0, 12.0, 45.0, 20.0])]
    clips = [None, None, None, [{"start": 0.0, "end": 30.0}, {"start": 30.0, "end": 45.0}], None]
    kw = dict(beam_size=1, batch_size=4, vad_filter=False, max_new_tokens=24, repetition_penalty=1.2, no_repeat_ngram_size=3)
    if which == "tiny_en":
        kw["language"] = "en"
    got = T.BatchedInferencePipeline(gpu).transcribe_many(audios, clip_timestamps=clips, **kw)
    want, file_margins = _oracle_per_file(cpu, mp, margins, audios, clips, kw)
    assert sum(len(s) for s, _ in want) >= 5
    _compare(got, want, file_margins)


def test_transcribe_many_beam5_batch16(tiny_en):
    """16 chunks of 9 files in one generate call at beam 5."""
    gpu, cpu, mp, margins = tiny_en
    audios = [synthetic_audio(500 + i, s) for i, s in enumerate([29.0, 5.0, 58.0, 12.0, 29.0, 88.0, 40.0, 20.0, 87.0])]
    clips = [[{"start": lo, "end": min(lo + 29.0, len(a) / 16000)} for lo in np.arange(0, len(a) / 16000, 29.0)] for a in audios]
    kw = dict(beam_size=5, batch_size=16, vad_filter=False, language="en", max_new_tokens=32, repetition_penalty=1.2,
              no_repeat_ngram_size=3)
    got = T.BatchedInferencePipeline(gpu).transcribe_many(audios, clip_timestamps=clips, **kw)
    want, file_margins = _oracle_per_file(cpu, mp, margins, audios, clips, kw)
    assert sum(len(c) for c in clips) == 16
    _compare(got, want, file_margins)
