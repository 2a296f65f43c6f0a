"""Voice-activity chunking (``faster_whisper/vad.py``).

The speech probabilities come from the Silero VAD v6 network, one per 512-sample window.  ``get_vad_model()`` loads it from
``B2W_SILERO_VAD`` or ``assets/silero_vad_v6.onnx`` next to this file, as the reference loads its asset (``vad.py:286-351``):
through onnxruntime on the CPU when onnxruntime is importable (``SileroVADModel``, exactly the reference's session), otherwise
on the GPU (``SileroGpuVAD``: the ONNX file is read by ``silero.py`` without onnxruntime, and the network runs as the CUDA
kernels of ``csrc/vad.cu``, fp32 throughout, checked against a float64 restatement).  A missing model file raises RuntimeError;
``set_vad_model`` installs any other ``audio -> probabilities per 512-sample window`` callable.
Everything around the network — the hysteresis segmenter (``vad.py:44-183``), ``collect_chunks`` and ``SpeechTimestampsMap``
(``vad.py:186-285``) — is implemented here and checked against the reference's functions on the same probabilities
(tests/test_dropin.py).
"""
from __future__ import annotations

import bisect
import os
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np


@dataclass
class VadOptions:
    threshold: float = 0.5
    neg_threshold: float = None
    min_speech_duration_ms: int = 0
    max_speech_duration_s: float = float("inf")
    min_silence_duration_ms: int = 2000
    speech_pad_ms: int = 400


_WINDOW = 512  # samples per probability (Silero v5+/v6 at 16 kHz)
_vad_model = None   # installed by set_vad_model
_silero: dict = {}  # default Silero models by (path, None for onnxruntime on the CPU or the GPU index)


def set_vad_model(model) -> None:
    """Installs the speech-probability model: ``model(padded_audio) -> array of one probability per 512-sample window``
    (None restores the default Silero loader)."""
    global _vad_model
    _vad_model = model


def get_vad_model(device_index: int = 0):
    """The installed model, else Silero: through onnxruntime when it is importable, otherwise on GPU ``device_index``
    (the transcription model's first device)."""
    if _vad_model is not None:
        return _vad_model
    path = os.environ.get("B2W_SILERO_VAD") or os.path.join(os.path.dirname(__file__), "assets", "silero_vad_v6.onnx")
    try:
        import onnxruntime  # noqa: F401
    except ImportError:
        key, make = (path, device_index), lambda: SileroGpuVAD(path, device=device_index)
    else:
        key, make = (path, None), lambda: SileroVADModel(path)
    if key not in _silero:
        _silero[key] = make()
    return _silero[key]


def _missing_model(path: str) -> RuntimeError:
    return RuntimeError(f"Silero VAD model not found at {path}; set B2W_SILERO_VAD or use vad_filter=False with clip_timestamps")


class SileroVADModel:
    """The Silero VAD ONNX graph through onnxruntime (inputs ``input [n, 64 + 512]``, ``h``, ``c`` -> probabilities, ``h``, ``c``)."""

    def __init__(self, path: str):
        try:
            import onnxruntime
        except ImportError as e:
            raise RuntimeError("Applying the VAD filter requires the onnxruntime package") from e
        if not os.path.isfile(path):
            raise _missing_model(path)
        opts = onnxruntime.SessionOptions()
        opts.inter_op_num_threads = 1
        opts.intra_op_num_threads = 1
        opts.enable_cpu_mem_arena = False
        opts.log_severity_level = 4
        self.session = onnxruntime.InferenceSession(path, providers=["CPUExecutionProvider"], sess_options=opts)

    def __call__(self, audio: np.ndarray, num_samples: int = _WINDOW, context: int = 64) -> np.ndarray:
        assert audio.ndim == 1 and audio.shape[0] % num_samples == 0
        frames = audio.reshape(-1, num_samples).copy()
        frames[-1, -context:] = 0  # the reference zeroes the tail of the last window in place (vad.py:323-324 writes through a view)
        # every window is preceded by the last 64 samples of the previous one (zeros before the first)
        tails = np.concatenate([np.zeros((1, context), frames.dtype), frames[:-1, -context:]], axis=0)
        x = np.concatenate([tails, frames], axis=1).astype(np.float32)
        h = np.zeros((1, 1, 128), np.float32)
        c = np.zeros((1, 1, 128), np.float32)
        outs = []
        for lo in range(0, x.shape[0], 10000):
            out, h, c = self.session.run(None, {"input": x[lo : lo + 10000], "h": h, "c": c})
            outs.append(out)
        return np.concatenate(outs, axis=0)


class SileroGpuVAD:
    """The Silero VAD ONNX graph on the GPU (csrc/vad.cu), with SileroVADModel's contract: padded audio in, one probability
    per 512-sample window out (same window context, same zeroed tail of the last window, LSTM state carried through)."""

    def __init__(self, path: str, device: int = 0, block_windows: Optional[int] = None):
        if not os.path.isfile(path):
            raise _missing_model(path)
        from . import engine, silero

        self.model = engine.SileroVad(silero.load_weights(path), device=device, block_windows=block_windows)

    def __call__(self, audio: np.ndarray, num_samples: int = _WINDOW, context: int = 64) -> np.ndarray:
        assert audio.ndim == 1 and audio.shape[0] % num_samples == 0
        assert num_samples == _WINDOW and context == 64, "the network takes 512-sample windows after 64 context samples"
        return self.model.probs(audio)

    def many(self, audios: Sequence[np.ndarray], num_samples: int = _WINDOW, context: int = 64) -> List[np.ndarray]:
        """``self(audio)`` for each of several padded recordings, all of them in one sequence of GPU launches."""
        assert all(a.ndim == 1 and a.shape[0] % num_samples == 0 for a in audios)
        assert num_samples == _WINDOW and context == 64, "the network takes 512-sample windows after 64 context samples"
        return self.model.probs_many(audios)


class _Segmenter:
    """Hysteresis over per-window speech probabilities (``vad.py:86-160``): speech starts at the first window >= threshold,
    ends after `min_silence` of windows < neg_threshold; overlong speech is cut at the last silence longer than 98 ms, else hard."""

    def __init__(self, o: VadOptions, sr: int):
        self.thr = o.threshold
        self.neg = o.neg_threshold if o.neg_threshold is not None else max(o.threshold - 0.15, 0.01)
        pad = sr * o.speech_pad_ms / 1000
        self.min_speech = sr * o.min_speech_duration_ms / 1000
        self.max_speech = sr * o.max_speech_duration_s - _WINDOW - 2 * pad
        self.min_silence = sr * o.min_silence_duration_ms / 1000
        self.min_silence_at_max = sr * 98 / 1000
        self.out: List[dict] = []
        self.cur: dict = {}
        self.active = False
        self.silence_from = 0  # start of the silence being tolerated (0 = none)
        self.cut_at = 0        # last silence start that is long enough to cut an overlong segment at
        self.resume = 0        # where speech resumed after that silence

    def _reset_marks(self):
        self.silence_from = self.cut_at = self.resume = 0

    def feed(self, i: int, p: float) -> None:
        pos = _WINDOW * i
        if p >= self.thr and self.silence_from:
            self.silence_from = 0
            if self.resume < self.cut_at:
                self.resume = pos
        if p >= self.thr and not self.active:
            self.active = True
            self.cur["start"] = pos
            return
        if self.active and pos - self.cur["start"] > self.max_speech:
            if self.cut_at:
                self.cur["end"] = self.cut_at
                self.out.append(self.cur)
                self.cur = {}
                if self.resume < self.cut_at:  # still inside that silence: wait for the next onset
                    self.active = False
                else:
                    self.cur["start"] = self.resume
                self._reset_marks()
            else:
                self.cur["end"] = pos
                self.out.append(self.cur)
                self.cur = {}
                self._reset_marks()
                self.active = False
                return
        if p < self.neg and self.active:
            if not self.silence_from:
                self.silence_from = pos
            if pos - self.silence_from > self.min_silence_at_max:
                self.cut_at = self.silence_from
            if pos - self.silence_from < self.min_silence:
                return
            self.cur["end"] = self.silence_from
            if self.cur["end"] - self.cur["start"] > self.min_speech:
                self.out.append(self.cur)
            self.cur = {}
            self._reset_marks()
            self.active = False

    def finish(self, n_samples: int) -> List[dict]:
        if self.cur and n_samples - self.cur["start"] > self.min_speech:
            self.cur["end"] = n_samples
            self.out.append(self.cur)
        return self.out


def get_speech_timestamps(audio: np.ndarray, vad_options: Optional[VadOptions] = None, sampling_rate: int = 16000,
                          device_index: int = 0, **kwargs) -> List[dict]:
    """Speech spans ``[{"start": sample, "end": sample}, ...]`` (``vad.py:44-183``); ``device_index``: the GPU of the default
    Silero model when it runs on the GPU."""
    o = vad_options if vad_options is not None else VadOptions(**kwargs)
    return _spans(audio, get_vad_model(device_index)(_padded(audio)), o, sampling_rate)


def get_speech_timestamps_many(audios: Sequence[np.ndarray], vad_options: Optional[VadOptions] = None,
                               sampling_rate: int = 16000, device_index: int = 0, **kwargs) -> List[List[dict]]:
    """``get_speech_timestamps`` of every recording: the default GPU model runs all of them in one multi-stream call
    (``SileroGpuVAD.many``); onnxruntime or a model installed by ``set_vad_model`` runs them one after another."""
    o = vad_options if vad_options is not None else VadOptions(**kwargs)
    model = get_vad_model(device_index)
    padded = [_padded(a) for a in audios]
    probs = model.many(padded) if hasattr(model, "many") else [model(a) for a in padded]
    return [_spans(a, p, o, sampling_rate) for a, p in zip(audios, probs)]


def _padded(audio: np.ndarray) -> np.ndarray:
    return np.pad(audio, (0, _WINDOW - audio.shape[0] % _WINDOW))


def _spans(audio: np.ndarray, probs: np.ndarray, o: VadOptions, sampling_rate: int) -> List[dict]:
    """The segmenter over one recording's probabilities, then the span padding."""
    n = len(audio)
    seg = _Segmenter(o, sampling_rate)
    for i, p in enumerate(probs):
        seg.feed(i, p)
    spans = seg.finish(n)
    # pad every span by speech_pad_ms, sharing short gaps between neighbours half and half
    pad = sampling_rate * o.speech_pad_ms / 1000
    for k, sp in enumerate(spans):
        if k == 0:
            sp["start"] = int(max(0, sp["start"] - pad))
        if k + 1 < len(spans):
            nxt = spans[k + 1]
            gap = nxt["start"] - sp["end"]
            if gap < 2 * pad:
                sp["end"] += int(gap // 2)
                nxt["start"] = int(max(0, nxt["start"] - gap // 2))
            else:
                sp["end"] = int(min(n, sp["end"] + pad))
                nxt["start"] = int(max(0, nxt["start"] - pad))
        else:
            sp["end"] = int(min(n, sp["end"] + pad))
    return spans


def collect_chunks(audio: np.ndarray, chunks: List[dict], sampling_rate: int = 16000,
                   max_duration: float = float("inf")) -> Tuple[List[np.ndarray], List[Dict[str, float]]]:
    """Greedily packs speech spans (sample offsets) into pieces of at most `max_duration` seconds."""
    if not chunks:
        return [np.array([], dtype=np.float32)], [{"offset": 0, "duration": 0, "segments": []}]
    limit = max_duration * sampling_rate
    pieces, metas = [], []
    spans, samples, consumed = [], 0, 0
    buf: List[np.ndarray] = []

    def flush():
        nonlocal spans, samples, consumed, buf
        pieces.append(np.concatenate(buf) if buf else np.array([], dtype=np.float32))
        metas.append({"offset": consumed / sampling_rate, "duration": samples / sampling_rate, "segments": spans})
        consumed += samples

    for span in chunks:
        n = span["end"] - span["start"]
        if samples + n > limit:
            flush()
            # the reference starts the next piece with this span's audio but does not list the span itself
            spans, buf, samples = [], [audio[span["start"] : span["end"]]], n
        else:
            spans.append(span)
            buf.append(audio[span["start"] : span["end"]])
            samples += n
    flush()
    return pieces, metas


class SpeechTimestampsMap:
    """Maps times on the silence-removed axis back to the original recording."""

    def __init__(self, chunks: List[dict], sampling_rate: int, time_precision: int = 2):
        self.sampling_rate = sampling_rate
        self.time_precision = time_precision
        self.chunk_end_sample: List[int] = []
        self.total_silence_before: List[float] = []
        cursor, removed = 0, 0
        for c in chunks:
            removed += c["start"] - cursor
            cursor = c["end"]
            self.chunk_end_sample.append(c["end"] - removed)
            self.total_silence_before.append(removed / sampling_rate)

    def get_chunk_index(self, time: float, is_end: bool = False) -> int:
        sample = int(time * self.sampling_rate)
        if is_end and sample in self.chunk_end_sample:
            return self.chunk_end_sample.index(sample)
        return min(bisect.bisect(self.chunk_end_sample, sample), len(self.chunk_end_sample) - 1)

    def get_original_time(self, time: float, chunk_index: Optional[int] = None, is_end: bool = False) -> float:
        if chunk_index is None:
            chunk_index = self.get_chunk_index(time, is_end)
        return round(self.total_silence_before[chunk_index] + time, self.time_precision)
