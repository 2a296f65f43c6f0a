"""ctypes binding of ``libb200whisper.so`` presenting the slice of the ``ctranslate2`` Python API that
faster-whisper consumes (reference ``faster_whisper/transcribe.py:13,689-698,209,215,222-236,1193,1400,
1446-1459,1709-1715,1823,1875``; SURVEY.md §8b): ``Whisper``, ``StorageView``, ``WhisperGenerationResult``.

There is no CPU path and no fallback: importing works anywhere (so host logic can be tested), but creating a
model, computing a log-mel or encoding raises ``RuntimeError`` unless the CUDA library loads and an H100 (sm_90) is present.
"""

from __future__ import annotations

import ctypes as C
import os
import threading
from dataclasses import dataclass, field
from typing import Dict, Iterable, List, Optional, Sequence, Tuple, Union

import numpy as np

from .config import MODEL_DIMS, SpecialTokens, WhisperDims, special_tokens

# B2W_LIBRARY: measurement hook — another build of the same C ABI (tools/step_ab.py compares kernel versions on one box)
_LIB_PATH = os.environ.get("B2W_LIBRARY") or os.path.join(os.path.dirname(os.path.abspath(__file__)), "libb200whisper.so")
_lib = None
_lib_lock = threading.Lock()

T_STAGES = ("mel", "encoder", "cross_kv", "prefill", "decode", "h2d", "d2h", "reserved")


class _Config(C.Structure):
    _fields_ = [(n, C.c_int32) for n in (
        "n_mels", "n_audio_ctx", "n_audio_state", "n_audio_head", "n_audio_layer",
        "n_vocab", "n_text_ctx", "n_text_state", "n_text_head", "n_text_layer",
        "eot", "sot", "lang_begin", "num_languages", "translate", "transcribe", "sot_lm", "sot_prev",
        "no_speech", "no_timestamps", "timestamp_begin", "n_suppress_begin")] + [("suppress_begin", C.c_int32 * 8)]


class _Tensor(C.Structure):
    _fields_ = [("name", C.c_char_p), ("data", C.c_void_p), ("dtype", C.c_int32), ("ndim", C.c_int32),
                ("shape", C.c_int64 * 4)]


class _GenOpts(C.Structure):
    _fields_ = [
        ("beam_size", C.c_int32), ("patience", C.c_float), ("num_hypotheses", C.c_int32),
        ("length_penalty", C.c_float), ("repetition_penalty", C.c_float), ("no_repeat_ngram_size", C.c_int32),
        ("max_length", C.c_int32), ("return_scores", C.c_int32), ("return_no_speech_prob", C.c_int32),
        ("max_initial_timestamp_index", C.c_int32), ("suppress_blank", C.c_int32),
        ("suppress_tokens", C.POINTER(C.c_int32)), ("n_suppress_tokens", C.c_int32),
        ("sampling_topk", C.c_int32), ("sampling_temperature", C.c_float), ("seed", C.c_uint64),
        ("debug_fake_logits", C.c_int32),
    ]


# every symbol include/b200whisper.h declares (checked by tests/test_abi.py)
ABI_SYMBOLS = (
    "b2w_last_error", "b2w_abi_version", "b2w_device_count", "b2w_model_create", "b2w_model_destroy",
    "b2w_model_info", "b2w_model_sync", "b2w_logmel", "b2w_logmel_frames", "b2w_encode", "b2w_encode_audio",
    "b2w_encoded_shape", "b2w_encoded_to_host", "b2w_encoded_free", "b2w_generate", "b2w_gen_opts_default",
    "b2w_detect_language", "b2w_align", "b2w_model_set_alignment_heads", "b2w_timing_enable", "b2w_timing_reset", "b2w_timing_get", "b2w_span_begin", "b2w_span_end",
    "b2w_counters_get", "b2w_debug_gemm", "b2w_debug_attention", "b2w_debug_gemv", "b2w_debug_logits", "b2w_debug_fetch",
)


def load_library():
    """Loads (building first if the sources are newer and nvcc exists) the CUDA library.  Raises RuntimeError
    when it cannot be loaded: the product has no other implementation."""
    global _lib
    with _lib_lock:
        if _lib is not None:
            return _lib
        if not os.path.exists(_LIB_PATH):
            try:
                from .build import build

                build()
            except Exception as e:  # noqa: BLE001
                raise RuntimeError(f"libb200whisper.so is missing and could not be built: {e}") from e
        try:
            lib = C.CDLL(_LIB_PATH)
        except OSError as e:
            raise RuntimeError(f"cannot load {_LIB_PATH}: {e}") from e
        lib.b2w_last_error.restype = C.c_char_p
        lib.b2w_model_create.argtypes = [C.POINTER(_Config), C.POINTER(_Tensor), C.c_int32, C.c_int32, C.c_char_p,
                                         C.POINTER(C.c_void_p)]
        lib.b2w_model_destroy.argtypes = [C.c_void_p]
        lib.b2w_model_destroy.restype = None
        lib.b2w_model_info.argtypes = [C.c_void_p, C.POINTER(_Config), C.POINTER(C.c_int32)]
        lib.b2w_model_sync.argtypes = [C.c_void_p]
        lib.b2w_logmel.argtypes = [C.c_int32, C.c_int32, C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_int64,
                                   C.POINTER(C.c_int32)]
        lib.b2w_logmel_frames.argtypes = [C.c_int64, C.c_int32]
        lib.b2w_encode.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.POINTER(C.c_void_p)]
        lib.b2w_encode_audio.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_int64), C.c_int32, C.c_void_p,
                                         C.POINTER(C.c_void_p)]
        lib.b2w_encoded_shape.argtypes = [C.c_void_p, C.POINTER(C.c_int64)]
        lib.b2w_encoded_to_host.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        lib.b2w_encoded_free.argtypes = [C.c_void_p]
        lib.b2w_encoded_free.restype = None
        lib.b2w_generate.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.POINTER(_GenOpts),
                                     C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        lib.b2w_gen_opts_default.argtypes = [C.POINTER(_GenOpts)]
        lib.b2w_gen_opts_default.restype = None
        lib.b2w_detect_language.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        lib.b2w_align.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_int32,
                                  C.c_void_p, C.c_int32, C.POINTER(C.c_int32), C.c_void_p]
        lib.b2w_model_set_alignment_heads.argtypes = [C.c_void_p, C.c_void_p, C.c_int32]
        lib.b2w_timing_enable.argtypes = [C.c_void_p, C.c_int32]
        lib.b2w_timing_reset.argtypes = [C.c_void_p]
        lib.b2w_timing_get.argtypes = [C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_int64)]
        lib.b2w_span_begin.argtypes = [C.c_void_p]
        lib.b2w_span_end.argtypes = [C.c_void_p, C.POINTER(C.c_double)]
        lib.b2w_counters_get.argtypes = [C.c_void_p, C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.POINTER(C.c_double)]
        lib.b2w_debug_gemm.argtypes = [C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32,
                                       C.c_int32, C.c_int32, C.c_void_p]
        lib.b2w_debug_attention.argtypes = [C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p]
        lib.b2w_debug_gemv.argtypes = [C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32,
                                       C.c_int32, C.c_void_p]
        lib.b2w_debug_logits.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p]
        lib.b2w_debug_fetch.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_int64]
        if lib.b2w_abi_version() != 1:
            raise RuntimeError("libb200whisper ABI version mismatch")
        _lib = lib
        return lib


def _check(rc: int):
    """status -> the exception type CTranslate2 would surface (ValueError for bad arguments)."""
    if rc == 0:
        return
    msg = (_lib.b2w_last_error() or b"unknown error").decode("utf-8", "replace")
    if rc == 2:
        raise ValueError(msg)
    if rc == 3:
        raise NotImplementedError(msg)
    raise RuntimeError(msg)


def _ptr(a: Optional[np.ndarray]):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def device_count() -> int:
    lib = load_library()
    n = C.c_int(0)
    lib.b2w_device_count(C.byref(n))
    return n.value


def log_mel(waveform: np.ndarray, n_mels: int, padding: int = 160, device: int = 0) -> np.ndarray:
    """FeatureExtractor.__call__ on the GPU (feature_extractor.py:198-230): float32 [n_mels, (N+padding)//160]."""
    lib = load_library()
    x = np.ascontiguousarray(waveform, dtype=np.float32)
    n_frames = (x.shape[0] + padding) // 160
    out = np.empty((n_mels, max(n_frames, 0)), dtype=np.float32)
    nf = C.c_int32(0)
    _check(lib.b2w_logmel(device, n_mels, _ptr(x) if x.size else None, x.shape[0], padding, _ptr(out) if out.size else None,
                          out.size, C.byref(nf)))
    assert nf.value == n_frames
    return out


class StorageView:
    """Stand-in for ``ctranslate2.StorageView``: either a zero-copy view of a host float32 array
    (``from_array``, transcribe.py:1875) or an opaque device-resident encoder output."""

    def __init__(self, array: Optional[np.ndarray] = None, handle=None, owner: "Whisper" = None, shape=None):
        self._array = array
        self._handle = handle
        self._owner = owner
        self.shape = list(shape if shape is not None else (array.shape if array is not None else ()))
        self.device = "cuda" if handle is not None else "cpu"

    @classmethod
    def from_array(cls, array: np.ndarray) -> "StorageView":
        if not isinstance(array, np.ndarray):
            raise ValueError("StorageView.from_array expects a NumPy array")
        if not array.flags["C_CONTIGUOUS"]:
            raise ValueError("StorageView.from_array expects a C-contiguous array")
        return cls(array=array)

    def __array__(self, dtype=None, copy=None):
        a = self.numpy()
        return a.astype(dtype) if dtype is not None else a

    def numpy(self) -> np.ndarray:
        if self._array is not None:
            return self._array
        if self._handle is None:
            raise ValueError("empty StorageView")
        out = np.empty(self.shape, dtype=np.float32)
        _check(_lib.b2w_encoded_to_host(self._owner._replica_for(self).handle, self._handle, _ptr(out)))
        return out

    def _release(self):
        """Frees the device buffer (idempotent).  Goes through the owning replica: an encoder output returns its memory to the
        model's pool, so it must never outlive the native model (``Whisper.unload_model`` releases live outputs first)."""
        h, self._handle = getattr(self, "_handle", None), None
        rep = getattr(self, "_replica", None)
        if h is None or _lib is None:
            return
        if rep is not None:
            rep.release_output(h, id(self))
        else:
            _lib.b2w_encoded_free(h)

    def __del__(self):
        try:
            self._release()
        except Exception:  # noqa: BLE001
            pass


@dataclass
class WhisperGenerationResult:
    sequences_ids: List[List[int]]
    scores: List[float]
    no_speech_prob: float
    sequences: List[List[str]] = field(default_factory=list)


@dataclass
class WhisperAlignmentResult:
    alignments: List[Tuple[int, int]]
    text_token_probs: List[float]


class _Replica:
    def __init__(self, lib, cfg: _Config, tensors, device: int, compute_type: str):
        self._lib = lib
        self.device = device
        h = C.c_void_p()
        arr = (_Tensor * len(tensors))(*tensors)
        _check(lib.b2w_model_create(C.byref(cfg), arr, len(tensors), device, compute_type.encode(), C.byref(h)))
        self._h = h
        self.lock = threading.Lock()
        self._outputs = {}  # id(StorageView) -> weakref: device-resident encoder outputs that borrow from this model's pool
        self._out_lock = threading.Lock()

    def track_output(self, sv) -> None:
        import weakref

        with self._out_lock:
            self._outputs[id(sv)] = weakref.ref(sv)

    def release_output(self, handle, key=None) -> None:
        with self._out_lock:
            self._outputs.pop(key, None)
            if self._h:  # after close() the native model (and every buffer it handed out) is already gone
                self._lib.b2w_encoded_free(handle)

    def close(self):
        """Destroys the native model.  Live encoder outputs are detached first: they become empty StorageViews instead of
        dangling pointers into a freed pool (ADVICE r1: use-after-free in b2w_encoded_free after unload_model)."""
        with self._out_lock:
            views = [r() for r in self._outputs.values()]
            self._outputs.clear()
        for sv in views:
            if sv is not None:
                sv._release()
        with self._out_lock:
            h, self._h = self._h, None
        if h:
            self._lib.b2w_model_destroy(h)

    @property
    def handle(self):
        if not self._h:
            raise RuntimeError("the model is unloaded: call load_model() first")
        return self._h

    def __del__(self):
        try:
            self.close()
        except Exception:  # noqa: BLE001
            pass


_COMPUTE_TYPES = ("default", "auto", "int8", "int8_float32", "int8_float16", "int8_bfloat16", "int16", "float16",
                  "bfloat16", "float32")


class Whisper:
    """``ctranslate2.models.Whisper`` as faster-whisper uses it, backed by libb200whisper.

    ``weights`` maps OpenAI-Whisper state-dict names to float32/float16 NumPy arrays; ``dims`` is the geometry.
    ``model_path`` may instead name a directory holding ``weights.npz`` + ``b2w_config.json`` (see
    ``faster_whisper_b200.checkpoint``)."""

    def __init__(self, model_path: str = "", device: str = "auto", *, device_index: Union[int, Sequence[int]] = 0,
                 compute_type: str = "default", inter_threads: int = 1, intra_threads: int = 0,
                 max_queued_batches: int = 0, flash_attention: bool = False, tensor_parallel: bool = False,
                 files: Optional[dict] = None, dims: Optional[WhisperDims] = None,
                 weights: Optional[Dict[str, np.ndarray]] = None, tokens: Optional[SpecialTokens] = None):
        if device not in ("auto", "cuda", "cpu"):
            raise ValueError(f"unsupported device {device}")
        if device == "cpu":
            raise ValueError("This engine is H100-only: device='cpu' is not available (no CPU fallback by design)")
        if compute_type not in _COMPUTE_TYPES:
            raise ValueError(f"Invalid compute type: {compute_type}")
        lib = load_library()
        if dims is None or weights is None:
            from .checkpoint import load_model_dir

            dims, weights = load_model_dir(model_path, files)
            from .checkpoint import read_alignment_heads

            self._config_alignment_heads = read_alignment_heads(model_path, files)
        self.dims = dims
        self.tokens = tokens or special_tokens(dims.n_vocab)
        cfg = _Config()
        for k in ("n_mels", "n_audio_ctx", "n_audio_state", "n_audio_head", "n_audio_layer", "n_vocab", "n_text_ctx",
                  "n_text_state", "n_text_head", "n_text_layer"):
            setattr(cfg, k, getattr(dims, k))
        for k in ("eot", "sot", "lang_begin", "num_languages", "translate", "transcribe", "sot_lm", "sot_prev",
                  "no_speech", "no_timestamps", "timestamp_begin"):
            setattr(cfg, k, getattr(self.tokens, k))
        begin = [220, self.tokens.eot]
        cfg.n_suppress_begin = len(begin)
        for i, t in enumerate(begin):
            cfg.suppress_begin[i] = t
        self._keep = []
        tensors = []
        for name, arr in weights.items():
            if arr.dtype not in (np.float32, np.float16):
                arr = arr.astype(np.float32)
            arr = np.ascontiguousarray(arr)
            self._keep.append(arr)
            t = _Tensor()
            t.name = name.encode()
            t.data = arr.ctypes.data
            t.dtype = 0 if arr.dtype == np.float32 else 1
            t.ndim = arr.ndim
            for i, s in enumerate(arr.shape):
                t.shape[i] = s
            tensors.append(t)
        idx = [device_index] if isinstance(device_index, int) else list(device_index)
        self._device_index = idx
        self.compute_type = "float16" if compute_type in ("default", "auto") else compute_type
        self._replicas = [_Replica(lib, cfg, tensors, d, compute_type) for d in idx for _ in range(max(1, inter_threads))]
        self._keep = []  # weights are on the device now
        # what load_model() needs to rebuild the replicas after unload_model() (a path is re-read; an in-memory dict is the caller's)
        self._reload = dict(model_path=model_path, files=files, dims=dims if model_path == "" or weights is not None else None,
                            weights=weights if not model_path else None, compute_type=compute_type, inter_threads=inter_threads)
        self._rr = 0
        self._rr_lock = threading.Lock()
        if getattr(self, "_config_alignment_heads", None):
            self.set_alignment_heads(self._config_alignment_heads)

    # ---- read-only properties faster-whisper touches (transcribe.py:379,472,1394) ----
    @property
    def is_multilingual(self) -> bool:
        return self.dims.is_multilingual

    @property
    def n_mels(self) -> int:
        return self.dims.n_mels

    @property
    def device(self) -> str:
        return "cuda"

    @property
    def device_index(self) -> List[int]:
        return list(self._device_index)

    @property
    def num_languages(self) -> int:
        return self.tokens.num_languages

    def _next_replica(self) -> _Replica:
        with self._rr_lock:
            r = self._replicas[self._rr % len(self._replicas)]
            self._rr += 1
            return r

    def _replica_for(self, sv: StorageView) -> _Replica:
        return getattr(sv, "_replica", None) or self._replicas[0]

    @property
    def model_is_loaded(self) -> bool:
        return bool(self._replicas) and all(r._h for r in self._replicas)

    def unload_model(self, to_cpu: bool = False):
        """``ctranslate2`` ``Whisper.unload_model``: frees the device memory of every replica.  Encoder outputs still alive are
        released first and read as empty afterwards; every other call raises until ``load_model()``."""
        for r in self._replicas:
            r.close()

    def load_model(self, keep_cache: bool = False):
        """``ctranslate2`` ``Whisper.load_model``: rebuilds the replicas dropped by ``unload_model`` (no-op while loaded)."""
        if self.model_is_loaded:
            return
        rl = self._reload
        fresh = Whisper(rl["model_path"], "cuda", device_index=self._device_index, compute_type=rl["compute_type"],
                        inter_threads=rl["inter_threads"], files=rl["files"], dims=rl["dims"] or (self.dims if rl["weights"] is not None else None),
                        weights=rl["weights"], tokens=self.tokens)
        self._replicas, fresh._replicas = fresh._replicas, []

    # ---- encode (transcribe.py:209,1400) ----
    def encode(self, features: Union[StorageView, np.ndarray], to_cpu: bool = False) -> StorageView:
        arr = features.numpy() if isinstance(features, StorageView) else np.asarray(features)
        if arr.dtype != np.float32 or not arr.flags["C_CONTIGUOUS"]:
            arr = np.ascontiguousarray(arr, dtype=np.float32)
        if arr.ndim != 3 or arr.shape[1] != self.dims.n_mels or arr.shape[2] != 3000:
            raise ValueError(f"Invalid input features shape: expected an input with shape (batch, {self.dims.n_mels}, 3000), "
                             f"but got an input with shape {tuple(arr.shape)} instead")
        rep = self._next_replica()
        h = C.c_void_p()
        with rep.lock:
            _check(rep._lib.b2w_encode(rep.handle, _ptr(arr), arr.shape[0], C.byref(h)))
        sv = StorageView(handle=h, owner=self, shape=(arr.shape[0], self.dims.n_audio_ctx, self.dims.n_audio_state))
        sv._replica = rep
        rep.track_output(sv)
        if to_cpu:
            return StorageView.from_array(sv.numpy())
        return sv

    def encode_audio(self, chunks: Sequence[np.ndarray], return_features: bool = False):
        """Fused log-mel + encoder for <=30 s chunks (the batched pipeline's hot path): PCM in, encoder output
        resident on the device.  Mirrors ``feature_extractor(chunk)[..., :-1]`` + ``pad_or_trim`` + ``encode``
        (transcribe.py:463-467,514-516,209)."""
        rep = self._next_replica()
        arrs = [np.ascontiguousarray(c, dtype=np.float32) for c in chunks]
        n = len(arrs)
        ptrs = (C.c_void_p * n)(*[a.ctypes.data if a.size else None for a in arrs])
        lens = (C.c_int64 * n)(*[a.shape[0] for a in arrs])
        feats = np.empty((n, self.dims.n_mels, 3000), dtype=np.float32) if return_features else None
        h = C.c_void_p()
        with rep.lock:
            _check(rep._lib.b2w_encode_audio(rep.handle, ptrs, lens, n, _ptr(feats), C.byref(h)))
        sv = StorageView(handle=h, owner=self, shape=(n, self.dims.n_audio_ctx, self.dims.n_audio_state))
        sv._replica = rep
        rep.track_output(sv)
        return (sv, feats) if return_features else sv

    def _as_encoded(self, features: Union[StorageView, np.ndarray]) -> StorageView:
        if isinstance(features, StorageView) and features._handle is not None:
            return features
        arr = features.numpy() if isinstance(features, StorageView) else np.asarray(features, dtype=np.float32)
        if arr.ndim == 3 and arr.shape[1] == self.dims.n_audio_ctx and arr.shape[2] == self.dims.n_audio_state:
            raise ValueError("a host copy of the encoder output cannot be fed back; keep the device StorageView")
        return self.encode(arr)

    # ---- generate (transcribe.py:222-236,1446-1459) ----
    def generate(self, features: Union[StorageView, np.ndarray], prompts: Sequence[Sequence[int]], *,
                 asynchronous: bool = False, beam_size: int = 5, patience: float = 1, num_hypotheses: int = 1,
                 length_penalty: float = 1, repetition_penalty: float = 1, no_repeat_ngram_size: int = 0,
                 max_length: int = 448, return_scores: bool = False, return_logits_vocab: bool = False,
                 return_no_speech_prob: bool = False, max_initial_timestamp_index: int = 50,
                 suppress_blank: bool = True, suppress_tokens: Optional[Sequence[int]] = (-1,),
                 sampling_topk: int = 1, sampling_temperature: float = 1, seed: int = 0,
                 _fake_logits: bool = False) -> List[WhisperGenerationResult]:
        if asynchronous:
            raise NotImplementedError("asynchronous generation is not supported")
        prompts = [list(map(int, p)) for p in prompts]
        if not prompts:
            return []
        P = len(prompts[0])
        if any(len(p) != P for p in prompts):
            raise ValueError("all prompts of one generate() call must have the same length")
        if P == 0:
            raise ValueError("empty prompt")
        enc = None if _fake_logits else self._as_encoded(features)
        if enc is not None and enc.shape[0] != len(prompts):
            raise ValueError("the number of prompts must match the batch size of the encoder output")
        rep = self._replica_for(enc) if enc is not None else self._replicas[0]
        B = len(prompts)
        sup = [int(t) for t in (suppress_tokens or []) if int(t) >= 0]
        sup_arr = np.asarray(sorted(set(sup)), dtype=np.int32)
        o = _GenOpts()
        rep._lib.b2w_gen_opts_default(C.byref(o))
        o.beam_size = int(beam_size)
        o.patience = float(patience)
        o.num_hypotheses = int(num_hypotheses)
        o.length_penalty = float(length_penalty)
        o.repetition_penalty = float(repetition_penalty)
        o.no_repeat_ngram_size = int(no_repeat_ngram_size)
        o.max_length = int(min(max_length, self.dims.n_text_ctx))
        o.return_scores = int(bool(return_scores))
        o.return_no_speech_prob = int(bool(return_no_speech_prob))
        o.max_initial_timestamp_index = int(max_initial_timestamp_index)
        o.suppress_blank = int(bool(suppress_blank))
        o.suppress_tokens = sup_arr.ctypes.data_as(C.POINTER(C.c_int32)) if sup_arr.size else None
        o.n_suppress_tokens = int(sup_arr.size)
        o.sampling_topk = int(sampling_topk)
        o.sampling_temperature = float(sampling_temperature)
        o.seed = int(seed)
        o.debug_fake_logits = int(bool(_fake_logits))
        H = max(1, o.num_hypotheses)
        pr = np.ascontiguousarray(np.asarray(prompts, dtype=np.int32))
        ids = np.zeros((B, H, o.max_length), dtype=np.int32)
        lens = np.zeros((B, H), dtype=np.int32)
        scores = np.zeros((B, H), dtype=np.float32)
        nsp = np.zeros((B,), dtype=np.float32)
        with rep.lock:
            _check(rep._lib.b2w_generate(rep.handle, enc._handle if enc is not None else None, _ptr(pr), P, B, C.byref(o),
                                         _ptr(ids), _ptr(lens), _ptr(scores), _ptr(nsp)))
        out = []
        for b in range(B):
            seqs = [ids[b, h, : lens[b, h]].tolist() for h in range(H)]
            out.append(WhisperGenerationResult(
                sequences_ids=seqs, scores=[float(s) for s in scores[b]] if return_scores else [],
                no_speech_prob=float(nsp[b]) if return_no_speech_prob else 0.0))
        return out

    # ---- detect_language (transcribe.py:215,1193,1823) ----
    def detect_language(self, features: Union[StorageView, np.ndarray]) -> List[List[Tuple[str, float]]]:
        from .config import LANGUAGE_CODES

        if not self.is_multilingual:
            raise RuntimeError("detect_language can only be called on multilingual models")
        enc = self._as_encoded(features)
        rep = self._replica_for(enc)
        nl = self.tokens.num_languages
        probs = np.zeros((enc.shape[0], nl), dtype=np.float32)
        with rep.lock:
            _check(rep._lib.b2w_detect_language(rep.handle, enc._handle, _ptr(probs)))
        names = (LANGUAGE_CODES + [f"xx{i}" for i in range(1, 8)])[:nl]
        out = []
        for b in range(enc.shape[0]):
            order = np.argsort(-probs[b], kind="stable")
            out.append([(f"<|{names[i]}|>", float(probs[b, i])) for i in order])
        return out

    # ---- align (transcribe.py:1709-1715) ----
    def align(self, features, start_sequence, text_tokens, num_frames, *, median_filter_width: int = 7):
        """``ctranslate2.models.Whisper.align`` (transcribe.py:1709-1715): one result per batch item with ``.alignments``
        (list of (text_token_index, time_index)) and ``.text_token_probs``."""
        enc = self._as_encoded(features)
        rep = self._replica_for(enc)
        start = np.ascontiguousarray(list(start_sequence), dtype=np.int32)
        if len(text_tokens) != enc.shape[0]:
            raise ValueError("align: one text token list per batch item is required")
        results = []
        for b, toks in enumerate(text_tokens):
            nf = int(num_frames[b] if isinstance(num_frames, (list, tuple)) else num_frames)
            toks = np.ascontiguousarray(list(toks), dtype=np.int32)
            cap = len(toks) + nf // 2 + 2
            pairs = np.zeros((cap, 2), np.int32)
            probs = np.zeros(max(1, len(toks)), np.float32)
            n_pairs = C.c_int32(0)
            with rep.lock:
                _check(rep._lib.b2w_align(rep.handle, enc._handle, b, _ptr(start), len(start), _ptr(toks), len(toks), nf, int(median_filter_width),
                                          _ptr(pairs), cap, C.byref(n_pairs), _ptr(probs)))
            results.append(WhisperAlignmentResult([(int(a), int(t)) for a, t in pairs[: n_pairs.value]], [float(p) for p in probs[: len(toks)]]))
        return results

    def set_alignment_heads(self, heads=None):
        """(layer, head) pairs from a converted model's config.json ``alignment_heads``; None restores the default."""
        flat = np.ascontiguousarray([x for p in (heads or []) for x in p], dtype=np.int32)
        for rep in self._replicas:
            _check(rep._lib.b2w_model_set_alignment_heads(rep.handle, _ptr(flat) if flat.size else None, flat.size // 2))

    # ---- measurement / test hooks ----
    def timing(self, enable: Optional[bool] = None, reset: bool = False, replica: int = 0) -> Dict[str, float]:
        rep = self._replicas[replica]
        if enable is not None:
            _check(rep._lib.b2w_timing_enable(rep.handle, int(enable)))
        if reset:
            _check(rep._lib.b2w_timing_reset(rep.handle))
        ms = (C.c_double * 8)()
        cnt = (C.c_int64 * 8)()
        _check(rep._lib.b2w_timing_get(rep.handle, ms, cnt))
        ln, st, by = C.c_int64(), C.c_int64(), C.c_double()
        _check(rep._lib.b2w_counters_get(rep.handle, C.byref(ln), C.byref(st), C.byref(by)))
        d = {f"{n}_ms": ms[i] for i, n in enumerate(T_STAGES)}
        d.update(launches=ln.value, decode_steps=st.value, decode_alg_bytes=by.value)
        return d

    def span_begin(self, replica: int = 0):
        """CUDA event on the engine stream: start of a device-timed region (bench.py)."""
        rep = self._replicas[replica]
        _check(rep._lib.b2w_span_begin(rep.handle))

    def span_end(self, replica: int = 0) -> float:
        """Second event + wait; milliseconds between the two events on the engine stream."""
        rep = self._replicas[replica]
        ms = C.c_double()
        _check(rep._lib.b2w_span_end(rep.handle, C.byref(ms)))
        return ms.value

    def sync(self):
        for r in self._replicas:
            _check(r._lib.b2w_model_sync(r.handle))

    def debug_logits(self, enc: StorageView, tokens: np.ndarray) -> np.ndarray:
        tokens = np.ascontiguousarray(tokens, dtype=np.int32)
        B, n = tokens.shape
        out = np.empty((B, n, self.dims.n_vocab), dtype=np.float32)
        rep = self._replica_for(enc)
        with rep.lock:
            _check(rep._lib.b2w_debug_logits(rep.handle, enc._handle, _ptr(tokens), n, B, _ptr(out)))
        return out


    def debug_fetch(self, which: int, n: int, replica: int = 0) -> np.ndarray:
        """Decoder workspace buffer `which` of the last decode step as float32 (tests / tools only)."""
        out = np.empty(int(n), dtype=np.float32)
        rep = self._replicas[replica]
        with rep.lock:
            _check(rep._lib.b2w_debug_fetch(rep.handle, int(which), _ptr(out), int(n)))
        return out


class models:  # namespace shim so `ctranslate2.models.Whisper` style access works on this module
    Whisper = Whisper
    WhisperGenerationResult = WhisperGenerationResult


def debug_gemm(a: np.ndarray, w: np.ndarray, bias: Optional[np.ndarray], impl: int = 0, gelu: bool = False, device: int = 0):
    lib = load_library()
    a = np.ascontiguousarray(a, np.float32)
    w = np.ascontiguousarray(w, np.float32)
    b = None if bias is None else np.ascontiguousarray(bias, np.float32)
    out = np.empty((a.shape[0], w.shape[0]), np.float32)
    _check(lib.b2w_debug_gemm(device, impl, _ptr(a), _ptr(w), _ptr(b), a.shape[0], w.shape[0], a.shape[1], int(gelu), _ptr(out)))
    return out


def debug_attention(qkv: np.ndarray, heads: int, impl: int = 0, device: int = 0):
    lib = load_library()
    qkv = np.ascontiguousarray(qkv, np.float32)
    B, T, _ = qkv.shape
    out = np.empty((B, T, heads * 64), np.float32)
    _check(lib.b2w_debug_attention(device, impl, _ptr(qkv), B, T, heads, _ptr(out)))
    return out


def debug_gemv(x: np.ndarray, w: np.ndarray, bias: Optional[np.ndarray], impl: int = 0, device: int = 0):
    lib = load_library()
    x = np.ascontiguousarray(x, np.float32)
    w = np.ascontiguousarray(w, np.float32)
    b = None if bias is None else np.ascontiguousarray(bias, np.float32)
    out = np.empty((x.shape[0], w.shape[0]), np.float32)
    _check(lib.b2w_debug_gemv(device, impl, _ptr(x), _ptr(w), _ptr(b), x.shape[0], w.shape[0], x.shape[1], _ptr(out)))
    return out
