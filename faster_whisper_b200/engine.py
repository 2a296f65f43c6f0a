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


class _GemmDesc(C.Structure):  # b2w_gemm_desc
    _fields_ = [
        ("a", C.c_void_p), ("a_elems", C.c_int64), ("a_batch", C.c_int32), ("a_rows", C.c_int32), ("a_cols", C.c_int32),
        ("a_row_stride", C.c_int64), ("a_batch_stride", C.c_int64), ("taps", C.c_int32), ("tap_row", C.c_int32 * 3),
        ("tap_col", C.c_int32 * 3), ("k_per_tap", C.c_int32), ("w", C.c_void_p), ("bias", C.c_void_p), ("N", C.c_int32),
        ("rows", C.c_int32), ("epilogue", C.c_int32), ("narrow_tiles", C.c_int32), ("out", C.c_void_p), ("out_elems", C.c_int64),
        ("out_ld", C.c_int64), ("out_batch_stride", C.c_int64), ("pos", C.c_void_p), ("xkv_d", C.c_int32), ("xkv_heads", C.c_int32),
        ("xkv_T", C.c_int32), ("xkv_B", C.c_int32), ("rowinfo", C.c_void_p), ("kcache", C.c_void_p), ("vcache", C.c_void_p),
        ("cache_elems", C.c_int64), ("qkv_d", C.c_int32), ("n_ctx", C.c_int32), ("slots", C.c_int32), ("max_ctas", C.c_int32),
        ("block_n_out", C.c_int32), ("grid_out", C.c_int32),
    ]


class _GemvDesc(C.Structure):  # b2w_gemv_desc
    _fields_ = [
        ("x", C.c_void_p), ("w", C.c_void_p), ("bias", C.c_void_p), ("R", C.c_int32), ("N", C.c_int32), ("K", C.c_int32),
        ("mode", C.c_int32), ("route", C.c_int32), ("rows", C.c_void_p), ("kcache", C.c_void_p), ("vcache", C.c_void_p),
        ("cache_elems", C.c_int64), ("d", C.c_int32), ("n_ctx", C.c_int32), ("slots", C.c_int32), ("out", C.c_void_p),
        ("out_elems", C.c_int64), ("ldo", C.c_int64), ("xres", C.c_void_p), ("ln_g", C.c_void_p), ("ln_b", C.c_void_p),
        ("xn", C.c_void_p), ("path_out", C.c_int32),
    ]


class _SearchDesc(C.Structure):  # b2w_search_desc
    _fields_ = [
        ("cfg", C.POINTER(_Config)), ("opts", C.POINTER(_GenOpts)), ("prompt", C.c_void_p), ("P", C.c_int32), ("n", C.c_int32),
        ("K", C.c_int32), ("t", C.c_int32), ("logits", C.c_void_p), ("hist", C.c_void_p), ("anc", C.c_void_p), ("cum", C.c_void_p),
        ("done", C.c_void_p), ("fin_count", C.c_void_p), ("fin_len", C.c_void_p), ("fin_score", C.c_void_p), ("fin_tok", C.c_void_p),
        ("cand_score", C.c_void_p), ("cand_tok", C.c_void_p), ("no_speech", C.c_void_p), ("tokens_in", C.c_void_p), ("pos", C.c_void_p),
        ("n_done", C.c_int32),
    ]


MAX_FINISHED = 48  # include/b200whisper.h B2W_MAX_FINISHED: finished-hypothesis slots per chunk


def _make_config(dims: WhisperDims, tokens: SpecialTokens) -> _Config:
    cfg = _Config()
    for k in ("n_mels", "n_audio_ctx", "n_audio_state", "n_audio_head", "n_audio_layer", "n_vocab", "n_text_ctx",
              "n_text_state", "n_text_head", "n_text_layer"):
        setattr(cfg, k, getattr(dims, k))
    for k in ("eot", "sot", "lang_begin", "num_languages", "translate", "transcribe", "sot_lm", "sot_prev",
              "no_speech", "no_timestamps", "timestamp_begin"):
        setattr(cfg, k, getattr(tokens, k))
    begin = [220, tokens.eot]
    cfg.n_suppress_begin = len(begin)
    for i, t in enumerate(begin):
        cfg.suppress_begin[i] = t
    return cfg


def _gen_opts(lib, n_text_ctx: int, *, beam_size: int = 5, patience: float = 1, num_hypotheses: int = 1, length_penalty: float = 1,
              repetition_penalty: float = 1, no_repeat_ngram_size: int = 0, max_length: int = 448, return_scores: bool = False,
              return_no_speech_prob: bool = False, max_initial_timestamp_index: int = 50, suppress_blank: bool = True,
              suppress_tokens: Optional[Sequence[int]] = (-1,), sampling_topk: int = 1, sampling_temperature: float = 1, seed: int = 0,
              fake_logits: bool = False) -> Tuple[_GenOpts, np.ndarray]:
    """b2w_gen_opts of Whisper.generate's keyword arguments, and the suppress-id array it points to (keep it alive).  Negative
    suppress_tokens (the -1 that faster-whisper expands to the model's list itself) are dropped."""
    sup = [int(t) for t in (suppress_tokens or []) if int(t) >= 0]
    sup_arr = np.asarray(sorted(set(sup)), dtype=np.int32)
    o = _GenOpts()
    lib.b2w_gen_opts_default(C.byref(o))
    o.beam_size = int(beam_size)
    o.patience = float(patience)
    o.num_hypotheses = int(num_hypotheses)
    o.length_penalty = float(length_penalty)
    o.repetition_penalty = float(repetition_penalty)
    o.no_repeat_ngram_size = int(no_repeat_ngram_size)
    o.max_length = int(min(max_length, n_text_ctx))
    o.return_scores = int(bool(return_scores))
    o.return_no_speech_prob = int(bool(return_no_speech_prob))
    o.max_initial_timestamp_index = int(max_initial_timestamp_index)
    o.suppress_blank = int(bool(suppress_blank))
    o.suppress_tokens = sup_arr.ctypes.data_as(C.POINTER(C.c_int32)) if sup_arr.size else None
    o.n_suppress_tokens = int(sup_arr.size)
    o.sampling_topk = int(sampling_topk)
    o.sampling_temperature = float(sampling_temperature)
    o.seed = int(seed)
    o.debug_fake_logits = int(bool(fake_logits))
    return o, sup_arr


# dense GEMM epilogues (include/b200whisper.h B2W_EPI_*) and decode GEMM modes (B2W_GV_*)
EPI_F16, EPI_GELU_F16, EPI_RESID_F32, EPI_GELU_POS_F32, EPI_F16_XKV, EPI_F32, EPI_QKV_CACHE = range(7)
EPI_F16_OUT = (EPI_F16, EPI_GELU_F16, EPI_F16_XKV, EPI_QKV_CACHE)
GV_QKV, GV_F16, GV_GELU_F16, GV_RESID_LN, GV_F32 = range(5)


# every symbol include/b200whisper.h declares (checked by tests/test_abi.py)
ABI_SYMBOLS = (
    "b2w_last_error", "b2w_abi_version", "b2w_device_count", "b2w_model_create", "b2w_model_destroy",
    "b2w_model_info", "b2w_model_sync", "b2w_logmel", "b2w_logmel_frames", "b2w_encode", "b2w_encode_audio",
    "b2w_encoded_shape", "b2w_encoded_to_host", "b2w_encoded_free", "b2w_encoded_split", "b2w_memory_get", "b2w_generate",
    "b2w_gen_opts_default", "b2w_detect_language", "b2w_align", "b2w_align_batch", "b2w_align_items", "b2w_model_set_alignment_heads", "b2w_timing_enable", "b2w_timing_reset", "b2w_timing_get", "b2w_span_begin", "b2w_span_end",
    "b2w_counters_get", "b2w_debug_gemm", "b2w_debug_gemm_fp8", "b2w_debug_quantize_e4m3", "b2w_debug_layernorm_e4m3", "b2w_debug_attention", "b2w_debug_gemv", "b2w_debug_logits", "b2w_debug_fetch",
    "b2w_debug_step_logits", "b2w_debug_self_attn", "b2w_debug_cross_attn", "b2w_debug_search", "b2w_debug_align_cost", "b2w_debug_dtw", "b2w_vad_create", "b2w_vad_destroy", "b2w_vad_probs", "b2w_vad_probs_multi", "b2w_vad_set_block", "b2w_vad_timing",
    "b2w_session_create", "b2w_session_push", "b2w_session_run", "b2w_session_pending", "b2w_session_counters", "b2w_session_destroy",
    "b2w_session_debug_record", "b2w_session_debug_logits",
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
        lib.b2w_encoded_split.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(C.c_void_p)]
        lib.b2w_memory_get.argtypes = [C.c_void_p, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]
        lib.b2w_generate.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.POINTER(_GenOpts),
                                     C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        lib.b2w_gen_opts_default.argtypes = [C.POINTER(_GenOpts)]
        lib.b2w_gen_opts_default.restype = None
        lib.b2w_detect_language.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        lib.b2w_align.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_int32,
                                  C.c_void_p, C.c_int32, C.POINTER(C.c_int32), C.c_void_p]
        lib.b2w_align_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32,
                                        C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]
        lib.b2w_align_items.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p,
                                        C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]
        lib.b2w_model_set_alignment_heads.argtypes = [C.c_void_p, C.c_void_p, C.c_int32]
        lib.b2w_timing_enable.argtypes = [C.c_void_p, C.c_int32]
        lib.b2w_timing_reset.argtypes = [C.c_void_p]
        lib.b2w_timing_get.argtypes = [C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_int64)]
        lib.b2w_span_begin.argtypes = [C.c_void_p]
        lib.b2w_span_end.argtypes = [C.c_void_p, C.POINTER(C.c_double)]
        lib.b2w_counters_get.argtypes = [C.c_void_p, C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.POINTER(C.c_double)]
        lib.b2w_debug_gemm.argtypes = [C.c_int32, C.c_int32, C.POINTER(_GemmDesc)]
        lib.b2w_debug_gemm_fp8.argtypes = [C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32,
                                           C.c_void_p, C.c_int32, C.c_void_p, C.c_int32]
        lib.b2w_debug_quantize_e4m3.argtypes = [C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]
        lib.b2w_debug_layernorm_e4m3.argtypes = [C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p,
                                                 C.c_void_p]
        lib.b2w_debug_attention.argtypes = [C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p]
        lib.b2w_debug_gemv.argtypes = [C.c_int32, C.c_int32, C.POINTER(_GemvDesc)]
        lib.b2w_debug_logits.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p]
        lib.b2w_debug_fetch.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_int64]
        lib.b2w_debug_step_logits.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                              C.c_void_p, C.c_void_p, C.c_void_p]
        lib.b2w_debug_self_attn.argtypes = [C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32,
                                            C.c_int32, C.c_int32, C.c_int32, C.c_void_p]
        lib.b2w_debug_cross_attn.argtypes = [C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p]
        lib.b2w_debug_search.argtypes = [C.c_int32, C.POINTER(_SearchDesc)]
        lib.b2w_debug_align_cost.argtypes = [C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                             C.c_void_p]
        lib.b2w_debug_dtw.argtypes = [C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.POINTER(C.c_int32)]
        lib.b2w_vad_create.argtypes = [C.c_int32, C.POINTER(_Tensor), C.c_int32, C.POINTER(C.c_void_p)]
        lib.b2w_vad_destroy.argtypes = [C.c_void_p]
        lib.b2w_vad_destroy.restype = None
        lib.b2w_vad_probs.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64]
        lib.b2w_vad_probs_multi.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_int64), C.c_int32, C.c_void_p,
                                            C.c_int64]
        lib.b2w_vad_set_block.argtypes = [C.c_void_p, C.c_int64]
        lib.b2w_vad_timing.argtypes = [C.c_void_p, C.POINTER(C.c_double)]
        lib.b2w_session_create.argtypes = [C.c_void_p, C.POINTER(_GenOpts), C.POINTER(C.c_int32), C.POINTER(C.c_void_p)]
        lib.b2w_session_push.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.POINTER(C.c_int32)]
        lib.b2w_session_run.argtypes = [C.c_void_p, C.POINTER(C.c_int32), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        lib.b2w_session_pending.argtypes = [C.c_void_p, C.POINTER(C.c_int32)]
        lib.b2w_session_counters.argtypes = [C.c_void_p, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]
        lib.b2w_session_debug_record.argtypes = [C.c_void_p]
        lib.b2w_session_debug_logits.argtypes = [C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.POINTER(C.c_int32)]
        lib.b2w_session_destroy.argtypes = [C.c_void_p]
        lib.b2w_session_destroy.restype = None
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


# float8_float16: the encoder's linear layers as e4m3 tensor-core GEMMs, everything else as float16 (include/b200whisper.h)
_COMPUTE_TYPES = ("default", "auto", "int8", "int8_float32", "int8_float16", "int8_bfloat16", "int16", "float16",
                  "bfloat16", "float32", "float8_float16")


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
        cfg = _make_config(dims, self.tokens)
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

    def _pick_replica(self, replica: Optional[int]) -> _Replica:
        return self._next_replica() if replica is None else self._replicas[replica]

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
    def encode(self, features: Union[StorageView, np.ndarray], to_cpu: bool = False, replica: Optional[int] = None) -> StorageView:
        """``replica``: the replica (index) that encodes and holds the output; None takes the next one in round-robin order."""
        arr = features.numpy() if isinstance(features, StorageView) else np.asarray(features)
        if arr.dtype != np.float32 or not arr.flags["C_CONTIGUOUS"]:
            arr = np.ascontiguousarray(arr, dtype=np.float32)
        if arr.ndim != 3 or arr.shape[1] != self.dims.n_mels or arr.shape[2] != 3000:
            raise ValueError(f"Invalid input features shape: expected an input with shape (batch, {self.dims.n_mels}, 3000), "
                             f"but got an input with shape {tuple(arr.shape)} instead")
        rep = self._pick_replica(replica)
        h = C.c_void_p()
        with rep.lock:
            _check(rep._lib.b2w_encode(rep.handle, _ptr(arr), arr.shape[0], C.byref(h)))
        sv = StorageView(handle=h, owner=self, shape=(arr.shape[0], self.dims.n_audio_ctx, self.dims.n_audio_state))
        sv._replica = rep
        rep.track_output(sv)
        if to_cpu:
            return StorageView.from_array(sv.numpy())
        return sv

    def encode_audio(self, chunks: Sequence[np.ndarray], return_features: bool = False, replica: Optional[int] = None):
        """Fused log-mel + encoder for <=30 s chunks (the batched pipeline's hot path): PCM in, encoder output
        resident on the device.  Mirrors ``feature_extractor(chunk)[..., :-1]`` + ``pad_or_trim`` + ``encode``
        (transcribe.py:463-467,514-516,209).  ``replica`` as in ``encode``."""
        rep = self._pick_replica(replica)
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
        o, sup_arr = _gen_opts(rep._lib, self.dims.n_text_ctx, beam_size=beam_size, patience=patience, num_hypotheses=num_hypotheses,
                               length_penalty=length_penalty, repetition_penalty=repetition_penalty,
                               no_repeat_ngram_size=no_repeat_ngram_size, max_length=max_length, return_scores=return_scores,
                               return_no_speech_prob=return_no_speech_prob, max_initial_timestamp_index=max_initial_timestamp_index,
                               suppress_blank=suppress_blank, suppress_tokens=suppress_tokens, sampling_topk=sampling_topk,
                               sampling_temperature=sampling_temperature, seed=seed, fake_logits=_fake_logits)
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

    def decode_queue(self, *, beam_size: int = 5, patience: float = 1, num_hypotheses: int = 1, length_penalty: float = 1,
                     repetition_penalty: float = 1, no_repeat_ngram_size: int = 0, max_length: int = 448, return_scores: bool = False,
                     return_no_speech_prob: bool = False, max_initial_timestamp_index: int = 50, suppress_blank: bool = True,
                     suppress_tokens: Optional[Sequence[int]] = (-1,), sampling_topk: int = 1, sampling_temperature: float = 1,
                     seed: int = 0, slots: int = 0, replica: Optional[int] = 0) -> "DecodeQueue":
        """A continuous-batching decoder with ``generate``'s options: ``push`` items, iterate ``(item_id, WhisperGenerationResult)``
        in completion order.  A finished item's rows take the next queued item instead of idling until a whole batch ends.
        ``slots``: chunks decoded at once (0: as many as one decode step takes, 80 // rows per chunk).  ``replica``: the replica
        (index) that decodes, and whose encoder outputs ``push`` takes (the queue's ``replica``); None takes the next one in
        round-robin order."""
        rep = self._pick_replica(replica)
        o, sup_arr = _gen_opts(rep._lib, self.dims.n_text_ctx, beam_size=beam_size, patience=patience, num_hypotheses=num_hypotheses,
                               length_penalty=length_penalty, repetition_penalty=repetition_penalty,
                               no_repeat_ngram_size=no_repeat_ngram_size, max_length=max_length, return_scores=return_scores,
                               return_no_speech_prob=return_no_speech_prob, max_initial_timestamp_index=max_initial_timestamp_index,
                               suppress_blank=suppress_blank, suppress_tokens=suppress_tokens, sampling_topk=sampling_topk,
                               sampling_temperature=sampling_temperature, seed=seed)
        return DecodeQueue(self, rep, o, sup_arr, slots)

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

    def split_encoded(self, storage_view: StorageView) -> List[StorageView]:
        """One single-item device encoder output per batch item of ``storage_view`` (from ``encode`` or ``encode_audio``), each a
        bit-identical copy in device memory of its own: a chunk's output can then be freed as soon as that chunk is done, whatever
        the rest of its batch does.  ``storage_view`` is unchanged."""
        if not isinstance(storage_view, StorageView) or storage_view._handle is None:
            raise ValueError("split_encoded takes a device encoder output (a StorageView from encode / encode_audio)")
        rep = self._replica_for(storage_view)
        B = storage_view.shape[0]
        hs = (C.c_void_p * B)()
        with rep.lock:
            _check(rep._lib.b2w_encoded_split(rep.handle, storage_view._handle, hs))
        out = []
        for b in range(B):
            sv = StorageView(handle=C.c_void_p(hs[b]), owner=self, shape=(1, self.dims.n_audio_ctx, self.dims.n_audio_state))
            sv._replica = rep
            rep.track_output(sv)
            out.append(sv)
        return out

    def memory(self, replica: int = 0) -> Dict[str, int]:
        """Device bytes of this model's live encoder outputs (``encoded_bytes``, including those only a decode queue still holds)
        and of the buffers parked in its pool for reuse (``pool_bytes``)."""
        rep = self._replicas[replica]
        enc, pool = C.c_int64(), C.c_int64()
        with rep.lock:
            _check(rep._lib.b2w_memory_get(rep.handle, C.byref(enc), C.byref(pool)))
        return dict(encoded_bytes=int(enc.value), pool_bytes=int(pool.value))

    # ---- align (transcribe.py:1709-1715) ----
    def align(self, features, start_sequence, text_tokens, num_frames, *, median_filter_width: int = 7):
        """``ctranslate2.models.Whisper.align`` (transcribe.py:1709-1715): one result per batch item with ``.alignments``
        (list of (text_token_index, time_index)) and ``.text_token_probs``."""
        enc = self._as_encoded(features)
        if len(text_tokens) != enc.shape[0]:
            raise ValueError("align: one text token list per batch item is required")
        B = enc.shape[0]
        frames = [num_frames[b] if isinstance(num_frames, (list, tuple)) else num_frames for b in range(B)]
        return self.align_items([(enc, b) for b in range(B)], start_sequence, text_tokens, frames, median_filter_width=median_filter_width)

    def align_items(self, pairs: Sequence[Tuple[StorageView, int]], start_sequence, text_tokens, num_frames, *,
                    median_filter_width: int = 7) -> List[WhisperAlignmentResult]:
        """``align`` over items of several encoder outputs: item j is batch index ``pairs[j][1]`` of the device encoder output
        ``pairs[j][0]``, with ``text_tokens[j]`` and ``num_frames[j]``.  One result per item, in order."""
        pairs = list(pairs)
        B = len(pairs)
        if len(text_tokens) != B or len(num_frames) != B:
            raise ValueError("align_items: one text token list and one frame count per item are required")
        if B == 0:
            return []
        for sv, _ in pairs:
            if not isinstance(sv, StorageView) or sv._handle is None:
                raise ValueError("align_items takes device encoder outputs (StorageViews from encode / encode_audio)")
        rep = self._replica_for(pairs[0][0])
        if any(self._replica_for(sv) is not rep for sv, _ in pairs):
            raise ValueError("align_items: every encoder output must belong to one replica")
        encs = (C.c_void_p * B)(*[sv._handle.value for sv, _ in pairs])
        items = np.ascontiguousarray([int(i) for _, i in pairs], np.int32)
        start = np.ascontiguousarray(list(start_sequence), dtype=np.int32)
        texts = [np.asarray(list(t), dtype=np.int32) for t in text_tokens]
        frames = np.ascontiguousarray([int(f) for f in num_frames], np.int32)
        offsets = np.zeros(B + 1, np.int32)
        offsets[1:] = np.cumsum([len(t) for t in texts])
        toks = np.ascontiguousarray(np.concatenate(texts) if offsets[-1] else np.zeros(1, np.int32), dtype=np.int32)
        cap = int(sum(len(t) + max(1, min(1500, nf // 2)) + 1 for t, nf in zip(texts, frames) if len(t)))
        out_pairs = np.zeros((max(1, cap), 2), np.int32)
        pair_offsets = np.zeros(B + 1, np.int32)
        probs = np.zeros(max(1, int(offsets[-1])), np.float32)
        with rep.lock:
            _check(rep._lib.b2w_align_items(rep.handle, encs, _ptr(items), B, _ptr(start), len(start), _ptr(toks), _ptr(offsets),
                                            _ptr(frames), int(median_filter_width), _ptr(out_pairs), cap, _ptr(pair_offsets), _ptr(probs)))
        return [WhisperAlignmentResult([tuple(p) for p in out_pairs[pair_offsets[b]:pair_offsets[b + 1]].tolist()],
                                       probs[offsets[b]:offsets[b + 1]].tolist()) for b in range(B)]

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

    def debug_step_logits(self, enc: StorageView, prompts: np.ndarray, tokens: np.ndarray, parents: Optional[np.ndarray] = None) -> np.ndarray:
        """Teacher-forced run of the decode-step path generate() would take for n chunks x K rows (tests only).

        prompts [n, P]: positions 0..P-2 are prefilled.  tokens [n_steps, n, K]: step t feeds tokens[t, b, k] at position P-1+t.
        parents [n_steps, n, K] (row 0 unused): the slot of the same chunk whose history the row continues, as after a beam
        search's reordering; None keeps every slot on its own history.  Returns logits [n_steps, n, K, n_vocab]."""
        prompts = np.ascontiguousarray(prompts, dtype=np.int32)
        tokens = np.ascontiguousarray(tokens, dtype=np.int32)
        n, P = prompts.shape
        n_steps, tn, K = tokens.shape
        if tn != n:
            raise ValueError("tokens must be [n_steps, n_chunks, rows_per_chunk]")
        if parents is not None:
            parents = np.ascontiguousarray(parents, dtype=np.int32)
            if parents.shape != tokens.shape:
                raise ValueError("parents must have the shape of tokens")
        out = np.empty((n_steps, n, K, self.dims.n_vocab), dtype=np.float32)
        rep = self._replica_for(enc)
        with rep.lock:
            _check(rep._lib.b2w_debug_step_logits(rep.handle, enc._handle, _ptr(prompts), P, n, K, n_steps, _ptr(tokens), _ptr(parents),
                                                  _ptr(out)))
        return out

    def debug_search(self, logits: np.ndarray, prompt: Sequence[int], t: int, **kw) -> Dict[str, np.ndarray]:
        """One step of the on-device search on caller-supplied state (tests only); see ``debug_search``.  The generate options
        (beam_size, suppress_tokens, ...) are taken as ``generate`` takes them."""
        return debug_search(self.dims, self.tokens, logits, prompt, t, device=self._device_index[0], **kw)

    def debug_fetch(self, which: int, n: int, replica: int = 0) -> np.ndarray:
        """Decoder workspace buffer `which` of the last decode step as float32 (tests / tools only)."""
        out = np.empty(int(n), dtype=np.float32)
        rep = self._replicas[replica]
        with rep.lock:
            _check(rep._lib.b2w_debug_fetch(rep.handle, int(which), _ptr(out), int(n)))
        return out


def check_queue_items(prompts, max_lengths, n_vocab: int, sot: int, max_length: int) -> List[Tuple[np.ndarray, int]]:
    """The checks b2w_session_push makes, over every item before any is queued, so a rejected push queues nothing."""
    if len(max_lengths) != len(prompts):
        raise ValueError("one max_length per prompt is required")
    items = []
    for p, ml in zip(prompts, max_lengths):
        pr = np.ascontiguousarray(np.asarray(list(map(int, p)), dtype=np.int32))
        if pr.size == 0:
            raise ValueError("empty prompt")
        if pr.min() < 0 or pr.max() >= n_vocab:
            raise ValueError("prompt token id out of range")
        if sot not in pr:
            raise ValueError("<|startoftranscript|> token was not found in the prompt")
        if not (pr.size < int(ml) <= max_length):
            raise ValueError("max_length must exceed the prompt length and be at most the session's max_length")
        items.append((pr, int(ml)))
    return items


class DecodeQueue:
    """A native decode session (``Whisper.decode_queue``).  Items are decoded in a fixed set of slots; ``push`` queues them,
    iteration yields ``(item_id, WhisperGenerationResult)`` as they finish (ids count pushes from 0).  Each pushed encoder output
    is kept alive on the device until the session no longer reads it."""

    def __init__(self, owner: "Whisper", rep: _Replica, opts: _GenOpts, sup_arr: np.ndarray, slots: int = 0):
        self._owner, self._rep, self._opts, self._sup = owner, rep, opts, sup_arr
        self.replica = owner._replicas.index(rep)
        self._return_scores = bool(opts.return_scores)
        self._return_ns = bool(opts.return_no_speech_prob)
        h, slots = C.c_void_p(), C.c_int32(int(slots))
        with rep.lock:
            _check(rep._lib.b2w_session_create(rep.handle, C.byref(opts), C.byref(slots), C.byref(h)))
        self._h = h
        self.slots = int(slots.value)
        H, L = max(1, opts.num_hypotheses), opts.max_length
        self._ids = np.zeros((self.slots, H, L), np.int32)
        self._lens = np.zeros((self.slots, H), np.int32)
        self._scores = np.zeros((self.slots, H), np.float32)
        self._ns = np.zeros((self.slots,), np.float32)
        self._items = np.zeros((self.slots,), np.int32)

    def push(self, storage_view: StorageView, prompts: Sequence[Sequence[int]], max_lengths: Optional[Sequence[int]] = None) -> List[int]:
        """Queues item i of ``storage_view`` (a device encoder output of this model) with ``prompts[i]`` (lengths may differ)
        and ``max_lengths[i]`` (default: the queue's ``max_length``).  Returns the items' ids."""
        if not isinstance(storage_view, StorageView) or storage_view._handle is None:
            raise ValueError("push takes a device encoder output (a StorageView from encode / encode_audio)")
        if self._owner._replica_for(storage_view) is not self._rep:
            raise ValueError("the encoder output belongs to another replica")
        if len(prompts) != storage_view.shape[0]:
            raise ValueError("the number of prompts must match the batch size of the encoder output")
        if max_lengths is None:
            max_lengths = [self._opts.max_length] * len(prompts)
        items = check_queue_items(prompts, max_lengths, self._owner.dims.n_vocab, self._owner.tokens.sot, self._opts.max_length)
        ids = []
        for i, (pr, ml) in enumerate(items):
            out = C.c_int32()
            with self._rep.lock:
                _check(self._rep._lib.b2w_session_push(self._handle(), storage_view._handle, i, _ptr(pr), pr.shape[0], int(ml), C.byref(out)))
            ids.append(int(out.value))
        return ids

    def _handle(self):
        if not self._h:
            raise RuntimeError("the decode queue is closed")
        return self._h

    def debug_record(self):
        """Test hook: record every step's raw logits of each occupied slot (one row per slot only); call before the first run."""
        with self._rep.lock:
            _check(self._rep._lib.b2w_session_debug_record(self._handle()))

    def debug_logits(self, item_id: int) -> np.ndarray:
        """[steps][n_vocab] logits recorded for a finished item, from its first step (the last ones may be idle steps)."""
        cap = self._owner.dims.n_text_ctx
        out = np.zeros((cap, self._owner.dims.n_vocab), np.float32)
        n = C.c_int32()
        with self._rep.lock:
            _check(self._rep._lib.b2w_session_debug_logits(self._handle(), int(item_id), _ptr(out), cap, C.byref(n)))
        return out[: n.value]

    def pending(self) -> int:
        n = C.c_int32()
        with self._rep.lock:
            _check(self._rep._lib.b2w_session_pending(self._handle(), C.byref(n)))
        return int(n.value)

    def counters(self) -> Tuple[int, int]:
        """(decode steps run, rows of occupied slots summed over the steps)."""
        st, rows = C.c_int64(), C.c_int64()
        with self._rep.lock:
            _check(self._rep._lib.b2w_session_counters(self._handle(), C.byref(st), C.byref(rows)))
        return int(st.value), int(rows.value)

    def run(self) -> List[Tuple[int, WhisperGenerationResult]]:
        """Decodes until at least one item finishes; [] when nothing is queued or decoding."""
        n = C.c_int32()
        with self._rep.lock:
            _check(self._rep._lib.b2w_session_run(self._handle(), C.byref(n), _ptr(self._items), _ptr(self._ids), _ptr(self._lens),
                                                  _ptr(self._scores), _ptr(self._ns)))
        out = []
        for j in range(n.value):
            H = self._lens.shape[1]
            out.append((int(self._items[j]), WhisperGenerationResult(
                sequences_ids=[self._ids[j, h, : self._lens[j, h]].tolist() for h in range(H)],
                scores=[float(x) for x in self._scores[j]] if self._return_scores else [],
                no_speech_prob=float(self._ns[j]) if self._return_ns else 0.0)))
        return out

    def __iter__(self):
        while True:
            done = self.run()
            if not done:
                return
            yield from done

    def close(self):
        h, self._h = getattr(self, "_h", None), None
        if h and self._rep._h:  # the session must go before its model; after unload_model its buffers go with the device context
            self._rep._lib.b2w_session_destroy(h)

    def __del__(self):
        try:
            self.close()
        except Exception:  # noqa: BLE001
            pass


class SileroVad:
    """The Silero VAD v6 network on one GPU (``b2w_vad_*``): ``probs(pcm)`` returns one speech probability per 512-sample window.
    ``weights`` are the arrays ``silero.load_weights`` returns (names and shapes in include/b200whisper.h)."""

    def __init__(self, weights: Dict[str, np.ndarray], device: int = 0, block_windows: Optional[int] = None):
        lib = load_library()
        keep, tensors = [], []
        for name, arr in weights.items():
            arr = np.ascontiguousarray(arr, dtype=np.float32)
            keep.append(arr)
            t = _Tensor(name=name.encode(), data=arr.ctypes.data, dtype=0, ndim=arr.ndim)
            for i, n in enumerate(arr.shape[:4]):
                t.shape[i] = n
            tensors.append(t)
        arr_t = (_Tensor * max(len(tensors), 1))(*tensors)
        h = C.c_void_p()
        _check(lib.b2w_vad_create(device, arr_t, len(tensors), C.byref(h)))
        self._lib, self._h = lib, h
        if block_windows is not None:
            _check(lib.b2w_vad_set_block(h, block_windows))

    def probs(self, pcm: np.ndarray) -> np.ndarray:
        x = np.ascontiguousarray(pcm, dtype=np.float32)
        out = np.empty(x.shape[0] // 512, np.float32)
        _check(self._lib.b2w_vad_probs(self._h, _ptr(x), x.shape[0], _ptr(out), out.shape[0]))
        return out

    def probs_many(self, pcms: Sequence[np.ndarray]) -> List[np.ndarray]:
        """``probs`` of several independent recordings in one sequence of launches (``b2w_vad_probs_multi``); each result is
        bit-identical to ``probs`` of that recording alone."""
        xs = [np.ascontiguousarray(p, dtype=np.float32) for p in pcms]
        if not xs:
            return []
        ptrs = (C.c_void_p * len(xs))(*[x.ctypes.data for x in xs])
        lens = (C.c_int64 * len(xs))(*[x.shape[0] for x in xs])
        out = np.empty(max(sum(x.shape[0] // 512 for x in xs), 1), np.float32)
        _check(self._lib.b2w_vad_probs_multi(self._h, ptrs, lens, len(xs), _ptr(out), out.shape[0]))
        bounds = np.cumsum([0] + [x.shape[0] // 512 for x in xs])
        return [out[lo:hi].copy() for lo, hi in zip(bounds[:-1], bounds[1:])]

    def timing(self) -> Dict[str, float]:
        """Device milliseconds of the last ``probs`` or ``probs_many`` call per kernel."""
        ms = (C.c_double * 3)()
        _check(self._lib.b2w_vad_timing(self._h, ms))
        return dict(zip(("window", "recurrence", "decoder"), ms))

    def close(self):
        if getattr(self, "_h", None):
            self._lib.b2w_vad_destroy(self._h)
            self._h = None

    def __del__(self):
        self.close()


class models:  # namespace shim so `ctranslate2.models.Whisper` style access works on this module
    Whisper = Whisper
    WhisperGenerationResult = WhisperGenerationResult


def _buf(x: Optional[np.ndarray], dtype, name: str) -> Optional[np.ndarray]:
    """A host buffer the hooks read or update in place: it must already have the dtype and be C-contiguous."""
    if x is None:
        return None
    if x.dtype != dtype or not x.flags["C_CONTIGUOUS"]:
        raise ValueError(f"{name} must be a C-contiguous {np.dtype(dtype).name} array")
    return x


def debug_gemm_desc(a: np.ndarray, w: np.ndarray, out: np.ndarray, *, epilogue: int, rows: int, a_batch: int = 1,
                    a_rows: Optional[int] = None, a_cols: Optional[int] = None, a_row_stride: Optional[int] = None,
                    a_batch_stride: int = 0, tap_row: Sequence[int] = (0,), tap_col: Sequence[int] = (0,),
                    bias: Optional[np.ndarray] = None, out_ld: Optional[int] = None, out_batch_stride: int = 0,
                    narrow_tiles: bool = False, pos: Optional[np.ndarray] = None, xkv: Tuple[int, int, int, int] = (0, 0, 0, 0),
                    rowinfo: Optional[np.ndarray] = None, kcache: Optional[np.ndarray] = None, vcache: Optional[np.ndarray] = None,
                    qkv_d: int = 0, n_ctx: int = 0, slots: int = 0, max_ctas: int = 0, impl: int = 0, device: int = 0) -> Tuple[int, int]:
    """One dense GEMM as the engine states it (b2w_gemm_desc; tests only).  a: float16 buffer of A, w: float16 [N, taps*k_per_tap],
    out (float16 or float32 by epilogue) and the caches are updated in place; xkv = (d, heads, T, B).  Returns the (tile width,
    grid) the plan chose (0, 0 for the reference)."""
    lib = load_library()
    a, w = _buf(a, np.float16, "a"), _buf(w, np.float16, "w")
    out = _buf(out, np.float16 if epilogue in EPI_F16_OUT else np.float32, "out")
    bias = None if bias is None else np.ascontiguousarray(bias, np.float32)
    pos = None if pos is None else np.ascontiguousarray(pos, np.float32)
    rowinfo = None if rowinfo is None else np.ascontiguousarray(rowinfo, np.int32)
    kcache, vcache = _buf(kcache, np.float16, "kcache"), _buf(vcache, np.float16, "vcache")
    if len(tap_row) != len(tap_col) or not 1 <= len(tap_row) <= 3:
        raise ValueError("1..3 taps, one row and one column offset each")
    N, K = w.shape
    taps = len(tap_row)
    d = _GemmDesc()
    d.a, d.a_elems, d.a_batch = _ptr(a), a.size, a_batch
    d.a_rows = rows if a_rows is None else a_rows
    d.a_cols = K // taps if a_cols is None else a_cols
    d.a_row_stride = d.a_cols if a_row_stride is None else a_row_stride
    d.a_batch_stride = a_batch_stride
    d.taps, d.k_per_tap = taps, K // taps
    d.tap_row[:] = list(tap_row) + [0] * (3 - taps)
    d.tap_col[:] = list(tap_col) + [0] * (3 - taps)
    d.w, d.bias, d.N, d.rows, d.epilogue, d.narrow_tiles = _ptr(w), _ptr(bias), N, rows, epilogue, int(narrow_tiles)
    d.out, d.out_elems = _ptr(out), out.size
    d.out_ld = N if out_ld is None else out_ld
    d.out_batch_stride, d.pos = out_batch_stride, _ptr(pos)
    d.xkv_d, d.xkv_heads, d.xkv_T, d.xkv_B = xkv
    d.rowinfo, d.kcache, d.vcache = _ptr(rowinfo), _ptr(kcache), _ptr(vcache)
    d.cache_elems = 0 if kcache is None else min(kcache.size, vcache.size if vcache is not None else 0)
    d.qkv_d, d.n_ctx, d.slots, d.max_ctas = qkv_d, n_ctx, slots, max_ctas
    _check(lib.b2w_debug_gemm(device, impl, C.byref(d)))
    return d.block_n_out, d.grid_out


def debug_gemm(a: np.ndarray, w: np.ndarray, bias: Optional[np.ndarray], impl: int = 0, gelu: bool = False, device: int = 0):
    """C = A W^T + bias (or fp16 GELU of it) for float32 A [M, K], W [N, K] rounded to fp16; float32 result."""
    a16 = np.ascontiguousarray(a, np.float32).astype(np.float16)
    w16 = np.ascontiguousarray(w, np.float32).astype(np.float16)
    out = np.zeros((a16.shape[0], w16.shape[0]), np.float16 if gelu else np.float32)
    debug_gemm_desc(a16, w16, out, epilogue=EPI_GELU_F16 if gelu else EPI_F32, rows=a16.shape[0], bias=bias, impl=impl, device=device)
    return out.astype(np.float32)


def debug_gemm_fp8(a: np.ndarray, a_scale: np.ndarray, w: np.ndarray, w_scale: np.ndarray, out: np.ndarray, *, epilogue: int,
                   bias: Optional[np.ndarray] = None, max_ctas: int = 0, device: int = 0) -> None:
    """The encoder's e4m3 GEMM (b2w_debug_gemm_fp8; tests only): a uint8 codes [rows, K], w uint8 codes [N, K], float32 row /
    channel scales; out (float16 [rows, N] for EPI_F16 / EPI_GELU_F16, float32 for EPI_RESID_F32) is updated in place."""
    lib = load_library()
    a, w = _buf(a, np.uint8, "a"), _buf(w, np.uint8, "w")
    a_scale, w_scale = _buf(a_scale, np.float32, "a_scale"), _buf(w_scale, np.float32, "w_scale")
    out = _buf(out, np.float16 if epilogue in EPI_F16_OUT else np.float32, "out")
    bias = None if bias is None else np.ascontiguousarray(bias, np.float32)
    (rows, K), N = a.shape, w.shape[0]
    if w.shape[1] != K or a_scale.shape != (rows,) or w_scale.shape != (N,) or out.shape != (rows, N) or (bias is not None and bias.shape != (N,)):
        raise ValueError("shapes: a [rows, K], w [N, K], a_scale [rows], w_scale [N], out [rows, N], bias [N]")
    _check(lib.b2w_debug_gemm_fp8(device, _ptr(a), _ptr(a_scale), rows, K, _ptr(w), _ptr(w_scale), N, _ptr(bias), epilogue, _ptr(out),
                                  max_ctas))


def debug_quantize_e4m3(x: np.ndarray, device: int = 0) -> Tuple[np.ndarray, np.ndarray]:
    """e4m3 codes (uint8 [rows, K]) and row scales (float32 [rows]) of float16 rows x [rows, K] (tests only)."""
    lib = load_library()
    x = _buf(x, np.float16, "x")
    rows, K = x.shape
    codes, scales = np.zeros((rows, K), np.uint8), np.zeros(rows, np.float32)
    _check(lib.b2w_debug_quantize_e4m3(device, _ptr(x), rows, K, _ptr(codes), _ptr(scales)))
    return codes, scales


def debug_layernorm_e4m3(x: np.ndarray, gamma: Optional[np.ndarray], beta: Optional[np.ndarray], device: int = 0) -> Tuple[np.ndarray, np.ndarray]:
    """e4m3 codes and row scales of the float32 LayerNorm(x) * gamma + beta of float32 rows x [rows, d] (tests only)."""
    lib = load_library()
    x = _buf(x, np.float32, "x")
    gamma = None if gamma is None else np.ascontiguousarray(gamma, np.float32)
    beta = None if beta is None else np.ascontiguousarray(beta, np.float32)
    rows, d = x.shape
    codes, scales = np.zeros((rows, d), np.uint8), np.zeros(rows, np.float32)
    _check(lib.b2w_debug_layernorm_e4m3(device, _ptr(x), _ptr(gamma), _ptr(beta), rows, d, _ptr(codes), _ptr(scales)))
    return codes, scales


def debug_attention(qkv: np.ndarray, heads: int, impl: int = 0, device: int = 0):
    lib = load_library()
    qkv = np.ascontiguousarray(qkv, np.float32)
    B, T, _ = qkv.shape
    out = np.empty((B, T, heads * 64), np.float32)
    _check(lib.b2w_debug_attention(device, impl, _ptr(qkv), B, T, heads, _ptr(out)))
    return out


def debug_gemv_desc(x: np.ndarray, w: np.ndarray, *, mode: int, bias: Optional[np.ndarray] = None, out: Optional[np.ndarray] = None,
                    ldo: int = 0, rows: Optional[np.ndarray] = None, kcache: Optional[np.ndarray] = None,
                    vcache: Optional[np.ndarray] = None, d: int = 0, n_ctx: int = 0, slots: int = 0, xres: Optional[np.ndarray] = None,
                    ln_g: Optional[np.ndarray] = None, ln_b: Optional[np.ndarray] = None, xn: Optional[np.ndarray] = None,
                    route: int = 1, impl: int = 0, device: int = 0) -> int:
    """One decoder GEMM of R = x.shape[0] <= 80 rows (b2w_gemv_desc; tests only).  x: float16 [R, K], w: float16 [N, K]; out
    (float32 for GV_F32, else float16), the caches, xres (float32) and xn (float16) are updated in place.  route 1 runs what the
    decoder runs for this shape, route 0 the skinny kernel.  Returns the path that ran: 0 skinny, 1 wgmma."""
    lib = load_library()
    x, w = _buf(x, np.float16, "x"), _buf(w, np.float16, "w")
    out = _buf(out, np.float32 if mode == GV_F32 else np.float16, "out")
    bias = None if bias is None else np.ascontiguousarray(bias, np.float32)
    rows = None if rows is None else np.ascontiguousarray(rows, np.int32)
    kcache, vcache = _buf(kcache, np.float16, "kcache"), _buf(vcache, np.float16, "vcache")
    xres, xn = _buf(xres, np.float32, "xres"), _buf(xn, np.float16, "xn")
    ln_g = None if ln_g is None else np.ascontiguousarray(ln_g, np.float32)
    ln_b = None if ln_b is None else np.ascontiguousarray(ln_b, np.float32)
    R, K = x.shape
    desc = _GemvDesc()
    desc.x, desc.w, desc.bias, desc.R, desc.N, desc.K, desc.mode, desc.route = _ptr(x), _ptr(w), _ptr(bias), R, w.shape[0], K, mode, route
    desc.rows, desc.kcache, desc.vcache = _ptr(rows), _ptr(kcache), _ptr(vcache)
    desc.cache_elems = 0 if kcache is None else min(kcache.size, vcache.size if vcache is not None else 0)
    desc.d, desc.n_ctx, desc.slots = d, n_ctx, slots
    desc.out, desc.out_elems, desc.ldo = _ptr(out), 0 if out is None else out.size, ldo
    desc.xres, desc.ln_g, desc.ln_b, desc.xn = _ptr(xres), _ptr(ln_g), _ptr(ln_b), _ptr(xn)
    _check(lib.b2w_debug_gemv(device, impl, C.byref(desc)))
    return desc.path_out


def debug_search(dims: WhisperDims, tokens: SpecialTokens, logits: np.ndarray, prompt: Sequence[int], t: int, *,
                 hist: Optional[np.ndarray] = None, anc: Optional[np.ndarray] = None, cum: Optional[np.ndarray] = None,
                 done: Optional[np.ndarray] = None, fin_count: Optional[np.ndarray] = None, fin_len: Optional[np.ndarray] = None,
                 fin_score: Optional[np.ndarray] = None, n_done: int = 0, device: int = 0, **opts) -> Dict[str, np.ndarray]:
    """One decode step of the on-device search (b2w_search_desc; tests only) for n chunks x K rows at step t.

    logits [n, K, n_vocab]; hist [n, K, t] generated tokens; anc [n, K, P-1+t] self-KV slot ancestry; cum [n, K]; done and fin_count
    [n]; fin_len / fin_score [n, MAX_FINISHED] (fin_len -1 = empty).  Missing state starts empty.  ``opts`` are generate's keyword
    arguments.  Returns the state after the step: cand_score / cand_tok [n, K, ncand], no_speech [n], hist [n, K, t+1],
    anc [n, K, P+t], cum, tokens_in, pos [n, K], done, fin_count, n_done, fin_len, fin_score, and fin_tok [n, MAX_FINISHED, t+1]
    (-1 in slots the step did not write)."""
    lib = load_library()
    logits = np.ascontiguousarray(logits, np.float32)
    n, K, V = logits.shape
    prompt = np.ascontiguousarray(list(prompt), np.int32)
    P = prompt.shape[0]
    o, sup_arr = _gen_opts(lib, dims.n_text_ctx, **opts)
    ncand = 2 * K if o.beam_size > 1 else 1

    def state(x, shape, dtype, fill=0):
        return np.full(shape, fill, dtype) if x is None else np.array(np.broadcast_to(np.asarray(x, dtype), shape), dtype)

    hist_in = state(hist, (n, K, t), np.int32)
    anc_in = state(anc, (n, K, P - 1 + t), np.uint8)
    out = dict(
        hist=np.zeros((n, K, t + 1), np.int32), anc=np.zeros((n, K, P + t), np.uint8), cum=state(cum, (n, K), np.float32),
        done=state(done, (n,), np.int32), fin_count=state(fin_count, (n,), np.int32),
        fin_len=state(fin_len, (n, MAX_FINISHED), np.int32, -1), fin_score=state(fin_score, (n, MAX_FINISHED), np.float32),
        fin_tok=np.zeros((n, MAX_FINISHED, t + 1), np.int32), cand_score=np.zeros((n, K, ncand), np.float32),
        cand_tok=np.zeros((n, K, ncand), np.int32), no_speech=np.zeros(n, np.float32), tokens_in=np.zeros((n, K), np.int32),
        pos=np.zeros((n, K), np.int32))
    # hist and anc are in / out with the step's extra column: the input is packed into the front of the output buffers
    out["hist"].reshape(-1)[: hist_in.size] = hist_in.reshape(-1)
    out["anc"].reshape(-1)[: anc_in.size] = anc_in.reshape(-1)
    cfg = _make_config(dims, tokens)
    d = _SearchDesc()
    d.cfg, d.opts, d.prompt = C.pointer(cfg), C.pointer(o), _ptr(prompt)
    d.P, d.n, d.K, d.t = P, n, K, int(t)
    d.logits = _ptr(logits)
    for k in ("hist", "anc", "cum", "done", "fin_count", "fin_len", "fin_score", "fin_tok", "cand_score", "cand_tok", "no_speech",
              "tokens_in", "pos"):
        setattr(d, k, _ptr(out[k]))
    d.n_done = int(n_done)
    _check(lib.b2w_debug_search(device, C.byref(d)))
    out["n_done"] = d.n_done
    return out


def debug_align_cost(capture: np.ndarray, n_start: int, n_text: int, median_filter_width: int = 7, device: int = 0) -> np.ndarray:
    """The DTW cost matrix [n_text + 1, nf] (float64) of Whisper.align from a float32 capture [n_heads, n_tok, nf] (tests only)."""
    lib = load_library()
    cap = np.ascontiguousarray(capture, np.float32)
    n_heads, n_tok, nf = cap.shape
    out = np.zeros((max(0, n_text) + 1, nf), np.float64)
    _check(lib.b2w_debug_align_cost(device, _ptr(cap), n_heads, n_tok, nf, n_start, n_text, median_filter_width, _ptr(out)))
    return out


def debug_dtw(cost: np.ndarray, capacity: Optional[int] = None, device: int = 0) -> List[Tuple[int, int]]:
    """The DTW path of Whisper.align through a float64 cost [N, M] as (row, frame) pairs (tests only)."""
    lib = load_library()
    c = np.ascontiguousarray(cost, np.float64)
    N, M = c.shape
    cap = N + M if capacity is None else capacity
    pairs = np.zeros((max(1, cap), 2), np.int32)
    n = C.c_int32(0)
    _check(lib.b2w_debug_dtw(device, _ptr(c), N, M, _ptr(pairs), cap, C.byref(n)))
    return [(int(a), int(b)) for a, b in pairs[: n.value]]


def debug_self_attn(q: np.ndarray, kcache: np.ndarray, vcache: np.ndarray, anc: np.ndarray, rows: np.ndarray, device: int = 0) -> np.ndarray:
    """The decoder's masked self-attention kernel (tests only): q float16 [R, 64 H], caches float16 [n_chunks, n_ctx, slots, 64 H],
    anc uint8 [2, n_chunks, slots, n_ctx] (a row at position p reads buffer p & 1), rows int32 [R, 4] = (chunk, slot, pos, -).
    Returns float16 [R, 64 H]."""
    lib = load_library()
    q, kcache, vcache = (np.ascontiguousarray(x, np.float16) for x in (q, kcache, vcache))
    anc, rows = np.ascontiguousarray(anc, np.uint8), np.ascontiguousarray(rows, np.int32)
    if q.ndim != 2 or q.shape[1] % 64 or kcache.ndim != 4 or kcache.shape != vcache.shape or kcache.shape[3] != q.shape[1]:
        raise ValueError("q must be [R, 64 H] and both caches [n_chunks, n_ctx, slots, 64 H]")
    n_chunks, n_ctx, slots, _ = kcache.shape
    if anc.shape != (2, n_chunks, slots, n_ctx) or rows.shape != (q.shape[0], 4):
        raise ValueError("anc must be [2, n_chunks, slots, n_ctx] and rows [R, 4]")
    out = np.zeros_like(q)
    _check(lib.b2w_debug_self_attn(device, _ptr(q), _ptr(kcache), _ptr(vcache), _ptr(anc), _ptr(rows), q.shape[0], q.shape[1] // 64,
                                   n_chunks, slots, n_ctx, _ptr(out)))
    return out


def debug_cross_attn(q: np.ndarray, kv: np.ndarray, device: int = 0) -> np.ndarray:
    """The decoder's beam-shared cross-attention kernel (tests only): q float16 [n_chunks, rows_per_chunk, 64 H], kv float16
    [2, n_chunks, H, 1500, 64] as the encoder output stores it (16-byte chunk c of key t at c ^ (t & 7)).  Returns float16
    [n_chunks, rows_per_chunk, 64 H]."""
    lib = load_library()
    q, kv = np.ascontiguousarray(q, np.float16), np.ascontiguousarray(kv, np.float16)
    if q.ndim != 3 or kv.ndim != 5 or kv.shape[0] != 2 or kv.shape[1] != q.shape[0] or kv.shape[3:] != (1500, 64) or q.shape[2] != 64 * kv.shape[2]:
        raise ValueError("q must be [n_chunks, rows_per_chunk, 64 H] and kv [2, n_chunks, H, 1500, 64]")
    out = np.zeros_like(q)
    _check(lib.b2w_debug_cross_attn(device, _ptr(q), _ptr(kv), q.shape[0], q.shape[1], kv.shape[2], _ptr(out)))
    return out


def debug_gemv(x: np.ndarray, w: np.ndarray, bias: Optional[np.ndarray], impl: int = 0, device: int = 0):
    """y = x W^T + bias through the skinny kernel (impl 0) or its reference (impl 1), float32 x [R, K], W [N, K] rounded to fp16."""
    x16 = np.ascontiguousarray(x, np.float32).astype(np.float16)
    w16 = np.ascontiguousarray(w, np.float32).astype(np.float16)
    out = np.zeros((x16.shape[0], w16.shape[0]), np.float32)
    debug_gemv_desc(x16, w16, mode=GV_F32, bias=bias, out=out, ldo=w16.shape[0], route=0, impl=impl, device=device)
    return out
