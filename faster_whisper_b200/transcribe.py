"""``WhisperModel`` and ``BatchedInferencePipeline`` with faster-whisper's public surface, driving the H100 engine.

Interface mirrored from ``faster_whisper/transcribe.py`` (reference tree): result/option dataclasses ``:31-108``,
``BatchedInferencePipeline`` ``:111-617``, ``WhisperModel`` ``:620-1841`` and the helper functions ``:1844-1941``.
Same argument names, defaults, return types and error behaviour, so a caller (or the reference's tests) can switch
imports.  The engine underneath is ``faster_whisper_b200.engine.Whisper`` (libb200whisper through ctypes) where the
reference has ``ctranslate2.models.Whisper``; the batched pipeline additionally uses the fused audio->log-mel->encoder
entry point so features never leave HBM.
"""

from __future__ import annotations

import itertools
import json
import logging
import os
import zlib
from dataclasses import asdict, dataclass
from inspect import signature
from math import ceil
from typing import BinaryIO, Iterable, Iterator, List, Optional, Tuple, Union
from warnings import warn

import numpy as np

from . import engine
from .audio import decode_audio, pad_or_trim
from .config import MODEL_DIMS
from .feature_extractor import FeatureExtractor
from .tokenizer import _LANGUAGE_CODES, Tokenizer
from .utils import download_model, format_timestamp, get_end, get_logger
from .vad import SpeechTimestampsMap, VadOptions, collect_chunks, get_speech_timestamps

_DEFAULT_TEMPERATURES = [0.0, 0.2, 0.4, 0.6, 0.8, 1.0]
_PREPEND_PUNCT = "\"'“¿([{-"
_APPEND_PUNCT = "\"'.。,，!！?？:：”)]}、"


# --------------------------------------------------------------------------------------------------
# result / option records (transcribe.py:31-108)
# --------------------------------------------------------------------------------------------------
def _deprecated_asdict(obj, name):
    warn(f"{name}._asdict() method is deprecated, use dataclasses.asdict({name}) instead", DeprecationWarning, 3)
    return asdict(obj)


@dataclass
class Word:
    start: float
    end: float
    word: str
    probability: float

    def _asdict(self):
        return _deprecated_asdict(self, "Word")


@dataclass
class Segment:
    id: int
    seek: int
    start: float
    end: float
    text: str
    tokens: List[int]
    avg_logprob: float
    compression_ratio: float
    no_speech_prob: float
    words: Optional[List[Word]]
    temperature: Optional[float]

    def _asdict(self):
        return _deprecated_asdict(self, "Segment")


@dataclass
class TranscriptionOptions:
    beam_size: int
    best_of: int
    patience: float
    length_penalty: float
    repetition_penalty: float
    no_repeat_ngram_size: int
    log_prob_threshold: Optional[float]
    no_speech_threshold: Optional[float]
    compression_ratio_threshold: Optional[float]
    condition_on_previous_text: bool
    prompt_reset_on_temperature: float
    temperatures: List[float]
    initial_prompt: Optional[Union[str, Iterable[int]]]
    prefix: Optional[str]
    suppress_blank: bool
    suppress_tokens: Optional[List[int]]
    without_timestamps: bool
    max_initial_timestamp: float
    word_timestamps: bool
    prepend_punctuations: str
    append_punctuations: str
    multilingual: bool
    max_new_tokens: Optional[int]
    clip_timestamps: Union[str, List[float]]
    hallucination_silence_threshold: Optional[float]
    hotwords: Optional[str]


@dataclass
class TranscriptionInfo:
    language: str
    language_probability: float
    duration: float
    duration_after_vad: float
    all_language_probs: Optional[List[Tuple[str, float]]]
    transcription_options: TranscriptionOptions
    vad_options: VadOptions


# --------------------------------------------------------------------------------------------------
# module-level helpers (transcribe.py:1844-1941)
# --------------------------------------------------------------------------------------------------
def get_ctranslate2_storage(segment: np.ndarray) -> engine.StorageView:
    """The host->engine hand-off: a C-contiguous float32 view (transcribe.py:1873-1876)."""
    return engine.StorageView.from_array(np.ascontiguousarray(segment))


def get_compression_ratio(text: str) -> float:
    raw = text.encode("utf-8")
    return len(raw) / len(zlib.compress(raw))


def get_suppressed_tokens(tokenizer: Tokenizer, suppress_tokens) -> Optional[Tuple[int, ...]]:
    """Expands -1 to the tokenizer's non-speech set and always adds the task/control tokens
    (transcribe.py:1884-1907); returns a sorted tuple."""
    if -1 in suppress_tokens:
        ids = [t for t in suppress_tokens if t >= 0]
        ids.extend(tokenizer.non_speech_tokens)
    elif suppress_tokens is None or len(suppress_tokens) == 0:
        ids = []
    else:
        assert isinstance(suppress_tokens, list), "suppress_tokens must be a list"
        ids = list(suppress_tokens)
    ids += [tokenizer.transcribe, tokenizer.translate, tokenizer.sot, tokenizer.sot_prev, tokenizer.sot_lm, tokenizer.no_speech]
    return tuple(sorted(set(ids)))


def merge_punctuations(alignment: List[dict], prepended: str, appended: str) -> None:
    """Glue leading punctuation onto the following word and trailing punctuation onto the previous one."""
    nxt = len(alignment) - 1
    for cur in range(len(alignment) - 2, -1, -1):
        a, b = alignment[cur], alignment[nxt]
        if a["word"].startswith(" ") and a["word"].strip() in prepended:
            b["word"] = a["word"] + b["word"]
            b["tokens"] = a["tokens"] + b["tokens"]
            a["word"], a["tokens"] = "", []
        else:
            nxt = cur
    prev = 0
    for cur in range(1, len(alignment)):
        a, b = alignment[prev], alignment[cur]
        if not a["word"].endswith(" ") and b["word"] in appended:
            a["word"] = a["word"] + b["word"]
            a["tokens"] = a["tokens"] + b["tokens"]
            b["word"], b["tokens"] = "", []
        else:
            prev = cur


def restore_speech_timestamps(segments: Iterable[Segment], speech_chunks: List[dict], sampling_rate: int) -> Iterable[Segment]:
    """Maps segment (and word) times from the VAD-concatenated axis back to the original recording."""
    ts_map = SpeechTimestampsMap(speech_chunks, sampling_rate)
    for seg in segments:
        if seg.words:
            for w in seg.words:
                idx = ts_map.get_chunk_index((w.start + w.end) / 2)  # keep both ends of a word in one chunk
                w.start = ts_map.get_original_time(w.start, idx)
                w.end = ts_map.get_original_time(w.end, idx)
            seg.start, seg.end = seg.words[0].start, seg.words[-1].end
        else:
            seg.start = ts_map.get_original_time(seg.start)
            seg.end = ts_map.get_original_time(seg.end, is_end=True)
        yield seg


def _as_temperature_list(temperature) -> List[float]:
    return list(temperature) if isinstance(temperature, (list, tuple)) else [temperature]


def _score_to_avg_logprob(score: float, n_tokens: int, length_penalty: float) -> float:
    """The engine returns cum_logprob / len**length_penalty (EOS not counted in len); Whisper's
    avg_logprob divides by len + 1 (transcribe.py:241-246, 1463-1466)."""
    return score * (n_tokens**length_penalty) / (n_tokens + 1)


def _check_max_length(prompt_len: int, max_new_tokens: Optional[int], limit: int) -> int:
    total = limit if max_new_tokens is None else prompt_len + max_new_tokens
    if total > limit:
        raise ValueError(
            f"The length of the prompt is {prompt_len}, and the `max_new_tokens` {total - prompt_len}. Thus, the combined "
            f"length of the prompt and `max_new_tokens` is: {total}. This exceeds the `max_length` of the Whisper model: "
            f"{limit}. You should either reduce the length of your prompt, or reduce the value of `max_new_tokens`, so that "
            f"their combined length is less that {limit}.")
    return total


# --------------------------------------------------------------------------------------------------
# batched pipeline (transcribe.py:111-617)
# --------------------------------------------------------------------------------------------------
class BatchedInferencePipeline:
    def __init__(self, model):
        self.model: WhisperModel = model
        self.last_speech_timestamp = 0.0

    # -- one batch: encode + one generate call + timestamp splitting ---------------------------------
    def forward(self, features, tokenizer, chunks_metadata, options):
        encoder_output, outputs = self.generate_segment_batched(features, tokenizer, options)
        model = self.model
        batch_results, frame_counts = [], []
        for meta, out in zip(chunks_metadata, outputs):
            n_frames = int(ceil(meta["duration"]) * model.frames_per_second)
            frame_counts.append(n_frames)
            pieces, _, _ = model._split_segments_by_timestamps(
                tokenizer=tokenizer, tokens=out["tokens"], time_offset=meta["offset"], segment_size=n_frames,
                segment_duration=meta["duration"], seek=0)
            rows = []
            for piece in pieces:
                text = tokenizer.decode(piece["tokens"])
                rows.append(dict(
                    text=text, avg_logprob=out["avg_logprob"], no_speech_prob=out["no_speech_prob"], tokens=piece["tokens"],
                    start=piece["start"], end=piece["end"], compression_ratio=get_compression_ratio(text),
                    seek=int(meta["offset"] * model.frames_per_second)))
            batch_results.append(rows)
        if options.word_timestamps:
            self.last_speech_timestamp = model.add_word_timestamps(
                batch_results, tokenizer, encoder_output, frame_counts, options.prepend_punctuations,
                options.append_punctuations, self.last_speech_timestamp)
        return batch_results

    def generate_segment_batched(self, features, tokenizer: Tokenizer, options: TranscriptionOptions):
        """`features` is either the stacked float32 array [n, n_mels, 3000] (reference contract) or an encoder
        output already produced by the fused audio path."""
        model = self.model
        n = features.shape[0]
        history = tokenizer.encode(options.initial_prompt) if options.initial_prompt is not None else []
        prompt = model.get_prompt(tokenizer, previous_tokens=history, without_timestamps=options.without_timestamps,
                                  hotwords=options.hotwords)
        max_length = _check_max_length(len(prompt), options.max_new_tokens, model.max_length)
        encoder_output = features if isinstance(features, engine.StorageView) else model.encode(features)
        prompts = [list(prompt) for _ in range(n)]
        if options.multilingual:
            where = prompt.index(tokenizer.language)
            for row, langs in zip(prompts, model.model.detect_language(encoder_output)):
                row[where] = tokenizer.tokenizer.token_to_id(langs[0][0])
        results = model.model.generate(
            encoder_output, prompts, beam_size=options.beam_size, patience=options.patience,
            length_penalty=options.length_penalty, max_length=max_length, suppress_blank=options.suppress_blank,
            suppress_tokens=options.suppress_tokens, return_scores=True, return_no_speech_prob=True,
            sampling_temperature=options.temperatures[0], repetition_penalty=options.repetition_penalty,
            no_repeat_ngram_size=options.no_repeat_ngram_size)
        outputs = []
        for r in results:
            toks = r.sequences_ids[0]
            outputs.append(dict(avg_logprob=_score_to_avg_logprob(r.scores[0], len(toks), options.length_penalty),
                                no_speech_prob=r.no_speech_prob, tokens=toks))
        return encoder_output, outputs

    def transcribe(
        self,
        audio: Union[str, BinaryIO, np.ndarray],
        language: Optional[str] = None,
        task: str = "transcribe",
        log_progress: bool = False,
        beam_size: int = 5,
        best_of: int = 5,
        patience: float = 1,
        length_penalty: float = 1,
        repetition_penalty: float = 1,
        no_repeat_ngram_size: int = 0,
        temperature: Union[float, List[float], Tuple[float, ...]] = [0.0, 0.2, 0.4, 0.6, 0.8, 1.0],
        compression_ratio_threshold: Optional[float] = 2.4,
        log_prob_threshold: Optional[float] = -1.0,
        no_speech_threshold: Optional[float] = 0.6,
        condition_on_previous_text: bool = True,
        prompt_reset_on_temperature: float = 0.5,
        initial_prompt: Optional[Union[str, Iterable[int]]] = None,
        prefix: Optional[str] = None,
        suppress_blank: bool = True,
        suppress_tokens: Optional[List[int]] = [-1],
        without_timestamps: bool = True,
        max_initial_timestamp: float = 1.0,
        word_timestamps: bool = False,
        prepend_punctuations: str = _PREPEND_PUNCT,
        append_punctuations: str = _APPEND_PUNCT,
        multilingual: bool = False,
        vad_filter: bool = True,
        vad_parameters: Optional[Union[dict, VadOptions]] = None,
        max_new_tokens: Optional[int] = None,
        chunk_length: Optional[int] = None,
        clip_timestamps: Optional[List[dict]] = None,
        hallucination_silence_threshold: Optional[float] = None,
        batch_size: int = 8,
        hotwords: Optional[str] = None,
        language_detection_threshold: Optional[float] = 0.5,
        language_detection_segments: int = 1,
    ) -> Tuple[Iterable[Segment], TranscriptionInfo]:
        """Transcribes `audio` in independent chunks of at most `chunk_length` seconds, `batch_size` chunks per
        engine call.  Arguments, defaults and the ignored ones (compression/log-prob/no-speech thresholds,
        condition_on_previous_text, prefix, max_initial_timestamp, hallucination_silence_threshold) follow the
        reference (transcribe.py:254-375).  Returns (lazy segment generator, TranscriptionInfo)."""
        model = self.model
        sr = model.feature_extractor.sampling_rate
        if multilingual and not model.model.is_multilingual:
            model.logger.warning("The current model is English-only but the multilingual parameter is set to"
                                 "True; setting to False instead.")
            multilingual = False
        if not isinstance(audio, np.ndarray):
            audio = decode_audio(audio, sampling_rate=sr)
        duration = audio.shape[0] / sr
        model.logger.info("Processing audio with duration %s", format_timestamp(duration))
        chunk_length = chunk_length or model.feature_extractor.chunk_length

        # ---- carve the audio into <= chunk_length pieces -------------------------------------------------
        if clip_timestamps:
            from_user = True
            clip_timestamps = [{k: int(v * sr) for k, v in clip.items()} for clip in clip_timestamps]
            audio_chunks, chunks_metadata = [], []
            for i, clip in enumerate(clip_timestamps):
                audio_chunks.append(audio[clip["start"] : clip["end"]])
                seconds = (clip["end"] - clip["start"]) / sr
                if seconds > 30:
                    model.logger.warning("Segment %d is longer than 30 seconds, only the first 30 seconds will be transcribed", i)
                chunks_metadata.append({"offset": clip["start"] / sr, "duration": seconds, "segments": [clip]})
        else:
            from_user = False
            if vad_filter:
                if vad_parameters is None:
                    vad_parameters = VadOptions(max_speech_duration_s=chunk_length, min_silence_duration_ms=160)
                elif isinstance(vad_parameters, dict):
                    vad_parameters = VadOptions(**{**{k: v for k, v in vad_parameters.items() if k != "max_speech_duration_s"},
                                                   "max_speech_duration_s": chunk_length})
                clip_timestamps = get_speech_timestamps(audio, vad_parameters)
            elif duration < chunk_length:
                clip_timestamps = [{"start": 0, "end": audio.shape[0]}]
            else:
                raise RuntimeError("No clip timestamps found. Set 'vad_filter' to True or provide 'clip_timestamps'.")
            audio_chunks, chunks_metadata = collect_chunks(audio, clip_timestamps, max_duration=chunk_length)

        duration_after_vad = sum(c["end"] - c["start"] for c in clip_timestamps) / sr
        model.logger.info("VAD filter removed %s of audio", format_timestamp(duration - duration_after_vad))
        if not duration_after_vad:
            audio_chunks, chunks_metadata = [], []
        # (a chunk longer than 30 s — only possible with user-supplied clips — is not cut here: like the reference, its log-mel is computed
        #  over the whole clip and the FEATURES are trimmed to 3000 frames, see _batched_segments_generator)

        # ---- language ---------------------------------------------------------------------------------------
        all_language_probs = None
        if language is None:
            if not model.model.is_multilingual:
                language, language_probability = "en", 1
            else:
                # the reference concatenates the features of ALL chunks and detect_language reads the first
                # `language_detection_segments` windows of 3000 frames (transcribe.py:478-489): short leading chunks are followed by the
                # next chunks' frames inside a window.  Only the chunks that reach into those windows are computed here.
                feats, need = [], max(1, language_detection_segments) * model.feature_extractor.nb_max_frames
                for c in audio_chunks:
                    if sum(f.shape[-1] for f in feats) >= need:
                        break
                    feats.append(model.feature_extractor(c)[..., :-1])
                feats.append(np.full((model.model.n_mels, 1), -1.5, dtype="float32"))  # keeps empty audio well-formed
                language, language_probability, all_language_probs = model.detect_language(
                    features=np.concatenate(feats, axis=1), language_detection_segments=language_detection_segments,
                    language_detection_threshold=language_detection_threshold)
                model.logger.info("Detected language '%s' with probability %.2f", language, language_probability)
        else:
            if not model.model.is_multilingual and language != "en":
                model.logger.warning("The current model is English-only but the language parameter is set to '%s'; "
                                     "using 'en' instead." % language)
                language = "en"
            language_probability = 1

        tokenizer = Tokenizer(model.hf_tokenizer, model.model.is_multilingual, task=task, language=language)
        options = TranscriptionOptions(
            beam_size=beam_size, best_of=best_of, patience=patience, length_penalty=length_penalty,
            repetition_penalty=repetition_penalty, no_repeat_ngram_size=no_repeat_ngram_size,
            log_prob_threshold=log_prob_threshold, no_speech_threshold=no_speech_threshold,
            compression_ratio_threshold=compression_ratio_threshold, temperatures=_as_temperature_list(temperature)[:1],
            initial_prompt=initial_prompt, prefix=prefix, suppress_blank=suppress_blank,
            suppress_tokens=get_suppressed_tokens(tokenizer, suppress_tokens) if suppress_tokens else suppress_tokens,
            prepend_punctuations=prepend_punctuations, append_punctuations=append_punctuations,
            max_new_tokens=max_new_tokens, hotwords=hotwords, word_timestamps=word_timestamps,
            hallucination_silence_threshold=None, condition_on_previous_text=False, clip_timestamps=clip_timestamps,
            prompt_reset_on_temperature=0.5, multilingual=multilingual, without_timestamps=without_timestamps,
            max_initial_timestamp=0.0)
        info = TranscriptionInfo(
            language=language, language_probability=language_probability, duration=duration,
            duration_after_vad=duration_after_vad, transcription_options=options, vad_options=vad_parameters,
            all_language_probs=all_language_probs)
        segments = self._batched_segments_generator(audio_chunks, tokenizer, chunks_metadata, batch_size, options, log_progress)
        if not from_user:
            segments = restore_speech_timestamps(segments, clip_timestamps, sr)
        return segments, info

    def _batched_segments_generator(self, features, tokenizer, chunks_metadata, batch_size, options, log_progress):
        """`features`: list of PCM chunks (fused audio->mel->encoder path, the default here) or the reference's
        stacked feature array [n, n_mels, 3000]."""
        from tqdm import tqdm

        fused = isinstance(features, list)
        total = len(features)
        bar = tqdm(total=total, disable=not log_progress, position=0)
        seg_id = 0
        for lo in range(0, total, batch_size):
            block = features[lo : lo + batch_size]
            if fused:
                if any(len(c) > 30 * self.model.feature_extractor.sampling_rate for c in block):
                    # the reference's order of operations (transcribe.py:463-467,514-516): log-mel of the whole clip — its clamp maximum and
                    # its last frames see the audio beyond 30 s — then pad_or_trim of the features
                    fe = self.model.feature_extractor
                    block = self.model.encode(np.stack([pad_or_trim(fe(c)[..., :-1]) for c in block]))
                else:
                    block = self.model.model.encode_audio(block)
            for rows in self.forward(block, tokenizer, chunks_metadata[lo : lo + batch_size], options):
                for row in rows:
                    seg_id += 1
                    yield Segment(
                        seek=row["seek"], id=seg_id, text=row["text"], start=round(row["start"], 3), end=round(row["end"], 3),
                        words=[Word(**w) for w in row["words"]] if options.word_timestamps else None, tokens=row["tokens"],
                        avg_logprob=row["avg_logprob"], no_speech_prob=row["no_speech_prob"],
                        compression_ratio=row["compression_ratio"], temperature=options.temperatures[0])
                bar.update(1)
        bar.close()
        self.last_speech_timestamp = 0.0


# --------------------------------------------------------------------------------------------------
# sequential model (transcribe.py:620-1841)
# --------------------------------------------------------------------------------------------------
class WhisperModel:
    def __init__(
        self,
        model_size_or_path: str,
        device: str = "auto",
        device_index: Union[int, List[int]] = 0,
        compute_type: str = "default",
        cpu_threads: int = 0,
        num_workers: int = 1,
        download_root: Optional[str] = None,
        local_files_only: bool = False,
        files: dict = None,
        revision: Optional[str] = None,
        use_auth_token: Optional[Union[str, bool]] = None,
        **model_kwargs,
    ):
        """Same arguments as the reference (transcribe.py:621-670).  Additionally, because no checkpoint can be
        downloaded here: ``WhisperModel("large-v3", synthetic_seed=0)`` builds a seeded random-weight model and a
        synthetic tokenizer at the exact shapes of that size, and ``weights=``/``dims=`` accept an in-memory state dict."""
        self.logger = get_logger()
        synthetic_seed = model_kwargs.pop("synthetic_seed", None)
        weights = model_kwargs.pop("weights", None)
        dims = model_kwargs.pop("dims", None)
        tokenizer_bytes = preprocessor_bytes = None
        model_path = model_size_or_path
        if files:
            tokenizer_bytes = files.pop("tokenizer.json", None)
            preprocessor_bytes = files.pop("preprocessor_config.json", None)
        elif weights is not None or synthetic_seed is not None:
            from .synthetic import make_weights

            dims = dims or MODEL_DIMS[model_size_or_path]
            if weights is None:
                weights = make_weights(dims, seed=int(synthetic_seed))
        elif not os.path.isdir(model_size_or_path):
            model_path = download_model(model_size_or_path, local_files_only=local_files_only, cache_dir=download_root,
                                        revision=revision, use_auth_token=use_auth_token)

        self.model = engine.Whisper(model_path, device=device, device_index=device_index, compute_type=compute_type,
                                    intra_threads=cpu_threads, inter_threads=num_workers, files=files, dims=dims,
                                    weights=weights, **model_kwargs)

        import tokenizers

        tokenizer_file = os.path.join(model_path, "tokenizer.json") if isinstance(model_path, str) else ""
        if tokenizer_bytes:
            self.hf_tokenizer = tokenizers.Tokenizer.from_buffer(tokenizer_bytes)
        elif tokenizer_file and os.path.isfile(tokenizer_file):
            self.hf_tokenizer = tokenizers.Tokenizer.from_file(tokenizer_file)
        else:
            # the reference would fetch openai/whisper-tiny's tokenizer from the hub; offline we synthesise one with
            # Whisper's control-token layout
            from .synthetic import make_tokenizer

            self.hf_tokenizer = make_tokenizer(self.model.dims.n_vocab)
        self.feat_kwargs = self._get_feature_kwargs(model_path, preprocessor_bytes)
        self.feat_kwargs.setdefault("feature_size", self.model.n_mels)
        self.feature_extractor = FeatureExtractor(**self.feat_kwargs, device_index=self.model.device_index[0])
        self.input_stride = 2
        self.num_samples_per_token = self.feature_extractor.hop_length * self.input_stride
        self.frames_per_second = self.feature_extractor.sampling_rate // self.feature_extractor.hop_length
        self.tokens_per_second = self.feature_extractor.sampling_rate // self.num_samples_per_token
        self.time_precision = 0.02
        self.max_length = 448

    @property
    def supported_languages(self) -> List[str]:
        return list(_LANGUAGE_CODES) if self.model.is_multilingual else ["en"]

    def _get_feature_kwargs(self, model_path, preprocessor_bytes=None) -> dict:
        config = {}
        try:
            path = os.path.join(model_path, "preprocessor_config.json") if isinstance(model_path, str) else ""
            if preprocessor_bytes:
                config = json.loads(preprocessor_bytes)
            elif path and os.path.isfile(path):
                with open(path, "r", encoding="utf-8") as f:
                    config = json.load(f)
            else:
                return config
            accepted = set(signature(FeatureExtractor.__init__).parameters) - {"self", "device_index"}
            return {k: v for k, v in config.items() if k in accepted}
        except json.JSONDecodeError as e:
            self.logger.warning("Could not load preprocessor config: %s", e)
        return config

    # ------------------------------------------------------------------------------------------------------
    def transcribe(
        self,
        audio: Union[str, BinaryIO, np.ndarray],
        language: Optional[str] = None,
        task: str = "transcribe",
        log_progress: bool = False,
        beam_size: int = 5,
        best_of: int = 5,
        patience: float = 1,
        length_penalty: float = 1,
        repetition_penalty: float = 1,
        no_repeat_ngram_size: int = 0,
        temperature: Union[float, List[float], Tuple[float, ...]] = [0.0, 0.2, 0.4, 0.6, 0.8, 1.0],
        compression_ratio_threshold: Optional[float] = 2.4,
        log_prob_threshold: Optional[float] = -1.0,
        no_speech_threshold: Optional[float] = 0.6,
        condition_on_previous_text: bool = True,
        prompt_reset_on_temperature: float = 0.5,
        initial_prompt: Optional[Union[str, Iterable[int]]] = None,
        prefix: Optional[str] = None,
        suppress_blank: bool = True,
        suppress_tokens: Optional[List[int]] = [-1],
        without_timestamps: bool = False,
        max_initial_timestamp: float = 1.0,
        word_timestamps: bool = False,
        prepend_punctuations: str = _PREPEND_PUNCT,
        append_punctuations: str = _APPEND_PUNCT,
        multilingual: bool = False,
        vad_filter: bool = False,
        vad_parameters: Optional[Union[dict, VadOptions]] = None,
        max_new_tokens: Optional[int] = None,
        chunk_length: Optional[int] = None,
        clip_timestamps: Union[str, List[float]] = "0",
        hallucination_silence_threshold: Optional[float] = None,
        hotwords: Optional[str] = None,
        language_detection_threshold: Optional[float] = 0.5,
        language_detection_segments: int = 1,
    ) -> Tuple[Iterable[Segment], TranscriptionInfo]:
        """Window-by-window transcription with text conditioning and temperature fallback; arguments and
        defaults as in the reference (transcribe.py:747-865).  Returns (lazy segment generator, TranscriptionInfo)."""
        sr = self.feature_extractor.sampling_rate
        if multilingual and not self.model.is_multilingual:
            self.logger.warning("The current model is English-only but the multilingual parameter is set to"
                                "True; setting to False instead.")
            multilingual = False
        if not isinstance(audio, np.ndarray):
            audio = decode_audio(audio, sampling_rate=sr)
        duration = duration_after_vad = audio.shape[0] / sr
        self.logger.info("Processing audio with duration %s", format_timestamp(duration))

        speech_chunks = None
        if vad_filter and clip_timestamps == "0":
            if vad_parameters is None:
                vad_parameters = VadOptions()
            elif isinstance(vad_parameters, dict):
                vad_parameters = VadOptions(**vad_parameters)
            speech_chunks = get_speech_timestamps(audio, vad_parameters)
            pieces, _ = collect_chunks(audio, speech_chunks)
            audio = np.concatenate(pieces, axis=0)
            duration_after_vad = audio.shape[0] / sr
            self.logger.info("VAD filter removed %s of audio", format_timestamp(duration - duration_after_vad))
            if self.logger.isEnabledFor(logging.DEBUG):
                self.logger.debug("VAD filter kept the following audio segments: %s", ", ".join(
                    "[%s -> %s]" % (format_timestamp(c["start"] / sr), format_timestamp(c["end"] / sr)) for c in speech_chunks))

        features = self.feature_extractor(audio, chunk_length=chunk_length)
        encoder_output = None
        all_language_probs = None
        if language is None:
            if not self.model.is_multilingual:
                language, language_probability = "en", 1
            else:
                first = float(clip_timestamps.split(",")[0]) if isinstance(clip_timestamps, str) else clip_timestamps[0]
                content_frames = features.shape[-1] - 1
                start_frame = first * self.frames_per_second
                seek = int(start_frame) if start_frame < content_frames else 0
                language, language_probability, all_language_probs = self.detect_language(
                    features=features[..., seek:], language_detection_segments=language_detection_segments,
                    language_detection_threshold=language_detection_threshold)
                self.logger.info("Detected language '%s' with probability %.2f", language, language_probability)
        else:
            if not self.model.is_multilingual and language != "en":
                self.logger.warning("The current model is English-only but the language parameter is set to '%s'; "
                                    "using 'en' instead." % language)
                language = "en"
            language_probability = 1

        tokenizer = Tokenizer(self.hf_tokenizer, self.model.is_multilingual, task=task, language=language)
        options = TranscriptionOptions(
            beam_size=beam_size, best_of=best_of, patience=patience, length_penalty=length_penalty,
            repetition_penalty=repetition_penalty, no_repeat_ngram_size=no_repeat_ngram_size,
            log_prob_threshold=log_prob_threshold, no_speech_threshold=no_speech_threshold,
            compression_ratio_threshold=compression_ratio_threshold, condition_on_previous_text=condition_on_previous_text,
            prompt_reset_on_temperature=prompt_reset_on_temperature, temperatures=_as_temperature_list(temperature),
            initial_prompt=initial_prompt, prefix=prefix, suppress_blank=suppress_blank,
            suppress_tokens=get_suppressed_tokens(tokenizer, suppress_tokens) if suppress_tokens else suppress_tokens,
            without_timestamps=without_timestamps, max_initial_timestamp=max_initial_timestamp,
            word_timestamps=word_timestamps, prepend_punctuations=prepend_punctuations,
            append_punctuations=append_punctuations, multilingual=multilingual, max_new_tokens=max_new_tokens,
            clip_timestamps=clip_timestamps, hallucination_silence_threshold=hallucination_silence_threshold,
            hotwords=hotwords)
        segments = self.generate_segments(features, tokenizer, options, log_progress, encoder_output)
        if speech_chunks:
            segments = restore_speech_timestamps(segments, speech_chunks, sr)
        info = TranscriptionInfo(
            language=language, language_probability=language_probability, duration=duration,
            duration_after_vad=duration_after_vad, transcription_options=options, vad_options=vad_parameters,
            all_language_probs=all_language_probs)
        return segments, info

    # ------------------------------------------------------------------------------------------------------
    def _split_segments_by_timestamps(self, tokenizer: Tokenizer, tokens: List[int], time_offset: float,
                                      segment_size: int, segment_duration: float, seek: int):
        """Cuts a decoded window at consecutive timestamp pairs (transcribe.py:1024-1101).
        Returns (sub-segments, new seek, single_timestamp_ending)."""
        ts0 = tokenizer.timestamp_begin
        is_ts = [t >= ts0 for t in tokens]
        single_ending = len(tokens) >= 2 and not is_ts[-2] and is_ts[-1]
        cuts = [i for i in range(1, len(tokens)) if is_ts[i] and is_ts[i - 1]]
        pieces = []
        if cuts:
            if single_ending:
                cuts.append(len(tokens))
            begin = 0
            for cut in cuts:
                part = tokens[begin:cut]
                pieces.append(dict(seek=seek, start=time_offset + (part[0] - ts0) * self.time_precision,
                                   end=time_offset + (part[-1] - ts0) * self.time_precision, tokens=part))
                begin = cut
            if single_ending:
                seek += segment_size  # nothing spoken after the last timestamp
            else:
                seek += (tokens[begin - 1] - ts0) * self.input_stride  # resume at the last closed timestamp
        else:
            span = segment_duration
            stamps = [t for t in tokens if t >= ts0]
            if stamps and stamps[-1] != ts0:
                span = (stamps[-1] - ts0) * self.time_precision
            pieces.append(dict(seek=seek, start=time_offset, end=time_offset + span, tokens=tokens))
            seek += segment_size
        return pieces, seek, single_ending

    def generate_segments(self, features: np.ndarray, tokenizer: Tokenizer, options: TranscriptionOptions, log_progress,
                          encoder_output: Optional[engine.StorageView] = None) -> Iterator[Segment]:
        """The seek loop (transcribe.py:1103-1389): one encoder pass + decode per <=30 s window, windows chained by
        the timestamps the decoder emits and (optionally) by the previous text."""
        from tqdm import tqdm

        fe = self.feature_extractor
        content_frames = features.shape[-1] - 1
        content_duration = float(content_frames * fe.time_per_frame)
        if isinstance(options.clip_timestamps, str):
            options.clip_timestamps = [float(x) for x in options.clip_timestamps.split(",")] if options.clip_timestamps else []
        marks = [round(t * self.frames_per_second) for t in options.clip_timestamps] or [0]
        if len(marks) % 2:
            marks.append(content_frames)
        clips = list(zip(marks[::2], marks[1::2]))
        punctuation = _PREPEND_PUNCT + _APPEND_PUNCT

        all_tokens: List[int] = []
        if options.initial_prompt is not None:
            if isinstance(options.initial_prompt, str):
                all_tokens.extend(tokenizer.encode(" " + options.initial_prompt.strip()))
            else:
                all_tokens.extend(options.initial_prompt)
        prompt_reset_since = 0
        seg_id = 0
        last_speech_timestamp = 0.0
        bar = tqdm(total=content_duration, unit="seconds", disable=not log_progress)

        def anomaly(word: dict) -> float:
            p, dur = word.get("probability", 0.0), word["end"] - word["start"]
            return (1.0 if p < 0.15 else 0.0) + ((0.133 - dur) * 15 if dur < 0.133 else 0.0) + (dur - 2.0 if dur > 2.0 else 0.0)

        def is_anomalous(seg: Optional[dict]) -> bool:
            if seg is None or not seg["words"]:
                return False
            ws = [w for w in seg["words"] if w["word"] not in punctuation][:8]
            score = sum(anomaly(w) for w in ws)
            return score >= 3 or score + 0.01 >= len(ws)

        def first_with_words(segs: List[dict]) -> Optional[dict]:
            return next((s for s in segs if s["words"]), None)

        for clip_start, clip_end in clips:
            clip_end = min(clip_end, content_frames)
            seek = clip_start
            while seek < clip_end:
                time_offset = seek * fe.time_per_frame
                window_end_time = float((seek + fe.nb_max_frames) * fe.time_per_frame)
                segment_size = min(fe.nb_max_frames, content_frames - seek, clip_end - seek)
                segment_duration = segment_size * fe.time_per_frame
                window = pad_or_trim(features[:, seek : seek + segment_size])
                if self.logger.isEnabledFor(logging.DEBUG):
                    self.logger.debug("Processing segment at %s", format_timestamp(time_offset))
                previous_tokens = all_tokens[prompt_reset_since:]
                if seek > 0 or encoder_output is None:
                    encoder_output = self.encode(window)
                if options.multilingual:
                    token, _ = self.model.detect_language(encoder_output)[0][0]
                    tokenizer.language = tokenizer.tokenizer.token_to_id(token)
                    tokenizer.language_code = token[2:-2]
                prompt = self.get_prompt(tokenizer, previous_tokens, without_timestamps=options.without_timestamps,
                                         prefix=options.prefix if seek == 0 else None, hotwords=options.hotwords)
                result, avg_logprob, temperature, compression_ratio = self.generate_with_fallback(
                    encoder_output, prompt, tokenizer, options)

                if options.no_speech_threshold is not None:
                    silent = result.no_speech_prob > options.no_speech_threshold
                    if options.log_prob_threshold is not None and avg_logprob > options.log_prob_threshold:
                        silent = False  # confident text wins over the no-speech probability
                    if silent:
                        self.logger.debug("No speech threshold is met (%f > %f)", result.no_speech_prob, options.no_speech_threshold)
                        seek += segment_size
                        continue

                tokens = result.sequences_ids[0]
                previous_seek = seek
                current, seek, single_ending = self._split_segments_by_timestamps(
                    tokenizer=tokenizer, tokens=tokens, time_offset=time_offset, segment_size=segment_size,
                    segment_duration=segment_duration, seek=seek)

                if options.word_timestamps:
                    self.add_word_timestamps([current], tokenizer, encoder_output, segment_size, options.prepend_punctuations,
                                             options.append_punctuations, last_speech_timestamp=last_speech_timestamp)
                    if not single_ending:
                        last_word_end = get_end(current)
                        if last_word_end is not None and last_word_end > time_offset:
                            seek = round(last_word_end * self.frames_per_second)
                    threshold = options.hallucination_silence_threshold
                    if threshold is not None:
                        restart = False
                        head = first_with_words(current)
                        if head is not None and is_anomalous(head):
                            gap = head["start"] - time_offset
                            if gap > threshold:
                                seek = previous_seek + round(gap * self.frames_per_second)
                                restart = True
                        if restart:
                            continue
                        hal_last_end = last_speech_timestamp
                        for si, seg in enumerate(current):
                            if not seg["words"]:
                                continue
                            if is_anomalous(seg):
                                nxt = first_with_words(current[si + 1 :])
                                nxt_start = nxt["words"][0]["start"] if nxt is not None else time_offset + segment_duration
                                quiet_before = (seg["start"] - hal_last_end > threshold or seg["start"] < threshold
                                                or seg["start"] - time_offset < 2.0)
                                quiet_after = (nxt_start - seg["end"] > threshold or is_anomalous(nxt)
                                               or window_end_time - seg["end"] < 2.0)
                                if quiet_before and quiet_after:
                                    seek = round(max(time_offset + 1, seg["start"]) * self.frames_per_second)
                                    if content_duration - seg["end"] < threshold:
                                        seek = content_frames
                                    del current[si:]
                                    break
                            hal_last_end = seg["end"]
                    last_word_end = get_end(current)
                    if last_word_end is not None:
                        last_speech_timestamp = last_word_end

                for seg in current:
                    text = tokenizer.decode(seg["tokens"])
                    if seg["start"] == seg["end"] or not text.strip():
                        continue
                    all_tokens.extend(seg["tokens"])
                    seg_id += 1
                    yield Segment(
                        id=seg_id, seek=previous_seek, start=seg["start"], end=seg["end"], text=text, tokens=seg["tokens"],
                        temperature=temperature, avg_logprob=avg_logprob, compression_ratio=compression_ratio,
                        no_speech_prob=result.no_speech_prob,
                        words=[Word(**w) for w in seg["words"]] if options.word_timestamps else None)

                if not options.condition_on_previous_text or temperature > options.prompt_reset_on_temperature:
                    if options.condition_on_previous_text:
                        self.logger.debug("Reset prompt. prompt_reset_on_temperature threshold is met %f > %f",
                                          temperature, options.prompt_reset_on_temperature)
                    prompt_reset_since = len(all_tokens)
                bar.update((min(content_frames, seek) - previous_seek) * fe.time_per_frame)
        bar.close()

    def encode(self, features: np.ndarray) -> engine.StorageView:
        """[n_mels, 3000] or [batch, n_mels, 3000] float32 -> device-resident encoder output (transcribe.py:1391-1400).
        With several GPUs the reference bounces the output through host memory because the next call may land on
        another device; here an encoder output remembers its replica, so it stays in HBM."""
        if features.ndim == 2:
            features = np.expand_dims(features, 0)
        return self.model.encode(get_ctranslate2_storage(features), to_cpu=False)

    def generate_with_fallback(self, encoder_output, prompt: List[int], tokenizer: Tokenizer, options: TranscriptionOptions):
        """Decodes one window, retrying at higher temperatures when the text is too repetitive or too unlikely
        (transcribe.py:1402-1530).  Returns (result, avg_logprob, temperature, compression_ratio)."""
        max_initial_timestamp_index = int(round(options.max_initial_timestamp / self.time_precision))
        max_length = _check_max_length(len(prompt), options.max_new_tokens, self.max_length)
        attempts, acceptable = [], []
        chosen = None
        for temperature in options.temperatures:
            if temperature > 0:
                search = dict(beam_size=1, num_hypotheses=options.best_of, sampling_topk=0, sampling_temperature=temperature)
            else:
                search = dict(beam_size=options.beam_size, patience=options.patience)
            result = self.model.generate(
                encoder_output, [prompt], length_penalty=options.length_penalty, repetition_penalty=options.repetition_penalty,
                no_repeat_ngram_size=options.no_repeat_ngram_size, max_length=max_length, return_scores=True,
                return_no_speech_prob=True, suppress_blank=options.suppress_blank, suppress_tokens=options.suppress_tokens,
                max_initial_timestamp_index=max_initial_timestamp_index, **search)[0]
            tokens = result.sequences_ids[0]
            avg_logprob = _score_to_avg_logprob(result.scores[0], len(tokens), options.length_penalty)
            compression_ratio = get_compression_ratio(tokenizer.decode(tokens).strip())
            chosen = (result, avg_logprob, temperature, compression_ratio)
            attempts.append(chosen)
            retry = False
            if options.compression_ratio_threshold is not None:
                if compression_ratio > options.compression_ratio_threshold:
                    retry = True
                    self.logger.debug("Compression ratio threshold is not met with temperature %.1f (%f > %f)",
                                      temperature, compression_ratio, options.compression_ratio_threshold)
                else:
                    acceptable.append(chosen)
            too_unlikely = options.log_prob_threshold is not None and avg_logprob < options.log_prob_threshold
            if too_unlikely:
                retry = True
                self.logger.debug("Log probability threshold is not met with temperature %.1f (%f < %f)",
                                  temperature, avg_logprob, options.log_prob_threshold)
            if (options.no_speech_threshold is not None and result.no_speech_prob > options.no_speech_threshold and too_unlikely):
                retry = False  # silence: do not burn more temperatures on it
            if not retry:
                return chosen
        # every temperature failed: keep the most likely attempt, report the last temperature tried
        best = max(acceptable or attempts, key=lambda a: a[1])
        return (best[0], best[1], options.temperatures[-1], best[3])

    def get_prompt(self, tokenizer: Tokenizer, previous_tokens: List[int], without_timestamps: bool = False,
                   prefix: Optional[str] = None, hotwords: Optional[str] = None) -> List[int]:
        """[sot_prev, hotwords..., previous text...]? + sot sequence + [no_timestamps]? + [timestamp_begin? + prefix...]
        (transcribe.py:1532-1565)."""
        cap = self.max_length // 2 - 1
        prompt: List[int] = []
        use_hotwords = bool(hotwords) and not prefix
        if previous_tokens or use_hotwords:
            prompt.append(tokenizer.sot_prev)
            if use_hotwords:
                prompt.extend(tokenizer.encode(" " + hotwords.strip())[:cap])
            if previous_tokens:
                prompt.extend(previous_tokens[-cap:])
        prompt.extend(tokenizer.sot_sequence)
        if without_timestamps:
            prompt.append(tokenizer.no_timestamps)
        if prefix:
            if not without_timestamps:
                prompt.append(tokenizer.timestamp_begin)
            prompt.extend(tokenizer.encode(" " + prefix.strip())[:cap])
        return prompt

    # -- word timestamps (SURVEY.md §8f row 3: needs Whisper.align) ---------------------------------------------
    def add_word_timestamps(self, segments: List[dict], tokenizer: Tokenizer, encoder_output, num_frames,
                            prepend_punctuations: str, append_punctuations: str, last_speech_timestamp: float) -> float:
        if len(segments) == 0:
            return last_speech_timestamp
        per_segment_tokens = [[[t for t in sub["tokens"] if t < tokenizer.eot] for sub in seg] for seg in segments]
        text_tokens = [list(itertools.chain.from_iterable(parts)) for parts in per_segment_tokens]
        alignments = self.find_alignment(tokenizer, text_tokens, encoder_output, num_frames)
        limits = []
        for alignment in alignments:
            spans = np.array([w["end"] - w["start"] for w in alignment])
            spans = spans[spans.nonzero()]
            median = min(0.7, float(np.median(spans))) if len(spans) > 0 else 0.0
            longest = median * 2
            if len(spans) > 0:
                for i in range(1, len(alignment)):  # clamp over-long words next to sentence ends
                    if alignment[i]["end"] - alignment[i]["start"] > longest:
                        if alignment[i]["word"] in ".。!！?？":
                            alignment[i]["end"] = alignment[i]["start"] + longest
                        elif alignment[i - 1]["word"] in ".。!！?？":
                            alignment[i]["start"] = alignment[i]["end"] - longest
            merge_punctuations(alignment, prepend_punctuations, append_punctuations)
            limits.append((median, longest))
        for si, seg in enumerate(segments):
            cursor = 0
            offset = seg[0]["seek"] / self.frames_per_second
            median, longest = limits[si]
            for sj, sub in enumerate(seg):
                taken, words = 0, []
                want = len(per_segment_tokens[si][sj])
                while cursor < len(alignments[si]) and taken < want:
                    w = alignments[si][cursor]
                    if w["word"]:
                        words.append(dict(word=w["word"], start=round(offset + w["start"], 2), end=round(offset + w["end"], 2),
                                          probability=w["probability"]))
                    taken += len(w["tokens"])
                    cursor += 1
                if words:
                    first = words[0]
                    if first["end"] - last_speech_timestamp > median * 4 and (
                            first["end"] - first["start"] > longest
                            or (len(words) > 1 and words[1]["end"] - first["start"] > longest * 2)):
                        if len(words) > 1 and words[1]["end"] - words[1]["start"] > longest:
                            edge = max(words[1]["end"] / 2, words[1]["end"] - longest)
                            first["end"] = words[1]["start"] = edge
                        first["start"] = max(0, first["end"] - longest)
                    if sub["start"] < first["end"] and sub["start"] - 0.5 > first["start"]:
                        first["start"] = max(0, min(first["end"] - median, sub["start"]))
                    else:
                        sub["start"] = first["start"]
                    last = words[-1]
                    if sub["end"] > last["start"] and sub["end"] + 0.5 < last["end"]:
                        last["end"] = max(last["start"] + median, sub["end"])
                    else:
                        sub["end"] = last["end"]
                    last_speech_timestamp = sub["end"]
                segments[si][sj]["words"] = words
        return last_speech_timestamp

    def find_alignment(self, tokenizer: Tokenizer, text_tokens, encoder_output, num_frames, median_filter_width: int = 7):
        if len(text_tokens) == 0:
            return []
        results = self.model.align(encoder_output, tokenizer.sot_sequence, text_tokens, num_frames,
                                   median_filter_width=median_filter_width)
        out = []
        for result, toks in zip(results, text_tokens):
            words, word_tokens = tokenizer.split_to_word_tokens(toks + [tokenizer.eot])
            if len(word_tokens) <= 1:
                out.append([])
                continue
            bounds = np.pad(np.cumsum([len(t) for t in word_tokens[:-1]]), (1, 0))
            if len(bounds) <= 1:
                out.append([])
                continue
            text_idx = np.array([p[0] for p in result.alignments])
            time_idx = np.array([p[1] for p in result.alignments])
            jumps = np.pad(np.diff(text_idx), (1, 0), constant_values=1).astype(bool)
            jump_times = time_idx[jumps] / self.tokens_per_second
            probs = result.text_token_probs
            out.append([
                dict(word=w, tokens=t, start=s, end=e, probability=float(np.mean(probs[i:j])))
                for w, t, s, e, i, j in zip(words, word_tokens, jump_times[bounds[:-1]], jump_times[bounds[1:]], bounds[:-1], bounds[1:])
            ])
        return out

    def detect_language(self, audio: Optional[np.ndarray] = None, features: Optional[np.ndarray] = None,
                        vad_filter: bool = False, vad_parameters: Union[dict, VadOptions] = None,
                        language_detection_segments: int = 1, language_detection_threshold: float = 0.5):
        """Returns (language, probability, all_language_probs) from up to `language_detection_segments` 30 s windows
        (transcribe.py:1768-1841): first window above the threshold wins, else majority vote."""
        assert audio is not None or features is not None, "Either `audio` or `features` must be provided."
        fe = self.feature_extractor
        if audio is not None:
            if vad_filter:
                spans = get_speech_timestamps(audio, vad_parameters)
                pieces, _ = collect_chunks(audio, spans)
                audio = np.concatenate(pieces, axis=0)
            features = fe(audio[: language_detection_segments * fe.n_samples])
        features = features[..., : language_detection_segments * fe.nb_max_frames]
        votes = {}
        language = language_probability = all_language_probs = None
        for lo in range(0, features.shape[-1], fe.nb_max_frames):
            enc = self.encode(pad_or_trim(features[..., lo : lo + fe.nb_max_frames]))
            ranked = self.model.detect_language(enc)[0]
            all_language_probs = [(tok[2:-2], p) for tok, p in ranked]
            language, language_probability = all_language_probs[0]
            if language_probability > language_detection_threshold:
                return language, language_probability, all_language_probs
            votes.setdefault(language, []).append(language_probability)
        language = max(votes, key=lambda k: len(votes[k]))
        return language, max(votes[language]), all_language_probs
