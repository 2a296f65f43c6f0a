"""CPU: our host layer (tokenizer wrapper, prompt building, timestamp splitting, chunk bookkeeping, helper functions)
against outputs recorded from the reference (tests/golden/host_golden.json, made by oracle/make_golden.py)."""
import inspect
import json
import os

import numpy as np
import pytest

from faster_whisper_b200 import transcribe as T
from faster_whisper_b200 import utils, vad
from faster_whisper_b200.config import MODEL_DIMS, special_tokens
from faster_whisper_b200.synthetic import make_tokenizer
from faster_whisper_b200.tokenizer import Tokenizer
from oracle.refload import RecordedReference, canon


def recorded_reference():
    """What the reference returned for the comparisons below (tests/golden/reference_golden.json.gz, recorded by oracle/refload.py)."""
    return RecordedReference(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_golden.json.gz"))

GOLD = os.path.join(os.path.dirname(__file__), "golden")


@pytest.fixture(scope="module")
def gold():
    with open(os.path.join(GOLD, "host_golden.json")) as f:
        return json.load(f)


@pytest.fixture(scope="module")
def tok():
    return Tokenizer(make_tokenizer(51865), True, task="transcribe", language="en")


@pytest.fixture(scope="module")
def bare_model():
    m = T.WhisperModel.__new__(T.WhisperModel)
    m.time_precision, m.input_stride, m.max_length = 0.02, 2, 448
    return m


def test_special_token_layout_matches_reference_goldens(tok, gold):
    # tests/test_tokenizer.py:96-110 of the reference pins the tiny.en ids; the derived layout must agree
    en = special_tokens(51864)
    assert (en.eot, en.sot, en.translate, en.transcribe, en.sot_lm, en.sot_prev, en.no_speech, en.no_timestamps, en.timestamp_begin) == (
        50256, 50257, 50357, 50358, 50359, 50360, 50361, 50362, 50363)
    ml = special_tokens(51865)
    assert (tok.sot, tok.eot, tok.timestamp_begin, tok.no_speech) == (ml.sot, ml.eot, ml.timestamp_begin, ml.no_speech)
    g = gold["special"]
    assert (tok.sot, tok.eot, tok.timestamp_begin, tok.no_speech, tok.sot_sequence) == (g["sot"], g["eot"], g["ts0"], g["no_speech"], g["sot_sequence"])
    v3 = special_tokens(51866)
    assert v3.timestamp_begin == 50365 and v3.num_languages == 100
    for name, d in MODEL_DIMS.items():
        special_tokens(d.n_vocab)


def test_split_segments_by_timestamps(tok, bare_model, gold):
    for case in gold["split"]:
        segs, seek, single = bare_model._split_segments_by_timestamps(tok, list(case["tokens"]), 12.5, 2800, 28.0, 100)
        assert seek == case["seek"] and bool(single) == case["single"], case["tokens"]
        assert len(segs) == len(case["segments"])
        for a, b in zip(segs, case["segments"]):
            assert a["tokens"] == b["tokens"] and a["seek"] == b["seek"]
            assert a["start"] == pytest.approx(b["start"]) and a["end"] == pytest.approx(b["end"])


def test_get_prompt(tok, bare_model, gold):
    for case in gold["prompts"]:
        assert bare_model.get_prompt(tok, **case["kwargs"]) == case["prompt"]


def test_get_suppressed_tokens(tok, gold):
    for case in gold["suppressed"]:
        assert list(T.get_suppressed_tokens(tok, list(case["arg"]))) == case["out"]
    assert isinstance(T.get_suppressed_tokens(tok, [-1]), tuple)


def test_chunk_bookkeeping(gold):
    g = gold["vad"]
    audio = np.arange(16000 * 100, dtype=np.float32)
    chunks, metas = vad.collect_chunks(audio, g["spans"], max_duration=30)
    assert [int(c.shape[0]) for c in chunks] == g["chunk_lens"]
    assert [float(c[0]) if c.size else None for c in chunks] == g["chunk_first"]
    assert metas == g["metas"]
    tsm = vad.SpeechTimestampsMap(g["spans"], 16000)
    assert [tsm.get_original_time(t) for t in (0.0, 5.0, 12.4, 30.0, 60.0)] == g["orig"]
    assert [tsm.get_original_time(t, is_end=True) for t in (12.4375, 37.4375)] == g["orig_end"]
    c, m = vad.collect_chunks(audio, [])
    assert len(c) == 1 and c[0].size == 0 and m == [{"offset": 0, "duration": 0, "segments": []}]


def test_small_helpers(gold):
    for s, a, b in gold["format_timestamp"]:
        assert utils.format_timestamp(s) == a and utils.format_timestamp(s, True, ",") == b
    al = [dict(word=" (", tokens=[1]), dict(word=" hello", tokens=[2, 3]), dict(word=",", tokens=[4]), dict(word=" world", tokens=[5]),
          dict(word=".", tokens=[6]), dict(word=" \"", tokens=[7]), dict(word=" yes", tokens=[8])]
    T.merge_punctuations(al, "\"'“¿([{-", "\"'.。,，!！?？:：”)]}、")
    assert al == gold["merged"]
    for s, r in gold["compression"]:
        assert T.get_compression_ratio(s) == pytest.approx(r)
    assert utils.get_end([{"end": 1.0, "words": []}, {"end": 2.0, "words": [{"end": 1.7}]}]) == 1.7
    assert utils.get_end([]) is None
    assert "large-v3" in utils.available_models() and len(utils.available_models()) == 19


def test_transcribe_signatures():
    """The reference's own structural test (tests/test_transcribe.py:237-244): both transcribe() methods take the same
    arguments apart from batch_size — and here additionally match the reference's names and defaults exactly."""
    seq = inspect.signature(T.WhisperModel.transcribe).parameters
    bat = inspect.signature(T.BatchedInferencePipeline.transcribe).parameters
    assert set(bat) - set(seq) == {"batch_size"} and not set(seq) - set(bat)
    from oracle.refload import load_reference

    rec = recorded_reference()
    R = load_reference().transcribe if rec.record else None

    def signature(fn):  # parameter names and the repr of their defaults
        return [[k, repr(v.default)] for k, v in inspect.signature(fn).parameters.items()]

    for name in ("WhisperModel.transcribe", "BatchedInferencePipeline.transcribe", "WhisperModel.__init__", "WhisperModel.detect_language",
                 "WhisperModel.get_prompt"):
        cls, meth = name.split(".")
        want = rec.get("signature/" + name, lambda: signature(getattr(getattr(R, cls), meth)))
        assert canon(signature(getattr(getattr(T, cls), meth))) == want, name
    for cls in ("Word", "Segment", "TranscriptionOptions", "TranscriptionInfo"):
        assert [f for f in getattr(T, cls).__dataclass_fields__] == rec.get("fields/" + cls, lambda: list(getattr(R, cls).__dataclass_fields__))


def test_tokenizer_wrapper(tok):
    ids = tok.encode(" hello world")
    assert tok.decode(ids + [tok.eot, tok.timestamp_begin + 3]) == " hello world"
    assert tok.decode_with_timestamps([tok.timestamp_begin, *ids, tok.timestamp_begin + 50]) == "<|0.00|> hello world<|1.00|>"
    words, groups = tok.split_to_word_tokens(ids + [tok.eot])
    assert "".join(words[:-1]) == " hello world" and sum(len(g) for g in groups) == len(ids) + 1
    assert len(tok.non_speech_tokens) > 20 and tok.non_speech_tokens == tuple(sorted(tok.non_speech_tokens))
    with pytest.raises(ValueError):
        Tokenizer(tok.tokenizer, True, task="nope", language="en")
    with pytest.raises(ValueError):
        Tokenizer(tok.tokenizer, True, task="transcribe", language="klingon")
    en = Tokenizer(make_tokenizer(51864), False)
    assert en.sot_sequence == [50257] and en.language_code == "en"


# ---- CTranslate2 model directory (model.bin) reader/writer round trip --------------------------------------------------------
def test_ct2_model_bin_round_trip(tmp_path):
    from faster_whisper_b200 import checkpoint, ct2_format
    from faster_whisper_b200.synthetic import custom_dims, make_weights

    dims = custom_dims(name="rt", n_mels=80, d=64, heads=1, enc_layers=2, dec_layers=2, n_vocab=51864)
    w = make_weights(dims, seed=3)
    d = tmp_path / "m"
    ct2_format.save_ct2_dir(str(d), dims, w, alignment_heads=[(1, 0)], dtype=np.float32)
    spec, rev, variables, aliases = ct2_format.read_model_bin(str(d / "model.bin"))
    assert spec == "WhisperSpec" and aliases["decoder/projection/weight"] == "decoder/embeddings/weight"
    assert variables["decoder/layer_1/attention/linear_1/weight"].shape == (2 * dims.n_text_state, dims.n_text_state)
    dims2, w2 = checkpoint.load_model_dir(str(d))
    assert dims2.to_dict() | {"name": "x"} == dims.to_dict() | {"name": "x"}
    assert set(w2) == set(w)
    for k in w:
        assert np.array_equal(w2[k], w[k].astype(np.float32)), k
    assert checkpoint.read_alignment_heads(str(d)) == [(1, 0)]
    # int8 storage with per-row scales de-quantises to within half a quantisation step
    d8 = tmp_path / "m8"
    ct2_format.save_ct2_dir(str(d8), dims, w, quantize_int8=True)
    _, w8 = checkpoint.load_model_dir(str(d8))
    k = "decoder.blocks.0.mlp.0.weight"
    step = np.abs(w[k]).max(axis=1, keepdims=True) / 127.0
    assert np.all(np.abs(w8[k] - w[k]) <= 0.5 * step + 1e-7)
    with pytest.raises(ValueError):
        ct2_format.read_model_bin(b"\\xff\\xff\\xff\\xff garbage")


def test_unloaded_model_is_never_dereferenced():
    """ADVICE r1: StorageViews that outlive unload_model() used to free into a destroyed native model.  Pure host logic here (no
    GPU): a replica hands its live outputs back before it is destroyed, and every later call raises instead of passing NULL."""
    import ctypes
    import gc

    from faster_whisper_b200 import engine as E

    class FakeLib:
        def __init__(self):
            self.freed, self.destroyed = [], []

        def b2w_encoded_free(self, h):
            assert not self.destroyed, "encoder output freed after its model"
            self.freed.append(h)

        def b2w_model_destroy(self, h):
            self.destroyed.append(h)

    rep = E._Replica.__new__(E._Replica)
    rep._lib, rep.device, rep._h = FakeLib(), 0, ctypes.c_void_p(1234)
    import threading

    rep.lock, rep._out_lock, rep._outputs = threading.Lock(), threading.Lock(), {}
    old_lib, E._lib = E._lib, rep._lib
    try:
        a = E.StorageView(handle=ctypes.c_void_p(1), shape=(1, 1500, 8))
        b = E.StorageView(handle=ctypes.c_void_p(2), shape=(1, 1500, 8))
        for sv in (a, b):
            sv._replica = rep
            rep.track_output(sv)
        del b, sv
        gc.collect()
        assert len(rep._lib.freed) == 1 and len(rep._outputs) == 1
        rep.close()
        assert len(rep._lib.freed) == 2 and rep._lib.destroyed and a._handle is None
        with pytest.raises(ValueError):
            a.numpy()
        with pytest.raises(RuntimeError, match="unloaded"):
            rep.handle
        del a
        gc.collect()
        assert len(rep._lib.freed) == 2  # nothing is freed into the destroyed model
        rep.close()  # idempotent
        assert len(rep._lib.destroyed) == 1
    finally:
        E._lib = old_lib


def test_tokenizer_matches_the_reference_class_on_random_sequences():
    """Our Tokenizer wrapper against the reference's own class (faster_whisper/tokenizer.py, imported unmodified) over the same HF tokenizer:
    sot sequence, non-speech set, decode, decode_with_timestamps and the word splitting (space-based languages and the unicode path of
    zh / ja / th / yue) on random token sequences, with and without a trailing eot."""
    import sys

    from oracle.refload import load_reference

    rec = recorded_reference()
    ref_cls = sys.modules[load_reference().__name__ + ".tokenizer"].Tokenizer if rec.record else None
    hf = make_tokenizer(51866)
    rng = np.random.default_rng(0)

    def specials(t):
        return [t.sot_sequence, t.non_speech_tokens, [t.transcribe, t.translate, t.sot, t.sot_lm, t.sot_prev, t.eot, t.no_timestamps, t.no_speech,
                                                      t.timestamp_begin]]

    def outputs(t, ids, ts):
        return [t.split_to_word_tokens(ids), t.decode_with_timestamps(ts), t.decode(ids), t.encode(" hello wor")]

    for lang in ["en", "zh", "ja", "th", "de", "yue"]:
        ours = Tokenizer(hf, True, task="transcribe", language=lang)
        ref = ref_cls(hf, True, task="transcribe", language=lang) if rec.record else None
        assert canon(specials(ours)) == rec.get(f"tokenizer/{lang}/specials", lambda: specials(ref))
        for trial in range(120):
            n = int(rng.integers(1, 24))
            ids = [int(x) for x in rng.integers(0, ours.eot, size=n)] + ([ours.eot] if trial % 3 == 0 else [])
            ts = [ours.timestamp_begin + 3] + ids[: n // 2] + [ours.timestamp_begin + 40] * 2 + ids[n // 2:] + [ours.timestamp_begin + 90]
            assert canon(outputs(ours, ids, ts)) == rec.get(f"tokenizer/{lang}/{trial}", lambda: outputs(ref, ids, ts)), (lang, ids)


def test_model_names_and_hub_repositories_match_the_reference():
    """available_models() and the size -> hub repository table are the reference's (utils.py:12-47), entry for entry and in order."""
    import sys

    from faster_whisper_b200 import utils as ours
    from oracle.refload import load_reference

    rec = recorded_reference()
    ref = sys.modules[load_reference().__name__ + ".utils"] if rec.record else None
    assert ours.available_models() == rec.get("utils/available_models", lambda: ref.available_models())
    assert list(ours._HUB_REPOS.items()) == [tuple(kv) for kv in rec.get("utils/models", lambda: list(ref._MODELS.items()))]
    assert ours.format_timestamp(3723.456, always_include_hours=True, decimal_marker=",") == rec.get(
        "utils/format_timestamp_hours", lambda: ref.format_timestamp(3723.456, always_include_hours=True, decimal_marker=","))
    assert ours.format_timestamp(59.999) == rec.get("utils/format_timestamp", lambda: ref.format_timestamp(59.999))
