"""CPU: the C-ABI library builds, loads, exports every symbol the header declares, and fails loudly without a GPU."""
import ctypes
import os
import re

import numpy as np
import pytest

from faster_whisper_b200 import engine

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_symbols():
    text = open(os.path.join(ROOT, "include", "b200whisper.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(b2w_[a-z0-9_]+)\s*\(", text)))


def test_library_exports_every_declared_symbol():
    lib = engine.load_library()
    declared = header_symbols()
    assert len(declared) >= 20
    for name in declared:
        assert hasattr(lib, name), f"{name} is declared in include/b200whisper.h but not exported"
    assert set(declared) == set(engine.ABI_SYMBOLS)
    assert lib.b2w_abi_version() == 1


def test_struct_layout_matches_header():
    # b2w_gen_opts: the ctypes mirror must have the size the C side fills in
    lib = engine.load_library()
    o = engine._GenOpts()
    ctypes.memset(ctypes.byref(o), 0xFF, ctypes.sizeof(o))
    lib.b2w_gen_opts_default(ctypes.byref(o))
    assert (o.beam_size, o.num_hypotheses, o.max_length, o.max_initial_timestamp_index, o.suppress_blank, o.sampling_topk) == (5, 1, 448, 50, 1, 1)
    assert (o.patience, o.length_penalty, o.repetition_penalty, o.sampling_temperature) == (1.0, 1.0, 1.0, 1.0)
    assert o.debug_fake_logits == 0 and o.seed == 0 and o.n_suppress_tokens == 0


def test_gemm_hooks_check_arguments_before_the_device():
    """Bad GEMM descriptors are refused (ValueError) before anything touches a device, GPU or not."""
    a, out = np.zeros(64 * 64, np.float16), np.zeros(64 * 128, np.float32)
    w = np.zeros((128, 64), np.float16)
    with pytest.raises(ValueError, match="N must be a multiple of 32"):
        engine.debug_gemm_desc(a, np.zeros((48, 64), np.float16), out, epilogue=engine.EPI_F32, rows=64)
    with pytest.raises(ValueError, match="K per tap"):
        engine.debug_gemm_desc(a, np.zeros((128, 96), np.float16), out, epilogue=engine.EPI_F32, rows=64, a_cols=96)
    with pytest.raises(ValueError, match="exceeds its buffer"):
        engine.debug_gemm_desc(a, w, out, epilogue=engine.EPI_F32, rows=65, a_rows=64)
    kc = np.zeros((1, 4, 2, 64), np.float16)
    rows = np.array([[0, 1, 3, 0]] * 63 + [[0, 2, 0, 0]], np.int32)  # slot 2 of 2
    with pytest.raises(ValueError, match="row table"):
        engine.debug_gemm_desc(a, np.zeros((192, 64), np.float16), np.zeros(64 * 64, np.float16), epilogue=engine.EPI_QKV_CACHE, rows=64,
                               rowinfo=rows, kcache=kc, vcache=kc.copy(), qkv_d=64, n_ctx=4, slots=2)
    with pytest.raises(ValueError, match="1..80 rows"):
        engine.debug_gemv_desc(np.zeros((81, 64), np.float16), w, mode=engine.GV_F32, out=np.zeros(81 * 128, np.float32), ldo=128)


def test_attention_hooks_check_arguments_before_the_device():
    """Bad inputs of the decoder attention hooks are refused (ValueError) before anything touches a device, GPU or not."""
    q, kc = np.zeros((2, 128), np.float16), np.zeros((1, 8, 4, 128), np.float16)
    anc, rows = np.zeros((2, 1, 4, 8), np.uint8), np.array([[0, 1, 3, 0], [0, 3, 7, 0]], np.int32)
    for r, field, v in ((1, 2, 8), (0, 1, 4), (1, 0, 1), (0, 2, -1)):
        bad = rows.copy()
        bad[r, field] = v
        with pytest.raises(ValueError, match="row table"):
            engine.debug_self_attn(q, kc, kc.copy(), anc, bad)
    bad = anc.copy()
    bad[1, 0, 2, 5] = 4
    with pytest.raises(ValueError, match="ancestry slot"):
        engine.debug_self_attn(q, kc, kc.copy(), bad, rows)
    with pytest.raises(ValueError, match="slots in 1..16"):
        engine.debug_self_attn(q, np.zeros((1, 8, 17, 128), np.float16), np.zeros((1, 8, 17, 128), np.float16),
                               np.zeros((2, 1, 17, 8), np.uint8), rows)
    with pytest.raises(ValueError, match="n_ctx"):
        engine.debug_self_attn(q, np.zeros((1, 449, 4, 128), np.float16), np.zeros((1, 449, 4, 128), np.float16),
                               np.zeros((2, 1, 4, 449), np.uint8), rows)
    with pytest.raises(ValueError, match="caches"):
        engine.debug_self_attn(q[:, :64], kc, kc.copy(), anc, rows)
    kv = np.zeros((2, 17, 1, 1500, 64), np.float16)
    with pytest.raises(ValueError, match="n_chunks"):
        engine.debug_cross_attn(np.zeros((17, 1, 64), np.float16), kv)
    with pytest.raises(ValueError, match="rows_per_chunk"):
        engine.debug_cross_attn(np.zeros((1, 17, 64), np.float16), kv[:, :1])
    with pytest.raises(ValueError, match="heads"):
        engine.debug_cross_attn(np.zeros((1, 1, 21 * 64), np.float16), np.zeros((2, 1, 21, 1500, 64), np.float16))
    with pytest.raises(ValueError, match="kv"):
        engine.debug_cross_attn(np.zeros((1, 1, 64), np.float16), np.zeros((2, 1, 1, 1499, 64), np.float16))


def test_search_hook_checks_arguments_before_the_device():
    """Bad search-step descriptors are refused (ValueError) before anything touches a device, GPU or not."""
    from faster_whisper_b200.config import special_tokens
    from faster_whisper_b200.synthetic import custom_dims

    dims = custom_dims(n_vocab=51865)
    st = special_tokens(dims.n_vocab)
    V = dims.n_vocab

    def call(K=2, t=1, prompt=(st.sot, st.no_timestamps), **kw):
        opts = dict(beam_size=2, max_length=20)
        opts.update(kw)
        return engine.debug_search(dims, st, np.zeros((1, K, V), np.float32), prompt, t, **opts)

    with pytest.raises(ValueError, match="K must be"):
        call(beam_size=3)
    with pytest.raises(ValueError, match="beam_size must be in"):
        call(K=17, beam_size=17)
    with pytest.raises(ValueError, match="beam_size \\* patience"):
        call(K=16, beam_size=16, patience=2.1)
    with pytest.raises(ValueError, match="num_hypotheses must be <= beam_size"):
        call(num_hypotheses=3)
    with pytest.raises(ValueError, match="startoftranscript"):
        call(prompt=(st.no_timestamps,))
    with pytest.raises(ValueError, match="prompt token id"):
        call(prompt=(st.sot, V))
    with pytest.raises(ValueError, match="step must be"):
        call(t=18)
    with pytest.raises(ValueError, match="history token id"):
        call(hist=[[[V], [0]]])
    with pytest.raises(ValueError, match="ancestry slot"):
        call(anc=2)
    with pytest.raises(ValueError, match="done is 0 or 1"):
        call(done=[2])
    with pytest.raises(ValueError, match="K free finished slots"):
        call(fin_count=[engine.MAX_FINISHED - 1])
    with pytest.raises(ValueError, match="fin_len"):
        call(fin_len=-2)
    with pytest.raises(ValueError, match="n_done"):
        engine.debug_search(dims, st, np.zeros((1, 2, V), np.float32), (st.sot,), 0, beam_size=2, n_done=2)
    with pytest.raises(ValueError, match="chunks x rows"):
        engine.debug_search(dims, st, np.zeros((6, 16, V), np.float32), (st.sot,), 0, beam_size=16)


def test_no_cpu_fallback():
    if engine.device_count() > 0:
        pytest.skip("a GPU is present")
    with pytest.raises(RuntimeError, match="no CUDA device|CPU path"):
        engine.log_mel(np.zeros(1600, np.float32), 80)
    from faster_whisper_b200.synthetic import custom_dims

    dims = custom_dims()
    with pytest.raises((RuntimeError, ValueError)):
        engine.Whisper(dims=dims, weights={}, device="cuda")
    with pytest.raises(ValueError):
        engine.Whisper(dims=dims, weights={}, device="cpu")


def test_product_never_imports_the_oracle():
    pkg = os.path.join(ROOT, "faster_whisper_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(dirpath, f), errors="replace").read()
                assert not re.search(r"^\s*(import|from)\s+oracle\b", src, flags=re.M), f
                assert not re.search(r"#include\s+[\"<].*oracle", src), f
