"""CPU: the decode-session entry points are exported and refuse bad arguments before any device work."""
import ctypes as C

import pytest

from faster_whisper_b200 import engine


def test_session_symbols_are_exported():
    lib = engine.load_library()
    for name in ("b2w_session_create", "b2w_session_push", "b2w_session_run", "b2w_session_pending", "b2w_session_counters",
                 "b2w_session_destroy"):
        assert hasattr(lib, name) and name in engine.ABI_SYMBOLS


def test_session_calls_check_arguments_before_the_device():
    lib = engine.load_library()
    o = engine._GenOpts()
    lib.b2w_gen_opts_default(C.byref(o))
    slots, h, n = C.c_int32(0), C.c_void_p(), C.c_int32()
    with pytest.raises(ValueError, match="null model"):
        engine._check(lib.b2w_session_create(None, C.byref(o), C.byref(slots), C.byref(h)))
    with pytest.raises(ValueError, match="null argument"):
        engine._check(lib.b2w_session_push(None, None, 0, None, 1, 2, C.byref(n)))
    with pytest.raises(ValueError, match="null argument"):
        engine._check(lib.b2w_session_run(None, C.byref(n), None, None, None, None, None))
    with pytest.raises(ValueError, match="null argument"):
        engine._check(lib.b2w_session_pending(None, C.byref(n)))
    with pytest.raises(ValueError, match="null argument"):
        engine._check(lib.b2w_session_counters(None, None, None))
    lib.b2w_session_destroy(None)  # a no-op, as b2w_encoded_free(NULL)


def test_push_checks_every_item_before_queueing_any():
    """DecodeQueue.push runs these checks over all items first, so a rejected push leaves nothing queued."""
    sot, V = 50258, 51866
    good = [[sot, 1], [50360, sot, 2, 3]]
    items = engine.check_queue_items(good, [10, 448], V, sot, 448)
    assert [p.tolist() for p, _ in items] == good and [ml for _, ml in items] == [10, 448]
    for prompts, mls, match in (
        (good + [[5, 6]], [10, 10, 10], "startoftranscript"),
        (good + [[sot, V]], [10, 10, 10], "token id"),
        (good + [[]], [10, 10, 10], "empty prompt"),
        (good, [10, 449], "max_length"),
        (good, [2, 10], "max_length"),
        (good, [10], "one max_length"),
    ):
        with pytest.raises(ValueError, match=match):
            engine.check_queue_items(prompts, mls, V, sot, 448)
