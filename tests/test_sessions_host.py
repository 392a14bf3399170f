"""Host-side validation of the session entry points: refused before any device work, so these run without a GPU."""
import ctypes


def test_session_of_null_context_is_null(ext):
    assert ext.L.minigpt4_b200_session_create(None, 1) is None
    assert ext.L.minigpt4_b200_session_info(None, None, None, None) != 0


def test_empty_or_null_batches_are_errors(ext):
    ids = (ctypes.c_int32 * 8)()
    out = (ctypes.c_int32 * 8)()
    assert ext.L.minigpt4_b200_decode_batch(None, 0, ids, out) == 8          # FailedToAddString
    assert ext.L.minigpt4_b200_decode_batch(None, 3, ids, out) == 8
    ctxs = (ctypes.c_void_p * 9)()
    assert ext.L.minigpt4_b200_decode_batch(ctypes.cast(ctxs, ctypes.c_void_p), 9, ids, out) == 8
    assert ext.L.minigpt4_b200_decode_batch(ctypes.cast(ctxs, ctypes.c_void_p), 2, ids, out) == 8   # NULL entries
    toks = (ctypes.c_char_p * 8)()
    assert ext.L.minigpt4_b200_end_chat_batch(None, 0, ctypes.cast(toks, ctypes.c_void_p), 0.8, 40, 0.9, 1.0, 1.0, 64, 1.1, 1.0, 1.0, 0, 5.0, 1.0, 1) == 8
