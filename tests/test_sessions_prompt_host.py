"""Host-side validation of minigpt4_b200_flush_batch: refused before any device work, so these run without a GPU."""
import ctypes


def test_empty_null_or_long_batches_are_errors(ext):
    assert ext.L.minigpt4_b200_flush_batch(None, 0) == 8          # FailedToAddString
    assert ext.L.minigpt4_b200_flush_batch(None, 3) == 8
    ctxs = (ctypes.c_void_p * 9)()
    assert ext.L.minigpt4_b200_flush_batch(ctypes.cast(ctxs, ctypes.c_void_p), 9) == 8
    assert ext.L.minigpt4_b200_flush_batch(ctypes.cast(ctxs, ctypes.c_void_p), 0) == 8
    assert ext.L.minigpt4_b200_flush_batch(ctypes.cast(ctxs, ctypes.c_void_p), 2) == 8   # NULL entries
