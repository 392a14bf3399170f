"""Host-side validation of minigpt4_b200_sample_until and its seam minigpt4_b200_op_reply_stop: refused before any device work, so these
run without a GPU."""
import ctypes


def _until(ext, ctxs, n, max_steps, ids, n_out, stop=None):
    return ext.L.minigpt4_b200_sample_until(ctxs, n, max_steps, stop, 0.8, 40, 0.9, 1.0, 1.0, ids, n_out, None, None)


def test_null_and_out_of_range_calls_are_errors(ext):
    ids, n_out = (ctypes.c_int32 * 64)(), (ctypes.c_int32 * 8)()
    nulls = ctypes.cast((ctypes.c_void_p * 9)(), ctypes.c_void_p)
    assert _until(ext, None, 1, 1, ids, n_out) == 8                            # FailedToAddString
    assert _until(ext, nulls, 1, 1, None, n_out) == 8                          # NULL ids_out
    assert _until(ext, nulls, 1, 1, ids, None) == 8                            # NULL n_out
    assert _until(ext, nulls, 0, 1, ids, n_out) == 8                           # n outside 1..8
    assert _until(ext, nulls, 9, 1, ids, n_out) == 8
    assert _until(ext, nulls, 2, 1, ids, n_out) == 8                           # NULL contexts
    assert _until(ext, nulls, 1, 0, ids, n_out) == 8                           # max_steps < 1 (and a NULL context)
    assert _until(ext, nulls, 1, 4, ids, n_out, b"#" * 33) == 8                # stop text over 32 bytes (and a NULL context)


def test_reply_stop_seam_refuses_a_null_context(ext):
    at = ctypes.c_int32(0)
    ids = (ctypes.c_int32 * 2)(1, 2)
    assert ext.L.minigpt4_b200_op_reply_stop(None, ids, 2, None, None, ctypes.byref(at)) == 8
