"""Host-side validation of the batched entry points at their widest: n = 1..64 contexts of one group.  n = 0 and n = 65 are refused by
all seven calls before any device work, and n = 64 passes the range check and is refused by the NULL check, so these run without a GPU."""
import ctypes

import pytest

N_MAX = 64


def _calls(ext):
    """the seven batched entry points, each as f(ctxs, n) with every other argument valid"""
    L = ext.L
    ids = (ctypes.c_int32 * (N_MAX + 1))()
    out = (ctypes.c_int32 * (4 * (N_MAX + 1)))()
    n_out = (ctypes.c_int32 * (N_MAX + 1))()
    toks = (ctypes.c_char_p * (N_MAX + 1))()
    keep = (ids, out, n_out, toks)
    return keep, {
        "decode_batch": lambda c, n: L.minigpt4_b200_decode_batch(c, n, ids, out),
        "flush_batch": lambda c, n: L.minigpt4_b200_flush_batch(c, n),
        "end_chat_batch": lambda c, n: L.minigpt4_b200_end_chat_batch(c, n, ctypes.cast(toks, ctypes.c_void_p), 0.8, 40, 0.9, 1.0, 1.0, 64,
                                                                      1.1, 1.0, 1.0, 0, 5.0, 1.0, 1),
        "sample_steps": lambda c, n: L.minigpt4_b200_sample_steps(c, n, 1, 0.8, 40, 0.9, 1.0, 1.0, out, None),
        "sample_until": lambda c, n: L.minigpt4_b200_sample_until(c, n, 1, None, 0.8, 40, 0.9, 1.0, 1.0, out, n_out, None, None),
        "sample_steps_mirostat": lambda c, n: L.minigpt4_b200_sample_steps_mirostat(c, n, 1, 0.8, 2, 5.0, 0.1, out, None),
        "sample_until_mirostat": lambda c, n: L.minigpt4_b200_sample_until_mirostat(c, n, 1, None, 0.8, 2, 5.0, 0.1, out, n_out, None, None),
    }


@pytest.mark.parametrize("name", ["decode_batch", "flush_batch", "end_chat_batch", "sample_steps", "sample_until", "sample_steps_mirostat",
                                  "sample_until_mirostat"])
def test_batch_sizes_outside_1_to_64_are_refused(ext, name):
    keep, calls = _calls(ext)
    f = calls[name]
    nulls = ctypes.cast((ctypes.c_void_p * (N_MAX + 1))(), ctypes.c_void_p)
    assert f(nulls, 0) == 8                    # FailedToAddString: n outside 1..64
    assert f(nulls, N_MAX + 1) == 8
    assert f(None, N_MAX + 1) == 8
    assert f(None, 0) == 8
    assert f(nulls, N_MAX) == 8                # in range, NULL contexts
    assert f(nulls, 9) == 8
    del keep
