"""Host-side validation of minigpt4_b200_score_tokens: the refusals that need no device.  NULL arrays, n outside 1..64 and NULL contexts
are refused before any context is looked at, so these run without a GPU."""
import ctypes

import pytest

N_MAX = 64


def _call(ext, ctxs, n, ids=True, n_ids=True, logprob=True, keep=0):
    a = (ctypes.c_int32 * (N_MAX + 1))(*([1] * (N_MAX + 1)))
    lens = (ctypes.c_int32 * (N_MAX + 1))(*([1] * (N_MAX + 1)))
    lp = (ctypes.c_float * (N_MAX + 1))()
    rk = (ctypes.c_int32 * (N_MAX + 1))()
    return ext.L.minigpt4_b200_score_tokens(ctxs, n, a if ids else None, lens if n_ids else None, keep, lp if logprob else None, rk, None)


@pytest.mark.parametrize("n", [0, N_MAX + 1, 9, N_MAX])
def test_null_or_out_of_range_batches_are_refused(ext, n):
    nulls = ctypes.cast((ctypes.c_void_p * (N_MAX + 1))(), ctypes.c_void_p)
    assert _call(ext, nulls, n) == 8            # FailedToAddString: n outside 1..64, or NULL contexts
    assert _call(ext, None, n) == 8


@pytest.mark.parametrize("missing", ["ids", "n_ids", "logprob"])
def test_null_arrays_are_refused(ext, missing):
    nulls = ctypes.cast((ctypes.c_void_p * (N_MAX + 1))(), ctypes.c_void_p)
    assert _call(ext, nulls, 1, **{missing: False}) == 8


def test_score_tokens_is_declared(ext):
    import minigpt4_cpp_b200.minigpt4_library as ml
    assert "minigpt4_b200_score_tokens" in ml.EXT_SYMBOLS
    assert hasattr(ext.L, "minigpt4_b200_score_tokens")
