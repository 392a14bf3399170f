"""Host-side validation of the device sampler's entry points (minigpt4_b200_sample_steps, op_sample, op_check_libm): refused before any
device work, so these run without a GPU."""
import ctypes

import numpy as np


def _steps(ext, ctxs, n, steps, ids):
    return ext.L.minigpt4_b200_sample_steps(ctxs, n, steps, 0.8, 40, 0.9, 1.0, 1.0, ids, None)


def test_null_and_out_of_range_calls_are_errors(ext):
    ids = (ctypes.c_int32 * 64)()
    assert _steps(ext, None, 1, 1, ids) == 8                                   # FailedToAddString
    nulls = ctypes.cast((ctypes.c_void_p * 9)(), ctypes.c_void_p)
    assert _steps(ext, nulls, 1, 1, None) == 8                                 # NULL ids_out
    assert _steps(ext, nulls, 0, 1, ids) == 8                                  # n outside 1..8
    assert _steps(ext, nulls, 9, 1, ids) == 8
    assert _steps(ext, nulls, 2, 1, ids) == 8                                  # NULL contexts
    assert _steps(ext, nulls, 1, 0, ids) == 8                                  # steps < 1 (and a NULL context)


def test_op_hooks_refuse_bad_arguments(ext):
    lg = np.zeros(16, np.float32)
    out = np.zeros(4, np.int32)
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    assert ext.L.minigpt4_b200_op_sample(p(lg), 16, 1, 0.0, 40, 0.9, 1.0, 1.0, 4, p(out)) == 8     # greedy: not the sampler
    assert ext.L.minigpt4_b200_op_sample(None, 16, 1, 0.8, 40, 0.9, 1.0, 1.0, 4, p(out)) == 8
    assert ext.L.minigpt4_b200_op_sample(p(lg), 16, 1, 0.8, 40, 0.9, 1.0, 1.0, 0, p(out)) == 8
    bad = ctypes.c_longlong(0)
    assert ext.L.minigpt4_b200_op_check_libm(2, 0, 1, ctypes.byref(bad)) == 8
    assert ext.L.minigpt4_b200_op_check_libm(0, 5, 4, ctypes.byref(bad)) == 8
