"""Host-side validation of the mirostat entry points of the device sampler (minigpt4_b200_sample_steps_mirostat, sample_until_mirostat and
their seams op_sample_mirostat, op_check_log2f, op_check_powf): refused before any device work, so these run without a GPU."""
import ctypes

import numpy as np


def _steps(ext, ctxs, n, steps, ids, mirostat=2):
    return ext.L.minigpt4_b200_sample_steps_mirostat(ctxs, n, steps, 0.8, mirostat, 5.0, 0.1, ids, None)


def _until(ext, ctxs, n, max_steps, ids, n_out, stop=None, mirostat=2):
    return ext.L.minigpt4_b200_sample_until_mirostat(ctxs, n, max_steps, stop, 0.8, mirostat, 5.0, 0.1, ids, n_out, None, None)


def test_sample_steps_mirostat_refusals(ext):
    ids = (ctypes.c_int32 * 64)()
    nulls = ctypes.cast((ctypes.c_void_p * 9)(), ctypes.c_void_p)
    assert _steps(ext, None, 1, 1, ids) == 8                                   # FailedToAddString
    assert _steps(ext, nulls, 1, 1, None) == 8                                 # NULL ids_out
    assert _steps(ext, nulls, 0, 1, ids) == 8                                  # n outside 1..8
    assert _steps(ext, nulls, 9, 1, ids) == 8
    assert _steps(ext, nulls, 2, 1, ids) == 8                                  # NULL contexts
    assert _steps(ext, nulls, 1, 0, ids) == 8                                  # steps < 1 (and a NULL context)
    for m in (0, 3, -1):                                                       # mirostat outside 1..2
        assert _steps(ext, nulls, 1, 1, ids, mirostat=m) == 8


def test_sample_until_mirostat_refusals(ext):
    ids, n_out = (ctypes.c_int32 * 64)(), (ctypes.c_int32 * 8)()
    nulls = ctypes.cast((ctypes.c_void_p * 9)(), ctypes.c_void_p)
    assert _until(ext, None, 1, 1, ids, n_out) == 8
    assert _until(ext, nulls, 1, 1, None, n_out) == 8                          # NULL ids_out
    assert _until(ext, nulls, 1, 1, ids, None) == 8                            # NULL n_out
    assert _until(ext, nulls, 0, 1, ids, n_out) == 8                           # n outside 1..8
    assert _until(ext, nulls, 9, 1, ids, n_out) == 8
    assert _until(ext, nulls, 2, 1, ids, n_out) == 8                           # NULL contexts
    assert _until(ext, nulls, 1, 0, ids, n_out) == 8                           # max_steps < 1
    assert _until(ext, nulls, 1, 4, ids, n_out, b"#" * 33) == 8                # stop text over 32 bytes
    for m in (0, 3):
        assert _until(ext, nulls, 1, 1, ids, n_out, mirostat=m) == 8


def test_seams_refuse_bad_arguments(ext):
    lg = np.zeros(16, np.float32)
    ids, mu = np.zeros(4, np.int32), np.zeros(4, np.float32)
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    f = ext.L.minigpt4_b200_op_sample_mirostat
    assert f(None, 16, 1, 0.8, 1, 5.0, 1.0, 4, 0, p(ids), p(mu), None) == 8
    assert f(p(lg), 16, 1, 0.8, 1, 5.0, 1.0, 4, 0, None, p(mu), None) == 8
    assert f(p(lg), 16, 1, 0.8, 1, 5.0, 1.0, 4, 0, p(ids), None, None) == 8
    assert f(p(lg), 0, 1, 0.8, 1, 5.0, 1.0, 4, 0, p(ids), p(mu), None) == 8    # n_vocab < 1
    assert f(p(lg), 16, 1, 0.8, 1, 5.0, 1.0, 0, 0, p(ids), p(mu), None) == 8   # n_draws < 1
    assert f(p(lg), 16, 1, 0.8, 0, 5.0, 1.0, 4, 0, p(ids), p(mu), None) == 8   # mirostat 0 / 3
    assert f(p(lg), 16, 1, 0.8, 3, 5.0, 1.0, 4, 0, p(ids), p(mu), None) == 8
    assert f(p(lg), 16, 1, 0.8, 1, 5.0, 1.0, 4, 2, p(ids), p(mu), None) == 8   # on_device outside 0..1
    assert f(p(lg), 16, 1, 0.0, 1, 5.0, 1.0, 4, 1, p(ids), p(mu), None) == 8   # greedy on the device: not the sampler
    bad = ctypes.c_longlong(0)
    assert ext.L.minigpt4_b200_op_check_log2f(5, 4, ctypes.byref(bad)) == 8
    assert ext.L.minigpt4_b200_op_check_log2f(0, 1, None) == 8
    assert ext.L.minigpt4_b200_op_check_powf(2.0, 5, 4, ctypes.byref(bad)) == 8
    assert ext.L.minigpt4_b200_op_check_powf(2.0, 0, 1, None) == 8


def test_host_seam_starts_mu_at_twice_tau(ext):
    """the host side of op_sample_mirostat needs no GPU: μ starts at 2 tau and moves by eta (surprise - tau) per draw"""
    logits = np.random.default_rng(3).standard_normal(64).astype(np.float32) * 3
    for mode in (1, 2):
        ids, mu = ext.op_sample_mirostat(logits, 7, 8, temp=0.8, mirostat=mode, mirostat_tau=5.0, mirostat_eta=0.0, on_device=False)
        assert mu.tolist() == [10.0] * 8                                       # eta 0: μ stays 2 tau
        assert ids.tolist() == ext.host_sample(logits, 7, 8, temp=0.8, mirostat=mode, mirostat_tau=5.0, mirostat_eta=0.0).tolist()
