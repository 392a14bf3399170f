"""Log-probabilities of generated replies, without a GPU: minigpt4_b200_sample_until_logprobs and minigpt4_b200_op_logprobs refuse bad
arguments (return 8) before they touch a context or the device, and both symbols are in the extension table."""
import ctypes

import numpy as np
import pytest

import minigpt4_cpp_b200.minigpt4_library as ml

REFUSED = 8


def _until(lib, ctxs, n, top_n=5, mirostat=0, logprob=True, top_ids=True, ids=True, n_out=True, max_steps=4):
    L = lib.library
    L.minigpt4_b200_sample_until_logprobs.argtypes, L.minigpt4_b200_sample_until_logprobs.restype = ml._EXT["minigpt4_b200_sample_until_logprobs"]
    size = max_steps * max(1, n)
    buf = lambda dt, k=1: np.zeros(size * k, dt)   # noqa: E731
    a_ids, a_n, a_st, a_lp, a_rk = buf(np.int32), np.zeros(max(1, n), np.int32), np.zeros(max(1, n), np.int32), buf(np.float32), buf(np.int32)
    a_tid, a_tlp = buf(np.int32, max(1, top_n)), buf(np.float32, max(1, top_n))
    ms = ctypes.c_float(0)
    return L.minigpt4_b200_sample_until_logprobs(ctxs, n, max_steps, None, 0.8, 40, 0.9, 1.0, 1.0, mirostat, 5.0, 1.0, top_n,
                                                 ml._ptr(a_ids) if ids else None, ml._ptr(a_n) if n_out else None, ml._ptr(a_st),
                                                 ml._ptr(a_lp) if logprob else None, ml._ptr(a_rk), ml._ptr(a_tid) if top_ids else None,
                                                 ml._ptr(a_tlp), ctypes.byref(ms))


def _null_ctxs(n):
    return ctypes.cast((ctypes.c_void_p * max(1, n))(), ctypes.c_void_p)   # n NULL contexts: refused if a check ever reaches them


def test_symbols_in_the_extension_table():
    assert "minigpt4_b200_sample_until_logprobs" in ml.EXT_SYMBOLS
    assert "minigpt4_b200_op_logprobs" in ml.EXT_SYMBOLS


@pytest.mark.parametrize("case", ["null-ctxs", "null-logprob", "null-ids", "null-n_out", "null-top_ids", "n-0", "n-65", "top_n--1", "top_n-21",
                                  "mirostat--1", "mirostat-3"])
def test_sample_until_logprobs_refusals(lib, case):
    kw = {"null-logprob": dict(logprob=False), "null-ids": dict(ids=False), "null-n_out": dict(n_out=False), "null-top_ids": dict(top_ids=False),
          "top_n--1": dict(top_n=-1), "top_n-21": dict(top_n=21), "mirostat--1": dict(mirostat=-1), "mirostat-3": dict(mirostat=3)}.get(case, {})
    n = {"n-0": 0, "n-65": 65}.get(case, 2)
    ctxs = None if case == "null-ctxs" else _null_ctxs(n)
    assert _until(lib, ctxs, n, **kw) == REFUSED


def test_top_n_zero_needs_no_top_arrays(lib):
    # top_n 0 with NULL top_ids passes the argument checks and is refused only at the NULL contexts
    assert _until(lib, _null_ctxs(1), 1, top_n=0, top_ids=False) == REFUSED


def _op(lib, logits, ids, top_n, rows=None, n_vocab=None, logprob=True, top_ids=True):
    L = lib.library
    L.minigpt4_b200_op_logprobs.argtypes, L.minigpt4_b200_op_logprobs.restype = ml._EXT["minigpt4_b200_op_logprobs"]
    rows = len(ids) if rows is None else rows
    V = logits.shape[1] if n_vocab is None else n_vocab
    k = max(1, top_n)
    lp, rk, tid, tlp = np.zeros(max(1, rows), np.float32), np.zeros(max(1, rows), np.int32), np.zeros(max(1, rows) * k, np.int32), np.zeros(max(1, rows) * k, np.float32)
    return L.minigpt4_b200_op_logprobs(ml._ptr(logits), rows, V, ml._ptr(np.ascontiguousarray(ids, np.int32)), top_n, ml._ptr(lp) if logprob else None,
                                       ml._ptr(rk), ml._ptr(tid) if top_ids else None, ml._ptr(tlp), None)


@pytest.mark.parametrize("case", ["rows-0", "rows-65", "n_vocab-0", "top_n-21", "top_n--1", "id-out-of-range", "id-negative", "null-logprob",
                                  "null-top_ids"])
def test_op_logprobs_refusals(lib, case):
    lg = np.zeros((2, 16), np.float32)
    ids = {"id-out-of-range": [0, 16], "id-negative": [-1, 0]}.get(case, [0, 1])
    kw = {"rows-0": dict(rows=0), "rows-65": dict(rows=65), "n_vocab-0": dict(n_vocab=0), "null-logprob": dict(logprob=False),
          "null-top_ids": dict(top_ids=False)}.get(case, {})
    top_n = {"top_n-21": 21, "top_n--1": -1}.get(case, 3)
    assert _op(lib, lg, ids, top_n, **kw) == REFUSED
