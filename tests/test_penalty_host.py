"""Repetition, presence and frequency penalties without a GPU: the host sampler's penalize (minigpt4_b200_op_penalize, on_device 0) bit for
bit against a numpy float32 restatement of the semantics in include/minigpt4_b200.h, and every refusal that needs no device."""
import ctypes

import numpy as np
import pytest

import minigpt4_cpp_b200.minigpt4_library as ml

REFUSED = 8
N_CTX = 32768
VOCABS = [1, 13, 14, 32000, 32001]
PENALTIES = [1.0, 1.1, 0.5, 2.0]
ALPHAS = [(0.0, 0.0), (1.0, 0.0), (0.0, 1.0), (-0.5, -0.5), (1.0, -0.5)]   # (alpha_presence, alpha_frequency)
WINDOWS = [0, 1, 64, N_CTX]


def np_penalize(lg, hist, repeat_last_n, repeat_penalty, alpha_presence, alpha_frequency, penalize_nl):
    """the header's semantics in numpy float32: every operation rounds to float32 on its own"""
    out = np.array(lg, np.float32)
    V = out.size
    w = np.asarray(hist, np.int64)[len(hist) - min(repeat_last_n, len(hist)):]
    ids, counts = np.unique(w, return_counts=True)
    if not penalize_nl and V > 13:
        counts, ids = counts[ids != 13], ids[ids != 13]
    rp, ap, af = np.float32(repeat_penalty), np.float32(alpha_presence), np.float32(alpha_frequency)
    z = out[ids]
    z1 = z if rp == np.float32(1) else np.where(z <= 0, z * rp, z / rp).astype(np.float32)
    z2 = z1 if (af == 0 and ap == 0) else (z1 - (counts.astype(np.float32) * af + ap)).astype(np.float32)
    out[ids] = z2
    return out


def bits(x):
    return np.asarray(x, np.float32).view(np.uint32)


def penalty_rows(V, rng):
    """rows with +-0, negative and equal logits, and histories that hold ids 0, 13 and n_vocab - 1 with repeats: one longer than n_ctx, one
    empty, one short"""
    lg = rng.normal(0, 3, size=(3, V)).astype(np.float32)
    for r in range(3):
        lg[r, 0] = (-0.0, 0.0, -2.5)[r]
        lg[r, min(13, V - 1)] = (0.0, -0.0, 1.5)[r]
        lg[r, V - 1] = lg[r, V // 2]          # equal logits
        lg[r, rng.integers(0, V, size=min(V, 50))] = -1.0
    long = rng.integers(0, min(V, 300), size=N_CTX + 1000)
    long[rng.integers(0, long.size, size=200)] = min(13, V - 1)
    long[-5:] = [0, min(13, V - 1), V - 1, V - 1, 0]
    short = [min(13, V - 1), V - 1, 0, 0, min(13, V - 1)]
    return lg, [long.tolist(), [], short]


@pytest.mark.parametrize("penalize_nl", [0, 1])
@pytest.mark.parametrize("alphas", ALPHAS, ids=[f"ap{a}-af{f}" for a, f in ALPHAS])
@pytest.mark.parametrize("repeat_penalty", PENALTIES)
@pytest.mark.parametrize("V", VOCABS)
def test_host_penalize_against_numpy(ext, V, repeat_penalty, alphas, penalize_nl):
    rng = np.random.default_rng(V + int(repeat_penalty * 10))
    lg, hist = penalty_rows(V, rng)
    ap, af = alphas
    for n in WINDOWS:
        got, ms = ext.op_penalize(lg, hist, n, repeat_penalty, ap, af, bool(penalize_nl), on_device=False)
        assert ms == 0.0
        for r in range(lg.shape[0]):
            want = np_penalize(lg[r], hist[r], n, repeat_penalty, ap, af, penalize_nl)
            assert np.array_equal(bits(got[r]), bits(want)), f"row {r} window {n}: {np.nonzero(bits(got[r]) != bits(want))[0][:8]}"


def test_neutral_penalties_change_nothing(ext):
    rng = np.random.default_rng(5)
    lg, hist = penalty_rows(32000, rng)
    for n, rp, ap, af in ((64, 1.0, 0.0, 0.0), (0, 1.3, 1.0, 1.0)):
        got, _ = ext.op_penalize(lg, hist, n, rp, ap, af, False, on_device=False)
        assert np.array_equal(bits(got), bits(lg))


def test_symbols_in_the_extension_table():
    for s in ("minigpt4_b200_sample_until_penalized", "minigpt4_b200_end_chat_penalized", "minigpt4_b200_op_penalize"):
        assert s in ml.EXT_SYMBOLS


# ---- refusals ----------------------------------------------------------------------------------------------------------------------
def _op(lib, case):
    L = lib.library
    L.minigpt4_b200_op_penalize.argtypes, L.minigpt4_b200_op_penalize.restype = ml._EXT["minigpt4_b200_op_penalize"]
    lg, out = np.zeros((2, 16), np.float32), np.zeros((2, 16), np.float32)
    hist, n_last = np.array([1, 2, 3, 4], np.int32), np.array([2, 2], np.int32)
    a = dict(rows=2, n_vocab=16, repeat_last_n=64, rp=1.1, ap=0.0, af=0.0, nl=1, on_device=0, hist=hist, n_last=n_last, logits=lg, out=out)
    if case.startswith("id-"):
        hist[3] = {"id-negative": -1, "id-n_vocab": 16}[case]
    elif case == "n_last-negative":
        n_last[1] = -1
    elif case == "null-last_ids":
        a["hist"] = None
    else:
        a.update({"rows-0": dict(rows=0), "rows-65": dict(rows=65), "n_vocab-0": dict(n_vocab=0), "on_device-2": dict(on_device=2),
                  "repeat_last_n--1": dict(repeat_last_n=-1), "penalty-0": dict(rp=0.0), "penalty--1": dict(rp=-1.0),
                  "penalty-inf": dict(rp=float("inf")), "penalty-nan": dict(rp=float("nan")), "presence-inf": dict(ap=float("inf")),
                  "frequency-nan": dict(af=float("nan")), "penalize_nl-2": dict(nl=2), "penalize_nl--1": dict(nl=-1),
                  "null-logits": dict(logits=None), "null-out": dict(out=None)}[case])
    return L.minigpt4_b200_op_penalize(ml._ptr(a["logits"]), a["rows"], a["n_vocab"], ml._ptr(a["hist"]), ml._ptr(a["n_last"]), a["repeat_last_n"],
                                       a["rp"], a["ap"], a["af"], a["nl"], a["on_device"], ml._ptr(a["out"]), None)


OP_CASES = ["rows-0", "rows-65", "n_vocab-0", "on_device-2", "repeat_last_n--1", "penalty-0", "penalty--1", "penalty-inf", "penalty-nan",
            "presence-inf", "frequency-nan", "penalize_nl-2", "penalize_nl--1", "null-logits", "null-out", "id-negative", "id-n_vocab",
            "n_last-negative", "null-last_ids"]


@pytest.mark.parametrize("case", OP_CASES)
def test_op_penalize_refusals(lib, case):
    assert _op(lib, case) == REFUSED


def _until(lib, ctxs, n, mirostat=0, repeat_last_n=64, rp=1.1, ap=0.0, af=0.0, nl=1, ids=True, n_out=True):
    L = lib.library
    L.minigpt4_b200_sample_until_penalized.argtypes, L.minigpt4_b200_sample_until_penalized.restype = ml._EXT["minigpt4_b200_sample_until_penalized"]
    a_ids, a_n, a_st = np.zeros(4 * max(1, n), np.int32), np.zeros(max(1, n), np.int32), np.zeros(max(1, n), np.int32)
    return L.minigpt4_b200_sample_until_penalized(ctxs, n, 4, None, 0.8, 40, 0.9, 1.0, 1.0, mirostat, 5.0, 1.0, repeat_last_n, rp, ap, af, nl, None, None,
                                                  ml._ptr(a_ids) if ids else None, ml._ptr(a_n) if n_out else None, ml._ptr(a_st),
                                                  ctypes.byref(ctypes.c_float(0)))


def _null_ctxs(n):
    return ctypes.cast((ctypes.c_void_p * max(1, n))(), ctypes.c_void_p)   # n NULL contexts: refused if a check ever reaches them


UNTIL_CASES = {"null-ctxs": {}, "n-0": {}, "n-65": {}, "null-ids": dict(ids=False), "null-n_out": dict(n_out=False), "mirostat--1": dict(mirostat=-1),
               "mirostat-3": dict(mirostat=3), "repeat_last_n--1": dict(repeat_last_n=-1), "penalty-0": dict(rp=0.0),
               "penalty-nan": dict(rp=float("nan")), "presence-inf": dict(ap=float("-inf")), "frequency-nan": dict(af=float("nan")),
               "penalize_nl-2": dict(nl=2)}


@pytest.mark.parametrize("case", list(UNTIL_CASES))
def test_sample_until_penalized_refusals(lib, case):
    n = {"n-0": 0, "n-65": 65}.get(case, 2)
    ctxs = None if case == "null-ctxs" else _null_ctxs(n)
    assert _until(lib, ctxs, n, **UNTIL_CASES[case]) == REFUSED


def test_end_chat_penalized_refuses_a_null_context(lib):
    L = lib.library
    L.minigpt4_b200_end_chat_penalized.argtypes, L.minigpt4_b200_end_chat_penalized.restype = ml._EXT["minigpt4_b200_end_chat_penalized"]
    tok = ctypes.c_char_p()
    assert L.minigpt4_b200_end_chat_penalized(None, ctypes.byref(tok), 0.8, 40, 0.9, 1.0, 1.0, 64, 1.1, 0.0, 0.0, 1, 0, 5.0, 1.0, None, 0, None) == REFUSED
