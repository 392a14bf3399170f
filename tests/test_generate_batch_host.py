"""Per-conversation settings without a GPU (minigpt4_b200_generate_batch): the ctypes mirror of struct MiniGPT4B200GenParams against the layout
include/minigpt4_b200.h states, GenParams' defaults against B200.sample_until's, and the refusals that need no context."""
import ctypes
import inspect
import re
from pathlib import Path

import minigpt4_cpp_b200.minigpt4_library as ml

REFUSED = 8
HEADER = Path(__file__).resolve().parent.parent / "include" / "minigpt4_b200.h"
# the offsets the header's comment states
OFFSETS = dict(size=0, max_steps=4, stop=8, temp=16, top_k=20, top_p=24, tfs_z=28, typical_p=32, mirostat=36, mirostat_tau=40, mirostat_eta=44,
               repeat_last_n=48, repeat_penalty=52, alpha_presence=56, alpha_frequency=60, penalize_nl=64, n_last=68, last_ids=72)


def test_struct_layout_matches_header():
    assert ctypes.sizeof(ml.GenParamsC) == 80
    for name, off in OFFSETS.items():
        assert getattr(ml.GenParamsC, name).offset == off, name
    text = HEADER.read_text()
    body = re.search(r"struct MiniGPT4B200GenParams \{(.*?)\n\};", text, re.S).group(1)
    declared = re.findall(r"(\w+)(?=\s*[,;])", re.sub(r"/\*.*?\*/", "", body, flags=re.S))
    assert declared == [f for f, _ in ml.GenParamsC._fields_], "the header's field order"
    stated = dict((k, int(v)) for v, k in re.findall(r"(\d+) (\w+)", text[text.index("offset  0"):text.index("struct MiniGPT4B200GenParams {")]))
    assert stated == OFFSETS


def test_gen_params_defaults_are_sample_until_defaults():
    sig = inspect.signature(ml.B200.sample_until).parameters
    g = ml.GenParams(max_steps=7)
    for name in ("stop", "temp", "top_k", "top_p", "tfs_z", "typical_p", "mirostat", "mirostat_tau", "mirostat_eta"):
        assert getattr(g, name) == sig[name].default, name
    assert g.repeat_penalty == 1.0 and g.alpha_presence == 0.0 and g.alpha_frequency == 0.0, "neutral penalties"
    assert g.last_ids is None


def test_extension_table_has_generate_batch():
    assert "minigpt4_b200_generate_batch" in ml.EXT_SYMBOLS


def _call(lib, params, n=1, top_n=0, logprob=False):
    """generate_batch over n stand-in context pointers: every call here is refused before a context is read"""
    ctxs = (ctypes.c_void_p * n)(*([1] * n))
    ids, n_out = (ctypes.c_int32 * 64)(), (ctypes.c_int32 * 8)()
    lp = (ctypes.c_float * 64)() if logprob else None
    fn = lib.library.minigpt4_b200_generate_batch
    fn.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int] + [ctypes.c_void_p] * 7 + [ctypes.POINTER(ctypes.c_float)]
    fn.restype = ctypes.c_int
    return fn(ctypes.cast(ctxs, ctypes.c_void_p), n, params, top_n, ctypes.cast(ids, ctypes.c_void_p), ctypes.cast(n_out, ctypes.c_void_p), None,
              ctypes.cast(lp, ctypes.c_void_p) if lp is not None else None, None, None, None, None)


def test_refusals_before_any_context_is_read(lib):
    arr, _keep = ml.B200.gen_params_c([ml.GenParams(max_steps=4)] * 3)
    assert _call(lib, None, 3) == REFUSED, "NULL params"
    for bad in (0, ctypes.sizeof(ml.GenParamsC) - 8, ctypes.sizeof(ml.GenParamsC) + 8):
        arr[1].size = bad
        assert _call(lib, ctypes.cast(arr, ctypes.c_void_p), 3) == REFUSED, f"size {bad}"
    arr[1].size = ctypes.sizeof(ml.GenParamsC)
    assert _call(lib, ctypes.cast(arr, ctypes.c_void_p), 0) == REFUSED, "no contexts"
    assert _call(lib, ctypes.cast(arr, ctypes.c_void_p), 65) == REFUSED, "65 contexts"
    assert _call(lib, ctypes.cast(arr, ctypes.c_void_p), 3, top_n=5) == REFUSED, "top_n without records"
