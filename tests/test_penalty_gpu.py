"""Repetition, presence and frequency penalties on the GPU (minigpt4_b200_sample_until_penalized; llama_penalty.cuh, DESIGN.md §4.15):

- the kernel (op_penalize) bit for bit against numpy, at 1 .. 64 rows;
- neutral parameters: ids, stops and end state of sample_until / sample_until_mirostat, with the same kernel launches;
- against the host twin: a group driven by sample_until_penalized and a twin group driven by a loop of end_chat_penalized give the same
  ids, n_past, logits bits, greedy id and next draw, on every tiny weight type and at B = 1, 3, 9 and 64 with greedy, the web UI chain,
  top_k 0 / top_p 0.95, mirostat 1 / 2 and constrained contexts;
- greedy against a numpy loop over raw logits (no host sampler);
- chunked replies, stops at different steps, a stop text across two calls, max_steps and the last slot of n_ctx, a 4096-wide 32000-id model;
- refusals, the penalty scratch's memory, and MiniGPT4ChatBot.generate_on_device."""
import ctypes

import numpy as np
import pytest

from minigpt4_cpp_b200.minigpt4_library import _ptr, choices_dfa
from test_logprobs_gpu import files, free, group  # noqa: F401  (files: the module's model fixture)
from test_penalty_host import ALPHAS, PENALTIES, VOCABS, WINDOWS, bits, np_penalize, penalty_rows
from test_reply_gpu import ref_stop

pytestmark = pytest.mark.gpu

WEBUI = dict(temp=0.8, top_k=40, top_p=0.9)
PARAMS = {"greedy": dict(temp=0.0), "webui": WEBUI, "top_k-0-top_p-0.95": dict(temp=0.8, top_k=0, top_p=0.95),
          "mirostat-1": dict(temp=0.8, mirostat=1), "mirostat-2": dict(temp=0.8, mirostat=2)}
# every stage at work (penalize_nl 0: id 13 keeps its raw logit)
PEN = dict(repeat_last_n=16, repeat_penalty=1.5, alpha_presence=0.5, alpha_frequency=0.25, penalize_nl=False)
REFUSED = 8


def histories(n, seed=3, V=1000):
    """context i's history: none for every third context, otherwise 1 .. 40 ids with repeats (13 among them)"""
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n):
        h = [] if i % 3 == 2 else rng.integers(3, min(V, 60), size=1 + (7 * i) % 40).tolist()
        if h:
            h[len(h) // 2] = 13
        out.append(h)
    return out


def end_chat(lib, c, p):
    tok = ctypes.c_char_p()
    assert lib.library.minigpt4_end_chat(c.ptr, ctypes.byref(tok), 0, p.get("temp", 0.8), p.get("top_k", 40), p.get("top_p", 0.9), 1.0, 1.0,
                                         64, 1.1, 1.0, 1.0, p.get("mirostat", 0), 5.0, 1.0, 1) == 0
    return tok.value


def same_state(lib, ext, a, b, p):
    """n_past, raw logits, greedy id, and the generators and μ through one more (unpenalised) end_chat"""
    assert ext.n_past(a) == ext.n_past(b)
    assert np.array_equal(bits(ext.logits(a)), bits(ext.logits(b)))
    assert ext.greedy_id(a) == ext.greedy_id(b)
    assert end_chat(lib, a, p) == end_chat(lib, b, p)
    assert np.array_equal(bits(ext.logits(a)), bits(ext.logits(b)))


def twin_loop(ext, ctxs, steps, hist, p, pen):
    """the host twin: steps[i] calls of end_chat_penalized on context i, each with the history and the ids fed so far"""
    out = []
    for c, k, h in zip(ctxs, steps, hist):
        fed = []
        for _ in range(k):
            fed.append(ext.end_chat_penalized(c, h + fed, **pen, **p)[1])
        out.append(fed)
    return out


# ---- the kernel --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("penalize_nl", [0, 1])
@pytest.mark.parametrize("repeat_penalty", PENALTIES)
@pytest.mark.parametrize("V", VOCABS)
def test_kernel_against_numpy(ext, V, repeat_penalty, penalize_nl):
    rng = np.random.default_rng(V * 3 + int(repeat_penalty * 10))
    lg3, hist3 = penalty_rows(V, rng)
    for rows in (1, 3, 64):
        lg = np.concatenate([lg3] * 22)[:rows]
        lg[3:] += rng.normal(0, 1, size=lg[3:].shape).astype(np.float32)
        hist = (hist3 * 22)[:rows]
        for ap, af in ALPHAS:
            for n in WINDOWS:
                got, ms = ext.op_penalize(lg, hist, n, repeat_penalty, ap, af, bool(penalize_nl), on_device=True)
                assert ms > 0
                for r in range(rows):
                    want = np_penalize(lg[r], hist[r], n, repeat_penalty, ap, af, penalize_nl)
                    assert np.array_equal(bits(got[r]), bits(want)), (rows, r, n, ap, af)


# ---- neutral parameters ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 3, 9, 64])
@pytest.mark.parametrize("params", ["greedy", "webui", "mirostat-2"])
def test_neutral_parameters_are_sample_until(lib, ext, files, n, params):
    p = PARAMS[params]
    for neutral in (dict(repeat_penalty=1.0, alpha_presence=0.0, alpha_frequency=0.0, penalize_nl=False), dict(repeat_last_n=0, repeat_penalty=1.3)):
        a, b = group(ext, files["q4_1"], n), group(ext, files["q4_1"], n)
        l0 = [ext.stats(c).kernel_launches for c in a + b]
        ids_a, st_a, _ = ext.sample_until(a, 12, None, **p)
        ids_b, st_b, _ = ext.sample_until_penalized(b, 12, None, histories(n), **neutral, **p)
        assert ids_a == ids_b and st_a == st_b
        l1 = [ext.stats(c).kernel_launches for c in a + b]
        assert [y - x for x, y in zip(l0[:n], l1[:n])] == [y - x for x, y in zip(l0[n:], l1[n:])], "the same work"
        owned = [ext.session_info(c)[1] for c in a]
        assert [ext.session_info(c)[1] for c in b] == owned, "neutral penalties allocate nothing"
        for x, y in zip(a, b):
            same_state(lib, ext, x, y, p)
        free(ext, a)
        free(ext, b)


# ---- against the host twin ---------------------------------------------------------------------------------------------------------
def _twins(lib, ext, path, n, p, pen=PEN, max_steps=12, cons=None):
    a, b = group(ext, path, n), group(ext, path, n)
    V = ext.L.minigpt4_b200_n_vocab(a[0].ptr)
    hist = histories(n, V=V)
    handles = []
    if cons is not None:
        for g in (a, b):
            h = ext.constraint_create(g[0], *choices_dfa([b"cat", b"car", b"dog", b"no animal", b"yes"]))
            handles.append(h)
            for i in cons:
                ext.constraint_attach(g[i], h)
    ids_a, st_a, _ = ext.sample_until_penalized(a, max_steps, "", hist, **pen, **p)
    ids_b = twin_loop(ext, b, [len(x) for x in ids_a], hist, p, pen)
    assert ids_a == ids_b
    for i, (x, y) in enumerate(zip(a, b)):
        q = p if cons is None or i not in cons else dict(p, mirostat=0)
        same_state(lib, ext, x, y, q)
    for g in (a, b):
        free(ext, g)
    for h in handles:
        ext.constraint_free(h)
    return ids_a, st_a


@pytest.mark.parametrize("wtype", ["q4_0", "q4_1", "q4_0-no-gemm", "q4_1-no-gemm", "q5_k", "q6_k", "f16", "mixed"])
def test_host_twin_weight_types(lib, ext, files, wtype, monkeypatch):
    if wtype.endswith("-no-gemm"):
        monkeypatch.setenv("MINIGPT4_B200_NO_PREFILL_GEMM", "1")
    _twins(lib, ext, files[wtype.split("-")[0]], 3, WEBUI, pen=dict(repeat_last_n=64, repeat_penalty=1.1, alpha_presence=0.0, alpha_frequency=0.0,
                                                                     penalize_nl=True))


@pytest.mark.parametrize("n", [1, 3, 9, 64])
@pytest.mark.parametrize("params", list(PARAMS))
def test_host_twin_batches(lib, ext, files, n, params):
    _twins(lib, ext, files["q4_1"], n, PARAMS[params])


@pytest.mark.parametrize("params", ["greedy", "webui"])
def test_host_twin_constrained_mix(lib, ext, files, params):
    ids, stopped = _twins(lib, ext, files["q4_1"], 9, PARAMS[params], cons=[0, 2, 3, 7])
    for i in (0, 2, 3, 7):
        assert stopped[i] and ids[i][-1] == 2, "a constrained reply ends after </s>"


# ---- greedy against numpy ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 9])
def test_greedy_against_numpy(ext, files, n):
    steps = 16
    pen = dict(repeat_last_n=32, repeat_penalty=3.0, alpha_presence=2.0, alpha_frequency=1.0, penalize_nl=False)
    g = group(ext, files["q4_1"], n)
    plain, _, _ = ext.sample_until(g, steps, "", temp=0.0)
    free(ext, g)
    # (the unpenalised reply in the history, so that the penalties change it from its first step)
    hist = [h + x for h, x in zip(histories(n), plain)]
    a, b = group(ext, files["q4_1"], n), group(ext, files["q4_1"], n)
    ids, _, _ = ext.sample_until_penalized(a, steps, "", hist, **pen, temp=0.0)
    assert any(x != y for x, y in zip(ids, plain)), "the penalties change a greedy reply"
    for i, c in enumerate(b):
        fed = []
        for _ in range(steps):
            z = np_penalize(ext.logits(c), hist[i] + fed, pen["repeat_last_n"], pen["repeat_penalty"], pen["alpha_presence"],
                            pen["alpha_frequency"], pen["penalize_nl"])
            t = int(np.argmax(z))   # the first arg-max
            fed.append(t)
            ext.eval_tokens(c, [t])
        assert ids[i] == fed, f"context {i}"
        assert np.array_equal(bits(ext.logits(a[i])), bits(ext.logits(c)))
    free(ext, a)
    free(ext, b)


# ---- chunking and stops --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("params", ["greedy", "webui", "mirostat-2"])
def test_chunked_reply_equals_one_call(lib, ext, files, params):
    p, n = PARAMS[params], 3
    hist = histories(n)
    one, many = group(ext, files["q4_1"], n), group(ext, files["q4_1"], n)
    ids1, _, _ = ext.sample_until_penalized(one, 23, "", hist, **PEN, **p)
    got = [[] for _ in range(n)]
    while len(got[0]) < 23:
        ids, _, _ = ext.sample_until_penalized(many, min(5, 23 - len(got[0])), "", [h + g for h, g in zip(hist, got)], **PEN, **p)
        for g, x in zip(got, ids):
            g += x
    assert got == ids1
    for x, y in zip(one, many):
        same_state(lib, ext, x, y, p)
    free(ext, one)
    free(ext, many)


def _texts(ext, c, ids):
    return [ext.L.minigpt4_b200_token_text(c.ptr, int(t)) for t in ids]


def test_stops_at_different_steps(lib, ext, files):
    n, max_steps = 8, 24
    hist = histories(n)
    probe = group(ext, files["hash"], n)
    ids, _, _ = ext.sample_until_penalized(probe, max_steps, "", hist, **PEN, **WEBUI)
    texts = [_texts(ext, probe[0], x) for x in ids]
    free(ext, probe)
    best = None
    for ch in sorted({bytes([b]) for tx in texts for t in tx for b in t}):
        firsts = [ref_stop(tx, ch) for tx in texts]
        if min(firsts) < 0:
            continue
        score = (len(set(firsts)), -max(firsts))
        if best is None or score > best[0]:
            best = (score, ch, firsts)
    assert best is not None and best[0][0] >= 3, "no stop text spreads the stops"
    _, stop, firsts = best
    a, b = group(ext, files["hash"], n), group(ext, files["hash"], n)
    got, stopped, _ = ext.sample_until_penalized(a, max_steps, stop, hist, **PEN, **WEBUI)
    assert [len(x) for x in got] == [f + 1 for f in firsts] and all(stopped)
    assert got == [x[:f + 1] for x, f in zip(ids, firsts)]
    # a context that stopped early holds what its own steps left, not the steps the others still ran
    assert twin_loop(ext, b, [len(x) for x in got], hist, WEBUI, PEN) == got
    for x, y in zip(a, b):
        same_state(lib, ext, x, y, WEBUI)
    free(ext, a)
    free(ext, b)


def test_stop_text_across_two_calls(ext, files):
    for seed in range(40):
        probe = group(ext, files["hash"], 1, seed0=100 + seed)
        ids, _, _ = ext.sample_until_penalized(probe, 30, "", None, **PEN, **WEBUI)
        tx = _texts(ext, probe[0], ids[0])
        free(ext, probe)
        hit = next((k for k in range(2, 29, 3) if tx[k] and tx[k + 1] and tx[k + 1] != b"##"
                    and ref_stop(tx, tx[k][-1:] + tx[k + 1][:1]) == k + 1), None)
        if hit is not None:
            break
    assert hit is not None, "no stop text across a call boundary in 40 seeds"
    stop = tx[hit][-1:] + tx[hit + 1][:1]
    one = group(ext, files["hash"], 1, seed0=100 + seed)
    ids1, st1, _ = ext.sample_until_penalized(one, 30, stop, None, **PEN, **WEBUI)
    many = group(ext, files["hash"], 1, seed0=100 + seed)
    ids2, st2 = [], False
    while len(ids2) < 30 and not st2:
        got, st, _ = ext.sample_until_penalized(many, 3, stop, [ids2], **PEN, **WEBUI)
        ids2 += got[0]
        st2 = st[0]
    assert ids2 == ids1[0] and st2 == st1[0] and len(ids2) == hit + 2
    assert np.array_equal(bits(ext.logits(one[0])), bits(ext.logits(many[0])))
    free(ext, one)
    free(ext, many)


def test_max_steps_and_the_last_slot_of_n_ctx(lib, ext, files):
    a, b = group(ext, files["hash"], 2, n_ctx=64), group(ext, files["hash"], 2, n_ctx=64)
    hist = histories(2)
    room = [64 - ext.n_past(c) for c in a]
    ids, stopped, _ = ext.sample_until_penalized(a, min(room), "", hist, **PEN, **WEBUI)
    assert [len(x) for x in ids] == [min(room)] * 2 and stopped == [False, False]
    assert twin_loop(ext, b, [min(room)] * 2, hist, WEBUI, PEN) == ids
    full = a[int(np.argmin(room))]
    assert ext.n_past(full) == 64
    buf = [np.zeros(1, np.int32) for _ in range(3)]
    assert ext.L.minigpt4_b200_sample_until_penalized(ctypes.cast(ext._ctx_array([full]), ctypes.c_void_p), 1, 1, b"", 0.8, 40, 0.9, 1.0, 1.0, 0, 5.0,
                                                      1.0, 16, 1.5, 0.5, 0.25, 0, None, None, _ptr(buf[0]), _ptr(buf[1]), _ptr(buf[2]), None) == REFUSED
    for x, y in zip(a, b):
        assert np.array_equal(bits(ext.logits(x)), bits(ext.logits(y)))
    free(ext, a)
    free(ext, b)


# ---- 7B width ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 16])
def test_7b_width(lib, ext, files, n):
    a, b = group(ext, files["w7b"], n, n_ctx=64), group(ext, files["w7b"], n, n_ctx=64)
    if n == 1:
        assert ext.stats(a[0]).decode_megakernel >= 6
    hist = histories(n, V=32000)
    pen = dict(repeat_last_n=64, repeat_penalty=1.1, alpha_presence=0.0, alpha_frequency=0.0, penalize_nl=True)
    for p in (WEBUI, PARAMS["greedy"]):
        ids, _, _ = ext.sample_until_penalized(a, 8, "", hist, **pen, **p)
        assert twin_loop(ext, b, [8] * n, hist, p, pen) == ids
        hist = [h + x for h, x in zip(hist, ids)]
    for x, y in zip(a, b):
        same_state(lib, ext, x, y, WEBUI)
    free(ext, a)
    free(ext, b)


# ---- refusals and memory -------------------------------------------------------------------------------------------------------------
def _raw(ext, ctxs, hist, n_last, mirostat=0, repeat_penalty=1.5):
    n, max_steps = len(ctxs), 4
    ids, n_out, stopped = np.zeros(max_steps * n, np.int32), np.zeros(n, np.int32), np.zeros(n, np.int32)
    return ext.L.minigpt4_b200_sample_until_penalized(ctypes.cast(ext._ctx_array(ctxs), ctypes.c_void_p), n, max_steps, None, 0.8, 40, 0.9, 1.0, 1.0,
                                                      mirostat, 5.0, 1.0, 16, repeat_penalty, 0.5, 0.25, 0, _ptr(hist), _ptr(n_last), _ptr(ids),
                                                      _ptr(n_out), _ptr(stopped), None)


@pytest.mark.parametrize("case", ["n_last-negative", "null-last_ids", "id-negative", "id-n_vocab", "penalty-0", "mirostat-constrained"])
def test_refusals_change_nothing(ext, files, case):
    c = ext.llm_load(files["q4_1"], n_ctx=128)
    twin = ext.llm_load(files["q4_1"], n_ctx=128)
    c1 = ext.session_create(c, 5)
    for x in (c, c1, twin):
        ext.eval_tokens(x, [1, 15, 27, 300])
        ext.flush(x)
        ext.eval_tokens(x, [41, 9, 77])   # queued
    hist, n_last = np.array([5, 6, 7, 8, 9], np.int32), np.array([2, 3], np.int32)
    h = None
    if case == "n_last-negative":
        n_last[1] = -1
    elif case == "id-negative":
        hist[4] = -1
    elif case == "id-n_vocab":
        hist[4] = 1024
    elif case == "mirostat-constrained":
        h = ext.constraint_create(c, *choices_dfa([b"cat", b"dog"]))
        ext.constraint_attach(c1, h)
    launches = [ext.stats(x).kernel_launches for x in (c, c1)]
    owned = [ext.session_info(x)[1] for x in (c, c1)]
    code = _raw(ext, [c, c1], None if case == "null-last_ids" else hist, n_last, mirostat=1 if case == "mirostat-constrained" else 0,
                repeat_penalty=0.0 if case == "penalty-0" else 1.5)
    assert code == REFUSED
    assert [ext.stats(x).kernel_launches for x in (c, c1)] == launches, "device work before the refusal"
    assert [ext.session_info(x)[1] for x in (c, c1)] == owned
    assert ext.n_past(c) == ext.n_past(twin)
    assert np.array_equal(ext.logits(c), ext.logits(twin))   # the queue was still there, and evaluates as the twin's does
    if h is not None:
        ext.constraint_attach(c1, None)
        ext.constraint_free(h)
    for x in (c1, c, twin):
        ext.base.minigpt4_free(x)


def test_penalty_memory(ext, files):
    n_ctx, V = 128, 1024
    c = group(ext, files["q4_1"], 1, n_ctx=n_ctx)[0]
    ext.sample_until([c], 2, "", **WEBUI)                     # the sampler and stop state
    o0 = ext.session_info(c)[1]
    ext.sample_until_penalized([c], 2, "", [[5, 6]], repeat_penalty=1.0)   # neutral: nothing allocated
    assert ext.session_info(c)[1] == o0
    ext.sample_until_penalized([c], 2, "", [[5, 6]], **PEN)
    o1 = ext.session_info(c)[1]
    assert o1 - o0 == 8 * V + 4 * n_ctx
    ext.sample_until_penalized([c], 2, "", None, **PEN)
    ext.sample_until([c], 2, "", **WEBUI)
    assert ext.session_info(c)[1] == o1
    # a window reaching further back than n_ctx history ids grows the history buffer to them
    ext.sample_until_penalized([c], 2, "", [list(range(3, 203))], **dict(PEN, repeat_last_n=200))
    assert ext.session_info(c)[1] - o1 == 4 * (200 - n_ctx)
    ext.base.minigpt4_free(c)


# ---- chat bot ------------------------------------------------------------------------------------------------------------------------
def test_chat_bot(mg, ext, files):
    import minigpt4_cpp_b200 as m
    bots = [m.MiniGPT4ChatBot(files["vision"], files["hash"]) for _ in range(4)]
    for bot in bots:
        bot.upload_image(mg.synth_image(3).reshape(1, 3, 224, 224))
    # defaults: exactly the sample_until chunks generate_on_device issued before it took penalties
    got = list(bots[0].generate_on_device("what is this?", limit=60, chunk=5))
    b = bots[1]
    b.is_image_chat = False
    b.library.minigpt4_begin_chat_image(b.ctx, b.embedding, "what is this?", b.n_threads)
    want, done = [], 0
    while done < 60:
        ids, stopped, _ = ext.sample_until([b.ctx], min(5, 60 - done), None, **WEBUI)
        done += len(ids[0])
        texts = [ext.L.minigpt4_b200_token_text(b.ctx.ptr, int(t)).decode("utf-8", errors="ignore") for t in ids[0]]
        keep = [t for k, t in enumerate(texts) if not (stopped[0] and k == len(texts) - 1) and not b.library.minigpt4_contains_eos_token(t)]
        want += keep
        if stopped[0]:
            break
    assert got == want and got
    assert ext.stats(bots[0].ctx).kernel_launches == ext.stats(b.ctx).kernel_launches
    # repeat_penalty 1.1: what a loop of end_chat_penalized over the reply's ids yields, with generate()'s stop rule
    got = list(bots[2].generate_on_device("what is this?", limit=60, chunk=5, repeat_penalty=1.1))
    b = bots[3]
    b.is_image_chat = False
    b.library.minigpt4_begin_chat_image(b.ctx, b.embedding, "what is this?", b.n_threads)
    want, reply, chat = [], [], ""
    for _ in range(60):
        token, t = ext.end_chat_penalized(b.ctx, reply, repeat_last_n=64, repeat_penalty=1.1, **WEBUI)
        reply.append(t)
        chat += token
        if b.library.minigpt4_contains_eos_token(token):
            continue
        if b.library.minigpt4_is_eos(chat):
            break
        want.append(token)
    assert got == want and got
    for bot in bots:
        bot.free()
