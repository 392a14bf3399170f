"""Constrained replies on the GPU (minigpt4_b200_constraint_*; llama_sample.cuh's constrained kernels, DESIGN.md §4.12).

- the device handle's tables equal the host compiler's;
- greedy and sampled steps over allowed(s) only, against a Python loop and the host Sampler (end_chat / end_chat_batch) on twins;
- sample_steps / sample_until at B = 1, 2, 8, 9, 64, constrained and mixed with unconstrained contexts;
- the state's lifetime (turns, session_copy, state_load, detach, a freed handle) and the refused calls."""
import ctypes

import numpy as np
import pytest

from minigpt4_cpp_b200.minigpt4_library import choices_dfa

pytestmark = pytest.mark.gpu

WEBUI = dict(temp=0.8, top_k=40, top_p=0.9)
PARAMS = {"webui": WEBUI, "top_k-0-top_p-0.95": dict(temp=0.8, top_k=0, top_p=0.95), "tfs_z-0.95": dict(temp=0.8, top_k=40, top_p=1.0, tfs_z=0.95),
          "typical_p-0.9": dict(temp=0.8, top_k=40, top_p=1.0, typical_p=0.9)}
CHOICES = [b"cat", b"car", b"cart", b"dog", b"no animal", b"yes", b"no"]


def _word(alphabet: bytes, max_len: int):
    """alphabet{1,max_len}: state k = k bytes so far"""
    nx, ac = np.full((max_len + 1, 256), -1, np.int32), np.zeros(max_len + 1, np.uint8)
    for s in range(max_len):
        nx[s, list(alphabet)] = s + 1
    ac[1:] = 1
    return nx, ac


LOWER = b"abcdefghijklmnopqrstuvwxyz "


@pytest.fixture(scope="module")
def files(tiny, mg, tmp_path_factory):
    d = tmp_path_factory.mktemp("constraint")
    out = dict(tiny)
    out["v32000"] = str(d / "llama-32000.bin")
    mg.write_llama_ggjt(out["v32000"], mg.LlamaSpec(n_vocab=32000, n_embd=512, n_head=4, n_layer=2, wtype="q4_1"))
    out["w4096"] = str(d / "llama-4096.bin")
    mg.write_llama_ggjt(out["w4096"], mg.LlamaSpec(n_vocab=2048, n_embd=4096, n_head=32, n_layer=2, wtype="q4_1"))
    return out


def _sessions(ext, path, seeds, n_ctx=128, prompt_seed=17):
    p = ext.llm_load(path, n_ctx=n_ctx, seed=seeds[0])
    ses = [p] + [ext.session_create(p, s) for s in seeds[1:]]
    rng = np.random.default_rng(prompt_seed)
    for i, c in enumerate(ses):
        ext.eval_tokens(c, rng.integers(3, 1000, size=3 + (i % 5)).tolist())
        ext.flush(c)
    return ses


def _free(ext, ctxs):
    for c in ctxs[1:] + ctxs[:1]:
        ext.base.minigpt4_free(c)


def _allowed(ext, h, state):
    return ext.constraint_allowed(h, state)


def _replay(ext, h, ids):
    """the states a run of ids passes through, asserting each id is allowed where it is fed; -1 = finished"""
    s = 0
    for t in ids:
        if s == -1:
            assert t == 2
            continue
        al, nx = _allowed(ext, h, s)
        j = np.searchsorted(al, t)
        assert j < len(al) and al[j] == t, f"id {t} not allowed in state {s}"
        s = int(nx[j])
    return s


def _rng_probe(lib, ext, c):
    """the generator's next draw, unconstrained (detaches c)"""
    ext.constraint_attach(c, None)
    return lib.minigpt4_end_chat(c, **WEBUI)


# ---- compiler on the device ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("which", ["q4_1", "v32000"])
def test_device_tables_equal_host_seam(ext, files, which):
    c = ext.llm_load(files[which], n_ctx=64)
    for nx, ac in (choices_dfa(CHOICES), _word(b"0123456789", 6), _word(LOWER, 3)):
        h = ext.constraint_create(c, nx, ac)
        for s in range(len(ac)):
            dev, host = ext.constraint_allowed(h, s), ext.host_constraint_allowed(files[which], nx, ac, s)
            assert (dev is None) == (host is None), s
            if dev is not None:
                assert np.array_equal(dev[0], host[0]) and np.array_equal(dev[1], host[1]), s
        ext.constraint_free(h)
    ext.base.minigpt4_free(c)


# ---- greedy -----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mega", [True, False], ids=["megakernel", "per-op"])
def test_greedy_equals_python_loop(ext, files, mega, monkeypatch):
    if not mega:
        monkeypatch.setenv("MINIGPT4_B200_NO_MEGAKERNEL", "1")
    a, b = _sessions(ext, files["w4096"], [1, 2])
    ext.session_copy(a, [b])
    assert (ext.stats(a).decode_megakernel >= 6) == mega
    nx, ac = _word(LOWER, 20)
    h = ext.constraint_create(a, nx, ac)
    ext.constraint_attach(a, h)
    ids, _ = ext.sample_steps([a], 24, temp=0.0)
    s, want = 0, []
    for _ in range(24):
        lg = ext.logits(b)
        al, nxt = _allowed(ext, h, s) if s >= 0 else (np.array([2]), np.array([-1]))
        j = int(np.argmax(lg[al]))   # the first maximum: the lower id on ties
        want.append(int(al[j])); s = int(nxt[j])
        ext.eval_tokens(b, [want[-1]]); ext.flush(b)
    assert ids[:, 0].tolist() == want
    assert ext.n_past(a) == ext.n_past(b) and np.array_equal(ext.logits(a), ext.logits(b))
    assert ext.constraint_state(a) == (s, s == -1)
    ext.constraint_free(h)
    _free(ext, [a, b])


def test_greedy_batch_equals_one_context(ext, files):
    ses = _sessions(ext, files["q4_1"], [1, 2, 3, 4])
    one = _sessions(ext, files["q4_1"], [1, 2, 3, 4])
    h = ext.constraint_create(ses[0], *_word(LOWER, 30))
    for c in ses:
        ext.constraint_attach(c, h)
    ids, _ = ext.sample_steps(ses, 16, temp=0.0)
    h1 = ext.constraint_create(one[0], *_word(LOWER, 30))
    for i, c in enumerate(one):
        ext.constraint_attach(c, h1)
        got, _ = ext.sample_steps([c], 16, temp=0.0)
        assert got[:, 0].tolist() == ids[:, i].tolist(), i
        assert np.array_equal(ext.logits(c), ext.logits(ses[i]))
    for hh in (h, h1):
        ext.constraint_free(hh)
    _free(ext, ses); _free(ext, one)


# ---- the host Sampler over allowed(s) ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("params", list(PARAMS))
@pytest.mark.parametrize("automaton", ["choices", "lower"], ids=["few-allowed", "many-allowed"])
def test_first_end_chat_is_host_sample_over_allowed(lib, ext, files, params, automaton):
    kw = PARAMS[params]
    c = ext.llm_load(files["v32000"], n_ctx=64, seed=4242)
    ext.eval_tokens(c, [1, 500, 600, 700])
    nx, ac = choices_dfa(CHOICES) if automaton == "choices" else _word(LOWER, 8)
    h = ext.constraint_create(c, nx, ac)
    al, _ = _allowed(ext, h, 0)
    assert (len(al) < 40) == (automaton == "choices")
    ext.constraint_attach(c, h)
    lg = ext.logits(c)
    j = int(ext.host_sample(lg[al], 4242, 1, **kw)[0])
    assert lib.minigpt4_end_chat(c, **kw) == ext.L.minigpt4_b200_token_text(c.ptr, int(al[j])).decode("utf-8", errors="ignore")
    ext.constraint_free(h)
    ext.base.minigpt4_free(c)


# ---- device against host ---------------------------------------------------------------------------------------------------------
def _text(ext, c, ids):
    return [ext.L.minigpt4_b200_token_text(c.ptr, int(i)).decode("utf-8", errors="ignore") for i in ids]


@pytest.mark.parametrize("n", [1, 2, 8, 9, 64])
@pytest.mark.parametrize("mixed", [False, True], ids=["all-constrained", "mixed"])
def test_sample_steps_equals_end_chat(lib, ext, files, n, mixed):
    seeds = [100 + 7 * i for i in range(n)]
    a, b, u = (_sessions(ext, files["q4_1"], seeds) for _ in range(3))
    nx, ac = _word(LOWER, 40)
    ha, hb = ext.constraint_create(a[0], nx, ac), ext.constraint_create(b[0], nx, ac)
    on = [not (mixed and i % 2 == 1) for i in range(n)]
    for i in range(n):
        if on[i]:
            ext.constraint_attach(a[i], ha); ext.constraint_attach(b[i], hb)
    steps = 12
    ids, _ = ext.sample_steps(a, steps, **WEBUI)
    if n == 1:
        want = [[lib.minigpt4_end_chat(b[0], **WEBUI)] for _ in range(steps)]
    else:
        want = [ext.end_chat_batch(b, **WEBUI) for _ in range(steps)]
    for i in range(n):
        assert _text(ext, a[i], ids[:, i]) == [w[i] for w in want], f"context {i}"
        assert ext.n_past(a[i]) == ext.n_past(b[i]) and np.array_equal(ext.logits(a[i]), ext.logits(b[i])), f"context {i}"
        if on[i]:
            assert ext.constraint_state(a[i]) == ext.constraint_state(b[i]) and ext.constraint_state(a[i])[0] == _replay(ext, ha, ids[:, i])
    if mixed:   # the unconstrained contexts draw what the same call draws with no constraint attached anywhere
        got, _ = ext.sample_steps(u, steps, **WEBUI)
        for i in range(n):
            if not on[i]:
                assert ids[:, i].tolist() == got[:, i].tolist(), f"context {i}"
    assert [_rng_probe(lib, ext, c) for c in a] == [_rng_probe(lib, ext, c) for c in b]   # the generators continue alike
    for h in (ha, hb):
        ext.constraint_free(h)
    for s in (a, b, u):
        _free(ext, s)


@pytest.mark.parametrize("n", [1, 2, 9])
@pytest.mark.parametrize("params", ["webui", "top_k-0-top_p-0.95"])
def test_sample_until_equals_end_chat_loop(lib, ext, files, n, params):
    """choices replies: each stops after </s>; the host loop is end_chat until it returns </s>"""
    kw = PARAMS[params]
    seeds = [300 + 11 * i for i in range(n)]
    a, b = _sessions(ext, files["q4_1"], seeds), _sessions(ext, files["q4_1"], seeds)
    nx, ac = choices_dfa(CHOICES)
    ha, hb = ext.constraint_create(a[0], nx, ac), ext.constraint_create(b[0], nx, ac)
    for x, y in zip(a, b):
        ext.constraint_attach(x, ha); ext.constraint_attach(y, hb)
    ids, stopped, _ = ext.sample_until(a, 24, "", **kw)
    for i in range(n):
        want = []
        while not want or want[-1] != "</s>":
            want.append(lib.minigpt4_end_chat(b[i], **kw))
        assert _text(ext, a[i], ids[i]) == want, f"context {i}"
        assert stopped[i] and ids[i][-1] == 2
        assert b"".join(ext.L.minigpt4_b200_token_text(a[i].ptr, t) for t in ids[i][:-1]) in CHOICES
        assert ext.n_past(a[i]) == ext.n_past(b[i]) and np.array_equal(ext.logits(a[i]), ext.logits(b[i]))
        assert ext.constraint_state(a[i]) == (-1, True) == ext.constraint_state(b[i])
    assert [_rng_probe(lib, ext, c) for c in a] == [_rng_probe(lib, ext, c) for c in b]
    for h in (ha, hb):
        ext.constraint_free(h)
    _free(ext, a); _free(ext, b)


def test_sample_until_in_chunks_equals_one_call(ext, files):
    seeds = [5, 6, 7]
    a, b = _sessions(ext, files["q4_1"], seeds), _sessions(ext, files["q4_1"], seeds)
    ha, hb = ext.constraint_create(a[0], *_word(LOWER, 60)), ext.constraint_create(b[0], *_word(LOWER, 60))
    for x, y in zip(a, b):
        ext.constraint_attach(x, ha); ext.constraint_attach(y, hb)
    one, st1, _ = ext.sample_until(a, 48, "e ", **WEBUI)
    parts, live = [[] for _ in b], list(range(3))
    for _ in range(3):
        ids, st, _ = ext.sample_until([b[i] for i in live], 16, "e ", **WEBUI)
        for k, i in enumerate(live):
            parts[i] += ids[k]
        live = [i for k, i in enumerate(live) if not st[k]]
        if not live:
            break
    assert parts == one
    for x, y in zip(a, b):
        assert ext.constraint_state(x) == ext.constraint_state(y) and np.array_equal(ext.logits(x), ext.logits(y))
    for h in (ha, hb):
        ext.constraint_free(h)
    _free(ext, a); _free(ext, b)


def test_choices_reply_is_one_of_the_choices(ext, files):
    ses = _sessions(ext, files["v32000"], [11 * i + 1 for i in range(8)])
    h = ext.constraint_create(ses[0], *choices_dfa(CHOICES))
    for c in ses:
        ext.constraint_attach(c, h)
    ids, stopped, _ = ext.sample_until(ses, 32, None, temp=1.5, top_k=0, top_p=1.0)
    for i, c in enumerate(ses):
        assert stopped[i] and ids[i][-1] == 2
        _replay(ext, h, ids[i])
        assert b"".join(ext.L.minigpt4_b200_token_text(c.ptr, t) for t in ids[i][:-1]) in CHOICES
    ext.constraint_free(h)
    _free(ext, ses)


# ---- lifetime ---------------------------------------------------------------------------------------------------------------------
def test_lifetime(lib, ext, files):
    a, b, c = _sessions(ext, files["q4_1"], [1, 2, 3])
    _, _, shared0 = ext.session_info(a)
    nx, ac = _word(LOWER, 200)
    h, h2 = ext.constraint_create(a, nx, ac), ext.constraint_create(a, *choices_dfa(CHOICES))
    _, _, shared1 = ext.session_info(a)
    assert shared1 > shared0
    ext.constraint_attach(a, h); ext.constraint_attach(b, h); ext.constraint_attach(c, h2)
    ext.sample_steps([a], 3, **WEBUI)
    s = ext.constraint_state(a)
    assert s[0] >= 3 and not s[1]
    # session_copy: the same constraint takes the source's state, another restarts
    ext.session_copy(a, [b, c])
    assert ext.constraint_state(b) == s and ext.constraint_state(c) == (0, False)
    # a new turn restarts it
    ext.eval_tokens(a, [5, 6])
    assert ext.constraint_state(a) == (0, False)
    ext.sample_steps([a], 2, **WEBUI)
    lib.minigpt4_begin_chat(a, "hi")
    assert ext.constraint_state(a) == (0, False)
    # state_load restarts it
    blob = ext.state_save(b)
    ext.state_load(b, blob)
    assert ext.constraint_state(b) == (0, False)
    # a freed handle keeps its attached contexts working
    ext.constraint_free(h)
    ids, _ = ext.sample_steps([a, b], 4, **WEBUI)
    for i, x in enumerate((a, b)):
        assert all(t != 2 and all(ch in LOWER for ch in ext.L.minigpt4_b200_token_text(x.ptr, int(t))) for t in ids[:, i])
    # detach restores unconstrained results; the last detach frees the tables
    ref, = _sessions(ext, files["q4_1"], [9])
    twin, = _sessions(ext, files["q4_1"], [9])
    h3 = ext.constraint_create(twin, *choices_dfa(CHOICES))
    ext.constraint_attach(twin, h3)
    ext.constraint_attach(twin, None)
    with pytest.raises(RuntimeError):
        ext.constraint_state(twin)
    assert ext.sample_steps([twin], 6, **WEBUI)[0].tolist() == ext.sample_steps([ref], 6, **WEBUI)[0].tolist()
    ext.constraint_free(h3)
    # the tables leave the shared bytes with their last reference
    shared2 = ext.session_info(a)[2]
    for x in (a, b):
        ext.constraint_attach(x, None)
    assert ext.session_info(a)[2] < shared2
    ext.constraint_attach(c, None)
    ext.constraint_free(h2)
    assert ext.session_info(a)[2] == shared2 - (shared1 - shared0)
    _free(ext, [a, b, c]); ext.base.minigpt4_free(ref); ext.base.minigpt4_free(twin)


# ---- refusals ---------------------------------------------------------------------------------------------------------------------
def test_refused_calls_change_nothing(lib, ext, files):
    a, b = _sessions(ext, files["q4_1"], [21, 22])
    twin_a, twin_b = _sessions(ext, files["q4_1"], [21, 22])
    h, ht = ext.constraint_create(a, *_word(LOWER, 200)), ext.constraint_create(twin_a, *_word(LOWER, 200))
    ext.constraint_attach(a, h); ext.constraint_attach(twin_a, ht)
    ext.sample_steps([a], 2, **WEBUI); ext.sample_steps([twin_a], 2, **WEBUI)   # (a mid-reply state)
    before = (ext.n_past(a), ext.logits(a), ext.constraint_state(a))
    ctxs = ctypes.cast(ext._ctx_array([a, b]), ctypes.c_void_p)
    ids = (ctypes.c_int32 * 64)()
    ms = ctypes.c_float(0)
    L = ext.L
    assert L.minigpt4_b200_decode_chain(a.ptr, 2, ids, ctypes.byref(ms)) == 8
    assert L.minigpt4_b200_decode_batch(ctxs, 2, ids, ids) == 8
    assert L.minigpt4_b200_sample_steps_mirostat(ctxs, 2, 2, 0.8, 2, 5.0, 0.1, ids, None) == 8
    assert L.minigpt4_b200_sample_until_mirostat(ctxs, 2, 2, None, 0.8, 1, 5.0, 0.1, ids, ids, ids, None) == 8
    tok = ctypes.c_char_p()
    for mode in (1, 2):
        assert lib.library.minigpt4_end_chat(a.ptr, ctypes.byref(tok), 0, 0.8, 40, 0.9, 1.0, 1.0, 64, 1.1, 1.0, 1.0, mode, 5.0, 0.1, 1) == 8
        toks = (ctypes.c_char_p * 2)()
        assert L.minigpt4_b200_end_chat_batch(ctxs, 2, toks, 0.8, 40, 0.9, 1.0, 1.0, 64, 1.1, 1.0, 1.0, mode, 5.0, 0.1, 1) == 8
    assert ext.n_past(a) == before[0] and np.array_equal(ext.logits(a), before[1]) and ext.constraint_state(a) == before[2]
    assert before[2] == ext.constraint_state(twin_a) and np.array_equal(before[1], ext.logits(twin_a))
    assert ext.n_past(b) == ext.n_past(twin_b) and np.array_equal(ext.logits(b), ext.logits(twin_b))
    assert [_rng_probe(lib, ext, c) for c in (a, b)] == [_rng_probe(lib, ext, c) for c in (twin_a, twin_b)]
    # another group
    other = ext.llm_load(files["q4_1"], n_ctx=32)
    assert L.minigpt4_b200_constraint_attach(other.ptr, h) == 8
    ext.constraint_free(h); ext.constraint_free(ht)
    _free(ext, [a, b]); _free(ext, [twin_a, twin_b]); ext.base.minigpt4_free(other)
