"""Mirostat on the device sampler (minigpt4_b200_sample_steps_mirostat / sample_until_mirostat; llama_sample.cuh): the ids and the μ of the
host Sampler for the same generator.

- glibc's log2f / powf restated on the device, bit for bit, NaNs included;
- the mirostat kernel against the host Sampler through op_sample_mirostat, draw for draw and μ for μ, over a parameter sweep and crafted
  logits (all equal, a spike that leaves one candidate, k above n_vocab or past the int range, two candidates);
- one context, batches and whole replies against minigpt4_end_chat / end_chat_batch twins: ids, n_past, logits, then μ and the generator
  continuing on the host;
- greedy, refused calls, and MiniGPT4ChatBot.generate_on_device against generate()."""
import ctypes
import itertools
import struct

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

UNUSED = (64, 1.1, 1.0, 1.0)   # repeat_last_n .. alpha_frequency of end_chat (never applied)
M1 = dict(temp=0.8, mirostat=1, mirostat_tau=5.0, mirostat_eta=0.1)
M2 = dict(temp=0.8, mirostat=2, mirostat_tau=5.0, mirostat_eta=1.0)


def bits(x: float) -> int:
    return struct.unpack("<I", struct.pack("<f", x))[0]


# ---- libm -----------------------------------------------------------------------------------------------------------------------------
def test_log2f_bit_exact(ext):
    """every positive float (the finite ones, inf and every NaN pattern), -0 and the negative default NaN"""
    assert ext.op_check_log2f(0x00000000, 0x7FFFFFFF) == 0
    assert ext.op_check_log2f(0x80000000, 0x80000000) == 0
    assert ext.op_check_log2f(0xFFC00000, 0xFFC00000) == 0


@pytest.mark.parametrize("x", [2.0, 2048.0, 32000.0, 32001.0])
def test_powf_bit_exact_for_every_y(ext, x):
    """powf(2, μ) and powf(n_vocab, -eps) of mirostat v1: every y bit pattern"""
    assert ext.op_check_powf(x, 0x00000000, 0xFFFFFFFF) == 0


def _powf_xs():
    special = [0.0, -0.0, 1e-45, 1e-40, 1.0, -1.0, -2.0, -0.5, -3.5, -1e10, float("inf"), float("-inf"), float("nan"), 0.99999994, 1.0000001,
               2048.0]
    return special + np.logspace(-30, 30, 48).astype(np.float32).tolist()


def test_powf_bit_exact_over_y_in_minus_128_to_128(ext):
    """~64 values of x (0, subnormals, 1, up to 1e30, negatives, inf, NaN), each against y in [-128, 128]: windows of 2^12 consecutive
    bit patterns around every integer of the range, which covers the odd / even / non-integer y that decide the sign for negative x and
    |y log2 x| on both sides of the overflow and underflow limits"""
    for x in _powf_xs():
        bad = 0
        for y in range(-128, 129):
            c = bits(float(y))
            bad += ext.op_check_powf(x, max(0, c - 0x800), min(0xFFFFFFFF, c + 0x7FF))
        assert bad == 0, x


# ---- kernel against host --------------------------------------------------------------------------------------------------------------
def _same(logits, temp, got, want, what):
    """draw for draw the same id and bit for bit the same μ; a different id only where the two candidates' logit / temp are equal as float32
    (the documented tie rule, after temperature: equal probabilities, so μ and the generator stay in step)"""
    gi, gm = got
    wi, wm = want
    scaled = logits.astype(np.float32) / np.float32(temp)
    for d, (g, w) in enumerate(zip(gi.tolist(), wi.tolist())):
        assert g == w or scaled[g] == scaled[w], f"draw {d}: {g} != {w}, {what}"
    assert np.array_equal(gm.view(np.uint32), wm.view(np.uint32)), f"μ {gm} != {wm}, {what}"


def _both(ext, logits, seed, n, **kw):
    return ext.op_sample_mirostat(logits, seed, n, **kw), ext.op_sample_mirostat(logits, seed, n, on_device=False, **kw)


@pytest.mark.parametrize("n_vocab", [2, 2048, 32000])
@pytest.mark.parametrize("sigma", [1.0, 3.0, 10.0, 40.0])
@pytest.mark.parametrize("mode", [1, 2])
def test_kernel_draws_and_mu_equal_host(ext, n_vocab, sigma, mode):
    """64 draws from one generator per case: tau x eta x temp x seed"""
    logits = (np.random.default_rng(int(sigma * 1000) + n_vocab).standard_normal(n_vocab) * sigma).astype(np.float32)
    for tau, eta, temp, seed in itertools.product((3.0, 5.0, 8.0), (0.1, 1.0), (0.1, 0.8, 1.5), (1, 77, 4242)):
        kw = dict(temp=temp, mirostat=mode, mirostat_tau=tau, mirostat_eta=eta)
        got, want = _both(ext, logits, seed, 64, **kw)
        _same(logits, temp, got, want, kw | dict(seed=seed))


def _zipf(n, s):
    return (-s * np.log(np.arange(1, n + 1))).astype(np.float32)


@pytest.mark.parametrize("name,logits,tau", [
    ("all-equal", np.full(32000, 0.25, np.float32), 5.0),
    ("spike", np.where(np.arange(32000) == 1234, 1000.0, -1000.0).astype(np.float32), 5.0),   # p 0 / 0 in v1's fit: kf NaN, one candidate
    ("k-above-n_vocab", _zipf(2048, 1.1), 10.0),                                               # kf ~ 6e4 > 2048: every candidate
    ("k-past-int", _zipf(2048, 1.01), 20.0),                                                   # kf ~ 1e11: cvttss2si gives INT_MIN, one candidate
    ("two", np.array([0.5, -0.25], np.float32), 5.0),
    ("two-equal", np.array([1.0, 1.0], np.float32), 5.0)],
    ids=lambda v: v if isinstance(v, str) else None)
@pytest.mark.parametrize("mode", [1, 2])
def test_crafted_logits(ext, name, logits, tau, mode):
    for eta, temp, seed in itertools.product((0.1, 1.0), (0.8, 1.0), (3, 11)):
        kw = dict(temp=temp, mirostat=mode, mirostat_tau=tau, mirostat_eta=eta)
        got, want = _both(ext, logits, seed, 32, **kw)
        _same(logits, temp, got, want, kw | dict(case=name, seed=seed))
    if name == "spike":
        assert got[0].tolist() == [1234] * 32


# ---- end to end -----------------------------------------------------------------------------------------------------------------------
def hash_vocab(mg, n_vocab, seed=5):
    """make_vocab with the byte tokens 0x80..0xff and the last third of the pieces replaced by distinct '#'-bearing ASCII pieces, so that
    sampled replies reach "###" within a few dozen tokens"""
    v = mg.make_vocab(n_vocab)
    seen = {p for p, _ in v}
    rng = np.random.default_rng(seed)
    slots = list(range(3 + 0x80, 259)) + list(range(n_vocab - n_vocab // 3, n_vocab))
    fresh = []
    while len(fresh) < len(slots):
        p = bytes(rng.choice(list(b"#ab #"), size=int(rng.integers(1, 7))).tolist())
        if p not in seen:
            seen.add(p)
            fresh.append(p)
    for i, p in zip(slots, fresh):
        v[i] = (p, v[i][1] if i >= 259 else -2.0)
    return v


@pytest.fixture(scope="module")
def files(tiny, mg, tmp_path_factory):
    d = tmp_path_factory.mktemp("mirostat")
    wide = dict(n_embd=4096, n_head=32, n_layer=2)
    out = {}
    for name, kw in (("q4_1", dict(wide, n_vocab=2048, wtype="q4_1")), ("q5_k", dict(wide, n_vocab=2048, wtype="q5_k", output_type="q6_k")),
                     ("q4_1_32000", dict(wide, n_vocab=32000, wtype="q4_1")),
                     ("hash", dict(wide, n_vocab=2048, wtype="q4_1", vocab=hash_vocab(mg, 2048))),
                     ("hash_tiny", dict(n_embd=512, n_head=4, n_layer=2, n_vocab=1024, wtype="q4_1", vocab=hash_vocab(mg, 1024)))):
        out[name] = str(d / f"llama-{name}.bin")
        mg.write_llama_ggjt(out[name], mg.LlamaSpec(**kw))
    out["vision"] = tiny["vision"]
    return out


def _chat(lib, mg, vision, llm, seed, n_ctx=512):
    import minigpt4_cpp_b200 as m
    c = lib.minigpt4_model_load(vision, llm, 1, seed, n_ctx, 8, 0)
    im = mg.synth_image(3)
    mi = m.MiniGPT4Image(im.ctypes.data_as(ctypes.c_void_p), 224, 224, 3, m.ImageFormat.F32)
    emb = lib.minigpt4_encode_image(c, mi)
    lib.minigpt4_system_prompt(c)
    lib.minigpt4_begin_chat_image(c, emb, "what is this?")
    lib.minigpt4_free_embedding(emb)
    return c


def text(ext, c, i):
    return ext.L.minigpt4_b200_token_text(c.ptr, int(i))


def end_chat(lib, c, p):
    """minigpt4_end_chat with mirostat arguments p: the token's bytes"""
    tok = ctypes.c_char_p()
    assert lib.library.minigpt4_end_chat(c.ptr, ctypes.byref(tok), 0, p["temp"], 40, 0.9, 1.0, 1.0, *UNUSED, p["mirostat"], p["mirostat_tau"],
                                         p["mirostat_eta"], 1) == 0
    return tok.value


def end_chat_batch(ext, ctxs, p):
    toks = (ctypes.c_char_p * len(ctxs))()
    assert ext.L.minigpt4_b200_end_chat_batch(ctypes.cast(ext._ctx_array(ctxs), ctypes.c_void_p), len(ctxs), ctypes.cast(toks, ctypes.c_void_p),
                                              p["temp"], 40, 0.9, 1.0, 1.0, *UNUSED, p["mirostat"], p["mirostat_tau"], p["mirostat_eta"], 1) == 0
    return [toks[i] for i in range(len(ctxs))]


def _same_state(lib, ext, a, b, p, steps=8):
    assert ext.n_past(a) == ext.n_past(b)
    assert np.array_equal(ext.logits(a), ext.logits(b))
    assert ext.greedy_id(a) == ext.greedy_id(b)
    assert [end_chat(lib, a, p) for _ in range(steps)] == [end_chat(lib, b, p) for _ in range(steps)]   # μ and the generators
    assert np.array_equal(ext.logits(a), ext.logits(b))


@pytest.mark.parametrize("name,mega", [("q4_1", True), ("q5_k", False), ("q4_1_32000", True)],
                         ids=["q4_1-megakernel", "q5_k-q6_k-per-op", "n_vocab-32000"])
@pytest.mark.parametrize("p", [M1, M2], ids=["mirostat1", "mirostat2"])
def test_one_context_equals_end_chat(lib, ext, mg, files, name, mega, p):
    a = _chat(lib, mg, files["vision"], files[name], seed=1234)
    b = _chat(lib, mg, files["vision"], files[name], seed=1234)
    assert (ext.stats(a).decode_megakernel >= 6) == mega
    ids, _ = ext.sample_steps([a], 48, **p)
    assert [text(ext, a, i) for i in ids[:, 0]] == [end_chat(lib, b, p) for _ in range(48)]
    _same_state(lib, ext, a, b, p)
    # the other mode on the same contexts: its own μ starts at 2 tau on both, the generator goes on
    q = M2 if p is M1 else M1
    ids, _ = ext.sample_steps([a], 16, **q)
    assert [text(ext, a, i) for i in ids[:, 0]] == [end_chat(lib, b, q) for _ in range(16)]
    _same_state(lib, ext, a, b, q)
    _same_state(lib, ext, a, b, p)
    for c in (a, b):
        lib.minigpt4_free(c)


@pytest.mark.parametrize("mode", [1, 2])
def test_greedy_leaves_mu_alone(lib, ext, mg, files, mode):
    """temp 0: the ids of decode_chain, and μ is neither read nor set (before and after the mode's first use)"""
    p = dict(temp=0.8, mirostat=mode, mirostat_tau=5.0, mirostat_eta=1.0)
    a = _chat(lib, mg, files["vision"], files["q4_1"], seed=9)
    b = _chat(lib, mg, files["vision"], files["q4_1"], seed=9)
    for first in (True, False):
        ids, _ = ext.sample_steps([a], 16, temp=0.0, mirostat=mode, mirostat_tau=3.0, mirostat_eta=1.0)
        want, _ = ext.decode_chain(b, 16)
        assert ids[:, 0].tolist() == want.tolist()
        assert ext.n_past(a) == ext.n_past(b) and np.array_equal(ext.logits(a), ext.logits(b))
        assert end_chat(lib, a, p) == end_chat(lib, b, p), first   # μ unset (first) / as the host left it
    for c in (a, b):
        lib.minigpt4_free(c)


def _sessions(ext, path, seeds, prompts, n_ctx=256):
    p = ext.llm_load(path, n_ctx=n_ctx, seed=seeds[0])
    ses = [p] + [ext.session_create(p, s) for s in seeds[1:]]
    for c, pr in zip(ses, prompts):
        ext.eval_tokens(c, pr)
    return ses


@pytest.mark.parametrize("which,n", [("tiny", 2), ("tiny", 3), ("tiny", 5), ("tiny", 8), ("wide", 3)],
                         ids=["tiny-B2", "tiny-B3", "tiny-B5", "tiny-B8", "4096-B3"])
@pytest.mark.parametrize("p", [M1, M2], ids=["mirostat1", "mirostat2"])
def test_sessions_equal_end_chat_batch(lib, ext, tiny, files, which, n, p):
    path = tiny["q4_1"] if which == "tiny" else files["q4_1"]
    rng = np.random.default_rng(17 + n)
    prompts = [rng.integers(3, 1000, size=3 + 4 * i).tolist() for i in range(n)]
    seeds = [101 + 7 * i for i in range(n)]
    a = _sessions(ext, path, seeds, prompts)
    b = _sessions(ext, path, seeds, prompts)
    ids, _ = ext.sample_steps(a, 24, **p)
    want = [end_chat_batch(ext, b, p) for _ in range(24)]
    for i in range(n):
        assert [text(ext, a[i], t) for t in ids[:, i]] == [w[i] for w in want], f"session {i}"
        assert ext.n_past(a[i]) == ext.n_past(b[i])
        assert np.array_equal(ext.logits(a[i]), ext.logits(b[i])), f"session {i}"
    assert [end_chat_batch(ext, a, p) for _ in range(4)] == [end_chat_batch(ext, b, p) for _ in range(4)]   # μ and generators
    for c in a + b:
        ext.base.minigpt4_free(c)


# ---- whole replies --------------------------------------------------------------------------------------------------------------------
def ref_reply(lib, c, max_steps, p, stop=b"###"):
    texts, chat = [], b""
    for _ in range(max_steps):
        t = end_chat(lib, c, p)
        texts.append(t)
        chat += t
        if t != b"##" and chat.endswith(stop):
            return texts, True
    return texts, False


@pytest.mark.parametrize("chunk", [0, 1, 3, 16], ids=["one-call", "chunk1", "chunk3", "chunk16"])
@pytest.mark.parametrize("p", [M1, M2], ids=["mirostat1", "mirostat2"])
def test_reply_equals_the_end_chat_loop(lib, ext, mg, files, chunk, p):
    a = _chat(lib, mg, files["vision"], files["hash"], seed=1234)
    b = _chat(lib, mg, files["vision"], files["hash"], seed=1234)
    want, want_stopped = ref_reply(lib, b, 96, p)
    got, stopped = [], False
    while len(got) < 96 and not stopped:
        step = 96 - len(got) if chunk == 0 else min(chunk, 96 - len(got))
        ids, st, _ = ext.sample_until([a], step, None, **p)
        got, stopped = got + ids[0], st[0]
    assert [text(ext, a, i) for i in got] == want
    assert stopped == want_stopped
    _same_state(lib, ext, a, b, p)
    for c in (a, b):
        lib.minigpt4_free(c)


@pytest.mark.parametrize("p", [M1, M2], ids=["mirostat1", "mirostat2"])
def test_batched_replies_equal_end_chat_batch(lib, ext, files, p):
    n = 5
    rng = np.random.default_rng(23)
    prompts = [rng.integers(3, 1000, size=3 + 4 * i).tolist() for i in range(n)]
    seeds = [41 + 3 * i for i in range(n)]
    a = _sessions(ext, files["hash_tiny"], seeds, prompts)
    b = _sessions(ext, files["hash_tiny"], seeds, prompts)
    texts, chat, stopped, live = [[] for _ in range(n)], [b""] * n, [False] * n, list(range(n))
    for _ in range(48):
        if not live:
            break
        nxt = []
        for i, t in zip(live, end_chat_batch(ext, [b[i] for i in live], p)):
            texts[i].append(t)
            chat[i] += t
            if t != b"##" and chat[i].endswith(b"###"):
                stopped[i] = True
            else:
                nxt.append(i)
        live = nxt
    got, got_stopped, _ = ext.sample_until(a, 48, None, **p)
    for i in range(n):
        assert [text(ext, a[i], t) for t in got[i]] == texts[i], f"session {i}"
        assert got_stopped[i] == stopped[i]
        assert ext.n_past(a[i]) == ext.n_past(b[i]) and np.array_equal(ext.logits(a[i]), ext.logits(b[i]))
    assert [end_chat_batch(ext, a, p) for _ in range(4)] == [end_chat_batch(ext, b, p) for _ in range(4)]
    for c in a + b:
        ext.base.minigpt4_free(c)


# ---- refusals -------------------------------------------------------------------------------------------------------------------------
def test_refused_calls_change_nothing(lib, ext, files):
    path = files["hash_tiny"]
    a = _sessions(ext, path, [5, 6], [[3, 4, 5, 6], [7, 8]], n_ctx=16)
    b = _sessions(ext, path, [5, 6], [[3, 4, 5, 6], [7, 8]], n_ctx=16)
    for x, y in zip(a, b):   # μ of both modes set and moved on both twins
        for p in (M1, M2):
            assert end_chat(lib, x, p) == end_chat(lib, y, p)
    before = [(ext.n_past(c), ext.logits(c)) for c in a]
    arr = ctypes.cast(ext._ctx_array(a), ctypes.c_void_p)
    ids, n_out = (ctypes.c_int32 * 128)(), (ctypes.c_int32 * 8)()
    steps = lambda n, k, m=1: ext.L.minigpt4_b200_sample_steps_mirostat(arr, n, k, 0.8, m, 5.0, 0.1, ids, None)
    until = lambda n, k, m=2, stop=None: ext.L.minigpt4_b200_sample_until_mirostat(arr, n, k, stop, 0.8, m, 5.0, 1.0, ids, n_out, None, None)
    assert steps(2, 11) == 8          # 6 + 11 > 16
    assert steps(2, 0) == 8
    assert steps(2, 2, 3) == 8        # mirostat 3
    assert steps(2, 2, 0) == 8
    assert until(2, 11) == 8
    assert until(2, 2, 0) == 8
    assert until(2, 2, 2, b"#" * 33) == 8
    for c, (n, lg) in zip(a, before):
        assert ext.n_past(c) == n and np.array_equal(ext.logits(c), lg)
    for p in (M1, M2):
        assert [end_chat(lib, c, p) for c in a] == [end_chat(lib, c, p) for c in b]   # μ and generators untouched
    for c in a + b:
        ext.base.minigpt4_free(c)


# ---- Python ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("p", [M1, M2], ids=["mirostat1", "mirostat2"])
def test_generate_on_device_yields_what_generate_yields(mg, files, p):
    import minigpt4_cpp_b200 as m
    bots = [m.MiniGPT4ChatBot(files["vision"], files["hash"]) for _ in range(2)]
    for bot in bots:
        bot.upload_image(mg.synth_image(3).reshape(1, 3, 224, 224))
    want = list(bots[0].generate("what is this?", limit=200, **p))
    got = list(bots[1].generate_on_device("what is this?", limit=200, chunk=16, **p))
    assert got == want and len(want) < 199
    assert list(bots[1].generate_on_device("and then?", limit=200, **p)) == list(bots[0].generate("and then?", limit=200, **p))
    for bot in bots:
        bot.free()
