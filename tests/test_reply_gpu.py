"""Whole replies on the GPU (minigpt4_b200_sample_until): each context stops where the reference's chat loop stops its reply.

- the device's stop rule (op_reply_stop) against a Python restatement of the loop, on bytes, over a vocabulary full of '#' pieces;
- one context against the end_chat loop on a twin: ids, n_out, stopped, n_past, logits bit for bit, greedy id, then the generator;
  in one call and in chunks, after a few end_chat tokens, and greedy against decode_chain;
- batches against end_chat_batch twins that drop each context when its reply ends;
- the steps run past the last stop, from the kernel launch count;
- refused calls that change nothing;
- MiniGPT4ChatBot.generate_on_device against generate()."""
import ctypes

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

WEBUI = dict(temp=0.8, top_k=40, top_p=0.9)
CHUNK = 4   # LlamaDevice::kReplyChunk: at most 2 CHUNK - 1 steps run past the last stop
UNUSED = (64, 1.1, 1.0, 1.0, 0, 5.0, 1.0, 1)   # repeat_last_n .. penalize_nl of end_chat (mirostat 0)


# ---- the reference's loop, on bytes -------------------------------------------------------------------------------------------------
def ref_stop(texts, stop=b"###", chat=b""):
    """MiniGPT4ChatBot.generate's loop over these token texts from a reply `chat`: the index of the token that ends it, -1 if none"""
    for i, t in enumerate(texts):
        chat += t
        if t == b"##":
            continue
        if stop and chat.endswith(stop):
            return i
    return -1


def hash_vocab(mg, n_vocab, seed=5):
    """make_vocab with the byte tokens 0x80..0xff and the last third of the pieces replaced by '#'-bearing ASCII pieces: every piece is
    valid UTF-8 on its own, and random replies reach "###" within a few dozen tokens"""
    v = mg.make_vocab(n_vocab)
    seen = {p for p, _ in v}
    rng = np.random.default_rng(seed)
    fresh = [p for p in (b"a#", b"#b", b"#a#", b" #", b"# ", b"##a", b"b##", b"\n#", b"####", b"#\n") if p not in seen]
    seen.update(fresh)
    slots = list(range(3 + 0x80, 259)) + list(range(n_vocab - n_vocab // 3, n_vocab))
    while len(fresh) < len(slots):
        p = bytes(rng.choice(list(b"#ab #"), size=int(rng.integers(1, 7))).tolist())
        if p not in seen:
            seen.add(p)
            fresh.append(p)
    for i, p in zip(slots, fresh):
        v[i] = (p, v[i][1] if i >= 259 else -2.0)
    return v


def text(ext, c, i):
    return ext.L.minigpt4_b200_token_text(c.ptr, int(i))


def end_chat(lib, c, p):
    tok = ctypes.c_char_p()
    assert lib.library.minigpt4_end_chat(c.ptr, ctypes.byref(tok), 0, p["temp"], p["top_k"], p["top_p"], 1.0, 1.0, *UNUSED) == 0
    return tok.value


def end_chat_batch(ext, ctxs, p):
    toks = (ctypes.c_char_p * len(ctxs))()
    assert ext.L.minigpt4_b200_end_chat_batch(ctypes.cast(ext._ctx_array(ctxs), ctypes.c_void_p), len(ctxs), ctypes.cast(toks, ctypes.c_void_p),
                                              p["temp"], p["top_k"], p["top_p"], 1.0, 1.0, *UNUSED) == 0
    return [toks[i] for i in range(len(ctxs))]


def ref_reply(lib, c, max_steps, stop, p, chat=b""):
    """the end_chat loop on c until its reply ends with stop: (texts, stopped)"""
    texts = []
    for _ in range(max_steps):
        t = end_chat(lib, c, p)
        texts.append(t)
        chat += t
        if t != b"##" and stop and chat.endswith(stop):
            return texts, True
    return texts, False


def until_chunks(ext, c, max_steps, stop, p, chunk):
    """sample_until over calls of `chunk` steps until the reply ends: (ids, stopped)"""
    ids = []
    while len(ids) < max_steps:
        got, stopped, _ = ext.sample_until([c], min(chunk, max_steps - len(ids)), stop, **p)
        ids += got[0]
        if stopped[0]:
            return ids, True
    return ids, False


# ---- files --------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def files(tiny, mg, tmp_path_factory):
    d = tmp_path_factory.mktemp("reply")
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


def _same_state(lib, ext, a, b, p):
    assert ext.n_past(a) == ext.n_past(b)
    assert np.array_equal(ext.logits(a), ext.logits(b))
    assert ext.greedy_id(a) == ext.greedy_id(b)
    assert [end_chat(lib, a, p) for _ in range(8)] == [end_chat(lib, b, p) for _ in range(8)]   # the generators
    assert np.array_equal(ext.logits(a), ext.logits(b))


# ---- the stop rule ------------------------------------------------------------------------------------------------------------------
def test_stop_rule_equals_the_reference_loop(lib, ext, mg, files):
    c = ext.llm_load(files["hash_tiny"], n_ctx=64)
    V = ext.L.minigpt4_b200_n_vocab(c.ptr)
    texts = [text(ext, c, i) for i in range(V)]
    by = {t: i for i, t in enumerate(texts)}
    assert texts[2] == b"</s>" and texts[3] == b""                    # id 2, and the NUL byte token cut at its NUL
    hashy = [i for i, t in enumerate(texts) if b"#" in t]
    rng = np.random.default_rng(11)
    for case in range(400):
        pool = hashy if case % 2 == 0 else list(range(V))
        ids = rng.choice(pool, size=int(rng.integers(1, 40))).tolist()
        stop = [None, b"###", b"#", b"a#b", b"## #", b"", b"#" * 32][case % 7]
        tail = [b"", b"#", b"##", b"x" * 40 + b"#"][case % 4]
        want = ref_stop([texts[i] for i in ids], b"###" if stop is None else stop, tail)
        assert ext.op_reply_stop(c, ids, stop, tail) == want, (ids, stop, tail)
    # "##" then "#": the "##" is no stop even when it completes "###"; the "#" after it is
    assert ext.op_reply_stop(c, [by[b"#"], by[b"##"], by[b"#"]]) == 2
    assert ext.op_reply_stop(c, [by[b"##"]], None, b"#") == -1
    # a stop text over three tokens, from a non-empty tail, with the NUL token (empty text) between
    assert ext.op_reply_stop(c, [by[b"a#"], 3, by[b"#b"], by[b" #"]], b"a##b #", b"zz") == 3
    assert ext.op_reply_stop(c, [3], b"###", b"x###") == 0           # an empty piece on a reply that already ends with the stop
    assert ext.op_reply_stop(c, [by[b"a#"], by[b"#b"]], b"a##b") == 1
    assert ext.op_reply_stop(c, [5, 2, 7], b"</s>") == 1             # id 2 is "</s>"
    assert ext.op_reply_stop(c, [by[b"###"]] * 4, b"") == -1          # no text stop
    # the table, id by id
    for i, t in enumerate(texts):
        if t and len(t) <= 32 and t != b"##":
            assert ext.op_reply_stop(c, [i], t) == 0, (i, t)
    ext.base.minigpt4_free(c)


# ---- one context ---------------------------------------------------------------------------------------------------------------------
_STREAMS = {}


def _forced_stop(lib, mg, ext, files, name, p, k, span):
    """a stop text that first ends the reply at step k of the twins' stream (span: longer than that step's text, so over two tokens)"""
    if name not in _STREAMS:
        c = _chat(lib, mg, files["vision"], files[name], seed=1234)
        _STREAMS[name] = [end_chat(lib, c, p) for _ in range(24)]
        lib.minigpt4_free(c)
    texts = _STREAMS[name][:k + 1]
    reply = b"".join(texts)
    for n in range(1, 33):
        stop = reply[-n:]
        if len(stop) == n and (not span or n > len(texts[k])) and ref_stop(texts, stop) == k:
            return stop
    pytest.skip(f"no stop text ends this reply first at step {k}")


@pytest.mark.parametrize("name,mega,p", [("q4_1", True, WEBUI), ("q5_k", False, WEBUI), ("q4_1_32000", True, dict(temp=0.8, top_k=0, top_p=0.95)),
                                         ("hash", True, WEBUI)],
                         ids=["q4_1-megakernel", "q5_k-q6_k-per-op", "n_vocab-32000-top_k-0", "hash-vocab"])
@pytest.mark.parametrize("chunk", [0, 1, 3, 16], ids=["one-call", "chunk1", "chunk3", "chunk16"])
def test_one_context_equals_the_end_chat_loop(lib, ext, mg, files, name, mega, p, chunk):
    stops = [None] if name == "hash" else [_forced_stop(lib, mg, ext, files, name, p, 17, True)]
    if chunk == 0 and name != "hash":
        stops.insert(0, _forced_stop(lib, mg, ext, files, name, p, 9, False))
    for stop in stops:
        for pre in ((0, 3) if chunk == 0 else (3,)):
            a = _chat(lib, mg, files["vision"], files[name], seed=1234)
            b = _chat(lib, mg, files["vision"], files[name], seed=1234)
            assert (ext.stats(a).decode_megakernel >= 6) == mega
            head = [end_chat(lib, a, p) for _ in range(pre)]
            assert head == [end_chat(lib, b, p) for _ in range(pre)]
            want, want_stopped = ref_reply(lib, b, 64, b"###" if stop is None else stop, p, b"".join(head))
            if chunk == 0:
                got, stopped, _ = ext.sample_until([a], 64, stop, **p)
                got, stopped = got[0], stopped[0]
            else:
                got, stopped = until_chunks(ext, a, 64, stop, p, chunk)
            assert [text(ext, a, i) for i in got] == want, (stop, pre)
            assert stopped == want_stopped and (stopped or stop is None)
            _same_state(lib, ext, a, b, p)
            for c in (a, b):
                lib.minigpt4_free(c)


def test_greedy_stops_where_the_decode_chain_text_meets_the_rule(lib, ext, mg, files):
    a = _chat(lib, mg, files["vision"], files["hash"], seed=9)
    b = _chat(lib, mg, files["vision"], files["hash"], seed=9)
    c = _chat(lib, mg, files["vision"], files["hash"], seed=9)
    chain, _ = ext.decode_chain(b, 96)
    k = ref_stop([text(ext, b, i) for i in chain], b"#")
    assert k >= 0
    got, stopped, _ = ext.sample_until([a], 96, "#", temp=0.0)
    assert got[0] == chain[:k + 1].tolist() and stopped == [True]
    ext.decode_chain(c, k + 1)
    assert ext.n_past(a) == ext.n_past(c) and np.array_equal(ext.logits(a), ext.logits(c)) and ext.greedy_id(a) == ext.greedy_id(c)
    assert end_chat(lib, a, WEBUI) == end_chat(lib, c, WEBUI)   # the generator was not touched
    for x in (a, b, c):
        lib.minigpt4_free(x)


# ---- batches --------------------------------------------------------------------------------------------------------------------------
def _sessions(ext, path, seeds, prompts, n_ctx=256):
    p = ext.llm_load(path, n_ctx=n_ctx, seed=seeds[0])
    ses = [p] + [ext.session_create(p, s) for s in seeds[1:]]
    for c, pr in zip(ses, prompts):
        ext.eval_tokens(c, pr)
    return ses


def ref_batch(ext, ctxs, max_steps, stop, p):
    """end_chat_batch over the contexts whose replies have not ended: (texts per context, stopped per context)"""
    n = len(ctxs)
    texts, chat, stopped, live = [[] for _ in range(n)], [b""] * n, [False] * n, list(range(n))
    for _ in range(max_steps):
        if not live:
            break
        nxt = []
        for i, t in zip(live, end_chat_batch(ext, [ctxs[i] for i in live], p)):
            texts[i].append(t)
            chat[i] += t
            if t != b"##" and stop and chat[i].endswith(stop):
                stopped[i] = True
            else:
                nxt.append(i)
        live = nxt
    return texts, stopped


@pytest.mark.parametrize("which,n,stop", [("hash_tiny", 2, None), ("hash_tiny", 3, None), ("hash_tiny", 5, "#a"), ("hash_tiny", 8, None),
                                          ("hash_tiny", 8, "##a"), ("hash", 3, None)],
                         ids=["tiny-B2", "tiny-B3", "tiny-B5-stop-#a", "tiny-B8", "tiny-B8-stop-##a", "4096-B3"])
def test_sessions_equal_end_chat_batch(lib, ext, files, which, n, stop):
    rng = np.random.default_rng(17 + n)
    prompts = [rng.integers(3, 1000, size=3 + 4 * i).tolist() for i in range(n)]
    seeds = [101 + 7 * i for i in range(n)]
    a = _sessions(ext, files[which], seeds, prompts)
    b = _sessions(ext, files[which], seeds, prompts)
    want, want_stopped = ref_batch(ext, b, 40, b"###" if stop is None else stop.encode(), WEBUI)
    got, stopped, _ = ext.sample_until(a, 40, stop, **WEBUI)
    for i in range(n):
        assert [text(ext, a[i], t) for t in got[i]] == want[i], f"session {i}"
        assert stopped[i] == want_stopped[i]
        assert ext.n_past(a[i]) == ext.n_past(b[i])
        assert np.array_equal(ext.logits(a[i]), ext.logits(b[i])), f"session {i}"
        assert ext.greedy_id(a[i]) == ext.greedy_id(b[i])
    # the generators continue on the host, also for the contexts that stopped while the batch ran on
    assert [ext.end_chat_batch(a, **WEBUI) for _ in range(4)] == [ext.end_chat_batch(b, **WEBUI) for _ in range(4)]
    for i in range(n):
        assert np.array_equal(ext.logits(a[i]), ext.logits(b[i])), f"session {i}"
    for c in a + b:
        ext.base.minigpt4_free(c)


# ---- overshoot ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 3])
def test_steps_past_the_last_stop_are_bounded(ext, files, n):
    a = _sessions(ext, files["hash_tiny"], [31 + i for i in range(n)], [[5, 6, 7 + i] for i in range(n)])
    launches = lambda: ext.stats(a[0]).kernel_launches
    x = launches()
    ext.sample_steps(a, 1, **WEBUI)
    per_step = launches() - x
    x = launches()
    got, stopped, _ = ext.sample_until(a, 96, "#", **WEBUI)
    s = max(len(g) for g in got)
    assert all(stopped)
    assert launches() - x <= (s + 2 * CHUNK - 1) * per_step
    for c in a:
        ext.base.minigpt4_free(c)


# ---- refusals -------------------------------------------------------------------------------------------------------------------------
def test_refused_calls_change_nothing(lib, ext, files):
    path = files["hash_tiny"]
    a = _sessions(ext, path, [5, 6], [[3, 4, 5, 6], [7, 8]], n_ctx=16)
    b = _sessions(ext, path, [5, 6], [[3, 4, 5, 6], [7, 8]], n_ctx=16)
    other = ext.llm_load(path, n_ctx=16, seed=5)
    for c in a + b + [other]:
        ext.flush(c)
    before = [(ext.n_past(c), ext.logits(c)) for c in a]
    ids, n_out = (ctypes.c_int32 * 128)(), (ctypes.c_int32 * 8)()

    def call(ctxs, n, max_steps, stop=None, ids=ids, n_out=n_out):
        arr = ctypes.cast((ctypes.c_void_p * len(ctxs))(*[c.ptr if c else None for c in ctxs]), ctypes.c_void_p)
        return ext.L.minigpt4_b200_sample_until(arr, n, max_steps, stop, 0.8, 40, 0.9, 1.0, 1.0, ids, n_out, None, None)

    assert call(a, 2, 13) == 8                          # 4 + 13 > 16
    assert call(a, 1, 0) == 8                           # max_steps < 1
    assert call(a, 2, 4, b"#" * 33) == 8                # stop text over 32 bytes
    assert call(a, 2, 4, n_out=None) == 8               # NULL n_out
    assert call(a, 2, 4, ids=None) == 8                 # NULL ids_out
    assert call([a[0], a[0]], 2, 4) == 8                # duplicate context
    assert call([a[0], other], 2, 4) == 8               # another group
    assert call(a + [None], 3, 4) == 8                  # NULL context
    assert call(a * 5, 9, 4) == 8                       # n outside 1..8
    for c, (n, lg) in zip(a, before):
        assert ext.n_past(c) == n and np.array_equal(ext.logits(c), lg)
    assert [end_chat(lib, c, WEBUI) for c in a] == [end_chat(lib, c, WEBUI) for c in b]   # generators untouched
    for c in a + b + [other]:
        ext.base.minigpt4_free(c)


# ---- Python ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("chunk", [1, 16])
def test_generate_on_device_yields_what_generate_yields(mg, files, chunk):
    import minigpt4_cpp_b200 as m
    bots = [m.MiniGPT4ChatBot(files["vision"], files["hash"]) for _ in range(2)]
    for bot in bots:
        bot.upload_image(mg.synth_image(3).reshape(1, 3, 224, 224))
    want = list(bots[0].generate("what is this?", limit=200))
    got = list(bots[1].generate_on_device("what is this?", limit=200, chunk=chunk))
    assert got == want and len(want) < 199
    # the next turn starts a new reply on both
    assert list(bots[1].generate_on_device("and then?", limit=200, chunk=chunk)) == list(bots[0].generate("and then?", limit=200))
    for bot in bots:
        bot.free()
