"""Beam search on the GPU (minigpt4_b200_beam_search) against its restatement in Python (tests/beam_spec.py):

- the candidate order of the rank and merge kernels (op_beam_rank) against numpy, with exact ties;
- one beam against sample_until(temp 0): ids, n_out, stopped and the context's state, with and without the prefill GEMM;
- 2, 4, 8 and 16 beams against the restatement run on CPU-oracle logits, over a '#'-heavy vocabulary so replies end early; every
  entry's S against the float32 left fold of score_tokens' log-probabilities, bit for bit;
- the contexts afterwards: ctxs[0] as a twin that fed the best ids, the others as a session_copy of the conversation;
- stop texts, limits and refusals."""
import numpy as np
import pytest

import beam_spec as bs
from test_reply_gpu import hash_vocab

pytestmark = pytest.mark.gpu

PROMPT = [1, 15, 27, 300, 41, 9, 77]
# the prompts a comparison with the Python model may use: the first on which that model meets no near tie (the device's log-probabilities
# may differ from numpy's in the last place, so only decisions between values more than TIE_ULPS apart are compared exactly)
PROMPTS = [PROMPT] + [[1] + np.random.default_rng(s).integers(3, 1000, 6).tolist() for s in range(23)]
TIE_ULPS = 4


@pytest.fixture(scope="module")
def files(tiny, mg, orc, tmp_path_factory):
    d = tmp_path_factory.mktemp("beam")
    out = dict(tiny)
    for name, kw in (("hash", dict(n_embd=512, n_head=4, n_layer=2, n_vocab=1024, wtype="q4_1", vocab=hash_vocab(mg, 1024))),
                     ("hash_q4_0", dict(n_embd=512, n_head=4, n_layer=2, n_vocab=1024, wtype="q4_0", vocab=hash_vocab(mg, 1024, seed=7))),
                     ("wide", dict(n_embd=4096, n_head=32, n_layer=2, n_vocab=2048, wtype="q4_1", vocab=hash_vocab(mg, 2048)))):
        out[name] = str(d / f"llama-{name}.bin")
        mg.write_llama_ggjt(out[name], mg.LlamaSpec(**kw))
    # "hash_exempt": hash_q4_0's weights with the texts of its greedy id after PROMPT and of "##" swapped (the texts do not touch the
    # weights), so the first candidate of every search from PROMPT is "##", which stop "#" would end without the exception
    z = orc.OracleEngine(None, out["hash_q4_0"], n_ctx=64).eval_tokens(PROMPT)
    v = hash_vocab(mg, 1024, seed=7)
    x = int(np.argmax(z))
    h = next((i for i, (p, _) in enumerate(v) if p == b"##"), None)
    if h is None:
        h = len(v) - 1
        v[h] = (b"##", v[h][1])
    v[x], v[h] = (v[h][0], v[x][1]), (v[x][0], v[h][1])
    out["hash_exempt"] = str(d / "llama-hash_exempt.bin")
    mg.write_llama_ggjt(out["hash_exempt"], mg.LlamaSpec(n_embd=512, n_head=4, n_layer=2, n_vocab=1024, wtype="q4_0", vocab=v))
    return out


def texts_of(ext, c):
    return [ext.L.minigpt4_b200_token_text(c.ptr, i) for i in range(ext.L.minigpt4_b200_n_vocab(c.ptr))]


def load(ext, path, n_beams, n_ctx=256, prompt=PROMPT):
    c = ext.llm_load(path, n_ctx=n_ctx)
    ext.eval_tokens(c, prompt)
    return [c] + [ext.session_create(c) for _ in range(n_beams - 1)]


def free(ext, ctxs):
    for c in ctxs:
        ext.base.minigpt4_free(c)


class OracleLogits:
    """logits after the prompt and ids, from the CPU oracle: rows are re-evaluated from the longest prefix its cache still holds"""

    def __init__(self, orc, path, prompt, n_ctx):
        self.e = orc.OracleEngine(None, path, n_ctx=n_ctx)
        self.n0 = len(prompt)
        self.cache = {(): self.e.eval_tokens(prompt).copy()}
        self.cur = ()

    def __call__(self, ids):
        ids = tuple(ids)
        if ids not in self.cache:
            k = 0
            while k < min(len(ids), len(self.cur)) and ids[k] == self.cur[k]:
                k += 1
            k = min(k, len(ids) - 1)
            self.e.n_past = self.n0 + k
            self.cache[ids] = self.e.eval_tokens(list(ids[k:])).copy()
            self.cur = ids
        return self.cache[ids]


def fold(lps):
    s = np.float32(0.0)
    for x in lps:
        s = np.float32(s + np.float32(x))
    return float(s)


# ---- the kernels' order ---------------------------------------------------------------------------------------------------------------
def _check_rank(ext, logits, S, n_beams):
    par, ids, c = ext.op_beam_rank(logits, S, n_beams)
    n_live, V = logits.shape
    k = min(2 * n_beams, n_live * V)
    assert len(par) == k
    keys = [(c[r], int(par[r]), logits[par[r], ids[r]], int(ids[r])) for r in range(k)]
    assert keys == sorted(keys, key=bs.order_key), "not in the search's order"
    assert len(set(zip(par.tolist(), ids.tolist()))) == k
    for b in range(n_live):
        lp = bs.lp_row(logits[b])
        top = np.lexsort((np.arange(V), -logits[b]))
        mine = [int(ids[r]) for r in range(k) if par[r] == b]
        assert mine == top[:len(mine)].tolist(), "a beam's candidates are not its best ids"
        for r in range(k):
            if par[r] == b:
                want = np.float32(S[b] + lp[ids[r]])
                assert bs.ulps(c[r], want) <= 1, (b, int(ids[r]), c[r], want)
        if len(mine) < min(2 * n_beams, V):   # the next candidate of this beam orders after the last one returned
            v = int(top[len(mine)])
            nxt = (np.float32(S[b] + lp[v]), b, logits[b, v], v)
            last = keys[-1]
            assert bs.order_key(nxt) >= bs.order_key(last) or bs.ulps(nxt[0], last[0]) <= 1


@pytest.mark.parametrize("n_beams", [1, 2, 4, 16])
def test_rank_order_against_numpy(ext, n_beams):
    rng = np.random.default_rng(n_beams)
    for case in range(6):
        n_live = int(rng.integers(1, n_beams + 1))
        V = [32000, 1024, 37, 2048, 5000, 64][case]
        lg = (rng.standard_normal((n_live, V)) * 4).astype(np.float32)
        S = (-rng.random(n_live) * 10).astype(np.float32)
        if case % 3 == 1:                          # duplicate rows across beams with equal S: exact ties across beams
            lg[:] = lg[0]
            S[:] = S[0]
        if case % 3 == 2:                          # few distinct values: equal logits within a row
            lg = np.round(lg).astype(np.float32)
        _check_rank(ext, lg, S, n_beams)


# ---- one beam is greedy sample_until -------------------------------------------------------------------------------------------------
def _same_state(ext, a, b):
    assert ext.n_past(a) == ext.n_past(b)
    assert np.array_equal(ext.logits(a), ext.logits(b))
    assert ext.greedy_id(a) == ext.greedy_id(b)


@pytest.mark.parametrize("name", ["q4_0", "q4_1", "q5_k", "q6_k", "hash"])
@pytest.mark.parametrize("gemm", [True, False], ids=["prefill-gemm", "no-prefill-gemm"])
def test_one_beam_equals_greedy_sample_until(ext, files, monkeypatch, name, gemm):
    if not gemm:
        monkeypatch.setenv("MINIGPT4_B200_NO_PREFILL_GEMM", "1")
    for stop, steps in ((None, 40), (b"", 24), (b"a", 30)):
        a, = load(ext, files[name], 1)
        b, = load(ext, files[name], 1)
        hyps, _ = ext.beam_search([a], steps, stop)
        ids, stopped, _ = ext.sample_until([b], steps, stop, temp=0.0)
        assert (hyps[0][0], hyps[0][3]) == (ids[0], stopped[0]), (name, stop)
        _same_state(ext, a, b)
        assert ext.sample_until([a], 12, None, temp=0.0)[:2] == ext.sample_until([b], 12, None, temp=0.0)[:2]   # the tail and the state go on
        _same_state(ext, a, b)
        free(ext, [a, b])


# ---- several beams against the restatement (the reply tail a search leaves is checked through sample_until above) ------------------------------------------------------------------------------------------
def _spec(ext, orc, path, n_beams, max_steps, stop, lp_pen, n_ctx, ctx, logits_fn=None, need=None):
    """(prompt, H of the Python model) on the first of PROMPTS where the model meets no near tie (and need(stats) holds)"""
    ties = []
    for prompt in PROMPTS:
        fn = logits_fn(prompt) if logits_fn else OracleLogits(orc, path, prompt, n_ctx)
        stats = {}
        try:
            want = bs.beam_search(fn, n_beams, max_steps, texts_of(ext, ctx), stop, lp_pen, tie_ulps=TIE_ULPS, stats=stats)
        except bs.NearTie as t:
            ties.append(str(t))
            continue
        if need is None or need(stats):
            return prompt, want
    pytest.fail("no prompt gives a comparison the Python model can make exactly (near ties: " + "; ".join(ties) + ")")


def _check_search(ext, files, name, n_beams, max_steps, stop, lp_pen, spec, n_ctx=256):
    prompt, want = spec
    ctxs = load(ext, files[name], n_beams, n_ctx, prompt)
    twin = load(ext, files[name], 1, n_ctx, prompt)[0]
    copy = ext.session_create(twin)
    ext.session_copy(twin, [copy])
    texts = texts_of(ext, twin)
    hyps, ms = ext.beam_search(ctxs, max_steps, stop, lp_pen, n_beams)
    assert ms > 0
    got = [h for h in hyps if h[0]]
    assert [(h[0], h[3]) for h in got] == [(w[0], w[3]) for w in want]
    assert [h[1] for h in got] == pytest.approx([w[1] for w in want], rel=1e-5)
    assert all(h[1] == -np.inf and not h[0] for h in hyps[len(got):])
    for h in got:   # S: the float32 left fold of score_tokens' log-probabilities, bit for bit
        lp, = ext.score_tokens([twin], [h[0]])[0][:1]
        assert h[2] == fold(lp), (h[0], h[2], fold(lp))
    # the others: the conversation as it was, also in the K / V rows below n0 that the next steps read
    after = ext.sample_until([copy], 8, b"", temp=0.0)[0][0]
    for c in ctxs[1:]:
        assert ext.n_past(c) == len(prompt) and np.array_equal(ext.logits(c), ext.logits(twin))
        assert ext.sample_until([c], 8, b"", temp=0.0)[0][0] == after
    # ctxs[0]: the twin fed the best ids: logits, greedy id, the next 8 greedy ids, and the reply tail (where a later sample_until stops)
    best = got[0][0]
    ext.eval_tokens(twin, best)
    assert ext.n_past(ctxs[0]) == len(prompt) + len(best)
    _same_state(ext, ctxs[0], twin)
    if ext.n_past(twin) + 24 <= n_ctx:
        nxt = ext.sample_until([ctxs[0]], 8, b"", temp=0.0)[0][0]
        assert nxt == ext.sample_until([twin], 8, b"", temp=0.0)[0][0]
        _same_state(ext, ctxs[0], twin)
        tail = b"".join(texts[i] for i in best + nxt)[-bs.KEEP:]   # the twin's own tail restarted at eval_tokens; compute where it stops
        more = ext.sample_until([twin], 16, b"", temp=0.0)[0][0]
        k = next((j for j in range(len(more)) if bs.ends(tail + b"".join(texts[i] for i in more[:j]), texts[more[j]], b"#")), None)
        ids, stopped, _ = ext.sample_until([ctxs[0]], 16, b"#", temp=0.0)
        assert (ids[0], stopped[0]) == ((more[:k + 1], True) if k is not None else (more, False))
    free(ext, ctxs + [twin, copy])


@pytest.mark.parametrize("n_beams", [2, 4, 8, 16])
@pytest.mark.parametrize("lp_pen", [1.0, 0.0, 2.0])
def test_beams_equal_the_restatement(ext, orc, files, n_beams, lp_pen):
    c = ext.llm_load(files["hash"], n_ctx=256)
    spec = _spec(ext, orc, files["hash"], n_beams, 32, None, lp_pen, 256, c)
    ext.base.minigpt4_free(c)
    _check_search(ext, files, "hash", n_beams, 32, None, lp_pen, spec)


@pytest.mark.parametrize("name,stop,max_steps", [("hash_q4_0", b"", 20), ("hash_q4_0", b"a#b", 40), ("hash_exempt", b"#", 12),
                                                 ("hash_q4_0", None, 24)],
                         ids=["no-stop", "spanning-stop", "hash-exempt", "default-stop"])
def test_stops_and_limits(ext, orc, files, name, stop, max_steps):
    """a stop text over several ids, none, the chat's "###", and the "##" exception: on hash_exempt a search from PROMPT walks "##" first,
    which stop "#" would end without the exception; the prompt taken is the first without near ties on which the Python model walks
    such a candidate (it counts them)"""
    c = ext.llm_load(files[name], n_ctx=256)
    need = (lambda st: st["hash_exempt"] > 0) if name == "hash_exempt" else None
    spec = _spec(ext, orc, files[name], 4, max_steps, stop, 1.0, 256, c, need=need)
    ext.base.minigpt4_free(c)
    if stop == b"":
        assert all(len(w[0]) == max_steps and not w[3] for w in spec[1])
    _check_search(ext, files, name, 4, max_steps, stop, 1.0, spec)


def test_the_last_slot_of_n_ctx(ext, orc, files):
    n_ctx = len(PROMPT) + 9
    c = ext.llm_load(files["hash"], n_ctx=n_ctx)
    spec = _spec(ext, orc, files["hash"], 8, 9, b"", 1.0, n_ctx, c)
    ext.base.minigpt4_free(c)
    _check_search(ext, files, "hash", 8, 9, b"", 1.0, spec, n_ctx=n_ctx)


@pytest.mark.parametrize("n_beams", [4, 16])
def test_wide_model(ext, files, n_beams):
    """4096 wide Q4_1: per-op batched layers at 4 beams, the tensor-core batched layers at 16; the restatement runs on the device's own
    row logits (score_tokens, which the oracle matches bit for bit on this path in test_score_gpu.py)"""
    c = ext.llm_load(files["wide"], n_ctx=256)
    made = []

    def rows(prompt):
        d = load(ext, files["wide"], 1, 256, prompt)[0]
        made.append(d)

        def fn(ids):
            return ext.logits(d) if not ids else ext.score_tokens([d], [list(ids)], logits=True)[0][2][-1]
        return fn
    spec = _spec(ext, None, None, n_beams, 24, None, 1.0, 256, c, rows)
    free(ext, [c] + made)
    _check_search(ext, files, "wide", n_beams, 24, None, 1.0, spec)


# ---- refusals ----------------------------------------------------------------------------------------------------------------------------
def test_refusals_change_nothing(ext, files, lib):
    import ctypes as C
    ctxs = load(ext, files["q4_1"], 4, n_ctx=64)
    other = ext.llm_load(files["q4_1"], n_ctx=64)
    ext.eval_tokens(other, PROMPT)
    empty = ext.session_create(ctxs[0])
    before = [(ext.n_past(c), ext.logits(c)) for c in ctxs]

    def call(cs, n=None, max_steps=8, stop=None, lp=1.0, n_hyp=1, null=None):
        out = np.zeros(64 * 16, np.int32)
        n_out, score = np.zeros(16, np.int32), np.zeros(16, np.float32)
        arr = C.cast(ext._ctx_array(cs), C.c_void_p) if null != "ctxs" else None
        return ext.L.minigpt4_b200_beam_search(arr, len(cs) if n is None else n, max_steps, stop, lp, n_hyp,
                                               None if null == "ids" else out.ctypes.data_as(C.c_void_p),
                                               None if null == "n_out" else n_out.ctypes.data_as(C.c_void_p),
                                               None if null == "score" else score.ctypes.data_as(C.c_void_p), None, None, None)
    for null in ("ctxs", "ids", "n_out", "score"):
        assert call(ctxs, null=null) == 8
    assert call(ctxs, n=0) == 8 and call(ctxs * 5, n=17) == 8
    assert call([ctxs[0], ctxs[1], ctxs[1]]) == 8                     # duplicate
    assert call([ctxs[0], other]) == 8                                # another group
    assert call(ctxs, max_steps=0) == 8
    assert call(ctxs, n_hyp=0) == 8 and call(ctxs, n_hyp=5) == 8
    assert call(ctxs, stop=b"#" * 33) == 8
    assert call(ctxs, lp=float("nan")) == 8 and call(ctxs, lp=float("inf")) == 8
    assert call([empty] + ctxs[1:]) == 8                               # n_past 0
    assert call(ctxs, max_steps=64 - len(PROMPT) + 1) == 8             # past n_ctx
    arr = (C.c_void_p * 2)(ctxs[0].ptr, None)                          # a NULL context among them
    out, n_out, score = np.zeros(16, np.int32), np.zeros(2, np.int32), np.zeros(2, np.float32)
    assert ext.L.minigpt4_b200_beam_search(C.cast(arr, C.c_void_p), 2, 8, None, 1.0, 1, out.ctypes.data_as(C.c_void_p),
                                           n_out.ctypes.data_as(C.c_void_p), score.ctypes.data_as(C.c_void_p), None, None, None) == 8
    # queued rows count: nothing evaluated yet is no empty conversation, and rows that fit only before counting the queue are refused
    queued = ext.session_create(ctxs[0])
    ext.eval_tokens(queued, PROMPT + list(range(40, 60)))
    n_q = len(PROMPT) + 20
    assert ext.n_past(queued) == n_q
    assert call([queued] + ctxs[1:], max_steps=64 - n_q + 1) == 8
    assert ext.n_past(queued) == n_q
    h = ext.constraint_create(ctxs[1], *__import__("minigpt4_cpp_b200").minigpt4_library.choices_dfa([b"a"]))
    ext.constraint_attach(ctxs[1], h)
    assert call(ctxs) == 8                                             # a constrained context
    ext.constraint_attach(ctxs[1], None)
    ext.constraint_free(h)
    for c, (n, lg) in zip(ctxs, before):
        assert ext.n_past(c) == n and np.array_equal(ext.logits(c), lg)
    assert call(ctxs, max_steps=64 - len(PROMPT)) == 0                 # the last slot of n_ctx is allowed
    assert call([queued] + ctxs[1:], max_steps=64 - n_q) == 0          # a conversation still in the queue is evaluated first
    assert ext.n_past(queued) > n_q
    free(ext, ctxs + [other, empty, queued])


def test_chatbot_generate_beam(lib, ext, mg, files):
    import minigpt4_cpp_b200 as m
    bot = m.MiniGPT4ChatBot.__new__(m.MiniGPT4ChatBot)
    bot.library, bot.n_threads, bot.embedding, bot.is_image_chat, bot._keep = lib, 0, None, False, None
    bot.ctx = lib.minigpt4_model_load(files["vision"], files["hash"], 1, 1337, 512, 8, 0)
    twin = lib.minigpt4_model_load(files["vision"], files["hash"], 1, 1337, 512, 8, 0)
    lib.minigpt4_begin_chat(twin, "hi", 0)
    ids, stopped, _ = ext.sample_until([twin], 64, None, temp=0.0)
    words = [ext.L.minigpt4_b200_token_text(twin.ptr, t).decode("utf-8", errors="ignore") for t in ids[0]]
    if stopped[0]:
        words = words[:-1]
    assert list(bot.generate_beam("hi", num_beams=1, limit=64)) == [w for w in words if not lib.minigpt4_contains_eos_token(w)]
    got4 = list(bot.generate_beam("again", num_beams=4, limit=64))
    assert len(bot._beams) == 3 and all(t != "##" for t in got4)
    bot.free()
    lib.minigpt4_free(twin)
