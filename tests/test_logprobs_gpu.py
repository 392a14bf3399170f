"""Log-probabilities of generated replies on the GPU (minigpt4_b200_sample_until_logprobs; llama_logprob.cuh, DESIGN.md §4.14):

- the kernel (op_logprobs) against numpy: random and tied rows, offset logits, vocabularies 1 .. 32001, top_n 0 .. 20 and above n_vocab;
- generation unchanged: a group running sample_until and a twin group running sample_until_logprobs leave the same ids and state, on every
  tiny weight type and at B = 1, 3, 9 and 64 with greedy, the web UI chain, top_k 0 / top_p 0.95, mirostat 1 / 2 and constrained contexts;
- every record bit for bit against score_tokens on a session_copy of the conversation, and the top lists against numpy;
- stops at different steps, a stop text across two calls, max_steps, the last slot of n_ctx, a 4096-wide 32000-id model;
- refusals, the record buffer's memory, and MiniGPT4ChatBot.generate_with_logprobs."""
import ctypes

import numpy as np
import pytest

from minigpt4_cpp_b200.minigpt4_library import _ptr, choices_dfa
from test_reply_gpu import hash_vocab, ref_stop

pytestmark = pytest.mark.gpu

WEBUI = dict(temp=0.8, top_k=40, top_p=0.9)
PARAMS = {"greedy": dict(temp=0.0), "webui": WEBUI, "top_k-0-top_p-0.95": dict(temp=0.8, top_k=0, top_p=0.95),
          "mirostat-1": dict(temp=0.8, mirostat=1), "mirostat-2": dict(temp=0.8, mirostat=2)}
RECORD_BYTES = 168
TOP = 20
REFUSED = 8


@pytest.fixture(scope="module")
def files(tiny, mg, tmp_path_factory):
    d = tmp_path_factory.mktemp("logprobs")
    out = dict(tiny)
    for name, kw in (("hash", dict(n_embd=512, n_head=4, n_layer=2, n_vocab=1024, wtype="q4_1", vocab=hash_vocab(mg, 1024))),
                     ("w7b", dict(n_embd=4096, n_head=32, n_layer=2, n_vocab=32000, wtype="q4_1"))):
        out[name] = str(d / f"llama-{name}.bin")
        mg.write_llama_ggjt(out[name], mg.LlamaSpec(**kw))
    return out


# ---- numpy -------------------------------------------------------------------------------------------------------------------------
def np_lps(lg):
    """every id's log-probability: float64, rounded to float32"""
    z = lg.astype(np.float64)
    m = z.max()
    return ((z - m) - np.log(np.exp(z - m).sum())).astype(np.float32)


def np_rank(lg, t):
    return int(np.count_nonzero(lg > lg[t]) + np.count_nonzero(lg[:t] == lg[t]))


def np_top(lg, k):
    return np.lexsort((np.arange(lg.size), -lg))[:k]


def within_ulp(got, want):
    got, want = np.float64(got), np.float64(want)
    return abs(got - want) <= np.spacing(np.abs(np.float32(want)))


def bits(x):
    return np.asarray(x, np.float32).view(np.uint32)


def check_top(tid, tlp, lg, top_n, tag=""):
    """a record's top list against numpy over the logits it was taken from"""
    k = min(top_n, lg.size)
    want = np_top(lg, k)
    assert tid[:k].tolist() == want.tolist(), f"{tag} top ids"
    lps = np_lps(lg)
    for j in range(k):
        assert within_ulp(tlp[j], lps[want[j]]), f"{tag} top {j}: {tlp[j]!r} vs {lps[want[j]]!r}"
    assert (tid[k:] == -1).all() and np.isnan(tlp[k:]).all(), f"{tag} padding"


# ---- the kernel --------------------------------------------------------------------------------------------------------------------
def _rows(kind, rows, V, rng):
    if kind == "ties":
        return (rng.integers(0, 4, size=(rows, V)) * 0.5).astype(np.float32)
    lg = rng.normal(0, 3, size=(rows, V)).astype(np.float32)
    return lg + np.float32({"random": 0, "plus-1e4": 1e4, "minus-1e4": -1e4}[kind])


@pytest.mark.parametrize("V", [1, 7, 20, 21, 2048, 32000, 32001])
@pytest.mark.parametrize("kind", ["random", "ties", "plus-1e4", "minus-1e4"])
def test_kernel_against_numpy(ext, V, kind):
    rng = np.random.default_rng(V * 7 + len(kind))
    for rows in (1, 8, 64):
        lg = _rows(kind, rows, V, rng)
        ids = rng.integers(0, V, size=rows)
        if V > 1:
            ids[0] = int(np.argmax(lg[0]))   # a rank-0 row
        for top_n in sorted({0, 1, 5, 20, min(20, V + 3)}):
            lp, rk, tid, tlp, ms = ext.op_logprobs(lg, ids, top_n)
            assert ms > 0
            for r in range(rows):
                t = int(ids[r])
                want = np_lps(lg[r])[t]
                assert within_ulp(lp[r], want), (r, lp[r], want)
                assert rk[r] == np_rank(lg[r], t), r
                if top_n:
                    check_top(tid[r], tlp[r], lg[r], top_n, f"row {r} top_n {top_n}")
                    if rk[r] == 0:
                        assert bits(tlp[r, 0]) == bits(lp[r])
                        assert tid[r, 0] == t


# ---- groups ------------------------------------------------------------------------------------------------------------------------
def group(ext, path, n, n_ctx=128, seed0=11, prompt_seed=17):
    p = ext.llm_load(path, n_ctx=n_ctx, seed=seed0)
    ses = [p] + [ext.session_create(p, seed0 + i) for i in range(1, n)]
    rng = np.random.default_rng(prompt_seed)
    for i, c in enumerate(ses):
        ext.eval_tokens(c, [1] + rng.integers(3, 1000, size=2 + (i % 5)).tolist())
        ext.flush(c)
    return ses


def free(ext, ctxs):
    for c in ctxs[1:] + ctxs[:1]:
        ext.base.minigpt4_free(c)


def end_chat(lib, c, p):
    tok = ctypes.c_char_p()
    assert lib.library.minigpt4_end_chat(c.ptr, ctypes.byref(tok), 0, p.get("temp", 0.8), p.get("top_k", 40), p.get("top_p", 0.9), 1.0, 1.0,
                                         64, 1.1, 1.0, 1.0, p.get("mirostat", 0), 5.0, 1.0, 1) == 0
    return tok.value


def same_state(lib, ext, a, b, p):
    assert ext.n_past(a) == ext.n_past(b)
    assert np.array_equal(ext.logits(a), ext.logits(b))
    assert ext.greedy_id(a) == ext.greedy_id(b)
    assert end_chat(lib, a, p) == end_chat(lib, b, p)   # the generators and μ carried on
    assert np.array_equal(ext.logits(a), ext.logits(b))


def scorers_of(ext, ctxs):
    """one session per context holding a copy of its conversation, and the logits before the call"""
    sc = [ext.session_create(ctxs[0]) for _ in ctxs]
    for c, s in zip(ctxs, sc):
        ext.session_copy(c, [s])
    return sc, [ext.logits(c) for c in ctxs]


def check_against_score(ext, scorers, before, ids, recs, top_n, tag=""):
    """each context's records bit for bit against score_tokens over its fed ids, and the top lists against numpy over the same rows"""
    live = [i for i in range(len(ids)) if ids[i]]
    got = ext.score_tokens([scorers[i] for i in live], [ids[i] for i in live], keep=False, logits=True)
    for i, (lp_s, rk_s, rows) in zip(live, got):
        lp, rk, tid, tlp = recs[i]
        assert len(lp) == len(ids[i])
        assert np.array_equal(bits(lp), bits(lp_s)), f"{tag} context {i}: log-probabilities differ from score_tokens"
        assert np.array_equal(rk, rk_s), f"{tag} context {i}: ranks differ from score_tokens"
        for s, t in enumerate(ids[i]):
            lg = before[i] if s == 0 else rows[s - 1]
            if top_n:
                check_top(tid[s], tlp[s], lg, top_n, f"{tag} context {i} step {s}")
                hit = np.nonzero(tid[s] == t)[0]
                if hit.size:
                    assert hit[0] == rk[s] and bits(tlp[s, hit[0]]) == bits(lp[s]), f"{tag} context {i} step {s}"


# ---- generation unchanged ----------------------------------------------------------------------------------------------------------
def _twins(lib, ext, path, n, p, top_n, max_steps=12, stop=None, cons=None):
    a, b = group(ext, path, n), group(ext, path, n)
    handles = []
    if cons is not None:
        for g in (a, b):
            h = ext.constraint_create(g[0], *choices_dfa([b"cat", b"car", b"dog", b"no animal", b"yes"]))
            handles.append(h)
            for i in cons:
                ext.constraint_attach(g[i], h)
    ids_a, st_a, _ = ext.sample_until(a, max_steps, stop, **p)
    ids_b, st_b, recs, _ = ext.sample_until_logprobs(b, max_steps, stop, top_n, **p)
    assert ids_a == ids_b and st_a == st_b
    for x, y in zip(a, b):
        same_state(lib, ext, x, y, p if cons is None else dict(p, mirostat=0))
    for g in (a, b):
        free(ext, g)
    for h in handles:
        ext.constraint_free(h)
    return ids_b, recs


@pytest.mark.parametrize("wtype", ["q4_0", "q4_1", "q4_0-no-gemm", "q4_1-no-gemm", "q5_k", "q6_k", "f16", "mixed"])
def test_generation_unchanged_weight_types(lib, ext, files, wtype, monkeypatch):
    if wtype.endswith("-no-gemm"):
        monkeypatch.setenv("MINIGPT4_B200_NO_PREFILL_GEMM", "1")
    _twins(lib, ext, files[wtype.split("-")[0]], 3, WEBUI, 5)


@pytest.mark.parametrize("n", [1, 3, 9, 64])
@pytest.mark.parametrize("params", list(PARAMS))
def test_generation_unchanged_batches(lib, ext, files, n, params):
    ids, recs = _twins(lib, ext, files["q4_1"], n, PARAMS[params], TOP if n < 64 else 5)
    for i in range(n):
        assert len(recs[i][0]) == len(ids[i])
        if params == "greedy":
            assert (recs[i][1] == 0).all(), "the greedy id has rank 0"


@pytest.mark.parametrize("params", ["greedy", "webui"])
def test_generation_unchanged_constrained_mix(lib, ext, files, params):
    _twins(lib, ext, files["q4_1"], 9, PARAMS[params], 5, cons=[0, 2, 3, 7])


# ---- bit for bit against score_tokens ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 8, 9])
@pytest.mark.parametrize("params", ["greedy", "webui", "top_k-0-top_p-0.95", "mirostat-2"])
def test_records_equal_score_tokens(ext, files, n, params):
    ctxs = group(ext, files["q4_1"], n)
    sc, before = scorers_of(ext, ctxs)
    ids, _, recs, _ = ext.sample_until_logprobs(ctxs, 16, "", TOP, **PARAMS[params])
    check_against_score(ext, sc, before, ids, recs, TOP, params)
    free(ext, sc)
    free(ext, ctxs)


def test_records_of_a_constrained_context_are_unconstrained(ext, files):
    ctxs = group(ext, files["q4_1"], 3)
    h = ext.constraint_create(ctxs[0], *choices_dfa([b"cat", b"car", b"dog"]))
    ext.constraint_attach(ctxs[1], h)
    sc, before = scorers_of(ext, ctxs)
    ids, stopped, recs, _ = ext.sample_until_logprobs(ctxs, 12, "", 5, **WEBUI)
    assert stopped[1] and ids[1][-1] == 2
    check_against_score(ext, sc, before, ids, recs, 5, "constrained")
    free(ext, sc)
    free(ext, ctxs)
    ext.constraint_free(h)


# ---- stops ---------------------------------------------------------------------------------------------------------------------------
def _texts(ext, c, ids):
    return [ext.L.minigpt4_b200_token_text(c.ptr, int(t)) for t in ids]


def test_stops_at_different_steps(ext, files):
    # a host run without a stop text picks a one-byte stop that the 8 contexts reach at different steps
    probe = group(ext, files["hash"], 8)
    ids, _, _ = ext.sample_until(probe, 24, "", **WEBUI)
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
    ctxs = group(ext, files["hash"], 8)
    sc, before = scorers_of(ext, ctxs)
    L = ext.L
    n, max_steps, top_n = 8, 24, 5
    a_ids, a_lp, a_rk = (np.zeros(max_steps * n, dt) for dt in (np.int32, np.float32, np.int32))
    a_tid, a_tlp = np.zeros(max_steps * n * top_n, np.int32), np.zeros(max_steps * n * top_n, np.float32)
    n_out, stopped, ms = np.zeros(n, np.int32), np.zeros(n, np.int32), ctypes.c_float(0)
    assert L.minigpt4_b200_sample_until_logprobs(ctypes.cast(ext._ctx_array(ctxs), ctypes.c_void_p), n, max_steps, stop, WEBUI["temp"], WEBUI["top_k"],
                                                 WEBUI["top_p"], 1.0, 1.0, 0, 5.0, 1.0, top_n, _ptr(a_ids), _ptr(n_out), _ptr(stopped), _ptr(a_lp),
                                                 _ptr(a_rk), _ptr(a_tid), _ptr(a_tlp), ctypes.byref(ms)) == 0
    assert n_out.tolist() == [f + 1 for f in firsts] and stopped.all()
    ids, recs = [], []
    for i in range(n):
        e = np.arange(max_steps) * n + i
        k = int(n_out[i])
        ids.append(a_ids[e[:k]].tolist())
        recs.append((a_lp[e[:k]], a_rk[e[:k]], a_tid.reshape(-1, top_n)[e[:k]], a_tlp.reshape(-1, top_n)[e[:k]]))
        # every entry after the stop, including the steps the device ran past it: -1 / NaN
        after = e[k:]
        assert (a_ids[after] == -1).all() and (a_rk[after] == -1).all() and np.isnan(a_lp[after]).all()
        assert (a_tid.reshape(-1, top_n)[after] == -1).all() and np.isnan(a_tlp.reshape(-1, top_n)[after]).all()
    check_against_score(ext, sc, before, ids, recs, top_n, "stops")
    free(ext, sc)
    free(ext, ctxs)


def test_stop_text_across_two_calls(ext, files):
    # find a two-byte stop whose first byte ends the last token of a 3-step call and whose second byte starts the next call's first token
    for seed in range(40):
        probe = group(ext, files["hash"], 1, seed0=100 + seed)
        ids, _, _ = ext.sample_until(probe, 30, "", **WEBUI)
        tx = _texts(ext, probe[0], ids[0])
        free(ext, probe)
        hit = next((k for k in range(2, 29, 3) if tx[k] and tx[k + 1] and tx[k + 1] != b"##"
                    and ref_stop(tx, tx[k][-1:] + tx[k + 1][:1]) == k + 1), None)
        if hit is not None:
            break
    assert hit is not None, "no stop text across a call boundary in 40 seeds"
    stop = tx[hit][-1:] + tx[hit + 1][:1]
    one = group(ext, files["hash"], 1, seed0=100 + seed)
    ids1, st1, rec1, _ = ext.sample_until_logprobs(one, 30, stop, 5, **WEBUI)
    many = group(ext, files["hash"], 1, seed0=100 + seed)
    ids2, rec2, st2 = [], [], False
    while len(ids2) < 30 and not st2:
        got, st, rec, _ = ext.sample_until_logprobs(many, 3, stop, 5, **WEBUI)
        ids2 += got[0]; rec2.append(rec[0]); st2 = st[0]
    assert ids2 == ids1[0] and st2 == st1[0] and len(ids2) == hit + 2
    for j in range(4):   # logprob, rank, top ids, top log-probabilities: the bits of one call
        cat = np.concatenate([r[j] for r in rec2])
        assert np.array_equal(cat.view(np.uint32), rec1[0][j].view(np.uint32)), j
    free(ext, one)
    free(ext, many)


def test_max_steps_and_the_last_slot_of_n_ctx(ext, files):
    ctxs = group(ext, files["hash"], 2, n_ctx=64)
    sc, before = scorers_of(ext, ctxs)
    room = [64 - ext.n_past(c) for c in ctxs]
    ids, stopped, recs, _ = ext.sample_until_logprobs(ctxs, min(room), "", 5, **WEBUI)
    assert [len(x) for x in ids] == [min(room)] * 2 and stopped == [False, False]
    check_against_score(ext, sc, before, ids, recs, 5, "max_steps")
    full = ctxs[int(np.argmin(room))]
    assert ext.n_past(full) == 64
    lp = np.zeros(1, np.float32)
    buf = [np.zeros(1, np.int32) for _ in range(3)]
    assert ext.L.minigpt4_b200_sample_until_logprobs(ctypes.cast(ext._ctx_array([full]), ctypes.c_void_p), 1, 1, b"", 0.8, 40, 0.9, 1.0, 1.0, 0, 5.0,
                                                     1.0, 0, _ptr(buf[0]), _ptr(buf[1]), _ptr(buf[2]), _ptr(lp), None, None, None, None) == REFUSED
    free(ext, sc)
    free(ext, ctxs)


# ---- 7B width ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 16])
def test_7b_width(lib, ext, files, n):
    a = group(ext, files["w7b"], n, n_ctx=64)
    if n == 1:
        assert ext.stats(a[0]).decode_megakernel >= 6
    sc, before = scorers_of(ext, a)
    ids, stopped, recs, _ = ext.sample_until_logprobs(a, 8, "", TOP, **WEBUI)
    check_against_score(ext, sc, before, ids, recs, TOP, f"7b B{n}")
    b = group(ext, files["w7b"], n, n_ctx=64)
    assert ext.sample_until(b, 8, "", **WEBUI)[0] == ids
    for x, y in zip(a, b):
        same_state(lib, ext, x, y, WEBUI)
    for g in (sc, a, b):
        free(ext, g)


# ---- refusals and memory -------------------------------------------------------------------------------------------------------------
def _raw(ext, ctxs, top_n=5, mirostat=0):
    n, max_steps = len(ctxs), 4
    ids, lp, rk = np.zeros(max_steps * n, np.int32), np.zeros(max_steps * n, np.float32), np.zeros(max_steps * n, np.int32)
    tid, tlp = np.zeros(max_steps * n * max(1, top_n), np.int32), np.zeros(max_steps * n * max(1, top_n), np.float32)
    n_out, stopped = np.zeros(n, np.int32), np.zeros(n, np.int32)
    return ext.L.minigpt4_b200_sample_until_logprobs(ctypes.cast(ext._ctx_array(ctxs), ctypes.c_void_p), n, max_steps, None, 0.8, 40, 0.9, 1.0, 1.0,
                                                     mirostat, 5.0, 1.0, top_n, _ptr(ids), _ptr(n_out), _ptr(stopped), _ptr(lp), _ptr(rk), _ptr(tid),
                                                     _ptr(tlp), None)


@pytest.mark.parametrize("case", ["empty", "top_n-21", "mirostat-constrained"])
def test_refusals_change_nothing(ext, files, case):
    c = ext.llm_load(files["q4_1"], n_ctx=128)
    twin = ext.llm_load(files["q4_1"], n_ctx=128)
    h = None
    if case != "empty":
        for x in (c, twin):
            ext.eval_tokens(x, [1, 15, 27, 300])
            ext.flush(x)
            ext.eval_tokens(x, [41, 9, 77])   # queued
    if case == "mirostat-constrained":
        h = ext.constraint_create(c, *choices_dfa([b"cat", b"dog"]))
        ext.constraint_attach(c, h)
    launches = ext.stats(c).kernel_launches
    n_past = ext.n_past(c)
    code = _raw(ext, [c], top_n=21 if case == "top_n-21" else 5, mirostat=1 if case == "mirostat-constrained" else 0)
    assert code == REFUSED
    assert ext.stats(c).kernel_launches == launches, "device work before the refusal"
    assert ext.n_past(c) == n_past
    if case != "empty":
        assert np.array_equal(ext.logits(c), ext.logits(twin))   # the queue was still there, and evaluates as the twin's does
    if h is not None:
        ext.constraint_attach(c, None)
        ext.constraint_free(h)
    for x in (c, twin):
        ext.base.minigpt4_free(x)


def test_record_buffer_memory(ext, files):
    c = group(ext, files["q4_1"], 1, n_ctx=128)[0]
    ext.sample_until([c], 2, "", **WEBUI)               # the sampler and stop state
    o0 = ext.session_info(c)[1]
    ext.sample_until_logprobs([c], 2, "", 5, **WEBUI)
    o1 = ext.session_info(c)[1]
    assert o1 - o0 == RECORD_BYTES * 128
    ext.sample_until_logprobs([c], 2, "", 20, **WEBUI)
    ext.sample_until([c], 2, "", **WEBUI)
    assert ext.session_info(c)[1] == o1
    ext.base.minigpt4_free(c)


# ---- chat bot ------------------------------------------------------------------------------------------------------------------------
def test_chat_bot_generate_with_logprobs(mg, ext, files):
    import minigpt4_cpp_b200 as m
    bots = [m.MiniGPT4ChatBot(files["vision"], files["hash"]) for _ in range(3)]
    for bot in bots:
        bot.upload_image(mg.synth_image(3).reshape(1, 3, 224, 224))
    want = list(bots[0].generate_on_device("what is this?", limit=60, chunk=5))
    got = list(bots[1].generate_with_logprobs("what is this?", top_n=5, limit=60, chunk=5))
    assert [g[0] for g in got] == want and want
    # the same reply's ids on a third bot, scored from a copy of its conversation
    b = bots[2]
    b.is_image_chat = False
    b.library.minigpt4_begin_chat_image(b.ctx, b.embedding, "what is this?", b.n_threads)
    scorer = ext.session_create(b.ctx)
    ext.session_copy(b.ctx, [scorer])
    ids, stopped, _ = ext.sample_until([b.ctx], 60, None, **WEBUI)
    lps = ext.score_tokens([scorer], [ids[0]])[0][0]
    texts = [ext.L.minigpt4_b200_token_text(b.ctx.ptr, int(t)).decode("utf-8", errors="ignore") for t in ids[0]]
    keep = [k for k, t in enumerate(texts) if not (stopped[0] and k == len(texts) - 1) and not b.library.minigpt4_contains_eos_token(t)]
    assert [texts[k] for k in keep] == want
    assert [np.float32(g[1]).view(np.uint32) for g in got] == [lps[k].view(np.uint32) for k in keep]
    for _, lp, alts in got:
        assert len(alts) == 5 and all(alts[j][1] >= alts[j + 1][1] for j in range(4))
    ext.base.minigpt4_free(scorer)
    for bot in bots:
        bot.free()
