"""Batched calls over 9..64 sessions of one group (LlamaDevice::kMaxBatch = 64): decode_batch, flush_batch, end_chat_batch, sample_steps,
sample_until and their mirostat forms.

Every session of a wide batch must end where the same work leaves it on a context of its own, bit for bit: each case compares with
np.array_equal against a separate context (stepped alone, or in the B <= 8 calls that are tested elsewhere), and against the CPU oracle
where noted.  Steps of more than 8 columns run their layers on the tensor-core prefill GEMM (Q4_0 / Q4_1 files, from the crossover
width on) or on the per-op matvecs; both paths are checked against each other at every width tested."""
import ctypes

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

N_CTX = 256
STEPS = 24
WIDTHS = (9, 16, 33, 64)
PASS = 512     # LlamaDevice::kPrefillMax
WEBUI = dict(temp=0.8, top_k=40, top_p=0.9)
TOPK0 = dict(temp=0.8, top_k=0, top_p=0.95)
M1 = dict(temp=0.8, mirostat=1, mirostat_tau=5.0, mirostat_eta=0.1)
M2 = dict(temp=0.8, mirostat=2, mirostat_tau=5.0, mirostat_eta=1.0)
UNUSED = (64, 1.1, 1.0, 1.0)   # repeat_last_n .. alpha_frequency of end_chat (never applied)


def _prompts(n_vocab, k, seed=5):
    rng = np.random.default_rng(seed)
    return [rng.integers(3, n_vocab, size=2 + (3 * i) % 29).tolist() for i in range(k)]   # 2..30 rows: every session at its own n_past


def _group(ext, path, n, n_ctx=N_CTX, seed=100):
    p = ext.llm_load(path, n_ctx=n_ctx, seed=seed)
    return [p] + [ext.session_create(p, seed=seed + 1 + i) for i in range(n - 1)]


def _free(ext, ctxs):
    for c in ctxs:
        ext.base.minigpt4_free(c)


def _alone(lib, ext, path, prompts, steps, n_ctx=N_CTX, mega=None):
    """each prompt on a context of its own (one context, reset between prompts), `steps` greedy steps: [(ids, logits after each step)]"""
    c = ext.llm_load(path, n_ctx=n_ctx)
    if mega is not None:
        assert (ext.stats(c).decode_megakernel >= 6) == mega
    out = []
    for pr in prompts:
        lib.minigpt4_reset_chat(c)
        ext.eval_tokens(c, pr)
        ids, lg = [], []
        for _ in range(steps):
            ext.eval_tokens(c, [ext.greedy_id(c)])
            ids.append(ext.greedy_id(c)); lg.append(ext.logits(c))
        out.append((ids, lg))
    ext.base.minigpt4_free(c)
    return out


def _oracle(orc, path, prompt, steps, n_ctx=N_CTX):
    e = orc.OracleEngine(None, path, n_ctx=n_ctx)
    e.eval_tokens(prompt)
    lg = []
    for _ in range(steps):
        e.end_chat_greedy(); lg.append(e.logits.copy())
    return lg


def _batched(ext, path, prompts, steps, n_ctx=N_CTX):
    ctxs = _group(ext, path, len(prompts), n_ctx)
    for c, pr in zip(ctxs, prompts):
        ext.eval_tokens(c, pr)                     # queued: the first decode_batch evaluates them in one batched flush
    ids, lg = [], []
    for _ in range(steps):
        ids.append(ext.decode_batch(ctxs).tolist())
        lg.append([ext.logits(c) for c in ctxs])
    for c, pr in zip(ctxs, prompts):
        assert ext.n_past(c) == len(pr) + steps
    _free(ext, ctxs)
    return ids, lg


def _check(ids, lg, refs, oracle=None):
    for i, (rid, rlg) in enumerate(refs):
        assert [s[i] for s in ids] == rid, f"session {i}"
        for k in range(len(rid)):
            assert np.array_equal(lg[k][i], rlg[k]), f"session {i} step {k}"
            if oracle is not None:
                assert np.array_equal(lg[k][i], oracle[i][k]), f"session {i} step {k} (oracle)"


# ---- decode steps ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("wt", ["q4_1", "q4_0", "q5_k", "q6_k", "f16", "mixed"])
def test_wide_steps_are_bit_exact(lib, ext, orc, tiny, wt):
    """B = 9, 16, 33, 64 sessions from prompts of different lengths, 24 greedy batched steps: every session's ids and logits after every
    step equal its own context's (and, for q4_1 and q5_k, the oracle's)"""
    path = tiny[wt]
    n_vocab = 1001 if wt == "mixed" else 1024
    prompts = _prompts(n_vocab, 64)
    refs = _alone(lib, ext, path, prompts, STEPS)
    oracle = [_oracle(orc, path, p, STEPS) for p in prompts] if wt in ("q4_1", "q5_k") else None
    for B in WIDTHS:
        ids, lg = _batched(ext, path, prompts[:B], STEPS)
        _check(ids, lg, refs[:B], oracle[:B] if oracle else None)


def test_tensor_core_and_per_op_layers_agree(ext, tiny, monkeypatch):
    """the tiny q4_1 file loaded with and without the tensor-core prefill GEMM: wide steps on both groups give equal ids and logits, so both
    sides of the crossover are covered whatever its width"""
    path = tiny["q4_1"]
    prompts = _prompts(1024, 64, seed=11)
    a = _group(ext, path, 64)
    monkeypatch.setenv("MINIGPT4_B200_NO_PREFILL_GEMM", "1")
    b = _group(ext, path, 64)
    monkeypatch.delenv("MINIGPT4_B200_NO_PREFILL_GEMM")
    assert ext.stats(a[0]).prefill_gemm and not ext.stats(b[0]).prefill_gemm
    for c, d, pr in zip(a, b, prompts):
        ext.eval_tokens(c, pr); ext.eval_tokens(d, pr)
    for B in WIDTHS:
        for k in range(4):
            ga, gb = ext.decode_batch(a[:B]), ext.decode_batch(b[:B])
            assert ga.tolist() == gb.tolist(), f"B {B} step {k}"
            for i in range(B):
                assert np.array_equal(ext.logits(a[i]), ext.logits(b[i])), f"B {B} step {k} session {i}"
    _free(ext, a + b)


@pytest.mark.parametrize("spec,B", [(dict(n_embd=4096, n_head=32, wtype="q4_1"), 64), (dict(n_embd=5120, n_head=40, wtype="q5_k"), 16)],
                         ids=["7b-wide-q4_1-B64", "13b-wide-q5_k-B16"])
def test_wide_steps_at_full_width(lib, ext, mg, tmp_path, spec, B):
    """7B width at B = 64 (tensor-core layers) and 13B width at B = 16 (per-op layers), 2 layers each: == contexts stepped alone on the
    megakernel"""
    path = str(tmp_path / "llama-wide.bin")
    mg.write_llama_ggjt(path, mg.LlamaSpec(n_vocab=2048, n_layer=2, **spec))
    prompts = _prompts(2048, B, seed=13)
    refs = _alone(lib, ext, path, prompts, 8, mega=True)
    ids, lg = _batched(ext, path, prompts, 8)
    _check(ids, lg, refs)


# ---- prompt passes --------------------------------------------------------------------------------------------------------------------
def _queue(rng, n_vocab, n_embd, n):
    """n queued rows: tokens, with a run of embedding rows in the middle from 5 rows on"""
    if n < 5:
        return [("t", rng.integers(3, n_vocab, size=n).tolist())]
    k = n // 3
    a = (n - k) // 2
    return [("t", rng.integers(3, n_vocab, size=a).tolist()), ("e", rng.standard_normal((k, n_embd)).astype(np.float32) * 0.1),
            ("t", rng.integers(3, n_vocab, size=n - k - a).tolist())]


def _put(ext, c, q):
    for kind, v in q:
        if kind == "t": ext.eval_tokens(c, v)
        else: ext.eval_embd(c, v)


def _last_pass(lens):
    """rows of each queue in the shared pass that evaluates its last row (queues concatenated in order, PASS rows per pass)"""
    out, pos = [], 0
    for n in lens:
        end = pos + n
        out.append(end - max(pos, (end - 1) // PASS * PASS))
        pos = end
    return out


@pytest.mark.parametrize("wt", ["q4_1", "q5_k"])
def test_flush_batch_over_64_sessions(lib, ext, tiny, wt):
    """64 queues of 2..28 rows in two 512-row passes: one session is split across them and more than 8 sessions end in each.  n_past,
    logits, greedy id and the hidden rows of the last pass equal each session's own flush; then 8 batched steps equal its own steps."""
    path = tiny[wt]
    rng = np.random.default_rng(60)
    lens = [2 + (5 * i) % 27 for i in range(64)]
    queues = [_queue(rng, 1024, 512, n) for n in lens]
    ends = np.cumsum(lens)
    assert any(e - n < PASS < e for e, n in zip(ends, lens)), "a session is split across the passes"
    assert np.sum(ends <= PASS) > 8 and np.sum(ends > PASS) > 8
    r = ext.llm_load(path, n_ctx=N_CTX)
    gemm = bool(ext.stats(r).prefill_gemm)
    refs = []
    for q, n in zip(queues, lens):
        lib.minigpt4_reset_chat(r)
        _put(ext, r, q)
        ext.flush(r)
        own = n if gemm else (n - 1) % 8 + 1    # rows of its own last pass: all of them on the tensor-core path, the last 8-row chunk per-op
        st = dict(n_past=ext.n_past(r), logits=ext.logits(r), greedy=ext.greedy_id(r), hidden=ext.hidden(r, own), ids=[], lg=[])
        for _ in range(8):
            ext.eval_tokens(r, [ext.greedy_id(r)])
            st["ids"].append(ext.greedy_id(r)); st["lg"].append(ext.logits(r))
        refs.append(st)
    ext.base.minigpt4_free(r)
    ses = _group(ext, path, 64)
    for c, q in zip(ses, queues):
        _put(ext, c, q)
    ext.flush_batch(ses)
    for i, (c, k, ref) in enumerate(zip(ses, _last_pass(lens), refs)):
        assert ext.n_past(c) == ref["n_past"], f"session {i}"
        assert np.array_equal(ext.logits(c), ref["logits"]), f"session {i}"
        assert ext.greedy_id(c) == ref["greedy"], f"session {i}"
        m = min(k, len(ref["hidden"]))
        assert np.array_equal(ext.hidden(c, k)[k - m:], ref["hidden"][len(ref["hidden"]) - m:]), f"session {i} (hidden)"
    for s in range(8):
        got = ext.decode_batch(ses).tolist()
        for i, (c, ref) in enumerate(zip(ses, refs)):
            assert got[i] == ref["ids"][s], f"session {i} step {s}"
            assert np.array_equal(ext.logits(c), ref["lg"][s]), f"session {i} step {s}"
    _free(ext, ses)


# ---- device sampling ------------------------------------------------------------------------------------------------------------------
def _args(p):
    return (p["temp"], p.get("top_k", 40), p.get("top_p", 0.9), 1.0, 1.0, *UNUSED, p.get("mirostat", 0), p.get("mirostat_tau", 5.0),
            p.get("mirostat_eta", 0.1), 1)


def _end_chat_batch(ext, ctxs, p):
    toks = (ctypes.c_char_p * len(ctxs))()
    assert ext.L.minigpt4_b200_end_chat_batch(ctypes.cast(ext._ctx_array(ctxs), ctypes.c_void_p), len(ctxs), ctypes.cast(toks, ctypes.c_void_p),
                                              *_args(p)) == 0
    return [toks[i] for i in range(len(ctxs))]


def _end_chat(lib, c, p):
    tok = ctypes.c_char_p()
    assert lib.library.minigpt4_end_chat(c.ptr, ctypes.byref(tok), 0, *_args(p)) == 0
    return tok.value


def _text(ext, c, i):
    return ext.L.minigpt4_b200_token_text(c.ptr, int(i))


def _sessions(ext, path, n, seed=17):
    rng = np.random.default_rng(seed + n)
    ses = _group(ext, path, n, seed=101)
    for c in ses:
        ext.eval_tokens(c, rng.integers(3, 1000, size=int(rng.integers(3, 30))).tolist())
    return ses


def _same_after(lib, ext, a, b, p):
    """n_past, logits and greedy id equal; then 4 end_chat calls on each side give equal tokens (generators and μ were written back)"""
    for i, (x, y) in enumerate(zip(a, b)):
        assert ext.n_past(x) == ext.n_past(y), f"session {i}"
        assert np.array_equal(ext.logits(x), ext.logits(y)), f"session {i}"
        assert ext.greedy_id(x) == ext.greedy_id(y), f"session {i}"
    for i, (x, y) in enumerate(zip(a, b)):
        assert [_end_chat(lib, x, p) for _ in range(4)] == [_end_chat(lib, y, p) for _ in range(4)], f"session {i}"


SAMPLE_CASES = [(24, WEBUI), (64, WEBUI), (24, TOPK0), (24, M1), (64, M1), (24, M2), (64, M2)]
SAMPLE_IDS = ["B24-webui", "B64-webui", "B24-top_k0", "B24-mirostat1", "B64-mirostat1", "B24-mirostat2", "B64-mirostat2"]


@pytest.mark.parametrize("n,p", SAMPLE_CASES, ids=SAMPLE_IDS)
def test_sample_steps_equal_end_chat_batch(lib, ext, tiny, n, p):
    path = tiny["q4_1"]
    a, b = _sessions(ext, path, n), _sessions(ext, path, n)
    ids, _ = ext.sample_steps(a, 24, **p)
    want = [_end_chat_batch(ext, b, p) for _ in range(24)]
    for i in range(n):
        assert [_text(ext, a[i], t) for t in ids[:, i]] == [w[i] for w in want], f"session {i}"
    _same_after(lib, ext, a, b, p)
    _free(ext, a + b)


def _hash_vocab(mg, n_vocab, seed=5):
    """make_vocab with the byte tokens 0x80..0xff and the last third of the pieces replaced by '#'-bearing ASCII pieces, so that random
    replies reach "###" within a few dozen tokens"""
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


@pytest.fixture(scope="module")
def hash_tiny(mg, tmp_path_factory):
    path = str(tmp_path_factory.mktemp("wide_reply") / "llama-hash-tiny.bin")
    mg.write_llama_ggjt(path, mg.LlamaSpec(n_embd=512, n_head=4, n_layer=2, n_vocab=1024, wtype="q4_1", vocab=_hash_vocab(mg, 1024)))
    return path


def _ref_replies(ext, ctxs, max_steps, p, stop=b"###"):
    """end_chat_batch over the sessions whose replies have not ended: (texts per session, stopped per session)"""
    n = len(ctxs)
    texts, chat, stopped, live = [[] for _ in range(n)], [b""] * n, [False] * n, list(range(n))
    for _ in range(max_steps):
        if not live:
            break
        nxt = []
        for i, t in zip(live, _end_chat_batch(ext, [ctxs[i] for i in live], p)):
            texts[i].append(t)
            chat[i] += t
            if t != b"##" and chat[i].endswith(stop):
                stopped[i] = True
            else:
                nxt.append(i)
        live = nxt
    return texts, stopped


@pytest.mark.parametrize("n,p", SAMPLE_CASES, ids=SAMPLE_IDS)
def test_sample_until_equals_end_chat_batch(lib, ext, hash_tiny, n, p):
    a, b = _sessions(ext, hash_tiny, n), _sessions(ext, hash_tiny, n)
    want, want_stopped = _ref_replies(ext, b, 40, p)
    got, stopped, _ = ext.sample_until(a, 40, None, **p)
    for i in range(n):
        assert [_text(ext, a[i], t) for t in got[i]] == want[i], f"session {i}"
        assert stopped[i] == want_stopped[i], f"session {i}"
    assert 0 < sum(stopped) < n      # replies end at different steps, and some run to max_steps
    _same_after(lib, ext, a, b, p)
    _free(ext, a + b)


# ---- mixing and refusals --------------------------------------------------------------------------------------------------------------
def test_mixing_paths(lib, ext, tiny):
    """wide steps interleaved with B <= 8 batches, single end_chat steps, decode_chain and queued prompt rows on the same 20 sessions == the
    same operations on separate contexts"""
    path = tiny["q4_1"]
    n = 20
    prompts = _prompts(1024, n, seed=21)
    ses = _group(ext, path, n)
    ref = [ext.llm_load(path, n_ctx=N_CTX) for _ in range(n)]
    for s, r, p in zip(ses, ref, prompts):
        ext.eval_tokens(s, p); ext.eval_tokens(r, p)

    def batch(idx, ids=None):
        got = ext.decode_batch([ses[i] for i in idx], ids)
        for j, i in enumerate(idx):
            ext.eval_tokens(ref[i], [ext.greedy_id(ref[i]) if ids is None or ids[j] < 0 else ids[j]])
            assert got[j] == ext.greedy_id(ref[i])

    def same():
        for i, (s, r) in enumerate(zip(ses, ref)):
            assert ext.n_past(s) == ext.n_past(r), f"session {i}"
            assert np.array_equal(ext.logits(s), ext.logits(r)), f"session {i}"

    everyone = list(range(n))
    batch(everyone); same()
    ext.eval_tokens(ses[3], [17, 18, 19]); ext.eval_tokens(ref[3], [17, 18, 19])     # queued rows, flushed by the next batch
    batch([3, 1, 0]); same()
    batch(everyone[::-1][:12]); same()
    for _ in range(3):                                                                # single steps through each session's own graph
        assert lib.minigpt4_end_chat(ses[1], temp=0.0) == lib.minigpt4_end_chat(ref[1], temp=0.0)
    a, _ = ext.decode_chain(ses[2], 5); b, _ = ext.decode_chain(ref[2], 5)
    assert a.tolist() == b.tolist(); same()
    batch(everyone, [40 + i if i % 3 else -1 for i in everyone]); same()
    batch([5, 6, 7, 8, 9, 10, 11, 12]); same()
    ext.eval_tokens(ses[0], list(range(50, 61))); ext.eval_tokens(ref[0], list(range(50, 61)))
    for _ in range(4):
        batch(everyone)
    same()
    a, _ = ext.decode_chain(ses[0], 4); b, _ = ext.decode_chain(ref[0], 4)
    assert a.tolist() == b.tolist(); same()
    _free(ext, ses + ref)


def _refused(ext, ctxs):
    """every batched entry point refuses ctxs"""
    arr = ctypes.cast(ext._ctx_array(ctxs), ctypes.c_void_p)
    n = len(ctxs)
    ids = np.full(n, -1, np.int32)
    out = np.zeros(4 * n, np.int32)
    n_out = np.zeros(n, np.int32)
    toks = (ctypes.c_char_p * n)()
    p = lambda x: x.ctypes.data_as(ctypes.c_void_p)
    L = ext.L
    assert L.minigpt4_b200_decode_batch(arr, n, p(ids), p(out)) == 8
    assert L.minigpt4_b200_end_chat_batch(arr, n, ctypes.cast(toks, ctypes.c_void_p), *_args(WEBUI)) == 8
    assert L.minigpt4_b200_sample_steps(arr, n, 2, 0.8, 40, 0.9, 1.0, 1.0, p(out), None) == 8
    assert L.minigpt4_b200_sample_until(arr, n, 2, None, 0.8, 40, 0.9, 1.0, 1.0, p(out), p(n_out), None, None) == 8
    assert L.minigpt4_b200_sample_steps_mirostat(arr, n, 2, 0.8, 2, 5.0, 1.0, p(out), None) == 8
    assert L.minigpt4_b200_sample_until_mirostat(arr, n, 2, None, 0.8, 2, 5.0, 1.0, p(out), p(n_out), None, None) == 8


def test_refused_wide_batches_change_nothing(lib, ext, tiny):
    """65 sessions; a full context inside a 40-wide batch; a duplicate at position 50: refused, and no session changes"""
    path = tiny["q4_1"]
    ses = _group(ext, path, 65, n_ctx=16)
    for i, c in enumerate(ses):
        ext.eval_tokens(c, [3 + i % 50, 4, 5]); ext.flush(c)
    ext.eval_tokens(ses[20], list(range(3, 16))); ext.flush(ses[20])                     # full: 16 of 16
    twin = ext.llm_load(path, n_ctx=16, seed=100)
    ext.eval_tokens(twin, [3, 4, 5]); ext.flush(twin)
    before = [(ext.n_past(c), ext.logits(c)) for c in ses]
    _refused(ext, ses)
    with pytest.raises(RuntimeError, match="FailedToAddString"):
        ext.flush_batch(ses)
    _refused(ext, ses[:40])
    dup = ses[:50] + [ses[7]]
    _refused(ext, dup)
    with pytest.raises(RuntimeError, match="FailedToAddString"):
        ext.flush_batch(dup)
    for i, (c, (n, lg)) in enumerate(zip(ses, before)):
        assert ext.n_past(c) == n and np.array_equal(ext.logits(c), lg), f"session {i}"
    assert _end_chat(lib, ses[0], WEBUI) == _end_chat(lib, twin, WEBUI)                  # the parent's generator was not touched
    ok = [c for i, c in enumerate(ses[:41]) if i != 20]                                 # still usable: 40 wide
    ext.decode_batch(ok)
    assert all(ext.n_past(c) == 4 for c in ok[1:])
    _free(ext, ses + [twin])
