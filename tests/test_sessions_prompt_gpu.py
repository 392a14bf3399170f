"""The batched prompt pass (minigpt4_b200_flush_batch, and the flush inside decode_batch / end_chat_batch): the queued rows of several
sessions share passes over the weights, and every session must end exactly where its own flush leaves it.

Each case compares with np.array_equal against independent single contexts loaded from the same file that flush on their own: n_past,
logits, greedy id, the hidden rows of the last pass, then greedy steps continued through decode_batch and, for the first session,
decode_chain and minigpt4_end_chat (which read the KV cache and the device state the flush left).  Where noted, also the CPU oracle."""
import ctypes

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

PASS = 512     # LlamaDevice::kPrefillMax
STEPS = 8


def _queue(n_vocab, n_embd, n, seed):
    """a queue of n rows: n == 1 is one embedding row (a lone token would take the decode step, not the queue); otherwise tokens with a
    run of embedding rows in the middle when n > 4"""
    rng = np.random.default_rng(seed)
    if n == 1:
        return [("e", rng.standard_normal((1, n_embd)).astype(np.float32) * 0.1)]
    if n <= 4:
        return [("t", rng.integers(3, n_vocab, size=n).tolist())]
    k = n // 3
    a = (n - k) // 2
    q = [("t", rng.integers(3, n_vocab, size=a).tolist()), ("e", rng.standard_normal((k, n_embd)).astype(np.float32) * 0.1)]
    if n - k - a == 1:
        q.append(("e", rng.standard_normal((1, n_embd)).astype(np.float32) * 0.1))
    else:
        q.append(("t", rng.integers(3, n_vocab, size=n - k - a).tolist()))
    return q


def _put(ext, c, q):
    for kind, v in q:
        if kind == "t": ext.eval_tokens(c, v)
        else: ext.eval_embd(c, v)


def _put_oracle(e, q):
    for kind, v in q:
        if kind == "t": e.eval_tokens(v)
        else: e.eval_embd(v)


def _rows(q):
    return sum(len(v) for _, v in q)


def _last_chunk(ext, c, n):
    """rows of the context's own last prefill pass: all of them on the tensor-core path, the last 8-row chunk on the per-op path"""
    return n if n == 1 or ext.stats(c).prefill_gemm else (n - 1) % 8 + 1


def _last_pass(lens):
    """rows of each queue in the shared pass that evaluates its last row (queues concatenated in order, PASS rows per pass)"""
    out, pos = [], 0
    for n in lens:
        end = pos + n
        out.append(end - max(pos, (end - 1) // PASS * PASS))
        pos = end
    return out


def _state(ext, c, nh):
    return dict(n_past=ext.n_past(c), logits=ext.logits(c), greedy=ext.greedy_id(c), hidden=ext.hidden(c, nh))


def _same_state(ext, c, got_hidden_rows, ref, tag):
    assert ext.n_past(c) == ref["n_past"], tag
    assert np.array_equal(ext.logits(c), ref["logits"]), tag
    assert ext.greedy_id(c) == ref["greedy"], tag
    k = min(got_hidden_rows, len(ref["hidden"]))
    assert np.array_equal(ext.hidden(c, got_hidden_rows)[got_hidden_rows - k:], ref["hidden"][len(ref["hidden"]) - k:]), tag + " (hidden)"


def _reference(lib, ext, path, q, n_ctx, first):
    """a context of its own: queue, own flush, STEPS greedy steps (+ decode_chain and end_chat for the first session)"""
    c = ext.llm_load(path, n_ctx=n_ctx)
    _put(ext, c, q)
    ext.flush(c)
    n = _rows(q)
    st = _state(ext, c, _last_chunk(ext, c, n))
    ids, lg = [], []
    for _ in range(STEPS):
        ext.eval_tokens(c, [ext.greedy_id(c)])
        ids.append(ext.greedy_id(c)); lg.append(ext.logits(c))
    if first:
        st["chain"] = ext.decode_chain(c, 3)[0].tolist()
        st["end_chat"] = [lib.minigpt4_end_chat(c, temp=0.0) for _ in range(2)]
        st["tail"] = ext.logits(c)
    st["ids"], st["lg"] = ids, lg
    ext.base.minigpt4_free(c)
    return st


def _group(ext, path, n, n_ctx):
    p = ext.llm_load(path, n_ctx=n_ctx)
    return [p] + [ext.session_create(p, seed=100 + i) for i in range(n - 1)]


def _run_batch(lib, ext, path, queues, refs, n_ctx):
    """queues on B sessions, one batched flush, then STEPS batched greedy steps; every session == its reference"""
    ses = _group(ext, path, len(queues), n_ctx)
    for c, q in zip(ses, queues):
        _put(ext, c, q)
    ext.flush_batch(ses)
    lens = [_rows(q) for q in queues]
    kb = _last_pass(lens) if len(ses) > 1 else [_last_chunk(ext, ses[0], lens[0])]
    for i, (c, r) in enumerate(zip(ses, refs)):
        _same_state(ext, c, kb[i], r, f"session {i} of {len(ses)}")
    for k in range(STEPS):
        got = ext.decode_batch(ses).tolist()
        for i, (c, r) in enumerate(zip(ses, refs)):
            assert got[i] == r["ids"][k], f"session {i} step {k}"
            assert np.array_equal(ext.logits(c), r["lg"][k]), f"session {i} step {k}"
    assert ext.decode_chain(ses[0], 3)[0].tolist() == refs[0]["chain"]
    assert [lib.minigpt4_end_chat(ses[0], temp=0.0) for _ in range(2)] == refs[0]["end_chat"]
    assert np.array_equal(ext.logits(ses[0]), refs[0]["tail"])
    for c in ses:
        ext.base.minigpt4_free(c)


def _refs(lib, ext, path, queues, n_ctx):
    return [_reference(lib, ext, path, q, n_ctx, i == 0) for i, q in enumerate(queues)]


def _oracle_logits(orc, path, q, n_ctx):
    e = orc.OracleEngine(None, path, n_ctx=n_ctx)
    _put_oracle(e, q)
    return e.logits.copy()


LENS = [9, 1, 8, 7, 23, 2, 16, 5]    # 8-row chunks mix sessions; the single-row queue lands at a chunk start and mid-chunk


@pytest.mark.parametrize("wt,gemm", [("q4_1", True), ("q4_0", True), ("q5_k", True), ("q6_k", True), ("f16", True), ("mixed", True),
                                     ("q4_1", False), ("q4_0", False)],
                         ids=["q4_1", "q4_0", "q5_k", "q6_k", "f16", "mixed", "q4_1-per-op", "q4_0-per-op"])
def test_flush_batch_is_bit_exact(lib, ext, orc, tiny, monkeypatch, wt, gemm):
    """B = 2, 3, 5, 8 sessions with queues of 1..23 rows: tensor-core path (Q4 files) or per-op path (the rest, and Q4 files loaded with
    MINIGPT4_B200_NO_PREFILL_GEMM); == single contexts and the oracle"""
    if not gemm: monkeypatch.setenv("MINIGPT4_B200_NO_PREFILL_GEMM", "1")
    path = tiny[wt]
    n_vocab = 1001 if wt == "mixed" else 1024
    queues = [_queue(n_vocab, 512, n, seed=50 + i) for i, n in enumerate(LENS)]
    refs = _refs(lib, ext, path, queues, 256)
    c = ext.llm_load(path, n_ctx=256)
    assert bool(ext.stats(c).prefill_gemm) == (gemm and wt in ("q4_1", "q4_0"))
    ext.base.minigpt4_free(c)
    for q, r in zip(queues, refs):
        assert np.array_equal(r["logits"], _oracle_logits(orc, path, q, 256))
    for B in (2, 3, 5, 8):
        _run_batch(lib, ext, path, queues[:B], refs[:B], 256)


@pytest.mark.parametrize("wt", ["q4_1", "q5_k"])
@pytest.mark.parametrize("lens", [[300, 300, 300], [20, 512, 37]], ids=["3x300", "20-512-37"])
def test_passes_split_a_session(lib, ext, orc, tiny, wt, lens):
    """more than 512 rows in all: a session's rows are split across two passes"""
    path = tiny[wt]
    queues = [[("t", np.random.default_rng(70 + i).integers(3, 1024, size=n).tolist())] for i, n in enumerate(lens)]
    refs = _refs(lib, ext, path, queues, 1024)
    for q, r in zip(queues, refs):
        assert np.array_equal(r["logits"], _oracle_logits(orc, path, q, 1024))
    _run_batch(lib, ext, path, queues, refs, 1024)


@pytest.mark.parametrize("wt", ["q4_1", "q5_k"])
def test_sessions_mid_conversation(lib, ext, tiny, wt):
    """sessions at different positions after own prompts, single steps and batched steps; empty queues in the batch; a batch of one"""
    path = tiny[wt]
    ses = _group(ext, path, 4, 256)
    ref = [ext.llm_load(path, n_ctx=256) for _ in range(4)]
    rng = np.random.default_rng(90)

    def same():
        for i, (s, r) in enumerate(zip(ses, ref)):
            assert ext.n_past(s) == ext.n_past(r), i
            assert np.array_equal(ext.logits(s), ext.logits(r)), i
            assert ext.greedy_id(s) == ext.greedy_id(r), i

    first = [rng.integers(3, 1024, size=n).tolist() for n in (5, 12, 30, 3)]
    for s, r, p in zip(ses, ref, first):
        ext.eval_tokens(s, p); ext.eval_tokens(r, p); ext.flush(s); ext.flush(r)
    for i in (1, 2):
        for c in (ses[i], ref[i]):
            ext.eval_tokens(c, [ext.greedy_id(c)])
    ext.decode_batch(ses)
    for r in ref:
        ext.eval_tokens(r, [ext.greedy_id(r)])
    same()
    more = {0: _queue(1024, 512, 11, 91), 1: _queue(1024, 512, 1, 92), 3: _queue(1024, 512, 40, 93)}   # session 2: empty queue
    for i, q in more.items():
        _put(ext, ses[i], q); _put(ext, ref[i], q)
    ext.flush_batch([ses[2], ses[3], ses[0], ses[1]])
    for r in ref:
        ext.flush(r)
    same()
    for i, n in ((3, 40), (0, 11)):
        nh = _last_chunk(ext, ref[i], n)
        kb = {3: 40, 0: 11}[i]          # order ses[3], ses[0], ses[1]: 40 + 11 + 1 rows, one pass
        k = min(nh, kb)
        assert np.array_equal(ext.hidden(ses[i], kb)[kb - k:], ext.hidden(ref[i], nh)[nh - k:])
    q = _queue(1024, 512, 17, 94)
    _put(ext, ses[1], q); _put(ext, ref[1], q)
    ext.flush_batch([ses[1]]); ext.flush(ref[1])
    same()
    for _ in range(4):
        ext.decode_batch(ses)
        for r in ref:
            ext.eval_tokens(r, [ext.greedy_id(r)])
    same()
    for c in ses + ref:
        ext.base.minigpt4_free(c)


@pytest.fixture(scope="module")
def wide(tmp_path_factory, mg):
    d = tmp_path_factory.mktemp("wide")
    paths = {}
    for name, spec in (("7b-q4_1", dict(n_embd=4096, n_head=32, wtype="q4_1")), ("13b-q5_k", dict(n_embd=5120, n_head=40, wtype="q5_k"))):
        paths[name] = str(d / f"llama-{name}.bin")
        mg.write_llama_ggjt(paths[name], mg.LlamaSpec(n_vocab=2048, n_layer=2, **spec))
    return paths


@pytest.mark.parametrize("explicit", [True, False], ids=["flush_batch", "end_chat_batch"])
def test_image_chat_turns(lib, ext, wide, explicit):
    """system prompt + begin_chat_image with different embeddings on 4 sessions, then one batched flush (explicit, or inside
    end_chat_batch) and greedy turns == the same turn on a context of its own"""
    import minigpt4_cpp_b200 as m
    path = wide["7b-q4_1"]
    rng = np.random.default_rng(110)
    embs = [rng.standard_normal((32, 4096)).astype(np.float32) * 0.05 for _ in range(4)]
    qs = ["what is this?", "describe it", "which color?", "how many are there in the picture?"]

    def turn(c, e, q):
        lib.minigpt4_system_prompt(c)
        lib.minigpt4_begin_chat_image(c, m.MiniGPT4Embedding(e.ctypes.data_as(ctypes.POINTER(ctypes.c_float)), e.size), q)

    ses = _group(ext, path, 4, 512)
    for c, e, q in zip(ses, embs, qs):
        turn(c, e, q)
    if explicit:
        ext.flush_batch(ses)
        got_lg = [ext.logits(c) for c in ses]
        got = [[lib.minigpt4_end_chat(c, temp=0.0) for _ in range(12)] for c in ses]
    else:
        steps = [ext.end_chat_batch(ses, temp=0.0) for _ in range(12)]
        got = [[s[i] for s in steps] for i in range(4)]
    r = ext.llm_load(path, n_ctx=512)
    for i, (e, q) in enumerate(zip(embs, qs)):
        lib.minigpt4_reset_chat(r)
        turn(r, e, q)
        ext.flush(r)
        if explicit:
            assert np.array_equal(got_lg[i], ext.logits(r)), f"session {i}"
        assert got[i] == [lib.minigpt4_end_chat(r, temp=0.0) for _ in range(12)], f"session {i}"
        assert ext.n_past(ses[i]) == ext.n_past(r)
    for c in ses + [r]:
        ext.base.minigpt4_free(c)


@pytest.mark.parametrize("name,lens", [("7b-q4_1", [32, 300, 45, 77, 120, 33, 260, 90]), ("13b-q5_k", [40, 9, 70, 23])],
                         ids=["7b-wide-q4_1-B8", "13b-wide-q5_k-B4"])
def test_flush_batch_at_full_width(lib, ext, wide, name, lens):
    """4096-wide Q4_1 on the tensor-core path (K split, qkv scatter at 4096; 957 rows = two passes) and 5120-wide Q5_K on the per-op path"""
    path = wide[name]
    E = 4096 if name.startswith("7b") else 5120
    queues = [_queue(2048, E, n, seed=130 + i) for i, n in enumerate(lens)]
    refs = _refs(lib, ext, path, queues, 512)
    _run_batch(lib, ext, path, queues, refs, 512)


def test_refused_batches_change_nothing(ext, tiny):
    path = tiny["q4_1"]
    ses = _group(ext, path, 3, 256)
    other = ext.llm_load(path, n_ctx=256)
    queues = [_queue(1024, 512, n, seed=150 + i) for i, n in enumerate((6, 13, 1, 9))]
    refs = []
    for q in queues:
        r = ext.llm_load(path, n_ctx=256)
        _put(ext, r, q); ext.flush(r)
        refs.append((ext.n_past(r), ext.logits(r)))
        ext.base.minigpt4_free(r)
    everyone = ses + [other]
    for c, q in zip(everyone, queues):
        _put(ext, c, q)
    for ctxs in ([], ses * 3, [ses[0], ses[1], ses[0]], [ses[0], other]):
        with pytest.raises(RuntimeError, match="FailedToAddString"):
            ext.flush_batch(ctxs)
    arr = (ctypes.c_void_p * 2)(ses[0].ptr, None)
    assert ext.L.minigpt4_b200_flush_batch(None, 2) == 8
    assert ext.L.minigpt4_b200_flush_batch(ctypes.cast(arr, ctypes.c_void_p), 2) == 8
    for c, (n, lg) in zip(everyone, refs):   # every queue is still pending: its own flush gives the expected bits
        assert ext.n_past(c) == n
        ext.flush(c)
        assert np.array_equal(ext.logits(c), lg)
    for c in everyone:
        ext.base.minigpt4_free(c)
