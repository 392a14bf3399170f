"""minigpt4_b200_session_copy and the state save / restore entry points: a copied or restored conversation continues with the bits of the
conversation it came from.

The reference for a destination is a fresh session with the destination's seed that evaluated the source's whole history itself; the
source is checked against a twin that was never copied.  Every comparison is np.array_equal."""
import ctypes

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

N_CTX = 256
TYPES = ("q4_1", "q4_0", "q5_k", "q6_k", "f16", "mixed")
SAMPLE = dict(temp=0.8, top_k=40, top_p=0.9)


def _ids(n_vocab, n, seed):
    return np.random.default_rng(seed).integers(3, n_vocab, size=n).astype(np.int32).tolist()


def _rows(n_embd, n, seed):
    return (np.random.default_rng(seed).standard_normal((n, n_embd)) * 0.1).astype(np.float32)


def _history(ext, c, seed=1):
    """tokens (evaluated), one decode step, 32 embedding rows and tokens (queued): what an image-chat turn leaves"""
    V, E = ext.L.minigpt4_b200_n_vocab(c.ptr), ext.L.minigpt4_b200_n_embd(c.ptr)
    ext.eval_tokens(c, _ids(V, 9, seed)); ext.flush(c)
    ext.eval_tokens(c, _ids(V, 1, seed + 1))
    ext.eval_embd(c, _rows(E, 32, seed + 2))
    ext.eval_tokens(c, _ids(V, 6, seed + 3))


def _oracle_history(orc, path, ext, c, seed=1):
    V, E = ext.L.minigpt4_b200_n_vocab(c.ptr), ext.L.minigpt4_b200_n_embd(c.ptr)
    e = orc.OracleEngine(None, path, n_ctx=N_CTX)
    e.eval_tokens(_ids(V, 9, seed)); e.eval_tokens(_ids(V, 1, seed + 1)); e.eval_embd(_rows(E, 32, seed + 2)); e.eval_tokens(_ids(V, 6, seed + 3))
    return e


def _free(ext, ctxs):
    for c in ctxs:
        ext.base.minigpt4_free(c)


def _snap(ext, c):
    return ext.n_past(c), ext.logits(c), ext.greedy_id(c)


def _same(a, b):
    return a[0] == b[0] and np.array_equal(a[1], b[1]) and a[2] == b[2]


def _chunks(ctxs):
    return [ctxs[i:i + 64] for i in range(0, len(ctxs), 64)]   # a batched call takes 64 contexts


def _greedy_steps(ext, ctxs, steps):
    """decode_batch over ctxs (in calls of up to 64): ids [steps, n] and every column's logits after each step"""
    ids, lg = [], []
    for _ in range(steps):
        ids.append(np.concatenate([ext.decode_batch(b) for b in _chunks(ctxs)]))
        lg.append([ext.logits(c) for c in ctxs])
    return np.array(ids), lg


def _sample_steps(ext, ctxs, steps):
    return np.concatenate([ext.sample_steps(b, steps, **SAMPLE)[0] for b in _chunks(ctxs)], axis=1)


# ---- bit-exact continuation --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("wt,n", [(wt, n) for wt in TYPES for n in (1, 3)] + [("q4_1", 64)])
def test_copies_continue_bit_exact(ext, orc, tiny, wt, n):
    """copies of a mixed history into n destinations: greedy decode_batch over [src] + dsts, then sample_steps, equal each column's
    reference (and the oracle for the greedy steps); the source equals its twin; the copy is one launch and allocates nothing"""
    path = tiny[wt]
    p = ext.llm_load(path, n_ctx=N_CTX, seed=100)
    dsts = [ext.session_create(p, seed=101 + i) for i in range(n)]
    twin = ext.session_create(p, seed=100)
    refs = [ext.session_create(p, seed=101 + i) for i in range(n)]
    _history(ext, p)
    for c in [twin] + refs:
        _history(ext, c)
    for b in _chunks([twin] + refs):
        ext.flush_batch(b)
    if n == 1:   # otherwise the source's queued pieces are evaluated by the copy
        ext.flush(p)
    launches = ext.stats(p).kernel_launches
    info = [ext.session_info(c) for c in [p] + dsts]
    ext.session_copy(p, dsts)
    if n == 1:
        assert ext.stats(p).kernel_launches == launches + 1
    assert [ext.session_info(c) for c in [p] + dsts] == info
    want = _snap(ext, twin)
    assert _same(_snap(ext, p), want)
    for c in dsts:
        assert _same(_snap(ext, c), want)

    ids, lg = _greedy_steps(ext, [p] + dsts, 16)
    rids, rlg = _greedy_steps(ext, [twin] + refs, 16)
    assert np.array_equal(ids, rids)
    for s in range(16):
        for j in range(n + 1):
            assert np.array_equal(lg[s][j], rlg[s][j]), f"{wt} step {s} column {j}"
    e = _oracle_history(orc, path, ext, p)
    for s in range(16):   # the oracle feeds its greedy id; decode_batch returned the greedy id after each step
        t, _ = e.end_chat_greedy()
        assert t == (want[2] if s == 0 else ids[s - 1][0]), f"{wt} step {s} vs oracle"
        assert np.array_equal(lg[s][0], e.logits) and ids[s][0] == int(np.argmax(e.logits)), f"{wt} step {s} vs oracle"

    sids = _sample_steps(ext, [p] + dsts, 8)
    rsids = _sample_steps(ext, [twin] + refs, 8)
    assert np.array_equal(sids, rsids)
    for c, r in zip([p] + dsts, [twin] + refs):
        assert _same(_snap(ext, c), _snap(ext, r))
    if n >= 3:   # own samplers: the columns of different seeds drew different replies
        assert len({tuple(sids[:, j]) for j in range(n + 1)}) > 1
    _free(ext, [p, twin] + dsts + refs)


# ---- destinations that held a conversation of their own ----------------------------------------------------------------------------------
@pytest.mark.parametrize("wt", ["q4_1", "q5_k"])
def test_stale_destinations_behave_like_fresh_ones(ext, tiny, wt):
    """destinations with a longer conversation and queued pieces: after the copy, greedy steps and score_tokens equal fresh references"""
    p = ext.llm_load(tiny[wt], n_ctx=N_CTX, seed=7)
    V = ext.L.minigpt4_b200_n_vocab(p.ptr)
    dsts = [ext.session_create(p, seed=8 + i) for i in range(3)]
    refs = [ext.session_create(p, seed=8 + i) for i in range(3)]
    for i, c in enumerate(dsts):
        ext.eval_tokens(c, _ids(V, 150 + 10 * i, 50 + i)); ext.flush(c)
        ext.decode_batch([c])
        ext.eval_tokens(c, _ids(V, 7, 60 + i))   # queued: discarded by the copy
    _history(ext, p)
    for c in refs:
        _history(ext, c)
    ext.flush_batch(refs)
    ext.session_copy(p, dsts)
    for c, r in zip(dsts, refs):
        assert _same(_snap(ext, c), _snap(ext, r))
    cont = [_ids(V, 20, 70 + i) for i in range(3)]
    got = ext.score_tokens(dsts, cont, logits=True)
    want = ext.score_tokens(refs, cont, logits=True)
    for g, w in zip(got, want):
        assert all(np.array_equal(a, b, equal_nan=True) for a, b in zip(g, w))
    ids, lg = _greedy_steps(ext, dsts, 6)
    rids, rlg = _greedy_steps(ext, refs, 6)
    assert np.array_equal(ids, rids)
    assert all(np.array_equal(a, b) for s in range(6) for a, b in zip(lg[s], rlg[s]))
    _free(ext, [p] + dsts + refs)


# ---- the reply tail ----------------------------------------------------------------------------------------------------------------------
def test_reply_tail_spans_the_copy_point(ext, tiny):
    """a copy taken mid-reply stops its greedy sample_until where the source's reply would stop, with a stop text that began before the copy"""
    p = ext.llm_load(tiny["q4_1"], n_ctx=N_CTX, seed=3)
    twin = ext.session_create(p, seed=3)
    dsts = [ext.session_create(p, seed=30 + i) for i in range(2)]
    for c in (p, twin):
        _history(ext, c)
    full, _, _ = ext.sample_until([twin], 24, "", temp=0.0)
    texts = [ext.L.minigpt4_b200_token_text(twin.ptr, t) for t in full[0]]

    def first_stop(stop):
        chat = b""
        for i, t in enumerate(texts):
            chat += t
            if t != b"##" and chat.endswith(stop):
                return i
        return -1

    pick = None
    for k in range(3, 12):           # the copy after k steps, the stop text ends at step j >= k and starts before step k
        for j in range(k, k + 3):
            tail = b"".join(texts[:j + 1])
            after = len(b"".join(texts[k:j + 1]))
            for L in range(after + 1, min(32, len(tail)) + 1):
                if first_stop(tail[-L:]) == j:
                    pick = (k, j, tail[-L:])
                    break
            if pick:
                break
        if pick:
            break
    assert pick, texts
    k, j, stop = pick
    got, stopped, _ = ext.sample_until([p], k, stop, temp=0.0)
    assert got[0] == full[0][:k] and not stopped[0]
    ext.session_copy(p, dsts)
    got, stopped, _ = ext.sample_until(dsts + [p], 16, stop, temp=0.0)
    for i in range(3):
        assert got[i] == full[0][k:j + 1] and stopped[i], (i, k, j, stop)
    _free(ext, [p, twin] + dsts)


# ---- full width, full context ------------------------------------------------------------------------------------------------------------
def test_full_width_to_the_last_position(ext, mg, tmp_path):
    """4096-wide Q4_1 at n_ctx 2048: a 2040-row history copied into 3 sessions; 8 megakernel end_chat steps on one copy and 8 decode_batch
    steps of the others and the source equal the twin's steps; then every context refuses the step past n_ctx"""
    path = str(tmp_path / "llama-wide.bin")
    mg.write_llama_ggjt(path, mg.LlamaSpec(n_vocab=2048, n_embd=4096, n_head=32, n_layer=2, wtype="q4_1"))
    p = ext.llm_load(path, n_ctx=2048, seed=1)
    assert ext.stats(p).decode_megakernel > 0
    dsts = [ext.session_create(p, seed=2 + i) for i in range(3)]
    twin = ext.session_create(p, seed=1)
    hist = _ids(2048, 2040, 9)
    for c in (p, twin):
        ext.eval_tokens(c, hist)
    ext.session_copy(p, dsts)
    ref = []
    for _ in range(8):
        ext.base.minigpt4_end_chat(twin, temp=0.0)
        ref.append(_snap(ext, twin))
    for s in range(8):
        ext.base.minigpt4_end_chat(dsts[0], temp=0.0)
        assert _same(_snap(ext, dsts[0]), ref[s]), f"end_chat step {s}"
    batch = [p] + dsts[1:]
    for s in range(8):
        ids = ext.decode_batch(batch)
        assert all(t == ref[s][2] for t in ids)
        for c in batch:
            assert _same(_snap(ext, c), ref[s]), f"decode_batch step {s}"
    arr = ext._ctx_array([p])
    ids, out = (ctypes.c_int32 * 1)(-1), (ctypes.c_int32 * 1)()
    for c in [p, twin] + dsts:
        before = _snap(ext, c)
        assert before[0] == 2048
        arr[0] = c.ptr
        assert ext.L.minigpt4_b200_decode_batch(ctypes.cast(arr, ctypes.c_void_p), 1, ids, out) == 8
        assert _same(_snap(ext, c), before)
    _free(ext, [p, twin] + dsts)


# ---- refusals ----------------------------------------------------------------------------------------------------------------------------
def test_refused_copies_change_nothing(ext, tiny):
    p = ext.llm_load(tiny["q4_1"], n_ctx=N_CTX, seed=1)
    dsts = [ext.session_create(p, seed=2 + i) for i in range(3)]
    other = ext.llm_load(tiny["q4_1"], n_ctx=N_CTX, seed=9)
    V = ext.L.minigpt4_b200_n_vocab(p.ptr)
    for i, c in enumerate([p] + dsts + [other]):
        ext.eval_tokens(c, _ids(V, 20 + i, i)); ext.flush(c)
    snaps = [_snap(ext, c) for c in dsts + [other]]
    ext.eval_tokens(p, _ids(V, 5, 99))   # queued: a refused call must not evaluate it
    launches = ext.stats(p).kernel_launches
    L = ext.L

    def arr(cs):
        a = (ctypes.c_void_p * max(1, len(cs)))(*[None if c is None else c.ptr for c in cs])
        return ctypes.cast(a, ctypes.c_void_p)

    assert L.minigpt4_b200_session_copy(None, arr(dsts), 3) == 8
    assert L.minigpt4_b200_session_copy(p.ptr, None, 3) == 8
    assert L.minigpt4_b200_session_copy(p.ptr, arr(dsts), 0) == 8
    assert L.minigpt4_b200_session_copy(p.ptr, arr(dsts), 65) == 8
    assert L.minigpt4_b200_session_copy(p.ptr, arr([dsts[0], None, dsts[1]]), 3) == 8
    assert L.minigpt4_b200_session_copy(p.ptr, arr([dsts[0], dsts[1], dsts[0]]), 3) == 8
    assert L.minigpt4_b200_session_copy(p.ptr, arr([dsts[0], p]), 2) == 8
    assert L.minigpt4_b200_session_copy(p.ptr, arr([dsts[0], other]), 2) == 8
    assert ext.stats(p).kernel_launches == launches
    assert ext.n_past(p) == 20 + 5
    for c, before in zip(dsts + [other], snaps):
        assert _same(_snap(ext, c), before)
    # the state the refused calls left is the state a context that saw none of them has
    twin = ext.session_create(p, seed=1)
    ext.eval_tokens(twin, _ids(V, 20, 0)); ext.flush(twin); ext.eval_tokens(twin, _ids(V, 5, 99))
    assert _same(_snap(ext, p), _snap(ext, twin))
    _free(ext, [p, other, twin] + dsts)


# ---- save / restore ----------------------------------------------------------------------------------------------------------------------
def _continue(ext, c, steps=6):
    ids, lg = _greedy_steps(ext, [c], steps)
    return ids[:, 0], [x[0] for x in lg]


def test_state_round_trip(ext, tiny):
    """save at n_past 0, after a prompt and mid-reply; restore into a session of the group and into a second load at a larger n_ctx;
    both continue bit for bit, reply tail included"""
    path = tiny["q5_k"]
    p = ext.llm_load(path, n_ctx=N_CTX, seed=5)
    sess = ext.session_create(p, seed=6)
    big = ext.llm_load(path, n_ctx=2 * N_CTX, seed=7)
    V = ext.L.minigpt4_b200_n_vocab(p.ptr)
    E = ext.L.minigpt4_b200_n_embd(p.ptr)
    for stage in range(3):
        if stage == 1:
            _history(ext, p)   # queued rows: state_size counts them, state_save evaluates them
        if stage == 2:
            ext.sample_until([p], 5, "", temp=0.0)
        size = ext.L.minigpt4_b200_state_size(p.ptr)
        assert size == 144 + 4 * V + 4 * 2 * ext.n_past(p) * E
        data = ext.state_save(p)
        assert len(data) == size
        written = ctypes.c_longlong(0)
        buf = np.empty(size, np.uint8)
        assert ext.L.minigpt4_b200_state_save(p.ptr, buf.ctypes.data_as(ctypes.c_void_p), size, ctypes.byref(written)) == 0
        assert written.value == size and buf.tobytes() == data
        for c in (sess, big):
            ext.eval_tokens(c, _ids(V, 30, 11)); ext.flush(c)   # a conversation to replace
            ext.state_load(c, data)
            assert ext.n_past(c) == ext.n_past(p)
            assert ext.state_save(c) == data   # rows, logits, device state and reply tail, whatever the n_ctx
        if stage == 0:
            for c in (sess, big):
                assert ext.n_past(c) == 0
            ext.eval_tokens(p, _ids(V, 4, 12))
            for c in (sess, big):
                ext.eval_tokens(c, _ids(V, 4, 12))
        want = _snap(ext, p)
        for c in (sess, big):
            assert _same(_snap(ext, c), want), stage
        gi, gl = _continue(ext, p)
        for c in (sess, big):
            ci, cl = _continue(ext, c)
            assert np.array_equal(ci, gi) and all(np.array_equal(a, b) for a, b in zip(cl, gl)), stage
    _free(ext, [p, sess, big])


def test_state_restores_the_reply_tail(ext, tiny):
    """a state saved mid-reply carries the reply tail: the restored context's sample_until stops where the source's does"""
    path = tiny["q4_1"]
    p = ext.llm_load(path, n_ctx=N_CTX, seed=3)
    other = ext.llm_load(path, n_ctx=N_CTX, seed=4)
    _history(ext, p)
    ext.sample_until([p], 4, "", temp=0.0)
    data = ext.state_save(p)
    nxt, _, _ = ext.sample_until([p], 1, "", temp=0.0)
    first = ext.L.minigpt4_b200_token_text(p.ptr, nxt[0][0])
    n_tail = int(np.frombuffer(data[44:48], np.int32)[0])
    tail = data[48:48 + n_tail]
    assert 0 < n_tail <= 32 and first != b"##"
    stop = tail[-1:] + first   # begins before the save point: only the carried tail lets the first step end the reply
    ext.state_load(other, data)
    got, stopped, _ = ext.sample_until([other], 8, stop, temp=0.0)
    assert stopped[0] and got[0] == nxt[0]
    _free(ext, [p, other])


def test_state_refusals_change_nothing(ext, tiny, mg, tmp_path):
    seed_file = str(tmp_path / "llama-q4_1-seed9.bin")
    mg.write_llama_ggjt(seed_file, mg.LlamaSpec(n_vocab=1024, n_embd=512, n_head=4, n_layer=2, wtype="q4_1", seed=9))
    src = ext.llm_load(tiny["q4_1"], n_ctx=512, seed=1)
    V = ext.L.minigpt4_b200_n_vocab(src.ptr)
    ext.eval_tokens(src, _ids(V, 300, 1)); ext.flush(src)
    long_state = ext.state_save(src)
    short = ext.llm_load(tiny["q4_1"], n_ctx=N_CTX, seed=2)
    ext.eval_tokens(short, _ids(V, 17, 2)); ext.flush(short)
    short_state = ext.state_save(short)
    targets = {name: ext.llm_load(tiny[name], n_ctx=N_CTX, seed=3) for name in ("q4_1", "q4_0", "mixed")}
    targets["seed"] = ext.llm_load(seed_file, n_ctx=N_CTX, seed=3)
    for name, c in targets.items():
        v = ext.L.minigpt4_b200_n_vocab(c.ptr)
        ext.eval_tokens(c, _ids(v, 11, 3)); ext.flush(c)

    def bad(blob, **patch):
        b = bytearray(blob)
        for off, val in patch.values():
            b[off:off + len(val)] = val
        return bytes(b)

    i32 = lambda x: np.int32(x).tobytes()   # noqa: E731
    cases = [("q4_1", short_state[:-1]), ("q4_1", short_state + b"\0"), ("q4_1", short_state[:100]), ("q4_1", b""),
             ("q4_1", bad(short_state, m=(0, b"MG4STATF"))), ("q4_1", bad(short_state, v=(8, i32(2)))),
             ("q4_1", bad(short_state, d=(12, i32(1000)))), ("q4_1", bad(short_state, f=(32, bytes([short_state[32] ^ 1])))),
             ("q4_1", bad(short_state, s=(80, i32(16)))), ("q4_1", bad(short_state, r=(44, i32(33)))),
             ("q4_1", long_state),                                     # n_past 300 > n_ctx 256
             ("q4_0", short_state), ("mixed", short_state), ("seed", short_state)]
    for name, blob in cases:
        c = targets[name]
        before = _snap(ext, c)
        a = np.frombuffer(blob, np.uint8) if blob else np.zeros(1, np.uint8)
        assert ext.L.minigpt4_b200_state_load(c.ptr, a.ctypes.data_as(ctypes.c_void_p), len(blob)) == 8, name
        assert _same(_snap(ext, c), before), name
    assert ext.L.minigpt4_b200_state_load(targets["q4_1"].ptr, None, len(short_state)) == 8
    # a save into too small a buffer writes nothing and evaluates nothing
    ext.eval_tokens(short, _ids(V, 3, 5))
    size = ext.L.minigpt4_b200_state_size(short.ptr)
    buf = np.full(size, 0xAB, np.uint8)
    launches = ext.stats(short).kernel_launches
    assert ext.L.minigpt4_b200_state_save(short.ptr, buf.ctypes.data_as(ctypes.c_void_p), size - 1, None) == 8
    assert (buf == 0xAB).all() and ext.stats(short).kernel_launches == launches
    ext.state_load(targets["q4_1"], short_state)   # the same state is accepted
    assert ext.n_past(targets["q4_1"]) == 17
    _free(ext, [src, short] + list(targets.values()))
