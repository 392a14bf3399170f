"""Long contexts on the GPU: positions up to n_ctx - 1, against the CPU oracle bit for bit and against a float64 attention.

1. Kernel level (minigpt4_b200_op_llama_attention): attn_kernel (path 0) and attn_sessions_kernel (path 1) from position 0 to 32767 at
   n_ctx 32768, == the oracle's attention op bit for bit and the float64 attention of tests/test_long_context_host.py within 2e-3 of
   max|ref|; K / V rows above a row's position hold NaN / inf (the stale rows keep = 0 scoring and sample_until's overshoot leave there),
   scores whose differences leave the F16 range, probabilities in F16 subnormals, several heads, mixed positions in one launch.
2. The tiny models at n_ctx 2048: a ~1900-row prompt in one flush, then greedy decode to position 2047 through the megakernel and the
   per-op graph (decode_chain over the middle stretch), every row of a score_tokens call ending at position 2047, and every entry point
   refused at n_past = n_ctx without changing anything; decode_batch at B = 4 and 16 with contexts spread over 0 .. 2040, a batched prompt
   pass that fills a context to n_ctx, sample_until to the last slot; Q4_1 filled to n_ctx 4096.
3. 1-layer 4096-wide files at n_ctx 4096 .. 32768: the megakernel's plan (its attention scratch of 6 n_ctx bytes shares shared memory with
   the weight stream) or the per-op fallback, == the oracle; and 8 megakernel steps past position 2048 with 32 heads."""
import ctypes
import os
import time

import numpy as np
import pytest

from conftest import rel_err
from test_long_context_host import BAR, err_of, ref_attention
from test_wide13b_gpu import _load, _mega_plan, _smem_optin

pytestmark = pytest.mark.gpu

POSITIONS = [0, 1, 15, 16, 191, 192, 193, 383, 384, 1023, 2047, 4095, 8191, 16383]
STALE = (np.nan, np.inf, -np.inf)


# ---- 1. kernel level ------------------------------------------------------------------------------------------------------------------
def _cache(rng, n_ctx, n_head, valid, k_scale=1.0):
    """F16 K / V [n_ctx][n_head * 128]; rows from `valid` on hold NaN, +inf and -inf in turn"""
    E = 128 * n_head
    k = (k_scale * rng.standard_normal((n_ctx, E))).astype(np.float16)
    v = rng.standard_normal((n_ctx, E)).astype(np.float16)
    for i, x in enumerate(STALE):
        k[valid + i::3] = x
        v[valid + (i + 1) % 3::3] = x
    return k, v


def _check(ext, orc, q, k, v, pos, path):
    """the hook on `path` == the oracle op bit for bit, == float64 within BAR; returns the error against float64"""
    got = ext.op_llama_attention(q, k, v, pos if path else pos[0], path)
    want = orc.llama_attention(q, k, v, pos)
    assert np.isfinite(got).all()
    assert np.array_equal(got, want), f"path {path}, positions {pos}: {rel_err(got, want)}"
    err = err_of(got, ref_attention(q, k, v, pos))
    assert err < BAR, (path, pos, err)
    return err


@pytest.mark.parametrize("path", [0, 1])
@pytest.mark.parametrize("p", POSITIONS + [32767])
def test_attention_at_every_position_scale(ext, orc, path, p):
    """three consecutive rows ending at p (path 0: one launch at pos[0] + t) over 4 heads, stale rows right above p"""
    n_ctx = 32768 if p == 32767 else 16384
    rng = np.random.default_rng(p + 7 * path)
    pos = list(range(max(0, p - 2), p + 1))
    k, v = _cache(rng, n_ctx, 4, p + 1)
    q = (2.0 * rng.standard_normal((len(pos), 512))).astype(np.float32)
    err = _check(ext, orc, q, k, v, pos, path)
    print(f"path {path}, position {p}: {err:.2e} of max|ref|")


def test_sessions_kernel_mixed_positions_in_one_launch(ext, orc):
    """path 1: every position of POSITIONS (and repeats) as rows of one launch, in shuffled order, 4 heads"""
    rng = np.random.default_rng(11)
    pos = POSITIONS + [16383, 0, 192]
    rng.shuffle(pos)
    k, v = _cache(rng, 16384, 4, 16384)
    q = (4.0 * rng.standard_normal((len(pos), 512))).astype(np.float32)
    _check(ext, orc, q, k, v, pos, 1)
    k, v = _cache(rng, 16384, 4, 2048)   # stale rows above the furthest row's position
    pos = [p for p in pos if p < 2048]
    _check(ext, orc, q[:len(pos)], k, v, pos, 1)


@pytest.mark.parametrize("path", [0, 1])
def test_32_heads_at_n_ctx_4096(ext, orc, path):
    rng = np.random.default_rng(32 + path)
    k, v = _cache(rng, 4096, 32, 4096)
    pos = [4093, 4094, 4095] if path == 0 else [4095, 0, 2048, 191]
    q = rng.standard_normal((len(pos), 4096)).astype(np.float32)
    _check(ext, orc, q, k, v, pos, path)


@pytest.mark.parametrize("path", [0, 1])
def test_scores_beyond_the_f16_range(ext, orc, path):
    """|s - max| > 65504: the F16 argument of the exp table is -inf and P = 0 exactly; one key per head wins, on either side of a pass
    boundary and at the last key"""
    rng = np.random.default_rng(5)
    n_ctx, p = 4096, 4000
    k, v = _cache(rng, n_ctx, 4, p + 1)
    k[:p + 1] = np.where(rng.random((p + 1, 512)) < 0.5, -60000.0, 60000.0).astype(np.float16)
    q = np.zeros((1, 512), np.float32)
    for h, win in enumerate((191, 192, p, 0)):
        q[0, 128 * h:128 * h + 128] = np.sign(k[win, 128 * h:128 * h + 128].astype(np.float32)) * 1000.0
    got = ext.op_llama_attention(q, k, v, [p] if path else p, path)
    assert np.array_equal(got, orc.llama_attention(q, k, v, [p]))
    for h, win in enumerate((191, 192, p, 0)):
        assert np.array_equal(got[0, 128 * h:128 * h + 128], v[win, 128 * h:128 * h + 128].astype(np.float32)), h


@pytest.mark.parametrize("path", [0, 1])
@pytest.mark.parametrize("n_keys", [20000, 32768])
def test_subnormal_probabilities(ext, orc, path, n_keys):
    """long uniform (q = 0) and near-uniform rows: every P is a subnormal F16 (1 / n < 2^-14); the uniform row's output is the mean of V"""
    rng = np.random.default_rng(n_keys)
    k, v = _cache(rng, 32768, 2, n_keys)
    v[:n_keys] = (1.0 + 0.5 * rng.standard_normal((n_keys, 256))).astype(np.float16)
    q = np.zeros((2, 256), np.float32)
    q[1] = 1e-3 * rng.standard_normal(256)
    pos = [n_keys - 2, n_keys - 1]
    _check(ext, orc, q, k, v, pos, path)
    got = ext.op_llama_attention(q, k, v, pos if path else pos[0], path)
    assert err_of(got[:1], v[:n_keys - 1].astype(np.float64).mean(axis=0, keepdims=True)) < BAR


def test_hook_refuses_bad_arguments(ext):
    q = np.zeros((2, 128), np.float32)
    k = np.zeros((64, 128), np.float16)
    for pos, path in (([64, 0], 1), ([-1, 0], 1), ([63, 63], 0), ([0, 0], 2)):
        with pytest.raises(RuntimeError, match="FailedToAddString"):
            ext.op_llama_attention(q, k, k, pos if path != 0 else pos[0], path)


# ---- 2. whole model at n_ctx 2048 -------------------------------------------------------------------------------------------------
N_CTX = 2048
MEGA_TYPES = ("q4_0", "q4_1", "q5_k")


def _load_ctx(ext, path, monkeypatch, per_op: bool, n_ctx=N_CTX):
    if per_op: monkeypatch.setenv("MINIGPT4_B200_NO_MEGAKERNEL", "1")
    c = ext.llm_load(path, n_ctx=n_ctx)
    monkeypatch.delenv("MINIGPT4_B200_NO_MEGAKERNEL", raising=False)
    return c


def _prompt(V, E, n, seed):
    """n rows: ids, 32 embedding rows after the first third, ids (feed order)"""
    rng = np.random.default_rng(seed)
    a = (n - 32) // 3
    return rng.integers(3, V, size=a).tolist(), (0.05 * rng.standard_normal((32, E))).astype(np.float32), rng.integers(3, V, size=n - 32 - a).tolist()


def _feed(ext, c, pr):
    ext.eval_tokens(c, pr[0]); ext.eval_embd(c, pr[1]); ext.eval_tokens(c, pr[2])


def _feed_oracle(e, pr):
    e.eval_tokens(pr[0]); e.eval_embd(pr[1]); e.eval_tokens(pr[2])


def _refusals(ext, c, n_ctx):
    """at n_past = n_ctx every entry point that would add a row refuses, and nothing changes"""
    assert ext.n_past(c) == n_ctx
    before = ext.logits(c)
    t = int(np.argmax(before))
    calls = (lambda: ext.eval_tokens(c, [t]), lambda: ext.decode_chain(c, 1), lambda: ext.decode_batch([c]),
             lambda: ext.sample_steps([c], 1), lambda: ext.score_tokens([c], [[t]]), lambda: ext.sample_until([c], 1, ""))
    for i, call in enumerate(calls):
        with pytest.raises(RuntimeError):
            call()
        assert ext.n_past(c) == n_ctx, i
        assert np.array_equal(ext.logits(c), before), i


@pytest.mark.parametrize("wt", ["q4_1", "q4_0", "q5_k", "q6_k", "f16", "mixed"])
def test_one_context_to_the_last_slot(ext, orc, tiny, monkeypatch, wt):
    """1899 prompt rows in one flush (four 512-row passes), greedy decode to position 2047 on the default path (the megakernel on Q4_0 /
    Q4_1 / Q5_K) and the per-op graph: the oracle's logits after the prompt, after the first step and at every step of the last 48; the
    middle stretch through decode_chain == host-driven greedy; score_tokens over the last 48 ids == the oracle row for row; then every
    entry point refused at n_past = 2048"""
    path = tiny[wt]
    a, b = _load_ctx(ext, path, monkeypatch, False), _load_ctx(ext, path, monkeypatch, True)
    assert ext.stats(a).decode_megakernel == (6 if wt in MEGA_TYPES else 0) and ext.stats(b).decode_megakernel == 0
    e = orc.OracleEngine(None, path, n_ctx=N_CTX)
    pr = _prompt(e.n_vocab, e.n_embd, 1899, 3)
    for c in (a, b): _feed(ext, c, pr); ext.flush(c)
    _feed_oracle(e, pr)
    assert np.array_equal(ext.logits(a), e.logits) and np.array_equal(ext.logits(b), e.logits), "prompt"

    def step_both():
        t = ext.greedy_id(a)
        assert ext.greedy_id(b) == t
        ext.eval_tokens(a, [t]); ext.eval_tokens(b, [t])
        return t

    t = step_both(); e.eval_tokens([t])   # position 1899
    assert np.array_equal(ext.logits(a), e.logits) and np.array_equal(ext.logits(b), e.logits), "first step"
    mid = 2000 - ext.n_past(a)
    chain, _ = ext.decode_chain(a, mid)
    host = []
    for _ in range(mid):
        u = ext.greedy_id(b); host.append(u); ext.eval_tokens(b, [u])
    assert chain.tolist() == host and np.array_equal(ext.logits(a), ext.logits(b)), "decode_chain"
    e.eval_tokens(host)
    assert ext.n_past(a) == ext.n_past(b) == e.n_past == 2000
    tail, want = [], []
    for _ in range(N_CTX - 2000):   # positions 2000 .. 2047 on b, per step against the oracle
        u = ext.greedy_id(b)
        assert u == int(np.argmax(e.logits))
        ext.eval_tokens(b, [u]); e.eval_tokens([u]); tail.append(u); want.append(e.logits.copy())
        assert np.array_equal(ext.logits(b), e.logits), f"per-op graph at position {ext.n_past(b) - 1}: {rel_err(ext.logits(b), e.logits)}"
    (_, _, lg), = ext.score_tokens([a], [tail], logits=True)   # rows at positions 2000 .. 2047, a left at 2000
    for j in range(len(tail)):
        assert np.array_equal(lg[j], want[j]), f"score_tokens row at position {2000 + j}"
    for j, u in enumerate(tail):
        assert ext.greedy_id(a) == u
        ext.eval_tokens(a, [u])
        assert np.array_equal(ext.logits(a), want[j]), f"default path at position {2000 + j}"
    _refusals(ext, a, N_CTX); _refusals(ext, b, N_CTX)
    for c in (a, b): ext.base.minigpt4_free(c)


def _stepped_alone(ext, path, prompt_ids, steps):
    c = ext.llm_load(path, n_ctx=N_CTX)
    ext.eval_tokens(c, prompt_ids)
    ids, logits = [], []
    for _ in range(steps):
        t = ext.greedy_id(c); ids.append(t); ext.eval_tokens(c, [t]); logits.append(ext.logits(c))
    ext.base.minigpt4_free(c)
    return ids, logits


@pytest.mark.parametrize("wt,B", [("q4_0", 4), ("q4_1", 16)])
def test_decode_batch_at_long_positions(ext, orc, tiny, wt, B):
    """contexts at positions spread over 1 .. 2040 step together (B = 4: the sessions kernels; B = 16: the tensor-core layers) until the
    furthest reaches 2047: every column == its context stepped alone, two columns == the oracle"""
    path = tiny[wt]
    V = 1024
    starts = np.linspace(1, 2040, B).astype(int).tolist()
    rng = np.random.default_rng(B)
    prompts = [rng.integers(3, V, size=n).tolist() for n in starts]
    root = ext.llm_load(path, n_ctx=N_CTX)
    ctxs = [root] + [ext.session_create(root) for _ in range(B - 1)]
    for c, p in zip(ctxs, prompts): ext.eval_tokens(c, p)
    ext.flush_batch(ctxs)
    steps = N_CTX - max(starts)
    cols, logits = [], []
    for _ in range(steps):
        cols.append(ext.decode_batch(ctxs).tolist())
        logits.append([ext.logits(c) for c in ctxs])
    for i in range(B):
        ids, alone = _stepped_alone(ext, path, prompts[i], steps)
        assert [ids[0]] + [cols[s][i] for s in range(steps - 1)] == ids, i   # decode_batch feeds each context's greedy id, returns the next
        for s in range(steps):
            assert np.array_equal(logits[s][i], alone[s]), (i, s)
    for i in (0, B - 1):
        e = orc.OracleEngine(None, path, n_ctx=N_CTX)
        e.eval_tokens(prompts[i])
        for s in range(steps):
            e.eval_tokens([int(np.argmax(e.logits))])
            assert np.array_equal(logits[s][i], e.logits), (i, s)
    assert ext.n_past(ctxs[-1]) == N_CTX
    with pytest.raises(RuntimeError):
        ext.decode_batch(ctxs)
    for c in ctxs[::-1]: ext.base.minigpt4_free(c)


@pytest.mark.parametrize("wt", ["q4_1", "q5_k"])
def test_flush_batch_fills_a_context_to_n_ctx(ext, tiny, wt):
    """a batched prompt pass whose rows take one context from 0 to exactly n_ctx next to a short one: == each flushed alone"""
    path = tiny[wt]
    rng = np.random.default_rng(9)
    full, short = rng.integers(3, 1024, size=N_CTX).tolist(), rng.integers(3, 1024, size=37).tolist()
    root = ext.llm_load(path, n_ctx=N_CTX)
    other = ext.session_create(root)
    ext.eval_tokens(other, short[:5]); ext.flush(other)
    ext.eval_tokens(root, full); ext.eval_tokens(other, short[5:])
    ext.flush_batch([root, other])
    assert ext.n_past(root) == N_CTX
    for c, ids in ((root, full), (other, short)):
        twin = ext.llm_load(path, n_ctx=N_CTX)
        ext.eval_tokens(twin, ids); ext.flush(twin)
        assert np.array_equal(ext.logits(c), ext.logits(twin))
        ext.base.minigpt4_free(twin)
    _refusals(ext, root, N_CTX)
    ext.base.minigpt4_free(other); ext.base.minigpt4_free(root)


def test_sample_until_stops_at_the_last_slot(lib, ext, tiny):
    """sample_until with max_steps = n_ctx - n_past and a stop text that never occurs returns exactly at the end, with the ids of the end_chat
    loop on a twin; then nothing more is accepted"""
    path = tiny["q4_1"]
    ids = np.random.default_rng(4).integers(3, 1024, size=N_CTX - 40).tolist()
    a, b = ext.llm_load(path, n_ctx=N_CTX), ext.llm_load(path, n_ctx=N_CTX)
    for c in (a, b): ext.eval_tokens(c, ids)
    p = dict(temp=0.8, top_k=40, top_p=0.9)
    got, stopped, _ = ext.sample_until([a], 40, "", **p)
    assert len(got[0]) == 40 and not stopped[0] and ext.n_past(a) == N_CTX
    texts = []
    for _ in range(40):
        tok = ctypes.c_char_p()
        assert lib.library.minigpt4_end_chat(b.ptr, ctypes.byref(tok), 0, p["temp"], p["top_k"], p["top_p"], 1.0, 1.0, 64, 1.1, 1.0, 1.0, 0, 5.0, 1.0, 1) == 0
        texts.append(tok.value)
    assert [ext.L.minigpt4_b200_token_text(a.ptr, int(i)) for i in got[0]] == texts
    assert ext.n_past(b) == N_CTX and np.array_equal(ext.logits(a), ext.logits(b))
    _refusals(ext, a, N_CTX)
    for c in (a, b): ext.base.minigpt4_free(c)


def test_q4_1_filled_to_n_ctx_4096(ext, orc, tiny, monkeypatch):
    """the only model-level case past 2048: 4064 prompt rows, then 32 greedy steps to position 4095 on the megakernel and the per-op graph,
    the last 8 against the oracle (which follows the GPU's ids in one batch before that)"""
    path = tiny["q4_1"]
    a, b = _load_ctx(ext, path, monkeypatch, False, 4096), _load_ctx(ext, path, monkeypatch, True, 4096)
    assert ext.stats(a).decode_megakernel == 6
    e = orc.OracleEngine(None, path, n_ctx=4096)
    pr = _prompt(e.n_vocab, e.n_embd, 4064, 8)
    for c in (a, b): _feed(ext, c, pr); ext.flush(c)
    assert np.array_equal(ext.logits(a), ext.logits(b))
    fed = []
    for _ in range(24):
        t = ext.greedy_id(a)
        assert ext.greedy_id(b) == t
        ext.eval_tokens(a, [t]); ext.eval_tokens(b, [t]); fed.append(t)
    _feed_oracle(e, pr)
    e.eval_tokens(fed)
    assert np.array_equal(ext.logits(a), e.logits) and np.array_equal(ext.logits(b), e.logits)
    for _ in range(8):
        t = int(np.argmax(e.logits))
        assert ext.greedy_id(a) == t and ext.greedy_id(b) == t
        ext.eval_tokens(a, [t]); ext.eval_tokens(b, [t]); e.eval_tokens([t])
        assert np.array_equal(ext.logits(a), e.logits) and np.array_equal(ext.logits(b), e.logits), ext.n_past(a)
    _refusals(ext, a, 4096)
    for c in (a, b): ext.base.minigpt4_free(c)


# ---- 3. larger n_ctx at 7B width: the megakernel's plan and its fallback -------------------------------------------------------------------
WIDE = {"q4_1": 3, "q4_0": 2, "q5_k": 13}
N_CTXS = (4096, 8192, 16384, 24576, 32768)
# stream warps an H100 (227 KB opt-in shared memory per block) must get for a 4096-wide file (< 4: the per-op graph)
H100_W = {"q4_1": (14, 12, 8, 5, 1), "q4_0": (15, 13, 9, 6, 2), "q5_k": (13, 11, 8, 4, 1)}


@pytest.fixture(scope="module")
def wide7b(tmp_path_factory, mg):
    d = tmp_path_factory.mktemp("long7b")
    out = {}
    for wt in WIDE:
        out[wt] = str(d / f"llama-7b-{wt}.bin")
        mg.write_llama_ggjt(out[wt], mg.LlamaSpec(n_vocab=2048, n_embd=4096, n_head=32, n_layer=1, wtype=wt))
    yield out
    for p in out.values(): os.remove(p)


def test_sizing_rule_at_h100_numbers():
    for wt, ws in H100_W.items():
        assert tuple(_mega_plan(wt, 4096, 11008, n, 227 * 1024)[0] for n in N_CTXS) == ws, wt


@pytest.mark.parametrize("wt", list(WIDE))
def test_plan_and_fallback_up_to_n_ctx_32768(ext, orc, wide7b, capfd, wt):
    """at each n_ctx the load takes the megakernel with the planned (W, slot, act) when W >= 4 and the per-op graph otherwise; a 24-row
    prompt and 8 greedy steps == the oracle either way"""
    path = wide7b[wt]
    e = orc.OracleEngine(None, path, n_ctx=64)
    ids = np.random.default_rng(24).integers(3, 2048, size=24).tolist()
    want = [e.eval_tokens(ids).copy()]
    for _ in range(8):
        e.eval_tokens([int(np.argmax(e.logits))]); want.append(e.logits.copy())
    for i, n_ctx in enumerate(N_CTXS):
        c, plan = _load(ext, capfd, path, n_ctx)
        W, slot, act, _ = _mega_plan(wt, 4096, 11008, n_ctx, _smem_optin())
        if _smem_optin() == 227 * 1024:
            assert W == H100_W[wt][i], (n_ctx, W)
        if W >= 4:
            assert ext.stats(c).decode_megakernel == 6 and plan is not None and plan[1:4] == (W, slot, act), (n_ctx, plan)
        else:
            assert ext.stats(c).decode_megakernel == 0 and plan is None, n_ctx
        ext.eval_tokens(c, ids)
        assert np.array_equal(ext.logits(c), want[0]), n_ctx
        for s in range(8):
            t = ext.greedy_id(c)
            assert t == int(np.argmax(want[s])), (n_ctx, s)
            ext.eval_tokens(c, [t])
            assert np.array_equal(ext.logits(c), want[s + 1]), (n_ctx, s)
        ext.base.minigpt4_free(c)


def test_megakernel_past_2048_keys_with_32_heads(ext, orc, wide7b, capfd):
    """Q4_1 at n_ctx 4096 (W = 14 on an H100): 2100 prompt rows, then 8 megakernel steps at positions 2100 .. 2107 == the oracle"""
    path = wide7b["q4_1"]
    c, plan = _load(ext, capfd, path, 4096)
    assert ext.stats(c).decode_megakernel == 6 and plan is not None
    e = orc.OracleEngine(None, path, n_ctx=4096)
    ids = np.random.default_rng(2100).integers(3, 2048, size=2100).tolist()
    ext.eval_tokens(c, ids)
    t0 = time.time()
    e.eval_tokens(ids)
    print(f"oracle: 2100 rows at 4096 wide in {time.time() - t0:.1f} s")
    assert np.array_equal(ext.logits(c), e.logits)
    for s in range(8):
        t = ext.greedy_id(c)
        assert t == int(np.argmax(e.logits)), s
        ext.eval_tokens(c, [t]); e.eval_tokens([t])
        assert np.array_equal(ext.logits(c), e.logits), f"step {s}: {rel_err(ext.logits(c), e.logits)}"
    ext.base.minigpt4_free(c)
