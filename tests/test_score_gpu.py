"""minigpt4_b200_score_tokens: the log-probability, rank and logits of every id of a known continuation, for 1..64 contexts of one group in
shared prompt passes.

Every row's logits must be the bits a context holds after evaluating its ids up to that row (a twin context fed the same ids, and the CPU
oracle); log-probabilities are checked against numpy in float64 to one float32 ulp, ranks exactly.  A batch must give each context what it
gets scored alone; keep = 0 must leave a context exactly as it was and keep = 1 exactly where eval_tokens + flush leaves it."""
import ctypes
import sys
from pathlib import Path

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parent.parent
N_CTX = 1200
PASS = 512     # LlamaDevice::kPrefillMax


def _ids(n_vocab, n, seed):
    return np.random.default_rng(seed).integers(3, n_vocab, size=n).astype(np.int32).tolist()


def _np_score(lg, t):
    """numpy's log-probability (float64, rounded to float32) and tie-ruled rank of id t under the float32 logits lg"""
    m = np.float64(lg.max())
    s = np.exp(lg.astype(np.float64) - m).sum()
    lp = np.float32((np.float64(lg[t]) - m) - np.log(s))
    rank = int(np.count_nonzero(lg > lg[t]) + np.count_nonzero(lg[:t] == lg[t]))
    return lp, rank


def _check_scores(lp, rk, before, rows, ids, tag=""):
    """lp / rk of ids against numpy over the logits before the call (None: n_past 0) and the call's logits rows"""
    for j, t in enumerate(ids):
        lg = before if j == 0 else rows[j - 1]
        if lg is None:
            assert np.isnan(lp[j]) and rk[j] == -1, f"{tag} entry 0 at n_past 0"
            continue
        want, wr = _np_score(lg, t)
        assert abs(np.float64(lp[j]) - np.float64(want)) <= np.spacing(np.abs(want)), f"{tag} entry {j}: {lp[j]!r} vs {want!r}"
        assert rk[j] == wr, f"{tag} entry {j}: rank {rk[j]} vs {wr}"


def _twin_rows(ext, path, prefix, ids, n_ctx=N_CTX):
    """a context of its own fed prefix, then ids one at a time: its logits before the ids and after each of them"""
    c = ext.llm_load(path, n_ctx=n_ctx)
    before = None
    if prefix:
        ext.eval_tokens(c, prefix); before = ext.logits(c)
    rows = []
    for t in ids:
        ext.eval_tokens(c, [t]); rows.append(ext.logits(c))
    ext.base.minigpt4_free(c)
    return before, rows


def _oracle_rows(orc, path, prefix, ids, n_ctx=N_CTX):
    e = orc.OracleEngine(None, path, n_ctx=n_ctx)
    if prefix:
        e.eval_tokens(prefix)
    rows = []
    for t in ids:
        e.eval_tokens([t]); rows.append(e.logits.copy())
    return rows


def _group(ext, path, n, n_ctx=N_CTX, seed=100):
    p = ext.llm_load(path, n_ctx=n_ctx, seed=seed)
    return [p] + [ext.session_create(p, seed=seed + 1 + i) for i in range(n - 1)]


def _free(ext, ctxs):
    for c in ctxs:
        ext.base.minigpt4_free(c)


# ---- every row's logits, log-probabilities and ranks ------------------------------------------------------------------------------------
@pytest.mark.parametrize("wt,gemm", [("q4_1", True), ("q4_1", False), ("q4_0", True), ("q4_0", False), ("q5_k", True), ("q6_k", True),
                                     ("f16", True), ("mixed", True)])
def test_every_row_is_bit_exact(ext, orc, tiny, monkeypatch, wt, gemm):
    """logits_out row j == a twin's logits after ids[:j + 1] == the oracle's; logprob / rank == numpy; on every tiny weight type, Q4 also
    on the per-op layers"""
    if not gemm:
        monkeypatch.setenv("MINIGPT4_B200_NO_PREFILL_GEMM", "1")
    path = tiny[wt]
    c = ext.llm_load(path, n_ctx=N_CTX)
    V = ext.L.minigpt4_b200_n_vocab(c.ptr)
    prefix, ids = _ids(V, 6, 1), _ids(V, 21, 2)
    ext.eval_tokens(c, prefix)
    (lp, rk, lg), = ext.score_tokens([c], [ids], logits=True)
    ext.base.minigpt4_free(c)
    before, rows = _twin_rows(ext, path, prefix, ids)
    orows = _oracle_rows(orc, path, prefix, ids)
    for j in range(len(ids)):
        assert np.array_equal(lg[j], rows[j]), f"{wt} row {j} vs twin"
        assert np.array_equal(lg[j], orows[j]), f"{wt} row {j} vs oracle"
    _check_scores(lp, rk, before, rows, ids, wt)


@pytest.mark.parametrize("spec", [dict(n_embd=4096, n_head=32, wtype="q4_1", n_vocab=32000), dict(n_embd=5120, n_head=40, wtype="q5_k", n_vocab=2048)],
                         ids=["7b-wide-q4_1", "13b-wide-q5_k"])
def test_full_width(ext, orc, mg, tmp_path, spec):
    """7B width with a 32000 vocabulary (tensor-core layers) and 13B width (per-op layers): == a twin on the megakernel and the oracle"""
    path = str(tmp_path / "llama-wide.bin")
    mg.write_llama_ggjt(path, mg.LlamaSpec(n_layer=1, **spec))
    V = spec["n_vocab"]
    prefix, ids = _ids(V, 5, 3), _ids(V, 24, 4)
    c = ext.llm_load(path, n_ctx=256)
    ext.eval_tokens(c, prefix)
    (lp, rk, lg), = ext.score_tokens([c], [ids], logits=True)
    ext.base.minigpt4_free(c)
    before, rows = _twin_rows(ext, path, prefix, ids, n_ctx=256)
    orows = _oracle_rows(orc, path, prefix, ids[:6], n_ctx=256)
    for j in range(len(ids)):
        assert np.array_equal(lg[j], rows[j]), f"row {j} vs twin"
    for j in range(len(orows)):
        assert np.array_equal(lg[j], orows[j]), f"row {j} vs oracle"
    _check_scores(lp, rk, before, rows, ids)


def _tied_model(mg, path, dup):
    """a tiny F16 model whose output rows dup[1:] are copies of row dup[0]: those ids always have equal logits"""
    spec = mg.LlamaSpec(n_vocab=1024, n_embd=512, n_head=4, n_layer=2, wtype="f16")
    mg.write_llama_ggjt(path, spec)
    raw = bytearray(Path(path).read_bytes())
    name = b"output.weight"
    p = raw.index(name) + len(name)
    p += (-p) % 32
    rb = mg.gg_row_bytes(mg.GG_NAMES["f16"], spec.n_embd)
    src = bytes(raw[p + dup[0] * rb:p + (dup[0] + 1) * rb])
    for r in dup[1:]:
        raw[p + r * rb:p + (r + 1) * rb] = src
    Path(path).write_bytes(bytes(raw))


def test_ranks_with_tied_logits(ext, mg, tmp_path):
    """ids whose logits are equal by construction: the rank counts the tied ids below the target, as numpy does"""
    path = str(tmp_path / "tied.bin")
    dup = [40, 7, 300, 1000]
    _tied_model(mg, path, dup)
    ids = [40, 7, 300, 1000, 5, 40, 1000, 7] * 3
    c = ext.llm_load(path, n_ctx=256)
    ext.eval_tokens(c, [1, 9, 11])
    before = ext.logits(c)
    assert before[40] == before[7] == before[300] == before[1000]
    (lp, rk, lg), = ext.score_tokens([c], [ids], logits=True)
    assert all(r[40] == r[7] == r[300] == r[1000] for r in lg)
    _check_scores(lp, rk, before, lg, ids, "tied")
    ext.base.minigpt4_free(c)


def test_first_entry_at_n_past_0_is_nan(ext, tiny):
    c = ext.llm_load(tiny["q4_1"], n_ctx=64)
    (lp, rk), = ext.score_tokens([c], [[1, 50, 60]])
    assert np.isnan(lp[0]) and rk[0] == -1
    assert np.all(np.isfinite(lp[1:])) and np.all(rk[1:] >= 0)
    assert ext.n_past(c) == 0
    ext.base.minigpt4_free(c)


# ---- sequence lengths and passes --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("m", [1, 7, 8, 9, 511, 512, 513, 1000])
def test_sequence_lengths(ext, tiny, m):
    """one context, m ids (up to two 512-row passes): every row == the twin's, scores == numpy"""
    path = tiny["q4_1"]
    c = ext.llm_load(path, n_ctx=N_CTX)
    prefix, ids = _ids(1024, 4, 10 + m), _ids(1024, m, 20 + m)
    ext.eval_tokens(c, prefix)
    (lp, rk, lg), = ext.score_tokens([c], [ids], logits=True)
    ext.base.minigpt4_free(c)
    before, rows = _twin_rows(ext, path, prefix, ids)
    for j in range(m):
        assert np.array_equal(lg[j], rows[j]), f"m {m} row {j}"
    _check_scores(lp, rk, before, rows, ids, f"m {m}")


def _alone(ext, path, prefixes, id_lists, queued=None, n_ctx=N_CTX):
    """each context scored on its own (a fresh context per prefix): [(lp, rk, logits)]"""
    out = []
    for i, (pr, ids) in enumerate(zip(prefixes, id_lists)):
        c = ext.llm_load(path, n_ctx=n_ctx)
        if pr: ext.eval_tokens(c, pr)
        if queued and queued[i] is not None: ext.eval_embd(c, queued[i])
        out.append(ext.score_tokens([c], [ids], logits=True)[0])
        ext.base.minigpt4_free(c)
    return out


@pytest.mark.parametrize("wt", ["q4_1", "q5_k"])
@pytest.mark.parametrize("n,lens", [(1, [700]), (2, [300, 400]), (3, [300, 400, 500]), (9, [1, 7, 8, 9, 100, 200, 300, 333, 60]),
                                    (64, [2 + (37 * i) % 29 for i in range(64)])],
                         ids=["n1-two-passes", "n2-split", "n3-three-passes", "n9", "n64"])
def test_batch_equals_alone(ext, tiny, wt, n, lens):
    """contexts at different positions, every third with queued embedding rows that the call flushes first: each context's results equal
    the same context scored alone; n_past unchanged (keep = 0)"""
    path = tiny[wt]
    rng = np.random.default_rng(30 + n)
    prefixes = [_ids(1024, 1 + (5 * i) % 17, 40 + i) for i in range(n)]
    queued = [rng.standard_normal((3 + i % 5, 512)).astype(np.float32) * 0.1 if i % 3 == 0 else None for i in range(n)]
    id_lists = [_ids(1024, k, 60 + i) for i, k in enumerate(lens)]
    ses = _group(ext, path, n)
    for c, pr, q in zip(ses, prefixes, queued):
        ext.eval_tokens(c, pr)
        if q is not None: ext.eval_embd(c, q)
    got = ext.score_tokens(ses, id_lists, logits=True)
    for c, pr, q in zip(ses, prefixes, queued):
        assert ext.n_past(c) == len(pr) + (0 if q is None else q.shape[0])
    _free(ext, ses)
    ref = _alone(ext, path, prefixes, id_lists, queued)
    for i, ((lp, rk, lg), (lp2, rk2, lg2)) in enumerate(zip(got, ref)):
        assert np.array_equal(lg, lg2), f"context {i}: logits"
        assert np.array_equal(lp, lp2) and np.array_equal(rk, rk2), f"context {i}: scores"


def test_image_chat_turn_then_answers(lib, ext, mg, tmp_path):
    """a queued image-chat turn (4096 wide, as the image rows are), then K candidate answers scored on one context with keep = 0: each
    equals the answer scored on a fresh context after the same turn"""
    import minigpt4_cpp_b200 as m
    path = str(tmp_path / "llama-7b-wide.bin")
    mg.write_llama_ggjt(path, mg.LlamaSpec(n_vocab=1024, n_embd=4096, n_head=32, n_layer=1, wtype="q4_1"))
    emb = np.random.default_rng(7).standard_normal((32, 4096)).astype(np.float32) * 0.05
    answers = [_ids(1024, k, 80 + k) for k in (3, 9, 17, 1)]

    def turn(c):
        lib.minigpt4_system_prompt(c)
        lib.minigpt4_begin_chat_image(c, m.MiniGPT4Embedding(emb.ctypes.data_as(ctypes.POINTER(ctypes.c_float)), emb.size), "what is this?")
        ext.eval_tokens(c, _ids(1024, 5, 6))

    c = ext.llm_load(path, n_ctx=512)
    turn(c)
    got = [ext.score_tokens([c], [a], logits=True)[0] for a in answers]
    for a, (lp, rk, lg) in zip(answers, got):
        r = ext.llm_load(path, n_ctx=512)
        turn(r)
        lp2, rk2, lg2 = ext.score_tokens([r], [a], logits=True)[0]
        assert np.array_equal(lg, lg2) and np.array_equal(lp, lp2) and np.array_equal(rk, rk2)
        ext.base.minigpt4_free(r)
    ext.base.minigpt4_free(c)


# ---- keep = 0 / keep = 1 -----------------------------------------------------------------------------------------------------------------
def _same(ext, a, b, hidden_rows, tag):
    assert ext.n_past(a) == ext.n_past(b), tag
    assert np.array_equal(ext.logits(a), ext.logits(b)), tag
    assert ext.greedy_id(a) == ext.greedy_id(b), tag
    assert np.array_equal(ext.hidden(a, hidden_rows), ext.hidden(b, hidden_rows)), tag


@pytest.mark.parametrize("path_kind", ["megakernel", "per-op", "wide-batch"])
def test_keep0_leaves_contexts_as_they_were(lib, ext, tiny, monkeypatch, path_kind):
    """after keep = 0 scoring a context equals a twin that never scored: state, then decode_chain, sample_steps and sample_until (ids,
    logits, generator) on the megakernel, the per-op graph and 16-wide batches"""
    if path_kind == "per-op":
        monkeypatch.setenv("MINIGPT4_B200_NO_MEGAKERNEL", "1")
    path = tiny["q4_1"]
    n = 16 if path_kind == "wide-batch" else 1
    prompts = [_ids(1024, 9 + i, 90 + i) for i in range(n)]
    a, b = _group(ext, path, n, seed=200), _group(ext, path, n, seed=200)
    if path_kind == "megakernel":
        assert ext.stats(a[0]).decode_megakernel >= 6
    if path_kind == "per-op":
        assert ext.stats(a[0]).decode_megakernel == 0
    for x, y, pr in zip(a, b, prompts):
        ext.eval_tokens(x, pr); ext.eval_tokens(y, pr); ext.flush(x); ext.flush(y)
    for k in (5, 600, 40):
        ext.score_tokens(a, [_ids(1024, k + i, 100 + k + i) for i in range(n)], logits=True)
    for i, (x, y) in enumerate(zip(a, b)):
        _same(ext, x, y, len(prompts[i]), f"{path_kind} context {i}")
    if n == 1:
        ia, _ = ext.decode_chain(a[0], 6); ib, _ = ext.decode_chain(b[0], 6)
        assert ia.tolist() == ib.tolist()
    else:
        for _ in range(3):
            assert ext.decode_batch(a).tolist() == ext.decode_batch(b).tolist()
    sa, _ = ext.sample_steps(a, 8); sb, _ = ext.sample_steps(b, 8)
    assert np.array_equal(sa, sb)
    ua = ext.sample_until(a, 12, stop=b""); ub = ext.sample_until(b, 12, stop=b"")
    assert ua[:2] == ub[:2]
    for x, y in zip(a, b):
        assert np.array_equal(ext.logits(x), ext.logits(y)) and ext.n_past(x) == ext.n_past(y)
    assert lib.minigpt4_end_chat(a[0]) == lib.minigpt4_end_chat(b[0])   # the generator
    _free(ext, a + b)


@pytest.mark.parametrize("m", [1, 37, 600])
def test_keep1_equals_eval_tokens(lib, ext, tiny, m):
    """keep = 1 leaves a context where eval_tokens + flush does: n_past, logits, greedy id, the hidden rows of its last pass, the following
    decode_chain ids, and a following sample_until stops at the same step"""
    path = tiny["q4_1"]
    prefix, ids = _ids(1024, 8, 5), _ids(1024, m, 6 + m)
    a, b, d = (ext.llm_load(path, n_ctx=N_CTX, seed=300) for _ in range(3))
    for c in (a, b, d):
        ext.eval_tokens(c, prefix)
        ext.sample_steps([c], 3)              # a reply tail that the call must clear as eval_tokens does
    ext.score_tokens([a], [ids], keep=True)
    ext.eval_tokens(b, ids); ext.flush(b)
    ext.eval_tokens(d, ids); ext.flush(d)
    last = m - (m - 1) // PASS * PASS
    assert ext.n_past(a) == ext.n_past(b) == 8 + 3 + m
    assert np.array_equal(ext.logits(a), ext.logits(b)) and ext.greedy_id(a) == ext.greedy_id(b)
    if m > 1:                                 # (a single id on its own goes through the decode step, which leaves no prompt rows)
        assert np.array_equal(ext.hidden(a, last), ext.hidden(b, last))
    probe, _ = ext.decode_chain(d, 6)
    stop = ext.L.minigpt4_b200_token_text(d.ptr, int(probe[3]))
    ia, _ = ext.decode_chain(a, 2); ib, _ = ext.decode_chain(b, 2)
    assert ia.tolist() == ib.tolist()
    ua = ext.sample_until([a], 16, stop=stop, temp=0.0); ub = ext.sample_until([b], 16, stop=stop, temp=0.0)
    assert ua[:2] == ub[:2]
    _free(ext, [a, b, d])


# ---- refusals -----------------------------------------------------------------------------------------------------------------------------
def test_refused_calls_change_nothing(ext, tiny):
    path = tiny["q4_1"]
    ses = _group(ext, path, 3, n_ctx=64)
    other = ext.llm_load(path, n_ctx=64)
    for i, c in enumerate(ses + [other]):
        ext.eval_tokens(c, _ids(1024, 4 + i, 120 + i))
    ext.eval_embd(ses[1], np.ones((3, 512), np.float32) * 0.01)   # queued: a refused call must not flush it
    before = [ext.n_past(c) for c in ses]
    L = ext.L
    arr = lambda cs: ctypes.cast(ext._ctx_array(cs), ctypes.c_void_p)
    p = lambda x: x.ctypes.data_as(ctypes.c_void_p)
    ids = np.full(200, 5, np.int32)
    lp, rk = np.zeros(200, np.float32), np.zeros(200, np.int32)

    def call(cs, lens, keep=0, ids=ids):
        lens = np.asarray(lens, np.int32)
        return L.minigpt4_b200_score_tokens(arr(cs), len(cs), p(ids), p(lens), keep, p(lp), p(rk), None)

    assert call(ses, [2, 2, 2], keep=2) == 8
    assert call(ses, [2, 2, -1]) == 8
    assert call(ses, [2, 0, 2]) == 8
    assert call(ses, [2, 70, 2]) == 8                            # n_past + n_ids > n_ctx
    assert call([ses[0], ses[1], ses[0]], [2, 2, 2]) == 8
    assert call([ses[0], other], [2, 2]) == 8
    bad = ids.copy(); bad[3] = 1024
    assert call(ses, [2, 2, 2], ids=bad) == 8
    bad[3] = -1
    assert call(ses, [2, 2, 2], ids=bad) == 8
    assert L.minigpt4_b200_score_tokens(arr(ses), 3, None, p(np.array([1, 1, 1], np.int32)), 0, p(lp), None, None) == 8
    assert L.minigpt4_b200_score_tokens(arr(ses), 3, p(ids), p(np.array([1, 1, 1], np.int32)), 0, None, None, None) == 8
    assert L.minigpt4_b200_score_tokens(arr(ses), 0, p(ids), p(np.array([1], np.int32)), 0, p(lp), None, None) == 8
    assert [ext.n_past(c) for c in ses] == before
    ref = ext.llm_load(path, n_ctx=64)
    ext.eval_tokens(ref, _ids(1024, 5, 121)); ext.eval_embd(ref, np.ones((3, 512), np.float32) * 0.01)
    got = ext.score_tokens(ses, [[5, 6], [7, 8, 9], [10]], logits=True)     # accepted now: the queue is still intact
    want = ext.score_tokens([ref], [[7, 8, 9]], logits=True)[0]
    assert all(np.array_equal(x, y) for x, y in zip(got[1], want))
    _free(ext, ses + [other, ref])


# ---- perplexity tool -------------------------------------------------------------------------------------------------------------------
def test_perplexity_tool(ext, tiny):
    """tools/perplexity.py == the perplexity numpy computes from logits_out over the same chunks"""
    sys.path.insert(0, str(ROOT / "tools"))
    import perplexity as ppl_tool
    path, n_ctx = tiny["q4_1"], 64
    parent = ext.llm_load(path, n_ctx=n_ctx)
    tokens = [1] + _ids(1024, 5 * n_ctx + 17, 140)
    got, n_chunks, n_tok = ppl_tool.perplexity(ext, parent, tokens, n_ctx)
    assert n_chunks == len(tokens) // n_ctx
    nll, count = 0.0, 0
    for ck in ppl_tool.chunks(tokens, n_ctx):
        _, _, lg = ext.score_tokens([parent], [ck], logits=True)[0]
        for j in range(n_ctx // 2 + 1, n_ctx):
            nll -= float(_np_score(lg[j - 1], ck[j])[0]); count += 1
    assert count == n_tok
    assert np.isclose(got, np.exp(nll / count), rtol=1e-6, atol=0), (got, np.exp(nll / count))
    ext.base.minigpt4_free(parent)
