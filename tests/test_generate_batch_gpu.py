"""Per-conversation settings in one batched reply call on the GPU (minigpt4_b200_generate_batch; DESIGN.md §4.16):

- uniform settings are today's calls: generate_batch with the same settings for every context equals sample_until / _mirostat /
  _penalized / _logprobs on a twin group, with the same kernel launches, on every tiny weight type and at B = 1, 3, 9 and 64;
- mixed settings are each context alone: every context of a mixed call (samplers, penalties, constraints, stops, budgets 1..40) ends where
  it ends run alone with its own settings, at B = 3, 9, 16 and 64 and on a 4096-wide 32000-id model;
- a budget that ends at n_ctx while others run on leaves exactly the state its alone twin leaves;
- streaming over a changing membership, records of a mixed call against score_tokens, refusals and memory."""
import numpy as np
import pytest

from minigpt4_cpp_b200.minigpt4_library import GenParams, choices_dfa
from test_logprobs_gpu import check_against_score, files, free, group, scorers_of  # noqa: F401  (files: the module's model fixture)
from test_penalty_gpu import PEN, histories

pytestmark = pytest.mark.gpu

REFUSED = 8
WEBUI = dict(temp=0.8, top_k=40, top_p=0.9)
KINDS = {"greedy": dict(temp=0.0), "webui": WEBUI, "top_k-0-top_p-0.95": dict(temp=0.8, top_k=0, top_p=0.95),
         "mirostat-1": dict(temp=0.8, mirostat=1), "mirostat-2": dict(temp=0.8, mirostat=2)}
CHOICES = [b"cat", b"car", b"dog", b"no animal", b"yes"]


def bits(x):
    return np.asarray(x, np.float32).view(np.uint32)


def launches(ext, ctxs):
    return [ext.stats(c).kernel_launches for c in ctxs]


def end_state(lib, ext, c, p, constrained=False):
    """n_past, logits bits, greedy id, the constraint state, then one further end_chat draw (generator and μ) and its logits"""
    from test_logprobs_gpu import end_chat
    out = [ext.n_past(c), bits(ext.logits(c)).tobytes(), ext.greedy_id(c), ext.constraint_state(c) if constrained else None]
    out.append(end_chat(lib, c, p))
    out.append(bits(ext.logits(c)).tobytes())
    return out


def single_call(ext, ctxs, g: GenParams, logprobs=False, top_n=0):
    """the existing call that g's settings select, on ctxs"""
    p = dict(temp=g.temp, top_k=g.top_k, top_p=g.top_p, tfs_z=g.tfs_z, typical_p=g.typical_p, mirostat=g.mirostat, mirostat_tau=g.mirostat_tau,
             mirostat_eta=g.mirostat_eta)
    neutral = g.repeat_penalty == 1.0 and g.alpha_presence == 0.0 and g.alpha_frequency == 0.0 or g.repeat_last_n == 0
    if logprobs:
        ids, st, recs, _ = ext.sample_until_logprobs(ctxs, g.max_steps, g.stop, top_n, **p)
        return ids, st, recs
    if not neutral:
        ids, st, _ = ext.sample_until_penalized(ctxs, g.max_steps, g.stop, [g.last_ids] * len(ctxs), g.repeat_last_n, g.repeat_penalty,
                                                g.alpha_presence, g.alpha_frequency, g.penalize_nl, **p)
        return ids, st, None
    ids, st, _ = ext.sample_until(ctxs, g.max_steps, g.stop, **p)
    return ids, st, None


# ---- uniform settings ------------------------------------------------------------------------------------------------------------------
UNIFORM = dict(KINDS, **{"penalized": dict(WEBUI, **PEN, last_ids=[5, 13, 7, 5]), "records": dict(WEBUI)})


def _uniform(lib, ext, path, n, kind):
    kw = dict(UNIFORM[kind])
    g = GenParams(max_steps=12, stop="", **kw)
    a, b = group(ext, path, n), group(ext, path, n)
    rec = kind == "records"
    l0 = launches(ext, a + b)
    got = ext.generate_batch(a, [g] * n, top_n=5 if rec else 0, logprobs=rec)
    want = single_call(ext, b, g, logprobs=rec, top_n=5)
    l1 = launches(ext, a + b)
    assert got[0] == want[0] and got[1] == want[1]
    if rec:
        for x, y in zip(got[2], want[2]):
            for u, v in zip(x, y):
                assert np.array_equal(np.asarray(u).view(np.uint32), np.asarray(v).view(np.uint32))
    assert [y - x for x, y in zip(l0[:n], l1[:n])] == [y - x for x, y in zip(l0[n:], l1[n:])], "the same kernel launches"
    p = dict(temp=g.temp, top_k=g.top_k, top_p=g.top_p, mirostat=g.mirostat)
    for x, y in zip(a, b):
        assert end_state(lib, ext, x, p) == end_state(lib, ext, y, p)
    free(ext, a)
    free(ext, b)


@pytest.mark.parametrize("n", [1, 3, 9, 64])
@pytest.mark.parametrize("kind", list(UNIFORM))
def test_uniform_is_the_single_call(lib, ext, files, n, kind):
    _uniform(lib, ext, files["q4_1"], n, kind)


@pytest.mark.parametrize("wtype", ["q4_0", "q4_1", "q4_0-no-gemm", "q5_k", "q6_k", "f16", "mixed"])
def test_uniform_weight_types(lib, ext, files, wtype, monkeypatch):
    if wtype.endswith("-no-gemm"):
        monkeypatch.setenv("MINIGPT4_B200_NO_PREFILL_GEMM", "1")
    for kind in ("webui", "mirostat-2"):
        _uniform(lib, ext, files[wtype.split("-")[0]], 3, kind)


# ---- mixed settings --------------------------------------------------------------------------------------------------------------------
def pool(n, seed=5):
    """context i's settings and whether it is constrained: every kind, penalised greedy / mirostat, constrained chain / greedy, the stops
    NULL, "", "a" and a multi-byte one, budgets 1 .. 40"""
    rng = np.random.default_rng(seed)
    kinds = list(KINDS) + ["pen-greedy", "pen-mirostat", "pen-webui", "cons-webui", "cons-greedy"]
    stops = [None, "", "a", "ét"]
    out = []
    for i in range(n):
        k = kinds[i % len(kinds)]
        base = k.split("-", 1)[1] if k.startswith(("pen-", "cons-")) else k
        kw = dict(KINDS["mirostat-2" if base == "mirostat" else base])
        if k.startswith("pen-"):
            kw.update(PEN, last_ids=histories(3, seed=i)[i % 2])
        budget = 1 if i == 1 else int(rng.integers(2, 41))
        out.append((GenParams(max_steps=budget, stop=stops[(i // 2) % len(stops)], **kw), k.startswith("cons-")))
    return out


def _attach(ext, ctxs, flags):
    handles = []
    if any(flags):
        h = ext.constraint_create(ctxs[0], *choices_dfa(CHOICES))
        handles.append(h)
        for c, f in zip(ctxs, flags):
            if f:
                ext.constraint_attach(c, h)
    return handles


def _mixed(lib, ext, path, n, grouped=False):
    settings = pool(n)
    params, flags = [g for g, _ in settings], [f for _, f in settings]
    a, b = group(ext, path, n), group(ext, path, n)
    ha, hb = _attach(ext, a, flags), _attach(ext, b, flags)
    ids, stopped, _ = ext.generate_batch(a, params)
    for i in range(n):
        assert 1 <= len(ids[i]) <= params[i].max_steps
    if grouped:   # one single-settings call per distinct setting, over the contexts that have it
        groups = {}
        for i, (g, f) in enumerate(settings):
            groups.setdefault((repr(g), f), []).append(i)
        twin_ids, twin_st = [None] * n, [None] * n
        for members in groups.values():
            x, s, _ = single_call(ext, [b[i] for i in members], params[members[0]])
            for j, i in enumerate(members):
                twin_ids[i], twin_st[i] = x[j], s[j]
    else:         # each context alone, through the single call its settings select
        twin_ids, twin_st = [], []
        for i in range(n):
            x, s, _ = single_call(ext, [b[i]], params[i])
            twin_ids.append(x[0])
            twin_st.append(s[0])
    for i in range(n):
        assert ids[i] == twin_ids[i] and stopped[i] == twin_st[i], f"context {i}"
        p = dict(temp=params[i].temp, top_k=params[i].top_k, top_p=params[i].top_p, mirostat=0 if flags[i] else params[i].mirostat)
        assert end_state(lib, ext, a[i], p, flags[i]) == end_state(lib, ext, b[i], p, flags[i]), f"context {i}"
    # the reply tails: both continue alike
    more_a, _, _ = ext.sample_until(a, 8, None, temp=0.0)
    more_b, _, _ = ext.sample_until(b, 8, None, temp=0.0)
    assert more_a == more_b
    for g in (a, b):
        free(ext, g)
    for h in ha + hb:
        ext.constraint_free(h)


@pytest.mark.parametrize("n", [3, 9, 16, 64])
def test_mixed_is_each_alone(lib, ext, files, n):
    _mixed(lib, ext, files["q4_1"], n)


@pytest.mark.parametrize("n", [3, 9, 16, 64])
def test_mixed_is_grouped_single_calls(lib, ext, files, n):
    _mixed(lib, ext, files["q4_1"], n, grouped=True)


def test_mixed_wide_model(lib, ext, files):
    _mixed(lib, ext, files["w7b"], 9)


# ---- budgets at the edge of the context ------------------------------------------------------------------------------------------------
def _edge_group(ext, path, n, n_ctx):
    g = group(ext, path, n, n_ctx=n_ctx)
    fill = n_ctx - 4 - ext.n_past(g[0])
    ext.eval_tokens(g[0], (np.arange(fill) % 900 + 3).tolist())
    ext.flush(g[0])
    return g


@pytest.mark.parametrize("n", [3, 16])
def test_budget_ends_at_n_ctx(lib, ext, files, n):
    n_ctx = 96
    a, b = _edge_group(ext, files["q4_1"], n, n_ctx), _edge_group(ext, files["q4_1"], n, n_ctx)
    assert ext.n_past(a[0]) == n_ctx - 4
    params = [GenParams(max_steps=4, stop="", **WEBUI)] + [GenParams(max_steps=60, stop="", **(WEBUI if i % 2 else dict(temp=0.0)))
                                                           for i in range(1, n)]
    ids, stopped, _ = ext.generate_batch(a, params)
    assert len(ids[0]) == 4 and not stopped[0] and ext.n_past(a[0]) == n_ctx
    assert all(len(x) == 60 for x in ids[1:])
    twin = [ext.generate_batch([b[i]], [params[i]])[0][0] for i in range(n)]
    assert ids == twin
    assert ext.state_save(a[0]) == ext.state_save(b[0]), "K / V rows, logits and state of the full context"
    for i in range(1, n):
        assert ext.state_save(a[i]) == ext.state_save(b[i]), f"context {i}"
    # the others continue alike: a scored continuation (keep 0) and one more draw
    got = ext.score_tokens(a[1:], [[5, 6, 7]] * (n - 1))
    want = ext.score_tokens(b[1:], [[5, 6, 7]] * (n - 1))
    for (x, _), (y, _) in zip(got, want):
        assert np.array_equal(bits(x), bits(y))
    for x, y in zip(a[1:], b[1:]):
        assert end_state(lib, ext, x, WEBUI) == end_state(lib, ext, y, WEBUI)
    for g in (a, b):
        free(ext, g)


def test_budget_refusals_are_per_context(lib, ext, files):
    n_ctx = 96
    g = _edge_group(ext, files["q4_1"], 3, n_ctx)
    before = [(ext.n_past(c), bits(ext.logits(c)).tobytes()) for c in g]
    with pytest.raises(Exception):
        ext.generate_batch(g, [GenParams(max_steps=5)] + [GenParams(max_steps=4)] * 2)
    assert [(ext.n_past(c), bits(ext.logits(c)).tobytes()) for c in g] == before
    # a budget that fits is taken although another context's longer one would not fit in it
    ids, _, _ = ext.generate_batch(g, [GenParams(max_steps=4, stop="")] + [GenParams(max_steps=50, stop="")] * 2)
    assert [len(x) for x in ids] == [4, 50, 50]
    free(ext, g)


# ---- streaming -------------------------------------------------------------------------------------------------------------------------
def test_streaming_over_changing_membership(lib, ext, files):
    n = 6
    settings = [GenParams(max_steps=40, stop="", **KINDS["webui"]), GenParams(max_steps=40, stop="", **KINDS["mirostat-1"]),
                GenParams(max_steps=40, stop="", temp=0.0), GenParams(max_steps=40, stop="", **dict(WEBUI, **PEN)),
                GenParams(max_steps=40, stop="###", **KINDS["top_k-0-top_p-0.95"]), GenParams(max_steps=40, stop="a", **KINDS["mirostat-2"])]
    a, b = group(ext, files["hash"], n), group(ext, files["hash"], n)
    want = [ext.generate_batch([b[i]], [settings[i]])[0][0] for i in range(n)]
    got = [[] for _ in range(n)]
    done = [False] * n
    live = [0, 1, 2]   # 3, 4, 5 join one per chunk
    joining = [3, 4, 5]
    while live:
        chunk = []
        for i in live:
            g = settings[i]
            left = g.max_steps - len(got[i])
            extra = dict(last_ids=list(g.last_ids or []) + got[i]) if g.repeat_penalty != 1.0 else {}
            chunk.append(GenParams(**dict(vars(g), max_steps=min(16, left), **extra)))
        ids, stopped, _ = ext.generate_batch([a[i] for i in live], chunk)
        for i, x, s in zip(list(live), ids, stopped):
            got[i] += x
            done[i] = s or len(got[i]) == settings[i].max_steps
        live = [i for i in live if not done[i]] + joining[:1]
        joining = joining[1:]
    assert got == want
    for g in (a, b):
        free(ext, g)


# ---- records ---------------------------------------------------------------------------------------------------------------------------
def test_records_of_a_mixed_call(lib, ext, files):
    n = 9
    params = [g for g, f in pool(n) if not f] + [GenParams(max_steps=9, stop="", **dict(WEBUI, **PEN))]
    params = params[:n]
    a = group(ext, files["q4_1"], n)
    scorers, before = scorers_of(ext, a)
    ids, _, recs, _ = ext.generate_batch(a, params, top_n=5, logprobs=True)
    check_against_score(ext, scorers, before, ids, recs, 5)
    free(ext, scorers)
    free(ext, a)


# ---- refusals and memory ---------------------------------------------------------------------------------------------------------------
def test_refusals_in_context_5_of_9(lib, ext, files):
    n = 9
    g = group(ext, files["q4_1"], n)
    V = ext.L.minigpt4_b200_n_vocab(g[0].ptr)
    ext.eval_tokens(g[2], [5, 6, 7])   # queued rows stay queued
    h = ext.constraint_create(g[0], *choices_dfa(CHOICES))
    ext.constraint_attach(g[5], h)
    snap = [(ext.L.minigpt4_b200_n_past(c.ptr), ext.stats(c).kernel_launches) for c in g]
    ok = GenParams(max_steps=4)
    bad = [dict(max_steps=0), dict(max_steps=200), dict(stop="x" * 33), dict(mirostat=3), dict(mirostat=-1), dict(mirostat=1),
           dict(repeat_last_n=-1, repeat_penalty=1.1), dict(repeat_penalty=0.0), dict(repeat_penalty=float("nan")),
           dict(alpha_presence=float("inf")), dict(penalize_nl=2), dict(repeat_penalty=1.1, last_ids=[V + 5]), dict(last_ids=[-1])]
    for kw in bad:
        params = [ok] * n
        params[5] = GenParams(**dict(vars(ok), **kw))
        with pytest.raises(Exception):
            ext.generate_batch(g, params)
    for top_n in (-1, 21):
        with pytest.raises(Exception):
            ext.generate_batch(g, [ok] * n, top_n=top_n, logprobs=True)
    arr, _keep = ext.gen_params_c([ok] * n)
    arr[5].size = 72
    import ctypes
    ids, n_out = np.zeros((4, n), np.int32), np.zeros(n, np.int32)
    assert ext.L.minigpt4_b200_generate_batch(ctypes.cast(ext._ctx_array(g), ctypes.c_void_p), n, ctypes.cast(arr, ctypes.c_void_p), 0,
                                              ids.ctypes.data_as(ctypes.c_void_p), n_out.ctypes.data_as(ctypes.c_void_p), None, None, None, None,
                                              None, None) == REFUSED
    assert ext.L.minigpt4_b200_generate_batch(ctypes.cast(ext._ctx_array(g), ctypes.c_void_p), n, None, 0, ids.ctypes.data_as(ctypes.c_void_p),
                                              n_out.ctypes.data_as(ctypes.c_void_p), None, None, None, None, None, None) == REFUSED
    # an empty conversation with records
    e = ext.session_create(g[0], 99)
    with pytest.raises(Exception):
        ext.generate_batch(g[:5] + [e], [ok] * 6, logprobs=True)
    assert [(ext.L.minigpt4_b200_n_past(c.ptr), ext.stats(c).kernel_launches) for c in g] == snap, "nothing ran"
    ext.base.minigpt4_free(e)
    ext.constraint_attach(g[5], None)
    ext.constraint_free(h)
    free(ext, g)


def test_memory_follows_the_scratch_rules(lib, ext, files):
    n = 4
    a, b = group(ext, files["w7b"], n), group(ext, files["w7b"], n)
    params = [GenParams(max_steps=6, **WEBUI), GenParams(max_steps=6, **dict(WEBUI, **PEN)), GenParams(max_steps=3, temp=0.0),
              GenParams(max_steps=6, mirostat=2)]
    ext.generate_batch(a, params)
    for i in range(n):
        ext.generate_batch([b[i]], [params[i]])
    assert [ext.session_info(c)[1] for c in a] == [ext.session_info(c)[1] for c in b]
    owned = [ext.session_info(c)[1] for c in a]
    assert owned[1] > owned[0] and owned[0] == owned[2] == owned[3], "only the penalised context holds penalty scratch"
    for g in (a, b):
        free(ext, g)


def test_gen_params_defaults_reproduce_sample_until(lib, ext, files):
    n = 3
    a, b = group(ext, files["q4_1"], n), group(ext, files["q4_1"], n)
    assert ext.generate_batch(a, [GenParams(max_steps=10)] * n)[:2] == ext.sample_until(b, 10)[:2]
    for x, y in zip(a, b):
        assert end_state(lib, ext, x, WEBUI) == end_state(lib, ext, y, WEBUI)
    for g in (a, b):
        free(ext, g)
