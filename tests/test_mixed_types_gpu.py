"""LLaMA files whose tensors do not all share one block type, the way real ggjt files come: a token embedding of its own type, k-quant
"_M"-like mixes that give `wv` and `w2` more bits in some layers, q / k / v of different types, Q4_0 and Q4_1 layers side by side.

The engine picks its paths per tensor (decode megakernel, tensor-core prefill, fused qkv, shared activation staging of q / k / v), so each
case pins the path plan it must get and then checks, bit for bit:
- one context against the CPU oracle: prompt, embedding rows, a queued tokens / rows / tokens flush, greedy steps and decode_chain;
- the same file with the megakernel and the tensor-core prefill switched off, step for step;
- the batched paths (flush_batch, decode_batch, score_tokens, sample_steps at B = 1 and 3, and B = 16 where the wide step is a GEMM pass)
  against contexts stepped on their own.

test_token_embedding_the_megakernel_cannot_decode is the regression test for token embeddings the megakernel's embed op does not decode
(Q4_K / Q5_0 / Q5_1 / Q8_0): such files must take the per-op decode graph, whose embed kernels decode every type."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

N_CTX = 256
WEBUI = dict(temp=0.8, top_k=40, top_p=0.9)
TINY = dict(n_vocab=1024, n_embd=512, n_head=4, n_layer=2)
MATS = ("attention.wq.weight", "attention.wk.weight", "attention.wv.weight", "attention.wo.weight", "feed_forward.w1.weight",
        "feed_forward.w2.weight", "feed_forward.w3.weight")


def _layer(i, types):
    """overrides for layer i: {matrix suffix: type}"""
    return {f"layers.{i}.{m}": t for m, t in types.items()}


ALL_Q4_0 = {m: "q4_0" for m in MATS}

# name -> (modelgen.LlamaSpec fields, (decode megakernel, tensor-core prefill) the load must choose)
CASES = {
    "tok-q8_0": (dict(TINY, wtype="q4_1", tok_type="q8_0"), (False, True)),
    "tok-q5_0": (dict(TINY, wtype="q4_0", tok_type="q5_0"), (False, True)),
    "tok-q5_1-k": (dict(TINY, wtype="q5_k", tok_type="q5_1"), (False, False)),
    "tok-q4_k": (dict(TINY, wtype="q4_1", tok_type="q4_k"), (False, True)),
    "tok-f16": (dict(TINY, wtype="q4_0", tok_type="f16"), (True, True)),
    "tok-f32": (dict(TINY, wtype="q4_1", tok_type="f32"), (True, True)),
    "tok-q6_k": (dict(TINY, wtype="q4_1", tok_type="q6_k"), (True, True)),
    "q4-layer-mix": (dict(TINY, wtype="q4_1", overrides={**_layer(0, ALL_Q4_0), **_layer(1, {"attention.wo.weight": "q4_0"})}),
                     (False, True)),
    "q4_k-M-like": (dict(TINY, wtype="q4_k", output_type="q6_k",
                         overrides=_layer(0, {"attention.wv.weight": "q6_k", "feed_forward.w2.weight": "q6_k"})), (False, False)),
    "q5_k-M-like": (dict(TINY, wtype="q5_k", output_type="q6_k",
                         overrides=_layer(1, {"attention.wv.weight": "q6_k", "feed_forward.w2.weight": "q6_k"})), (False, False)),
    # q / k / v of three types: layer 0 stages one Q8_0 activation for all three parts, layer 1 one Q8_K, layer 2 restages every part
    "qkv-act-reuse": (dict(TINY, n_layer=3, wtype="q4_1", overrides={
        **_layer(0, {"attention.wq.weight": "q4_0", "attention.wk.weight": "q5_0", "attention.wv.weight": "q8_0"}),
        **_layer(1, {"attention.wq.weight": "q4_k", "attention.wk.weight": "q5_k", "attention.wv.weight": "q6_k"}),
        **_layer(2, {"attention.wq.weight": "q4_1", "attention.wk.weight": "q4_0", "attention.wv.weight": "f16"})}), (False, False)),
    # 7B row widths (n_embd 4096, n_ff 11008): the K-split plans of the prefill GEMM, on Q4_1 and Q4_0 layers
    "wide-q4-mix": (dict(n_vocab=2048, n_embd=4096, n_head=32, n_layer=2, wtype="q4_1", tok_type="q8_0", overrides=_layer(1, ALL_Q4_0)),
                    (False, True)),
}

# the regression cases: token embeddings outside the megakernel's embed op, under layers the megakernel would otherwise run
REG_TOK = ("q4_k", "q5_0", "q5_1", "q8_0")
REG_LAYERS = ("q4_0", "q4_1", "q5_k")
REG_CASES = {f"reg-{t}-{w}": (dict(TINY, wtype=w, tok_type=t), (False, w != "q5_k")) for t in REG_TOK for w in REG_LAYERS}


@pytest.fixture(scope="module")
def model(mg, tmp_path_factory):
    """name -> path of the case's file, written on first use"""
    d = tmp_path_factory.mktemp("mixed")
    paths = {}

    def get(name):
        if name not in paths:
            spec = {**CASES, **REG_CASES}[name][0]
            paths[name] = str(d / f"llama-{name}.bin")
            mg.write_llama_ggjt(paths[name], mg.LlamaSpec(**spec))
        return paths[name]
    return get


def _plan(ext, c):
    s = ext.stats(c)
    return s.decode_megakernel == 6, s.prefill_gemm == 1


def _dims(name):
    spec = {**CASES, **REG_CASES}[name][0]
    return spec["n_vocab"], spec["n_embd"]


def _script(name, seed=21):
    n_vocab, n_embd = _dims(name)
    rng = np.random.default_rng(seed)
    return dict(ids=rng.integers(3, n_vocab, size=21).tolist(), rows=rng.standard_normal((7, n_embd)).astype(np.float32),
                head=rng.integers(3, n_vocab, size=9).tolist(), mid=rng.standard_normal((6, n_embd)).astype(np.float32),
                tail=rng.integers(3, n_vocab, size=4).tolist())


STAGES = ("21-token prompt", "7 embedding rows", "queued tokens / rows / tokens")


def _oracle(orc, path, s, steps):
    """the oracle's logits after each prompt stage and each of `steps` greedy steps, and the greedy ids"""
    e = orc.OracleEngine(None, path, n_ctx=N_CTX)
    lg = [e.eval_tokens(s["ids"]).copy(), e.eval_embd(s["rows"]).copy()]
    e.eval_tokens(s["head"]); e.eval_embd(s["mid"])
    lg.append(e.eval_tokens(s["tail"]).copy())
    ids = []
    for _ in range(steps):
        ids.append(e.end_chat_greedy()[0]); lg.append(e.logits.copy())
    return lg, ids


def _device(ext, path, s, steps, chain):
    """one context through the same script: the plan, logits after each stage and step, greedy ids; then decode_chain's ids and logits"""
    c = ext.llm_load(path, n_ctx=N_CTX)
    plan = _plan(ext, c)
    ext.eval_tokens(c, s["ids"]); lg = [ext.logits(c)]
    ext.eval_embd(c, s["rows"]); lg.append(ext.logits(c))
    ext.eval_tokens(c, s["head"]); ext.eval_embd(c, s["mid"]); ext.eval_tokens(c, s["tail"]); ext.flush(c)
    lg.append(ext.logits(c))
    ids = []
    for _ in range(steps):
        t = ext.greedy_id(c); ids.append(t); ext.eval_tokens(c, [t]); lg.append(ext.logits(c))
    ch = ext.decode_chain(c, chain)[0].tolist() if chain else []
    if chain:
        lg.append(ext.logits(c))
    ext.base.minigpt4_free(c)
    return plan, lg, ids, ch


def _label(k):
    return STAGES[k] if k < len(STAGES) else f"greedy step {k - len(STAGES)}"


def _first_difference(got, want):
    for k, (g, w) in enumerate(zip(got, want)):
        if not np.array_equal(g, w):
            return k
    return None


@pytest.mark.parametrize("name", list(CASES))
def test_one_context_matches_oracle_on_both_arms(ext, orc, model, monkeypatch, name):
    steps, chain = 24, 8
    path, want_plan = model(name), CASES[name][1]
    s = _script(name)
    want, want_ids = _oracle(orc, path, s, steps + chain)
    plan, lg, ids, ch = _device(ext, path, s, steps, chain)
    assert plan == want_plan, f"(megakernel, prefill GEMM) = {plan}"
    k = _first_difference(lg[:-1], want[:len(STAGES) + steps])
    assert k is None, f"logits differ from the oracle after the {_label(k)}"
    assert ids == want_ids[:steps]
    assert ch == want_ids[steps:], "decode_chain"
    assert np.array_equal(lg[-1], want[-1]), "logits after decode_chain"
    # the per-op arm: the general decode graph and the 8-row matvec prefill
    monkeypatch.setenv("MINIGPT4_B200_NO_MEGAKERNEL", "1")
    monkeypatch.setenv("MINIGPT4_B200_NO_PREFILL_GEMM", "1")
    plan2, lg2, ids2, ch2 = _device(ext, path, s, steps, chain)
    monkeypatch.delenv("MINIGPT4_B200_NO_MEGAKERNEL")
    monkeypatch.delenv("MINIGPT4_B200_NO_PREFILL_GEMM")
    assert plan2 == (False, False)
    k = _first_difference(lg2, lg)
    assert k is None, f"the per-op arm differs after the {_label(k) if k <= len(STAGES) + steps - 1 else 'decode_chain'}"
    assert ids2 == ids and ch2 == ch


# ---- batched paths against contexts stepped on their own ------------------------------------------------------------------------------
def _queues(name, n, seed):
    """n prompt queues of different lengths; the second one also holds embedding rows between its tokens"""
    n_vocab, n_embd = _dims(name)
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n):
        if i % 3 == 1:
            out.append([("t", rng.integers(3, n_vocab, size=5 + i).tolist()), ("e", rng.standard_normal((4, n_embd)).astype(np.float32)),
                        ("t", rng.integers(3, n_vocab, size=3).tolist())])
        else:
            out.append([("t", rng.integers(3, n_vocab, size=3 + 4 * i + (i % 3)).tolist())])
    return out


def _put(ext, c, q):
    for kind, v in q:
        if kind == "t": ext.eval_tokens(c, v)
        else: ext.eval_embd(c, v)


def _group(ext, path, n, seed):
    p = ext.llm_load(path, n_ctx=N_CTX, seed=seed)
    return [p] + [ext.session_create(p, seed=seed + 1 + i) for i in range(n - 1)]


def _free(ext, ctxs):
    for c in ctxs:
        ext.base.minigpt4_free(c)


def _np_score(lg, t):
    """numpy's log-probability (float64, rounded to float32) and tie-ruled rank of id t under the float32 logits lg"""
    m = np.float64(lg.max())
    lp = np.float32((np.float64(lg[t]) - m) - np.log(np.exp(lg.astype(np.float64) - m).sum()))
    return lp, int(np.count_nonzero(lg > lg[t]) + np.count_nonzero(lg[:t] == lg[t]))


def _text(ext, c, ids):
    return [ext.L.minigpt4_b200_token_text(c.ptr, int(i)).decode("utf-8", errors="ignore") for i in ids]


def _batch_equals_own_steps(ext, path, queues, steps, tag):
    """queues on a group flushed with flush_batch, then `steps` decode_batch steps; a second group runs each context on its own (own flush,
    greedy steps through eval_tokens): n_past, logits and ids equal at every step.  Returns both groups."""
    ses, ref = _group(ext, path, len(queues), 100), _group(ext, path, len(queues), 100)
    for c, r, q in zip(ses, ref, queues):
        _put(ext, c, q); _put(ext, r, q); ext.flush(r)
    ext.flush_batch(ses)
    for i, (c, r) in enumerate(zip(ses, ref)):
        assert ext.n_past(c) == ext.n_past(r) and np.array_equal(ext.logits(c), ext.logits(r)), f"{tag}: flush_batch, session {i}"
    for k in range(steps):
        got = ext.decode_batch(ses).tolist()
        for i, (c, r) in enumerate(zip(ses, ref)):
            ext.eval_tokens(r, [ext.greedy_id(r)])
            assert got[i] == ext.greedy_id(r), f"{tag}: decode_batch step {k}, session {i}"
            assert np.array_equal(ext.logits(c), ext.logits(r)), f"{tag}: decode_batch step {k}, session {i}"
    return ses, ref


@pytest.mark.parametrize("name", list(CASES))
def test_batched_paths_equal_own_steps(lib, ext, model, name):
    path, (_, gemm) = model(name), CASES[name][1]
    n_vocab = _dims(name)[0]
    queues = _queues(name, 3, seed=7)
    ses, ref = _batch_equals_own_steps(ext, path, queues, 8, "B = 3")
    # score_tokens (ids kept) against the same ids evaluated one at a time
    rng = np.random.default_rng(8)
    lists = [rng.integers(3, n_vocab, size=n).tolist() for n in (5, 2, 7)]
    before = [ext.logits(r) for r in ref]
    scored = ext.score_tokens(ses, lists, keep=True, logits=True)
    for i, (r, ids, (lp, rk, rows)) in enumerate(zip(ref, lists, scored)):
        for j, t in enumerate(ids):
            want_lp, want_rk = _np_score(before[i] if j == 0 else rows[j - 1], t)
            assert abs(np.float64(lp[j]) - np.float64(want_lp)) <= np.spacing(np.abs(want_lp)) and rk[j] == want_rk, f"session {i} id {j}"
            ext.eval_tokens(r, [t])
            assert np.array_equal(rows[j], ext.logits(r)), f"score_tokens: session {i}, row {j}"
        assert ext.n_past(ses[i]) == ext.n_past(r) and np.array_equal(ext.logits(ses[i]), ext.logits(r)), f"score_tokens kept, session {i}"
    _free(ext, ses + ref)
    # device-sampled steps at B = 1 (the context's own decode graph) and B = 3 against end_chat / end_chat_batch on twins
    a, b = _group(ext, path, 3, 300), _group(ext, path, 3, 300)
    for c, d, q in zip(a, b, queues):
        _put(ext, c, q); _put(ext, d, q)
    ids, _ = ext.sample_steps([a[0]], 12, **WEBUI)
    assert _text(ext, a[0], ids[:, 0]) == [lib.minigpt4_end_chat(b[0], **WEBUI) for _ in range(12)], "sample_steps at B = 1"
    assert ext.n_past(a[0]) == ext.n_past(b[0]) and np.array_equal(ext.logits(a[0]), ext.logits(b[0])), "sample_steps at B = 1"
    ids, _ = ext.sample_steps(a, 12, **WEBUI)
    want = [ext.end_chat_batch(b, **WEBUI) for _ in range(12)]
    for i in range(3):
        assert _text(ext, a[i], ids[:, i]) == [w[i] for w in want], f"sample_steps at B = 3, session {i}"
        assert ext.n_past(a[i]) == ext.n_past(b[i]) and np.array_equal(ext.logits(a[i]), ext.logits(b[i])), f"sample_steps at B = 3, session {i}"
    _free(ext, a + b)
    if gemm:   # from 16 columns the batched step runs the layers as the tensor-core GEMM pass
        ses, ref = _batch_equals_own_steps(ext, path, _queues(name, 16, seed=9), 6 if name.startswith("wide") else 8, "B = 16")
        _free(ext, ses + ref)


# ---- regression: token embeddings the megakernel does not decode ------------------------------------------------------------------
@pytest.mark.parametrize("name", list(REG_CASES))
def test_token_embedding_the_megakernel_cannot_decode(ext, orc, model, name):
    """Q4_0 / Q4_1 / Q5_K layers and output with a Q4_K / Q5_0 / Q5_1 / Q8_0 token embedding.  The megakernel's embed op decodes F32, F16,
    Q4_0, Q4_1, Q5_K and Q6_K rows only; given another type it embedded every decoded token as zeros, so the prompt's logits matched the
    oracle and the first greedy step did not.  Such files take the per-op decode graph."""
    steps = 16
    path = model(name)
    s = _script(name)
    want, want_ids = _oracle(orc, path, s, steps)
    plan, lg, ids, _ = _device(ext, path, s, steps, 0)
    k = _first_difference(lg, want)
    assert k is None, f"logits differ from the oracle after the {_label(k)} (megakernel, prefill GEMM) = {plan}"
    assert ids == want_ids
    assert plan == REG_CASES[name][1], f"(megakernel, prefill GEMM) = {plan}"
