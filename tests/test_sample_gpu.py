"""The device sampler (minigpt4_b200_sample_steps; llama_sample.cuh): the ids of the host Sampler for the same generator state.

- glibc's expf / logf restated on the device, checked bit for bit over every input the sampler can give them;
- the sampling kernel against minigpt4_b200_host_sample, draw for draw, over a sweep of the chain's parameters;
- sample_steps against minigpt4_end_chat / end_chat_batch on twin contexts: ids, n_past and logits bit for bit, and the generator
  continuing where the device left it."""
import ctypes
import itertools

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

WEBUI = dict(temp=0.8, top_k=40, top_p=0.9)


# ---- libm -----------------------------------------------------------------------------------------------------------------------
def test_expf_bit_exact_over_every_softmax_argument(ext):
    """every finite float <= 0 (logit - max): -0, the negative normals and subnormals, down to -FLT_MAX; and +0"""
    assert ext.op_check_libm(0, 0x00000000, 0x00000000) == 0
    assert ext.op_check_libm(0, 0x80000000, 0xFF7FFFFF) == 0


def test_logf_bit_exact_over_every_probability(ext):
    """every float in (0, 1]"""
    assert ext.op_check_libm(1, 0x00000001, 0x3F800000) == 0


# ---- kernel against host --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_vocab", [2048, 32000])
@pytest.mark.parametrize("sigma", [1.0, 3.0, 10.0])
@pytest.mark.parametrize("top_k", [0, 1, 5, 40, 100, -1], ids=["0", "1", "5", "40", "100", "n_vocab"])
def test_kernel_draws_equal_host_draws(ext, n_vocab, sigma, top_k):
    """32 draws from one generator per case: top_p x tfs_z x typical_p x temp x seed"""
    k = n_vocab if top_k < 0 else top_k
    logits = (np.random.default_rng(int(sigma * 1000) + n_vocab).standard_normal(n_vocab) * sigma).astype(np.float32)
    for top_p, tfs_z, typical_p, temp, seed in itertools.product((1.0, 0.95, 0.9, 0.5), (1.0, 0.95), (1.0, 0.9), (0.1, 0.8, 1.5), (1, 77, 4242)):
        kw = dict(temp=temp, top_k=k, top_p=top_p, tfs_z=tfs_z, typical_p=typical_p)
        want = ext.host_sample(logits, seed, 32, **kw)
        got = ext.op_sample(logits, seed, 32, **kw)
        _same_up_to_ties(got, want, logits, kw | dict(seed=seed))


def _same_up_to_ties(got, want, logits, what):
    """draw for draw the same id, except that a draw may return another id of EQUAL logit (normal float32 logits over 32000 ids hold a few
    ties; the device orders tied ids by id, libstdc++'s sort in an order of its own).  Every draw takes the same two generator outputs, so
    the streams stay aligned after a tie."""
    for i, (g, w) in enumerate(zip(got.tolist(), want.tolist())):
        assert g == w or logits[g] == logits[w], f"draw {i}: {g} != {w}, {what}"


def test_ties_go_to_the_lower_id(ext):
    """all-equal logits: top_k 1 keeps id 0 every time (the documented tie rule)"""
    logits = np.full(32000, 0.25, np.float32)
    assert ext.op_sample(logits, 5, 32, temp=0.8, top_k=1, top_p=0.9).tolist() == [0] * 32


# ---- end to end -------------------------------------------------------------------------------------------------------------------
def _chat(lib, mg, vision, llm, seed, n_ctx=512, image_seed=3, q="what is this?"):
    import minigpt4_cpp_b200 as m
    c = lib.minigpt4_model_load(vision, llm, 1, seed, n_ctx, 8, 0)
    im = mg.synth_image(image_seed)
    mi = m.MiniGPT4Image(im.ctypes.data_as(ctypes.c_void_p), 224, 224, 3, m.ImageFormat.F32)
    emb = lib.minigpt4_encode_image(c, mi)
    lib.minigpt4_system_prompt(c)
    lib.minigpt4_begin_chat_image(c, emb, q)
    lib.minigpt4_free_embedding(emb)
    return c


def _text(ext, c, ids):
    return [ext.L.minigpt4_b200_token_text(c.ptr, int(i)).decode("utf-8", errors="ignore") for i in ids]


@pytest.fixture(scope="module")
def files(tiny, mg, tmp_path_factory):
    d = tmp_path_factory.mktemp("sample")
    spec = dict(n_embd=4096, n_head=32, n_layer=2)
    out = {}
    for name, kw in (("q4_1", dict(n_vocab=2048, wtype="q4_1")), ("q5_k", dict(n_vocab=2048, wtype="q5_k", output_type="q6_k")),
                     ("q4_1_32000", dict(n_vocab=32000, wtype="q4_1"))):
        out[name] = str(d / f"llama-{name}.bin")
        mg.write_llama_ggjt(out[name], mg.LlamaSpec(**spec, **kw))
    out["vision"] = tiny["vision"]
    return out


@pytest.mark.parametrize("name,mega,params", [("q4_1", True, WEBUI), ("q5_k", False, WEBUI),
                                              ("q4_1_32000", True, dict(temp=0.8, top_k=0, top_p=0.95))],
                         ids=["q4_1-megakernel", "q5_k-q6_k-per-op", "n_vocab-32000-top_k-0"])
def test_one_context_equals_end_chat(lib, ext, mg, files, name, mega, params):
    a = _chat(lib, mg, files["vision"], files[name], seed=1234)
    b = _chat(lib, mg, files["vision"], files[name], seed=1234)
    assert (ext.stats(a).decode_megakernel >= 6) == mega
    ids, _ = ext.sample_steps([a], 48, tfs_z=1.0, typical_p=1.0, **params)
    want = [lib.minigpt4_end_chat(b, **params) for _ in range(48)]
    assert _text(ext, a, ids[:, 0]) == want
    assert ext.n_past(a) == ext.n_past(b)
    assert np.array_equal(ext.logits(a), ext.logits(b))
    assert ext.greedy_id(a) == ext.greedy_id(b)
    # one generator: end_chat continues the device's stream
    assert [lib.minigpt4_end_chat(a, **params) for _ in range(8)] == [lib.minigpt4_end_chat(b, **params) for _ in range(8)]
    assert np.array_equal(ext.logits(a), ext.logits(b))
    for c in (a, b):
        lib.minigpt4_free(c)


def test_greedy_equals_decode_chain(lib, ext, mg, files):
    a = _chat(lib, mg, files["vision"], files["q4_1"], seed=9)
    b = _chat(lib, mg, files["vision"], files["q4_1"], seed=9)
    ids, _ = ext.sample_steps([a], 32, temp=0.0)
    want, _ = ext.decode_chain(b, 32)
    assert ids[:, 0].tolist() == want.tolist()
    assert ext.n_past(a) == ext.n_past(b) and np.array_equal(ext.logits(a), ext.logits(b))
    assert lib.minigpt4_end_chat(a, **WEBUI) == lib.minigpt4_end_chat(b, **WEBUI)   # the generator was not touched
    for c in (a, b):
        lib.minigpt4_free(c)


def _sessions(ext, path, seeds, prompts, n_ctx=256):
    p = ext.llm_load(path, n_ctx=n_ctx, seed=seeds[0])
    ses = [p] + [ext.session_create(p, s) for s in seeds[1:]]
    for c, pr in zip(ses, prompts):
        ext.eval_tokens(c, pr)
    return ses


@pytest.mark.parametrize("which,n", [("tiny", 8), ("wide", 3)], ids=["tiny-q4_1-B8", "4096-q4_1-B3"])
def test_sessions_equal_end_chat_batch(lib, ext, tiny, files, which, n):
    path = tiny["q4_1"] if which == "tiny" else files["q4_1"]
    rng = np.random.default_rng(17)
    prompts = [rng.integers(3, 1024, size=3 + 4 * i).tolist() for i in range(n)]
    seeds = [101 + 7 * i for i in range(n)]
    a = _sessions(ext, path, seeds, prompts)
    b = _sessions(ext, path, seeds, prompts)
    ids, _ = ext.sample_steps(a, 24, **WEBUI)
    want = [ext.end_chat_batch(b, **WEBUI) for _ in range(24)]
    for i in range(n):
        assert _text(ext, a[i], ids[:, i]) == [w[i] for w in want], f"session {i}"
        assert ext.n_past(a[i]) == ext.n_past(b[i])
        assert np.array_equal(ext.logits(a[i]), ext.logits(b[i])), f"session {i}"
    # the generators continue on the host
    assert [ext.end_chat_batch(a, **WEBUI) for _ in range(4)] == [ext.end_chat_batch(b, **WEBUI) for _ in range(4)]
    for c in a + b:
        ext.base.minigpt4_free(c)


def test_refused_calls_change_nothing(lib, ext, tiny):
    path = tiny["q4_1"]
    a = _sessions(ext, path, [5, 6], [[3, 4, 5, 6], [7, 8]], n_ctx=16)
    b = _sessions(ext, path, [5, 6], [[3, 4, 5, 6], [7, 8]], n_ctx=16)
    for c in a + b:
        ext.flush(c)
    before = [(ext.n_past(c), ext.logits(c)) for c in a]
    ctxs = ext._ctx_array(a)
    ids = (ctypes.c_int32 * 64)()
    assert ext.L.minigpt4_b200_sample_steps(ctypes.cast(ctxs, ctypes.c_void_p), 2, 13, 0.8, 40, 0.9, 1.0, 1.0, ids, None) == 8   # 4 + 13 > 16
    assert ext.L.minigpt4_b200_sample_steps(ctypes.cast(ctxs, ctypes.c_void_p), 1, 0, 0.8, 40, 0.9, 1.0, 1.0, ids, None) == 8
    for c, (n, lg) in zip(a, before):
        assert ext.n_past(c) == n and np.array_equal(ext.logits(c), lg)
    assert [lib.minigpt4_end_chat(c, **WEBUI) for c in a] == [lib.minigpt4_end_chat(c, **WEBUI) for c in b]   # generators untouched
    for c in a + b:
        ext.base.minigpt4_free(c)
