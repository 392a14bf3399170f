"""Sessions (contexts that share one loaded model) and the batched decode step (minigpt4_b200_decode_batch / end_chat_batch).

Every conversation stepped in a batch must get the logits it gets when stepped alone, bit for bit: each case compares with np.array_equal
against independent single contexts loaded from the same file, and against the CPU oracle where noted."""
import ctypes

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

N_CTX = 256
STEPS = 24


def _prompts(n_vocab: int, k: int, seed: int = 5) -> list[list[int]]:
    rng = np.random.default_rng(seed)
    return [rng.integers(3, n_vocab, size=4 + 5 * i).tolist() for i in range(k)]   # different lengths: every session at its own n_past


def _single(ext, path, prompt, steps, n_ctx=N_CTX):
    """greedy continuation on a context of its own: ([greedy id after each step], [logits after each step])"""
    c = ext.llm_load(path, n_ctx=n_ctx)
    ext.eval_tokens(c, prompt)
    ids, lg = [], []
    for _ in range(steps):
        ext.eval_tokens(c, [ext.greedy_id(c)])
        ids.append(ext.greedy_id(c)); lg.append(ext.logits(c))
    ext.base.minigpt4_free(c)
    return ids, lg


def _oracle(orc, path, prompt, steps, n_ctx=N_CTX):
    e = orc.OracleEngine(None, path, n_ctx=n_ctx)
    e.eval_tokens(prompt)
    lg = []
    for _ in range(steps):
        e.end_chat_greedy(); lg.append(e.logits.copy())
    return lg


def _group(ext, path, n, n_ctx=N_CTX):
    p = ext.llm_load(path, n_ctx=n_ctx)
    return [p] + [ext.session_create(p, seed=100 + i) for i in range(n - 1)]


def _batched(ext, path, prompts, steps, n_ctx=N_CTX):
    ctxs = _group(ext, path, len(prompts), n_ctx)
    for c, pr in zip(ctxs, prompts):
        ext.eval_tokens(c, pr)                     # queued: decode_batch evaluates each context's prompt first
    ids, lg = [], []
    for _ in range(steps):
        ids.append(ext.decode_batch(ctxs).tolist())
        lg.append([ext.logits(c) for c in ctxs])
    for c, pr in zip(ctxs, prompts):
        assert ext.n_past(c) == len(pr) + steps
    for c in ctxs:
        ext.base.minigpt4_free(c)
    return ids, lg


def _check(ids, lg, refs, oracle=None):
    for i, (rid, rlg) in enumerate(refs):
        assert [s[i] for s in ids] == rid, f"session {i}"
        for k in range(len(rid)):
            assert np.array_equal(lg[k][i], rlg[k]), f"session {i} step {k}"
            if oracle is not None:
                assert np.array_equal(lg[k][i], oracle[i][k]), f"session {i} step {k} (oracle)"


@pytest.mark.parametrize("wt", ["q4_1", "q4_0", "q5_k", "q6_k", "f16", "mixed"])
def test_batched_steps_are_bit_exact(ext, orc, tiny, wt):
    """B = 2, 3, 5, 8 sessions from prompts of different lengths, 24 greedy batched steps: every session's logits after every step equal the
    single context's and the oracle's"""
    path = tiny[wt]
    n_vocab = 1001 if wt == "mixed" else 1024
    prompts = _prompts(n_vocab, 8)
    refs = [_single(ext, path, p, STEPS) for p in prompts]
    oracle = [_oracle(orc, path, p, STEPS) for p in prompts]
    for B in (2, 3, 5, 8):
        ids, lg = _batched(ext, path, prompts[:B], STEPS)
        _check(ids, lg, refs[:B], oracle[:B])


@pytest.mark.parametrize("name", ["q4_k", "q5_0", "q5_1", "q8_0"])
def test_batched_steps_other_block_types(ext, mg, tmp_path, name):
    """the block types the tiny models miss (dot2_q4k, dot2_b32 and their token-embedding kernels), written like test_block_types_gpu.py"""
    path = str(tmp_path / f"llama-{name}.bin")
    extra = {"output_type": "q6_k"} if name == "q4_k" else {}
    mg.write_llama_ggjt(path, mg.LlamaSpec(n_vocab=1024, n_embd=512, n_head=4, n_layer=2, wtype=name, **extra))
    prompts = _prompts(1024, 3, seed=9)
    refs = [_single(ext, path, p, 12) for p in prompts]
    ids, lg = _batched(ext, path, prompts, 12)
    _check(ids, lg, refs)


@pytest.mark.parametrize("spec,B", [(dict(n_embd=4096, n_head=32, wtype="q4_1"), 8), (dict(n_embd=5120, n_head=40, wtype="q5_k"), 4)],
                         ids=["7b-wide-q4_1-B8", "13b-wide-q5_k-B4"])
def test_batched_steps_at_full_width(ext, mg, tmp_path, spec, B):
    """NT = 8 at 7B width and NT = 4 at 13B width (2 layers each); the single contexts decode on the megakernel"""
    path = str(tmp_path / "llama-wide.bin")
    mg.write_llama_ggjt(path, mg.LlamaSpec(n_vocab=2048, n_layer=2, **spec))
    prompts = _prompts(2048, B, seed=13)
    refs = [_single(ext, path, p, 8) for p in prompts]
    ids, lg = _batched(ext, path, prompts, 8)
    _check(ids, lg, refs)


def test_mixing_paths(lib, ext, tiny):
    """batched steps interleaved with single end_chat steps (megakernel), decode_chain and queued prompt rows on the same sessions == the same
    operations on separate contexts"""
    path = tiny["q4_1"]
    prompts = _prompts(1024, 4, seed=21)
    ses = _group(ext, path, 4)
    ref = [ext.llm_load(path, n_ctx=N_CTX) for _ in range(4)]
    assert ext.stats(ses[1]).decode_megakernel >= 6
    for s, r, p in zip(ses, ref, prompts):
        ext.eval_tokens(s, p); ext.eval_tokens(r, p)

    def batch(idx, ids=None):
        got = ext.decode_batch([ses[i] for i in idx], ids)
        for j, i in enumerate(idx):
            ext.eval_tokens(ref[i], [ext.greedy_id(ref[i]) if ids is None or ids[j] < 0 else ids[j]])
            assert got[j] == ext.greedy_id(ref[i])

    def same():
        for s, r in zip(ses, ref):
            assert ext.n_past(s) == ext.n_past(r)
            assert np.array_equal(ext.logits(s), ext.logits(r))

    batch([0, 1, 2, 3]); same()
    ext.eval_tokens(ses[3], [17, 18, 19]); ext.eval_tokens(ref[3], [17, 18, 19])      # queued rows, flushed by the next batch
    batch([3, 1, 0]); same()
    for _ in range(3):                                                                 # single steps through each session's own graph
        assert lib.minigpt4_end_chat(ses[1], temp=0.0) == lib.minigpt4_end_chat(ref[1], temp=0.0)
    a, _ = ext.decode_chain(ses[2], 5); b, _ = ext.decode_chain(ref[2], 5)
    assert a.tolist() == b.tolist(); same()
    batch([2, 0, 3], [40, -1, 41]); same()
    batch([1]); same()                                                                 # a batch of one: the context's own decode graph
    ext.eval_tokens(ses[0], list(range(50, 61))); ext.eval_tokens(ref[0], list(range(50, 61)))
    for _ in range(4):
        batch([0, 1, 2, 3])
    same()
    a, _ = ext.decode_chain(ses[0], 4); b, _ = ext.decode_chain(ref[0], 4)
    assert a.tolist() == b.tolist(); same()
    for c in ses + ref:
        ext.base.minigpt4_free(c)


def test_chat_flow_through_the_reference_abi(lib, ext, mg, tiny):
    """system prompt + begin_chat_image on three sessions with different images encoded on the sessions, 32 greedy end_chat_batch steps ==
    minigpt4_end_chat on a separate context"""
    import minigpt4_cpp_b200 as m
    big = tiny["q4_1"].replace("llama-tiny-q4_1.bin", "llama-4096-sessions.bin")
    mg.write_llama_ggjt(big, mg.LlamaSpec(n_vocab=2048, n_embd=4096, n_head=32, n_layer=2, wtype="q4_1"))
    p = lib.minigpt4_model_load(tiny["vision"], big, 1, 1337, 512, 8, 0)
    ses = [p, ext.session_create(p, 1), ext.session_create(p, 2)]
    imgs = [mg.synth_image(s) for s in (3, 4, 5)]
    qs = ["what is this?", "describe it", "which color?"]
    keep = []
    for c, im, q in zip(ses, imgs, qs):
        mi = m.MiniGPT4Image(im.ctypes.data_as(ctypes.c_void_p), 224, 224, 3, m.ImageFormat.F32)
        emb = lib.minigpt4_encode_image(c, mi)
        keep.append(emb)
        lib.minigpt4_system_prompt(c)
        lib.minigpt4_begin_chat_image(c, emb, q)
    got = [ext.end_chat_batch(ses, temp=0.0) for _ in range(32)]
    r = lib.minigpt4_model_load(tiny["vision"], big, 1, 1337, 512, 8, 0)
    for i, (im, q) in enumerate(zip(imgs, qs)):
        lib.minigpt4_reset_chat(r)
        mi = m.MiniGPT4Image(im.ctypes.data_as(ctypes.c_void_p), 224, 224, 3, m.ImageFormat.F32)
        emb = lib.minigpt4_encode_image(r, mi)
        lib.minigpt4_system_prompt(r)
        lib.minigpt4_begin_chat_image(r, emb, q)
        want = [lib.minigpt4_end_chat(r, temp=0.0) for _ in range(32)]
        assert [g[i] for g in got] == want, f"session {i}"
        assert ext.n_past(ses[i]) == ext.n_past(r)
        lib.minigpt4_free_embedding(emb)
    for e in keep:
        lib.minigpt4_free_embedding(e)
    for c in ses + [r]:
        lib.minigpt4_free(c)


def test_sampling_uses_each_sessions_own_sampler(lib, ext, tiny):
    """temp 0.8, top_k 40, top_p 0.9: each session's sequence == a separate context created with the same seed"""
    path = tiny["q4_1"]
    p = ext.llm_load(path, n_ctx=N_CTX, seed=7)
    ses = [p, ext.session_create(p, 11), ext.session_create(p, 12)]
    for c in ses:
        lib.minigpt4_begin_chat(c, "tell me a story")
    got = [ext.end_chat_batch(ses, temp=0.8, top_k=40, top_p=0.9) for _ in range(24)]
    for i, seed in enumerate((7, 11, 12)):
        r = ext.llm_load(path, n_ctx=N_CTX, seed=seed)
        lib.minigpt4_begin_chat(r, "tell me a story")
        want = [lib.minigpt4_end_chat(r, temp=0.8, top_k=40, top_p=0.9) for _ in range(24)]
        assert [g[i] for g in got] == want, f"session {i}"
        ext.base.minigpt4_free(r)
    for c in ses:
        ext.base.minigpt4_free(c)


def test_refused_batches_change_nothing(lib, ext, tiny):
    path = tiny["q4_1"]
    ses = _group(ext, path, 3)
    other = ext.llm_load(path, n_ctx=N_CTX)
    for c, pr in zip(ses + [other], _prompts(1024, 4, seed=31)):
        ext.eval_tokens(c, pr); ext.flush(c)
    small = _group(ext, path, 2, n_ctx=16)
    ext.eval_tokens(small[0], list(range(3, 19))); ext.eval_tokens(small[1], [5, 6])
    everyone = ses + [other] + small
    before = [(ext.n_past(c), ext.logits(c)) for c in everyone]
    bad = [([], None), (ses * 3, None), ([ses[0], ses[1], ses[0]], None), ([ses[0], other], None), ([small[1], small[0]], None),
           ([ses[0], ses[1]], [5, 1024]), ([ses[0], ses[1]], [5, 10 ** 6])]
    for ctxs, ids in bad:
        with pytest.raises(RuntimeError, match="FailedToAddString"):
            ext.decode_batch(ctxs, ids)
    with pytest.raises(RuntimeError, match="FailedToAddString"):
        ext.end_chat_batch([ses[1], ses[1]], temp=0.8)
    assert ext.L.minigpt4_b200_decode_batch(None, 2, None, None) != 0
    for c, (n, lg) in zip(everyone, before):
        assert ext.n_past(c) == n and np.array_equal(ext.logits(c), lg)
    ext.decode_batch([small[1]]); ext.decode_batch(ses)    # still usable
    for c in everyone:
        ext.base.minigpt4_free(c)


def test_lifetime_and_sharing(ext, tiny):
    """the parent freed first, the sessions keep stepping; n_contexts counts down; the weights are shared and a context owns its KV cache plus
    its scratch"""
    path = tiny["q4_1"]
    prompts = _prompts(1024, 4, seed=41)
    refs = [_single(ext, path, p, 12) for p in prompts]
    ses = _group(ext, path, 4)
    st = ext.stats(ses[0])
    E, L, FF, V = st.n_embd, st.n_layer, st.n_ff, st.n_vocab
    infos = [ext.session_info(c) for c in ses]
    assert all(i[0] == 4 for i in infos)
    shared = infos[0][2]
    assert all(i[2] == shared for i in infos) and shared >= st.llm_weight_bytes_per_token
    kv = 2 * L * N_CTX * E * 2
    scratch = 512 * (3 * E + FF) * 4 + 8 * E * 4 + 8 * (max(E, FF) * 2 + 4096) + (V + 1) * 4 + 4096
    for _, owned, _ in infos:
        assert kv <= owned <= kv + scratch and owned * 4 < shared
    for c, p in zip(ses, prompts):
        ext.eval_tokens(c, p)
    got = {i: [] for i in range(4)}

    def step(idx):
        for i, t in zip(idx, ext.decode_batch([ses[i] for i in idx]).tolist()):
            got[i].append(t)

    for _ in range(4):
        step([0, 1, 2, 3])
    ext.base.minigpt4_free(ses[0])                       # the parent goes first
    assert ext.session_info(ses[1])[0] == 3
    for _ in range(4):
        step([1, 2, 3])
    ext.base.minigpt4_free(ses[2])
    assert ext.session_info(ses[1])[0] == 2
    for _ in range(4):
        step([3, 1])
    assert got[0] == refs[0][0][:4] and got[2] == refs[2][0][:8]
    assert got[1] == refs[1][0] and got[3] == refs[3][0]
    assert np.array_equal(ext.logits(ses[1]), refs[1][1][11]) and np.array_equal(ext.logits(ses[3]), refs[3][1][11])
    ext.base.minigpt4_free(ses[1])
    assert ext.session_info(ses[3])[0] == 1
    ext.decode_batch([ses[3]])
    ext.base.minigpt4_free(ses[3])
