"""The Vicuna-13B geometry (n_embd 5120, 40 heads, n_ff 13824) against the CPU oracle, bit for bit.

The 512- and 4096-wide models of the other tests never reach the paths these widths select: the megakernel with five register-resident
Q8 blocks per lane (NBL = 5), RMS staging with 5 items per thread and un-normed staging with 8, a non-power-of-two RMS divisor, fewer than
15 stream warps, Q5_K staging over 20 / 54 super-blocks per row, prefill GEMM classes with padded tiles (S = 8 for 160 blocks), per-op F16
staging next to the shared-memory cap, and a 5120-wide llama_proj / image prefix.  The load log is parsed to prove that the intended
megakernel configuration ran.  The files are 13B-wide with 1-2 layers (370-450 MB each), written once per module."""
import ctypes
import functools
import os
import re

import numpy as np
import pytest

from conftest import rel_err

pytestmark = pytest.mark.gpu

E13, FF13, N_CTX = 5120, 13824, 512
TYPES = {"q4_0": 2, "q4_1": 3, "q5_0": 6, "q5_1": 7, "q8_0": 8, "q4_k": 12, "q5_k": 13, "q6_k": 14, "f16": 1}
K_QUANTS = (12, 13, 14)

SPECS = {   # n_vocab 2048 throughout
    "q4_1": dict(n_embd=5120, n_head=40, n_layer=2, wtype="q4_1"),
    "q5_k": dict(n_embd=5120, n_head=40, n_layer=2, wtype="q5_k"),
    "q4_0": dict(n_embd=5120, n_head=40, n_layer=1, wtype="q4_0"),
    "q5_k+q6_k": dict(n_embd=5120, n_head=40, n_layer=1, wtype="q5_k", output_type="q6_k"),   # the layout of the 13B q5_k download
    "7b-q4_1": dict(n_embd=4096, n_head=32, n_layer=1, wtype="q4_1"),
    "7b-q5_k": dict(n_embd=4096, n_head=32, n_layer=1, wtype="q5_k"),
}


@pytest.fixture(scope="module")
def wide(tmp_path_factory, mg):
    """name -> path of the file, written on first use (about 3 s each) and deleted when the module is done"""
    d = tmp_path_factory.mktemp("wide13b")
    made = {}

    def get(name):
        if name not in made:
            p = str(d / f"{name}.bin")
            if name == "vision":
                mg.write_minigpt4(p, mg.VisionSpec(n_blocks=2, n_qformer_layers=2, n_embd_llm=5120))
            else:
                mg.write_llama_ggjt(p, mg.LlamaSpec(n_vocab=2048, **SPECS[name]))
            made[name] = p
        return made[name]
    yield get
    for p in made.values():
        os.remove(p)


# ---- which megakernel configuration a file must get ------------------------------------------------------------------------------------
_MEGA_LOG = re.compile(r"decode megakernel \(generation 6\): (\d+) ops/token, (\d+) stream warps x 2 slots x (\d+) B, act (\d+) B, "
                       r"(\d+) B dynamic shared per CTA, register-resident blocks per lane (\d+), grid (\d+)")
_LIBC = ctypes.CDLL(None)


@functools.lru_cache(maxsize=None)
def _smem_optin() -> int:
    import torch
    return int(torch.cuda.get_device_properties(0).shared_memory_per_block_optin)


def _row_bytes(wt: str, cols: int) -> int:   # device row of a megakernel weight matrix (16-byte padded Q4 rows, row-packed Q5_K)
    return {"q4_0": (cols // 32 * 18 + 15) & ~15, "q4_1": (cols // 32 * 20 + 15) & ~15, "q5_k": cols // 256 * 176}[wt]


def _mega_plan(wt: str, E: int, FF: int, n_ctx: int, smem_optin: int, w_cap: int = 15) -> tuple[int, int, int, int]:
    """(stream warps, slot bytes, activation bytes, register-resident blocks per lane) the megakernel must choose: two slots per stream warp
    hold a row pair of an E-wide or one row of an FF-wide matrix; the activation region holds the widest staged vector (or the attention
    scratch); all of it, 10 KB of static shared memory and 2 x 15 mbarriers must fit in the opt-in shared memory of one block."""
    if wt == "q5_k":
        act = max(((c + c // 256 * 4 + c // 16 * 2) + 15) & ~15 for c in (E, FF))   # Q8_K: int8 q, float d per 256, int16 sums per 16
    else:
        act = max(c + 64 + c // 32 * 8 for c in (E, FF))                               # Q8_0 / Q8_1 planes + 64 B pad + {d, s} per block
    act = (max(act, 6 * n_ctx) + 127) & ~127
    slot = (max(2 * _row_bytes(wt, E), _row_bytes(wt, FF)) + 15) & ~15
    room = smem_optin - 10240 - act - 2 * 15 * 8
    W = min(15, w_cap, room // (2 * slot))
    return W, slot, act, 0 if wt == "q5_k" else {4096: 4, 5120: 5}.get(E, 0)


# W an H100 (227 KB opt-in shared memory per block) must get at n_ctx 512
H100_W = {("q4_1", 5120): 11, ("q4_0", 5120): 13, ("q5_k", 5120): 10, ("q4_1", 4096): 15, ("q5_k", 4096): 13}


def _load(ext, capfd, path: str, n_ctx: int = N_CTX):
    """load at verbosity 2; returns (ctx, numbers of the megakernel line of the load log or None):
    (ops per token, stream warps, slot bytes, act bytes, dynamic shared bytes, register-resident blocks per lane, grid)"""
    capfd.readouterr()
    c = ext.llm_load(path, n_ctx=n_ctx, verbosity=2)
    _LIBC.fflush(None)   # the C stdout buffer -> the captured file descriptor
    m = _MEGA_LOG.search(capfd.readouterr().out)
    return c, (tuple(int(g) for g in m.groups()) if m else None)


def _check_plan(ext, c, plan, name: str, w_cap: int = 15):
    s = SPECS[name]
    wt, E = s["wtype"], s["n_embd"]
    FF = 13824 if E == 5120 else 11008
    W, slot, act, nbl = _mega_plan(wt, E, FF, N_CTX, _smem_optin(), w_cap)
    assert ext.stats(c).decode_megakernel == 6 and plan is not None, "the megakernel did not take this file"
    assert plan[0] == 5 * s["n_layer"] + 3
    assert plan[1:4] == (W, slot, act), (plan, (W, slot, act))
    assert plan[5] == nbl
    return plan[1]


# ---- 1. kernel level ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("wt", list(TYPES))
@pytest.mark.parametrize("shape", [(64, 5120), (48, 13824), (34, 5120)])
@pytest.mark.parametrize("n", [1, 8, 11])
def test_matvec_at_13b_widths_matches_oracle(ext, orc, mg, wt, shape, n):
    """per-op dequant-matvec at 5120 / 13824 columns (F16 x 13824 x 8 rows stages 221 184 B: the widest shared-memory staging of any shape)"""
    rows, cols = shape
    gt = TYPES[wt]
    rng = np.random.default_rng(rows * 7 + cols + n + gt)
    raw = mg.synth_quant(rng, gt, rows, cols, 0.02)
    x = rng.standard_normal((n, cols)).astype(np.float32)
    x[0, :256 if gt in K_QUANTS else 32] = 0.0   # an all-zero (super-)block: the amax == 0 path
    got, want = ext.op_matvec(gt, raw, rows, cols, x), orc.mul_mat(gt, raw, rows, cols, x)
    assert got.shape == want.shape
    assert np.array_equal(got, want), rel_err(got, want)


# ---- 2./3. the files take the 13B paths ---------------------------------------------------------------------------------------------------
def test_megakernel_sizing_on_h100():
    """the sizing rule, at the numbers of an H100: 13B files run with fewer than 15 stream warps"""
    for (wt, E), W in H100_W.items():
        assert _mega_plan(wt, E, 13824 if E == 5120 else 11008, N_CTX, 227 * 1024)[0] == W, (wt, E)


@pytest.mark.parametrize("name", ["q4_1", "q4_0", "q5_k", "q5_k+q6_k"])
def test_13b_files_take_the_wide_paths(ext, wide, capfd, name):
    s = SPECS[name]
    c, plan = _load(ext, capfd, wide(name))
    st = ext.stats(c)
    assert (st.n_embd, st.n_ff, st.n_layer) == (E13, FF13, s["n_layer"])
    assert st.prefill_gemm == (1 if s["wtype"] in ("q4_0", "q4_1") else 0)   # the int8 GEMM takes homogeneous Q4_0 / Q4_1 files
    if name == "q5_k+q6_k":
        assert st.decode_megakernel == 0 and plan is None   # the Q6_K output matrix sends decode to the per-op graph
    else:
        W = _check_plan(ext, c, plan, name)
        assert W < 15 and plan[5] == (0 if s["wtype"] == "q5_k" else 5)
        if _smem_optin() == 227 * 1024:
            assert W == H100_W[(s["wtype"], E13)]
        print(f"{name}: {W} stream warps, register-resident blocks per lane {plan[5]}")
    ext.base.minigpt4_free(c)


# ---- 4. megakernel decode ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["q4_1", "q4_0", "q5_k"])
def test_megakernel_decode_at_13b_is_bit_identical(ext, orc, wide, capfd, monkeypatch, name):
    """230-token prompt (past the 192-key single pass of the in-kernel attention, 40 heads), 24 greedy steps through the megakernel and the
    per-op graph with the oracle's logits at every step, then 8 device-chained steps == host-driven greedy"""
    path = wide(name)
    c2, plan = _load(ext, capfd, path)
    _check_plan(ext, c2, plan, name)
    monkeypatch.setenv("MINIGPT4_B200_NO_MEGAKERNEL", "1")
    c1 = ext.llm_load(path, n_ctx=N_CTX)
    monkeypatch.delenv("MINIGPT4_B200_NO_MEGAKERNEL")
    assert ext.stats(c1).decode_megakernel == 0
    e = orc.OracleEngine(None, path, n_ctx=N_CTX)
    ids = np.random.default_rng(13).integers(3, e.n_vocab, size=230).tolist()
    ext.eval_tokens(c1, ids); ext.eval_tokens(c2, ids); e.eval_tokens(ids)
    assert np.array_equal(ext.logits(c1), e.logits) and np.array_equal(ext.logits(c2), e.logits), "prompt"
    for step in range(24):
        t1, t2 = ext.greedy_id(c1), ext.greedy_id(c2)
        assert t1 == t2 == int(np.argmax(e.logits)), step
        ext.eval_tokens(c1, [t1]); ext.eval_tokens(c2, [t2]); e.eval_tokens([t1])
        assert np.array_equal(ext.logits(c2), e.logits), f"megakernel, step {step}: {rel_err(ext.logits(c2), e.logits)}"
        assert np.array_equal(ext.logits(c1), e.logits), f"per-op graph, step {step}: {rel_err(ext.logits(c1), e.logits)}"
    chain, _ = ext.decode_chain(c2, 8)
    host = []
    for _ in range(8):
        t = ext.greedy_id(c1); host.append(t); ext.eval_tokens(c1, [t])
    assert chain.tolist() == host
    assert np.array_equal(ext.logits(c1), ext.logits(c2))
    ext.base.minigpt4_free(c1); ext.base.minigpt4_free(c2)


# ---- 5. prefill GEMM ----------------------------------------------------------------------------------------------------------------------
def _load_prefill(ext, path, monkeypatch, gemm: bool):
    if gemm: monkeypatch.delenv("MINIGPT4_B200_NO_PREFILL_GEMM", raising=False)
    else: monkeypatch.setenv("MINIGPT4_B200_NO_PREFILL_GEMM", "1")
    c = ext.llm_load(path, n_ctx=N_CTX)
    monkeypatch.delenv("MINIGPT4_B200_NO_PREFILL_GEMM", raising=False)
    assert ext.stats(c).prefill_gemm == (1 if gemm else 0)
    return c


@pytest.mark.parametrize("name", ["q4_1", "q4_0"])
@pytest.mark.parametrize("n", [2, 33, 97])
def test_prefill_gemm_at_13b_is_bit_identical(ext, orc, wide, monkeypatch, name, n):
    """a 32-row embedding prefix, then n prompt rows: the GEMM (default K split and none), the per-op matvec path and the oracle agree on
    the logits and on the residual stream after the last layer"""
    path = wide(name)
    gemm, per_op, no_ksplit = _load_prefill(ext, path, monkeypatch, True), _load_prefill(ext, path, monkeypatch, False), _load_prefill(ext, path, monkeypatch, True)
    ctxs = (gemm, per_op, no_ksplit)
    e = orc.OracleEngine(None, path, n_ctx=N_CTX)
    last = SPECS[name]["n_layer"] - 1

    def run(feed, piece):   # one pass per piece on every context; the K split is chosen per launch
        for c in ctxs:
            if c is no_ksplit: monkeypatch.setenv("MINIGPT4_B200_PREFILL_NO_KSPLIT", "1")
            feed(c, piece); ext.flush(c)
            monkeypatch.delenv("MINIGPT4_B200_PREFILL_NO_KSPLIT", raising=False)

    rows = np.random.default_rng(n).standard_normal((32, E13)).astype(np.float32)
    run(ext.eval_embd, rows)
    want = e.eval_embd(rows).copy()
    assert all(np.array_equal(ext.logits(c), want) for c in ctxs), "prefix"
    assert np.array_equal(ext.hidden(gemm, 32), ext.hidden(no_ksplit, 32))
    assert np.array_equal(ext.hidden(gemm, 32)[24:], ext.hidden(per_op, 8))   # the per-op path keeps the residual stream of its last 8-row chunk
    ids = np.random.default_rng(100 + n).integers(3, e.n_vocab, size=n).tolist()
    run(ext.eval_tokens, ids)
    hid = e.eval_tokens(ids, tap_layer=last).copy()
    want = e.logits.copy()
    k = n - 8 * ((n - 1) // 8)
    h = ext.hidden(gemm, n)
    assert np.array_equal(h, hid), "residual stream differs between the GEMM prefill and the oracle"
    assert np.array_equal(h, ext.hidden(no_ksplit, n))
    assert np.array_equal(h[n - k:], ext.hidden(per_op, k))
    assert all(np.array_equal(ext.logits(c), want) for c in ctxs), "prompt"
    a, b = [], []
    for _ in range(4):   # decode continues from the KV rows the GEMM epilogue wrote
        t = ext.greedy_id(gemm); a.append(t); ext.eval_tokens(gemm, [t]); b.append(e.end_chat_greedy()[0])
    assert a == b
    for c in ctxs: ext.base.minigpt4_free(c)


# ---- 6. per-op path ----------------------------------------------------------------------------------------------------------------------
def test_per_op_path_at_13b_with_q6_k_output(ext, orc, wide):
    path = wide("q5_k+q6_k")
    c = ext.llm_load(path, n_ctx=N_CTX)
    st = ext.stats(c)
    assert st.decode_megakernel == 0 and st.prefill_gemm == 0 and (st.n_embd, st.n_ff) == (E13, FF13)
    e = orc.OracleEngine(None, path, n_ctx=N_CTX)
    ids = np.random.default_rng(61).integers(3, e.n_vocab, size=61).tolist()
    ext.eval_tokens(c, ids)
    assert np.array_equal(ext.logits(c), e.eval_tokens(ids))
    for step in range(16):
        t = ext.greedy_id(c)
        assert t == int(np.argmax(e.logits)), step
        ext.eval_tokens(c, [t]); e.eval_tokens([t])
        assert np.array_equal(ext.logits(c), e.logits), f"step {step}: {rel_err(ext.logits(c), e.logits)}"
    ext.base.minigpt4_free(c)


# ---- 7. vision + chat at 5120 -------------------------------------------------------------------------------------------------------------
def test_vision_and_chat_flow_at_13b_width(lib, ext, orc, mg, wide):
    """llama_proj with 5120 outputs, then system prompt -> begin_chat_image -> 32 x end_chat_image (greedy) == the oracle fed the GPU's
    embedding, token for token"""
    import minigpt4_cpp_b200 as m
    vis, llm = wide("vision"), wide("q4_1")
    c = lib.minigpt4_model_load(vis, llm, 1, 1337, N_CTX, 8, 0)
    e = orc.OracleEngine(vis, llm, n_ctx=N_CTX)
    img = mg.synth_image(7)
    mi = m.MiniGPT4Image(img.ctypes.data_as(ctypes.c_void_p), 224, 224, 3, m.ImageFormat.F32)
    emb = lib.minigpt4_encode_image(c, mi)
    assert emb.n_embeddings == 32 * E13
    gemb = np.ctypeslib.as_array(emb.data, shape=(32 * E13,)).copy().reshape(32, E13)
    want = e.encode_image(img)
    assert want.shape == (32, E13)
    assert rel_err(gemb, want) < 1e-2, rel_err(gemb, want)   # (measured 3.0e-4 on an H100)
    lib.minigpt4_system_prompt(c)
    lib.minigpt4_begin_chat_image(c, emb, "what is this?")
    e.system_prompt(); e.begin_chat_image(gemb, "what is this?")
    assert ext.n_past(c) == e.n_past
    assert np.array_equal(ext.logits(c), e.logits)
    got = [lib.minigpt4_end_chat_image(c, temp=0.0) for _ in range(32)]
    want = [e.end_chat_greedy()[1].decode("utf-8", errors="ignore") for _ in range(32)]
    assert got == want
    lib.minigpt4_begin_chat(c, "and the color?"); e.begin_chat("and the color?")
    assert lib.minigpt4_end_chat(c, temp=0.0) == e.end_chat_greedy()[1].decode("utf-8", errors="ignore")
    lib.minigpt4_free_embedding(emb)
    lib.minigpt4_free(c)


# ---- 8. stream-warp count -----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["7b-q4_1", "7b-q5_k"])
def test_stream_warp_count_does_not_change_a_bit(ext, orc, wide, capfd, monkeypatch, name):
    """MINIGPT4_B200_MEGA_W caps the stream warps: every W >= 4 gives the oracle's logits and ids (7B-wide rows, so that each CTA owns many
    row pairs and the W-strided walk wraps several times); W = 3 leaves decode to the per-op graph"""
    path = wide(name)
    ctxs = {}
    for w in (None, 4, 7, 11, 13, 3):
        if w is not None: monkeypatch.setenv("MINIGPT4_B200_MEGA_W", str(w))
        c, plan = _load(ext, capfd, path)
        monkeypatch.delenv("MINIGPT4_B200_MEGA_W", raising=False)
        if w == 3:
            assert ext.stats(c).decode_megakernel == 0 and plan is None
        else:
            W = _check_plan(ext, c, plan, name, 15 if w is None else w)
            if _smem_optin() == 227 * 1024:
                assert W == min(w or 15, H100_W[(SPECS[name]["wtype"], 4096)])
        ctxs[w] = c
    e = orc.OracleEngine(None, path, n_ctx=N_CTX)
    ids = np.random.default_rng(40).integers(3, e.n_vocab, size=40).tolist()
    for c in ctxs.values(): ext.eval_tokens(c, ids)
    e.eval_tokens(ids)
    for w, c in ctxs.items(): assert np.array_equal(ext.logits(c), e.logits), w
    for step in range(16):
        want = int(np.argmax(e.logits))
        for w, c in ctxs.items():
            assert ext.greedy_id(c) == want, (w, step)
            ext.eval_tokens(c, [want])
        e.eval_tokens([want])
        for w, c in ctxs.items(): assert np.array_equal(ext.logits(c), e.logits), (w, step)
    for c in ctxs.values(): ext.base.minigpt4_free(c)
