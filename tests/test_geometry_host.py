"""LLaMA geometries at the edges of the decode-megakernel and prefill-GEMM gates, host side (no GPU).

CASES is the table tests/test_geometry_gpu.py runs: each file's geometry, the gate or tier it is there for, and the path the load must
choose on an H100 (decode megakernel yes / no, tensor-core prefill yes / no, and the megakernel's stream warps).  The rules of
LlamaDevice::build_mega and build_prefill (csrc/llama.cu) are restated here in Python, so the expected paths are written down once and can
be read without a GPU; the GPU module asserts the load against the same functions.

The oracle the GPU paths are compared with bit for bit is itself checked here against a plain float64 LLaMA forward at two of these
geometries (n_embd 1280 with 32001 tokens, n_embd 256 with 259 tokens), where no other test looks at it."""
from dataclasses import dataclass, field

import numpy as np
import pytest

N_CTX = 777            # not a power of two: the attention scratch and KV planes of every case are off the usual sizes
SMEM_OPTIN_H100 = 227 * 1024
SM_COUNT_H100 = 132
K_MAX_OPS = 7 * 80 + 3     # mk6::kMaxOps: the op table holds the tensor-parallel program (7 ops per layer) of up to 80 layers
MEGA_TOK_TYPES = ("f32", "f16", "q4_0", "q4_1", "q5_k", "q6_k")   # token embeddings the megakernel's embed op decodes


@dataclass(frozen=True)
class Case:
    spec: dict             # modelgen.LlamaSpec fields
    probes: str            # the gate or tier the case is there for
    mega: bool             # the decode megakernel must take the file
    gemm: bool             # the tensor-core prefill must take the file
    w_h100: int = 0        # stream warps the megakernel must choose on an H100 (227 KB opt-in shared memory, n_ctx 777)
    n_ctx: int = N_CTX
    extra: dict = field(default_factory=dict)


def _g(n_vocab, n_embd, n_mult, n_layer, wtype):
    return dict(n_vocab=n_vocab, n_embd=n_embd, n_head=n_embd // 128, n_mult=n_mult, n_layer=n_layer, wtype=wtype)


CASES = {
    "e256-q4_1": Case(_g(259, 256, 32, 2, "q4_1"), "smallest width: wo (128 row pairs), down (128) and output (130) have fewer row pairs than "
                      "the grid has CTAs; odd vocabulary (259, the least make_vocab allows); n_ff 704 = 22 blocks, prefill classes 22..31 empty",
                      True, True, 15),
    "e256-q4_0": Case(_g(259, 256, 32, 2, "q4_0"), "as e256-q4_1 with Q4_0 rows (144 / 400 B: the other slot size)", True, True, 15),
    "e1280": Case(_g(32001, 1280, 32, 2, "q4_1"), "RMS divisor 1280 (not a power of two) below 4096; n_ff 3424 = 107 blocks (odd, not a multiple "
                  "of 64 or 256); 32001 tokens", True, True, 15),
    "e4352": Case(_g(32001, 4352, 32, 1, "q4_1"), "just past both staging tiers (RMS-normed 4352 > 4096: 5 items per thread, un-normed n_ff 11616 > "
                  "11520: 8 items); no register-resident blocks above 4096; 34 attention CTAs", True, True, 14),
    "e4352-q5k": Case(_g(2048, 4352, 256, 1, "q5_k"), "Q5_K staging over 17 and 46 super-blocks per row", True, False, 12),
    "7b-32001-q4_1": Case(_g(32001, 4096, 256, 2, "q4_1"), "the 7B Q4_1 download layout: 4 register-resident blocks per lane with an odd "
                          "vocabulary", True, True, 15),
    "7b-32001-q4_0": Case(_g(32001, 4096, 256, 2, "q4_0"), "the 7B Q4_0 download layout", True, True, 15),
    "deep80": Case(_g(259, 256, 32, 80, "q4_1"), "80 layers: the last program that fits the op table (7 x 80 + 3 ops)", True, True, 15),
    "deep81": Case(_g(259, 256, 32, 81, "q4_1"), "81 layers: the first program that must fall back to the per-op decode graph", False, True),
    "e640": Case(_g(1001, 640, 256, 2, "q4_1"), "just outside the n_embd % 256 gate: per-op decode, GEMM prefill", False, True),
}


def n_ff(spec: dict) -> int:
    """LlamaSpec.n_ff: 8 E / 3 rounded up to a multiple of n_mult"""
    E, m = spec["n_embd"], spec.get("n_mult", 256)
    return ((2 * (4 * E) // 3 + m - 1) // m) * m


def _types(spec: dict) -> tuple[set, str, str]:
    """(types of the layer matrices, output type, token-embedding type) of a file without overrides"""
    wt = spec["wtype"]
    assert not spec.get("overrides")
    return {wt}, spec.get("output_type") or wt, spec.get("tok_type") or wt


def _row_bytes(wt: str, cols: int) -> int:   # device row of a megakernel matrix (16-byte padded Q4 rows, row-packed Q5_K)
    return {"q4_0": (cols // 32 * 18 + 15) & ~15, "q4_1": (cols // 32 * 20 + 15) & ~15, "q5_k": cols // 256 * 176}[wt]


def mega_plan(spec: dict, n_ctx: int, smem_optin: int = SMEM_OPTIN_H100, sm_count: int = SM_COUNT_H100, w_cap: int = 15):
    """the megakernel configuration build_mega chooses on one GPU, or None when it refuses the file:
    (ops per token, stream warps W, slot bytes, activation bytes, register-resident blocks per lane)"""
    E, FF, L = spec["n_embd"], n_ff(spec), spec["n_layer"]
    layer_types, out_t, tok_t = _types(spec)
    if out_t not in ("q4_0", "q4_1", "q5_k") or layer_types != {out_t} or tok_t not in MEGA_TOK_TYPES:
        return None
    if E % 256 or FF % 32 or E > 1024 * 5 or FF > 4 * 480 * 8:          # RMS staging <= 5 items, plain staging <= 8 items per thread
        return None
    if E // 128 > sm_count or 7 * L + 3 > K_MAX_OPS:                      # one attention CTA per head; the op table
        return None
    wt = out_t
    if wt == "q5_k":
        if E % 256 or FF % 256 or FF > 256 * 15 * 4 or E > 256 * 15 * 2:
            return None
        act = max(((c + c // 256 * 4 + c // 16 * 2) + 15) & ~15 for c in (E, FF))   # Q8_K: int8 q, float d per 256, int16 sums per 16
    else:
        act = max(c + 64 + c // 32 * 8 for c in (E, FF))                           # Q8_0 / Q8_1 planes + 64 B pad + {d, s} per block
    act = (max(act, 6 * n_ctx) + 127) & ~127
    rb_e, rb_ff = _row_bytes(wt, E), _row_bytes(wt, FF)
    slot = (max(2 * rb_e, rb_ff) + 15) & ~15
    for rb in (rb_e, rb_ff):   # every slot-load a 16-byte multiple (the `uniform` rule)
        parts = 1 if 2 * rb <= slot else 2
        if (2 * rb // parts) % 16:
            return None
    W = min(15, w_cap, (smem_optin - 10240 - act - 2 * 15 * 8) // (2 * slot))
    if W < 4:
        return None
    nbl = 0 if wt == "q5_k" else {4096: 4, 5120: 5}.get(E, 0)
    return 5 * L + 3, W, slot, act, nbl


def prefill_gemm(spec: dict) -> bool:
    """build_prefill: every layer has one fused q / k / v matrix and Q4_0 / Q4_1 qkv, wo, w13 and w2 (output and token embedding may be
    anything); the operand cache fits in memory (it does, for every file here)"""
    layer_types, _, _ = _types(spec)
    return layer_types <= {"q4_0", "q4_1"}


def pf_slots(cols: int) -> int:
    """slots per class of the class-major prefill operand cache (a multiple of 4)"""
    return 4 * (((cols // 32 + 31) // 32 + 3) // 4)


# ---- the case table is right ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(CASES))
def test_case_arithmetic(name):
    c = CASES[name]
    s = c.spec
    assert s["n_embd"] == 128 * s["n_head"], "head_dim 128 (load refuses anything else)"
    assert s["n_vocab"] >= 259, "make_vocab needs the 3 specials and 256 byte tokens"
    plan = mega_plan(s, c.n_ctx)
    assert (plan is not None, prefill_gemm(s)) == (c.mega, c.gemm), name
    if plan is not None:
        assert plan[1] == c.w_h100, plan


def test_geometry_numbers():
    """the numbers each case's probe rests on"""
    ff = {k: n_ff(c.spec) for k, c in CASES.items()}
    assert ff["e256-q4_1"] == 704 and 704 // 32 == 22
    assert ff["e1280"] == 3424 and 3424 // 32 == 107 and 3424 % 64 and 3424 % 256
    assert ff["e4352"] == 11616 and 11616 > 4 * 480 * 6 and 4352 > 4096 and 4352 <= 4 * 480 * 3
    assert ff["e4352-q5k"] == 11776 and (4352 // 256, 11776 // 256) == (17, 46)
    assert ff["7b-32001-q4_1"] == 11008 and ff["e640"] == 1792 and 640 % 256
    assert 7 * 80 + 3 == K_MAX_OPS < 7 * 81 + 3
    # fewer row pairs than CTAs at n_embd 256: wo / down 128, output (259 rows padded to 260) 130
    assert 256 // 2 < SM_COUNT_H100 and (259 + 1) // 2 < SM_COUNT_H100
    # classes of the prefill cache: 22 blocks fill classes 0..21 once, 107 blocks fill 0..10 four times and 11..31 three times
    assert pf_slots(704) == 4 and pf_slots(3424) == 4 and pf_slots(11616) == 12 and pf_slots(4352) == 8
    assert mega_plan(CASES["e4352"].spec, N_CTX)[4] == 0 and mega_plan(CASES["7b-32001-q4_1"].spec, N_CTX)[4] == 4


def test_gates_refuse_what_they_must():
    base = CASES["e256-q4_1"].spec
    assert mega_plan(dict(base, wtype="q5_k", n_mult=256), N_CTX) is not None
    assert mega_plan(dict(base, output_type="q6_k"), N_CTX) is None
    assert mega_plan(dict(base, tok_type="q8_0"), N_CTX) is None
    assert mega_plan(dict(base, n_embd=5248, n_head=41), N_CTX) is None           # RMS staging holds 5120 at most
    assert mega_plan(dict(base, n_layer=81), N_CTX) is None and mega_plan(dict(base, n_layer=80), N_CTX)[0] == 403
    assert not prefill_gemm(dict(base, wtype="q5_k")) and prefill_gemm(dict(base, output_type="q6_k"))


# ---- the oracle against a float64 LLaMA at two of these geometries ----------------------------------------------------------------------
def _rms(x, w):
    return x / np.sqrt(np.mean(x * x, axis=-1, keepdims=True) + 1e-6) * w


def _rope_table(n_pos: int) -> np.ndarray:
    """[n_pos][64] angles, formed as the engine and ggml form them: float32 theta, multiplied by the float32 scale per pair"""
    scale = np.float32(10000.0 ** (-2.0 / 128.0))
    out = np.zeros((n_pos, 64))
    for p in range(n_pos):
        th = np.float32(p)
        for i in range(64):
            out[p, i] = th
            th = np.float32(th * scale)
    return out


def _rope(x, pos, ang):   # mode 0: adjacent pairs (2 i, 2 i + 1) of every 128-wide head
    y = x.reshape(x.shape[0], -1, 64, 2)
    c, s = np.cos(ang[pos])[:, None, :], np.sin(ang[pos])[:, None, :]
    a, b = y[..., 0], y[..., 1]
    return np.stack([a * c - b * s, a * s + b * c], axis=-1).reshape(x.shape)


def llama_forward_f64(path: str, ids: list[int]) -> np.ndarray:
    """logits of the last row of a float64 LLaMA forward: weights dequantised by gguf-py, K and V rounded to F16 as the cache holds them"""
    import gguf
    import gguf.quants as gq
    from oracle import oracle
    hp, _, t = oracle.read_ggjt(path)
    E, H = hp["n_embd"], hp["n_head"]

    def w(name, rows=None):
        tv = t[name]
        raw = np.asarray(tv.data).reshape(tv.ne[1], -1)
        if rows is not None:
            raw = raw[rows]
        return gq.dequantize(raw, gguf.GGMLQuantizationType(tv.gtype)).astype(np.float64)

    def v(name):
        return np.asarray(t[name].data).view(np.float32).astype(np.float64)

    n = len(ids)
    ang = _rope_table(n)
    pos = np.arange(n)
    x = w("tok_embeddings.weight", np.asarray(ids))
    for il in range(hp["n_layer"]):
        p = f"layers.{il}."
        h = _rms(x, v(p + "attention_norm.weight"))
        q = _rope(h @ w(p + "attention.wq.weight").T, pos, ang)
        k = _rope(h @ w(p + "attention.wk.weight").T, pos, ang).astype(np.float16).astype(np.float64)
        vv = (h @ w(p + "attention.wv.weight").T).astype(np.float16).astype(np.float64)
        att = np.zeros_like(q)
        for hd in range(H):
            c = slice(128 * hd, 128 * hd + 128)
            s = q[:, c] @ k[:, c].T / np.sqrt(128.0)
            s[np.triu_indices(n, 1)] = -np.inf
            e = np.exp(s - s.max(axis=1, keepdims=True))
            att[:, c] = (e / e.sum(axis=1, keepdims=True)) @ vv[:, c]
        x = x + att @ w(p + "attention.wo.weight").T
        h = _rms(x, v(p + "ffn_norm.weight"))
        g, u = h @ w(p + "feed_forward.w1.weight").T, h @ w(p + "feed_forward.w3.weight").T
        x = x + (g / (1.0 + np.exp(-g)) * u) @ w(p + "feed_forward.w2.weight").T
    h = _rms(x[-1:], v("norm.weight"))
    return (h @ w("output.weight").T)[0]


@pytest.mark.parametrize("name", ["e1280", "e256-q4_1"])
def test_oracle_matches_float64_llama(orc, mg, tmp_path, name):
    """one layer, a 13-token prompt that ends on the last token id: relative error under 2e-2 (the Q8 activation quantisation of ggml's
    quantised mul_mat, as in test_golden.py) and the same arg-max"""
    spec = dict(CASES[name].spec, n_layer=1)
    path = str(tmp_path / f"{name}-1l.bin")
    mg.write_llama_ggjt(path, mg.LlamaSpec(**spec))
    V = spec["n_vocab"]
    ids = np.random.default_rng(5).integers(3, V, size=12).tolist() + [V - 1]
    e = orc.OracleEngine(None, path, n_ctx=64)
    got = e.eval_tokens(ids).astype(np.float64)
    want = llama_forward_f64(path, ids)
    assert got.shape == want.shape == (V,)
    err = float(np.abs(got - want).max() / np.abs(want).max())
    assert err < 2e-2, err
    assert int(np.argmax(got)) == int(np.argmax(want))
    print(f"{name}: oracle vs float64 rel err {err:.2e}")
