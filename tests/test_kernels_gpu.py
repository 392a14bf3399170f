"""Kernel-level parity (GPU): each production CUDA kernel, driven through the C ABI, against the CPU oracle op
(the oracle replaces the 'plain PyTorch reference' for this tier).  Language-path kernels share the oracle's canonical
float reduction order and must be BIT-IDENTICAL; tensor-core GEMMs differ by accumulation order only (tolerances stated)."""
import math

import numpy as np
import pytest

from conftest import rel_err

pytestmark = pytest.mark.gpu

TYPES = {"q4_0": 2, "q4_1": 3, "q5_k": 13, "q6_k": 14, "f16": 1}


@pytest.mark.parametrize("wt", list(TYPES))
@pytest.mark.parametrize("shape", [(64, 512), (130, 4096), (48, 11008), (33, 256)])
@pytest.mark.parametrize("n", [1, 3, 8, 11])
def test_matvec_matches_oracle(ext, orc, mg, wt, shape, n):
    rows, cols = shape
    gt = TYPES[wt]
    rng = np.random.default_rng(rows * 7 + cols + n)
    raw = mg.synth_quant(rng, gt, rows, cols, 0.02)
    x = rng.standard_normal((n, cols)).astype(np.float32)
    x[0, :32] = 0.0  # an all-zero block (amax == 0 path)
    want = orc.mul_mat(gt, raw, rows, cols, x)
    got = ext.op_matvec(gt, raw, rows, cols, x)
    assert got.shape == want.shape
    assert np.array_equal(got, want)  # canonical reduction order on both sides -> bit-identical


def test_matvec_ragged_and_extreme(ext, orc, mg):
    rng = np.random.default_rng(5)
    raw = mg.synth_quant(rng, 3, 2, 32, 0.5)  # smallest legal matrix: 2 rows x one block
    x = np.array([[1e4] * 16 + [-1e-4] * 16], np.float32)
    assert np.array_equal(ext.op_matvec(3, raw, 2, 32, x), orc.mul_mat(3, raw, 2, 32, x))
    x0 = np.zeros((1, 32), np.float32)
    assert np.all(ext.op_matvec(3, raw, 2, 32, x0) == 0)


# ---- vision: wgmma GEMM --------------------------------------------------------------------------------------------------------
GE_BIAS, GE_QSCALE, GE_GELU, GE_RESID, GE_PATCH = 0, 1, 2, 3, 4
SENTINEL = -1234.0   # pre-filled into every output buffer (exact in F16 and F32): an element the kernel must not write comes back as this
U24 = 2.0 ** -24     # F32 unit roundoff
# |got - exact| <= C_GEMM * 2^-24 * (sum_k |w x| + |bias| + |resid| + |pos|) per element, exact = float64 sum of the exact F16 x F16 products:
# the accumulation-order error of the tensor-core F32 sums plus the F32 epilogue adds.  Measured on an H100 80GB HBM3 (700 W limit): at most
# 8.7 over every production shape and edge token count (K 6144 split-K slices and K 3072 highest, 3-5 at K 512); pinned with a 1.8x margin.
C_GEMM = 16.0


def _gemm_operands(rng, M, T, K):
    w = (rng.standard_normal((M, K)) * 0.02).astype(np.float16)
    x = rng.standard_normal((T, K)).astype(np.float16)
    bias = (rng.standard_normal(M) * 0.02).astype(np.float32)
    return w, x, bias


def _exact(w, x, k0=0, k1=None):
    """float64 sum of the exact F16 x F16 products over k0..k1, and the sum of their magnitudes"""
    xd, wd = x[:, k0:k1].astype(np.float64), w[:, k0:k1].astype(np.float64)
    return xd @ wd.T, np.abs(xd) @ np.abs(wd).T


def _gemm_c(got, want, mag):
    """the measured c of |got - want| <= c * 2^-24 * mag"""
    return float((np.abs(got.astype(np.float64) - want) / (U24 * mag)).max())


def _check_gemm(ext, M, K, T, epi, ksplit=1, in_place=False, tsplit=True, seed=0, expect_plan=None):
    rng = np.random.default_rng(seed or (M * 7 + K * 3 + T + epi))
    w, x, bias = _gemm_operands(rng, M, T, K)
    exact, mag = _exact(w, x)
    rows = T + 1 + (epi == GE_PATCH)
    dt = np.float16 if epi == GE_GELU else np.float32
    out = np.full((ksplit, rows, M), SENTINEL, dt)
    aux, qscale, qrows = None, 1.0, 0
    if epi == GE_QSCALE:
        qscale, qrows = 1.0 / math.sqrt(88.0), M // 3       # the ViT qkv: q rows scaled by 1 / sqrt(head_dim)
    if epi == GE_RESID:
        resid = rng.standard_normal((T, M)).astype(np.float32)
        if in_place:
            out[0, :T] = resid
        else:
            aux = resid
    if epi == GE_PATCH:
        aux = (rng.standard_normal((T + 1, M)) * 0.02).astype(np.float32)
    got, plan = ext.op_gemm_f16(w, x, bias, epi, aux=aux, qscale=qscale, qscale_rows=qrows, ksplit=ksplit, tsplit=tsplit, in_place=in_place,
                                out=out, plan=True)
    nt, gy, gz, kb = plan
    if expect_plan:
        assert plan == expect_plan, plan
    assert gy == -(-T // nt)
    b64 = bias.astype(np.float64)
    if gz > 1:   # split-K: slice z holds the raw sum over its own k-blocks (+ bias on slice 0) and nothing else
        worst = 0.0
        for z in range(gz):
            e, m = _exact(w, x, z * kb * 64, min(K, (z + 1) * kb * 64))
            want = e + (b64 if z == 0 else 0.0)
            m = m + (np.abs(b64) if z == 0 else 0.0)
            worst = max(worst, _gemm_c(got[z, :T], want, m))
            assert np.all(got[z, T:] == SENTINEL), f"slice {z}: a row past T was written"
        assert np.all(got[gz:] == SENTINEL), "a slice past grid.z was written"
        print(f"MEASURE gemm {M}x{K} T{T} epi{epi} split-K {gz}: c = {worst:.3f}")
        assert worst <= C_GEMM, worst
        return
    assert np.all(got[1:] == SENTINEL)
    g = got[0]
    if epi == GE_GELU:
        # the LUT is indexed by the F16-rounded pre-activation, which the GEMM bound places within +-d of the exact one: the result must be a
        # LUT value of that index range (near zero the range spans several F16 ulps), and it is the exact index's value on > 99 % of the entries
        pre, d = exact + b64, C_GEMM * U24 * (mag + np.abs(b64))
        lut = orc_table(0).view(np.float16)
        at = lambda h: lut[h.view(np.uint16)].astype(np.float32)
        lo, mid, hi = at((pre - d).astype(np.float16)), at(pre.astype(np.float32).astype(np.float16)), at((pre + d).astype(np.float16))
        got16 = g[:T].astype(np.float32)
        inside = (got16 >= np.minimum(np.minimum(lo, mid), hi)) & (got16 <= np.maximum(np.maximum(lo, mid), hi))
        frac = float(np.mean(got16 != mid))
        print(f"MEASURE gemm {M}x{K} T{T} gelu: {frac:.4%} of the entries off the exact LUT index")
        assert frac < 1e-2 and np.all(inside), (frac, int(np.sum(~inside)))
        assert np.all(g[T] == SENTINEL)
        return
    if epi == GE_PATCH:
        assert np.all(g[0] == SENTINEL), "row 0 belongs to the CLS kernel"
        want, m = (exact + b64) + aux[1:], mag + np.abs(b64) + np.abs(aux[1:])
        body, guard = g[1:T + 1], g[T + 1]
    else:
        want, m = exact + b64, mag + np.abs(b64)
        if epi == GE_QSCALE:
            s = np.where(np.arange(M) < qrows, qscale, 1.0)
            want, m = want * s, m * s
        if epi == GE_RESID:
            r = resid.astype(np.float64)
            want, m = want + r, m + np.abs(r)
        body, guard = g[:T], g[T]
    c = _gemm_c(body, want, m)
    print(f"MEASURE gemm {M}x{K} T{T} epi{epi}{' in-place' if in_place else ''}{'' if tsplit else ' plain grid'}: c = {c:.3f}")
    assert c <= C_GEMM, c
    assert np.all(guard == SENTINEL), "the guard row past T was written"
    if epi == GE_QSCALE:   # the scale stops exactly at qscale_rows
        assert np.all(np.abs(body[:, qrows:] - want[:, qrows:]) <= C_GEMM * U24 * m[:, qrows:])


def orc_table(which):
    from oracle import oracle
    return oracle.table(which)


# Every GEMM load() plans, at its production shape, epilogue and grid: (name, M, K, T, epi, ksplit, in_place, expected plan)
PRODUCTION_GEMMS = [
    ("patch", 1408, 640, 256, GE_PATCH, 1, False, (256, 1, 1, 0)),
    ("vit_qkv", 4224, 1408, 257, GE_QSCALE, 1, False, None),
    ("vit_proj_splitk", 1408, 1408, 257, GE_RESID, 3, False, (80, 4, 3, 8)),
    ("vit_proj_in_place", 1408, 1408, 257, GE_RESID, 1, True, None),
    ("vit_fc1", 6144, 1408, 257, GE_GELU, 1, False, None),
    ("vit_fc2_splitk", 1408, 6144, 257, GE_RESID, 3, False, (80, 4, 3, 32)),
    ("qf_self_qkv", 2304, 768, 32, GE_BIAS, 1, False, (32, 1, 1, 0)),
    ("qf_dense", 768, 768, 32, GE_RESID, 1, False, (32, 1, 1, 0)),
    ("qf_cross_kv", 1536, 1408, 257, GE_BIAS, 1, False, None),
    ("qf_ff1", 3072, 768, 32, GE_GELU, 1, False, None),
    ("qf_ff2", 768, 3072, 32, GE_RESID, 1, False, None),
    ("llama_proj_7b", 4096, 768, 32, GE_BIAS, 1, False, None),
    ("llama_proj_13b", 5120, 768, 32, GE_BIAS, 1, False, None),
]


@pytest.mark.parametrize("name,M,K,T,epi,ksplit,in_place,plan", PRODUCTION_GEMMS, ids=[g[0] for g in PRODUCTION_GEMMS])
def test_wgmma_gemm_production_shapes(ext, name, M, K, T, epi, ksplit, in_place, plan):
    _check_gemm(ext, M, K, T, epi, ksplit=ksplit, in_place=in_place, expect_plan=plan)


@pytest.mark.parametrize("T", [1, 31, 33, 79, 81, 128, 129, 143, 145, 255, 257, 272])
@pytest.mark.parametrize("cfg", ["qscale", "resid_splitk", "resid_in_place", "bias_plain_grid"])
def test_wgmma_gemm_edge_tokens(ext, cfg, T):
    """token counts on both sides of every token tile (32 / 80 / 144 / 256), of the token split (T > 128) and of the split-K switch"""
    if cfg == "qscale":
        _check_gemm(ext, 384, 640, T, GE_QSCALE)
    elif cfg == "resid_splitk":
        _check_gemm(ext, 1408, 1408, T, GE_RESID, ksplit=3)
    elif cfg == "resid_in_place":
        _check_gemm(ext, 256, 512, T, GE_RESID, in_place=True)
    else:
        _check_gemm(ext, 256, 512, T, GE_BIAS, tsplit=False)


def test_wgmma_gemm_token_split_is_bit_identical(ext):
    """the token split only moves tokens between CTAs: every element keeps its k order"""
    rng = np.random.default_rng(9)
    w, x, bias = _gemm_operands(rng, 1536, 257, 1408)
    a, pa = ext.op_gemm_f16(w, x, bias, GE_BIAS, tsplit=True, plan=True)
    b, pb = ext.op_gemm_f16(w, x, bias, GE_BIAS, tsplit=False, plan=True)
    assert pa[1] > pb[1] and np.array_equal(a, b)


def test_wgmma_gemm_refuses_out_of_range(ext):
    assert ext.op_gemm_f16_rc(128, 16, 64) == 0
    for M, T, K in [(130, 16, 64), (128, 16, 96), (128, 0, 64), (128, 273, 64)]:
        assert ext.op_gemm_f16_rc(M, T, K) == 8, (M, T, K)
    assert ext.op_gemm_f16_rc(128, 16, 64, epi=5) == 8        # GE_PARTIAL is planned, not requested
    assert ext.op_gemm_f16_rc(128, 16, 64, epi=GE_BIAS, ksplit=3) == 8
    assert ext.op_gemm_f16_rc(128, 16, 64, epi=GE_RESID, aux=False) == 8
    assert ext.op_gemm_f16_rc(128, 16, 64, epi=GE_PATCH, aux=False) == 8
    assert ext.op_gemm_f16_rc(128, 16, 64, epi=GE_BIAS, in_place=True) == 8


@pytest.mark.parametrize("M,T,K", [(128, 16, 64), (256, 32, 768), (1408, 257, 1408), (128, 257, 6144), (768, 256, 640), (384, 100, 128)])
def test_wgmma_gemm_matches_oracle(ext, orc, M, T, K):
    rng = np.random.default_rng(M + T + K)
    w = (rng.standard_normal((M, K)) * 0.05).astype(np.float16)
    x = rng.standard_normal((T, K)).astype(np.float16)
    bias = rng.standard_normal(M).astype(np.float32)
    want = orc.mul_mat(1, w.view(np.uint8).reshape(M, -1), M, K, x.astype(np.float32)) + bias
    got = ext.op_gemm_f16(w, x, bias, 0)
    assert rel_err(got, want) < 1e-5  # F16 products are exact in F32; accumulation order only


def test_wgmma_gemm_gelu_epilogue(ext, orc):
    rng = np.random.default_rng(3)
    M, T, K = 256, 257, 512
    w = (rng.standard_normal((M, K)) * 0.05).astype(np.float16)
    x = rng.standard_normal((T, K)).astype(np.float16)
    bias = rng.standard_normal(M).astype(np.float32)
    pre = orc.mul_mat(1, w.view(np.uint8).reshape(M, -1), M, K, x.astype(np.float32)) + bias
    want = orc.gelu(pre)
    got = ext.op_gemm_f16(w, x, bias, 2)
    # the fp16 LUT makes the op discontinuous at F16 rounding boundaries: allow 1 F16 ulp on <1 % of entries (measured 0.27 %)
    diff = np.abs(got - want)
    assert np.mean(diff > 0) < 1e-2 and diff.max() <= np.abs(want).max() * 2 ** -9


# ---- vision: LayerNorm ----------------------------------------------------------------------------------------------------------
def test_layernorm_matches_oracle(ext, orc):
    rng = np.random.default_rng(1)
    x = (rng.standard_normal((257, 1408)) * 3 + 0.5).astype(np.float32)
    w = rng.standard_normal(1408).astype(np.float32); b = rng.standard_normal(1408).astype(np.float32)
    assert rel_err(ext.op_layernorm(x, w, b), orc.layernorm(x, w, b)) < 1e-6


def _ln_rows(rng, kind, rows, n):
    if kind == "production":
        return (rng.standard_normal((rows, n)) * 3 + 0.5).astype(np.float32)
    if kind == "large_mean":       # mean ~1e3, spread ~1e-2: the centring must happen in F32 after an exact mean
        return (1e3 + 1e-2 * rng.standard_normal((rows, n))).astype(np.float32)
    if kind == "constant":         # zero variance: the output is the bias
        return np.full((rows, n), 0.37, np.float32) * rng.uniform(-2, 2, (rows, 1)).astype(np.float32)
    # values from 2^-20 to 2^20: the double sums are no longer exact, so their order shows
    return (rng.choice([-1.0, 1.0], (rows, n)) * np.exp2(rng.uniform(-20, 20, (rows, n))) * rng.uniform(1, 2, (rows, n))).astype(np.float32)


@pytest.mark.parametrize("kind", ["production", "large_mean", "constant", "wide_exponents"])
@pytest.mark.parametrize("rows", [1, 32, 257])
@pytest.mark.parametrize("n", [768, 1000, 1408, 1536])
def test_layernorm_shapes_and_inputs(ext, orc, n, rows, kind):
    rng = np.random.default_rng(n * 3 + rows + len(kind))
    x = _ln_rows(rng, kind, rows, n)
    w = (1.0 + 0.02 * rng.standard_normal(n)).astype(np.float32); b = (0.02 * rng.standard_normal(n)).astype(np.float32)
    got32, got16 = ext.op_layernorm(x, w, b, f16=True, f32=True)   # one launch writes both, as the Q-Former's LayerNorms do
    want = orc.layernorm(x, w, b)
    assert np.array_equal(got16, got32.astype(np.float16))
    if kind != "wide_exponents":   # both sides sum in double, exactly for this exponent spread: the order of the sums does not matter
        assert np.array_equal(got32, want), float(np.abs(got32 - want).max())
        assert np.array_equal(got16, want.astype(np.float16))
    else:
        ulps = np.abs(got32.astype(np.float64) - want) / np.spacing(np.abs(want)).astype(np.float64)
        # measured on an H100 80GB HBM3: 0 % of the outputs off (the double sums happen to round the same way at every shape here)
        print(f"MEASURE layernorm n{n} rows{rows} wide exponents: {np.mean(ulps > 0):.4%} of the outputs 1 ulp off, max {ulps.max():.0f}")
        assert ulps.max() <= 1


def test_layernorm_refuses_out_of_range(ext):
    assert ext.op_layernorm_rc(2, 1536) == 0
    assert ext.op_layernorm_rc(2, 1537) == 8 and ext.op_layernorm_rc(2, 0) == 8 and ext.op_layernorm_rc(0, 768) == 8


@pytest.mark.parametrize("rows,n,n_parts", [(257, 1408, 3), (257, 1408, 2), (1, 1408, 4), (32, 1000, 3)])
def test_layernorm_fold_matches_numpy(ext, orc, rows, n, n_parts):
    """the LayerNorm after a split-K residual GEMM folds the slices into the residual stream in slice order"""
    rng = np.random.default_rng(rows + n + n_parts)
    x = (rng.standard_normal((rows, n)) * 4).astype(np.float32)
    parts = (rng.standard_normal((n_parts, rows, n)) * np.array([1.0, 1e-3, 30.0, 0.5][:n_parts])[:, None, None]).astype(np.float32)
    w = (1.0 + 0.02 * rng.standard_normal(n)).astype(np.float32); b = (0.02 * rng.standard_normal(n)).astype(np.float32)
    folded, y16 = ext.op_layernorm_fold(x, parts, w, b)
    want = x.copy()
    for p in parts:
        want = want + p          # float32, one slice after the other
    assert np.array_equal(folded, want)
    assert np.array_equal(y16, orc.layernorm(want, w, b).astype(np.float16))


# ---- vision: attention ----------------------------------------------------------------------------------------------------------
# per output row: max_d |got - ref| / max_d |ref| against float64 scores with the fp16-LUT softmax; the output is F16 and an F16 rounding
# flip of one score's exp index moves one probability by an F16 ulp.  Measured on an H100 80GB HBM3 (700 W limit): worst row 6.7e-4 over
# every case below (ViT 4.8e-4 .. 6.7e-4, Q-Former 4.2e-4 .. 5.6e-4); pinned with a 2.2x margin.
ATTN_ROW_BOUND = 1.5e-3


def _attn_ref(q, k, v, div, tab):
    s = (q.astype(np.float64) @ k.astype(np.float64).T) / div
    idx = (s - s.max(axis=1, keepdims=True)).astype(np.float16).view(np.uint16)
    e = tab[idx].view(np.float16).astype(np.float64)
    return (e @ v.astype(np.float64)) / e.sum(axis=1, keepdims=True)


def _check_attention(ext, orc, buf, q_off, ldq, k_off, v_off, ldkv, nq, nk, heads, dh, div, qpc, seed):
    out = np.full((nq + 1, heads * dh), SENTINEL, np.float32)
    got = ext.op_attention_packed(buf, q_off, ldq, k_off, v_off, ldkv, nq, nk, heads, dh, div, q_per_cta=qpc, out=out)
    assert np.all(got[nq] == SENTINEL), "the guard row past nq was written"
    tab = orc.table(2)
    worst = 0.0
    for h in range(heads):
        c = slice(h * dh, (h + 1) * dh)
        rows = lambda off, ld, n: buf[off + np.arange(n)[:, None] * ld + h * dh + np.arange(dh)[None, :]]
        ref = _attn_ref(rows(q_off, ldq, nq), rows(k_off, ldkv, nk), rows(v_off, ldkv, nk), div, tab)
        err = np.abs(got[:nq, c] - ref).max(axis=1) / np.abs(ref).max(axis=1)
        worst = max(worst, float(err.max()))
    print(f"MEASURE attention nq{nq} nk{nk} heads{heads}x{dh} qpc{qpc}: worst row {worst:.3e}")
    assert worst <= ATTN_ROW_BOUND, worst


@pytest.mark.parametrize("nq", [257, 233, 234, 235])
def test_attention_vit_packed_qkv(ext, orc, nq):
    """the ViT launch: 16 heads of 88 read from the packed [T][3 D] qkv GEMM output, 29 queries per CTA (9 chunks)"""
    D, nk = 1408, 257
    rng = np.random.default_rng(nq)
    qkv = rng.standard_normal((max(nq, nk), 3 * D)).astype(np.float32)
    qkv[:, :D] *= 0.3
    _check_attention(ext, orc, qkv.reshape(-1), 0, 3 * D, D, 2 * D, 3 * D, nq, nk, 16, 88, 1.0, 29, nq)


@pytest.mark.parametrize("nq", [32, 29, 30, 31])
def test_attention_qformer_self_packed_qkv(ext, orc, nq):
    """the Q-Former self-attention: 12 heads of 64 from the packed [32][3 x 768] buffer, all queries in one CTA per head"""
    rng = np.random.default_rng(100 + nq)
    qkv = rng.standard_normal((32, 3 * 768)).astype(np.float32)
    _check_attention(ext, orc, qkv.reshape(-1), 0, 3 * 768, 768, 1536, 3 * 768, nq, 32, 12, 64, 8.0, 32, nq)


@pytest.mark.parametrize("nq,nk", [(32, 257), (32, 1), (32, 31), (32, 32), (32, 33), (32, 288), (29, 257), (30, 257), (31, 257)])
def test_attention_qformer_cross_packed_kv(ext, orc, nq, nk):
    """the cross-attention: q [32][768] against the packed [T][2 x 768] key / value GEMM output, 16 queries per CTA"""
    rng = np.random.default_rng(200 + nq * 300 + nk)
    q = rng.standard_normal((nq, 768)).astype(np.float32)
    kv = rng.standard_normal((nk, 2 * 768)).astype(np.float32)
    buf = np.concatenate([q.reshape(-1), kv.reshape(-1)])
    _check_attention(ext, orc, buf, 0, 768, nq * 768, nq * 768 + 768, 1536, nq, nk, 12, 64, 8.0, 16, nq + nk)


def test_attention_refuses_out_of_range(ext):
    assert ext.op_attention_rc(32, 288, 12, 64) == 0
    assert ext.op_attention_rc(32, 289, 12, 64) == 8
    assert ext.op_attention_rc(32, 257, 16, 88) == 0
    assert ext.op_attention_rc(32, 288, 16, 88) == 8       # more keys than the head_dim-88 kernel holds in shared memory
    assert ext.op_attention_rc(32, 32, 12, 72) == 8
    assert ext.op_attention_rc(32, 0, 12, 64) == 8


@pytest.mark.parametrize("nq,nk,heads,dh,div", [(257, 257, 16, 88, 1.0), (32, 32, 12, 64, 8.0), (32, 257, 12, 64, 8.0)])
def test_attention_matches_oracle(ext, orc, nq, nk, heads, dh, div):
    rng = np.random.default_rng(nq + nk)
    q = rng.standard_normal((nq, heads * dh)).astype(np.float32) * (0.3 if div == 1.0 else 1.0)
    k = rng.standard_normal((nk, heads * dh)).astype(np.float32)
    v = rng.standard_normal((nk, heads * dh)).astype(np.float32)
    got = ext.op_attention(q, k, v, heads, dh, div)
    want = np.empty_like(q)
    for h in range(heads):
        sl = slice(h * dh, (h + 1) * dh)
        s = (q[:, sl] @ k[:, sl].T) / div
        p = orc.softmax(s.astype(np.float32))
        want[:, sl] = p @ v[:, sl]
    want = want.astype(np.float16).astype(np.float32)
    assert rel_err(got, want) < 2e-3  # output is rounded to F16; exp LUT boundary flips allowed
