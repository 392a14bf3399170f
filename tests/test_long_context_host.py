"""The oracle's LLaMA attention op against a plain float64 attention, from 1 key to 32768 (the largest n_ctx a context may be loaded
with).  The GPU attention kernels are compared with this op bit for bit (tests/test_long_context_gpu.py), so this is what ties them to the
mathematical definition at long positions.

Inputs are what ggml's attention sees: Q, K and V rounded to F16.  The float64 side then computes scores, soft-max and P.V exactly; the op
differs from it by its own roundings only (the exp table's F16 argument and result, P rounded to F16, F32 accumulation).  Bar: 2e-3 of
max|ref|."""
import numpy as np
import pytest

BAR = 2e-3
LENGTHS = [1, 16, 17, 191, 192, 193, 384, 2047, 4096, 32768]


def ref_attention(q, k, v, pos):
    """float64 attention of row t over keys 0 .. pos[t], every head, from the F16-rounded inputs"""
    qd = np.asarray(q, np.float32).astype(np.float16).astype(np.float64)
    kd, vd = np.asarray(k, np.float64), np.asarray(v, np.float64)
    out = np.zeros(qd.shape)
    for t, p in enumerate(np.asarray(pos).reshape(-1)):
        for h in range(kd.shape[1] // 128):
            c = slice(128 * h, 128 * h + 128)
            s = kd[:p + 1, c] @ qd[t, c] / np.sqrt(128.0)
            e = np.exp(s - s.max())
            out[t, c] = (e @ vd[:p + 1, c]) / e.sum()
    return out


def err_of(got, want) -> float:
    return float(np.abs(np.asarray(got, np.float64) - want).max() / np.abs(want).max())


def random_case(rng, n_keys, n_head, score_scale, rows=1):
    """scores of standard deviation score_scale: K ~ N(0, 1), Q ~ N(0, score_scale^2) (the 1 / sqrt(128) cancels the dot's growth)"""
    E = 128 * n_head
    k = rng.standard_normal((n_keys, E)).astype(np.float16)
    v = rng.standard_normal((n_keys, E)).astype(np.float16)
    q = (score_scale * rng.standard_normal((rows, E))).astype(np.float32)
    return q, k, v


@pytest.mark.parametrize("n_keys", LENGTHS)
def test_oracle_attention_matches_float64(orc, n_keys):
    rng = np.random.default_rng(n_keys)
    worst = 0.0
    for scale in (0.5, 2.0, 8.0):
        q, k, v = random_case(rng, n_keys, 2, scale, rows=2)
        pos = [n_keys - 1, max(0, n_keys - 2)]   # the last key, and one short of it
        err = err_of(orc.llama_attention(q, k, v, pos), ref_attention(q, k, v, pos))
        assert err < BAR, (n_keys, scale, err)
        worst = max(worst, err)
    print(f"{n_keys} keys: worst error {worst:.2e} of max|ref|")


@pytest.mark.parametrize("n_keys", [193, 4096, 32768])
def test_one_dominant_key(orc, n_keys):
    """one key scores ~45 above the rest (their exp underflows F16): the output is that key's V row, wherever it sits - first key, either
    side of a 192-key pass boundary, last key"""
    rng = np.random.default_rng(7)
    q = np.full((1, 128), 0.5, np.float32)
    v = (1.0 + 0.5 * rng.standard_normal((n_keys, 128))).astype(np.float16)
    for at in sorted({0, 191, 192, 193, 383, 384, n_keys - 1} & set(range(n_keys))):
        k = (0.05 * rng.standard_normal((n_keys, 128))).astype(np.float16)
        k[at] = 8.0
        got = orc.llama_attention(q, k, v, [n_keys - 1])
        want = ref_attention(q, k, v, [n_keys - 1])
        assert err_of(got, want) < BAR, (n_keys, at)
        assert np.array_equal(got[0], v[at].astype(np.float32)), (n_keys, at)   # P = 1 exactly, every other P = 0


@pytest.mark.parametrize("n_keys", [17, 193, 4096, 30000, 32768])
def test_equal_scores_give_the_mean_of_v(orc, n_keys):
    """q = 0: every score is 0 and P = F16(1 / n), a subnormal F16 from n = 16385 on"""
    rng = np.random.default_rng(n_keys)
    q = np.zeros((1, 256), np.float32)
    k = rng.standard_normal((n_keys, 256)).astype(np.float16)
    v = (1.0 + 0.5 * rng.standard_normal((n_keys, 256))).astype(np.float16)
    got = orc.llama_attention(q, k, v, [n_keys - 1])
    mean = v.astype(np.float64).mean(axis=0, keepdims=True)
    assert err_of(got, ref_attention(q, k, v, [n_keys - 1])) < BAR
    assert err_of(got, mean) < BAR, err_of(got, mean)


def test_rows_see_only_their_own_prefix(orc):
    """row t reads keys 0 .. pos[t] and nothing above: NaN / inf rows past a row's position leave it unchanged"""
    rng = np.random.default_rng(3)
    q, k, v = random_case(rng, 1024, 2, 2.0, rows=3)
    pos = [100, 511, 0]
    clean = orc.llama_attention(q, k, v, pos)
    k2, v2 = k.copy(), v.copy()
    k2[512:] = np.inf; v2[512:] = np.nan; k2[600:] = -np.inf
    assert np.array_equal(orc.llama_attention(q, k2, v2, pos), clean)
    assert err_of(clean, ref_attention(q, k, v, pos)) < BAR


def test_positions_outside_the_cache_are_refused(orc):
    q, k, v = random_case(np.random.default_rng(0), 64, 1, 1.0)
    for p in (-1, 64):
        with pytest.raises(ValueError):
            orc.llama_attention(q, k, v, [p])
