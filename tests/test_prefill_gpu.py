"""Tensor-core prefill (csrc/llama_prefill.cuh, wgmma s8): prompt / prefix rows must be BIT-IDENTICAL to the per-op matvec path and
to the CPU oracle for any number of rows - the epilogue keeps the canonical float order (per-class sequential sums + xor-butterfly tree).
Reference behaviour: llama_eval_embd with N = 32 in one batch (minigpt4.cpp:2405-2412), llama_eval in n_batch chunks (:2369-2379)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _load(ext, path, monkeypatch, gemm: bool, n_ctx=512):
    if gemm: monkeypatch.delenv("MINIGPT4_B200_NO_PREFILL_GEMM", raising=False)
    else: monkeypatch.setenv("MINIGPT4_B200_NO_PREFILL_GEMM", "1")
    c = ext.llm_load(path, n_ctx=n_ctx)
    monkeypatch.delenv("MINIGPT4_B200_NO_PREFILL_GEMM", raising=False)
    assert ext.stats(c).prefill_gemm == (1 if gemm else 0)
    return c


@pytest.mark.parametrize("wt", ["q4_1", "q4_0"])
@pytest.mark.parametrize("n", [2, 5, 31, 32, 33, 97])
def test_prefill_gemm_equals_per_op_path_and_oracle(ext, orc, tiny, monkeypatch, wt, n):
    c1, c2 = _load(ext, tiny[wt], monkeypatch, True), _load(ext, tiny[wt], monkeypatch, False)
    e = orc.OracleEngine(None, tiny[wt], n_ctx=512)
    ids = np.random.default_rng(100 + n).integers(3, e.n_vocab, size=n).tolist()
    ext.eval_tokens(c1, ids); ext.eval_tokens(c2, ids)
    want = e.eval_tokens(ids).copy()
    k = n - 8 * ((n - 1) // 8)   # the per-op path works in chunks of 8 rows: its buffer holds the residual stream of the LAST chunk only
    assert np.array_equal(ext.hidden(c1, n)[n - k:], ext.hidden(c2, k)), "residual stream differs between the GEMM and the matvec prefill"
    assert np.array_equal(ext.logits(c1), ext.logits(c2)) and np.array_equal(ext.logits(c1), want)
    # a second pass (embedding rows) on top of the first: positions > 0, KV rows written by the GEMM epilogue are read back by attention
    rows = np.random.default_rng(n).standard_normal((7, e.n_embd)).astype(np.float32)
    ext.eval_embd(c1, rows); ext.eval_embd(c2, rows)
    want = e.eval_embd(rows).copy()
    assert np.array_equal(ext.logits(c1), ext.logits(c2)) and np.array_equal(ext.logits(c1), want)
    a, b = [], []
    for _ in range(8):  # decode continues from the prefilled cache
        t = ext.greedy_id(c1); a.append(t); ext.eval_tokens(c1, [t]); b.append(e.end_chat_greedy()[0])
    assert a == b
    ext.base.minigpt4_free(c1); ext.base.minigpt4_free(c2)


def test_prefill_gemm_7b_wide_layer(ext, orc, mg, tmp_path, monkeypatch):
    """production row widths: n_embd 4096 (4 blocks per class), n_ff 11008 (344 blocks: 11 / 10 per class, three 4-block tiles)"""
    llm = str(tmp_path / "llama-7bwide-1l.bin")
    mg.write_llama_ggjt(llm, mg.LlamaSpec(n_vocab=1024, n_embd=4096, n_head=32, n_layer=1, wtype="q4_1"))
    c = _load(ext, llm, monkeypatch, True, n_ctx=256)
    e = orc.OracleEngine(None, llm, n_ctx=256)
    rows = np.random.default_rng(5).standard_normal((32, 4096)).astype(np.float32)   # the 32-row image prefix
    ext.eval_embd(c, rows)
    assert np.array_equal(ext.logits(c), e.eval_embd(rows))
    ids = np.random.default_rng(6).integers(3, 1024, size=45).tolist()
    ext.eval_tokens(c, ids)
    assert np.array_equal(ext.logits(c), e.eval_tokens(ids))
    ext.base.minigpt4_free(c)
