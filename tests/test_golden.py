"""Oracle vs the committed golden vectors (tests/golden/, made by tools/make_golden.py from seeded tiny models) and
the stored independent cross-check against HuggingFace transformers.  The reference ships no golden vectors of its own
(SURVEY §8c: parity unpinned) — these fixtures pin the oracle against regressions and against an independent float model."""
import json
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tools"))
GOLD = ROOT / "tests" / "golden"


@pytest.fixture(scope="module")
def gold():
    return np.load(GOLD / "oracle_golden.npz")


@pytest.fixture(scope="module")
def models(tmp_path_factory, mg):
    import make_golden as g
    d = tmp_path_factory.mktemp("gold")
    mg.write_minigpt4(d / "vision.bin", mg.VisionSpec(**g.VISION_SPEC))
    for name, spec in g.LLAMA_SPECS.items():
        mg.write_llama_ggjt(d / f"llama-{name}.bin", mg.LlamaSpec(**spec))
    return d


def test_vision_golden(orc, mg, gold, models):
    e = orc.OracleEngine(str(models / "vision.bin"), None)
    img = mg.synth_image()
    emb = e.encode_image(img)
    assert np.abs(emb - gold["vision_embedding"]).max() <= 1e-5 * np.abs(gold["vision_embedding"]).max()
    assert np.allclose(e.encode_image(img, tap_kind=3)[0], gold["vision_ln_vision_row0"], rtol=0, atol=1e-5)
    assert np.allclose(e.encode_image(img, tap_kind=2, tap_idx=0)[5], gold["vision_block0_row5"], rtol=0, atol=1e-4)


@pytest.mark.parametrize("name", ["q4_1", "q4_0", "q5_k", "q6_k", "f16"])
def test_llama_golden(orc, gold, models, name):
    import make_golden as g
    e = orc.OracleEngine(None, str(models / f"llama-{name}.bin"), n_ctx=128)
    e.eval_tokens(g.TOKENS)
    want = gold[f"llama_{name}_logits"]
    assert np.abs(e.logits - want).max() <= 1e-5 * np.abs(want).max()
    ids = [e.end_chat_greedy()[0] for _ in range(16)]
    assert ids == gold[f"llama_{name}_greedy"].tolist()


def test_tokenizer_golden(orc, gold, models):
    import make_golden as g
    _, vocab, _ = orc.read_ggjt(str(models / "llama-q4_1.bin"))
    tk = orc.Tokenizer(vocab)
    for i, t in enumerate(g.TEXTS):
        assert tk.tokenize(t, True) == gold[f"tok_{i}"].tolist()


def test_independent_crosscheck_is_within_bounds():
    """HuggingFace float models on the same synthetic weights (see tools/make_golden.py)."""
    r = json.loads((GOLD / "crosscheck.json").read_text())
    assert r["vision_ln_vision_rel_err"] < 2e-3 and r["qformer_proj_rel_err"] < 2e-3
    assert r["llama_f16_logits_rel_err"] < 2e-3 and r["llama_f16_argmax_equal"]
    assert r["llama_f16_long_logits_rel_err"] < 2e-3 and r["llama_f16_long_argmax_equal"]   # 2048 tokens: positions to 2047
    assert r["llama_q4_1_logits_rel_err"] < 2e-2 and r["llama_q4_1_argmax_equal"]  # Q8 activation quantisation is deliberate
    assert r["vision_missing_keys"] == [] and r["qformer_missing_keys"] == []


def test_vision_all_stages_run_equals_single_taps(orc, mg, models):
    """encode_image_stages fills every stage in one run: each equals the single-tap run of that stage (tap kinds 1-4) and its
    output equals the plain encode_image, bit for bit."""
    e = orc.OracleEngine(str(models / "vision.bin"), None)
    img = mg.synth_image(7)
    st = e.encode_image_stages(img)
    assert np.array_equal(st["out"], e.encode_image(img))
    assert np.array_equal(st["embed"], e.encode_image(img, tap_kind=1))
    assert st["vit_blocks"].shape[0] >= 1 and st["qformer"].shape[0] >= 2
    for b in range(st["vit_blocks"].shape[0]):
        assert np.array_equal(st["vit_blocks"][b], e.encode_image(img, tap_kind=2, tap_idx=b))
    assert np.array_equal(st["ln_vision"], e.encode_image(img, tap_kind=3))
    for layer in range(st["qformer"].shape[0]):
        assert np.array_equal(st["qformer"][layer], e.encode_image(img, tap_kind=4, tap_idx=layer))
