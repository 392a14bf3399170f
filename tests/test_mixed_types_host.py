"""The mixed-type files of test_mixed_types_gpu.py, read back without a GPU: every tensor has the type its case asks for, layer by layer.
An override whose suffix matches no tensor name would otherwise leave a homogeneous file that the GPU tests check as if it were mixed."""
import importlib.util
from pathlib import Path

import pytest

_spec = importlib.util.spec_from_file_location("mixed_types_cases", Path(__file__).with_name("test_mixed_types_gpu.py"))
cases = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(cases)
ALL = {**cases.CASES, **cases.REG_CASES}


def _names(n_layer):
    return ["tok_embeddings.weight", "output.weight"] + [f"layers.{i}.{m}" for i in range(n_layer) for m in cases.MATS]


def _intended(spec, name):
    """the type the case asks for: its per-tensor overrides, else output_type / tok_type, else wtype"""
    hits = [t for suf, t in spec.get("overrides", {}).items() if name.endswith(suf)]
    assert len(hits) <= 1, f"{name} matches {len(hits)} overrides"
    if hits:
        return hits[0]
    if name == "output.weight" and spec.get("output_type"):
        return spec["output_type"]
    if name == "tok_embeddings.weight" and spec.get("tok_type"):
        return spec["tok_type"]
    return spec["wtype"]


@pytest.mark.parametrize("name", list(ALL))
def test_case_file_has_the_intended_types(mg, tmp_path, name):
    from oracle.oracle import read_ggjt
    spec = ALL[name][0]
    path = tmp_path / f"{name}.bin"
    mg.write_llama_ggjt(path, mg.LlamaSpec(**spec))
    hp, _, tensors = read_ggjt(str(path))
    assert (hp["n_vocab"], hp["n_embd"], hp["n_layer"]) == (spec["n_vocab"], spec["n_embd"], spec["n_layer"])
    names = _names(spec["n_layer"])
    for suf in spec.get("overrides", {}):
        assert any(n.endswith(suf) for n in names), f"override {suf!r} matches no tensor"
    for n in names:
        assert tensors[n].gtype == mg.GG_NAMES[_intended(spec, n)], n


def test_cases_mix_what_they_claim():
    """spot checks written out by hand, independent of the resolution above"""
    ov = cases.CASES["q4-layer-mix"][0]["overrides"]
    assert all(ov[f"layers.0.{m}"] == "q4_0" for m in cases.MATS) and ov["layers.1.attention.wo.weight"] == "q4_0" and len(ov) == 8
    ov = cases.CASES["qkv-act-reuse"][0]["overrides"]
    assert [ov[f"layers.{i}.attention.w{p}.weight"] for i in range(3) for p in "qkv"] == \
        ["q4_0", "q5_0", "q8_0", "q4_k", "q5_k", "q6_k", "q4_1", "q4_0", "f16"]
    assert len(cases.REG_CASES) == 12
