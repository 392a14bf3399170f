"""Shared fixtures.  `-m "not gpu"`: oracle vs golden vectors, host logic, ABI surface (no compute calls).
`-m gpu`: parity tests proper — every CUDA path is driven through the C ABI and compared with the CPU oracle."""
import os
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.fixture(scope="session")
def lib():
    import minigpt4_cpp_b200 as m
    return m.load_library()


@pytest.fixture(scope="session")
def ext(lib):
    import minigpt4_cpp_b200 as m
    return m.B200(lib)


@pytest.fixture(scope="session")
def orc():
    from oracle import oracle
    oracle.lib()
    return oracle


@pytest.fixture(scope="session")
def mg():
    from minigpt4_cpp_b200 import modelgen
    return modelgen


@pytest.fixture(scope="session")
def tiny(tmp_path_factory, mg):
    """Seeded tiny models: full-width ViT/Q-Former with 2 blocks / 2 layers, 2-layer LLaMA (n_embd 512, head_dim 128)."""
    d = tmp_path_factory.mktemp("models")
    paths = {}
    for wt in ("q4_1", "q4_0", "q5_k", "q6_k", "f16"):
        spec = mg.LlamaSpec(n_vocab=1024, n_embd=512, n_head=4, n_layer=2, wtype=wt)
        paths[wt] = str(d / f"llama-tiny-{wt}.bin")
        mg.write_llama_ggjt(paths[wt], spec)
    spec = mg.LlamaSpec(n_vocab=1001, n_embd=512, n_head=4, n_layer=2, wtype="q4_1", output_type="q6_k",
                        overrides={"attention.wv.weight": "q4_0"})
    paths["mixed"] = str(d / "llama-tiny-mixed.bin")
    mg.write_llama_ggjt(paths["mixed"], spec)
    paths["vision"] = str(d / "minigpt4-tiny.bin")
    mg.write_minigpt4(paths["vision"], mg.VisionSpec(n_blocks=2, n_qformer_layers=2, n_embd_llm=4096))
    paths["vision512"] = None
    return paths


def rel_err(a, b):
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / (np.abs(b).max() + 1e-30))
