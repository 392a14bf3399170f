"""Lean profiling target: Vicuna-7B-shaped Q4_1 model (synthetic), 32-row prefix, then N chained decode steps.
Run under a profiler (python tools/torch_prof.py tools/prof_decode.py prints the kernel table)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import minigpt4_cpp_b200 as m
import bench
from minigpt4_cpp_b200 import modelgen as mg
lib = m.load_library(); ext = m.B200(lib)
d = bench.model_dir()
llm = d / "llama-7b-q4_1.bin"
if not llm.exists():
    mg.write_llama_ggjt(llm, mg.LlamaSpec(wtype="q4_1", **mg.LLAMA_7B))
ctx = ext.llm_load(str(llm), n_ctx=2048)
rows = np.random.default_rng(0).standard_normal((32, 4096)).astype(np.float32)
ext.eval_embd(ctx, rows)
n = int(os.environ.get("STEPS", "24"))
ids, ms = ext.decode_chain(ctx, n)
print("chain ms/token", ms / n, "tok/s", 1e3 * n / ms)
