"""Profiling target for the prompt path: Vicuna-7B-shaped Q4_1 model (synthetic), a 32-row embedding prefix and a 45-row mixed prompt.
Run under a profiler (python tools/torch_prof.py tools/prof_prefill.py prints the kernel table)."""
import os, sys, time
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
for n_rep in range(int(os.environ.get("REPS", "2"))):
    lib.minigpt4_reset_chat(ctx)
    t0 = time.perf_counter(); ext.eval_embd(ctx, rows); ext.flush(ctx); t1 = time.perf_counter()
    ext.eval_tokens(ctx, list(range(5, 18))); ext.eval_embd(ctx, rows); ext.flush(ctx); t2 = time.perf_counter()
    print(f"32-row prefix {1e3 * (t1 - t0):.2f} ms, 45-row mixed pass {1e3 * (t2 - t1):.2f} ms")
