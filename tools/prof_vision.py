"""Lean profiling target for the vision graph: full-size ViT-g + Q-Former (synthetic F16 weights), two encodes.
Run under a profiler (python tools/torch_prof.py tools/prof_vision.py prints the kernel table)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import minigpt4_cpp_b200 as m
import bench
from minigpt4_cpp_b200 import modelgen as mg
lib = m.load_library(); ext = m.B200(lib)
d = bench.model_dir()
vis = d / "minigpt4-7b-f16-b39.bin"
if not vis.exists():
    mg.write_minigpt4(vis, mg.VisionSpec(n_blocks=39, n_embd_llm=4096, fast=True))
llm = d / "llama-4096-2l-q4_1.bin"
if not llm.exists():
    mg.write_llama_ggjt(llm, mg.LlamaSpec(n_vocab=2048, n_embd=4096, n_head=32, n_layer=2, wtype="q4_1"))
ctx = lib.minigpt4_model_load(str(vis), str(llm), 1, 1337, 256, 8, 0)
img = mg.synth_image()
for _ in range(int(os.environ.get("ENCODES", "2"))):
    emb = ext.encode_array(ctx, img)
print("encode ms", ext.stats(ctx).last_encode_ms)
