"""Profiling target: ONE chat turn through the reference ABI (7B q4_1 + ViT-g f16, synthetic): encode, system prompt + begin_chat_image (one merged
prefill pass), N greedy tokens.  Run under a profiler (python tools/torch_prof.py tools/prof_turn.py) for the kernel table of a step."""
import ctypes, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import minigpt4_cpp_b200 as m
import bench
from minigpt4_cpp_b200 import modelgen as mg
lib = m.load_library(); ext = m.B200(lib)
vis, llm, info = bench.ensure_models("7b", "q4_1", 39)
ctx = lib.minigpt4_model_load(vis, llm, 1, 1337, 2048, 512, 0)
img = mg.synth_image()
mi = m.MiniGPT4Image(img.ctypes.data_as(ctypes.c_void_p), 224, 224, 3, m.ImageFormat.F32)
for rep in range(int(os.environ.get("REPS", "1"))):
    lib.minigpt4_reset_chat(ctx)
    emb = lib.minigpt4_encode_image(ctx, mi)
    lib.minigpt4_system_prompt(ctx)
    lib.minigpt4_begin_chat_image(ctx, emb, bench.PROMPT)
    toks = [lib.minigpt4_end_chat_image(ctx, temp=0.0) for _ in range(int(os.environ.get("TOKENS", "16")))]
    lib.minigpt4_free_embedding(emb)
print("turn done,", len(toks), "tokens")
