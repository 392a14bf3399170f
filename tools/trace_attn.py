import os, sys
os.environ["MINIGPT4_B200_MEGA_TRACE"] = "1"
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import minigpt4_cpp_b200 as m, bench
from minigpt4_cpp_b200 import modelgen as mg
lib = m.load_library(); ext = m.B200(lib)
llm = str(bench.model_dir() / "llama-7bwide-4l-v32000-q4_1.bin")
if not os.path.exists(llm): mg.write_llama_ggjt(llm, mg.LlamaSpec(wtype="q4_1", n_vocab=32000, n_embd=4096, n_head=32, n_layer=4))
ctx = ext.llm_load(llm, n_ctx=2048)
ext.eval_embd(ctx, np.random.default_rng(0).standard_normal((32, 4096)).astype(np.float32))
ext.decode_chain(ctx, 128)
tr = ext.mega_trace(ctx).astype(np.float64)[0]
kinds = [0] + [1, 2, 3, 4, 5] * 4 + [6, 7]
for i, k in enumerate(kinds):
    if k == 2:
        t = tr[i]; f = 1 / 1965.0
        print(f"attn: barrier->entry {(t[12]-t[1])*f:.2f} | K+q loads+FMA {(t[13]-t[12])*f:.2f} | shuffles+sc {(t[14]-t[13])*f:.2f} | V issue+warp_max {(t[15]-t[14])*f:.2f} | sync wait {(t[8]-t[15])*f:.2f} | exp+sum {(t[9]-t[8])*f:.2f}")
