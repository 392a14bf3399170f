"""Fast GPU canary for the decode megakernel: bit-exact against the CPU oracle on seeded tiny models, at short AND long positions
(the in-kernel attention has a one-pass regime below 192 keys and a multi-pass regime above), Q4_1 and Q4_0, plus 7B- and 13B-wide
2-layer models (the production row widths; 13B: five register-resident blocks per lane, fewer stream warps).  ~30 s; run before spending
GPU minutes on anything else."""
import os, sys, tempfile
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import minigpt4_cpp_b200 as m
from minigpt4_cpp_b200 import modelgen as mg
from oracle import oracle as orc

lib = m.load_library(); ext = m.B200(lib)
assert ext.L.minigpt4_b200_device_count() > 0
ok = True
with tempfile.TemporaryDirectory() as d:
    cases = [("q4_1", dict(n_vocab=1024, n_embd=512, n_head=4, n_layer=2), 230, 12),
             ("q4_0", dict(n_vocab=1024, n_embd=512, n_head=4, n_layer=2), 40, 12),
             ("q4_1", dict(n_vocab=2048, n_embd=4096, n_head=32, n_layer=2), 180, 20),
             ("q5_k", dict(n_vocab=1024, n_embd=512, n_head=4, n_layer=2), 200, 12),
             ("q5_k", dict(n_vocab=2048, n_embd=4096, n_head=32, n_layer=2), 60, 12),
             ("q4_1", dict(n_vocab=2048, n_embd=5120, n_head=40, n_layer=2), 230, 12),
             ("q5_k", dict(n_vocab=2048, n_embd=5120, n_head=40, n_layer=2), 60, 12)]
    for wt, dims, n_prompt, n_gen in cases:
        p = f"{d}/llama-{wt}-{dims['n_embd']}.bin"
        mg.write_llama_ggjt(p, mg.LlamaSpec(wtype=wt, **dims))
        c = ext.llm_load(p, n_ctx=512)
        assert ext.stats(c).decode_megakernel >= 1, "megakernel not active"
        e = orc.OracleEngine(None, p, n_ctx=512)
        ids = [int(x) for x in np.random.default_rng(3).integers(3, dims["n_vocab"], n_prompt)]
        ext.eval_tokens(c, ids); e.eval_tokens(ids)
        same = np.array_equal(ext.logits(c), e.logits)
        for _ in range(n_gen):
            t = ext.greedy_id(c)
            same &= t == int(np.argmax(e.logits))
            ext.eval_tokens(c, [t]); e.eval_tokens([t])
            same &= bool(np.array_equal(ext.logits(c), e.logits))
        ch, _ = ext.decode_chain(c, 8)
        want = []
        for _ in range(8):
            t = int(np.argmax(e.logits)); want.append(t); e.eval_tokens([t])
        same &= ch.tolist() == want
        print(f"canary {wt} n_embd={dims['n_embd']} prompt={n_prompt}: {'bit-identical' if same else 'MISMATCH'}")
        ok &= bool(same)
        ext.base.minigpt4_free(c)
sys.exit(0 if ok else 1)
