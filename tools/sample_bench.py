"""Sampled decoding: the host sampler loop against the device sampler (minigpt4_b200_sample_steps).  One Vicuna-7B Q4_1 model (language
model only) at n_ctx 2048; every arm starts from fresh sessions with fixed seeds after one image-chat turn (minigpt4_system_prompt +
minigpt4_begin_chat_image with 32 seeded embedding rows, about 95 rows) and samples 128 tokens.  Alternated in the same run, best of
--rounds with the spread:

- one context: the minigpt4_end_chat loop, a sample_steps(steps=1) loop, one sample_steps(steps=128) call, and greedy decode_chain as
  the ceiling;
- B = 2, 4, 8 sessions: the minigpt4_b200_end_chat_batch loop against sample_steps(n=B, steps=1) loops and one steps=128 call;

for the web UI's parameters (temp 0.8, top_k 40, top_p 0.9), for top_k 0 / top_p 0.95, and for mirostat 1 (tau 5, eta 0.1) and
mirostat 2 (tau 5, eta 1.0) at temp 0.8 (minigpt4_b200_sample_steps_mirostat; both sort the whole vocabulary every step, as top_k 0 does).
The sampling kernel's own time is the CUDA-event average of one launch over a context's logits (minigpt4_b200_op_sample_timed /
op_sample_mirostat).  parity: every arm's ids equal the end_chat arm's; parity_mismatch lists the legs that differ, with the session
and step of their first differing token.  Prints one JSON line.

    python tools/sample_bench.py [--steps 128] [--rounds 3] [--params webui,top_k0_top_p0.95,mirostat1,mirostat2]"""
import argparse
import ctypes
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402

import bench  # noqa: E402
import minigpt4_cpp_b200 as m  # noqa: E402
from tools.sessions_bench import gpu_card  # noqa: E402

N_CTX = 2048
QUESTION = "Describe this image in detail, please."
PARAMS = {"webui": dict(temp=0.8, top_k=40, top_p=0.9), "top_k0_top_p0.95": dict(temp=0.8, top_k=0, top_p=0.95),
          "mirostat1": dict(temp=0.8, mirostat=1, mirostat_tau=5.0, mirostat_eta=0.1),
          "mirostat2": dict(temp=0.8, mirostat=2, mirostat_tau=5.0, mirostat_eta=1.0)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=128)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--params", default=",".join(PARAMS), help="comma-separated names of PARAMS to run")
    args = ap.parse_args()
    params = {pn: PARAMS[pn] for pn in args.params.split(",")}
    lib = m.load_library()
    ext = m.B200(lib)
    if ext.L.minigpt4_b200_device_count() < 1:
        sys.exit("sample_bench.py needs a CUDA device")
    _, llm, _ = bench.ensure_models("7b", "q4_1", 39)
    parent = ext.llm_load(llm, n_ctx=N_CTX, seed=1)
    rng = np.random.default_rng(0)
    embs = [rng.standard_normal((32, 4096)).astype(np.float32) * 0.05 for _ in range(8)]
    views = [m.MiniGPT4Embedding(e.ctypes.data_as(ctypes.POINTER(ctypes.c_float)), e.size) for e in embs]
    S = args.steps

    def fresh(B):
        cs = [ext.session_create(parent, seed=1000 + i) for i in range(B)]
        for i, c in enumerate(cs):
            lib.minigpt4_system_prompt(c)
            lib.minigpt4_begin_chat_image(c, views[i], QUESTION)
        ext.flush_batch(cs)
        return cs

    def text(c, ids):
        return [ext.L.minigpt4_b200_token_text(c.ptr, int(i)).decode("utf-8", errors="ignore") for i in ids]

    def run(arm, B, p):
        """(seconds, [B][S] token texts)"""
        cs = fresh(B)
        t0 = time.perf_counter()
        if arm == "host":
            if B == 1:
                toks = [[lib.minigpt4_end_chat(cs[0], **p) for _ in range(S)]]
            else:
                steps = [ext.end_chat_batch(cs, **p) for _ in range(S)]
                toks = [[s[i] for s in steps] for i in range(B)]
            t = time.perf_counter() - t0
        elif arm == "device_steps1":
            ids = np.concatenate([ext.sample_steps(cs, 1, **p)[0] for _ in range(S)], 0)
            t = time.perf_counter() - t0
            toks = [text(cs[i], ids[:, i]) for i in range(B)]
        elif arm == "device_steps_all":
            ids, _ = ext.sample_steps(cs, S, **p)
            t = time.perf_counter() - t0
            toks = [text(cs[i], ids[:, i]) for i in range(B)]
        else:   # greedy ceiling
            ext.decode_chain(cs[0], S)
            t = time.perf_counter() - t0
            toks = None
        for c in cs:
            ext.base.minigpt4_free(c)
        return t, toks

    arms = [(arm, B, pn) for pn in params for B in (1, 2, 4, 8) for arm in ("host", "device_steps1", "device_steps_all")]
    arms.append(("decode_chain", 1, "greedy"))
    for arm, B, pn in arms:   # warm-up: graphs of every batch size, scratch of every arm
        run(arm, B, PARAMS.get(pn, {}))
    wall = {a: [] for a in arms}
    toks = {}
    for _ in range(args.rounds):
        for a in arms:
            t, tk = run(a[0], a[1], PARAMS.get(a[2], {}))
            wall[a].append(t)
            toks.setdefault(a, tk)
    def first_diff(got, want):   # [session, step] of the first token that differs
        for i, (g, w) in enumerate(zip(got, want)):
            for s, (x, y) in enumerate(zip(g, w)):
                if x != y:
                    return [i, s]
        return None
    mismatch = {f"{pn}/B{B}/{arm}": first_diff(toks[(arm, B, pn)], toks[("host", B, pn)]) for arm, B, pn in arms if arm not in ("host", "decode_chain")}
    mismatch = {k: v for k, v in mismatch.items() if v}
    legs = {}
    for a in arms:
        arm, B, pn = a
        t = min(wall[a])
        legs[f"{pn}/B{B}/{arm}"] = {"tok_s": round(S * B / t, 1), "ms_per_step": round(t / S * 1e3, 3), "spread": round(max(wall[a]) / t - 1.0, 3)}
    # the sampling kernel alone, over the logits a context has after the turn
    c = fresh(1)[0]
    logits = ext.logits(c)
    ext.base.minigpt4_free(c)
    kernel = {}
    for pn, p in params.items():
        if p.get("mirostat"):
            _, _, ms = ext.op_sample_mirostat(logits, 1000, 64, timed=True, **p)
        else:
            _, ms = ext.op_sample(logits, 1000, 64, tfs_z=1.0, typical_p=1.0, timed=True, **p)
        kernel[pn] = {"us_per_launch": round(ms * 1e3, 1)}
    st = ext.stats(parent)
    out = {"metric": "sampled decode tokens/s, Vicuna-7B q4_1, n_ctx 2048, after one image-chat turn", "steps": S, "rounds": args.rounds,
           "timing": "best of rounds, wall clock around synchronous calls, arms alternated", "legs": legs, "sample_kernel": kernel,
           "decode_megakernel": st.decode_megakernel, "parity": not mismatch,
           "parity_mismatch": mismatch, **gpu_card()}
    print(json.dumps(out))
    ext.base.minigpt4_free(parent)


if __name__ == "__main__":
    main()
