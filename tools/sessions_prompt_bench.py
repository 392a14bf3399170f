"""Batched prompt evaluation across sessions: one Vicuna-7B model (language model only) serving a parent context and 7 sessions at n_ctx
2048.  Every context queues one chat turn: the system prompt, "Human: <Img>", 32 image rows (synthetic), "</Img> ", a question and
"### Assistant:" (minigpt4_system_prompt + minigpt4_begin_chat_image).  For B = 1, 2, 4, 8 contexts, alternated in the same run, it times
(wall clock around synchronous calls, queueing excluded):
  * flush: each context's own minigpt4_b200_flush one after another, against one minigpt4_b200_flush_batch;
  * first token: per-context flush + minigpt4_end_chat, against one minigpt4_b200_end_chat_batch (batched flush + sample + batched step).
The Q4_1 file takes the tensor-core prefill path; the Q5_K file (--types q4_1,q5_k, the default) the per-op path.  Prints one JSON line.

    python tools/sessions_prompt_bench.py [--rounds 3] [--types q4_1,q5_k]

parity: after a batched flush of all 8 contexts, every context's logits equal its logits after its own flush."""
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
N_CTXS = 8
QUESTIONS = ["What is in this picture?", "Describe the image in detail.", "Which colors do you see?", "How many people are there?",
             "Is this indoors or outdoors?", "What is the person on the left doing?", "Write a short poem about this image.",
             "What time of day was this taken?"]


def run(lib, ext, wtype: str, rounds: int) -> dict:
    _, llm, _ = bench.ensure_models("7b", wtype, 39)
    parent = ext.llm_load(llm, n_ctx=N_CTX, seed=1)
    ctxs = [parent] + [ext.session_create(parent, seed=2 + i) for i in range(N_CTXS - 1)]
    rng = np.random.default_rng(0)
    embs = [rng.standard_normal((32, 4096)).astype(np.float32) * 0.05 for _ in range(N_CTXS)]
    views = [m.MiniGPT4Embedding(e.ctypes.data_as(ctypes.POINTER(ctypes.c_float)), e.size) for e in embs]

    def queue(cs):
        for i, c in enumerate(cs):
            lib.minigpt4_reset_chat(c)
            lib.minigpt4_system_prompt(c)
            lib.minigpt4_begin_chat_image(c, views[i], QUESTIONS[i])
        return [ext.n_past(c) for c in cs]

    rows = queue(ctxs)
    ext.flush_batch(ctxs)
    batched = [ext.logits(c) for c in ctxs]
    queue(ctxs)
    own = []
    for c in ctxs:
        ext.flush(c); own.append(ext.logits(c))
    parity = all(np.array_equal(a, b) for a, b in zip(batched, own))

    legs = {}
    for B in (1, 2, 4, 8):
        sub = ctxs[:B]
        legs[f"flush_seq_B{B}"] = (sub, lambda s=sub: [ext.flush(c) for c in s])
        legs[f"flush_batch_B{B}"] = (sub, lambda s=sub: ext.flush_batch(s))
        legs[f"first_token_seq_B{B}"] = (sub, lambda s=sub: [(ext.flush(c), lib.minigpt4_end_chat(c, temp=0.0)) for c in s])
        legs[f"first_token_batch_B{B}"] = (sub, lambda s=sub: ext.end_chat_batch(s, temp=0.0))
    for sub, fn in legs.values():   # warm-up: every shape the timed legs use
        queue(sub); fn()
    wall = {k: [] for k in legs}
    for _ in range(rounds):
        for name, (sub, fn) in legs.items():   # alternated: every round runs every leg from the same queues
            queue(sub)
            t0 = time.perf_counter()
            fn()
            wall[name].append(time.perf_counter() - t0)
    res = {name: {"ms": round(min(t) * 1e3, 2), "spread": round(max(t) / min(t) - 1.0, 3)} for name, t in wall.items()}
    for B in (1, 2, 4, 8):
        res[f"speedup_flush_B{B}"] = round(res[f"flush_seq_B{B}"]["ms"] / res[f"flush_batch_B{B}"]["ms"], 3)
        res[f"speedup_first_token_B{B}"] = round(res[f"first_token_seq_B{B}"]["ms"] / res[f"first_token_batch_B{B}"]["ms"], 3)
    st = ext.stats(parent)
    out = {"rows_per_context": rows, "prefill_gemm": bool(st.prefill_gemm), "legs": res, "parity": parity}
    for c in ctxs:
        ext.base.minigpt4_free(c)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--types", default="q4_1,q5_k")
    args = ap.parse_args()
    lib = m.load_library()
    ext = m.B200(lib)
    if ext.L.minigpt4_b200_device_count() < 1:
        sys.exit("sessions_prompt_bench.py needs a CUDA device")
    out = {"metric": "wall ms to evaluate the queued chat turns of B contexts of one Vicuna-7B model (n_ctx 2048): own flushes vs one batched flush",
           "rounds": args.rounds, "timing": "best of rounds, wall clock around synchronous calls"}
    for wt in args.types.split(","):
        out[wt] = run(lib, ext, wt, args.rounds)
    out.update(gpu_card())
    print(json.dumps(out))


if __name__ == "__main__":
    main()
