"""Copying conversations between sessions and parking them in host memory, on Vicuna-7B-shaped models (language model only).

  * copy sweep (Q4_1, n_ctx 2048): a source history of 92, 512 and 2000 rows copied into 1, 8 and 16 sessions by minigpt4_b200_session_copy:
    the copy kernel's CUDA-event time, the wall time of the call, the algorithmic bytes (1 + n) * rows * 2 * n_layer * n_embd * 2 B and the
    kernel's share of the 3.35 TB/s HBM data-sheet bandwidth;
  * 64 questions about one image (Q4_1 and Q5_K, n_ctx 512 so that 64 caches fit): (a) every context queues a whole image-chat turn, then one
    end_chat_batch; (b) one context evaluates the system prompt, "Human: <Img>" and the 32 image rows, session_copy copies them into the 63
    others, each queues only "</Img> ", its question and "### Assistant:", then one end_chat_batch.  Time to the first token of all 64;
  * park / resume (Q4_1, n_ctx 2048): state_save and state_load of 92- and 2000-row conversations, ms and GB/s through pageable host memory.

Arms alternated, best of --rounds with the spread; wall clock around synchronous calls.  Parity: every copy's logits equal the source's; the
64 contexts' logits before sampling and their sampled ids (fresh sessions of the same seeds per arm) are equal across (a) and (b); a restored
context's 32 greedy ids equal the original's.  Prints one JSON line with the card name and power limit.

    python tools/session_copy_bench.py [--rounds 3]"""
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

HBM_GBS = 3350.0   # H100 SXM data sheet
ROWS, DSTS = (92, 512, 2000), (1, 8, 16)
N_Q = 64
WEBUI = dict(temp=0.8, top_k=40, top_p=0.9)


def spread(ts):
    return round(max(ts) / min(ts) - 1.0, 3)


def copy_sweep(lib, ext, rounds):
    _, llm, _ = bench.ensure_models("7b", "q4_1", 39)
    p = ext.llm_load(llm, n_ctx=2048, seed=1)
    st = ext.stats(p)
    dsts = [ext.session_create(p, seed=2 + i) for i in range(max(DSTS))]
    rng = np.random.default_rng(0)
    hist = {r: rng.integers(3, st.n_vocab, size=r).tolist() for r in ROWS}
    kern = {(r, n): [] for r in ROWS for n in DSTS}
    wall = {k: [] for k in kern}
    parity = True
    for _ in range(rounds):
        for r in ROWS:
            lib.minigpt4_reset_chat(p)
            ext.eval_tokens(p, hist[r]); ext.flush(p)
            src = ext.logits(p)
            for n in DSTS:
                t0 = time.perf_counter()
                ms = ext.session_copy(p, dsts[:n])
                wall[(r, n)].append((time.perf_counter() - t0) * 1e3)
                kern[(r, n)].append(ms)
                parity &= all(np.array_equal(ext.logits(c), src) for c in (dsts[0], dsts[n - 1]))
    out = []
    for (r, n), ks in kern.items():
        k = min(ks)
        nbytes = (1 + n) * r * 2 * st.n_layer * st.n_embd * 2
        gbs = nbytes / (k * 1e-3) / 1e9
        out.append({"rows": r, "destinations": n, "kernel_ms": round(k, 4), "kernel_spread": spread(ks), "call_ms": round(min(wall[(r, n)]), 3),
                    "call_spread": spread(wall[(r, n)]), "bytes": nbytes, "kernel_GBs": round(gbs, 1), "hbm_share": round(gbs / HBM_GBS, 3)})
    for c in [p] + dsts:
        ext.base.minigpt4_free(c)
    return out, parity


def image_questions(lib, ext, wtype, rounds):
    _, llm, _ = bench.ensure_models("7b", wtype, 39)
    p = ext.llm_load(llm, n_ctx=512, seed=1)   # holds the weights; the arms run on sessions
    rng = np.random.default_rng(1)
    emb = (rng.standard_normal((32, 4096)) * 0.05).astype(np.float32)
    view = m.MiniGPT4Embedding(emb.ctypes.data_as(ctypes.POINTER(ctypes.c_float)), emb.size)
    subjects = ["the sky", "the dog", "the man on the left", "the colours", "the weather", "the building", "the text", "the mood"]
    verbs = ["What is", "Describe", "Where is", "How many people see", "Why is", "What colour is", "Is there", "Who painted"]
    questions = [f"{verbs[i % 8]} {subjects[(i // 8) % 8]} in this picture?" for i in range(N_Q)]
    tok = lambda c, s: ext.tokenize(c, s, True)   # noqa: E731  (add_strings: always a BOS)

    def arm_a(cs):   # returns the prompt rows the arm evaluates
        for c, q in zip(cs, questions):
            lib.minigpt4_reset_chat(c)
            lib.minigpt4_system_prompt(c)
            lib.minigpt4_begin_chat_image(c, view, q)
        return sum(ext.n_past(c) for c in cs)

    def arm_b(cs):
        c0 = cs[0]
        lib.minigpt4_reset_chat(c0)
        lib.minigpt4_system_prompt(c0)
        ext.eval_tokens(c0, tok(c0, "Human: <Img>"))
        ext.eval_embd(c0, emb)
        prefix = ext.n_past(c0)
        ext.session_copy(c0, cs[1:])
        for c, q in zip(cs, questions):
            for piece in ("</Img> ", q, "### Assistant:"):
                ext.eval_tokens(c, tok(c, piece))
        return prefix + sum(ext.n_past(c) - prefix for c in cs)

    def fresh():
        return [ext.session_create(p, seed=1000 + i) for i in range(N_Q)]

    # parity: fresh sessions of the same seeds per arm, logits before sampling and the sampled ids
    seen, rows = {}, {}
    for name, arm in (("a", arm_a), ("b", arm_b)):
        cs = fresh()
        rows[name] = arm(cs)
        ext.flush_batch(cs)
        lg = [ext.logits(c) for c in cs]
        toks = ext.end_chat_batch(cs, **WEBUI)
        seen[name] = (lg, toks, [ext.n_past(c) for c in cs], [ext.greedy_id(c) for c in cs])
        for c in cs:
            ext.base.minigpt4_free(c)
    a, b = seen["a"], seen["b"]
    parity = all(np.array_equal(x, y) for x, y in zip(a[0], b[0])) and a[1:] == b[1:]

    cs = fresh()
    t = {"a": [], "b": []}
    for _ in range(rounds + 1):   # (the first round warms the batched graphs and is dropped)
        for name, arm in (("a", arm_a), ("b", arm_b)):
            t0 = time.perf_counter()
            arm(cs)
            ext.end_chat_batch(cs, **WEBUI)
            t[name].append((time.perf_counter() - t0) * 1e3)
    for c in cs + [p]:
        ext.base.minigpt4_free(c)
    ta, tb = min(t["a"][1:]), min(t["b"][1:])
    return {"first_token_ms_a": round(ta, 2), "spread_a": spread(t["a"][1:]), "first_token_ms_b": round(tb, 2), "spread_b": spread(t["b"][1:]),
            "speedup": round(ta / tb, 2), "prompt_rows_a": rows["a"], "prompt_rows_b": rows["b"], "parity": parity}


def park_resume(lib, ext, rounds):
    _, llm, _ = bench.ensure_models("7b", "q4_1", 39)
    p = ext.llm_load(llm, n_ctx=2048, seed=1)
    other = ext.session_create(p, seed=2)
    V = ext.L.minigpt4_b200_n_vocab(p.ptr)
    rng = np.random.default_rng(2)
    out, parity = [], True
    for r in (92, 2000):
        lib.minigpt4_reset_chat(p)
        ext.eval_tokens(p, rng.integers(3, V, size=r).tolist()); ext.flush(p)
        size = ext.L.minigpt4_b200_state_size(p.ptr)
        buf = np.empty(size, np.uint8)
        ptr = buf.ctypes.data_as(ctypes.c_void_p)
        ts, tl = [], []
        for _ in range(rounds):
            t0 = time.perf_counter()
            assert ext.L.minigpt4_b200_state_save(p.ptr, ptr, size, None) == 0
            t1 = time.perf_counter()
            assert ext.L.minigpt4_b200_state_load(other.ptr, ptr, size) == 0
            t2 = time.perf_counter()
            ts.append((t1 - t0) * 1e3); tl.append((t2 - t1) * 1e3)
        ids_o, _ = ext.decode_chain(p, 32)
        ids_r, _ = ext.decode_chain(other, 32)
        parity &= bool(np.array_equal(ids_o, ids_r))
        out.append({"rows": r, "bytes": size, "save_ms": round(min(ts), 3), "save_spread": spread(ts), "save_GBs": round(size / min(ts) / 1e6, 2),
                    "load_ms": round(min(tl), 3), "load_spread": spread(tl), "load_GBs": round(size / min(tl) / 1e6, 2)})
    for c in (p, other):
        ext.base.minigpt4_free(c)
    return out, parity


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    lib = m.load_library()
    ext = m.B200(lib)
    if ext.L.minigpt4_b200_device_count() < 1:
        sys.exit("session_copy_bench.py needs a CUDA device")
    card = gpu_card()
    sweep, copy_parity = copy_sweep(lib, ext, args.rounds)
    questions = {w: image_questions(lib, ext, w, args.rounds) for w in ("q4_1", "q5_k")}
    park, park_parity = park_resume(lib, ext, args.rounds)
    out = {"metric": "session_copy / state_save / state_load, Vicuna-7B-shaped", "rounds": args.rounds,
           "timing": "best of alternated rounds; kernel: CUDA events, calls: wall clock around synchronous calls", "hbm_datasheet_GBs": HBM_GBS,
           "copy_sweep": sweep, "image_questions_64": questions, "park_resume": park,
           "parity": {"copies": copy_parity, "questions": all(q["parity"] for q in questions.values()), "park_resume": park_parity}, **card}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
