"""Constrained replies (minigpt4_b200_constraint_*): compile time, the device sampler's cost over allowed(s), and whole constrained replies.
One Vicuna-7B-shaped Q4_1 model (language model only, n_vocab 32000) at n_ctx 512; sessions start from a seeded prompt of 64 ids.

1. compile time of minigpt4_b200_constraint_create (host compiler + upload) for three automata: 1000 labels (choices_dfa), digits
   [0-9]{1,6}, and a two-field JSON record {"color": "<string>", "count": <digits>} whose string state takes any byte but '"' and '\\';
2. device ms of sample_steps (64 steps) and of a sample_until call, constrained against unconstrained, at B = 1, 8 and 64, with the web UI's
   parameters and with top_k 0 / top_p 0.95 (the JSON record, whose string state allows most of the vocabulary);
3. whole constrained replies (B = 1, up to 64 ids, each ending after </s>) for the 1000 labels and the JSON record: the minigpt4_end_chat
   loop against one sample_until call, wall clock, with their parity.

Alternated, best of --rounds with the spread; card name and power limit.  Prints one JSON line.

    python tools/constrain_bench.py [--rounds 3]"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402

import bench  # noqa: E402
import minigpt4_cpp_b200 as m  # noqa: E402
from minigpt4_cpp_b200.minigpt4_library import choices_dfa  # noqa: E402
from tools.sessions_bench import gpu_card  # noqa: E402

N_CTX = 512
PARAMS = {"webui": dict(temp=0.8, top_k=40, top_p=0.9), "top_k0_top_p0.95": dict(temp=0.8, top_k=0, top_p=0.95)}


def labels(n=1000):
    rng = np.random.default_rng(0)
    words = set()
    while len(words) < n:
        words.add(bytes(rng.integers(ord("a"), ord("z") + 1, size=int(rng.integers(3, 12))).tolist()))
    return sorted(words)


def digits(k=6):
    nx, ac = np.full((k + 1, 256), -1, np.int32), np.zeros(k + 1, np.uint8)
    for s in range(k):
        nx[s, ord("0"):ord("9") + 1] = s + 1
    ac[1:] = 1
    return nx, ac


def json_record():
    """{"color": "<string>", "count": <1..6 digits>}"""
    nx, acc = [], []
    def new():
        nx.append([-1] * 256); acc.append(0)
        return len(nx) - 1
    def lit(s, text):
        for b in text.encode():
            t = new(); nx[s][b] = t; s = t
        return s
    s = lit(new(), '{"color": "')
    string = s
    for b in range(32, 256):
        if b not in (ord('"'), ord("\\")):
            nx[string][b] = string
    s = new(); nx[string][ord('"')] = s
    s = lit(s, ', "count": ')
    d = [new() for _ in range(6)]
    for b in range(ord("0"), ord("9") + 1):
        nx[s][b] = d[0]
        for i in range(5):
            nx[d[i]][b] = d[i + 1]
    end = new()
    for i in range(6):
        nx[d[i]][ord("}")] = end
    acc[end] = 1
    return np.array(nx, np.int32), np.array(acc, np.uint8)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    lib = m.load_library()
    ext = m.B200(lib)
    if ext.L.minigpt4_b200_device_count() < 1:
        sys.exit("constrain_bench.py needs a CUDA device")
    _, llm, _ = bench.ensure_models("7b", "q4_1", 39)
    parent = ext.llm_load(llm, n_ctx=N_CTX, seed=1)
    prompt = np.random.default_rng(1).integers(3, 32000, size=64).tolist()
    automata = {"labels_1000": choices_dfa(labels()), "digits_1_6": digits(), "json_record": json_record()}

    # 1. compile time
    compile_ms = {}
    for name, (nx, ac) in automata.items():
        ts = []
        for _ in range(args.rounds):
            t0 = time.perf_counter()
            h = ext.constraint_create(parent, nx, ac)
            ts.append((time.perf_counter() - t0) * 1e3)
            ext.constraint_free(h)
        compile_ms[name] = {"ms": round(min(ts), 2), "spread": round(max(ts) / min(ts) - 1.0, 3), "n_states": int(len(ac))}
    h = ext.constraint_create(parent, *automata["json_record"])
    pool = [ext.session_create(parent, seed=1000 + i) for i in range(64)]

    def fresh(B, constrained):
        cs = pool[:B]
        for c in cs:
            lib.minigpt4_reset_chat(c)
            ext.eval_tokens(c, prompt)
            ext.constraint_attach(c, h if constrained else None)
        ext.flush_batch(cs)
        return cs

    # 2. device ms, constrained against unconstrained
    legs = [(kind, B, pn, con) for kind in ("sample_steps", "sample_until") for B in (1, 8, 64) for pn in PARAMS for con in (False, True)]
    dev = {leg: [] for leg in legs}
    for r in range(args.rounds + 1):   # round 0 warms up
        for leg in legs:
            kind, B, pn, con = leg
            cs = fresh(B, con)
            if kind == "sample_steps":
                _, ms = ext.sample_steps(cs, 64, **PARAMS[pn])
                steps = 64
            else:
                ids, _, ms = ext.sample_until(cs, 64, "", **PARAMS[pn])
                steps = max(len(x) for x in ids)
            if r:
                dev[leg].append((ms, steps))
    device = {}
    for (kind, B, pn, con), v in dev.items():
        ms, steps = min(v)
        device[f"{kind}/{pn}/B{B}/{'constrained' if con else 'unconstrained'}"] = {
            "device_ms": round(ms, 2), "steps": steps, "ms_per_step": round(ms / steps, 3), "spread": round(max(x[0] for x in v) / ms - 1.0, 3)}

    # 3. whole replies: the end_chat loop against one sample_until call (up to 64 ids; a reply ends after </s>)
    p = PARAMS["webui"]
    handles = {"labels_1000": ext.constraint_create(parent, *automata["labels_1000"]), "json_record": h}

    def one(hh):   # a fresh session with the same seed for both arms
        c = ext.session_create(parent, seed=77)
        ext.eval_tokens(c, prompt)
        ext.constraint_attach(c, hh)
        ext.flush(c)
        return c

    whole, parity = {}, True
    for name, hh in handles.items():
        wall = {"end_chat_loop": [], "sample_until": []}
        replies = {}
        for _ in range(args.rounds + 1):   # (the first round warms up)
            c = one(hh)
            t0 = time.perf_counter()
            toks = []
            while len(toks) < 64 and (not toks or toks[-1] != "</s>"):
                toks.append(lib.minigpt4_end_chat(c, **p))
            wall["end_chat_loop"].append(time.perf_counter() - t0)
            replies["end_chat_loop"] = toks
            ext.base.minigpt4_free(c)
            c = one(hh)
            t0 = time.perf_counter()
            ids, _, _ = ext.sample_until([c], 64, "", **p)
            wall["sample_until"].append(time.perf_counter() - t0)
            replies["sample_until"] = [ext.L.minigpt4_b200_token_text(c.ptr, int(i)).decode("utf-8", errors="ignore") for i in ids[0]]
            ext.base.minigpt4_free(c)
        w = {k: {"ms": round(min(v[1:]) * 1e3, 2), "spread": round(max(v[1:]) / min(v[1:]) - 1.0, 3)} for k, v in wall.items()}
        w["reply_ids"] = len(replies["sample_until"])
        w["reply"] = "".join(replies["sample_until"])
        whole[name] = w
        parity = parity and replies["end_chat_loop"] == replies["sample_until"]
    ext.constraint_free(handles["labels_1000"])
    out = {"metric": "constrained replies, Vicuna-7B-shaped q4_1, n_vocab 32000, n_ctx 512", "rounds": args.rounds,
           "timing": "compile: wall clock of constraint_create; device: CUDA-event ms of the call's steps; whole replies: wall clock; best of rounds",
           "compile": compile_ms, "device": device, "whole_reply": whole, "parity": parity, **gpu_card()}
    print(json.dumps(out))
    for c in pool:
        ext.base.minigpt4_free(c)
    ext.constraint_free(h)
    ext.base.minigpt4_free(parent)


if __name__ == "__main__":
    main()
