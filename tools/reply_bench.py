"""Whole replies: the host chat loop against the device's stop rule (minigpt4_b200_sample_until).  One Vicuna-7B Q4_1 model (language
model only) at n_ctx 2048; every arm starts from fresh sessions with fixed seeds after one image-chat turn (minigpt4_system_prompt +
minigpt4_begin_chat_image with 32 seeded embedding rows) and runs each context's reply to its end.  The replies end at known, staggered
lengths: one host run per batch size picks the stop text (a token text of the replies) whose first stops come closest to 40..128 tokens
across the batch.  Alternated in the same run, best of --rounds with the spread:

- host: MiniGPT4ChatBot.generate's loop, minigpt4_end_chat (B = 1) or minigpt4_b200_end_chat_batch over the contexts whose replies
  have not ended, the text checked on the host;
- steps1: a sample_steps(steps=1) loop over those contexts, the text checked on the host;
- until: one sample_until call;
- until16: sample_until calls of 16 steps over those contexts;

at B = 1, 2, 4, 8, for the web UI's parameters (temp 0.8, top_k 40, top_p 0.9) and for top_k 0 / top_p 0.95.  Each leg reports the
whole-reply time, the aggregate tok/s (ids fed over that time) and, for the sample_until arms, the steps the device ran past the last stop
(from the kernel launch count).  parity: every arm's replies equal the host arm's.  Prints one JSON line.

    python tools/reply_bench.py [--rounds 3]"""
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
MAX = 160   # max_steps of every reply (the forced stops lie at or below 128)
QUESTION = "Describe this image in detail, please."
PARAMS = {"webui": dict(temp=0.8, top_k=40, top_p=0.9), "top_k0_top_p0.95": dict(temp=0.8, top_k=0, top_p=0.95)}
UNUSED = (64, 1.1, 1.0, 1.0, 0, 5.0, 1.0, 1)   # repeat_last_n .. penalize_nl (mirostat 0)


def first_stop(texts, stop):
    """the reference loop: index of the token after which the reply ends with stop, None if it never does"""
    chat = b""
    for i, t in enumerate(texts):
        chat += t
        if t != b"##" and chat.endswith(stop):
            return i
    return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    lib = m.load_library()
    ext = m.B200(lib)
    if ext.L.minigpt4_b200_device_count() < 1:
        sys.exit("reply_bench.py needs a CUDA device")
    _, llm, _ = bench.ensure_models("7b", "q4_1", 39)
    parent = ext.llm_load(llm, n_ctx=N_CTX, seed=1)
    rng = np.random.default_rng(0)
    embs = [rng.standard_normal((32, 4096)).astype(np.float32) * 0.05 for _ in range(8)]
    views = [m.MiniGPT4Embedding(e.ctypes.data_as(ctypes.POINTER(ctypes.c_float)), e.size) for e in embs]

    def fresh(B):
        cs = [ext.session_create(parent, seed=1000 + i) for i in range(B)]
        for i, c in enumerate(cs):
            lib.minigpt4_system_prompt(c)
            lib.minigpt4_begin_chat_image(c, views[i], QUESTION)
        ext.flush_batch(cs)
        return cs

    def text(c, i):
        return ext.L.minigpt4_b200_token_text(c.ptr, int(i))

    def end_chat_batch(cs, p):
        toks = (ctypes.c_char_p * len(cs))()
        if len(cs) == 1:
            assert lib.library.minigpt4_end_chat(cs[0].ptr, ctypes.cast(toks, ctypes.POINTER(ctypes.c_char_p)), 0, p["temp"], p["top_k"], p["top_p"], 1.0, 1.0, *UNUSED) == 0
        else:
            assert ext.L.minigpt4_b200_end_chat_batch(ctypes.cast(ext._ctx_array(cs), ctypes.c_void_p), len(cs), ctypes.cast(toks, ctypes.c_void_p),
                                                      p["temp"], p["top_k"], p["top_p"], 1.0, 1.0, *UNUSED) == 0
        return [toks[i] for i in range(len(cs))]

    def loop(cs, stop, step):
        """the host loop over the live contexts; step(live) -> each live context's fed text"""
        B = len(cs)
        texts, chat, live = [[] for _ in range(B)], [b""] * B, list(range(B))
        while live:
            nxt = []
            for i, t in zip(live, step([cs[i] for i in live])):
                texts[i].append(t)
                chat[i] += t
                if not (t != b"##" and chat[i].endswith(stop)) and len(texts[i]) < MAX:
                    nxt.append(i)
            live = nxt
        return texts

    def run(arm, B, p, stop):
        """(seconds, [B] reply texts, steps the device ran past the last stop)"""
        cs = fresh(B)
        L0 = ext.stats(cs[0]).kernel_launches
        over = None
        t0 = time.perf_counter()
        if arm == "host":
            texts = loop(cs, stop, lambda live: end_chat_batch(live, p))
        elif arm == "steps1":
            texts = loop(cs, stop, lambda live: [text(c, i) for c, i in zip(live, ext.sample_steps(live, 1, **p)[0][0])])
        elif arm == "until":
            ids, _, _ = ext.sample_until(cs, MAX, stop, **p)
            texts = [[text(c, i) for i in x] for c, x in zip(cs, ids)]
        else:   # until16
            texts, live = [[] for _ in range(B)], list(range(B))
            while live:
                ids, stopped, _ = ext.sample_until([cs[i] for i in live], min(16, MAX - len(texts[live[0]])), stop, **p)
                nxt = []
                for i, x, s in zip(live, ids, stopped):
                    texts[i] += [text(cs[i], t) for t in x]
                    if not s and len(texts[i]) < MAX:
                        nxt.append(i)
                live = nxt
        t = time.perf_counter() - t0
        if arm == "until":
            launches = ext.stats(cs[0]).kernel_launches - L0
            over = launches // per_step[B] - max(len(x) for x in texts)
        for c in cs:
            ext.base.minigpt4_free(c)
        return t, texts, over

    per_step = {}
    for B in (1, 2, 4, 8):   # kernel launches of one sampled step of B contexts (also warms the graphs of every batch size)
        cs = fresh(B)
        x = ext.stats(cs[0]).kernel_launches
        ext.sample_steps(cs, 1, **PARAMS["webui"])
        per_step[B] = ext.stats(cs[0]).kernel_launches - x
        for c in cs:
            ext.base.minigpt4_free(c)

    # the stop text of each (B, parameters): one host run without a stop, then the token text whose first stops come closest to the targets
    stops = {}
    for pn, p in PARAMS.items():
        for B in (1, 2, 4, 8):
            want = [int(x) for x in np.linspace(128, 40, B)] if B > 1 else [96]
            cs = fresh(B)
            texts = [[] for _ in range(B)]
            for _ in range(128):
                for i, t in enumerate(end_chat_batch(cs, p)):
                    texts[i].append(t)
            for c in cs:
                ext.base.minigpt4_free(c)
            cands = {t[-k:] for tx in texts for t in tx for k in (1, 2, 3) if len(t) >= k and t != b"##"}

            def score(s):
                firsts = [first_stop(tx, s) for tx in texts]
                return sum(abs((MAX if f is None else f + 1) - w) for f, w in zip(firsts, want))
            stops[(B, pn)] = min(sorted(cands), key=score)
            print(f"stop text of {pn}/B{B}: {stops[(B, pn)]!r}", file=sys.stderr, flush=True)

    arms = [(arm, B, pn) for pn in PARAMS for B in (1, 2, 4, 8) for arm in ("host", "steps1", "until", "until16")]
    for a in arms:   # warm-up: scratch and stop state of every arm
        run(a[0], a[1], PARAMS[a[2]], stops[(a[1], a[2])])
    wall = {a: [] for a in arms}
    replies, overs = {}, {a: [] for a in arms}
    for r in range(args.rounds):
        print(f"round {r + 1} of {args.rounds}", file=sys.stderr, flush=True)
        for a in arms:
            t, tx, over = run(a[0], a[1], PARAMS[a[2]], stops[(a[1], a[2])])
            wall[a].append(t)
            replies.setdefault(a, tx)
            if over is not None:
                overs[a].append(over)
    same = {a: replies[a] == replies[("host", a[1], a[2])] for a in arms}
    for a in arms:
        if not same[a]:
            host = replies[("host", a[1], a[2])]
            i = next(i for i in range(a[1]) if replies[a][i] != host[i])
            k = next((k for k, (x, y) in enumerate(zip(replies[a][i], host[i])) if x != y), min(len(replies[a][i]), len(host[i])))
            print(f"{a}: context {i} differs from the host arm at token {k}: {replies[a][i][k:k + 3]} vs {host[i][k:k + 3]}, "
                  f"lengths {len(replies[a][i])} / {len(host[i])}", file=sys.stderr, flush=True)
    parity = all(same.values())
    legs = {}
    for a in arms:
        arm, B, pn = a
        t = min(wall[a])
        fed = sum(len(x) for x in replies[a])
        legs[f"{pn}/B{B}/{arm}"] = {"reply_ms": round(t * 1e3, 1), "tok_s": round(fed / t, 1), "spread": round(max(wall[a]) / t - 1.0, 3),
                                    "parity": same[a]}
        if overs[a]:
            legs[f"{pn}/B{B}/{arm}"]["steps_past_last_stop"] = max(overs[a])
    lengths = {f"{pn}/B{B}": {"stop": stops[(B, pn)].decode("utf-8", "replace"), "reply_tokens": [len(x) for x in replies[("host", B, pn)]]}
               for pn in PARAMS for B in (1, 2, 4, 8)}
    st = ext.stats(parent)
    out = {"metric": "whole-reply time and tokens/s, Vicuna-7B q4_1, n_ctx 2048, after one image-chat turn", "rounds": args.rounds,
           "timing": "best of rounds, wall clock around synchronous calls, arms alternated", "reply_chunk": 4, "legs": legs, "replies": lengths,
           "decode_megakernel": st.decode_megakernel, "parity": parity, **gpu_card()}
    print(json.dumps(out))
    ext.base.minigpt4_free(parent)


if __name__ == "__main__":
    main()
