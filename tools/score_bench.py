"""Scoring known continuations on one Vicuna-7B-shaped model (language model only): minigpt4_b200_score_tokens against the per-token loop a
caller needs without it (minigpt4_b200_eval_tokens of one id, get_logits, a log-softmax on the host).

  * one context at n_ctx 2048 after an image-chat turn (system prompt, "Human: <Img>", 32 synthetic image rows, "</Img> ", a question,
    "### Assistant:"), continuations of 64, 512 and 1536 tokens: the loop against one call with keep = 0 and with keep = 1;
  * 64 contexts x 256 tokens (n_ctx 512, so that 64 KV caches fit beside the weights): one call against 64 calls of one context each.

The Q4_1 file takes the tensor-core layers, the Q5_K file (--types q4_1,q5_k, the default) the per-op layers.  Each leg starts from the same
state (the turn is queued again and flushed outside the timed region); wall clock around synchronous calls; legs alternated, best of
--rounds with the spread.  Parity: the loop's host log-probabilities (float64, rounded to float32) and ranks against the call's, and the
64 contexts of one call against the single calls.  Prints one JSON line with the card name and power limit.

    python tools/score_bench.py [--rounds 3] [--types q4_1,q5_k]"""
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

LENGTHS = (64, 512, 1536)
WIDE_N, WIDE_LEN, WIDE_CTX = 64, 256, 512


def host_score(lg, t):
    """the log-probability and rank the host loop computes from one get_logits row"""
    mx = np.float64(lg.max())
    s = np.exp(lg.astype(np.float64) - mx).sum()
    return np.float32((np.float64(lg[t]) - mx) - np.log(s)), int(np.count_nonzero(lg > lg[t]) + np.count_nonzero(lg[:t] == lg[t]))


def ulps(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return int(np.max(np.abs(a.view(np.int32).astype(np.int64) - b.view(np.int32).astype(np.int64)))) if a.size else 0


def run(lib, ext, wtype: str, rounds: int) -> dict:
    _, llm, _ = bench.ensure_models("7b", wtype, 39)
    rng = np.random.default_rng(0)
    emb = rng.standard_normal((32, 4096)).astype(np.float32) * 0.05
    view = m.MiniGPT4Embedding(emb.ctypes.data_as(ctypes.POINTER(ctypes.c_float)), emb.size)
    ctx = ext.llm_load(llm, n_ctx=2048, seed=1)
    V = ext.L.minigpt4_b200_n_vocab(ctx.ptr)
    conts = {n: rng.integers(3, V, size=n).tolist() for n in LENGTHS}

    def turn():
        lib.minigpt4_reset_chat(ctx)
        lib.minigpt4_system_prompt(ctx)
        lib.minigpt4_begin_chat_image(ctx, view, "What is in this picture?")
        ext.flush(ctx)

    def loop(ids):
        lp, rk = np.empty(len(ids), np.float32), np.empty(len(ids), np.int32)
        lg = ext.logits(ctx)
        for j, t in enumerate(ids):
            lp[j], rk[j] = host_score(lg, t)
            if j + 1 < len(ids):
                ext.eval_tokens(ctx, [t]); lg = ext.logits(ctx)
        return lp, rk

    legs = {}
    for n in LENGTHS:
        ids = conts[n]
        legs[f"loop_{n}"] = lambda ids=ids: loop(ids)
        legs[f"score_keep0_{n}"] = lambda ids=ids: ext.score_tokens([ctx], [ids])[0]
        legs[f"score_keep1_{n}"] = lambda ids=ids: ext.score_tokens([ctx], [ids], keep=True)[0]
    results = {}
    for name, fn in legs.items():   # warm-up, and the values the parity check compares
        turn(); results[name] = fn()
    wall = {k: [] for k in legs}
    for _ in range(rounds):
        for name, fn in legs.items():
            turn()
            t0 = time.perf_counter()
            fn()
            wall[name].append(time.perf_counter() - t0)
    res = {name: {"ms": round(min(t) * 1e3, 2), "spread": round(max(t) / min(t) - 1.0, 3)} for name, t in wall.items()}
    parity = {}
    for n in LENGTHS:
        res[f"speedup_keep0_{n}"] = round(res[f"loop_{n}"]["ms"] / res[f"score_keep0_{n}"]["ms"], 2)
        res[f"speedup_keep1_{n}"] = round(res[f"loop_{n}"]["ms"] / res[f"score_keep1_{n}"]["ms"], 2)
        (la, ra), (lb, rb), (lc, rc) = results[f"loop_{n}"], results[f"score_keep0_{n}"], results[f"score_keep1_{n}"]
        parity[n] = {"logprob_max_ulp": max(ulps(la, lb), ulps(la, lc)), "ranks_equal": bool(np.array_equal(ra, rb) and np.array_equal(ra, rc)),
                     "keep0_equals_keep1": bool(np.array_equal(lb, lc))}
    turn()
    prompt_rows = ext.n_past(ctx)
    ext.base.minigpt4_free(ctx)

    # ---- 64 contexts x 256 tokens: one call against 64 single calls
    parent = ext.llm_load(llm, n_ctx=WIDE_CTX, seed=1)
    ses = [parent] + [ext.session_create(parent, seed=2 + i) for i in range(WIDE_N - 1)]
    prompts = [rng.integers(3, V, size=16 + (7 * i) % 60).tolist() for i in range(WIDE_N)]
    wide = [rng.integers(3, V, size=WIDE_LEN).tolist() for _ in range(WIDE_N)]
    for c, p in zip(ses, prompts):
        ext.eval_tokens(c, p)
    ext.flush_batch(ses)
    one = ext.score_tokens(ses, wide)                                     # (warm-up)
    single = [ext.score_tokens([c], [w])[0] for c, w in zip(ses, wide)]
    wide_parity = all(np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) for a, b in zip(one, single))
    tw = {"one_call": [], "single_calls": []}
    for _ in range(rounds):
        t0 = time.perf_counter(); ext.score_tokens(ses, wide); tw["one_call"].append(time.perf_counter() - t0)
        t0 = time.perf_counter()
        for c, w in zip(ses, wide):
            ext.score_tokens([c], [w])
        tw["single_calls"].append(time.perf_counter() - t0)
    for name, t in tw.items():
        res[f"wide_{WIDE_N}x{WIDE_LEN}_{name}"] = {"ms": round(min(t) * 1e3, 2), "spread": round(max(t) / min(t) - 1.0, 3)}
    res[f"speedup_wide_{WIDE_N}x{WIDE_LEN}"] = round(min(tw["single_calls"]) / min(tw["one_call"]), 2)
    st = ext.stats(parent)
    _, owned, shared = ext.session_info(parent)
    for c in ses:
        ext.base.minigpt4_free(c)
    return {"prompt_rows": prompt_rows, "prefill_gemm": bool(st.prefill_gemm), "legs": res, "parity": parity, "wide_parity": wide_parity,
            "shared_bytes_after_scoring": shared, "owned_bytes_n_ctx_512": owned}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--types", default="q4_1,q5_k")
    args = ap.parse_args()
    lib = m.load_library()
    ext = m.B200(lib)
    if ext.L.minigpt4_b200_device_count() < 1:
        sys.exit("score_bench.py needs a CUDA device")
    out = {"metric": "wall ms to score a known continuation on a Vicuna-7B-shaped model: per-token eval_tokens + get_logits + host log-softmax "
                     "against one minigpt4_b200_score_tokens call", "rounds": args.rounds,
           "timing": "best of rounds, wall clock around synchronous calls, legs alternated"}
    for wt in args.types.split(","):
        out[wt] = run(lib, ext, wt, args.rounds)
    out.update(gpu_card())
    print(json.dumps(out))


if __name__ == "__main__":
    main()
