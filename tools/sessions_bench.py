"""Multi-session decode throughput: one Vicuna-7B Q4_1 model (language model only) serving a parent context and 7 sessions at n_ctx 2048,
each prefilled to a different length.  Times 128 host-driven greedy minigpt4_b200_decode_batch steps for B = 1, 2, 4, 8 (wall clock around
synchronous calls), alternated in the same run with the single-context legs: 128 device-chained steps (minigpt4_b200_decode_chain) and the
per-token minigpt4_end_chat loop.  Prints one JSON line.

    python tools/sessions_bench.py [--steps 128] [--rounds 3]

parity: each session's 32 greedy ids from batched B = 8 steps equal its 32 ids when it runs alone (each context's own decode path)."""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402

import bench  # noqa: E402
import minigpt4_cpp_b200 as m  # noqa: E402

N_CTX = 2048
N_CTXS = 8
PARITY_STEPS = 32


def gpu_card() -> dict:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(", ")
        return {"gpu": out[0], "power_limit": out[1], "sm_max_clock": out[2]}
    except (OSError, subprocess.SubprocessError, IndexError):
        return {"gpu": None, "power_limit": None, "sm_max_clock": None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=128)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    lib = m.load_library()
    ext = m.B200(lib)
    if ext.L.minigpt4_b200_device_count() < 1:
        sys.exit("sessions_bench.py needs a CUDA device")
    _, llm, _ = bench.ensure_models("7b", "q4_1", 39)
    parent = ext.llm_load(llm, n_ctx=N_CTX, seed=1)
    ctxs = [parent] + [ext.session_create(parent, seed=2 + i) for i in range(N_CTXS - 1)]
    rng = np.random.default_rng(0)
    prompts = [rng.integers(3, 32000, size=32 + 40 * i).tolist() for i in range(N_CTXS)]   # 32 .. 312 rows: every context at its own n_past

    def fresh(cs):
        for c in cs:
            lib.minigpt4_reset_chat(c)
        for c, p in zip(cs, prompts):
            ext.eval_tokens(c, p); ext.flush(c)

    # parity: batched ids == ids alone
    fresh(ctxs)
    batched = np.stack([ext.decode_batch(ctxs) for _ in range(PARITY_STEPS)], 1)
    fresh(ctxs)
    alone = []
    for c in ctxs:
        ids = []
        for _ in range(PARITY_STEPS):
            ext.eval_tokens(c, [ext.greedy_id(c)]); ids.append(ext.greedy_id(c))
        alone.append(ids)
    parity = bool(np.array_equal(batched, np.array(alone)))

    # warm-up: every batch size's graph, the chain and the end_chat loop
    fresh(ctxs)
    for B in (1, 2, 4, 8):
        for _ in range(4):
            ext.decode_batch(ctxs[:B])
    ext.decode_chain(parent, 4)
    for _ in range(4):
        lib.minigpt4_end_chat(parent, temp=0.0)

    S = args.steps
    legs = {f"batch_B{B}": B for B in (1, 2, 4, 8)}
    legs.update({"decode_chain": 0, "end_chat": -1})
    wall = {k: [] for k in legs}
    for _ in range(args.rounds):
        for name, B in legs.items():   # alternated: every round runs every leg from the same positions
            fresh(ctxs)
            t0 = time.perf_counter()
            if B > 0:
                sub = ctxs[:B]
                for _ in range(S):
                    ext.decode_batch(sub)
            elif B == 0:
                ext.decode_chain(parent, S)
            else:
                for _ in range(S):
                    lib.minigpt4_end_chat(parent, temp=0.0)
            wall[name].append(time.perf_counter() - t0)
    res = {}
    for name, B in legs.items():
        t = min(wall[name])
        n_tok = S * max(B, 1)
        res[name] = {"tok_s": round(n_tok / t, 1), "ms_per_step": round(t / S * 1e3, 3), "contexts": max(B, 1),
                     "spread": round(max(wall[name]) / t - 1.0, 3)}
    n, owned, shared = ext.session_info(ctxs[1])
    st = ext.stats(parent)
    out = {"metric": "aggregate decode tokens/s, Vicuna-7B q4_1, n_ctx 2048, 8 contexts of one model at 32..312 prompt rows",
           "steps": S, "rounds": args.rounds, "timing": "best of rounds, wall clock around synchronous calls", "legs": res,
           "owned_bytes_per_session": owned, "shared_bytes": shared, "n_contexts": n, "decode_megakernel": st.decode_megakernel,
           "parity": parity, **gpu_card()}
    print(json.dumps(out))
    for c in ctxs:
        ext.base.minigpt4_free(c)


if __name__ == "__main__":
    main()
