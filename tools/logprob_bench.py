"""Log-probabilities of generated replies: what minigpt4_b200_sample_until_logprobs costs over minigpt4_b200_sample_until.  A Vicuna-7B-shaped
Q4_1 model from modelgen (language model only, n_vocab 32000), after one image-chat turn (minigpt4_system_prompt +
minigpt4_begin_chat_image with 32 seeded embedding rows), copied into B = 1, 8 and 64 fresh sessions seeded alike for both arms.  B = 1
and 8 run at n_ctx 2048; B = 64 at n_ctx 1024, since 65 contexts of n_ctx 2048 (1 GiB of K / V each) do not fit in 80 GB.

- steps: wall ms per step of sample_until and of sample_until_logprobs (top_n 0, 5, 20) with stop "" (every call runs --steps steps), timed
  around the call, which ends in a device synchronise; the web UI's parameters and top_k 0 / top_p 0.95; the two arms alternated, best of
  --rounds with the spread, and the overhead of the best against the best.  parity: both arms fed the same ids.
- kernel: logprob_rows_kernel alone through minigpt4_b200_op_logprobs at 1, 8 and 64 rows of 32000 seeded logits, CUDA-event time of one
  launch averaged over 50.
- card: the name and power limit, read in the same run.  Prints one JSON line.

    python tools/logprob_bench.py [--rounds 3] [--steps 64]"""
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

WIDTHS = (1, 8, 64)
N_CTX = {1: 2048, 8: 2048, 64: 1024}
TOP_NS = (0, 5, 20)
PARAMS = {"webui": dict(temp=0.8, top_k=40, top_p=0.9), "top_k-0-top_p-0.95": dict(temp=0.8, top_k=0, top_p=0.95)}
QUESTION = "Describe this image in detail, please."


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=64)
    args = ap.parse_args()
    lib = m.load_library()
    ext = m.B200(lib)
    if ext.L.minigpt4_b200_device_count() < 1:
        sys.exit("logprob_bench.py needs a CUDA device")
    result = {"card": gpu_card(), "model": "7b-q4_1", "n_ctx": {f"B{b}": c for b, c in N_CTX.items()}, "steps_per_call": args.steps, "rounds": args.rounds}

    # ---- the kernel alone
    rng = np.random.default_rng(0)
    kern = {}
    for rows in WIDTHS:
        lg = (rng.standard_normal((rows, 32000)) * 3).astype(np.float32)
        ids = rng.integers(0, 32000, size=rows)
        for top_n in TOP_NS:
            ext.op_logprobs(lg, ids, top_n)   # warm
            kern[f"rows{rows}/top{top_n}"] = round(1e3 * ext.op_logprobs(lg, ids, top_n)[4], 2)
    result["kernel_us"] = kern
    print(f"kernel us: {json.dumps(kern)}", file=sys.stderr, flush=True)

    # ---- whole steps
    _, llm, _ = bench.ensure_models("7b", "q4_1", 39)
    emb = rng.standard_normal((32, 4096)).astype(np.float32) * 0.05
    view = m.MiniGPT4Embedding(emb.ctypes.data_as(ctypes.POINTER(ctypes.c_float)), emb.size)

    def arm(B, p, top_n):
        """one call on B fresh sessions (seeds 100..) holding the conversation: (wall s, device ms, ids)"""
        cs = [ext.session_create(parent, 100 + i) for i in range(B)]
        ext.session_copy(parent, cs)
        t0 = time.perf_counter()
        if top_n is None:
            ids, _, ms = ext.sample_until(cs, args.steps, b"", **p)
        else:
            ids, _, _, ms = ext.sample_until_logprobs(cs, args.steps, b"", top_n, **p)
        w = time.perf_counter() - t0
        for c in cs:
            ext.base.minigpt4_free(c)
        return w, ms, ids

    steps = {}
    for B in WIDTHS:
        parent = ext.llm_load(llm, n_ctx=N_CTX[B], seed=1)
        lib.minigpt4_system_prompt(parent)
        lib.minigpt4_begin_chat_image(parent, view, QUESTION)
        ext.flush(parent)
        for pn, p in PARAMS.items():
            arm(B, p, None); arm(B, p, 20)   # warm the batch graph and every context's scratch
            for top_n in TOP_NS:
                rec = {k: [] for k in ("plain_wall_ms_step", "logprobs_wall_ms_step", "plain_event_ms_step", "logprobs_event_ms_step")}
                parity = True
                for _ in range(args.rounds):
                    w0, ms0, ids0 = arm(B, p, None)
                    w1, ms1, ids1 = arm(B, p, top_n)
                    parity &= ids0 == ids1
                    rec["plain_wall_ms_step"].append(1e3 * w0 / args.steps)
                    rec["logprobs_wall_ms_step"].append(1e3 * w1 / args.steps)
                    rec["plain_event_ms_step"].append(ms0 / args.steps)
                    rec["logprobs_event_ms_step"].append(ms1 / args.steps)
                row = {k: {"best": round(min(v), 4), "spread": round(max(v) - min(v), 4)} for k, v in rec.items()}
                a, b = min(rec["plain_wall_ms_step"]), min(rec["logprobs_wall_ms_step"])
                row["overhead_wall_ms_step"] = round(b - a, 4)
                row["overhead_wall_share"] = round((b - a) / a, 4)
                row["parity"] = parity
                steps[f"{pn}/B{B}/top{top_n}"] = row
                print(f"{pn} B={B} top_n={top_n}: {json.dumps(row)}", file=sys.stderr, flush=True)
        ext.base.minigpt4_free(parent)
    result["steps"] = steps
    result["parity"] = all(r["parity"] for r in steps.values())
    print(json.dumps(result))


if __name__ == "__main__":
    main()
