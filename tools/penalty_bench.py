"""Repetition penalties on the GPU: what minigpt4_b200_sample_until_penalized costs over minigpt4_b200_sample_until.  A Vicuna-7B-shaped
Q4_1 model from modelgen (language model only, n_vocab 32000), after one image-chat turn (minigpt4_system_prompt +
minigpt4_begin_chat_image with 32 seeded embedding rows), copied into B = 1, 8 and 64 fresh sessions seeded alike for both arms.  B = 1
and 8 run at n_ctx 2048; B = 64 at n_ctx 1024, since 65 contexts of n_ctx 2048 (1 GiB of K / V each) do not fit in 80 GB.

- steps: wall ms per step of sample_until and of sample_until_penalized (repeat_penalty 1.1, alphas 0, repeat_last_n 64 and 1024, each
  context's history 1024 seeded ids) with stop "" (every call runs --steps steps), timed around the call, which ends in a device
  synchronise; the web UI's parameters and top_k 0 / top_p 0.95; the two arms alternated, best of --rounds with the spread, and the
  overhead of the best against the best.  The penalised arm feeds other ids than the plain one, so the check here is that each arm feeds
  the same ids in every round.
- kernel: penalty_rows_kernel alone through minigpt4_b200_op_penalize at 1, 8 and 64 rows of 32000 seeded logits, windows of 64 and
  1024 ids, CUDA-event time of one launch averaged over 50.
- card: the name and power limit, read in the same run.  Prints one JSON line.

    python tools/penalty_bench.py [--rounds 3] [--steps 64]"""
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
WINDOWS = (64, 1024)
HISTORY = 1024
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
        sys.exit("penalty_bench.py needs a CUDA device")
    result = {"card": gpu_card(), "model": "7b-q4_1", "n_ctx": {f"B{b}": c for b, c in N_CTX.items()}, "steps_per_call": args.steps,
              "rounds": args.rounds, "repeat_penalty": 1.1, "history_ids": HISTORY}

    # ---- the kernel alone
    rng = np.random.default_rng(0)
    kern = {}
    for rows in WIDTHS:
        lg = (rng.standard_normal((rows, 32000)) * 3).astype(np.float32)
        hist = [rng.integers(0, 32000, size=HISTORY).tolist() for _ in range(rows)]
        for w in WINDOWS:
            ext.op_penalize(lg, hist, w, 1.1)   # warm
            kern[f"rows{rows}/window{w}"] = round(1e3 * ext.op_penalize(lg, hist, w, 1.1)[1], 2)
    result["kernel_us"] = kern
    print(f"kernel us: {json.dumps(kern)}", file=sys.stderr, flush=True)

    # ---- whole steps
    _, llm, _ = bench.ensure_models("7b", "q4_1", 39)
    emb = rng.standard_normal((32, 4096)).astype(np.float32) * 0.05
    view = m.MiniGPT4Embedding(emb.ctypes.data_as(ctypes.POINTER(ctypes.c_float)), emb.size)

    def arm(B, p, window, hist):
        """one call on B fresh sessions (seeds 100..) holding the conversation: (wall s, device ms, ids)"""
        cs = [ext.session_create(parent, 100 + i) for i in range(B)]
        ext.session_copy(parent, cs)
        t0 = time.perf_counter()
        if window is None:
            ids, _, ms = ext.sample_until(cs, args.steps, b"", **p)
        else:
            ids, _, ms = ext.sample_until_penalized(cs, args.steps, b"", hist[:B], repeat_last_n=window, repeat_penalty=1.1, **p)
        w = time.perf_counter() - t0
        for c in cs:
            ext.base.minigpt4_free(c)
        return w, ms, ids

    steps = {}
    hist = [rng.integers(3, 32000, size=HISTORY).tolist() for _ in range(max(WIDTHS))]
    for B in WIDTHS:
        parent = ext.llm_load(llm, n_ctx=N_CTX[B], seed=1)
        lib.minigpt4_system_prompt(parent)
        lib.minigpt4_begin_chat_image(parent, view, QUESTION)
        ext.flush(parent)
        for pn, p in PARAMS.items():
            arm(B, p, None, hist); arm(B, p, WINDOWS[-1], hist)   # warm the batch graph and every context's scratch
            for window in WINDOWS:
                rec = {k: [] for k in ("plain_wall_ms_step", "penalized_wall_ms_step", "plain_event_ms_step", "penalized_event_ms_step")}
                same0, same1, ref0, ref1 = True, True, None, None
                for _ in range(args.rounds):
                    w0, ms0, ids0 = arm(B, p, None, hist)
                    w1, ms1, ids1 = arm(B, p, window, hist)
                    ref0, ref1 = ref0 or ids0, ref1 or ids1
                    same0 &= ids0 == ref0
                    same1 &= ids1 == ref1
                    rec["plain_wall_ms_step"].append(1e3 * w0 / args.steps)
                    rec["penalized_wall_ms_step"].append(1e3 * w1 / args.steps)
                    rec["plain_event_ms_step"].append(ms0 / args.steps)
                    rec["penalized_event_ms_step"].append(ms1 / args.steps)
                row = {k: {"best": round(min(v), 4), "spread": round(max(v) - min(v), 4)} for k, v in rec.items()}
                a, b = min(rec["plain_wall_ms_step"]), min(rec["penalized_wall_ms_step"])
                row["overhead_wall_ms_step"] = round(b - a, 4)
                row["overhead_wall_share"] = round((b - a) / a, 4)
                row["repeatable"] = same0 and same1
                row["ids_differ"] = ref0 != ref1
                steps[f"{pn}/B{B}/window{window}"] = row
                print(f"{pn} B={B} window={window}: {json.dumps(row)}", file=sys.stderr, flush=True)
        ext.base.minigpt4_free(parent)
    result["steps"] = steps
    result["repeatable"] = all(r["repeatable"] for r in steps.values())
    print(json.dumps(result))


if __name__ == "__main__":
    main()
