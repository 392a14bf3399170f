"""Wide batches: one Vicuna-7B Q4_1 model (language model only) loaded twice at n_ctx 512, each load serving 64 contexts prefilled to
32..350 rows.  The first load has the tensor-core prefill GEMM; the second is loaded with MINIGPT4_B200_NO_PREFILL_GEMM=1, so its decode
steps of more than 8 columns run every layer on the per-op matvecs.  Both layer paths of minigpt4_b200_decode_batch are timed in one
process (two such loads fit on an 80 GB card at n_ctx 512, not at 2048).  Prints one JSON line.

    python tools/wide_batch_bench.py [--steps 32] [--rounds 3]

legs (alternated; best of rounds, with the spread):
  decode_B{B}: `steps` host-driven greedy decode_batch steps at B = 8, 9, 12, 16, 24, 32, 48, 64 on both loads.  Each leg takes the B
      contexts with the most room left, so that the legs of a round share one prefill (a leg of 128 steps would need a fresh prefill of
      every context, and the per-op load's prefill is the slow part of the run).
  decode_8x8: the same 64 contexts as 8 sequential decode_batch calls of 8 per step, on the tensor-core load.
  sample_steps_B8 / _B64: one sample_steps(steps=128) call, web UI parameters, on the tensor-core load from a fresh prefill.
  sample_until_B64: sample_until in 16-step calls over the contexts still running, up to 128 steps, on the tensor-core load.
parity: 8 batched greedy steps at B = 64 on each load equal, for contexts 0, 31 and 63, 8 steps of the same prompt on a context of its own."""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import numpy as np  # noqa: E402

import bench  # noqa: E402
import minigpt4_cpp_b200 as m  # noqa: E402
from sessions_bench import gpu_card  # noqa: E402

N_CTX = 512
N_CTXS = 64
WIDTHS = (8, 9, 12, 16, 24, 32, 48, 64)
WEBUI = dict(temp=0.8, top_k=40, top_p=0.9)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=32)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    lib = m.load_library()
    ext = m.B200(lib)
    if ext.L.minigpt4_b200_device_count() < 1:
        sys.exit("wide_batch_bench.py needs a CUDA device")
    _, llm, _ = bench.ensure_models("7b", "q4_1", 39)
    rng = np.random.default_rng(0)
    lens = np.linspace(32, 350, N_CTXS).astype(int)
    prompts = [rng.integers(3, 32000, size=int(n)).tolist() for n in lens]

    def load(seed):
        parent = ext.llm_load(llm, n_ctx=N_CTX, seed=seed)
        return [parent] + [ext.session_create(parent, seed=seed + 1 + i) for i in range(N_CTXS - 1)]

    tc = load(1)
    os.environ["MINIGPT4_B200_NO_PREFILL_GEMM"] = "1"
    po = load(1)
    del os.environ["MINIGPT4_B200_NO_PREFILL_GEMM"]
    assert ext.stats(tc[0]).prefill_gemm and not ext.stats(po[0]).prefill_gemm
    groups = {"tensor_core_load": tc, "per_op_load": po}
    flush_s = {k: [] for k in groups}

    def fresh(name):
        cs = groups[name]
        for c in cs:
            lib.minigpt4_reset_chat(c)
        for c, p in zip(cs, prompts):
            ext.eval_tokens(c, p)
        t0 = time.perf_counter()
        ext.flush_batch(cs)
        flush_s[name].append(time.perf_counter() - t0)

    # parity: batched ids == ids alone (a session of the tensor-core load stepping on its own decode path)
    solo = ext.session_create(tc[0], seed=999)
    alone = {}
    for i in (0, 31, 63):
        lib.minigpt4_reset_chat(solo)
        ext.eval_tokens(solo, prompts[i]); ext.flush(solo)
        ids = []
        for _ in range(8):
            ext.eval_tokens(solo, [ext.greedy_id(solo)]); ids.append(ext.greedy_id(solo))
        alone[i] = ids
    parity = {}
    for name, cs in groups.items():
        fresh(name)
        got = np.stack([ext.decode_batch(cs) for _ in range(8)], 1)
        parity[name] = all(got[i].tolist() == alone[i] for i in alone)
    ext.base.minigpt4_free(solo)

    S = args.steps

    def roomiest(cs, B):
        return sorted(cs, key=ext.n_past)[:B]

    def ensure_room(name, need):
        if max(ext.n_past(c) for c in groups[name]) + need > N_CTX:
            fresh(name)

    # warm-up: every width's graph on both loads, the sampling kernels
    for name in groups:
        fresh(name)
        for B in WIDTHS:
            ext.decode_batch(groups[name][:B])
    fresh("tensor_core_load")
    ext.sample_steps(tc[:8], 2, **WEBUI); ext.sample_steps(tc, 2, **WEBUI); ext.sample_until(tc, 2, **WEBUI)

    wall = {}

    def timed(key, fn):
        t0 = time.perf_counter()
        r = fn()
        wall.setdefault(key, []).append(time.perf_counter() - t0)
        return r

    until_steps = []
    for _ in range(args.rounds):
        for name in groups:
            fresh(name)
        for B in WIDTHS:
            for name, cs in groups.items():
                ensure_room(name, S)
                sub = roomiest(cs, B)
                timed((name, f"decode_B{B}"), lambda: [ext.decode_batch(sub) for _ in range(S)])
        ensure_room("tensor_core_load", S)
        chunks = [tc[k:k + 8] for k in range(0, N_CTXS, 8)]
        timed(("tensor_core_load", "decode_8x8"), lambda: [[ext.decode_batch(ch) for ch in chunks] for _ in range(S)])
        for B in (8, 64):
            fresh("tensor_core_load")
            timed(("tensor_core_load", f"sample_steps_B{B}"), lambda: ext.sample_steps(tc[:B], 128, **WEBUI))
        fresh("tensor_core_load")

        def until():
            running, steps = list(tc), 0
            while running and steps < 128:
                got, stopped, _ = ext.sample_until(running, 16, **WEBUI)
                steps += 16
                running = [c for c, s in zip(running, stopped) if not s]
            return steps
        until_steps.append(timed(("tensor_core_load", "sample_until_B64"), until))

    def leg(key, n_tok, steps):
        t = min(wall[key])
        return {"tok_s": round(n_tok / t, 1), "ms_per_step": round(t / steps * 1e3, 3), "spread": round(max(wall[key]) / t - 1.0, 3)}

    res = {name: {} for name in groups}
    for name in groups:
        for B in WIDTHS:
            res[name][f"decode_B{B}"] = dict(leg((name, f"decode_B{B}"), S * B, S), contexts=B)
    res["tensor_core_load"]["decode_8x8"] = dict(leg(("tensor_core_load", "decode_8x8"), S * N_CTXS, S), contexts=N_CTXS,
                                                 calls_per_step=8)
    for B in (8, 64):
        res["tensor_core_load"][f"sample_steps_B{B}"] = dict(leg(("tensor_core_load", f"sample_steps_B{B}"), 128 * B, 128), contexts=B)
    us = max(until_steps)
    res["tensor_core_load"]["sample_until_B64"] = dict(leg(("tensor_core_load", "sample_until_B64"), us * N_CTXS, us), contexts=N_CTXS,
                                                       steps_issued=us, note="tok_s counts every issued step of every context")
    n, owned, shared = ext.session_info(tc[1])
    _, owned_po, shared_po = ext.session_info(po[1])
    out = {"metric": "aggregate decode tokens/s, Vicuna-7B q4_1, n_ctx 512, 64 contexts of one model at 32..350 prompt rows",
           "steps": S, "rounds": args.rounds, "timing": "best of rounds, wall clock around synchronous calls", "legs": res,
           "flush_batch_s": {k: round(min(v), 3) for k, v in flush_s.items()},
           "owned_bytes_per_session": owned, "shared_bytes": shared, "owned_bytes_per_session_per_op_load": owned_po,
           "shared_bytes_per_op_load": shared_po, "n_contexts": n, "parity_batched_vs_alone": parity, **gpu_card()}
    print(json.dumps(out))
    for c in tc + po:
        ext.base.minigpt4_free(c)


if __name__ == "__main__":
    main()
