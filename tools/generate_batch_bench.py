"""Per-conversation settings in one batched reply call: what minigpt4_b200_generate_batch buys a server whose users pick their own settings.
A Vicuna-7B-shaped Q4_1 model from modelgen (language model only, n_vocab 32000) at n_ctx 1024, after one image-chat turn
(minigpt4_system_prompt + minigpt4_begin_chat_image with 32 seeded embedding rows), copied into 64 fresh sessions seeded alike for every arm.

- mixed: 8 setting groups of 8 contexts (greedy, the web UI chain, top_k 0 / top_p 0.95, a cooler chain, mirostat 1, mirostat 2, and the
  web UI chain and greedy with repeat_penalty 1.1), each group with its own budget (40 .. 96 steps), stop "" (budgets end the replies).
  Arm (a): one generate_batch call per 16-step chunk over every unfinished session.  Arm (b): per chunk, one single-settings call
  (sample_until / _mirostat / _penalized) per unfinished group, one after another.  Whole-reply wall time, ms per step of the longest
  reply, aggregate tok/s; the two arms must feed the same ids.
- uniform: the web UI chain for every context, 64 steps, stop "": generate_batch against sample_until at B = 1, 8 and 64.
- parent: with --parent lib.so, sample_until, _mirostat, _penalized and _logprobs (top_n 5) at B = 1, 8 and 64 (n_ctx 512, 32 steps)
  through the given build and this one, alternated in one process, with id parity.
- card: the name and power limit, read in the same run.  Best of --rounds alternated rounds with the spread.  Prints one JSON line.

    python tools/generate_batch_bench.py [--rounds 3] [--parent build/ab/parent.so]"""
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
from minigpt4_cpp_b200.minigpt4_library import _EXT, GenParams, MiniGPT4SharedLibrary  # noqa: E402
from tools.sessions_bench import gpu_card  # noqa: E402

QUESTION = "Describe this image in detail, please."
WEBUI = dict(temp=0.8, top_k=40, top_p=0.9)
PEN = dict(repeat_last_n=64, repeat_penalty=1.1)
GROUPS = [dict(temp=0.0), WEBUI, dict(temp=0.8, top_k=0, top_p=0.95), dict(temp=0.5, top_k=20, top_p=0.8), dict(temp=0.8, mirostat=1),
          dict(temp=0.8, mirostat=2), dict(WEBUI, **PEN), dict(temp=0.0, **PEN)]
BUDGETS = [96, 80, 64, 48, 40, 88, 72, 56]
CHUNK = 16


class OtherBuild(m.B200):
    """B200 over a build that may predate some entry points (those are left unbound)"""

    def __init__(self, lib):
        self.base, self.L = lib, lib.library
        for name, (argtypes, restype) in _EXT.items():
            fn = getattr(self.L, name, None)
            if fn is not None:
                fn.argtypes, fn.restype = argtypes, restype


def stats(v):
    return {"best": round(min(v), 4), "spread": round(max(v) - min(v), 4)}


def conversation(lib, ext, llm, n_ctx, rng):
    parent = ext.llm_load(llm, n_ctx=n_ctx, seed=1)
    emb = (rng.standard_normal((32, 4096)) * 0.05).astype(np.float32)
    view = m.MiniGPT4Embedding(emb.ctypes.data_as(ctypes.POINTER(ctypes.c_float)), emb.size)
    lib.minigpt4_system_prompt(parent)
    lib.minigpt4_begin_chat_image(parent, view, QUESTION)
    ext.flush(parent)
    return parent


def sessions(ext, parent, B):
    cs = [ext.session_create(parent, 100 + i) for i in range(B)]
    ext.session_copy(parent, cs)
    return cs


def free(ext, cs):
    for c in cs:
        ext.base.minigpt4_free(c)


def single(ext, cs, g, steps, hist):
    """the single-settings call that g selects, `steps` steps, histories hist (penalised groups)"""
    if "repeat_penalty" in g:
        p = {k: v for k, v in g.items() if k not in PEN}
        return ext.sample_until_penalized(cs, steps, b"", hist, **PEN, **p)[0]
    return ext.sample_until(cs, steps, b"", **g)[0]


def mixed(ext, parent, batched):
    """one whole-reply run of 64 sessions in 8 groups: (wall s, ids per session)"""
    cs = sessions(ext, parent, 64)
    got = [[] for _ in range(64)]
    group_of = [i // 8 for i in range(64)]
    t0 = time.perf_counter()
    while True:
        live = [i for i in range(64) if len(got[i]) < BUDGETS[group_of[i]]]
        if not live:
            break
        if batched:
            params = []
            for i in live:
                g = GROUPS[group_of[i]]
                extra = dict(last_ids=got[i]) if "repeat_penalty" in g else {}
                params.append(GenParams(max_steps=min(CHUNK, BUDGETS[group_of[i]] - len(got[i])), stop=b"", **g, **extra))
            ids = ext.generate_batch([cs[i] for i in live], params)[0]
            for i, x in zip(live, ids):
                got[i] += x
        else:
            for k, g in enumerate(GROUPS):
                members = [i for i in live if group_of[i] == k]
                if members:
                    steps = min(CHUNK, BUDGETS[k] - len(got[members[0]]))
                    ids = single(ext, [cs[i] for i in members], g, steps, [got[i] for i in members])
                    for i, x in zip(members, ids):
                        got[i] += x
    w = time.perf_counter() - t0
    free(ext, cs)
    return w, got


def uniform(ext, parent, B, steps, batched):
    cs = sessions(ext, parent, B)
    t0 = time.perf_counter()
    if batched:
        ids = ext.generate_batch(cs, [GenParams(max_steps=steps, stop=b"", **WEBUI)] * B)[0]
    else:
        ids = ext.sample_until(cs, steps, b"", **WEBUI)[0]
    w = time.perf_counter() - t0
    free(ext, cs)
    return w, ids


def existing_call(ext, cs, kind, steps):
    if kind == "sample_until":
        return ext.sample_until(cs, steps, b"", **WEBUI)[0]
    if kind == "mirostat":
        return ext.sample_until(cs, steps, b"", temp=0.8, mirostat=2)[0]
    if kind == "penalized":
        return ext.sample_until_penalized(cs, steps, b"", None, **PEN, **WEBUI)[0]
    return ext.sample_until_logprobs(cs, steps, b"", 5, **WEBUI)[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--parent", default=None, help="another build of libminigpt4.so to time the existing calls against")
    args = ap.parse_args()
    lib = m.load_library()
    ext = m.B200(lib)
    if ext.L.minigpt4_b200_device_count() < 1:
        sys.exit("generate_batch_bench.py needs a CUDA device")
    result = {"card": gpu_card(), "model": "7b-q4_1", "rounds": args.rounds}
    rng = np.random.default_rng(0)
    _, llm, _ = bench.ensure_models("7b", "q4_1", 39)
    llm = str(llm)

    # ---- mixed settings: one call per chunk against one call per group per chunk
    parent = conversation(lib, ext, llm, 1024, rng)
    mixed(ext, parent, True); mixed(ext, parent, False)   # warm every batch graph and scratch
    rec = {"a": [], "b": []}
    ref, same = None, True
    for _ in range(args.rounds):
        for arm in ("a", "b"):
            w, ids = mixed(ext, parent, arm == "a")
            rec[arm].append(w)
            ref = ref or ids
            same &= ids == ref
    tok = sum(BUDGETS) * 8
    steps = max(BUDGETS)
    row = {}
    for arm, name in (("a", "generate_batch"), ("b", "one_call_per_group")):
        row[name] = {"wall_s": stats(rec[arm]), "ms_per_step": round(1e3 * min(rec[arm]) / steps, 3), "tok_s": round(tok / min(rec[arm]), 1)}
    row["speedup"] = round(min(rec["b"]) / min(rec["a"]), 3)
    row["same_ids"] = same
    result["mixed_64x8"] = row
    print(f"mixed: {json.dumps(row)}", file=sys.stderr, flush=True)

    # ---- uniform settings: generate_batch against sample_until
    uni = {}
    for B in (1, 8, 64):
        uniform(ext, parent, B, 64, True); uniform(ext, parent, B, 64, False)
        r = {"generate_batch": [], "sample_until": []}
        ids_same = True
        for _ in range(args.rounds):
            w0, i0 = uniform(ext, parent, B, 64, False)
            w1, i1 = uniform(ext, parent, B, 64, True)
            r["sample_until"].append(1e3 * w0 / 64)
            r["generate_batch"].append(1e3 * w1 / 64)
            ids_same &= i0 == i1
        u = {k + "_ms_step": stats(v) for k, v in r.items()}
        u["overhead_share"] = round(min(r["generate_batch"]) / min(r["sample_until"]) - 1, 4)
        u["same_ids"] = ids_same
        uni[f"B{B}"] = u
        print(f"uniform B={B}: {json.dumps(u)}", file=sys.stderr, flush=True)
    result["uniform"] = uni
    ext.base.minigpt4_free(parent)

    # ---- the existing calls through another build and this one
    if args.parent:
        builds = {"parent": OtherBuild(MiniGPT4SharedLibrary(os.path.abspath(args.parent))), "this": ext}
        parents = {k: conversation(e.base, e, llm, 512, np.random.default_rng(0)) for k, e in builds.items()}
        ab = {}
        for B in (1, 8, 64):
            for kind in ("sample_until", "mirostat", "penalized", "logprobs"):
                r, ids = {k: [] for k in builds}, {k: None for k in builds}
                same = True
                for rnd in range(args.rounds + 1):   # (round 0 warms)
                    for k, e in builds.items():
                        cs = sessions(e, parents[k], B)
                        t0 = time.perf_counter()
                        x = existing_call(e, cs, kind, 32)
                        w = time.perf_counter() - t0
                        free(e, cs)
                        ids[k] = ids[k] or x
                        same &= x == ids[k]
                        if rnd:
                            r[k].append(1e3 * w / 32)
                row = {k + "_ms_step": stats(v) for k, v in r.items()}
                row["this_vs_parent"] = round(min(r["this"]) / min(r["parent"]) - 1, 4)
                row["same_ids"] = same and ids["this"] == ids["parent"]
                ab[f"{kind}/B{B}"] = row
                print(f"{kind} B={B}: {json.dumps(row)}", file=sys.stderr, flush=True)
        result["existing_calls_vs_parent"] = ab
        for k, e in builds.items():
            e.base.minigpt4_free(parents[k])
    print(json.dumps(result))


if __name__ == "__main__":
    main()
