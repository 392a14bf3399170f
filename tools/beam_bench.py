"""Beam search: the device call (minigpt4_b200_beam_search) against a host-driven beam loop.  Vicuna-7B-shaped models from modelgen
(Q4_1, Q5_K; language model only) at n_ctx 2048, after one image-chat turn (minigpt4_system_prompt + minigpt4_begin_chat_image with 32
seeded embedding rows), at 1, 2, 4, 8 and 16 beams.  Arms, alternated in the same run, best of --rounds with the spread:

- device: one minigpt4_b200_beam_search call;
- host: a beam loop built from the public calls: minigpt4_b200_get_logits of every live beam, the log-softmax, top-k and the walk in numpy
  (tests/beam_spec.py's rules), minigpt4_b200_session_copy of the whole conversation into the slot of every beam that changes parent,
  and one minigpt4_b200_decode_batch step of the live beams;
- greedy: minigpt4_b200_sample_steps with temp 0 over the same contexts, the decode step the search runs under its kernels.

Every arm is timed by the wall clock around the whole call, which ends in a device synchronise: for the device arm that includes the copy
of the conversation into the working beams at the start and the prompt pass that evaluates the best reply into ctxs[0] at the end (2 or
more beams), which the call's own ms_out (also reported, "device_event_ms_step") leaves out.  Reported per model and width: wall ms per
step with stop "" (every arm runs --steps steps), the device call's overhead over the greedy arm on that clock, and the whole-reply wall
time of both arms with the chat's "###" (at most 256 steps; the reply length is reported).  parity: the device's hypotheses equal the
host loop's.  Prints one JSON line.

--profile: instead, one device call per width under torch.profiler (CUDA activities): the summed kernel time of beam_rank_kernel,
beam_merge_kernel and beam_reorder_kernel against the summed time of every kernel of the call (the kernels' share of the search).

    python tools/beam_bench.py [--rounds 3] [--steps 64] [--wtypes q4_1,q5_k] [--profile]"""
import argparse
import ctypes
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))

import numpy as np  # noqa: E402

import beam_spec as bs  # noqa: E402
import bench  # noqa: E402
import minigpt4_cpp_b200 as m  # noqa: E402
from tools.sessions_bench import gpu_card  # noqa: E402

N_CTX = 2048
WIDTHS = (1, 2, 4, 8, 16)
REPLY_MAX = 256
QUESTION = "Describe this image in detail, please."


def host_beam(ext, cs, max_steps, stop, texts, tail0=b""):
    """the search of minigpt4_b200_beam_search driven from the host over the contexts cs (cs[0] holds the conversation)"""
    B = len(cs)
    stop = b"###" if stop is None else stop
    if B > 1:
        ext.session_copy(cs[0], cs[1:])
    live = [(0, (), np.float32(0.0), tail0[-bs.KEEP:])]   # (slot, ids, S, tail) in beam order
    H, seq = [], 0
    for t in range(max_steps):
        cands = []
        for b, (s, ids, S, tail) in enumerate(live):
            z = ext.logits(cs[s])
            c = (S + bs.lp_row(z)).astype(np.float32)
            top = np.argpartition(-z, min(2 * B, z.size - 1))[:2 * B]
            top = top[np.lexsort((top, -z[top]))]
            cands += [(c[v], b, z[v], int(v)) for v in top]
        cands.sort(key=bs.order_key)
        nxt = []

        def offer(c, ids, stopped):
            nonlocal seq
            score = np.float32(float(c) / float(t + 1))
            if len(H) < B:
                H.append([score, c, ids, stopped, seq])
            else:
                w = min(range(B), key=lambda j: (float(H[j][0]), -H[j][4]))
                if score > H[w][0]:
                    H[w] = [score, c, ids, stopped, seq]
            seq += 1
        for r, (c, b, z, v) in enumerate(cands[:2 * B]):
            s, ids, S, tail = live[b]
            if bs.ends(tail, texts[v], stop):
                if r < B:
                    offer(c, ids + (v,), True)
            elif len(nxt) < B:
                nxt.append([s, ids + (v,), c, (tail + texts[v])[-bs.KEEP:], v])
        done = len(H) == B or not nxt
        if not done and t == max_steps - 1:
            for s, ids, c, tail, v in nxt:
                offer(c, ids, False)
            done = True
        if done:
            break
        # a parent keeps its first child in place; the other children take the slots of no parent, in order, by a whole-conversation copy
        parents = {x[0] for x in nxt}
        free = iter(s for s in range(B) if s not in parents)
        seen = set()
        for x in nxt:
            if x[0] in seen:
                d = next(free)
                ext.session_copy(cs[x[0]], [cs[d]])
                x[0] = d
            else:
                seen.add(x[0])
        ext.decode_batch([cs[x[0]] for x in nxt], [x[4] for x in nxt])
        live = [(x[0], x[1], x[2], x[3]) for x in nxt]
    out = sorted(H, key=lambda e: (-float(e[0]), e[4]))
    return [(list(e[2]), bool(e[3])) for e in out]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=64)
    ap.add_argument("--wtypes", default="q4_1,q5_k")
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    lib = m.load_library()
    ext = m.B200(lib)
    if ext.L.minigpt4_b200_device_count() < 1:
        sys.exit("beam_bench.py needs a CUDA device")
    result = {"card": gpu_card(), "steps": args.steps, "rounds": args.rounds, "models": {}}
    rng = np.random.default_rng(0)
    emb = rng.standard_normal((32, 4096)).astype(np.float32) * 0.05
    view = m.MiniGPT4Embedding(emb.ctypes.data_as(ctypes.POINTER(ctypes.c_float)), emb.size)
    for wtype in args.wtypes.split(","):
        _, llm, _ = bench.ensure_models("7b", wtype, 39)
        parent = ext.llm_load(llm, n_ctx=N_CTX, seed=1)
        texts = [ext.L.minigpt4_b200_token_text(parent.ptr, i) for i in range(ext.L.minigpt4_b200_n_vocab(parent.ptr))]
        pool = [ext.session_create(parent) for _ in range(max(WIDTHS))]

        def fresh(B):
            cs = pool[:B]
            lib.minigpt4_reset_chat(cs[0])
            lib.minigpt4_system_prompt(cs[0])
            lib.minigpt4_begin_chat_image(cs[0], view, QUESTION)
            ext.flush(cs[0])
            if B > 1:
                ext.session_copy(cs[0], cs[1:])
            return cs

        def arm(name, B, stop, max_steps):
            cs = fresh(B)
            t0 = time.perf_counter()
            if name == "device":
                hyps, ms = ext.beam_search(cs, max_steps, stop, 1.0, B)
                out = [(h[0], h[3]) for h in hyps if h[0]]
            elif name == "host":
                out = host_beam(ext, cs, max_steps, stop, texts)
                ms = None
            else:
                _, ms = ext.sample_steps(cs, max_steps, temp=0.0)
                out = None
            return time.perf_counter() - t0, ms, out

        res = {}
        if args.profile:
            from torch.profiler import ProfilerActivity, profile
            for B in WIDTHS:
                arm("device", B, b"", 4)
                cs = fresh(B)
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    ext.beam_search(cs, args.steps, b"", 1.0, 1)
                k = {"beam": 0.0, "all": 0.0}
                for e in prof.events():
                    if e.device_type.name != "CUDA":
                        continue
                    us = e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
                    k["all"] += us
                    if "beam_rank_kernel" in e.name or "beam_merge_kernel" in e.name or "beam_reorder_kernel" in e.name:
                        k["beam"] += us
                row = {"beam_kernels_us_step": round(k["beam"] / args.steps, 2), "all_kernels_us_step": round(k["all"] / args.steps, 2),
                       "beam_share": round(k["beam"] / k["all"], 4) if k["all"] else None}
                res[str(B)] = row
                print(f"{wtype} B={B}: {json.dumps(row)}", file=sys.stderr, flush=True)
            result["models"][wtype] = res
            for c in pool + [parent]:
                ext.base.minigpt4_free(c)
            continue
        for B in WIDTHS:
            arm("device", B, b"", 4)   # warm the graphs and the search state
            arm("greedy", B, b"", 4)
            rec = {k: [] for k in ("device_wall_ms_step", "device_event_ms_step", "host_wall_ms_step", "greedy_wall_ms_step", "greedy_event_ms_step",
                                   "device_reply_ms", "host_reply_ms")}
            parity = True
            for _ in range(args.rounds):
                w, ms, d_out = arm("device", B, b"", args.steps)
                rec["device_event_ms_step"].append(ms / args.steps)
                rec["device_wall_ms_step"].append(1e3 * w / args.steps)
                w, _, h_out = arm("host", B, b"", args.steps)
                rec["host_wall_ms_step"].append(1e3 * w / args.steps)
                w, ms, _ = arm("greedy", B, b"", args.steps)
                rec["greedy_wall_ms_step"].append(1e3 * w / args.steps)
                rec["greedy_event_ms_step"].append(ms / args.steps)
                parity &= d_out == h_out
                w, _, d_out = arm("device", B, None, REPLY_MAX)
                rec["device_reply_ms"].append(1e3 * w)
                w, _, h_out = arm("host", B, None, REPLY_MAX)
                rec["host_reply_ms"].append(1e3 * w)
                parity &= d_out == h_out
                reply_len = len(d_out[0][0])
            row = {k: {"best": round(min(v), 3), "spread": round(max(v) - min(v), 3)} for k, v in rec.items()}
            dev, gr, host = (min(rec[k]) for k in ("device_wall_ms_step", "greedy_wall_ms_step", "host_wall_ms_step"))
            row["overhead_wall_ms_step"] = round(dev - gr, 3)         # the whole call against greedy steps, one clock
            row["overhead_wall_share"] = round((dev - gr) / dev, 4)
            row["host_minus_device_wall_ms_step"] = round(host - dev, 3)
            row["best_reply_len"] = reply_len
            row["parity"] = parity
            res[str(B)] = row
            print(f"{wtype} B={B}: {json.dumps(row)}", file=sys.stderr, flush=True)
        result["models"][wtype] = res
        for c in pool + [parent]:
            ext.base.minigpt4_free(c)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
