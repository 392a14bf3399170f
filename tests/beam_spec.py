"""minigpt4_b200_beam_search restated in Python (include/minigpt4_b200.h, DESIGN.md §4.13), shared by test_beam_host.py and
test_beam_gpu.py.  Runs over any logits function, in float32 where the device computes in float32."""
import numpy as np

KEEP = 32   # the reply tail's bytes that every later stop check reads (LlamaDevice::kStopMax)


def lp_row(z: np.ndarray) -> np.ndarray:
    """lp[v] = (float)(((double)z[v] - M) - log sum exp((double)z - M)), M = max z (the device sums in another order: within an ulp)"""
    zd = z.astype(np.float64)
    M = float(z.max())
    return ((zd - M) - np.log(np.sum(np.exp(zd - M)))).astype(np.float32)


def ends(tail: bytes, text: bytes, stop: bytes) -> bool:
    """sample_until's stop rule: the text is not exactly "##", the stop text is not empty and the reply then ends with it"""
    return text != b"##" and bool(stop) and (tail + text).endswith(stop)


def order_key(x):
    """candidates (c, beam, z, id): c descending, beam ascending, z descending, id ascending"""
    c, b, z, v = x
    return (-float(c), b, -float(z), v)


def ulps(a: float, b: float) -> int:
    """the distance between two float32 values in units in the last place"""
    ia, ib = (int(np.float32(x).view(np.int32)) for x in (a, b))
    ia = ia if ia >= 0 else -(ia & 0x7fffffff)
    ib = ib if ib >= 0 else -(ib & 0x7fffffff)
    return abs(ia - ib)


class NearTie(AssertionError):
    pass


def beam_search(logits_fn, n_beams: int, max_steps: int, texts, stop=b"###", length_penalty: float = 1.0, tail0: bytes = b"",
                lp_fn=lp_row, tie_ulps: int = 0, stats: dict | None = None):
    """The search over logits_fn(ids) (float32 logits after the ids).  Returns H in output order: [(ids, score, S, stopped)].
    tie_ulps > 0: raise NearTie where a decision compares two different float32 values (or equal ones of different beams) closer than
    that, so that a caller whose lp may differ from the device's in the last place knows the comparison is not safe.
    stats (may be None) takes "hash_exempt": the walked candidates whose text is "##" and would have ended the reply without the
    exception."""
    if stats is not None:
        stats["hash_exempt"] = 0
    stop = b"###" if stop is None else stop
    live = [((), np.float32(0.0), tail0[-KEEP:])]
    H = []   # [score, S, ids, stopped, seq]
    seq = 0

    def near(a, b):
        return tie_ulps and a != b and ulps(a, b) <= tie_ulps

    def offer(t, c, ids, stopped):
        nonlocal seq
        score = np.float32(float(c) / float(t + 1) ** float(length_penalty))
        if len(H) < n_beams:
            H.append([score, c, ids, stopped, seq])
        else:
            w = min(range(len(H)), key=lambda j: (float(H[j][0]), -H[j][4]))
            if near(score, H[w][0]):
                raise NearTie(f"offer at step {t}: {score} against {H[w][0]}")
            if score > H[w][0]:
                H[w] = [score, c, ids, stopped, seq]
        seq += 1

    for t in range(max_steps):
        cands = []
        for b, (ids, S, tail) in enumerate(live):
            z = np.asarray(logits_fn(ids), np.float32)
            c = (S + lp_fn(z)).astype(np.float32)
            top = np.lexsort((np.arange(z.size), -z))[:2 * n_beams]
            cands += [(c[v], b, z[v], int(v)) for v in top]
        cands.sort(key=order_key)
        if tie_ulps:
            for x, y in zip(cands[:2 * n_beams], cands[1:2 * n_beams + 1]):
                if near(x[0], y[0]) or (x[0] == y[0] and x[1] != y[1]):
                    raise NearTie(f"candidates at step {t}: {x} and {y}")
        nxt = []
        for r, (c, b, z, v) in enumerate(cands[:2 * n_beams]):
            ids, S, tail = live[b]
            if stats is not None and texts[v] == b"##" and stop and (tail + texts[v]).endswith(stop):
                stats["hash_exempt"] += 1
            if ends(tail, texts[v], stop):
                if r < n_beams:
                    offer(t, c, ids + (v,), True)
            elif len(nxt) < n_beams:
                nxt.append((ids + (v,), c, (tail + texts[v])[-KEEP:]))
        live = nxt
        if len(H) == n_beams or not live:
            break
        if t == max_steps - 1:
            for ids, S, tail in live:
                offer(t, S, ids, False)
    out = sorted(H, key=lambda e: (-float(e[0]), e[4]))
    if tie_ulps:
        for x, y in zip(out, out[1:]):
            if near(x[0], y[0]):
                raise NearTie(f"final scores {x[0]} and {y[0]}")
    return [(list(e[2]), float(e[0]), float(e[1]), bool(e[3])) for e in out]
