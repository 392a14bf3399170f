"""Beam search (minigpt4_b200_beam_search) restated in Python (tests/beam_spec.py) and checked on synthetic logit functions, with no GPU:
the candidate order and its ties, one beam against the greedy loop, H's replacement rule and the early end, length_penalty 0 / 1 / 2,
and steps with fewer live beams than n_beams.  test_beam_gpu.py runs the same restatement against the device."""
import zlib

import numpy as np
import pytest

import beam_spec as bs


def texts_of(V, seed=3):
    """a vocabulary of short pieces, about a quarter of them holding '#'"""
    rng = np.random.default_rng(seed)
    return [bytes(rng.choice(list(b"#ab #"), size=int(rng.integers(1, 4))).tolist()) for _ in range(V)]


def hashed_logits(V, seed, ties=False):
    """logits that depend on the ids so far; ties: few distinct values, so equal logits and equal scores are common"""
    def fn(ids):
        rng = np.random.default_rng(zlib.crc32(np.asarray((seed,) + tuple(ids), np.int64).tobytes()))
        if ties:
            return rng.integers(0, 4, V).astype(np.float32)
        return (rng.standard_normal(V) * 3).astype(np.float32)
    return fn


def greedy(fn, texts, max_steps, stop=b"###"):
    """sample_until with temp 0: the first largest logit (lowest id on ties), the stopping id fed"""
    ids, tail = [], b""
    for _ in range(max_steps):
        v = int(np.argmax(fn(tuple(ids))))
        ids.append(v)
        if bs.ends(tail, texts[v], stop):
            return ids, True
        tail = (tail + texts[v])[-bs.KEEP:]
    return ids, False


@pytest.mark.parametrize("ties", [False, True])
@pytest.mark.parametrize("stop", [b"###", b"#", b""])
def test_one_beam_is_greedy(ties, stop):
    V = 64
    texts = texts_of(V)
    for seed in range(20):
        fn = hashed_logits(V, seed, ties)
        want, stopped = greedy(fn, texts, 30, stop)
        got = bs.beam_search(fn, 1, 30, texts, stop)
        assert len(got) == 1
        ids, score, S, st = got[0]
        assert (ids, st) == (want, stopped)
        lp = np.float32(0.0)
        for j, v in enumerate(ids):   # S is the float32 left fold of the log-probabilities
            lp = np.float32(lp + bs.lp_row(fn(tuple(ids[:j])))[v])
        assert S == float(lp) and score == float(np.float32(float(lp) / len(ids)))


def test_candidate_order_and_ties():
    # equal c across beams: the lower beam first; within a beam equal logits: the lower id first
    cands = [(np.float32(-1.0), 1, np.float32(2.0), 5), (np.float32(-1.0), 0, np.float32(1.0), 9), (np.float32(-0.5), 2, np.float32(0.0), 1),
             (np.float32(-1.0), 0, np.float32(1.0), 3), (np.float32(-1.0), 0, np.float32(1.5), 7)]
    got = [(b, v) for _, b, _, v in sorted(cands, key=bs.order_key)]
    assert got == [(2, 1), (0, 7), (0, 3), (0, 9), (1, 5)]
    # one beam, a row of equal logits: every id is a candidate of equal c, taken in id order
    V = 8
    texts = [b"a"] * V
    got = bs.beam_search(lambda ids: np.zeros(V, np.float32), 4, 1, texts, b"")
    assert [h[0] for h in got] == [[0], [1], [2], [3]]


def _three_offers(lp_pen):
    """n_beams 2: step 0 offers id 0 (r 0) and keeps ids 1 and 2; step 1 offers id 0 of both beams (r 0 and r 1)"""
    V = 4
    texts = [b"X#", b"a", b"b", b"c"]
    z0 = np.array([3.0, 2.99, 2.98, 0.0], np.float32)
    z1 = np.array([5.0, 0.0, 0.0, 0.0], np.float32)
    calls = []

    def fn(ids):
        calls.append(tuple(ids))
        return z0 if not ids else z1
    got = bs.beam_search(fn, 2, 10, texts, b"#", lp_pen)
    l0, l1 = bs.lp_row(z0), bs.lp_row(z1)
    offers = [([0], l0[0], 1), ([1, 0], np.float32(l0[1] + l1[0]), 2), ([2, 0], np.float32(l0[2] + l1[0]), 2)]
    return got, offers, calls


@pytest.mark.parametrize("lp_pen", [0.0, 1.0, 2.0])
def test_replacement_early_end_and_length_penalty(lp_pen):
    got, offers, calls = _three_offers(lp_pen)
    assert calls == [(), (1,), (2,)]   # the search ends after step 1: H is full, the live beams are not offered
    scores = [np.float32(float(c) / float(L) ** lp_pen) for _, c, L in offers]
    H = [0, 1]   # the first two fill H; the third replaces the worst only if strictly greater
    w = min(H, key=lambda j: (float(scores[j]), -j))
    if scores[2] > scores[w]:
        H[H.index(w)] = 2
    want = sorted(H, key=lambda j: (-float(scores[j]), j))
    assert [h[0] for h in got] == [offers[j][0] for j in want]
    assert [h[1] for h in got] == [float(scores[j]) for j in want]
    assert [h[2] for h in got] == [float(offers[j][1]) for j in want]
    assert all(h[3] for h in got)
    # which entries survive depends on the penalty: lp 0 keeps the one-id reply, 1 and 2 let the third offer replace it
    assert ([0] in [h[0] for h in got]) == (lp_pen == 0.0)


def test_fewer_live_beams_and_the_last_step():
    V = 8
    texts = [b"#"] * 6 + [b"a", b"b"]   # only ids 6 and 7 keep a reply going

    calls = []

    def fn(ids):
        calls.append(tuple(ids))
        z = np.zeros(V, np.float32)
        z[6], z[7] = 1.0, 0.5   # the non-ending ids rank first; then 6 ending ids with r >= 2 of n_beams 4 ... some r < 4
        return z
    got = bs.beam_search(fn, 4, 3, texts, b"#", 0.0)
    # step 0: r 0, 1 are ids 6, 7 (live), r 2, 3 end and are offered, r 4.. are dropped: two live beams, two entries
    assert calls[:3] == [(), (6,), (7,)]
    # step 1: two beams of 8 candidates; the first 8 in order: (6,6), (6,7), (7,6), (7,7) live, then ending ones of rank >= 4 dropped
    # step 2 (the last): 4 beams take their children; H has 2 entries, so the live beams are offered at the end, and with length_penalty
    # 0 the two best of them fill H
    assert len([c for c in calls if len(c) == 2]) == 4
    assert len(got) == 4 and sum(h[3] for h in got) == 2
    assert all(len(h[0]) == 3 for h in got if not h[3])


def test_near_tie_detection():
    V = 4
    texts = [b"a"] * V
    z = np.array([1.0, np.nextafter(np.float32(1.0), np.float32(0.0)), -5, -5], np.float32)
    with pytest.raises(bs.NearTie):
        bs.beam_search(lambda ids: z, 2, 2, texts, b"", tie_ulps=4)
    bs.beam_search(lambda ids: z, 2, 2, texts, b"")   # without the check the order is the float32 order
