"""The constraint compiler (minigpt4_b200_host_constraint_allowed; csrc/constraint.cpp) against a Python restatement of allowed(s): every
id's text walked byte by byte, id 2 special-cased, empty texts skipped, liveness pruned to a fixed point on the token transitions."""
import numpy as np
import pytest

from minigpt4_cpp_b200.minigpt4_library import choices_dfa


def _texts(mg, n_vocab):
    """the C strings minigpt4_end_chat returns: each piece up to its first NUL, id 2 as </s>"""
    t = [p.split(b"\0")[0] for p, _ in mg.make_vocab(n_vocab)]
    t[2] = b"</s>"
    return t


def _restated(texts, nxt, acc):
    S = len(acc)
    raw = [[] for _ in range(S)]
    for s in range(S):
        for i, t in enumerate(texts):
            if i == 2 or not t:
                continue
            q = s
            for b in t:
                q = int(nxt[q][b])
                if q < 0:
                    break
            if q >= 0:
                raw[s].append((i, q))
    live = [bool(a) for a in acc]
    changed = True
    while changed:
        changed = False
        for s in range(S):
            if not live[s] and any(live[q] for _, q in raw[s]):
                live[s] = changed = True
    out = []
    for s in range(S):
        if not live[s]:
            out.append(None)
            continue
        row = [(i, q) for i, q in raw[s] if live[q]] + ([(2, -1)] if acc[s] else [])
        out.append(sorted(row))
    return out


def _empty(n):
    return np.full((n, 256), -1, np.int32), np.zeros(n, np.uint8)


def _digits(k):
    nx, ac = _empty(k + 1)
    for s in range(k):
        nx[s, ord("0"):ord("9") + 1] = s + 1
    ac[1:] = 1
    return nx, ac


def _live_on_bytes_dead_on_tokens():
    """0 -a-> 1 -NUL-> 2 (accepts), 0 -b-> 3 (accepts): state 1 reaches an accepting state on bytes, but no piece carries NUL"""
    nx, ac = _empty(4)
    nx[0, ord("a")], nx[1, 0], nx[0, ord("b")] = 1, 2, 3
    ac[2] = ac[3] = 1
    return nx, ac


def _pairs_cycle():
    """(ab)*: a cycle through two states, accepting at the start"""
    nx, ac = _empty(2)
    nx[0, ord("a")], nx[1, ord("b")] = 1, 0
    ac[0] = 1
    return nx, ac


AUTOMATA = {
    "choices": lambda: choices_dfa([b"cat", b"car", b"cart", b"dog", b"no animal", b"no"]),
    "digits-1-3": lambda: _digits(3),
    "live-on-bytes-dead-on-tokens": _live_on_bytes_dead_on_tokens,
    "ab-cycle": _pairs_cycle,
}


@pytest.fixture(scope="module")
def vocab32000(mg, tmp_path_factory):
    p = str(tmp_path_factory.mktemp("constraint") / "llama-32000.bin")
    mg.write_llama_ggjt(p, mg.LlamaSpec(n_vocab=32000, n_embd=256, n_head=2, n_layer=1, wtype="q4_1"))
    return p


@pytest.mark.parametrize("name", list(AUTOMATA))
def test_allowed_equals_restatement(ext, mg, tiny, name):
    nx, ac = AUTOMATA[name]()
    want = _restated(_texts(mg, 1024), nx, ac)
    for s in range(len(ac)):
        got = ext.host_constraint_allowed(tiny["q4_1"], nx, ac, s)
        if want[s] is None:
            assert got is None, f"state {s} should be pruned"
        else:
            assert got is not None, f"state {s} pruned"
            assert list(zip(got[0].tolist(), got[1].tolist())) == want[s], f"state {s}"


def test_pruning_of_a_state_live_only_on_bytes(ext, tiny):
    nx, ac = _live_on_bytes_dead_on_tokens()
    assert ext.host_constraint_allowed(tiny["q4_1"], nx, ac, 1) is None
    ids, _ = ext.host_constraint_allowed(tiny["q4_1"], nx, ac, 0)
    assert ids.tolist() == [ord("b") + 3]   # the byte piece "b"; "a" leads to the dead state


def test_digits_at_n_vocab_32000(ext, mg, vocab32000):
    nx, ac = _digits(6)
    want = _restated(_texts(mg, 32000), nx, ac)
    for s in range(7):
        got = ext.host_constraint_allowed(vocab32000, nx, ac, s)
        assert list(zip(got[0].tolist(), got[1].tolist())) == want[s], f"state {s}"


def test_refusals(ext, tiny):
    path = tiny["q4_1"]
    nx, ac = _empty(2)
    nx[0, 0], ac[1] = 1, 1   # the only path needs byte 0x00, which no piece carries
    assert ext.host_constraint_refused(path, nx, ac)
    nx, ac = _digits(2)
    assert not ext.host_constraint_refused(path, nx, ac)
    assert ext.host_constraint_refused(path, nx[:0], ac[:0])                       # n_states 0
    bad = nx.copy(); bad[0, 5] = 3
    assert ext.host_constraint_refused(path, bad, ac)                              # a state past n_states - 1
    bad = nx.copy(); bad[1, 7] = -2
    assert ext.host_constraint_refused(path, bad, ac)                              # below -1
    nx, ac = _empty(1)
    assert ext.host_constraint_refused(path, nx, ac)                               # nothing accepts: start not live
    big = np.full((65537, 256), -1, np.int32)
    assert ext.host_constraint_refused(path, big, np.ones(65537, np.uint8))        # more than 65536 states


def test_allowed_reports_short_buffers_and_bad_states(ext, tiny):
    nx, ac = choices_dfa([b"yes", b"no"])
    ids, nxt = ext.host_constraint_allowed(tiny["q4_1"], nx, ac, 0)
    assert len(ids) >= 2
    nxa, aca = np.ascontiguousarray(nx), np.ascontiguousarray(ac)
    buf = np.zeros(1, np.int32)
    r = ext.L.minigpt4_b200_host_constraint_allowed(tiny["q4_1"].encode(), len(ac), nxa.ctypes.data, aca.ctypes.data, 0, buf.ctypes.data,
                                                    None, 1)
    assert r == -len(ids)
    for s in (-1, len(ac)):
        assert ext.L.minigpt4_b200_host_constraint_allowed(tiny["q4_1"].encode(), len(ac), nxa.ctypes.data, aca.ctypes.data, s, None, None,
                                                           0) == -1


def test_choices_dfa_accepts_exactly_the_choices():
    choices = [b"cat", b"car", b"cart", b"no"]
    nx, ac = choices_dfa(choices)
    def accepts(w):
        s = 0
        for b in w:
            s = nx[s, b]
            if s < 0:
                return False
        return bool(ac[s])
    for w in choices:
        assert accepts(w)
    for w in (b"", b"ca", b"carts", b"n", b"dog"):
        assert not accepts(w)
