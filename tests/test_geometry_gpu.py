"""LLaMA geometries at the edges of the decode-megakernel and prefill-GEMM gates, bit for bit against the CPU oracle.

The other GPU tests use three widths (512, 4096, 5120), n_ff on the 256 grid, 1-2 layers and an odd vocabulary only on a file that never
reaches the megakernel.  The cases here (tests/test_geometry_host.py CASES, each with the gate or tier it probes) move every geometry-derived
choice of the load off those values: the megakernel's slot size, stream warps, register-resident blocks and staging tiers, CTAs that own
no row pairs, the odd last pair of the output matrix, the prefill GEMM's class-major cache at odd block counts, and the 80-layer limit of
the op table.  For each case:
1. the load takes the path the gate rules give (and the megakernel configuration, parsed from the load log);
2. prompt pieces of 1, 7, 33 and 97 rows and embedding rows on top (530 rows: two GEMM passes) == the oracle, with and without the GEMM;
3. greedy steps on the decode graph and decode_chain == the oracle == the per-op decode graph;
4. decode_batch at 3 and 17 sessions and flush_batch == each session's own run == the oracle;
5. odd vocabularies: score_tokens rows, the device sampler, state save / load and session_copy carry all n_vocab logits;
6. the zero padding row of the odd last pair (logit exactly 0) never wins, and the last real row does when it is the largest."""
import ctypes
import functools
import itertools
import os
import re
import shutil

import numpy as np
import pytest

from conftest import rel_err
from test_geometry_host import CASES, mega_plan, n_ff

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def model(tmp_path_factory, mg):
    """name -> path of the case's file, written on first use and deleted when the module is done"""
    d = tmp_path_factory.mktemp("geometry")
    made = {}

    def get(name):
        if name not in made:
            p = str(d / f"{name}.bin")
            mg.write_llama_ggjt(p, mg.LlamaSpec(**CASES[name].spec))
            made[name] = p
        return made[name]
    yield get
    for p in made.values():
        os.remove(p)


_MEGA_LOG = re.compile(r"decode megakernel \(generation 6\): (\d+) ops/token, (\d+) stream warps x 2 slots x (\d+) B, act (\d+) B, "
                       r"(\d+) B dynamic shared per CTA, register-resident blocks per lane (\d+), grid (\d+)")
_LIBC = ctypes.CDLL(None)


@functools.lru_cache(maxsize=None)
def _smem_optin() -> int:
    import torch
    return int(torch.cuda.get_device_properties(0).shared_memory_per_block_optin)


def _load(ext, monkeypatch, name, path, no_mega=False, no_gemm=False, capfd=None, seed=1337):
    """a context of the case's file (MINIGPT4_B200_NO_MEGAKERNEL / NO_PREFILL_GEMM as asked), its path asserted; with capfd also the numbers
    of the megakernel line of the load log (ops, W, slot, act, dynamic shared, register-resident blocks, grid) or None"""
    for var, on in (("MINIGPT4_B200_NO_MEGAKERNEL", no_mega), ("MINIGPT4_B200_NO_PREFILL_GEMM", no_gemm)):
        if on: monkeypatch.setenv(var, "1")
        else: monkeypatch.delenv(var, raising=False)
    if capfd is not None:
        capfd.readouterr()
    c = ext.llm_load(path, n_ctx=CASES[name].n_ctx, seed=seed, verbosity=2 if capfd is not None else 1)
    plan = None
    if capfd is not None:
        _LIBC.fflush(None)   # the C stdout buffer -> the captured file descriptor
        m = _MEGA_LOG.search(capfd.readouterr().out)
        plan = tuple(int(g) for g in m.groups()) if m else None
    monkeypatch.delenv("MINIGPT4_B200_NO_MEGAKERNEL", raising=False)
    monkeypatch.delenv("MINIGPT4_B200_NO_PREFILL_GEMM", raising=False)
    st = ext.stats(c)
    assert st.decode_megakernel == (6 if CASES[name].mega and not no_mega else 0), f"{name}: decode megakernel {st.decode_megakernel}"
    assert st.prefill_gemm == (1 if CASES[name].gemm and not no_gemm else 0), f"{name}: prefill GEMM {st.prefill_gemm}"
    return c, plan


def _free(ext, ctxs):
    for c in ctxs:
        ext.base.minigpt4_free(c)


def _ids(name, n, seed):
    """n prompt ids that end on the last token id (its row is the real half of the padded last pair when n_vocab is odd)"""
    V = CASES[name].spec["n_vocab"]
    return np.random.default_rng(seed).integers(3, V, size=n - 1).tolist() + [V - 1]


# ---- 1. the path --------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(CASES))
def test_load_takes_the_gated_path(ext, model, capfd, monkeypatch, name):
    case, s = CASES[name], CASES[name].spec
    c, plan = _load(ext, monkeypatch, name, model(name), capfd=capfd)
    st = ext.stats(c)
    assert (st.n_embd, st.n_ff, st.n_layer, st.n_vocab, st.n_ctx) == (s["n_embd"], n_ff(s), s["n_layer"], s["n_vocab"], case.n_ctx)
    want = mega_plan(s, case.n_ctx, _smem_optin(), st.sm_count)
    assert (want is not None) == case.mega
    if case.mega:
        assert plan is not None, "the megakernel took the file but logged no configuration"
        ops, W, slot, act, _, nbl, grid = plan
        assert (ops, W, slot, act, nbl) == want, (plan, want)
        assert grid == st.sm_count
        if _smem_optin() == 227 * 1024:
            assert W == case.w_h100
        print(f"{name}: {ops} ops, W {W}, slot {slot} B, act {act} B, register-resident blocks {nbl}")
    else:
        assert plan is None
    _free(ext, [c])


# ---- 2. prompt and embedding rows ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(CASES))
def test_prompt_rows_equal_oracle(ext, orc, model, monkeypatch, name):
    """pieces of 1, 7, 33 and 97 token rows (530 more on e256-q4_1: a 512-row GEMM pass and an 18-row one), then 7 embedding rows, each
    flushed on its own: logits == the oracle's on the GEMM and the per-op prefill, residual stream of the last layer == the oracle's"""
    path = model(name)
    gemm, _ = _load(ext, monkeypatch, name, path)
    per_op, _ = _load(ext, monkeypatch, name, path, no_gemm=True)
    e = orc.OracleEngine(None, path, n_ctx=CASES[name].n_ctx)
    last = CASES[name].spec["n_layer"] - 1
    lengths = [1, 7, 33, 97] + ([530] if name == "e256-q4_1" else [])
    for i, n in enumerate(lengths):
        ids = _ids(name, n, 10 + i)
        for c in (gemm, per_op):
            ext.eval_tokens(c, ids); ext.flush(c)
        hid = e.eval_tokens(ids, tap_layer=last).copy()
        want = e.logits.copy()
        assert np.array_equal(ext.logits(gemm), want), f"{n} rows, GEMM prefill: {rel_err(ext.logits(gemm), want)}"
        assert np.array_equal(ext.logits(per_op), want), f"{n} rows, per-op prefill: {rel_err(ext.logits(per_op), want)}"
        k = n - 8 * ((n - 1) // 8)   # the per-op path keeps the residual stream of its last 8-row chunk, the GEMM that of its last pass
        tail = n - 512 * ((n - 1) // 512) if CASES[name].gemm and n > 1 else k
        assert np.array_equal(ext.hidden(gemm, tail), hid[n - tail:]), f"{n} rows: residual stream"
        assert np.array_equal(ext.hidden(per_op, k), hid[n - k:]), f"{n} rows: residual stream, per-op"
    rows = np.random.default_rng(3).standard_normal((7, CASES[name].spec["n_embd"])).astype(np.float32)
    for c in (gemm, per_op):
        ext.eval_embd(c, rows); ext.flush(c)
    want = e.eval_embd(rows).copy()
    assert np.array_equal(ext.logits(gemm), want) and np.array_equal(ext.logits(per_op), want), "embedding rows"
    assert ext.n_past(gemm) == ext.n_past(per_op) == e.n_past
    _free(ext, [gemm, per_op])


# ---- 3. decode ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(CASES))
def test_decode_equals_oracle_and_per_op(ext, orc, model, monkeypatch, name):
    """a 21-token prompt, the last token id fed as one decode step (the megakernel's embed op reads the padded pair's real row), 16 greedy
    steps and 16 decode_chain steps: ids and logits == the oracle == the per-op decode graph"""
    path = model(name)
    dev, _ = _load(ext, monkeypatch, name, path)
    ref, _ = _load(ext, monkeypatch, name, path, no_mega=True)
    e = orc.OracleEngine(None, path, n_ctx=CASES[name].n_ctx)
    V = CASES[name].spec["n_vocab"]
    ids = _ids(name, 21, 1)
    for c in (dev, ref):
        ext.eval_tokens(c, ids); ext.flush(c)
    e.eval_tokens(ids)
    for c in (dev, ref):
        ext.eval_tokens(c, [V - 1])
    e.eval_tokens([V - 1])
    assert np.array_equal(ext.logits(dev), e.logits) and np.array_equal(ext.logits(ref), e.logits), "the last token id as a decode step"
    for step in range(16):
        t = int(np.argmax(e.logits))
        assert ext.greedy_id(dev) == ext.greedy_id(ref) == t, step
        for c in (dev, ref):
            ext.eval_tokens(c, [t])
        e.eval_tokens([t])
        assert np.array_equal(ext.logits(dev), e.logits), f"step {step}: {rel_err(ext.logits(dev), e.logits)}"
        assert np.array_equal(ext.logits(ref), e.logits), f"per-op graph, step {step}"
    want = [e.end_chat_greedy()[0] for _ in range(16)]
    a, b = ext.decode_chain(dev, 16)[0].tolist(), ext.decode_chain(ref, 16)[0].tolist()
    assert a == b == want
    assert np.array_equal(ext.logits(dev), e.logits) and np.array_equal(ext.logits(ref), e.logits), "after decode_chain"
    _free(ext, [dev, ref])


# ---- 4. batched paths --------------------------------------------------------------------------------------------------------------------
def _oracle_run(orc, path, name, prompt, steps):
    """the oracle's logits after the prompt and after each of `steps` greedy steps"""
    e = orc.OracleEngine(None, path, n_ctx=CASES[name].n_ctx)
    out = [e.eval_tokens(prompt).copy()]
    for _ in range(steps):
        e.end_chat_greedy(); out.append(e.logits.copy())
    return out


@pytest.mark.parametrize("name", list(CASES))
def test_batched_paths_equal_own_runs(ext, orc, model, monkeypatch, name):
    """17 sessions with queued prompts of 2..34 tokens: flush_batch, 2 decode_batch steps of all 17 (the tensor-core columns on a GEMM file),
    then 2 of the first 3 (the matvec columns), at 17 different positions; each session == the same context run on its own == the oracle"""
    path, n = model(name), 17
    lens = [2 + 2 * i for i in range(n)]
    prompts = [_ids(name, k, 200 + i) for i, k in enumerate(lens)]
    groups = []
    for _ in range(2):
        p, _ = _load(ext, monkeypatch, name, path, seed=5)
        groups.append([p] + [ext.session_create(p, seed=6 + i) for i in range(n - 1)])
    ses, own = groups
    for c, r, q in zip(ses, own, prompts):
        ext.eval_tokens(c, q); ext.eval_tokens(r, q); ext.flush(r)
    ext.flush_batch(ses)
    steps = [4 if i < 3 else 2 for i in range(n)]
    want = [_oracle_run(orc, path, name, q, k) for q, k in zip(prompts, steps)]
    got = [[ext.logits(c)] for c in ses]
    for k in range(2):
        ids = ext.decode_batch(ses).tolist()
        for i, c in enumerate(ses):
            assert ids[i] == int(np.argmax(want[i][k + 1])), f"17 sessions, step {k}, session {i}"
            got[i].append(ext.logits(c))
    for k in range(2):
        ids = ext.decode_batch(ses[:3]).tolist()
        for i in range(3):
            assert ids[i] == int(np.argmax(want[i][k + 3])), f"3 sessions, step {k}, session {i}"
            got[i].append(ext.logits(ses[i]))
    for i, r in enumerate(own):
        mine = [ext.logits(r)]
        for _ in range(steps[i]):
            ext.eval_tokens(r, [ext.greedy_id(r)]); mine.append(ext.logits(r))
        for k in range(steps[i] + 1):
            assert np.array_equal(got[i][k], mine[k]), f"session {i}, {'flush_batch' if k == 0 else f'decode_batch step {k}'} != own run"
            assert np.array_equal(got[i][k], want[i][k]), f"session {i}, {'flush_batch' if k == 0 else f'decode_batch step {k}'} != oracle"
        assert ext.n_past(ses[i]) == ext.n_past(r) == lens[i] + steps[i]
    _free(ext, ses + own)


# ---- 5. odd vocabularies downstream ---------------------------------------------------------------------------------------------------------
ODD = ["e256-q4_1", "e1280", "7b-32001-q4_1"]


def _same_up_to_ties(got, want, logits, what):
    """the rule of test_sample_gpu.py: draw for draw the same id, or another id of equal logit"""
    for i, (g, w) in enumerate(zip(got.tolist(), want.tolist())):
        assert g == w or logits[g] == logits[w], f"draw {i}: {g} != {w}, {what}"


@pytest.mark.parametrize("name", ODD)
def test_odd_vocabulary_downstream(ext, model, monkeypatch, name):
    path = model(name)
    V = CASES[name].spec["n_vocab"]
    assert V % 2
    p, _ = _load(ext, monkeypatch, name, path, seed=9)
    ses = [p] + [ext.session_create(p, seed=10 + i) for i in range(4)]
    single, _ = _load(ext, monkeypatch, name, path)
    prompt = _ids(name, 9, 42)
    for c in ses + [single]:
        ext.eval_tokens(c, prompt); ext.flush(c)
    # score_tokens rows (stride n_vocab, odd) == the logits of one context evaluating the same ids one at a time
    lists = [[V - 1, 5, V - 2], [7, V - 1]]
    scored = ext.score_tokens(ses[:2], lists, logits=True)
    for i, ids in enumerate(lists):
        rows = scored[i][2]
        assert rows.shape == (len(ids), V)
        r, _ = _load(ext, monkeypatch, name, path)
        ext.eval_tokens(r, prompt); ext.flush(r)
        for j, t in enumerate(ids):
            ext.eval_tokens(r, [t])
            assert np.array_equal(rows[j], ext.logits(r)), f"score_tokens: list {i}, row {j}"
        _free(ext, [r])
    # the device sampler over all n_vocab logits (the model's own and a synthetic sweep) == the host sampler
    model_logits = ext.logits(single)
    synth = (np.random.default_rng(V).standard_normal(V) * 3.0).astype(np.float32)
    for logits in (model_logits, synth):
        for top_k, temp, top_p, seed in itertools.product((0, 1, 40), (0.1, 0.8, 1.5), (1.0, 0.9), (1, 4242)):
            kw = dict(temp=temp, top_k=top_k, top_p=top_p)
            got, want = ext.op_sample(logits, seed, 16, **kw), ext.host_sample(logits, seed, 16, **kw)
            assert got.max() < V
            _same_up_to_ties(got, want, logits, kw | dict(seed=seed))
    # state save / load and session_copy carry all n_vocab logits and the greedy id
    blob = ext.state_save(single)
    ext.state_load(ses[2], blob)
    ext.session_copy(ses[0], ses[3:5])   # (ses[0] holds the same prompt: score_tokens without keep left it as it was)
    for c in ses[2:5]:
        assert np.array_equal(ext.logits(c), model_logits) and ext.n_past(c) == ext.n_past(single)
        assert ext.greedy_id(c) == ext.greedy_id(single)
    ext.eval_tokens(single, [V - 1])
    for c in ses[2:5]:
        ext.eval_tokens(c, [V - 1])
        assert np.array_equal(ext.logits(c), ext.logits(single))
    _free(ext, ses + [single])


# ---- 6. the padding row --------------------------------------------------------------------------------------------------------------------
PAD = ["e256-q4_1", "e1280"]




# ---- 6. the padding row --------------------------------------------------------------------------------------------------------------------
PAD = ["e256-q4_1", "e1280"]


def _tensor_at(path, want: str) -> tuple[int, int, int]:
    """(byte offset of the data, rows, bytes per row) of one tensor of a ggjt file"""
    import struct
    with open(path, "rb") as f:
        b = f.read()
    n_vocab = struct.unpack_from("<I", b, 8)[0]
    pos = 8 + 28
    for _ in range(n_vocab):
        pos += 4 + struct.unpack_from("<I", b, pos)[0] + 4
    while pos < len(b):
        nd, nl, gt = struct.unpack_from("<III", b, pos); pos += 12
        ne = struct.unpack_from(f"<{nd}I", b, pos); pos += 4 * nd
        nm = b[pos:pos + nl].decode(); pos += nl
        pos = (pos + 31) & ~31
        rb = {3: ne[0] // 32 * 20, 2: ne[0] // 32 * 18, 0: ne[0] * 4}[gt]
        if nm == want:
            return pos, ne[1], rb
        pos += rb * (ne[1] if nd > 1 else 1)
    raise KeyError(want)


def _patch_output(src, dst, m):
    """a copy of src whose Q4_1 output row r has d = 0 and min m[r] in every block: its logit is m[r] times the sum of the staged Q8_1
    block sums of the final normed hidden state, whatever the nibbles hold"""
    shutil.copyfile(src, dst)
    off, rows, rb = _tensor_at(dst, "output.weight")
    assert rows == len(m)
    w = np.memmap(dst, dtype=np.uint8, mode="r+", offset=off, shape=(rows, rb // 20, 20))
    w[:, :, 0:2] = np.zeros(1, np.float16).view(np.uint8)
    w[:, :, 2:4] = np.asarray(m, np.float16).view(np.uint8).reshape(rows, 1, 2)
    w.flush()
    del w


@pytest.mark.parametrize("name", PAD)
def test_padding_row_never_wins(ext, orc, model, monkeypatch, tmp_path, name):
    """The output matrix of an odd vocabulary is padded with a zero row, whose logit is exactly 0.  Two patched files:
    - every real logit negative (d = 0, the min's sign against the hidden state's sum): the arg-max is a real row, on the decode graph
      (megakernel), the per-op graph, flush_batch / decode_batch, score_tokens rows and top_k 1 sampling;
    - row n_vocab - 1 (the real half of the last pair) the only positive logit: it wins on all of them.
    The output matrix does not change the hidden state, so the oracle's state before the patch gives the signs."""
    path = model(name)
    s = CASES[name].spec
    V, last = s["n_vocab"], s["n_layer"] - 1
    from oracle import oracle
    _, _, t = oracle.read_ggjt(path)
    nw = np.asarray(t["norm.weight"].data).view(np.float32).copy()
    for seed in range(256):   # a prompt whose normed hidden states, after it and after one more V - 1, have sums of one sign
        prompt = _ids(name, 13, 500 + seed)
        e = orc.OracleEngine(None, path, n_ctx=CASES[name].n_ctx)
        h = [orc.rms_norm_mul(e.eval_tokens(prompt, tap_layer=last)[-1:], nw)[0], orc.rms_norm_mul(e.eval_tokens([V - 1], tap_layer=last), nw)[0]]
        sums = [float(np.sum(x, dtype=np.float64)) for x in h]
        if np.sign(sums[0]) == np.sign(sums[1]) and min(abs(a) / np.abs(x).sum() for a, x in zip(sums, h)) > 0.02:
            break
    else:
        pytest.fail("no prompt with hidden-state sums of one sign")
    sgn = float(np.sign(sums[0]))
    mag = 0.02 + 0.03 * np.random.default_rng(V).random(V)
    star = V // 3
    neg = -sgn * mag; neg[star] = -sgn * 0.01         # every logit negative, row `star` the largest
    pos = -sgn * mag; pos[V - 1] = sgn * 0.02         # row V - 1 the only positive logit
    for tag, m, top in (("all negative", neg, star), ("last row largest", pos, V - 1)):
        f = str(tmp_path / f"{name}-{tag.replace(' ', '-')}.bin")
        _patch_output(path, f, m)
        e = orc.OracleEngine(None, f, n_ctx=CASES[name].n_ctx)
        want = [e.eval_tokens(prompt).copy(), e.eval_tokens([V - 1]).copy(), e.eval_tokens([V - 1]).copy()]
        assert int(np.argmax(want[0])) == top and want[0].shape == (V,)
        if top == star:
            assert want[0].max() < 0 and want[1].max() < 0, "the patch must leave every real logit negative"
        else:
            assert int(np.argmax(want[1])) == V - 1 and want[1][V - 1] > 0
        for no_mega in (False, True):   # the decode graph: megakernel (if the case has it) and per-op
            c, _ = _load(ext, monkeypatch, name, f, no_mega=no_mega)
            ext.eval_tokens(c, prompt); ext.flush(c)
            assert np.array_equal(ext.logits(c), want[0]) and ext.greedy_id(c) == top, (tag, no_mega)
            ext.eval_tokens(c, [V - 1])
            assert np.array_equal(ext.logits(c), want[1]), (tag, no_mega)
            assert ext.greedy_id(c) == int(np.argmax(want[1])) < V, (tag, no_mega)
            _free(ext, [c])
        p, _ = _load(ext, monkeypatch, name, f, seed=3)
        ses = [p] + [ext.session_create(p, seed=4 + i) for i in range(5)]
        for c in ses:
            ext.eval_tokens(c, prompt)
        ext.flush_batch(ses[:3])
        for c in ses[:3]:
            assert np.array_equal(ext.logits(c), want[0]) and ext.greedy_id(c) == top, (tag, "flush_batch")
        got = ext.decode_batch(ses[:3], [V - 1] * 3).tolist()
        assert got == [int(np.argmax(want[1]))] * 3, (tag, "decode_batch")
        for c in ses[:3]:
            assert np.array_equal(ext.logits(c), want[1]), (tag, "decode_batch")
        for c in ses[3:]:
            ext.flush(c)
        scored = ext.score_tokens(ses[3:5], [[V - 1, V - 1], [V - 1]], logits=True)
        for rows in (scored[0][2], scored[1][2]):
            for j in range(len(rows)):
                assert np.array_equal(rows[j], want[j + 1]), (tag, "score_tokens", j)
        ids, _ = ext.sample_steps([ses[5]], 2, temp=0.8, top_k=1, top_p=1.0)
        assert ids[0, 0] == top and ids[1, 0] < V, (tag, "top_k 1 sampling", ids.tolist())
        if top == V - 1:
            assert ids[1, 0] == V - 1
        _free(ext, ses)
