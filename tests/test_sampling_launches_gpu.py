"""Kernel launches of the device-driven step loops, as kernel_launches counts them on the first context of a call:

- sample_steps: every step is one sampling launch and the decode step (the context's own graph at B = 1, the batch graph at B >= 2);
- beam search: every step is rank, merge and (2 or more beams) the K / V reorder, then the decode step; 2 or more beams also copy the
  conversation into the other slots first and evaluate the best reply again afterwards.

Each decode step's share is measured on its own on twin contexts: decode_chain of one step, decode_batch of one step, the prompt pass of
the best reply."""
import pytest

pytestmark = pytest.mark.gpu

PROMPT = [1, 15, 27, 300, 41, 9, 77]
STEPS = 8   # two chunks of kReplyChunk steps: beam search issues all of them before it first reads its done flag


def launches(ext, c) -> int:
    return ext.stats(c).kernel_launches


def group(ext, path, n, evaluated):
    """n contexts of one group; the first `evaluated` of them have evaluated PROMPT"""
    c = ext.llm_load(path, n_ctx=256)
    ctxs = [c] + [ext.session_create(c, seed=7 + i) for i in range(n - 1)]
    for x in ctxs[:evaluated]:
        ext.eval_tokens(x, PROMPT)
        ext.flush(x)
    return ctxs


def free(ext, ctxs):
    for c in ctxs:
        ext.base.minigpt4_free(c)


def delta(ext, c, fn) -> int:
    before = launches(ext, c)
    fn()
    return launches(ext, c) - before


@pytest.mark.parametrize("B", [1, 9])
@pytest.mark.parametrize("mirostat", [0, 2], ids=["chain", "mirostat2"])
def test_sample_steps(ext, tiny, B, mirostat):
    ctxs = group(ext, tiny["q4_1"], B, B)
    decode = delta(ext, ctxs[0], (lambda: ext.decode_chain(ctxs[0], 1)) if B == 1 else (lambda: ext.decode_batch(ctxs)))
    assert decode > 0
    got = delta(ext, ctxs[0], lambda: ext.sample_steps(ctxs, STEPS, mirostat=mirostat))
    assert got == STEPS * (decode + 1), (B, decode)
    free(ext, ctxs)


@pytest.mark.parametrize("n_beams", [1, 2])
def test_beam_search(ext, tiny, n_beams):
    path = tiny["q4_1"]
    twins = group(ext, path, n_beams, n_beams)
    decode = delta(ext, twins[0], (lambda: ext.decode_chain(twins[0], 1)) if n_beams == 1 else (lambda: ext.decode_batch(twins)))
    ctxs = group(ext, path, n_beams, 1)
    hyps = []
    got = delta(ext, ctxs[0], lambda: hyps.append(ext.beam_search(ctxs, STEPS, b"")[0]))
    if n_beams == 1:
        assert got == STEPS * (2 + decode)
    else:
        best = hyps[0][0][0]
        assert len(best) == STEPS   # (no stop text: every hypothesis runs to max_steps)
        twin = group(ext, path, 1, 1)[0]
        ext.eval_tokens(twin, best)
        again = delta(ext, twin, lambda: ext.flush(twin))
        assert got == 1 + STEPS * (3 + decode) + again, (decode, again)
        free(ext, [twin])
    free(ext, twins + ctxs)
