"""Perplexity of a text under a LLaMA file, through the C ABI (minigpt4_b200_score_tokens), computed the way llama.cpp's perplexity tool
computes it: the text is tokenised with BOS and split into chunks of n_ctx tokens, each chunk starts a fresh conversation with BOS in its
first position, and the mean negative log-likelihood runs over the second half of every chunk (the tokens that see at least n_ctx / 2
tokens of context).  One session per chunk, up to 64 chunks per score_tokens call; the sessions are left as they were (keep = 0) and take
the next chunks.

    python tools/perplexity.py --model llama.bin --text wiki.test.raw [--n-ctx 512]

Prints one JSON line: perplexity, chunks, scored tokens, wall seconds.  On the synthetic models of the tests the value means nothing."""
import argparse
import json
import math
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

MAX_BATCH = 64   # contexts per score_tokens call (LlamaDevice::kMaxBatch)


def chunks(tokens: list[int], n_ctx: int, bos: int = 1) -> list[list[int]]:
    """the text's full n_ctx-token chunks, each with BOS in its first position"""
    out = []
    for i in range(len(tokens) // n_ctx):
        c = list(tokens[i * n_ctx:(i + 1) * n_ctx])
        c[0] = bos
        out.append(c)
    return out


def scored_entries(n_ctx: int) -> slice:
    """the entries of a chunk that count: llama.cpp's rows first .. n_ctx - 2 (first = n_ctx / 2) predict tokens first + 1 .. n_ctx - 1"""
    return slice(n_ctx // 2 + 1, n_ctx)


def chunk_logprobs(ext, parent, cks: list[list[int]]) -> list[np.ndarray]:
    """every chunk's per-token log-probabilities (entry 0 is NaN: a chunk starts a conversation)"""
    ses = [parent] + [ext.session_create(parent) for _ in range(min(len(cks), MAX_BATCH) - 1)]
    try:
        out = []
        for b in range(0, len(cks), MAX_BATCH):
            part = cks[b:b + MAX_BATCH]
            out += [lp for lp, _ in ext.score_tokens(ses[:len(part)], part, keep=False)]
        return out
    finally:
        for c in ses[1:]:
            ext.base.minigpt4_free(c)


def perplexity(ext, parent, tokens: list[int], n_ctx: int) -> tuple[float, int, int]:
    """(perplexity, chunks, scored tokens) of `tokens` in chunks of n_ctx; `parent` is a context of n_ctx >= n_ctx at n_past 0"""
    cks = chunks(tokens, n_ctx)
    if not cks:
        raise ValueError(f"{len(tokens)} tokens: fewer than one chunk of {n_ctx}")
    sel = scored_entries(n_ctx)
    nll, count = 0.0, 0
    for lp in chunk_logprobs(ext, parent, cks):
        v = lp[sel].astype(np.float64)
        nll -= float(v.sum()); count += v.size
    return math.exp(nll / count), len(cks), count


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--model", required=True, help="LLaMA ggjt file")
    ap.add_argument("--text", required=True, help="text file (UTF-8)")
    ap.add_argument("--n-ctx", type=int, default=512)
    a = ap.parse_args()
    import minigpt4_cpp_b200 as m
    ext = m.B200(m.load_library())
    if ext.L.minigpt4_b200_device_count() < 1:
        sys.exit("perplexity.py needs a CUDA device: the engine has no CPU path")
    parent = ext.llm_load(a.model, n_ctx=a.n_ctx, verbosity=0)
    tokens = ext.tokenize(parent, Path(a.text).read_bytes(), add_bos=True)
    t0 = time.perf_counter()
    ppl, n_chunks, n_tok = perplexity(ext, parent, tokens, a.n_ctx)
    print(json.dumps({"perplexity": ppl, "chunks": n_chunks, "scored_tokens": n_tok, "n_ctx": a.n_ctx, "seconds": round(time.perf_counter() - t0, 3)}))
    ext.base.minigpt4_free(parent)


if __name__ == "__main__":
    main()
