"""Python driver of the CPU oracle (TEST INFRASTRUCTURE — see oracle.cpp header; parity unpinned).

Holds the parts of the reference path that are host logic rather than arithmetic, restated
independently of the product's C++ implementation so they can check it:
  * file readers for the MiniGPT-4 container (reference minigpt4.cpp:1478-1596) and ggjt v3
    (llama.cpp@master-31cfbb1 llama_file_loader, SURVEY §B.2) — numpy memmaps, zero copy into the C oracle
  * llama.cpp's SentencePiece-style tokenizer (llama_tokenizer @ that tag: score-driven bigram merges over
    UTF-8 characters, byte fallback id = byte + 3; SURVEY §A.3)
  * the chat flow of the C API shims (minigpt4.cpp:2671-2753) incl. the BOS-per-add_strings quirk
  * greedy sampling = first arg-max (llama_sample_token_greedy)
Only tests/, __graft_entry__.smoke() and bench.py's CPU legs may import this module.
"""
from __future__ import annotations

import ctypes
import heapq
import json
import os
import struct
import subprocess
from pathlib import Path

import numpy as np

_HERE = Path(__file__).resolve().parent
_LIB = None

SYSTEM_PROMPT = ("Give the following image: <Img>ImageContent</Img>. You will be able to see the image once I provide it to you. "
                 "Please answer my questions.###")  # reference minigpt4.cpp:139

GG_BLOCK = {0: (1, 4), 1: (1, 2), 2: (32, 18), 3: (32, 20), 6: (32, 22), 7: (32, 24), 8: (32, 34), 12: (256, 144), 13: (256, 176), 14: (256, 210)}
# MiniGPT4DataType -> ggml type (reference minigpt4.cpp:555-739)
MG4_TO_GG = {0: 1, 1: 0, 4: 2, 5: 3, 6: 6, 7: 7, 8: 8, 12: 12, 13: 13, 14: 14}


def usable_cpus() -> int:
    """CPUs this process may actually use: the affinity mask capped by the cgroup CPU quota.  A GPU box shows 128 logical CPUs to a
    container that is throttled to 16; an OpenMP team of 128 spinning threads on a 16-CPU quota is 10-30x slower than a team of 16
    (this, not the arithmetic, made the GPU parity suite take 8 minutes)."""
    n = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 1)
    try:
        q, per = Path("/sys/fs/cgroup/cpu.max").read_text().split()
        if q != "max":
            n = max(1, min(n, int(int(q) / int(per))))
    except Exception:
        pass
    return n


def build(force: bool = False) -> Path:
    so = _HERE / "liboracle.so"
    src = _HERE / "oracle.cpp"
    if force or not so.exists() or so.stat().st_mtime < src.stat().st_mtime:
        subprocess.run(["make", "-C", str(_HERE), "-s"], check=True)
    return so


def lib() -> ctypes.CDLL:
    global _LIB
    if _LIB is None:
        L = ctypes.CDLL(str(build()))
        vp, i32, i64, fp = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64, ctypes.c_void_p
        L.oracle_model_new.restype = vp
        L.oracle_model_free.argtypes = [vp]
        L.oracle_model_add.argtypes = [vp, ctypes.c_char_p, i32, i32, ctypes.POINTER(i64), vp]
        L.oracle_vit_encode.argtypes = [vp, fp, fp, i32, i32, i32, fp]
        L.oracle_vit_encode_stages.argtypes = [vp, fp, fp, i32, fp, fp, fp, fp]
        L.oracle_llama_new.argtypes = [vp, i32]
        L.oracle_llama_new.restype = vp
        L.oracle_llama_free.argtypes = [vp]
        L.oracle_llama_eval.argtypes = [vp, vp, vp, i32, i32, i32, vp, vp, i32]
        L.oracle_llama_attention.argtypes = [vp, vp, vp, i32, i32, i32, vp, i32, vp]
        L.oracle_llama_n_vocab.argtypes = [vp]
        L.oracle_llama_n_embd.argtypes = [vp]
        L.oracle_mul_mat.argtypes = [i32, i64, i64, vp, vp, i32, vp]
        L.oracle_dequant_row.argtypes = [i32, i64, vp, vp]
        for n in ("oracle_quantize_q8_0", "oracle_quantize_q8_1", "oracle_quantize_q8_K"):
            getattr(L, n).argtypes = [vp, vp, i32]
        L.oracle_layernorm.argtypes = [vp, vp, i32, i32, vp, vp]
        L.oracle_rms_norm_mul.argtypes = [vp, vp, i32, i32, vp]
        L.oracle_softmax.argtypes = [vp, i32, i32]
        L.oracle_gelu.argtypes = [vp, vp, i32]
        L.oracle_silu.argtypes = [vp, vp, i32]
        L.oracle_table.argtypes = [i32]
        L.oracle_host_read_gbs.argtypes = [i64, i32, i32]; L.oracle_host_read_gbs.restype = ctypes.c_double
        L.oracle_table.restype = ctypes.POINTER(ctypes.c_uint16)
        L.oracle_init()
        L.oracle_set_num_threads(usable_cpus())  # default team for the single-op entry points (mul_mat, ...)
        _LIB = L
    return _LIB


def _p(a: np.ndarray):
    return a.ctypes.data_as(ctypes.c_void_p)


# ------------------------------------------------------------------------------------------------
# file readers
# ------------------------------------------------------------------------------------------------
class TensorView:
    __slots__ = ("name", "gtype", "ne", "data")

    def __init__(self, name, gtype, ne, data):
        self.name, self.gtype, self.ne, self.data = name, gtype, list(ne), data

    def nbytes(self):
        per, nb = GG_BLOCK[self.gtype]
        n = 1
        for d in self.ne:
            n *= d
        return n // per * nb


def read_minigpt4(path) -> tuple[dict, dict[str, TensorView]]:
    """-> (config, {"<model>.<tensor>": view}); views alias a read-only memmap."""
    mm = np.memmap(path, dtype=np.uint8, mode="r")
    pos = 0

    def s4():
        nonlocal pos
        v = struct.unpack_from("<i", mm, pos)[0]
        pos += 4
        return v

    def rstr():
        nonlocal pos
        n = s4()
        b = bytes(mm[pos:pos + n])
        pos += n
        return b.decode()

    if bytes(mm[0:4]) != b"ggml":
        raise ValueError("LoadModelFileHeader")
    pos = 4
    if s4() == 0:
        raise ValueError("LoadModelFileVersion")
    s4()  # file dtype
    config = json.loads(rstr())
    out: dict[str, TensorView] = {}
    while pos < mm.size:
        mname = rstr()
        n = s4()
        metas = []
        for _ in range(n):
            tname = rstr()
            nd = s4()
            ne = [s4() for _ in range(nd)]
            metas.append((tname, ne, MG4_TO_GG[s4()]))
        for tname, ne, gt in metas:
            if pos % 4096:
                pos = (pos + 4096) & ~4095
            tv = TensorView(f"{mname}.{tname}", gt, ne, None)
            nb = tv.nbytes()
            tv.data = mm[pos:pos + nb]
            pos += nb
            out[tv.name] = tv
    return config, out


def read_ggjt(path):
    """-> (hparams dict, vocab [(bytes, score)], {name: view})"""
    mm = np.memmap(path, dtype=np.uint8, mode="r")
    magic, ver = struct.unpack_from("<II", mm, 0)
    if magic != 0x67676A74 or ver != 3:
        raise ValueError("not ggjt v3")
    keys = ("n_vocab", "n_embd", "n_mult", "n_head", "n_layer", "n_rot", "ftype")
    hp = dict(zip(keys, struct.unpack_from("<7I", mm, 8)))
    pos = 8 + 28
    vocab = []
    for _ in range(hp["n_vocab"]):
        ln = struct.unpack_from("<I", mm, pos)[0]
        pos += 4
        text = bytes(mm[pos:pos + ln])
        pos += ln
        score = struct.unpack_from("<f", mm, pos)[0]
        pos += 4
        vocab.append((text, score))
    tensors: dict[str, TensorView] = {}
    while pos < mm.size:
        nd, nl, gt = struct.unpack_from("<III", mm, pos)
        pos += 12
        ne = list(struct.unpack_from(f"<{nd}I", mm, pos))
        pos += 4 * nd
        name = bytes(mm[pos:pos + nl]).decode()
        pos += nl
        pos = (pos + 31) & ~31
        tv = TensorView(name, gt, ne, None)
        nb = tv.nbytes()
        tv.data = mm[pos:pos + nb]
        pos += nb
        tensors[name] = tv
    return hp, vocab, tensors


class OracleModel:
    """name->tensor table living in the C oracle; keeps the memmaps alive."""

    def __init__(self, tensors: dict[str, TensorView]):
        self._keep = tensors
        self.h = lib().oracle_model_new()
        for name, tv in tensors.items():
            ne = (ctypes.c_int64 * 4)(*(tv.ne + [1] * (4 - len(tv.ne))))
            lib().oracle_model_add(self.h, name.encode(), tv.gtype, len(tv.ne), ne, ctypes.c_void_p(tv.data.ctypes.data))

    def __del__(self):
        try:
            lib().oracle_model_free(self.h)
        except Exception:
            pass


# ------------------------------------------------------------------------------------------------
# tokenizer (llama.cpp llama_tokenizer @ master-31cfbb1)
# ------------------------------------------------------------------------------------------------
class Tokenizer:
    def __init__(self, vocab):
        self.vocab = vocab
        self.tok2id: dict[bytes, int] = {}
        for i, (t, _) in enumerate(vocab):
            self.tok2id[t] = i  # later ids overwrite earlier ones, like the std::unordered_map assignment loop

    @staticmethod
    def _utf8_len(b: int) -> int:
        return (1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 2, 2, 3, 4)[b >> 4]

    def tokenize(self, text: bytes | str, bos: bool = True) -> list[int]:
        if isinstance(text, str):
            text = text.encode()
        if not text:
            return []  # llama_tokenize: empty text -> no tokens, not even BOS
        out = [1] if bos else []
        # symbols = utf-8 characters, doubly linked
        syms = []  # [start, length, prev, next]
        i = 0
        while i < len(text):
            n = min(self._utf8_len(text[i]), len(text) - i)
            syms.append([i, n, len(syms) - 1, len(syms) + 1])
            i += n
        syms[-1][3] = -1
        heap = []  # (-score, left_index, right_index, size) ; ties -> lower left index first

        def try_add(l, r):
            if l == -1 or r == -1:
                return
            piece = text[syms[l][0]:syms[l][0] + syms[l][1] + syms[r][1]]
            tid = self.tok2id.get(piece)
            if tid is None:
                return
            heapq.heappush(heap, (-self.vocab[tid][1], l, r, len(piece)))

        for k in range(1, len(syms)):
            try_add(k - 1, k)
        while heap:
            _, l, r, size = heapq.heappop(heap)
            L, R = syms[l], syms[r]
            if L[1] == 0 or R[1] == 0 or L[1] + R[1] != size:
                continue
            L[1] += R[1]
            R[1] = 0
            L[3] = R[3]
            if R[3] >= 0:
                syms[R[3]][2] = l
            try_add(L[2], l)
            try_add(l, L[3])
        k = 0
        while k != -1:
            st, n = syms[k][0], syms[k][1]
            piece = text[st:st + n]
            tid = self.tok2id.get(piece)
            if tid is None:
                out.extend(b + 3 for b in piece)
            else:
                out.append(tid)
            k = syms[k][3]
        return out

    def id_to_token(self, tid: int) -> bytes:
        return b"</s>" if tid == 2 else self.vocab[tid][0]  # minigpt4.cpp:2485-2497


# ------------------------------------------------------------------------------------------------
# engine mirror: MiniGPT4 class flow (minigpt4.cpp:1740-2522 + shims :2653-2753)
# ------------------------------------------------------------------------------------------------
class OracleEngine:
    def __init__(self, minigpt4_path=None, llama_path=None, n_ctx: int = 2048, n_batch: int = 512, n_threads: int = 0):
        self.n_threads = n_threads or usable_cpus()
        self.n_batch = n_batch
        self.n_past = 0
        self.vis = None
        self.llm = None
        if minigpt4_path is not None:
            self.config, vt = read_minigpt4(minigpt4_path)
            self._vis_names = set(vt)
            self.vis_d = vt["visual_encoder.pos_embed"].ne[0]
            self.vis = OracleModel(vt)
            self.n_embd_llm = vt["llama_proj.weight"].ne[1]
        if llama_path is not None:
            self.hp, vocab, lt = read_ggjt(llama_path)
            self.tok = Tokenizer(vocab)
            self.llm_model = OracleModel(lt)
            self.llm = lib().oracle_llama_new(self.llm_model.h, n_ctx)
            self.n_vocab = lib().oracle_llama_n_vocab(self.llm)
            self.n_embd = lib().oracle_llama_n_embd(self.llm)
            self.logits = np.zeros(self.n_vocab, np.float32)

    # -- vision ---------------------------------------------------------------------------
    def encode_image(self, image: np.ndarray, tap_kind: int = 0, tap_idx: int = 0) -> np.ndarray:
        image = np.ascontiguousarray(image, np.float32).reshape(3, 224, 224)
        out = np.zeros((32, self.n_embd_llm), np.float32)
        tap = None
        if tap_kind:
            tap = np.zeros((257, 1408), np.float32) if tap_kind in (1, 2, 3) else np.zeros((32, 768), np.float32)
        lib().oracle_vit_encode(self.vis.h, _p(image), _p(out), self.n_threads, tap_kind, tap_idx, _p(tap) if tap is not None else None)
        return tap if tap_kind else out

    def encode_image_stages(self, image: np.ndarray) -> dict:
        """every stage of one encode_image run: embed [257, D] (patches + CLS + positions), vit_blocks [n_blocks, 257, D] (residual stream
        after each block), ln_vision [257, D], qformer [q_layers, 32, 768] (hidden states after each layer) and out [32, n_embd_llm]"""
        image = np.ascontiguousarray(image, np.float32).reshape(3, 224, 224)
        D = self.vis_d
        nb = self._count("visual_encoder.blocks.{}.norm1.weight")
        nl = self._count("Qformer.bert.encoder.layer.{}.attention.self.query.weight")
        r = {"embed": np.zeros((257, D), np.float32), "vit_blocks": np.zeros((nb, 257, D), np.float32), "ln_vision": np.zeros((257, D), np.float32),
             "qformer": np.zeros((nl, 32, 768), np.float32), "out": np.zeros((32, self.n_embd_llm), np.float32)}
        lib().oracle_vit_encode_stages(self.vis.h, _p(image), _p(r["out"]), self.n_threads, _p(r["embed"]), _p(r["vit_blocks"]), _p(r["ln_vision"]),
                                       _p(r["qformer"]))
        return r

    def _count(self, pattern: str) -> int:
        n = 0
        while pattern.format(n) in self._vis_names:
            n += 1
        return n

    # -- language -------------------------------------------------------------------------
    def eval_tokens(self, ids, tap_layer: int = -1):
        ids = np.ascontiguousarray(ids, np.int32)
        tap = np.zeros((len(ids), self.n_embd), np.float32) if tap_layer >= 0 else None
        for i in range(0, len(ids), self.n_batch):  # add_tokens chunking minigpt4.cpp:2369-2379
            chunk = ids[i:i + self.n_batch]
            rc = lib().oracle_llama_eval(self.llm, _p(chunk), None, len(chunk), self.n_past, self.n_threads, _p(self.logits),
                                         _p(tap) if tap is not None else None, tap_layer)
            if rc:
                raise RuntimeError("FailedToAddString")
            self.n_past += len(chunk)
        return tap if tap is not None else self.logits

    def eval_embd(self, embd: np.ndarray):
        embd = np.ascontiguousarray(embd, np.float32).reshape(-1, self.n_embd)
        rc = lib().oracle_llama_eval(self.llm, None, _p(embd), embd.shape[0], self.n_past, self.n_threads, _p(self.logits), None, -1)
        if rc:
            raise RuntimeError("FailedToAddEmbedding")
        self.n_past += embd.shape[0]
        return self.logits

    def add_strings(self, s):
        self.eval_tokens(self.tok.tokenize(s, bos=True))  # add_bos=true ALWAYS (minigpt4.cpp:2387)

    def system_prompt(self):
        self.add_strings(SYSTEM_PROMPT)

    def begin_chat_image(self, emb: np.ndarray, s):
        self.add_strings("Human: <Img>")
        self.eval_embd(emb)
        self.add_strings("</Img> ")
        self.add_strings(s)
        self.add_strings("### Assistant:")

    def begin_chat(self, s):
        self.add_strings("Human: ")
        self.add_strings(s)
        self.add_strings("### Assistant:")

    def end_chat_greedy(self) -> tuple[int, bytes]:
        tid = int(np.argmax(self.logits))  # first max, like llama_sample_token_greedy
        self.eval_tokens([tid])
        return tid, self.tok.id_to_token(tid)

    def reset_chat(self):
        self.n_past = 0


# single-op helpers for kernel-level parity tests ----------------------------------------------------
def mul_mat(gtype: int, w_raw: np.ndarray, rows: int, cols: int, x: np.ndarray) -> np.ndarray:
    x = np.ascontiguousarray(x, np.float32).reshape(-1, cols)
    y = np.zeros((x.shape[0], rows), np.float32)
    w_raw = np.ascontiguousarray(w_raw)
    lib().oracle_mul_mat(gtype, rows, cols, _p(w_raw), _p(x), x.shape[0], _p(y))
    return y


def llama_attention(q: np.ndarray, k: np.ndarray, v: np.ndarray, pos) -> np.ndarray:
    """the language graph's attention op: q float32 [rows][n_head * 128], k / v float16 [n_ctx][n_head * 128]; row t sees keys 0 .. pos[t]"""
    q = np.ascontiguousarray(q, np.float32)
    k = np.ascontiguousarray(k, np.float16); v = np.ascontiguousarray(v, np.float16)
    pos = np.ascontiguousarray(pos, np.int32).reshape(-1)
    assert k.shape == v.shape and q.shape == (pos.size, k.shape[1]) and k.shape[1] % 128 == 0
    out = np.zeros_like(q)
    if lib().oracle_llama_attention(_p(q), _p(k), _p(v), k.shape[1] // 128, k.shape[0], pos.size, _p(pos), usable_cpus(), _p(out)):
        raise ValueError("a position lies outside the cache")
    return out


def dequant_rows(gtype: int, w_raw: np.ndarray, rows: int, cols: int) -> np.ndarray:
    w_raw = np.ascontiguousarray(w_raw).reshape(rows, -1)
    y = np.zeros((rows, cols), np.float32)
    for r in range(rows):
        lib().oracle_dequant_row(gtype, cols, ctypes.c_void_p(w_raw[r].ctypes.data), ctypes.c_void_p(y[r].ctypes.data))
    return y


def layernorm(x, w, b):
    x = np.ascontiguousarray(x, np.float32)
    y = np.empty_like(x)
    lib().oracle_layernorm(_p(x), _p(y), x.shape[-1], x.size // x.shape[-1], _p(np.ascontiguousarray(w, np.float32)), _p(np.ascontiguousarray(b, np.float32)))
    return y


def rms_norm_mul(x, w):
    x = np.ascontiguousarray(x, np.float32)
    y = np.empty_like(x)
    lib().oracle_rms_norm_mul(_p(x), _p(y), x.shape[-1], x.size // x.shape[-1], _p(np.ascontiguousarray(w, np.float32)))
    return y


def softmax(x):
    y = np.array(x, np.float32, copy=True)
    lib().oracle_softmax(_p(y), y.shape[-1], y.size // y.shape[-1])
    return y


def gelu(x):
    x = np.ascontiguousarray(x, np.float32)
    y = np.empty_like(x)
    lib().oracle_gelu(_p(x), _p(y), x.size)
    return y


def silu(x):
    x = np.ascontiguousarray(x, np.float32)
    y = np.empty_like(x)
    lib().oracle_silu(_p(x), _p(y), x.size)
    return y


def table(which: int) -> np.ndarray:
    return np.ctypeslib.as_array(lib().oracle_table(which), shape=(65536,)).copy()
