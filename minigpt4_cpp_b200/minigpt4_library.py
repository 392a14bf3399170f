"""Host-side Python mirror of the reference binding (reference minigpt4/minigpt4_library.py:74-689).

Same class names, method names, argument meaning and error behaviour as the reference's
``MiniGPT4SharedLibrary`` / ``MiniGPT4ChatBot`` so callers (webui, scripts, tests) switch by changing one
import; the reference's own unmodified file also binds to the new ``libminigpt4.so`` (same 18 symbols,
same struct layouts).  Written fresh as a table-driven ctypes binding.  ``B200`` adds the extension entry
points of ``include/minigpt4_b200.h``.
"""
from __future__ import annotations

import ctypes as C
import dataclasses
import enum
import os
import sys
from pathlib import Path
from typing import Optional

import numpy as np


class DataType(enum.IntEnum):  # include/minigpt4.h MiniGPT4DataType
    F16 = 0; F32 = 1; I32 = 2; L64 = 3; Q4_0 = 4; Q4_1 = 5; Q5_0 = 6; Q5_1 = 7; Q8_0 = 8; Q8_1 = 9
    Q2_K = 10; Q3_K = 11; Q4_K = 12; Q5_K = 13; Q6_K = 14; Q8_K = 15

    def __str__(self):
        return str(self.name)


class Verbosity(enum.IntEnum):
    SILENT = 0; ERR = 1; INFO = 2; DEBUG = 3


class ImageFormat(enum.IntEnum):
    UNKNOWN = 0; F32 = 1; U8 = 2


class MiniGPT4Context:
    def __init__(self, ptr):
        self.ptr = ptr


class MiniGPT4Image(C.Structure):
    _fields_ = [("data", C.c_void_p), ("width", C.c_int32), ("height", C.c_int32), ("channels", C.c_int32), ("format", C.c_int32)]


class MiniGPT4Embedding(C.Structure):
    _fields_ = [("data", C.POINTER(C.c_float)), ("n_embeddings", C.c_size_t)]


class MiniGPT4Images(C.Structure):
    _fields_ = [("images", C.POINTER(MiniGPT4Image)), ("n_images", C.c_size_t)]


class MiniGPT4Embeddings(C.Structure):
    _fields_ = [("embeddings", C.POINTER(MiniGPT4Embedding)), ("n_embeddings", C.c_size_t)]


_CTX, _I, _F, _S = C.c_void_p, C.c_int32, C.c_float, C.c_char_p
_SAMPLING = [_F, _I, _F, _F, _F, _I, _F, _F, _F, _I, _F, _F, _I]
# symbol -> (argtypes, restype); order and types follow include/minigpt4.h
_SIGNATURES = {
    "minigpt4_model_load": ([_S, _S, _I, _I, _I, _I, C.c_bool], _CTX),
    "minigpt4_image_load_from_file": ([_CTX, _S, C.POINTER(MiniGPT4Image), _I], _I),
    "minigpt4_preprocess_image": ([_CTX, C.POINTER(MiniGPT4Image), C.POINTER(MiniGPT4Image), _I], _I),
    "minigpt4_encode_image": ([_CTX, C.POINTER(MiniGPT4Image), C.POINTER(MiniGPT4Embedding), C.c_size_t], _I),
    "minigpt4_begin_chat_image": ([_CTX, C.POINTER(MiniGPT4Embedding), _S, C.c_size_t], _I),
    "minigpt4_end_chat_image": ([_CTX, C.POINTER(C.c_char_p), C.c_size_t] + _SAMPLING, _I),
    "minigpt4_system_prompt": ([_CTX, C.c_size_t], _I),
    "minigpt4_begin_chat": ([_CTX, _S, C.c_size_t], _I),
    "minigpt4_end_chat": ([_CTX, C.POINTER(C.c_char_p), C.c_size_t] + _SAMPLING, _I),
    "minigpt4_reset_chat": ([_CTX], _I),
    "minigpt4_contains_eos_token": ([_S], _I),
    "minigpt4_is_eos": ([_S], _I),
    "minigpt4_free": ([_CTX], _I),
    "minigpt4_free_image": ([C.POINTER(MiniGPT4Image)], _I),
    "minigpt4_free_embedding": ([C.POINTER(MiniGPT4Embedding)], _I),
    "minigpt4_error_code_to_string": ([_I], _S),
    "minigpt4_quantize_model": ([_S, _S, _I], _I),
    "minigpt4_set_verbosity": ([_I], None),
}
ABI_SYMBOLS = tuple(_SIGNATURES)


class MiniGPT4SharedLibrary:
    """Python wrapper around libminigpt4.so; one method per C function, 1:1 with the reference wrapper."""

    def __init__(self, shared_library_path: str):
        self.library = C.cdll.LoadLibrary(shared_library_path)
        for name, (argtypes, restype) in _SIGNATURES.items():
            fn = getattr(self.library, name)
            fn.argtypes, fn.restype = argtypes, restype

    def panic_if_error(self, error_code: int) -> None:
        if error_code != 0:
            raise RuntimeError(self.minigpt4_error_code_to_string(error_code))

    def minigpt4_model_load(self, model_path: str, llm_model_path: str, verbosity: int = 1, seed: int = 1337, n_ctx: int = 2048,
                            n_batch: int = 512, numa: int = 0) -> MiniGPT4Context:
        ptr = self.library.minigpt4_model_load(model_path.encode(), llm_model_path.encode(), int(verbosity), seed, n_ctx, n_batch, bool(numa))
        assert ptr is not None, "minigpt4_model_load failed"
        return MiniGPT4Context(ptr)

    def minigpt4_image_load_from_file(self, ctx: MiniGPT4Context, path: str, flags: int) -> MiniGPT4Image:
        image = MiniGPT4Image()
        self.panic_if_error(self.library.minigpt4_image_load_from_file(ctx.ptr, path.encode(), C.pointer(image), flags))
        return image

    def minigpt4_preprocess_image(self, ctx: MiniGPT4Context, image: MiniGPT4Image, flags: int = 0) -> MiniGPT4Image:
        out = MiniGPT4Image()
        self.panic_if_error(self.library.minigpt4_preprocess_image(ctx.ptr, C.pointer(image), C.pointer(out), flags))
        return out

    def minigpt4_encode_image(self, ctx: MiniGPT4Context, image: MiniGPT4Image, n_threads: int = 0) -> MiniGPT4Embedding:
        embedding = MiniGPT4Embedding()
        self.panic_if_error(self.library.minigpt4_encode_image(ctx.ptr, C.pointer(image), C.pointer(embedding), n_threads))
        return embedding

    def minigpt4_begin_chat_image(self, ctx: MiniGPT4Context, image_embedding: MiniGPT4Embedding, s: str, n_threads: int = 0):
        self.panic_if_error(self.library.minigpt4_begin_chat_image(ctx.ptr, C.pointer(image_embedding), s.encode(), n_threads))

    def _end(self, fn, ctx, n_threads, temp, top_k, top_p, tfs_z, typical_p, repeat_last_n, repeat_penalty, alpha_presence, alpha_frequency,
             mirostat, mirostat_tau, mirostat_eta, penalize_nl) -> str:
        token = C.c_char_p()
        self.panic_if_error(fn(ctx.ptr, C.byref(token), n_threads, temp, top_k, top_p, tfs_z, typical_p, repeat_last_n, repeat_penalty,
                               alpha_presence, alpha_frequency, mirostat, mirostat_tau, mirostat_eta, penalize_nl))
        return token.value.decode("utf-8", errors="ignore")

    def minigpt4_end_chat_image(self, ctx: MiniGPT4Context, n_threads: int = 0, temp: float = 0.8, top_k: int = 40, top_p: float = 0.9,
                                tfs_z: float = 1.0, typical_p: float = 1.0, repeat_last_n: int = 64, repeat_penalty: float = 1.1,
                                alpha_presence: float = 1.0, alpha_frequency: float = 1.0, mirostat: int = 0, mirostat_tau: float = 5.0,
                                mirostat_eta: float = 1.0, penalize_nl: int = 1) -> str:
        return self._end(self.library.minigpt4_end_chat_image, ctx, n_threads, temp, top_k, top_p, tfs_z, typical_p, repeat_last_n, repeat_penalty,
                         alpha_presence, alpha_frequency, mirostat, mirostat_tau, mirostat_eta, penalize_nl)

    def minigpt4_system_prompt(self, ctx: MiniGPT4Context, n_threads: int = 0):
        self.panic_if_error(self.library.minigpt4_system_prompt(ctx.ptr, n_threads))

    def minigpt4_begin_chat(self, ctx: MiniGPT4Context, s: str, n_threads: int = 0):
        self.panic_if_error(self.library.minigpt4_begin_chat(ctx.ptr, s.encode(), n_threads))

    def minigpt4_end_chat(self, ctx: MiniGPT4Context, n_threads: int = 0, temp: float = 0.8, top_k: int = 40, top_p: float = 0.9,
                          tfs_z: float = 1.0, typical_p: float = 1.0, repeat_last_n: int = 64, repeat_penalty: float = 1.1,
                          alpha_presence: float = 1.0, alpha_frequency: float = 1.0, mirostat: int = 0, mirostat_tau: float = 5.0,
                          mirostat_eta: float = 1.0, penalize_nl: int = 1) -> str:
        return self._end(self.library.minigpt4_end_chat, ctx, n_threads, temp, top_k, top_p, tfs_z, typical_p, repeat_last_n, repeat_penalty,
                         alpha_presence, alpha_frequency, mirostat, mirostat_tau, mirostat_eta, penalize_nl)

    def minigpt4_reset_chat(self, ctx: MiniGPT4Context):
        self.panic_if_error(self.library.minigpt4_reset_chat(ctx.ptr))

    def minigpt4_contains_eos_token(self, s: str) -> bool:
        return bool(self.library.minigpt4_contains_eos_token(s.encode()))

    def minigpt4_is_eos(self, s: str) -> bool:
        return bool(self.library.minigpt4_is_eos(s.encode()))

    def minigpt4_free(self, ctx: MiniGPT4Context) -> None:
        self.panic_if_error(self.library.minigpt4_free(ctx.ptr))
        ctx.ptr = None

    def minigpt4_free_image(self, image: MiniGPT4Image) -> None:
        self.panic_if_error(self.library.minigpt4_free_image(C.pointer(image)))

    def minigpt4_free_embedding(self, embedding: MiniGPT4Embedding) -> None:
        self.panic_if_error(self.library.minigpt4_free_embedding(C.pointer(embedding)))

    def minigpt4_error_code_to_string(self, error_code: int) -> str:
        return self.library.minigpt4_error_code_to_string(error_code).decode()

    def minigpt4_quantize_model(self, in_path: str, out_path: str, data_type: DataType):
        self.panic_if_error(self.library.minigpt4_quantize_model(in_path.encode(), out_path.encode(), int(data_type)))

    def minigpt4_set_verbosity(self, verbosity: Verbosity):
        self.library.minigpt4_set_verbosity(int(verbosity))


def library_path() -> Path:
    """In-tree build output (build/libminigpt4.so), built on demand; the extension must exist — no fallback."""
    from . import build as _build
    if os.environ.get("MINIGPT4_B200_LIB"):   # A/B of another build of the same ABI (tools/ab_lib.py, tools/mega_trace.py)
        return Path(os.environ["MINIGPT4_B200_LIB"]).resolve()
    return _build.build()


def load_library() -> MiniGPT4SharedLibrary:
    return MiniGPT4SharedLibrary(str(library_path()))


# ----------------------------------------------------------------------------------------------------
# extension entry points (include/minigpt4_b200.h)
# ----------------------------------------------------------------------------------------------------
class Stats(C.Structure):
    _fields_ = [("llm_weight_bytes_per_token", C.c_double), ("vision_flops_per_image", C.c_double), ("vision_weight_bytes", C.c_double),
                ("last_encode_ms", C.c_double), ("kernel_launches", C.c_ulonglong), ("n_layer", C.c_int), ("n_embd", C.c_int), ("n_ff", C.c_int),
                ("n_vocab", C.c_int), ("n_ctx", C.c_int), ("tp_rank", C.c_int), ("tp_world", C.c_int), ("sm_count", C.c_int), ("decode_megakernel", C.c_int),
                ("prefill_gemm", C.c_int)]


class GenParamsC(C.Structure):  # include/minigpt4_b200.h struct MiniGPT4B200GenParams
    _fields_ = [("size", C.c_int32), ("max_steps", C.c_int32), ("stop", C.c_char_p), ("temp", C.c_float), ("top_k", C.c_int32),
                ("top_p", C.c_float), ("tfs_z", C.c_float), ("typical_p", C.c_float), ("mirostat", C.c_int32), ("mirostat_tau", C.c_float),
                ("mirostat_eta", C.c_float), ("repeat_last_n", C.c_int32), ("repeat_penalty", C.c_float), ("alpha_presence", C.c_float),
                ("alpha_frequency", C.c_float), ("penalize_nl", C.c_int32), ("n_last", C.c_int32), ("last_ids", C.POINTER(C.c_int32))]


@dataclasses.dataclass
class GenParams:
    """one context's settings in B200.generate_batch: B200.sample_until's defaults (mirostat 1 / 2 ignores top_k .. typical_p), with
    neutral penalties (repeat_penalty 1, both alphas 0); last_ids is the penalty history (None: none)"""
    max_steps: int
    stop: str | bytes | None = None
    temp: float = 0.8
    top_k: int = 40
    top_p: float = 0.9
    tfs_z: float = 1.0
    typical_p: float = 1.0
    mirostat: int = 0
    mirostat_tau: float = 5.0
    mirostat_eta: float = 1.0
    repeat_last_n: int = 64
    repeat_penalty: float = 1.0
    alpha_presence: float = 0.0
    alpha_frequency: float = 0.0
    penalize_nl: bool = True
    last_ids: Optional[list] = None


_VP = C.c_void_p
_EXT = {
    "minigpt4_b200_device_count": ([], _I),
    "minigpt4_b200_set_device": ([_I], _I),
    "minigpt4_b200_tp_unique_id": ([_VP], _I),
    "minigpt4_b200_tp_configure": ([_I, _I, _VP], _I),
    "minigpt4_b200_llm_load": ([_S, _I, _I, _I], _CTX),
    "minigpt4_b200_n_vocab": ([_CTX], _I),
    "minigpt4_b200_n_embd": ([_CTX], _I),
    "minigpt4_b200_n_past": ([_CTX], _I),
    "minigpt4_b200_tokenize": ([_CTX, _S, _I, _VP, _I], _I),
    "minigpt4_b200_eval_tokens": ([_CTX, _VP, _I], _I),
    "minigpt4_b200_eval_embd": ([_CTX, _VP, _I], _I),
    "minigpt4_b200_flush": ([_CTX], _I),
    "minigpt4_b200_tp_time_allreduce": ([_CTX, _I, C.POINTER(C.c_float), C.POINTER(C.c_int)], _I),
    "minigpt4_b200_get_logits": ([_CTX, _VP], _I),
    "minigpt4_b200_greedy_id": ([_CTX], _I),
    "minigpt4_b200_get_hidden": ([_CTX, _VP, _I], _I),
    "minigpt4_b200_token_text": ([_CTX, _I], _S),
    "minigpt4_b200_decode_chain": ([_CTX, _I, _VP, C.POINTER(C.c_float)], _I),
    "minigpt4_b200_session_create": ([_CTX, _I], _CTX),
    "minigpt4_b200_session_info": ([_CTX, C.POINTER(C.c_int), C.POINTER(C.c_double), C.POINTER(C.c_double)], _I),
    "minigpt4_b200_decode_batch": ([_VP, _I, _VP, _VP], _I),
    "minigpt4_b200_flush_batch": ([_VP, _I], _I),
    "minigpt4_b200_score_tokens": ([_VP, _I, _VP, _VP, _I, _VP, _VP, _VP], _I),
    "minigpt4_b200_session_copy": ([_CTX, _VP, _I], _I),
    "minigpt4_b200_session_copy_timed": ([_CTX, _VP, _I, C.POINTER(C.c_float)], _I),
    "minigpt4_b200_state_size": ([_CTX], C.c_longlong),
    "minigpt4_b200_state_save": ([_CTX, _VP, C.c_longlong, C.POINTER(C.c_longlong)], _I),
    "minigpt4_b200_state_load": ([_CTX, _VP, C.c_longlong], _I),
    "minigpt4_b200_end_chat_batch": ([_VP, _I, _VP] + _SAMPLING, _I),
    "minigpt4_b200_sample_steps": ([_VP, _I, _I, _F, _I, _F, _F, _F, _VP, C.POINTER(C.c_float)], _I),
    "minigpt4_b200_sample_until": ([_VP, _I, _I, _S, _F, _I, _F, _F, _F, _VP, _VP, _VP, C.POINTER(C.c_float)], _I),
    "minigpt4_b200_beam_search": ([_VP, _I, _I, _S, _F, _I, _VP, _VP, _VP, _VP, _VP, C.POINTER(C.c_float)], _I),
    "minigpt4_b200_op_beam_rank": ([_VP, _I, _VP, _I, _I, _VP, _VP, _VP], _I),
    "minigpt4_b200_sample_steps_mirostat": ([_VP, _I, _I, _F, _I, _F, _F, _VP, C.POINTER(C.c_float)], _I),
    "minigpt4_b200_sample_until_mirostat": ([_VP, _I, _I, _S, _F, _I, _F, _F, _VP, _VP, _VP, C.POINTER(C.c_float)], _I),
    "minigpt4_b200_sample_until_logprobs": ([_VP, _I, _I, _S, _F, _I, _F, _F, _F, _I, _F, _F, _I, _VP, _VP, _VP, _VP, _VP, _VP, _VP,
                                             C.POINTER(C.c_float)], _I),
    "minigpt4_b200_op_logprobs": ([_VP, _I, _I, _VP, _I, _VP, _VP, _VP, _VP, C.POINTER(C.c_float)], _I),
    "minigpt4_b200_sample_until_penalized": ([_VP, _I, _I, _S, _F, _I, _F, _F, _F, _I, _F, _F, _I, _F, _F, _F, _I, _VP, _VP, _VP, _VP, _VP,
                                              C.POINTER(C.c_float)], _I),
    "minigpt4_b200_generate_batch": ([_VP, _I, _VP, _I, _VP, _VP, _VP, _VP, _VP, _VP, _VP, C.POINTER(C.c_float)], _I),
    "minigpt4_b200_end_chat_penalized": ([_CTX, C.POINTER(_S), _F, _I, _F, _F, _F, _I, _F, _F, _F, _I, _I, _F, _F, _VP, _I,
                                          C.POINTER(C.c_int32)], _I),
    "minigpt4_b200_op_penalize": ([_VP, _I, _I, _VP, _VP, _I, _F, _F, _F, _I, _I, _VP, C.POINTER(C.c_float)], _I),
    "minigpt4_b200_constraint_create": ([_CTX, _I, _VP, _VP], _VP),
    "minigpt4_b200_constraint_free": ([_VP], None),
    "minigpt4_b200_constraint_attach": ([_CTX, _VP], _I),
    "minigpt4_b200_constraint_state": ([_CTX, C.POINTER(_I), C.POINTER(_I)], _I),
    "minigpt4_b200_constraint_allowed": ([_VP, _I, _VP, _VP, _I], _I),
    "minigpt4_b200_host_constraint_allowed": ([_S, _I, _VP, _VP, _I, _VP, _VP, _I], _I),
    "minigpt4_b200_encode_images": ([_CTX, C.POINTER(MiniGPT4Images), C.POINTER(MiniGPT4Embeddings)], _I),
    "minigpt4_b200_stats": ([_CTX, C.POINTER(Stats)], _I),
    "minigpt4_b200_time_matvec": ([_CTX, _I, _I, C.POINTER(C.c_float), C.POINTER(C.c_double)], _I),
    "minigpt4_b200_mega_trace": ([_CTX, _VP, _I], _I),
    "minigpt4_b200_op_matvec": ([_I, _I, _I, _VP, _VP, _I, _VP], _I),
    "minigpt4_b200_op_gemm_f16": ([_I, _I, _I, _VP, _VP, _VP, _I, _VP, _F, _I, _I, _I, _I, _VP, _VP], _I),
    "minigpt4_b200_op_layernorm": ([_VP, _I, _I, _VP, _VP, _VP, _VP], _I),
    "minigpt4_b200_op_layernorm_fold": ([_VP, _I, _I, _VP, _VP, _VP, _I, C.c_longlong, _VP], _I),
    "minigpt4_b200_op_attention": ([_VP, C.c_longlong, C.c_longlong, _I, C.c_longlong, C.c_longlong, _I, _I, _I, _I, _I, _F, _I, _I, _VP], _I),
    "minigpt4_b200_encode_taps": ([_CTX, _VP, _VP, _VP, _VP, _VP, _VP], _I),
    "minigpt4_b200_op_llama_attention": ([_VP, _VP, _VP, _I, _I, _I, _VP, _I, _VP], _I),
    "minigpt4_b200_op_dequant_f16": ([_I, _VP, C.c_long, _VP], _I),
    "minigpt4_b200_host_quantize_row": ([_I, _VP, C.c_long, _VP], C.c_long),
    "minigpt4_b200_host_tokenize": ([_S, _S, _I, _VP, _I], _I),
    "minigpt4_b200_host_sample": ([_VP, _I, _I, _F, _I, _F, _F, _F, _I, _F, _F, _I, _VP], _I),
    "minigpt4_b200_op_sample": ([_VP, _I, _I, _F, _I, _F, _F, _F, _I, _VP], _I),
    "minigpt4_b200_op_sample_timed": ([_VP, _I, _I, _F, _I, _F, _F, _F, _I, _VP, C.POINTER(C.c_float)], _I),
    "minigpt4_b200_op_reply_stop": ([_CTX, _VP, _I, _S, _S, C.POINTER(C.c_int32)], _I),
    "minigpt4_b200_op_check_libm": ([_I, C.c_uint32, C.c_uint32, C.POINTER(C.c_longlong)], _I),
    "minigpt4_b200_op_sample_mirostat": ([_VP, _I, _I, _F, _I, _F, _F, _I, _I, _VP, _VP, C.POINTER(C.c_float)], _I),
    "minigpt4_b200_op_check_log2f": ([C.c_uint32, C.c_uint32, C.POINTER(C.c_longlong)], _I),
    "minigpt4_b200_op_check_powf": ([_F, C.c_uint32, C.c_uint32, C.POINTER(C.c_longlong)], _I),
    "minigpt4_b200_host_inspect_container": ([_S, C.POINTER(_I), C.POINTER(_I), C.POINTER(_I)], _I),
    "minigpt4_b200_host_inspect_ggjt": ([_S, C.POINTER(_I), C.POINTER(_I), C.POINTER(_I), C.POINTER(_I)], _I),
}
EXT_SYMBOLS = tuple(_EXT)


def _ptr(a: Optional[np.ndarray]):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def choices_dfa(choices: list[bytes]) -> tuple[np.ndarray, np.ndarray]:
    """The byte automaton of "exactly one of these answers": a trie over the choices' bytes, start state 0.  Returns (next [n_states,
    256] int32, -1 rejects; accept [n_states] uint8), the form minigpt4_b200_constraint_create takes."""
    nxt: list[list[int]] = [[-1] * 256]
    acc = [0]
    for ch in choices:
        s = 0
        for b in bytes(ch):
            if nxt[s][b] < 0:
                nxt[s][b] = len(nxt)
                nxt.append([-1] * 256)
                acc.append(0)
            s = nxt[s][b]
        acc[s] = 1
    return np.array(nxt, np.int32), np.array(acc, np.uint8)


def _automaton(next_states, accept) -> tuple[np.ndarray, np.ndarray]:
    nx = np.ascontiguousarray(next_states, np.int32)
    ac = np.ascontiguousarray(accept, np.uint8)
    assert nx.ndim == 2 and nx.shape[1] == 256 and ac.shape == (nx.shape[0],), "next [n_states, 256], accept [n_states]"
    return nx, ac


class B200:
    """numpy-friendly access to the extension ABI."""

    def __init__(self, lib: MiniGPT4SharedLibrary):
        self.base = lib
        self.L = lib.library
        for name, (argtypes, restype) in _EXT.items():
            fn = getattr(self.L, name)
            fn.argtypes, fn.restype = argtypes, restype

    def _chk(self, code: int):
        self.base.panic_if_error(code)

    def llm_load(self, llm_path: str, n_ctx: int = 2048, seed: int = 1337, verbosity: int = 1) -> MiniGPT4Context:
        ptr = self.L.minigpt4_b200_llm_load(llm_path.encode(), n_ctx, seed, verbosity)
        assert ptr is not None, "minigpt4_b200_llm_load failed"
        return MiniGPT4Context(ptr)

    def tokenize(self, ctx, text: str | bytes, add_bos: bool = True) -> list[int]:
        b = text.encode() if isinstance(text, str) else text
        buf = np.zeros(len(b) + 2, np.int32)
        n = self.L.minigpt4_b200_tokenize(ctx.ptr, b, int(add_bos), _ptr(buf), buf.size)
        assert n >= 0
        return buf[:n].tolist()

    def eval_tokens(self, ctx, ids):
        a = np.ascontiguousarray(ids, np.int32)
        self._chk(self.L.minigpt4_b200_eval_tokens(ctx.ptr, _ptr(a), a.size))

    def eval_embd(self, ctx, rows: np.ndarray):
        a = np.ascontiguousarray(rows, np.float32)
        self._chk(self.L.minigpt4_b200_eval_embd(ctx.ptr, _ptr(a), a.shape[0]))

    def tp_time_allreduce(self, ctx, reps: int = 64) -> tuple[float, bool]:
        us, peer = C.c_float(0), C.c_int(0)
        self._chk(self.L.minigpt4_b200_tp_time_allreduce(ctx.ptr, reps, C.byref(us), C.byref(peer)))
        return us.value, bool(peer.value)

    def flush(self, ctx) -> None:
        """evaluate the queued prompt rows now (they are otherwise evaluated together when the model state is first needed)"""
        self._chk(self.L.minigpt4_b200_flush(ctx.ptr))

    def logits(self, ctx) -> np.ndarray:
        out = np.empty(self.L.minigpt4_b200_n_vocab(ctx.ptr), np.float32)
        self._chk(self.L.minigpt4_b200_get_logits(ctx.ptr, _ptr(out)))
        return out

    def hidden(self, ctx, n_rows: int) -> np.ndarray:
        out = np.empty((n_rows, self.L.minigpt4_b200_n_embd(ctx.ptr)), np.float32)
        self._chk(self.L.minigpt4_b200_get_hidden(ctx.ptr, _ptr(out), n_rows))
        return out

    def greedy_id(self, ctx) -> int:
        return self.L.minigpt4_b200_greedy_id(ctx.ptr)

    def n_past(self, ctx) -> int:
        return self.L.minigpt4_b200_n_past(ctx.ptr)

    def decode_chain(self, ctx, steps: int) -> tuple[np.ndarray, float]:
        ids = np.zeros(steps, np.int32)
        ms = C.c_float(0)
        self._chk(self.L.minigpt4_b200_decode_chain(ctx.ptr, steps, _ptr(ids), C.byref(ms)))
        return ids, ms.value

    # multi-session serving: contexts that share one loaded model, stepped together
    def session_create(self, ctx, seed: int = 1337) -> MiniGPT4Context:
        """a new conversation over ctx's model (weights shared, own KV cache / state / sampler seeded with `seed`)"""
        ptr = self.L.minigpt4_b200_session_create(ctx.ptr, seed)
        assert ptr is not None, "minigpt4_b200_session_create failed"
        return MiniGPT4Context(ptr)

    def session_info(self, ctx) -> tuple[int, float, float]:
        """(live contexts of the group, device bytes ctx owns, device bytes it shares)"""
        n, owned, shared = C.c_int(0), C.c_double(0), C.c_double(0)
        self._chk(self.L.minigpt4_b200_session_info(ctx.ptr, C.byref(n), C.byref(owned), C.byref(shared)))
        return n.value, owned.value, shared.value

    @staticmethod
    def _ctx_array(ctxs):
        return (C.c_void_p * max(1, len(ctxs)))(*[c.ptr for c in ctxs])

    def decode_batch(self, ctxs, ids=None) -> np.ndarray:
        """one decode step of every context in `ctxs` (1..64 of one group; weights streamed once); ids[i] < 0 or ids None: each context's
        own greedy id.  Returns the new greedy ids."""
        n = len(ctxs)
        a = np.full(n, -1, np.int32) if ids is None else np.ascontiguousarray(ids, np.int32)
        out = np.zeros(max(1, n), np.int32)
        self._chk(self.L.minigpt4_b200_decode_batch(C.cast(self._ctx_array(ctxs), C.c_void_p), n, _ptr(a), _ptr(out)))
        return out[:n]

    def flush_batch(self, ctxs) -> None:
        """evaluate the queued prompt rows of every context in `ctxs` (1..64 of one group) in shared passes over the weights"""
        self._chk(self.L.minigpt4_b200_flush_batch(C.cast(self._ctx_array(ctxs), C.c_void_p), len(ctxs)))

    def score_tokens(self, ctxs, id_lists, keep: bool = False, logits: bool = False) -> list[tuple]:
        """the log-probability and rank of every id of id_lists[i] (>= 1 ids) as a continuation of context ctxs[i] (1..64 of one group), in
        shared passes over the weights; per context (logprob float32, rank int32[, logits float32 [n_ids, n_vocab]]).  Entry 0 is NaN with
        rank -1 on a context at n_past 0.  keep: the ids stay evaluated (as eval_tokens + flush); otherwise every context is left as it was."""
        n = len(ctxs)
        lens = np.array([len(x) for x in id_lists], np.int32)
        ids = np.ascontiguousarray(np.concatenate([np.asarray(x, np.int32).ravel() for x in id_lists]) if n else np.zeros(0, np.int32), np.int32)
        total = max(1, int(lens.sum()))
        lp, rk = np.empty(total, np.float32), np.empty(total, np.int32)
        lg = np.empty((total, self.L.minigpt4_b200_n_vocab(ctxs[0].ptr)), np.float32) if logits and n else None
        self._chk(self.L.minigpt4_b200_score_tokens(C.cast(self._ctx_array(ctxs), C.c_void_p), n, _ptr(ids), _ptr(lens), int(keep), _ptr(lp),
                                                    _ptr(rk), _ptr(lg)))
        out, o = [], 0
        for k in lens.tolist():
            out.append((lp[o:o + k], rk[o:o + k]) + ((lg[o:o + k],) if logits else ()))
            o += k
        return out

    def session_copy(self, src, dsts) -> float:
        """copy src's conversation (n_past, K / V rows, logits, greedy id, device state, reply tail) into every context in `dsts` (1..64 other
        contexts of src's group), each keeping its own sampler; src's queue is evaluated first.  Returns the copy kernel's device ms."""
        ms = C.c_float(0)
        self._chk(self.L.minigpt4_b200_session_copy_timed(src.ptr, C.cast(self._ctx_array(dsts), C.c_void_p), len(dsts), C.byref(ms)))
        return ms.value

    def state_save(self, ctx) -> bytes:
        """ctx's conversation as the state blob of minigpt4_b200_state_save (its queue is evaluated first)"""
        size = self.L.minigpt4_b200_state_size(ctx.ptr)
        assert size >= 0, "minigpt4_b200_state_size failed"
        buf = np.empty(size, np.uint8)
        written = C.c_longlong(0)
        self._chk(self.L.minigpt4_b200_state_save(ctx.ptr, _ptr(buf), size, C.byref(written)))
        return buf[:written.value].tobytes()

    def state_load(self, ctx, data: bytes) -> None:
        """replace ctx's conversation by a saved one (its sampler is kept, its queue discarded)"""
        a = np.frombuffer(data, np.uint8)
        self._chk(self.L.minigpt4_b200_state_load(ctx.ptr, _ptr(a), a.size))

    def end_chat_batch(self, ctxs, temp: float = 0.8, top_k: int = 40, top_p: float = 0.9, tfs_z: float = 1.0, typical_p: float = 1.0,
                       repeat_last_n: int = 64, repeat_penalty: float = 1.1, alpha_presence: float = 1.0, alpha_frequency: float = 1.0,
                       mirostat: int = 0, mirostat_tau: float = 5.0, mirostat_eta: float = 1.0, penalize_nl: int = 1) -> list[str]:
        """minigpt4_end_chat on each context (own logits, own sampler), the sampled tokens fed in one batched step; returns their texts"""
        n = len(ctxs)
        toks = (C.c_char_p * max(1, n))()
        self._chk(self.L.minigpt4_b200_end_chat_batch(C.cast(self._ctx_array(ctxs), C.c_void_p), n, C.cast(toks, C.c_void_p), temp, top_k, top_p,
                                                      tfs_z, typical_p, repeat_last_n, repeat_penalty, alpha_presence, alpha_frequency, mirostat,
                                                      mirostat_tau, mirostat_eta, penalize_nl))
        return [toks[i].decode("utf-8", errors="ignore") for i in range(n)]

    def sample_steps(self, ctxs, steps: int, temp: float = 0.8, top_k: int = 40, top_p: float = 0.9, tfs_z: float = 1.0,
                     typical_p: float = 1.0, mirostat: int = 0, mirostat_tau: float = 5.0, mirostat_eta: float = 1.0) -> tuple[np.ndarray, float]:
        """`steps` device-sampled decode steps of every context in `ctxs` (1..64 of one group) with no host round trip in between;
        returns the fed ids [steps, n] and the device ms of the steps.  mirostat 1 / 2: minigpt4_b200_sample_steps_mirostat (top_k ..
        typical_p do not apply)"""
        n = len(ctxs)
        ids = np.zeros((max(1, steps), max(1, n)), np.int32)
        ms = C.c_float(0)
        ctx = C.cast(self._ctx_array(ctxs), C.c_void_p)
        if mirostat:
            self._chk(self.L.minigpt4_b200_sample_steps_mirostat(ctx, n, steps, temp, mirostat, mirostat_tau, mirostat_eta, _ptr(ids), C.byref(ms)))
        else:
            self._chk(self.L.minigpt4_b200_sample_steps(ctx, n, steps, temp, top_k, top_p, tfs_z, typical_p, _ptr(ids), C.byref(ms)))
        return ids[:steps, :n], ms.value

    def sample_until(self, ctxs, max_steps: int, stop: str | bytes | None = None, temp: float = 0.8, top_k: int = 40, top_p: float = 0.9,
                     tfs_z: float = 1.0, typical_p: float = 1.0, mirostat: int = 0, mirostat_tau: float = 5.0,
                     mirostat_eta: float = 1.0) -> tuple[list[list[int]], list[bool], float]:
        """device-sampled steps of every context in `ctxs` (1..64 of one group), each until its reply ends with `stop` (None: "###"; "": never)
        or max_steps; returns each context's fed ids, whether the stop text ended it, and the device ms.  mirostat 1 / 2:
        minigpt4_b200_sample_until_mirostat"""
        n = len(ctxs)
        ids = np.zeros((max(1, max_steps), max(1, n)), np.int32)
        n_out, stopped = np.zeros(max(1, n), np.int32), np.zeros(max(1, n), np.int32)
        ms = C.c_float(0)
        st = stop.encode() if isinstance(stop, str) else stop
        ctx = C.cast(self._ctx_array(ctxs), C.c_void_p)
        if mirostat:
            self._chk(self.L.minigpt4_b200_sample_until_mirostat(ctx, n, max_steps, st, temp, mirostat, mirostat_tau, mirostat_eta, _ptr(ids),
                                                                 _ptr(n_out), _ptr(stopped), C.byref(ms)))
        else:
            self._chk(self.L.minigpt4_b200_sample_until(ctx, n, max_steps, st, temp, top_k, top_p, tfs_z, typical_p, _ptr(ids), _ptr(n_out),
                                                        _ptr(stopped), C.byref(ms)))
        return [ids[:n_out[i], i].tolist() for i in range(n)], [bool(x) for x in stopped[:n]], ms.value

    def sample_until_logprobs(self, ctxs, max_steps: int, stop: str | bytes | None = None, top_n: int = 0, temp: float = 0.8, top_k: int = 40,
                              top_p: float = 0.9, tfs_z: float = 1.0, typical_p: float = 1.0, mirostat: int = 0, mirostat_tau: float = 5.0,
                              mirostat_eta: float = 1.0) -> tuple[list[list[int]], list[bool], list[tuple], float]:
        """sample_until (mirostat 1 / 2: sample_until_mirostat) with the same ids and end state, which also reports each fed id's
        log-probability and rank under the raw logits it was drawn from, and the top_n (0..20) most likely ids there.  Returns each
        context's fed ids, whether the stop text ended it, its records (logprob float32 [k], rank int32 [k], top ids int32 [k, top_n], top
        log-probabilities float32 [k, top_n]; k its ids) and the device ms."""
        n = len(ctxs)
        shape = (max(1, max_steps), max(1, n))
        ids, lp, rk = np.zeros(shape, np.int32), np.zeros(shape, np.float32), np.zeros(shape, np.int32)
        tid, tlp = np.zeros(shape + (max(1, top_n),), np.int32), np.zeros(shape + (max(1, top_n),), np.float32)
        n_out, stopped = np.zeros(max(1, n), np.int32), np.zeros(max(1, n), np.int32)
        ms = C.c_float(0)
        st = stop.encode() if isinstance(stop, str) else stop
        self._chk(self.L.minigpt4_b200_sample_until_logprobs(C.cast(self._ctx_array(ctxs), C.c_void_p), n, max_steps, st, temp, top_k, top_p, tfs_z,
                                                             typical_p, mirostat, mirostat_tau, mirostat_eta, top_n, _ptr(ids), _ptr(n_out),
                                                             _ptr(stopped), _ptr(lp), _ptr(rk), _ptr(tid), _ptr(tlp), C.byref(ms)))
        recs = [(lp[:k, i].copy(), rk[:k, i].copy(), tid[:k, i, :top_n].copy(), tlp[:k, i, :top_n].copy()) for i, k in enumerate(n_out[:n].tolist())]
        return [ids[:n_out[i], i].tolist() for i in range(n)], [bool(x) for x in stopped[:n]], recs, ms.value

    def op_logprobs(self, logits: np.ndarray, ids, top_n: int) -> tuple[np.ndarray, np.ndarray, np.ndarray, np.ndarray, float]:
        """sample_until_logprobs' records through its kernel over host logits [rows, n_vocab] (rows 1..64) and one fed id per row:
        (logprob [rows], rank [rows], top ids [rows, top_n], top log-probabilities [rows, top_n], kernel ms per launch)"""
        lg = np.ascontiguousarray(logits, np.float32)
        rows, V = lg.shape
        t = np.ascontiguousarray(ids, np.int32)
        lp, rk = np.zeros(rows, np.float32), np.zeros(rows, np.int32)
        tid, tlp = np.zeros((rows, max(1, top_n)), np.int32), np.zeros((rows, max(1, top_n)), np.float32)
        ms = C.c_float(0)
        self._chk(self.L.minigpt4_b200_op_logprobs(_ptr(lg), rows, V, _ptr(t), top_n, _ptr(lp), _ptr(rk), _ptr(tid), _ptr(tlp), C.byref(ms)))
        return lp, rk, tid[:, :top_n], tlp[:, :top_n], ms.value

    @staticmethod
    def _histories(last_ids, n: int) -> tuple[np.ndarray, np.ndarray]:
        """each context's history (a list of id lists, None: none) as minigpt4_b200_*_penalized take them: (ids one after another, counts)"""
        lists = [[] if x is None else list(x) for x in (last_ids if last_ids is not None else [None] * n)]
        assert len(lists) == n, "one history per context"
        flat = np.ascontiguousarray(np.concatenate([np.asarray(x, np.int32).ravel() for x in lists]) if n else np.zeros(0, np.int32), np.int32)
        return (flat if flat.size else np.zeros(1, np.int32)), np.array([len(x) for x in lists] or [0], np.int32)

    def sample_until_penalized(self, ctxs, max_steps: int, stop: str | bytes | None = None, last_ids=None, repeat_last_n: int = 64,
                               repeat_penalty: float = 1.1, alpha_presence: float = 0.0, alpha_frequency: float = 0.0, penalize_nl: bool = True,
                               temp: float = 0.8, top_k: int = 40, top_p: float = 0.9, tfs_z: float = 1.0, typical_p: float = 1.0,
                               mirostat: int = 0, mirostat_tau: float = 5.0,
                               mirostat_eta: float = 1.0) -> tuple[list[list[int]], list[bool], float]:
        """sample_until (mirostat 1 / 2: sample_until_mirostat) that samples every step from the logits after llama.cpp's repetition,
        frequency and presence penalties over the last repeat_last_n ids of last_ids[i] (context i's history; None: none) and the ids the
        call has fed.  The defaults are llama.cpp main's.  Returns each context's fed ids, whether the stop text ended it, and the device ms."""
        n = len(ctxs)
        ids = np.zeros((max(1, max_steps), max(1, n)), np.int32)
        n_out, stopped = np.zeros(max(1, n), np.int32), np.zeros(max(1, n), np.int32)
        hist, n_last = self._histories(last_ids, n)
        ms = C.c_float(0)
        st = stop.encode() if isinstance(stop, str) else stop
        self._chk(self.L.minigpt4_b200_sample_until_penalized(C.cast(self._ctx_array(ctxs), C.c_void_p), n, max_steps, st, temp, top_k, top_p,
                                                              tfs_z, typical_p, mirostat, mirostat_tau, mirostat_eta, repeat_last_n, repeat_penalty,
                                                              alpha_presence, alpha_frequency, int(penalize_nl), _ptr(hist), _ptr(n_last),
                                                              _ptr(ids), _ptr(n_out), _ptr(stopped), C.byref(ms)))
        return [ids[:n_out[i], i].tolist() for i in range(n)], [bool(x) for x in stopped[:n]], ms.value

    @staticmethod
    def gen_params_c(params: list[GenParams]) -> tuple:
        """the C array of params and the buffers it points into (keep them alive for the call)"""
        arr = (GenParamsC * max(1, len(params)))()
        keep = []
        for i, g in enumerate(params):
            st = g.stop.encode() if isinstance(g.stop, str) else g.stop
            hist = np.ascontiguousarray(g.last_ids if g.last_ids is not None else [], np.int32)
            keep += [st, hist]
            arr[i] = GenParamsC(C.sizeof(GenParamsC), g.max_steps, st, g.temp, g.top_k, g.top_p, g.tfs_z, g.typical_p, g.mirostat, g.mirostat_tau,
                                g.mirostat_eta, g.repeat_last_n, g.repeat_penalty, g.alpha_presence, g.alpha_frequency, int(g.penalize_nl), hist.size,
                                hist.ctypes.data_as(C.POINTER(C.c_int32)) if hist.size else None)
        return arr, keep

    def generate_batch(self, ctxs, params: list[GenParams], top_n: int = 0, logprobs: bool = False) -> tuple:
        """device-sampled replies of every context in `ctxs` (1..64 of one group), context i with its own settings params[i] (sampler,
        penalties, stop text, budget), in one batched call; each context ends where it would end alone.  Returns each context's fed ids,
        whether the stop text ended it, with logprobs its records (as sample_until_logprobs returns them; top_n 0..20) and the device ms."""
        n = len(ctxs)
        arr, _keep = self.gen_params_c(params)
        S = max([g.max_steps for g in params] + [1])
        shape = (S, max(1, n))
        ids = np.zeros(shape, np.int32)
        n_out, stopped = np.zeros(max(1, n), np.int32), np.zeros(max(1, n), np.int32)
        lp, rk = np.zeros(shape, np.float32), np.zeros(shape, np.int32)
        tid, tlp = np.zeros(shape + (max(1, top_n),), np.int32), np.zeros(shape + (max(1, top_n),), np.float32)
        ms = C.c_float(0)
        self._chk(self.L.minigpt4_b200_generate_batch(C.cast(self._ctx_array(ctxs), C.c_void_p), n, C.cast(arr, C.c_void_p), top_n, _ptr(ids),
                                                      _ptr(n_out), _ptr(stopped), _ptr(lp) if logprobs else None, _ptr(rk) if logprobs else None,
                                                      _ptr(tid) if logprobs else None, _ptr(tlp) if logprobs else None, C.byref(ms)))
        out = [ids[:n_out[i], i].tolist() for i in range(n)], [bool(x) for x in stopped[:n]]
        if not logprobs:
            return (*out, ms.value)
        recs = [(lp[:k, i].copy(), rk[:k, i].copy(), tid[:k, i, :top_n].copy(), tlp[:k, i, :top_n].copy()) for i, k in enumerate(n_out[:n].tolist())]
        return (*out, recs, ms.value)

    def end_chat_penalized(self, ctx, last_ids=None, repeat_last_n: int = 64, repeat_penalty: float = 1.1, alpha_presence: float = 0.0,
                           alpha_frequency: float = 0.0, penalize_nl: bool = True, temp: float = 0.8, top_k: int = 40, top_p: float = 0.9,
                           tfs_z: float = 1.0, typical_p: float = 1.0, mirostat: int = 0, mirostat_tau: float = 5.0,
                           mirostat_eta: float = 1.0) -> tuple[str, int]:
        """minigpt4_end_chat with ctx's host sampler over its logits after the penalties of sample_until_penalized, the window being the last
        repeat_last_n ids of last_ids; returns the fed token's text and id"""
        hist = np.ascontiguousarray(last_ids if last_ids is not None else [], np.int32)
        tok, tid = C.c_char_p(), C.c_int32(0)
        self._chk(self.L.minigpt4_b200_end_chat_penalized(ctx.ptr, C.byref(tok), temp, top_k, top_p, tfs_z, typical_p, repeat_last_n, repeat_penalty,
                                                          alpha_presence, alpha_frequency, int(penalize_nl), mirostat, mirostat_tau, mirostat_eta,
                                                          _ptr(hist if hist.size else np.zeros(1, np.int32)), hist.size, C.byref(tid)))
        return tok.value.decode("utf-8", errors="ignore"), tid.value

    def op_penalize(self, logits: np.ndarray, last_ids=None, repeat_last_n: int = 64, repeat_penalty: float = 1.1, alpha_presence: float = 0.0,
                    alpha_frequency: float = 0.0, penalize_nl: bool = True, on_device: bool = True) -> tuple[np.ndarray, float]:
        """sample_until_penalized's penalised logits over host rows [rows, n_vocab] (rows 1..64), row r's window the last repeat_last_n ids
        of last_ids[r], through its kernel or (on_device False) the host sampler's penalize: (penalised rows, kernel ms per launch)"""
        lg = np.ascontiguousarray(logits, np.float32)
        rows, V = lg.shape
        hist, n_last = self._histories(last_ids, rows)
        out = np.zeros_like(lg)
        ms = C.c_float(0)
        self._chk(self.L.minigpt4_b200_op_penalize(_ptr(lg), rows, V, _ptr(hist), _ptr(n_last), repeat_last_n, repeat_penalty, alpha_presence,
                                                   alpha_frequency, int(penalize_nl), int(on_device), _ptr(out), C.byref(ms)))
        return out, ms.value

    def beam_search(self, ctxs, max_steps: int, stop: str | bytes | None = None, length_penalty: float = 1.0,
                    n_hyp: int = 1) -> tuple[list[tuple[list[int], float, float, bool]], float]:
        """the n_hyp best replies of ctxs[0]'s conversation by beam search with len(ctxs) (1..16) beams; ctxs[1:] are other sessions of
        its group used as working beams (their conversations are overwritten by ctxs[0]'s).  stop: None "###", "" no text stop.  Returns
        ([(ids, final score, sum of log-probabilities, stopped), ...] best first, device ms); afterwards ctxs[0] has fed the best ids."""
        n = len(ctxs)
        ids = np.full((max(1, n_hyp), max(1, max_steps)), -1, np.int32)
        n_out, stopped = np.zeros(max(1, n_hyp), np.int32), np.zeros(max(1, n_hyp), np.int32)
        score, lp = np.zeros(max(1, n_hyp), np.float32), np.zeros(max(1, n_hyp), np.float32)
        ms = C.c_float(0)
        st = stop.encode() if isinstance(stop, str) else stop
        self._chk(self.L.minigpt4_b200_beam_search(C.cast(self._ctx_array(ctxs), C.c_void_p), n, max_steps, st, length_penalty, n_hyp, _ptr(ids),
                                                   _ptr(n_out), _ptr(score), _ptr(lp), _ptr(stopped), C.byref(ms)))
        return [(ids[h, :n_out[h]].tolist(), float(score[h]), float(lp[h]), bool(stopped[h])) for h in range(n_hyp)], ms.value

    def op_beam_rank(self, logits: np.ndarray, S: np.ndarray, n_beams: int) -> tuple[np.ndarray, np.ndarray, np.ndarray]:
        """beam_search's candidate order through its kernels over host logits [n_live, n_vocab] and beam scores S [n_live]: the first
        2 n_beams candidates' (parent beam, id, c)"""
        lg = np.ascontiguousarray(logits, np.float32)
        s = np.ascontiguousarray(S, np.float32)
        n_live, V = lg.shape
        k = min(2 * n_beams, n_live * V)
        par, ids, c = np.zeros(2 * n_beams, np.int32), np.zeros(2 * n_beams, np.int32), np.zeros(2 * n_beams, np.float32)
        self._chk(self.L.minigpt4_b200_op_beam_rank(_ptr(lg), n_live, _ptr(s), n_beams, V, _ptr(par), _ptr(ids), _ptr(c)))
        return par[:k], ids[:k], c[:k]

    # constrained replies (minigpt4_b200_constraint_*): handles are plain ints (the C pointer)
    def constraint_create(self, ctx, next_states, accept) -> int:
        """compile the byte automaton (next [n_states, 256] int32, -1 rejects; accept [n_states]) against ctx's vocabulary; the handle"""
        nx, ac = _automaton(next_states, accept)
        h = self.L.minigpt4_b200_constraint_create(ctx.ptr, nx.shape[0], _ptr(nx), _ptr(ac))
        assert h, "minigpt4_b200_constraint_create refused the automaton"
        return h

    def constraint_free(self, handle: int) -> None:
        self.L.minigpt4_b200_constraint_free(handle)

    def constraint_attach(self, ctx, handle: Optional[int]) -> None:
        """attach the constraint (None: detach); its state starts at 0"""
        self._chk(self.L.minigpt4_b200_constraint_attach(ctx.ptr, handle))

    def constraint_state(self, ctx) -> tuple[int, bool]:
        """(state, finished) of ctx's constraint; state is -1 once finished"""
        st, fin = C.c_int(0), C.c_int(0)
        self._chk(self.L.minigpt4_b200_constraint_state(ctx.ptr, C.byref(st), C.byref(fin)))
        return st.value, bool(fin.value)

    @staticmethod
    def _allowed(call) -> Optional[tuple[np.ndarray, np.ndarray]]:
        # room for one pair first: -1 then means a pruned state, not a short buffer
        ids, nxt = np.zeros(1, np.int32), np.zeros(1, np.int32)
        n = call(_ptr(ids), _ptr(nxt), 1)
        if n == -1:
            return None
        if n < 0:
            ids, nxt = np.zeros(-n, np.int32), np.zeros(-n, np.int32)
            n = call(_ptr(ids), _ptr(nxt), ids.size)
            assert n == ids.size, n
        return ids[:n], nxt[:n]

    def constraint_allowed(self, handle: int, state: int) -> Optional[tuple[np.ndarray, np.ndarray]]:
        """allowed(state) as compiled: (ids ascending, next states with -1 for finished); None for a state that is not live"""
        return self._allowed(lambda ids, nxt, cap: self.L.minigpt4_b200_constraint_allowed(handle, state, ids, nxt, cap))

    def host_constraint_allowed(self, llm_path: str, next_states, accept, state: int) -> Optional[tuple[np.ndarray, np.ndarray]]:
        """constraint_allowed compiled on the host against the vocabulary of a ggjt file (no GPU); None for a state that is not live"""
        nx, ac = _automaton(next_states, accept)
        def call(ids, nxt, cap):
            r = self.L.minigpt4_b200_host_constraint_allowed(llm_path.encode(), nx.shape[0], _ptr(nx), _ptr(ac), state, ids, nxt, cap)
            assert r != -1000000, "unreadable file or refused automaton"
            return r
        return self._allowed(call)

    def host_constraint_refused(self, llm_path: str, next_states, accept) -> bool:
        """whether the host compiler refuses the automaton (next and accept taken as given)"""
        nx = np.ascontiguousarray(next_states, np.int32).reshape(-1)
        ac = np.ascontiguousarray(accept, np.uint8)
        return self.L.minigpt4_b200_host_constraint_allowed(llm_path.encode(), ac.size, _ptr(nx), _ptr(ac), 0, None, None, 0) == -1000000

    def time_matvec(self, ctx, kind: int, reps: int = 3) -> tuple[float, float]:
        ms, nb = C.c_float(0), C.c_double(0)
        self._chk(self.L.minigpt4_b200_time_matvec(ctx.ptr, kind, reps, C.byref(ms), C.byref(nb)))
        return ms.value, nb.value

    def mega_trace(self, ctx) -> np.ndarray:
        """per-op clock stamps [2 CTAs][n_ops][16] of the last megakernel launch (needs MINIGPT4_B200_MEGA_TRACE=1 at load)"""
        buf = np.zeros(2 * 403 * 16, np.int64)
        n = self.L.minigpt4_b200_mega_trace(ctx.ptr, _ptr(buf), buf.size)
        slots = 16 if self.stats(ctx).decode_megakernel >= 6 else 8
        return buf[:n].reshape(2, -1, slots) if n else buf[:0]

    def stats(self, ctx) -> Stats:
        s = Stats()
        self._chk(self.L.minigpt4_b200_stats(ctx.ptr, C.byref(s)))
        return s

    def encode_array(self, ctx, image: np.ndarray) -> np.ndarray:
        """encode a float32 CHW [3,224,224] array through minigpt4_encode_image; returns [32, n_embd] and frees the C buffer"""
        img = np.ascontiguousarray(image, np.float32)
        mi = MiniGPT4Image(img.ctypes.data_as(C.c_void_p), 224, 224, 3, ImageFormat.F32)
        emb = self.base.minigpt4_encode_image(ctx, mi)
        n = emb.n_embeddings
        out = np.ctypeslib.as_array(emb.data, shape=(n,)).copy().reshape(32, n // 32)
        self.base.minigpt4_free_embedding(emb)
        return out

    def encode_batch(self, ctx, images: list) -> tuple[list, float]:
        """encode float32 CHW [3,224,224] arrays through minigpt4_b200_encode_images (concurrent lanes over shared weights);
        returns ([32, n_embd] arrays, wall ms of the call) and frees the C buffers"""
        import time
        imgs = [np.ascontiguousarray(im, np.float32) for im in images]
        arr = (MiniGPT4Image * len(imgs))(*[MiniGPT4Image(im.ctypes.data_as(C.c_void_p), 224, 224, 3, ImageFormat.F32) for im in imgs])
        embs = (MiniGPT4Embedding * len(imgs))()
        ins, outs = MiniGPT4Images(arr, len(imgs)), MiniGPT4Embeddings(embs, len(imgs))
        t0 = time.perf_counter()
        self._chk(self.L.minigpt4_b200_encode_images(ctx.ptr, C.byref(ins), C.byref(outs)))
        ms = (time.perf_counter() - t0) * 1e3
        res = []
        for e in embs:
            n = e.n_embeddings
            res.append(np.ctypeslib.as_array(e.data, shape=(n,)).copy().reshape(32, n // 32))
            self.base.minigpt4_free_embedding(e)
        return res, ms

    # host-only seams (no GPU)
    def host_tokenize(self, llm_path: str, text: str | bytes, add_bos: bool = True) -> list[int]:
        b = text.encode() if isinstance(text, str) else text
        buf = np.zeros(len(b) + 2, np.int32)
        n = self.L.minigpt4_b200_host_tokenize(llm_path.encode(), b, int(add_bos), _ptr(buf), buf.size)
        assert n >= 0, n
        return buf[:n].tolist()

    def host_sample(self, logits: np.ndarray, seed: int, n_draws: int = 1, temp=0.8, top_k=40, top_p=0.9, tfs_z=1.0, typical_p=1.0,
                    mirostat=0, mirostat_tau=5.0, mirostat_eta=1.0) -> np.ndarray:
        lg = np.ascontiguousarray(logits, np.float32)
        out = np.zeros(n_draws, np.int32)
        self._chk(self.L.minigpt4_b200_host_sample(_ptr(lg), lg.size, seed, temp, top_k, top_p, tfs_z, typical_p, mirostat, mirostat_tau, mirostat_eta, n_draws, _ptr(out)))
        return out

    # kernel seams
    def op_sample(self, logits: np.ndarray, seed: int, n_draws: int = 1, temp=0.8, top_k=40, top_p=0.9, tfs_z=1.0, typical_p=1.0,
                  timed: bool = False):
        """the device twin of host_sample (no mirostat, temp > 0); timed: also the average ms of one sampling launch"""
        lg = np.ascontiguousarray(logits, np.float32)
        out = np.zeros(n_draws, np.int32)
        ms = C.c_float(0)
        self._chk(self.L.minigpt4_b200_op_sample_timed(_ptr(lg), lg.size, seed, temp, top_k, top_p, tfs_z, typical_p, n_draws, _ptr(out), C.byref(ms)))
        return (out, ms.value) if timed else out

    def op_reply_stop(self, ctx, ids, stop: str | bytes | None = None, tail: str | bytes = b"") -> int:
        """sample_until's stop rule on the device over `ids` from a reply ending with `tail`: the index of the id that ends the reply, -1 if none"""
        a = np.ascontiguousarray(ids, np.int32)
        at = C.c_int32(0)
        st = stop.encode() if isinstance(stop, str) else stop
        tl = tail.encode() if isinstance(tail, str) else tail
        self._chk(self.L.minigpt4_b200_op_reply_stop(ctx.ptr, _ptr(a), a.size, st, tl, C.byref(at)))
        return at.value

    def op_check_libm(self, fn: int, lo_bits: int, hi_bits: int) -> int:
        """device expf (fn 0) / logf (fn 1) against the host libm over the float bit patterns lo_bits..hi_bits; returns the mismatches"""
        bad = C.c_longlong(0)
        self._chk(self.L.minigpt4_b200_op_check_libm(fn, lo_bits, hi_bits, C.byref(bad)))
        return bad.value

    def op_check_log2f(self, lo_bits: int, hi_bits: int) -> int:
        """device log2f against the host libm over the float bit patterns lo_bits..hi_bits; returns the mismatches"""
        bad = C.c_longlong(0)
        self._chk(self.L.minigpt4_b200_op_check_log2f(lo_bits, hi_bits, C.byref(bad)))
        return bad.value

    def op_check_powf(self, x: float, lo_bits: int, hi_bits: int) -> int:
        """device powf(x, y) against the host libm for the y of the float bit patterns lo_bits..hi_bits; returns the mismatches"""
        bad = C.c_longlong(0)
        self._chk(self.L.minigpt4_b200_op_check_powf(x, lo_bits, hi_bits, C.byref(bad)))
        return bad.value

    def op_sample_mirostat(self, logits: np.ndarray, seed: int, n_draws: int = 1, temp=0.8, mirostat=1, mirostat_tau=5.0, mirostat_eta=1.0,
                           on_device: bool = True, timed: bool = False):
        """mirostat draws over the same logits from one generator and an unset μ, by the device kernel or (on_device False) the host
        Sampler: (ids, μ after each draw), and with timed the average ms of one sampling launch"""
        lg = np.ascontiguousarray(logits, np.float32)
        ids, mu = np.zeros(n_draws, np.int32), np.zeros(n_draws, np.float32)
        ms = C.c_float(0)
        self._chk(self.L.minigpt4_b200_op_sample_mirostat(_ptr(lg), lg.size, seed, temp, mirostat, mirostat_tau, mirostat_eta, n_draws, int(on_device),
                                                          _ptr(ids), _ptr(mu), C.byref(ms)))
        return (ids, mu, ms.value) if timed else (ids, mu)

    def op_matvec(self, gtype: int, w_raw: np.ndarray, rows: int, cols: int, x: np.ndarray) -> np.ndarray:
        x = np.ascontiguousarray(x, np.float32).reshape(-1, cols)
        w = np.ascontiguousarray(w_raw)
        y = np.zeros((x.shape[0], rows), np.float32)
        self._chk(self.L.minigpt4_b200_op_matvec(gtype, rows, cols, _ptr(w), _ptr(x), x.shape[0], _ptr(y)))
        return y

    def op_gemm_f16(self, w: np.ndarray, x: np.ndarray, bias: Optional[np.ndarray], epi: int = 0, aux: Optional[np.ndarray] = None,
                    qscale: float = 1.0, qscale_rows: int = 0, ksplit: int = 1, tsplit: bool = True, in_place: bool = False,
                    out: Optional[np.ndarray] = None, plan: bool = False):
        """minigpt4_b200_op_gemm_f16: w float16 [M, K], x float16 [T, K].  out: the pre-filled buffer [ksplit, T + 1 + (epi == 4), M] (float16
        for epi 2, float32 otherwise; default zeros), returned whole; plain epilogues without split-K return its first T rows (rows 1..T for
        epi 4) as before.  plan: also return (token tile, grid.y, grid.z, k-blocks per slice)."""
        w = np.ascontiguousarray(w, np.float16); x = np.ascontiguousarray(x, np.float16)
        M, K = w.shape
        T = x.shape[0]
        b = None if bias is None else np.ascontiguousarray(bias, np.float32)
        a = None if aux is None else np.ascontiguousarray(aux, np.float32)
        whole = out is not None
        if out is None:
            out = np.zeros((ksplit, T + 1 + (epi == 4), M), np.float16 if epi == 2 else np.float32)
        assert out.flags.c_contiguous and out.shape == (ksplit, T + 1 + (epi == 4), M) and out.dtype == (np.float16 if epi == 2 else np.float32)
        pl = np.zeros(4, np.int32)
        self._chk(self.L.minigpt4_b200_op_gemm_f16(M, T, K, _ptr(w), _ptr(x), _ptr(b), epi, _ptr(a), qscale, qscale_rows, ksplit, int(tsplit),
                                                   int(in_place), _ptr(out), _ptr(pl)))
        res = out if whole else out[0, (1 if epi == 4 else 0):(T + 1 if epi == 4 else T)].astype(np.float32)
        return (res, tuple(int(v) for v in pl)) if plan else res

    def op_gemm_f16_rc(self, M: int, T: int, K: int, epi: int = 0, ksplit: int = 1, aux: bool = True, in_place: bool = False) -> int:
        """the return code of minigpt4_b200_op_gemm_f16 for a shape / configuration, with zero operands of that shape (refusals do no device work)"""
        n = max(1, M * K), max(1, T * K)
        w, x = np.zeros(n[0], np.float16), np.zeros(n[1], np.float16)
        a = np.zeros(max(1, (T + 1) * M), np.float32) if aux else None
        out = np.zeros(max(1, ksplit * (T + 2) * M), np.float32)
        return self.L.minigpt4_b200_op_gemm_f16(M, T, K, _ptr(w), _ptr(x), None, epi, _ptr(a), 1.0, 0, ksplit, 1, int(in_place), _ptr(out), None)

    def op_layernorm(self, x, w, b, f16: bool = False, f32: bool = True):
        """float32 [rows, n] -> the F32 output, the F16 one, or (F32, F16) when both are asked for (one launch writes both)"""
        x = np.ascontiguousarray(x, np.float32); w = np.ascontiguousarray(w, np.float32)
        b = None if b is None else np.ascontiguousarray(b, np.float32)
        o32 = np.empty_like(x) if f32 else None
        o16 = np.empty(x.shape, np.float16) if f16 else None
        self._chk(self.L.minigpt4_b200_op_layernorm(_ptr(x), x.shape[0], x.shape[1], _ptr(w), _ptr(b), _ptr(o32), _ptr(o16)))
        return (o32, o16) if f32 and f16 else (o32 if f32 else o16)

    def op_layernorm_rc(self, rows: int, n: int) -> int:
        x = np.zeros(max(1, rows * n), np.float32); w = np.zeros(max(1, n), np.float32); o = np.zeros_like(x)
        return self.L.minigpt4_b200_op_layernorm(_ptr(x), rows, n, _ptr(w), None, _ptr(o), None)

    def op_layernorm_fold(self, x, parts, w, b) -> tuple[np.ndarray, np.ndarray]:
        """x float32 [rows, n], parts float32 [n_parts, rows, n] -> (x + parts[0] + parts[1] + ... in slice order, F16 LayerNorm of it)"""
        x = np.array(x, np.float32, order="C"); p = np.ascontiguousarray(parts, np.float32)
        w = np.ascontiguousarray(w, np.float32); b = None if b is None else np.ascontiguousarray(b, np.float32)
        o16 = np.empty(x.shape, np.float16)
        self._chk(self.L.minigpt4_b200_op_layernorm_fold(_ptr(x), x.shape[0], x.shape[1], _ptr(w), _ptr(b), _ptr(p), p.shape[0], x.size, _ptr(o16)))
        return x, o16

    def encode_taps(self, ctx, image: np.ndarray, n_blocks: int, q_layers: int, n_embd_llm: int, d: int = 1408) -> dict:
        """every stage of the encode of `image` on ctx (whose vision model has n_blocks ViT blocks and q_layers Q-Former layers): embed [257, d],
        vit_blocks [n_blocks, 257, d], ln_vision [257, d], qformer [q_layers, 32, 768], out [32, n_embd_llm]"""
        img = np.ascontiguousarray(image, np.float32)
        r = {"embed": np.zeros((257, d), np.float32), "vit_blocks": np.zeros((n_blocks, 257, d), np.float32),
             "ln_vision": np.zeros((257, d), np.float32), "qformer": np.zeros((q_layers, 32, 768), np.float32),
             "out": np.zeros((32, n_embd_llm), np.float32)}
        self._chk(self.L.minigpt4_b200_encode_taps(ctx.ptr, _ptr(img), _ptr(r["embed"]), _ptr(r["vit_blocks"]), _ptr(r["ln_vision"]),
                                                   _ptr(r["qformer"]), _ptr(r["out"])))
        return r

    def op_dequant_f16(self, gtype: int, raw: np.ndarray, n: int) -> np.ndarray:
        raw = np.ascontiguousarray(raw)
        out = np.zeros(n, np.float16)
        self._chk(self.L.minigpt4_b200_op_dequant_f16(gtype, _ptr(raw), n, _ptr(out)))
        return out

    def host_quantize_row(self, gtype: int, x: np.ndarray) -> np.ndarray:
        x = np.ascontiguousarray(x, np.float32).reshape(-1)
        out = np.zeros(x.size // 32 * 40, np.uint8)
        nb = self.L.minigpt4_b200_host_quantize_row(gtype, _ptr(x), x.size, _ptr(out))
        assert nb >= 0, "unsupported quantisation type"
        return out[:nb].copy()

    def op_attention(self, q, k, v, heads: int, dh: int, div: float) -> np.ndarray:
        """q [nq][heads * dh], k / v [nk][heads * dh] float32 -> the attention output [nq][heads * dh] (F16 precision), ceil(nq / 4) queries per CTA"""
        q = np.ascontiguousarray(q, np.float32); k = np.ascontiguousarray(k, np.float32); v = np.ascontiguousarray(v, np.float32)
        nq, nk, ld = q.shape[0], k.shape[0], heads * dh
        buf = np.concatenate([q.reshape(-1), k.reshape(-1), v.reshape(-1)])
        return self.op_attention_packed(buf, 0, ld, nq * ld, (nq + nk) * ld, ld, nq, nk, heads, dh, div)[:nq]

    def op_attention_packed(self, buf, q_off: int, ldq: int, k_off: int, v_off: int, ldkv: int, nq: int, nk: int, heads: int, dh: int,
                            div: float, q_per_cta: int = 0, ld_out: Optional[int] = None, out: Optional[np.ndarray] = None) -> np.ndarray:
        """minigpt4_b200_op_attention over one float32 buffer with q / k / v at element offsets and row pitches (as the vision graph passes its
        packed qkv outputs).  out: the pre-filled [nq + 1, ld_out] float32 buffer (default zeros), returned whole"""
        buf = np.ascontiguousarray(buf, np.float32).reshape(-1)
        ld_out = heads * dh if ld_out is None else ld_out
        if out is None:
            out = np.zeros((nq + 1, ld_out), np.float32)
        assert out.flags.c_contiguous and out.shape == (nq + 1, ld_out) and out.dtype == np.float32
        self._chk(self.L.minigpt4_b200_op_attention(_ptr(buf), buf.size, q_off, ldq, k_off, v_off, ldkv, nq, nk, heads, dh, div, q_per_cta, ld_out,
                                                    _ptr(out)))
        return out

    def op_attention_rc(self, nq: int, nk: int, heads: int, dh: int) -> int:
        ld = heads * dh
        buf = np.zeros((nq + 2 * nk) * ld, np.float32); out = np.zeros((nq + 1) * ld, np.float32)
        return self.L.minigpt4_b200_op_attention(_ptr(buf), buf.size, 0, ld, nq * ld, (nq + nk) * ld, ld, nq, nk, heads, dh, 1.0, 0, ld, _ptr(out))

    def op_llama_attention(self, q, k, v, pos, path: int) -> np.ndarray:
        """q float32 [rows][n_head * 128], k / v float16 [n_ctx][n_head * 128]; path 0: row t at pos[0] + t (pos may be one int), path 1:
        row t at pos[t]"""
        q = np.ascontiguousarray(q, np.float32)
        k = np.ascontiguousarray(k, np.float16); v = np.ascontiguousarray(v, np.float16)
        rows = q.shape[0]
        pos = np.full(rows, pos, np.int32) if np.ndim(pos) == 0 else np.ascontiguousarray(pos, np.int32)
        out = np.zeros_like(q)
        self._chk(self.L.minigpt4_b200_op_llama_attention(_ptr(q), _ptr(k), _ptr(v), k.shape[1] // 128, k.shape[0], rows, _ptr(pos), path, _ptr(out)))
        return out


class MiniGPT4ChatBot:
    """Chat driver with the reference's surface (reference minigpt4_library.py:568-689): generate() streams tokens,
    upload_image() encodes an image (PIL image -> torchvision transform like the reference, a file path -> the library's own decoder and
    Pillow-exact preprocess, or a ready float32 CHW array)."""

    def __init__(self, model_path: str, llm_model_path: str, verbosity: Verbosity = Verbosity.SILENT, n_threads: int = 0):
        self.library = load_library()
        self.ctx = self.library.minigpt4_model_load(model_path, llm_model_path, verbosity)
        self.n_threads = n_threads
        self.image_size = 224
        self.embedding: Optional[MiniGPT4Embedding] = None
        self.is_image_chat = False
        self.chat_history = []
        self._keep = None

    def free(self):
        for c in getattr(self, "_beams", []):
            self.library.minigpt4_free(c)
        self._beams = []
        if self.ctx and self.ctx.ptr:
            self.library.minigpt4_free(self.ctx)

    def _preprocess(self, image) -> np.ndarray:
        if isinstance(image, np.ndarray):
            return np.ascontiguousarray(image, np.float32).reshape(1, 3, 224, 224)
        if isinstance(image, (str, os.PathLike)):   # a file: the library's own decode + deterministic preprocess (examples/main.cpp's path)
            raw = self.library.minigpt4_image_load_from_file(self.ctx, os.fspath(image), 0)
            pre = self.library.minigpt4_preprocess_image(self.ctx, raw, 0)
            arr = np.ctypeslib.as_array(C.cast(pre.data, C.POINTER(C.c_float)), shape=(1, 3, 224, 224)).copy()
            self.library.minigpt4_free_image(raw); self.library.minigpt4_free_image(pre)
            return arr
        from torchvision import transforms
        from torchvision.transforms.functional import InterpolationMode
        tf = transforms.Compose([transforms.RandomResizedCrop(self.image_size, interpolation=InterpolationMode.BICUBIC), transforms.ToTensor(),
                                 transforms.Normalize((0.48145466, 0.4578275, 0.40821073), (0.26862954, 0.26130258, 0.27577711))])
        return tf(image).unsqueeze(0).numpy()

    def generate(self, message: str, limit: int = 1024, temp: float = 0.8, top_k: int = 40, top_p: float = 0.9, tfs_z: float = 1.0,
                 typical_p: float = 1.0, repeat_last_n: int = 64, repeat_penalty: float = 1.1, alpha_presence: float = 1.0,
                 alpha_frequency: float = 1.0, mirostat: int = 0, mirostat_tau: float = 5.0, mirostat_eta: float = 1.0, penalize_nl: int = 1):
        if self.is_image_chat:
            self.is_image_chat = False
            self.library.minigpt4_begin_chat_image(self.ctx, self.embedding, message, self.n_threads)
            step = self.library.minigpt4_end_chat_image
        else:
            self.library.minigpt4_begin_chat(self.ctx, message, self.n_threads)
            step = self.library.minigpt4_end_chat
        chat = ""
        for _ in range(limit):
            token = step(self.ctx, self.n_threads, temp, top_k, top_p, tfs_z, typical_p, repeat_last_n, repeat_penalty, alpha_presence,
                         alpha_frequency, mirostat, mirostat_tau, mirostat_eta, penalize_nl)
            chat += token
            if self.library.minigpt4_contains_eos_token(token):
                continue
            if self.library.minigpt4_is_eos(chat):
                break
            yield token

    def generate_on_device(self, message: str, limit: int = 1024, chunk: int = 16, temp: float = 0.8, top_k: int = 40, top_p: float = 0.9,
                           tfs_z: float = 1.0, typical_p: float = 1.0, mirostat: int = 0, mirostat_tau: float = 5.0, mirostat_eta: float = 1.0,
                           constraint: Optional[int] = None, repeat_last_n: int = 64, repeat_penalty: float = 1.0, alpha_presence: float = 0.0,
                           alpha_frequency: float = 0.0, penalize_nl: int = 1):
        """generate() with the sampling and the stop check on the GPU: minigpt4_b200_sample_until (mirostat 1 / 2: _mirostat) calls of up
        to `chunk` steps, each stopping where generate()'s loop stops.
        Yields what generate() yields for the same seed: no "##" token, and not the token that completes "###".

        The repetition arguments default to neutral values (repeat_penalty 1.0, alphas 0.0), and then the calls above are issued exactly,
        as generate() ignores them.  Otherwise every chunk is a minigpt4_b200_sample_until_penalized call whose history is the ids of this
        reply from the earlier chunks, so the penalties see the last repeat_last_n ids of the reply and a chunked reply equals one call; it
        yields what a loop of minigpt4_b200_end_chat_penalized over the same history yields (repeat_penalty 1.1 is the reference web UI's
        slider default, which generate() does not apply).

        One difference cannot be avoided: generate() decodes each token's bytes with errors="ignore" before it appends and checks them,
        so a piece that is not valid UTF-8 on its own drops out of its reply text, while the device compares the bytes.  The two can
        disagree only where such a piece sits inside or next to the stop text.

        constraint: a handle of B200.constraint_create (or None): the reply is drawn from the ids the automaton allows (no mirostat) and
        also ends after </s>, which is not yielded.  It is attached for this reply only."""
        ext = B200(self.library)
        pen = None
        if repeat_last_n != 0 and (repeat_penalty != 1.0 or alpha_presence != 0.0 or alpha_frequency != 0.0):
            pen = dict(repeat_last_n=repeat_last_n, repeat_penalty=repeat_penalty, alpha_presence=alpha_presence, alpha_frequency=alpha_frequency,
                       penalize_nl=penalize_nl)
        if constraint is None:
            yield from self._generate_on_device(ext, message, limit, chunk, temp, top_k, top_p, tfs_z, typical_p, mirostat, mirostat_tau,
                                                mirostat_eta, pen=pen)
            return
        ext.constraint_attach(self.ctx, constraint)
        try:
            yield from self._generate_on_device(ext, message, limit, chunk, temp, top_k, top_p, tfs_z, typical_p, mirostat, mirostat_tau,
                                                mirostat_eta, pen=pen)
        finally:
            ext.constraint_attach(self.ctx, None)

    def generate_with_logprobs(self, message: str, top_n: int = 5, limit: int = 1024, chunk: int = 16, temp: float = 0.8, top_k: int = 40,
                               top_p: float = 0.9, tfs_z: float = 1.0, typical_p: float = 1.0, mirostat: int = 0, mirostat_tau: float = 5.0,
                               mirostat_eta: float = 1.0, constraint: Optional[int] = None):
        """generate_on_device() that yields (token, logprob, [(alt_token, alt_logprob), ...]) for exactly the tokens generate_on_device
        yields with the same seed and arguments, through minigpt4_b200_sample_until_logprobs: the token's log-probability under the model's
        raw distribution at that step (temperature 1, no sampling cut or constraint), and the top_n (0..20) most likely tokens there."""
        ext = B200(self.library)
        if constraint is None:
            yield from self._generate_on_device(ext, message, limit, chunk, temp, top_k, top_p, tfs_z, typical_p, mirostat, mirostat_tau,
                                                mirostat_eta, top_n)
            return
        ext.constraint_attach(self.ctx, constraint)
        try:
            yield from self._generate_on_device(ext, message, limit, chunk, temp, top_k, top_p, tfs_z, typical_p, mirostat, mirostat_tau,
                                                mirostat_eta, top_n)
        finally:
            ext.constraint_attach(self.ctx, None)

    def _generate_on_device(self, ext, message, limit, chunk, temp, top_k, top_p, tfs_z, typical_p, mirostat, mirostat_tau, mirostat_eta,
                            top_n=None, pen=None):
        """the reply's tokens; with top_n (not None) each as (token, logprob, alternatives); pen (not None): the penalty arguments of
        sample_until_penalized, the reply's ids so far as the history"""
        if self.is_image_chat:
            self.is_image_chat = False
            self.library.minigpt4_begin_chat_image(self.ctx, self.embedding, message, self.n_threads)
        else:
            self.library.minigpt4_begin_chat(self.ctx, message, self.n_threads)

        def text(t):
            return ext.L.minigpt4_b200_token_text(self.ctx.ptr, int(t)).decode("utf-8", errors="ignore")
        done = 0
        reply = []
        while done < limit:
            steps = min(chunk, limit - done)
            if pen is not None:
                ids, stopped, _ = ext.sample_until_penalized([self.ctx], steps, None, [reply], temp=temp, top_k=top_k, top_p=top_p, tfs_z=tfs_z,
                                                             typical_p=typical_p, mirostat=mirostat, mirostat_tau=mirostat_tau,
                                                             mirostat_eta=mirostat_eta, **pen)
                reply += ids[0]
            elif top_n is None:
                ids, stopped, _ = ext.sample_until([self.ctx], steps, None, temp, top_k, top_p, tfs_z, typical_p, mirostat, mirostat_tau,
                                                   mirostat_eta)
            else:
                ids, stopped, recs, _ = ext.sample_until_logprobs([self.ctx], steps, None, top_n, temp, top_k, top_p, tfs_z, typical_p, mirostat,
                                                                  mirostat_tau, mirostat_eta)
            done += len(ids[0])
            for k, t in enumerate(ids[0]):
                if stopped[0] and k == len(ids[0]) - 1:
                    return
                token = text(t)
                if not self.library.minigpt4_contains_eos_token(token):
                    if top_n is None:
                        yield token
                    else:
                        lp, _, tid, tlp = recs[0]
                        yield token, float(lp[k]), [(text(a), float(b)) for a, b in zip(tid[k], tlp[k])]

    def generate_beam(self, message: str, num_beams: int = 4, limit: int = 1024, length_penalty: float = 1.0):
        """generate() with beam search on the GPU (minigpt4_b200_beam_search): the best of num_beams (1..16) beams, deterministic.  The
        num_beams - 1 working sessions are created on first use and kept.  Yields the best reply's tokens as generate_on_device does: no
        "##" token, and not the token that completes "###"."""
        ext = B200(self.library)
        if not hasattr(self, "_beams"):
            self._beams = []
        while len(self._beams) < num_beams - 1:
            self._beams.append(ext.session_create(self.ctx))
        if self.is_image_chat:
            self.is_image_chat = False
            self.library.minigpt4_begin_chat_image(self.ctx, self.embedding, message, self.n_threads)
        else:
            self.library.minigpt4_begin_chat(self.ctx, message, self.n_threads)
        steps = min(limit, self._room(ext))
        if steps < 1:   # the conversation fills the context: no reply
            return
        hyps, _ = ext.beam_search([self.ctx] + self._beams[:num_beams - 1], steps, None, length_penalty)
        ids, _, _, stopped = hyps[0]
        for k, t in enumerate(ids):
            if stopped and k == len(ids) - 1:
                return
            token = ext.L.minigpt4_b200_token_text(self.ctx.ptr, t).decode("utf-8", errors="ignore")
            if not self.library.minigpt4_contains_eos_token(token):
                yield token

    def _room(self, ext) -> int:
        """the positions left in the conversation (n_ctx - n_past, queued rows counted)"""
        return ext.stats(self.ctx).n_ctx - ext.n_past(self.ctx)

    def reset_chat(self):
        self.is_image_chat = False
        if self.embedding:
            self.library.minigpt4_free_embedding(self.embedding)
            self.embedding = None
        self.library.minigpt4_reset_chat(self.ctx)
        self.library.minigpt4_system_prompt(self.ctx, self.n_threads)

    def upload_image(self, image):
        self.reset_chat()
        arr = self._preprocess(image)
        self._keep = arr
        mi = MiniGPT4Image(arr.ctypes.data_as(C.c_void_p), self.image_size, self.image_size, 3, ImageFormat.F32)
        self.embedding = self.library.minigpt4_encode_image(self.ctx, mi, self.n_threads)
        self.is_image_chat = True
