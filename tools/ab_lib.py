"""A/B timing of several builds of libminigpt4.so on the SAME GPU in one process (bisection of a decode regression): 7B-wide 4-layer Q4_1 model, 32-row prefix,
128 device-chained greedy tokens, best of 3.  Only the oldest C entry points are used.   python tools/ab_lib.py build/ab/libA.so build/ab/libB.so ..."""
import ctypes, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import bench
from minigpt4_cpp_b200 import modelgen as mg
llm = str(bench.model_dir() / "llama-7bwide-4l-v32000-q4_1.bin")
if not os.path.exists(llm):
    mg.write_llama_ggjt(llm, mg.LlamaSpec(wtype="q4_1", n_vocab=32000, n_embd=4096, n_head=32, n_layer=4))
rows = np.random.default_rng(0).standard_normal((32, 4096)).astype(np.float32)
for rnd in range(2):
    for path in sys.argv[1:]:
        lib = ctypes.CDLL(os.path.abspath(path))
        lib.minigpt4_b200_llm_load.restype = ctypes.c_void_p
        lib.minigpt4_b200_llm_load.argtypes = [ctypes.c_char_p, ctypes.c_int, ctypes.c_int, ctypes.c_int]
        lib.minigpt4_b200_eval_embd.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int]
        lib.minigpt4_b200_decode_chain.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.POINTER(ctypes.c_float)]
        lib.minigpt4_reset_chat.argtypes = [ctypes.c_void_p]
        lib.minigpt4_free.argtypes = [ctypes.c_void_p]
        ctx = lib.minigpt4_b200_llm_load(llm.encode(), 2048, 1337, 1)
        best = 1e9
        for _ in range(3):
            lib.minigpt4_reset_chat(ctx)
            lib.minigpt4_b200_eval_embd(ctx, rows.ctypes.data_as(ctypes.c_void_p), 32)
            ids = np.zeros(128, np.int32); ms = ctypes.c_float(0)
            lib.minigpt4_b200_decode_chain(ctx, 128, ids.ctypes.data_as(ctypes.c_void_p), ctypes.byref(ms))
            best = min(best, ms.value / 128)
        print(f"round {rnd} {os.path.basename(path)}: {best * 1e3:.2f} us/token  ids[:4] {ids[:4].tolist()}", flush=True)
        lib.minigpt4_free(ctx)
