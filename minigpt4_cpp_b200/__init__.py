"""minigpt4.cpp_b200 — H100-native engine behind the minigpt4.h C ABI (hot path only: the vision graph behind
minigpt4_encode_image and the LLaMA step behind llama_eval).  The compute lives in build/libminigpt4.so (C++ host +
hand-written sm_90a CUDA); this package holds the host-side mirror of the reference's ctypes interface, the builder
and the synthetic-weight generators."""
from .minigpt4_library import (B200, DataType, ImageFormat, MiniGPT4ChatBot, MiniGPT4Context, MiniGPT4Embedding, MiniGPT4Image,  # noqa: F401
                               MiniGPT4SharedLibrary, Verbosity, choices_dfa, load_library, library_path)
