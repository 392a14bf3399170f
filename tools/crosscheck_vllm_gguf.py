"""Cross-check (needs a GPU and vLLM; NOT part of the test suite, never on the product path): pin the oracle's restatement of ggml's
quantised mul_mat against kernels that DESCEND from ggml itself.  vLLM (library code in this image) ships llama.cpp's CUDA MMVQ /
dequantise kernels as `torch.ops._C.ggml_mul_mat_vec_a8` / `ggml_dequantize`: activations quantised to q8_1, integer block dots,
the block layouts of ggml — i.e. the arithmetic this repo could only restate from memory ("parity unpinned", DESIGN.md §2).

Prints, per block type, (a) dequantiser: vLLM vs oracle, expected exact after rounding to F16; (b) matvec: vLLM vs oracle vs this repo's
CUDA kernel.  ggml-cuda's q8_1 keeps d and s as halves and reduces in another order, so (b) agrees to ~1e-3 relative, not bit for bit;
a layout or formula error (nibble order, the `- 8`, the m * s term, the K-quant scale packing) would show up as O(1).

    python tools/crosscheck_vllm_gguf.py            # on a machine with an H100 and vLLM installed
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main() -> int:
    import torch
    from vllm import _custom_ops as ops  # noqa: F401  (registers torch.ops._C.ggml_*)
    import minigpt4_cpp_b200 as m
    from minigpt4_cpp_b200 import modelgen as mg
    from oracle import oracle as orc

    lib = m.load_library()
    ext = m.B200(lib)
    rng = np.random.default_rng(0)
    rows, cols = 256, 4096
    worst = 0.0
    for name, gt in (("q4_0", 2), ("q4_1", 3), ("q5_k", 13), ("q6_k", 14)):
        raw = mg.synth_quant(rng, gt, rows, cols, 0.02)            # [rows][row_bytes] uint8, ggml block layout
        w_dev = torch.from_numpy(np.ascontiguousarray(raw).reshape(rows, -1)).cuda()
        deq = ops.ggml_dequantize(w_dev, gt, rows, cols, torch.float16).float().cpu().numpy()
        ref = orc.dequant_rows(gt, raw, rows, cols)
        e_deq = float(np.abs(deq - ref.astype(np.float16).astype(np.float32)).max())
        x = rng.standard_normal((1, cols)).astype(np.float32)
        y_vllm = ops.ggml_mul_mat_vec_a8(w_dev, torch.from_numpy(x).cuda().half(), gt, rows).float().cpu().numpy().reshape(-1)
        y_orc = orc.mul_mat(gt, raw, rows, cols, x).reshape(-1)
        y_ours = ext.op_matvec(gt, raw, rows, cols, x).reshape(-1)
        rel = lambda a, b: float(np.abs(a - b).max() / (np.abs(b).max() + 1e-30))
        print(f"{name}: dequant max |vllm - oracle(f16)| = {e_deq:.3e};  matvec rel err  vllm vs oracle {rel(y_vllm, y_orc):.3e},"
              f"  ours vs oracle {rel(y_ours, y_orc):.3e} (bit-identical: {bool(np.array_equal(y_ours, y_orc))})")
        worst = max(worst, rel(y_vllm, y_orc))
    print("worst vllm-vs-oracle matvec rel err:", worst, "(expect ~1e-3: half-precision activations / q8_1 scales in ggml-cuda)")
    return 0 if worst < 2e-2 else 1


if __name__ == "__main__":
    sys.exit(main())
