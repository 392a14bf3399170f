"""Run one of the prof_*.py targets under torch.profiler (CUDA activities) and print the kernel table: time per kernel name over the
target's launches.  The library's kernels are launched through ctypes; the profiler sees them through CUPTI like any other CUDA work.

    python tools/torch_prof.py tools/prof_decode.py [args of the target ...]"""
import runpy
import sys

import torch
from torch.profiler import ProfilerActivity, profile

target, sys.argv = sys.argv[1], sys.argv[1:]
torch.cuda.init()
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    runpy.run_path(target, run_name="__main__")
    torch.cuda.synchronize()
print(prof.key_averages().table(sort_by="cuda_time_total", row_limit=40, max_name_column_width=90))
