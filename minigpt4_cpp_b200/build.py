"""Build libminigpt4.so for sm_90a with nvcc (in-tree; output build/libminigpt4.so, where the reference's
ctypes loader looks: reference minigpt4/minigpt4_library.py:539-566)."""
from __future__ import annotations

import fcntl
import hashlib
import os
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
CSRC = Path(__file__).resolve().parent / "csrc"
OUT = ROOT / "build" / "libminigpt4.so"
SOURCES = ["llama.cu", "vision.cu", "api.cpp", "engine.cpp", "formats.cpp", "text.cpp", "tp.cpp", "quantize.cpp", "image.cpp", "jpeg.cpp"]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
# -fmad=false / -ffp-contract=off: no implicit FMA contraction — float expressions evaluate exactly as written so the
# language path is bit-identical to the CPU oracle's canonical reduction order (see oracle/oracle.cpp header)
FLAGS = ["-ccbin", "/usr/bin/g++", "-std=c++17", "-O3", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-fmad=false",
         "-Xcompiler", "-fPIC,-fvisibility=hidden,-Wall,-Wno-unused-function,-Wno-class-memaccess,-ffp-contract=off", "-I", str(ROOT / "include")]


def _digest() -> str:
    h = hashlib.sha256()
    for p in sorted(list(CSRC.glob("*")) + list((ROOT / "include").glob("*.h"))):
        h.update(p.name.encode())
        h.update(p.read_bytes())
    h.update(" ".join(FLAGS).encode())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False) -> Path:
    stamp = OUT.with_suffix(".stamp")
    dig = _digest()
    if not force and OUT.exists() and stamp.exists() and stamp.read_text() == dig:
        return OUT
    OUT.parent.mkdir(parents=True, exist_ok=True)
    # several ranks of one torchrun may get here together: one builds (into private object names, the .so is renamed into place), the others wait
    with open(OUT.parent / ".build.lock", "w") as lock:
        fcntl.flock(lock, fcntl.LOCK_EX)
        if not force and OUT.exists() and stamp.exists() and stamp.read_text() == dig:
            return OUT
        objs = []
        procs = []
        for s in SOURCES:
            o = OUT.parent / (s + ".o")
            cmd = [NVCC, *FLAGS, "-x", "cu", "-c", str(CSRC / s), "-o", str(o)]
            if verbose:
                print(" ".join(cmd))
            procs.append((s, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
            objs.append(str(o))
        failed = False
        for s, p in procs:
            out, _ = p.communicate()
            if p.returncode != 0:
                failed = True
                sys.stderr.write(f"--- nvcc failed on {s} ---\n{out}\n")
            elif verbose and out.strip():
                print(out)
        if failed:
            raise RuntimeError("libminigpt4.so: compilation failed")
        tmp = OUT.with_suffix(f".so.tmp{os.getpid()}")
        link = [NVCC, "-ccbin", "/usr/bin/g++", "-shared", "-o", str(tmp), *objs, "-gencode", "arch=compute_90a,code=sm_90a",
                "-Xlinker", "--no-undefined", "-ldl", "-lpthread", "-cudart", "static"]
        r = subprocess.run(link, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        if r.returncode != 0:
            raise RuntimeError("libminigpt4.so: link failed\n" + r.stdout)
        os.replace(tmp, OUT)
        stamp.write_text(dig)
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
