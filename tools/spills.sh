#!/bin/bash
# ptxas register / spill report (CPU-only check before spending GPU time).  Usage: [SRC=vision.cu] tools/spills.sh
# Prints every function that has a stack frame or spills, and the register count of every kernel whose name matches $1 (default: all).
# Exits non-zero (and shows the compiler output) when nvcc fails.
cd "$(dirname "$0")/.."
set -o pipefail
tmp=$(mktemp -d); trap 'rm -rf "$tmp"' EXIT
if ! ${NVCC:-/usr/local/cuda/bin/nvcc} -ccbin /usr/bin/g++ -std=c++17 -O3 -gencode arch=compute_90a,code=sm_90a -lineinfo -fmad=false \
  -Xcompiler -fPIC,-ffp-contract=off -I include -Xptxas -v -x cu -c minigpt4_cpp_b200/csrc/${SRC:-llama.cu} -o "$tmp/spills_check.o" > "$tmp/log" 2>&1; then
  cat "$tmp/log"; echo "spills.sh: nvcc failed on ${SRC:-llama.cu}" >&2; exit 1
fi
python3 -c '
import re, sys
pat = re.compile(sys.argv[1] if len(sys.argv) > 1 else ".")
fn = None; clean = 0
for line in sys.stdin:
    m = re.search(r"Function properties for (\S+)", line)
    if m: fn = m.group(1); continue
    m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
    if m and fn:
        if any(int(x) for x in m.groups()): print("SPILL/STACK", fn[:90], line.strip())
        else: clean += 1
        continue
    m = re.search(r"Used (\d+) registers", line)
    if m and fn and pat.search(fn): print(f"{m.group(1):>4} regs  {fn[:110]}")
print(clean, "functions without stack frame or spills")
' "$@" < "$tmp/log"
