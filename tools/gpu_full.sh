#!/bin/bash
# Full 1-GPU check-out on an H100: canary, GPU suite, prefill timing, bench (both arms), torch.profiler kernel tables, per-op trace, smoke.
# Logs go to $OUT (default: a fresh temporary directory, printed at the end).
OUT=${OUT:-$(mktemp -d)}
mkdir -p "$OUT"
run() { name=$1; shift; t=$1; shift; echo "=== $name"; timeout -k 5 $t "$@" > "$OUT/$name.log" 2>&1; rc=$?; echo "exit $rc"; tail -n ${TAILN:-12} "$OUT/$name.log"; return $rc; }
nvidia-smi --query-gpu=name,power.limit,clocks.max.sm --format=csv > "$OUT/gpu.csv"
TAILN=6 run canary6 300 python tools/canary.py || exit 1
TAILN=8 run pytest_gpu 1200 python -m pytest tests -m gpu -q -p no:cacheprovider
TAILN=3 run prefill_plain 300 python tools/prof_prefill.py
TAILN=3 run bench 600 python bench.py
TAILN=3 run bench_reference 600 python bench.py --impl reference --steps 2 --warmup 1
TAILN=40 run prof_decode 420 python tools/torch_prof.py tools/prof_decode.py
TAILN=40 run prof_turn 900 python tools/torch_prof.py tools/prof_turn.py
TAILN=30 run trace6 200 python tools/mega_trace.py
TAILN=2 run smoke 300 python -c "import __graft_entry__ as g; g.smoke()"
echo "done: logs in $OUT"
