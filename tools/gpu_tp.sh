#!/bin/bash
# Tensor-parallel check-out on N GPUs of one machine:   bash tools/gpu_tp.sh 2 [check]      (logs go to $OUT, default a temporary directory)
N=${1:-2}
OUT=${OUT:-$(mktemp -d)}
mkdir -p "$OUT"
run() { name=$1; shift; t=$1; shift; echo "=== $name"; timeout -k 5 $t "$@" > "$OUT/$name.log" 2>&1; rc=$?; echo "exit $rc"; tail -n ${TAILN:-12} "$OUT/$name.log"; return $rc; }
TR="python -m torch.distributed.run --nnodes=1 --nproc-per-node $N --master-addr 127.0.0.1"
if [ "$2" = "check" ]; then TAILN=6 run tp_check_$N 400 $TR --master-port 29511 tools/tp_check.py; fi
# bench.py's command line for N > 1 (replicas + the tp sub-record)
TAILN=4 run bench_dp_tp_$N 600 $TR --master-port 29512 bench.py --gpus $N --steps 2 --warmup 1 --no-cpu
echo "done: logs in $OUT"
