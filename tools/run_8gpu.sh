#!/bin/bash
# one N-GPU visit: [G == 1 check,] weak-scaling bench line, strong-scaling (configs[4] shape) bench line
#   bash tools/run_8gpu.sh 8 [nocheck]        (logs and JSON lines go to $OUT, default: a new temporary directory)
OUT=${OUT:-$(mktemp -d)}
mkdir -p "$OUT"
echo "output: $OUT"
N=${1:-8}
TR="python -m torch.distributed.run --nnodes=1 --nproc-per-node $N --master-addr 127.0.0.1"
if [ "${2:-}" != nocheck ]; then
  timeout 120 $TR --master-port 29521 tools/check_multi_gpu.py > "$OUT/mgpu_check_n$N.log" 2>&1; grep '"check"' "$OUT/mgpu_check_n$N.log" | cut -c1-200
fi
timeout 120 $TR --master-port 29522 bench.py --gpus $N --steps 60 --warmup 5 > "$OUT/bench_weak_n$N.json" 2> "$OUT/bench_weak_n$N.err"; tail -1 "$OUT/bench_weak_n$N.json" | cut -c1-250
timeout 200 $TR --master-port 29523 bench.py --gpus $N --steps 30 --warmup 5 --total-meshlets 50000000 > "$OUT/bench_strong50M_n$N.json" 2> "$OUT/bench_strong50M_n$N.err"; tail -1 "$OUT/bench_strong50M_n$N.json" | cut -c1-250
