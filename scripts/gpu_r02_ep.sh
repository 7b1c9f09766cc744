#!/bin/bash
# N GPUs: expert-parallel parity + S=4096 timing, then the bench with its ep record; logs under $OUT (default logs/)
N=${1:-2}
OUT=${OUT:-logs}
mkdir -p "$OUT"
TR="python -m torch.distributed.run --nnodes=1 --nproc-per-node $N --master-addr 127.0.0.1"
L=$([ "$N" -ge 8 ] && echo 32 || echo 8)
timeout 900 $TR --master-port 29541 tests/ep_check.py --layers 2 --seq 300 --time-seq 4096 --time-layers $L > $OUT/ep${N}.log 2>&1
echo "ep_check rc=$?" | tee -a $OUT/ep${N}.log; grep -E "EP x|bit-identical|Error|error" $OUT/ep${N}.log | tail -6 | cut -c1-300
timeout 1500 $TR --master-port 29543 bench.py --gpus $N --steps 2 --warmup 3 --no-parity > $OUT/bench_${N}gpu.json 2> $OUT/bench_${N}gpu.err
echo "bench rc=$?"; python - <<PY
import json
try:
    d = json.loads(open("$OUT/bench_${N}gpu.json").read().strip().splitlines()[-1])
    print("value", d["value"], "n_gpus", d["n_gpus"], "decode ms/tok", d["phases_ms"]["decode_per_token"])
    print("ep", json.dumps(d.get("ep"))[:1800])
except Exception as e:
    print("bench unreadable", e)
PY
tail -4 $OUT/bench_${N}gpu.err | cut -c1-300
