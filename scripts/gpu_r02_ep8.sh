#!/bin/bash
# 8 GPUs: sequence-sharded expert-parallel prefill at full depth: parity at small S + S=4096 timing (32 layers);
# logs under $OUT (default logs/)
N=8
OUT=${OUT:-logs}
mkdir -p "$OUT"
TR="python -m torch.distributed.run --nnodes=1 --nproc-per-node $N --master-addr 127.0.0.1"
timeout 600 $TR --master-port 29541 tests/ep_check.py --layers 2 --seq 301 --time-seq 4096 --time-layers 32 > $OUT/ep${N}.log 2>&1
echo "ep_check rc=$?" | tee -a $OUT/ep${N}.log; grep -E "EP x|bit-identical|Error" $OUT/ep${N}.log | tail -6 | cut -c1-300
