#!/bin/bash
# Tuning pass on an N-GPU machine (device-timed, CUDA-graph replayed).
set -x
W=${1:-8}
S="python scripts/bw_sweep.py --world $W"
# NVLS reduce phase in isolation (operands in the symmetric heap): CTA count
timeout 120 $S --symm --algos nvls --nvls-ctas 32,64,100,148 --min 67108864 --max 268435456 --step 4
# staged tensors: whole-grid CTA barriers (default) vs decoupled reduce phase
timeout 120 $S --algos nvls --nvls-ctas -1,64 --min 67108864 --max 1073741824 --step 4
# LL vs one-shot vs two-shot break-even
timeout 120 $S --algos ll,oneshot,twoshot --min 64 --max 1048576 --step 4
# the other collectives and the fused gradient kernel
for op in allgather reducescatter broadcast sendrecv grad; do
  timeout 100 $S --op $op --min 65536 --max 134217728 --step 8
done
