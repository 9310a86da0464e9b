#!/bin/bash
# Bring-up matrix of the fused tensor-core kernel's fusion switches (one process per configuration: a trap poisons the context).
#   tests/bringup/tc_matrix.sh <res> <n>
R=${1:-128}; N=${2:-2}
for fuse in 0 1 2 3; do
  echo "== MIGAN_FUSE=$fuse  (R=$R N=$N)"
  CUDA_LAUNCH_BLOCKING=1 MIGAN_FUSE=$fuse timeout 120 python tests/bringup/gpu_diag.py --path tc --res $R --n $N --taps 1 2>&1 | grep -E "FINAL|MISMATCH|FAILED|record" | head -12
done
