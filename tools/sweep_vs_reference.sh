#!/bin/bash
# Config-5 sweep with the reference beside it (run on a GPU box; N = number of GPUs, default 2):
#   tools/sweep_vs_reference.sh 2 > sweep_vs_reference_n2.jsonl
# Every line is bench.py's JSON line (ours and --impl reference, same metric / config / timing rules) for one total
# sequence length; the reference is lucidrains/ring-attention-pytorch's own Triton kernels + NCCL batch_isend_irecv ring
# (ring.py:51-60) from baseline/_ref, unmodified.
N=${1:-2}
SIZES=${2:-"4096 16384 65536 262144"}
PORT=29600
for S in $SIZES; do
  for IMPL in reference ours; do
    PORT=$((PORT+1))
    if [ "$N" -gt 1 ]; then
      python -m torch.distributed.run --nnodes=1 --nproc-per-node $N --master-addr 127.0.0.1 --master-port $PORT \
        bench.py --gpus $N --impl $IMPL --seq-len $S --steps 3 --warmup 2 --no-e2e --no-1m --check off 2>/dev/null | grep -E '^\{'
    else
      python bench.py --impl $IMPL --seq-len $S --steps 3 --warmup 2 --no-e2e --no-1m --check off 2>/dev/null | grep -E '^\{'
    fi
  done
done
