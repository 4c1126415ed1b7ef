#!/bin/bash
# Weak-scaling points and the NCCL CTA / SM-reserve sweep (run on one 8-GPU box: bash tools/scaling_sweep.sh).  Every line is bench.py's own JSON (CUDA events, max over ranks).
mkdir -p results
port=29540
for n in 8 4 2; do
  port=$((port + 1))
  timeout 600 python -m torch.distributed.run --nnodes=1 --nproc-per-node $n --master-addr 127.0.0.1 --master-port $port \
    bench.py --gpus $n --steps 30 --warmup 5 --no-extras > results/scale_n$n.json 2> results/scale_n$n.err
done
for c in 8 16 24 32; do
  port=$((port + 1))
  NCCL_MAX_CTAS=$c UNIVTG_DDP_SM_RESERVE=$c timeout 600 python -m torch.distributed.run --nnodes=1 --nproc-per-node 8 \
    --master-addr 127.0.0.1 --master-port $port bench.py --gpus 8 --steps 30 --warmup 5 --no-extras \
    > results/scale_n8_cta$c.json 2> results/scale_n8_cta$c.err
done
port=$((port + 1))
timeout 600 python -m torch.distributed.run --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 --master-port $port \
  bench.py --gpus 8 --steps 30 --warmup 5 --no-extras --no-overlap > results/scale_n8_nooverlap.json 2> results/scale_n8_nooverlap.err
timeout 300 python bench.py --steps 30 --warmup 5 --no-extras --no-cpu-baseline > results/scale_n1.json 2> results/scale_n1.err
