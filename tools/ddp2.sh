#!/bin/bash
# data-parallel timeline + train bench on N GPUs (default 2) next to 1 GPU: usage: bash tools/ddp2.sh [N]
N=${1:-2}
O=gpurun_out/ddp$N; mkdir -p $O
export NCCL_DEBUG=WARN
TR="python -m torch.distributed.run --nnodes=1 --nproc-per-node $N --master-addr 127.0.0.1"
timeout 300 $TR --master-port 29611 tools/ddp_timeline.py > $O/timeline.txt 2>&1
timeout 400 $TR --master-port 29612 bench.py --gpus $N --steps 20 --warmup 5 > $O/bench_train.json 2> $O/bench_train.err
timeout 400 python bench.py --gpus 1 --steps 20 --warmup 5 > $O/bench_train_1gpu.json 2>> $O/bench_train.err
grep -v "^\*\|OMP_NUM" $O/timeline.txt | tail -8; for f in bench_train bench_train_1gpu; do tail -1 $O/$f.json | cut -c1-330; echo; done; grep -v "^\*\|OMP_NUM\|^$" $O/bench_train.err | tail -3
