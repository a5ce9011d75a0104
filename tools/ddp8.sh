#!/bin/bash
# data-parallel timeline + train, noise and fullframe benches on N GPUs (default 8): usage: bash tools/ddp8.sh [N]
N=${1:-8}
O=gpurun_out/ddp$N; mkdir -p $O
export NCCL_DEBUG=WARN
TR="python -m torch.distributed.run --nnodes=1 --nproc-per-node $N --master-addr 127.0.0.1"
timeout 300 $TR --master-port 29621 tools/ddp_timeline.py > $O/timeline.txt 2>&1
timeout 300 $TR --master-port 29622 bench.py --gpus $N --steps 20 --warmup 5 > $O/bench_train.json 2> $O/bench_train.err
timeout 300 $TR --master-port 29623 bench.py --gpus $N --steps 20 --warmup 5 --workload noise --model ELD:P+G+B+R+U --batch 4 > $O/bench_noise_full.json 2> $O/bench_noise_full.err
timeout 300 $TR --master-port 29624 bench.py --gpus $N --steps 20 --warmup 5 --workload fullframe > $O/bench_fullframe.json 2> $O/bench_fullframe.err
timeout 300 python bench.py --gpus 1 --steps 20 --warmup 5 --no-cpu-baseline --no-onbox > $O/bench_train_1gpu.json 2>> $O/bench_train.err
grep -v "^\*\|OMP_NUM" $O/timeline.txt | tail -8; for f in bench_train bench_noise_full bench_fullframe bench_train_1gpu; do tail -1 $O/$f.json | cut -c1-420; echo; done; grep -v "^\*\|OMP_NUM\|^$" $O/*.err | tail -5
