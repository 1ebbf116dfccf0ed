#!/bin/bash
# developer check on an N-GPU box (default 2): correctness of the sharded solve against the single-GPU solve, the 2-GPU pytest, then bench.py
N=${1:-2}
mkdir -p ${OUT:-/tmp/mcba_out}
t0=$(date +%s)
timeout 300 python -m torch.distributed.run --nnodes=1 --nproc-per-node=$N --master-addr 127.0.0.1 --master-port 29511 scripts/multi_gpu_check.py > ${OUT:-/tmp/mcba_out}/mgc_n$N.log 2>&1
echo "multi_gpu_check N=$N rc=$? $(( $(date +%s) - t0 ))s"; tail -8 ${OUT:-/tmp/mcba_out}/mgc_n$N.log
timeout 600 python -m pytest tests/test_distributed.py -q -m gpu --tb=short > ${OUT:-/tmp/mcba_out}/pytest_distributed.log 2>&1; tail -3 ${OUT:-/tmp/mcba_out}/pytest_distributed.log
t1=$(date +%s)
timeout 600 python -m torch.distributed.run --nnodes=1 --nproc-per-node $N --master-addr 127.0.0.1 --master-port 29637 bench.py --gpus $N --steps 5 --warmup 3 > ${OUT:-/tmp/mcba_out}/bench_n$N.json 2> ${OUT:-/tmp/mcba_out}/bench_n$N.err
echo "bench N=$N rc=$? $(( $(date +%s) - t1 ))s"; tail -3 ${OUT:-/tmp/mcba_out}/bench_n$N.err
python scripts/show_bench.py ${OUT:-/tmp/mcba_out}/bench_n$N.json
