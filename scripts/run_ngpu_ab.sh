#!/bin/bash
# bench.py on N GPUs: peer-memory exchanges, NCCL only, and peer-memory exchanges with MCBA_FUSE=1 (five exchanges per LM iteration
# instead of six, four of them as the tail of the kernel that produces their values) -- developer A/B.  Run the correctness check
# first: MCBA_FUSE=1 torchrun ... scripts/multi_gpu_check.py
N=${1:-8}
mkdir -p ${OUT:-/tmp/mcba_out}
port=29700
for p in 1 0 fuse; do
  t1=$(date +%s); port=$((port+11))
  if [ $p = fuse ]; then export MCBA_FUSE=1; peer=1; else unset MCBA_FUSE; peer=$p; fi
  MCBA_PEER=$peer timeout 200 python -m torch.distributed.run --nnodes=1 --nproc-per-node $N --master-addr 127.0.0.1 --master-port $port bench.py --gpus $N --steps 10 --warmup 3 > ${OUT:-/tmp/mcba_out}/bench_n${N}_peer$p.json 2> ${OUT:-/tmp/mcba_out}/bench_n${N}_peer$p.err
  echo "bench N=$N peer=$p rc=$? $(( $(date +%s) - t1 ))s"
  python - <<PY
import json
try:
  txt = open("${OUT:-/tmp/mcba_out}/bench_n${N}_peer$p.json").read()
  d = json.loads([l for l in txt.splitlines() if l.startswith("{")][-1])
  print("N=$N peer=$p value %.4g ms_per_step %.3f evals %.1f lm_it/s %.0f e2e_ms %.3f launches %d" % (d["value"], d["ms_per_step"], d["nfev_plus_njev_per_step"], d["lm_iters_per_sec"], d["e2e"]["ms_per_step"], d["gpu_launches"]))
except Exception as e:
  print("no json:", e); print(open("${OUT:-/tmp/mcba_out}/bench_n${N}_peer$p.err").read()[-1500:])
PY
done
