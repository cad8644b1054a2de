#!/bin/bash
# Multi-GPU measurement suite: usage tools/run_suite.sh N [OUT_DIR]  (writes OUT_DIR/suite_nN.jsonl)
N=${1:-8}
OUT_DIR=${2:-suite_out}
OUT=$OUT_DIR/suite_n${N}.jsonl
mkdir -p $OUT_DIR; : > $OUT
TR="python -m torch.distributed.run --nnodes=1 --nproc-per-node $N --master-addr 127.0.0.1"
run() { # port, timeout, cmd...
  local port=$1; local to=$2; shift 2
  timeout $to $TR --master-port $port "$@" 2>&1 | grep -E '^\{' | tail -1 >> $OUT || echo "{\"failed\": \"$*\"}" >> $OUT
}
run 29601 240 bench.py --gpus $N --steps 50 --warmup 10
run 29602 240 bench.py --gpus $N --steps 50 --warmup 10 --column-slice-threshold none --no-e2e
SYN=examples/benchmarks/synthetic_models/main.py
run 29604 200 $SYN --model tiny --optimizer adagrad --batch_size 65536 --alpha 1.05 --num_steps 30 --num_data_batches 2 --amp
run 29605 240 $SYN --model small --optimizer adagrad --batch_size 65536 --alpha 1.05 --num_steps 30 --num_data_batches 2 --amp
run 29606 300 $SYN --model medium --optimizer adagrad --batch_size 65536 --alpha 1.05 --num_steps 20 --num_data_batches 1 --amp
run 29607 200 tools/bench_integer_lookup_dlrm.py --steps 30
# work-balancing placement (not in the reference) vs the memory_balanced lines above
run 29609 200 $SYN --model tiny --optimizer adagrad --batch_size 65536 --alpha 1.05 --num_steps 30 --num_data_batches 2 --amp --dist_strategy traffic_balanced
run 29610 240 $SYN --model small --optimizer adagrad --batch_size 65536 --alpha 1.05 --num_steps 30 --num_data_batches 2 --amp --dist_strategy traffic_balanced
if [ "$N" = "8" ]; then
  run 29608 420 $SYN --model large --optimizer rowwise_adagrad --batch_size 65536 --alpha 1.05 --num_steps 10 --num_data_batches 1 --amp --column_slice_threshold 1342177280
fi
cat $OUT
