#!/usr/bin/env python
"""Row threshold of the table update applied by the interaction backward, single-GPU DLRM step.

  python tools/bench_fused_table_update.py [--steps 30] [--warmup 5] [--repeats 3]

``DLRMTrainStep(fused_table_update=True, fused_update_min_rows=R)`` updates the tables with at
least R rows from the interaction backward and leaves the others to the staged scatter.  This
times the ``bench.py`` configuration (``dlrm-mlperf-20m``, global batch 65536, CUDA graph,
cuBLASLt, bf16 compute, SGD with the MLPerf schedule) with the update off and at every R of
``--rows``, on uniform ids and on the reference generator's power law (``--alphas``).  One model
and one step serve every configuration: R is switched between runs and the step recaptured.  The
configurations alternate within each repeat; the times are device-timed ms per step (CUDA events
around ``--steps`` graph replays), median and spread over the repeats.  The table sizes and the
id generator are imported from ``bench.py``.  Prints one JSON line.  Needs a GPU.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from bench import gen_ids, table_sizes_for  # noqa: E402


def gpu_info():
  out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True, check=True)
  name, power, clock = [x.strip() for x in out.stdout.splitlines()[0].split(",")]
  return {"name": name, "power_limit": power, "max_sm_clock": clock}


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--steps", type=int, default=30)
  ap.add_argument("--warmup", type=int, default=5)
  ap.add_argument("--repeats", type=int, default=3)
  ap.add_argument("--global-batch", type=int, default=65536)
  ap.add_argument("--alphas", default="0,1.05")
  ap.add_argument("--rows", default="2500,20000,100000,1000000,20000000")
  args = ap.parse_args()
  from distributed_embeddings_b200.models.dlrm import DLRM
  from distributed_embeddings_b200.models.dlrm_fast import DLRMTrainStep
  from distributed_embeddings_b200.utils.lr_schedule import LearningRateScheduler
  dev = torch.device("cuda", 0)
  torch.manual_seed(1234)
  sizes = table_sizes_for("dlrm-mlperf-20m")
  model = DLRM(sizes, device=dev, compute_dtype=torch.bfloat16, backend="fused")
  sched = LearningRateScheduler(24.0, warmup_steps=8000, decay_start_step=48000,
                                decay_steps=24000)
  step = DLRMTrainStep(model, lr=24.0, embedding_optimizer="sgd", use_cuda_graph=True,
                       scheduler=sched)
  b = args.global_batch
  pools = {}
  for a in [float(x) for x in args.alphas.split(",")]:
    g = torch.Generator().manual_seed(99)
    pools[a] = [(torch.rand(b, 13, generator=g).to(dev),
                 torch.stack([gen_ids(s, b, a, g) for s in sizes]).to(dev),
                 torch.randint(0, 2, (b, 1), generator=g).float().to(dev)) for _ in range(4)]
  configs = [None] + [int(x) for x in args.rows.split(",")]
  pos = [0]

  def run(pool, n):
    for _ in range(n):
      step.run_prefetched()
      pos[0] += 1
      step.prefetch(*pool[pos[0] % len(pool)])

  times = {}
  for _ in range(args.repeats):
    for a, pool in pools.items():
      for rows in configs:
        step.fused_table_update = rows is not None
        step.fused_update_min_rows = rows or 0
        step._graph = None  # recaptured with the new split by the next run
        if pos[0] == 0:
          step.prefetch(*pool[0])
        run(pool, args.warmup)
        torch.cuda.synchronize()
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        run(pool, args.steps)
        end.record()
        torch.cuda.synchronize()
        times.setdefault((a, rows), []).append(start.elapsed_time(end) / args.steps)
  rows_out = []
  for (a, rows), ts in times.items():
    ts = sorted(ts)
    rows_out.append({"alpha": a, "min_rows": rows,
                     "applied_tables": 0 if rows is None else sum(s >= rows for s in sizes),
                     "ms_per_step_median": ts[len(ts) // 2], "ms_per_step_min": ts[0],
                     "ms_per_step_max": ts[-1]})
  print(json.dumps({"gpu": gpu_info(), "steps": args.steps, "repeats": args.repeats,
                    "global_batch": b, "results": rows_out}))


if __name__ == "__main__":
  main()
