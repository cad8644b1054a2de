#!/usr/bin/env python
"""fp32 versus bf16 embedding tables in the single-GPU DLRM training step.

  python tools/bench_table_dtype.py [--steps 30] [--warmup 5] [--repeats 3] [--loss-steps 40]

One invocation, one GPU:

1. ``dlrm-mlperf-20m`` with fp32 and with bf16 tables, alternating, ``--repeats`` times each:
   device-timed ms per step (CUDA events around ``--steps`` graph replays; median and spread over
   the repeats), samples/s and ``torch.cuda.max_memory_allocated``;
2. ``dlrm-mlperf`` (40M-row cap, 89.5 GiB in fp32: does not fit one 80 GB card) with bf16 tables,
   the same numbers;
3. the loss after ``--loss-steps`` seeded steps for fp32 and bf16 tables of the 20m model and
   their relative difference (half-precision storage changes the result by design);
4. the card's name, power limit and max SM clock (``nvidia-smi --query-gpu``, read only).

The step is ``DLRMTrainStep`` (CUDA graph, cuBLASLt GEMMs, bf16 compute, SGD with the MLPerf
learning-rate schedule) at global batch 65536, the configuration ``bench.py`` times; the table
sizes and the id generator are imported from ``bench.py``.  Prints one JSON line.  Needs a GPU.
"""
import argparse
import gc
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from bench import gen_ids, table_sizes_for  # noqa: E402

_DTYPES = {"fp32": torch.float32, "bf16": torch.bfloat16}


def gpu_info():
  out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True, check=True)
  name, power, clock = [x.strip() for x in out.stdout.splitlines()[0].split(",")]
  return {"name": name, "power_limit": power, "max_sm_clock": clock}


def run(model_name, table_dtype, args, steps, timed=True):
  from distributed_embeddings_b200.models.dlrm import DLRM
  from distributed_embeddings_b200.models.dlrm_fast import DLRMTrainStep
  from distributed_embeddings_b200.utils.lr_schedule import LearningRateScheduler
  dev = torch.device("cuda", 0)
  torch.cuda.empty_cache()
  torch.cuda.reset_peak_memory_stats(dev)
  torch.manual_seed(1234)
  sizes = table_sizes_for(model_name)
  model = DLRM(sizes, device=dev, compute_dtype=torch.bfloat16, backend="fused",
               table_dtype=_DTYPES[table_dtype])
  sched = LearningRateScheduler(24.0, warmup_steps=8000, decay_start_step=48000,
                                decay_steps=24000)
  trainer = DLRMTrainStep(model, lr=24.0, embedding_optimizer="sgd", use_cuda_graph=True,
                          scheduler=sched)
  b = args.global_batch
  g = torch.Generator().manual_seed(99)
  pool = []
  for _ in range(4):
    num = torch.rand(b, 13, generator=g)
    cat = torch.stack([gen_ids(s, b, 0.0, g) for s in sizes])
    lab = torch.randint(0, 2, (b,), generator=g).float()
    pool.append((num.to(dev), cat.to(dev), lab.to(dev)))
  res = {"model": model_name, "table_dtype": table_dtype}
  if timed:
    for i in range(args.warmup):
      trainer.step(*pool[i % 4])
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for i in range(steps):
      trainer.step(*pool[i % 4])
    t1.record()
    torch.cuda.synchronize()
    ms = t0.elapsed_time(t1) / steps
    res.update(ms_per_step=ms, samples_per_s=b / ms * 1e3)
  else:
    loss = None
    for i in range(steps):
      loss = trainer.step(*pool[i % 4])
    torch.cuda.synchronize()
    res["loss"] = float(loss)
  res["max_memory_allocated_gib"] = torch.cuda.max_memory_allocated(dev) / 2**30
  trainer.ctx.check_errors()
  del trainer, model, pool
  gc.collect()
  torch.cuda.empty_cache()
  return res


def main():
  ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawTextHelpFormatter)
  ap.add_argument("--steps", type=int, default=30)
  ap.add_argument("--warmup", type=int, default=5)
  ap.add_argument("--repeats", type=int, default=3)
  ap.add_argument("--loss-steps", type=int, default=40)
  ap.add_argument("--global-batch", type=int, default=65536)
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("bench_table_dtype.py needs a CUDA GPU")
  torch.cuda.set_device(0)
  out = {"gpu": gpu_info(), "global_batch": args.global_batch, "steps": args.steps}
  runs = {"fp32": [], "bf16": []}
  for _ in range(args.repeats):
    for dt in ("fp32", "bf16"):
      runs[dt].append(run("dlrm-mlperf-20m", dt, args, args.steps))
  summary = {}
  for dt, rs in runs.items():
    ms = sorted(r["ms_per_step"] for r in rs)
    med = ms[len(ms) // 2]
    summary[dt] = {"ms_per_step_median": med, "ms_per_step_min": ms[0], "ms_per_step_max": ms[-1],
                   "samples_per_s": args.global_batch / med * 1e3,
                   "max_memory_allocated_gib": max(r["max_memory_allocated_gib"] for r in rs)}
  out["dlrm-mlperf-20m"] = summary
  out["dlrm-mlperf-20m"]["bf16_over_fp32_time"] = \
      summary["bf16"]["ms_per_step_median"] / summary["fp32"]["ms_per_step_median"]
  out["dlrm-mlperf"] = {"bf16": run("dlrm-mlperf", "bf16", args, args.steps)}
  l32 = run("dlrm-mlperf-20m", "fp32", args, args.loss_steps, timed=False)["loss"]
  l16 = run("dlrm-mlperf-20m", "bf16", args, args.loss_steps, timed=False)["loss"]
  out["loss_after_steps"] = {"steps": args.loss_steps, "fp32": l32, "bf16": l16,
                             "relative_difference": abs(l16 - l32) / abs(l32)}
  print(json.dumps(out))


if __name__ == "__main__":
  main()
