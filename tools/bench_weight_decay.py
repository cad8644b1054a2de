#!/usr/bin/env python
"""Cost of weight decay in the single-GPU DLRM training step: no decay, L2 decay and decoupled
(AdamW-style) decay, for the embedding optimizers that have a decoupled kernel.

  python tools/bench_weight_decay.py [--steps 30] [--warmup 5] [--repeats 3]
                                     [--optimizers adagrad,adam,rowwise_adam]
                                     [--max-rows 5000000] [--weight-decay 1e-5]

One invocation, one GPU, the MLPerf tables capped at ``--max-rows`` (default 5M, ids from
``bench.py``'s generator), ``DLRMTrainStep`` (CUDA graph, bf16 compute, dense SGD) at global
batch 65536.  For fp32 and bf16 tables the model is built once; then, ``--repeats`` times, every
optimizer x {none, l2, decoupled} runs in turn (the configurations alternate), each on a fresh
``DLRMTrainStep`` with the decay on both the tables and the dense parameters.  Reported per
configuration: device-timed ms per step (CUDA events around ``--steps`` graph replays; median and
spread over the repeats) and samples/s, and the card's name, power limit and max SM clock
(``nvidia-smi --query-gpu``, read only).

L2 decay makes the row pass of the row-wise kinds read the weights (the row mean of the decayed
gradient's square); decoupled decay does not.

Prints one JSON line.  Needs a GPU.
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

from bench import gen_ids  # noqa: E402
from distributed_embeddings_b200.models.dlrm import mlperf_table_sizes  # noqa: E402

_DTYPES = {"fp32": torch.float32, "bf16": torch.bfloat16}
_LR = {"adagrad": 0.01, "rowwise_adagrad": 0.01, "adam": 0.0001, "rowwise_adam": 0.0001}
DECAYS = ("none", "l2", "decoupled")


def gpu_info():
  out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True, check=True)
  name, power, clock = [x.strip() for x in out.stdout.splitlines()[0].split(",")]
  return {"name": name, "power_limit": power, "max_sm_clock": clock}


def make_pool(sizes, b):
  g = torch.Generator().manual_seed(99)
  pool = []
  for _ in range(4):
    num = torch.rand(b, 13, generator=g)
    cat = torch.stack([gen_ids(s, b, 0.0, g) for s in sizes])
    lab = torch.randint(0, 2, (b,), generator=g).float()
    pool.append((num, cat, lab))
  return pool


def time_step(model, kind, decay, args, batches):
  """ms per step of a fresh DLRMTrainStep with ``decay`` on ``model``."""
  from distributed_embeddings_b200.models.dlrm_fast import DLRMTrainStep
  kw = {} if decay == "none" else {"weight_decay": args.weight_decay, "weight_decay_mode": decay}
  trainer = DLRMTrainStep(model, lr=_LR[kind], embedding_optimizer=kind, use_cuda_graph=True,
                          embedding_optimizer_kwargs=kw, dense_optimizer_kwargs=kw)
  try:
    for i in range(args.warmup):
      trainer.step(*batches[i % 4])
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for i in range(args.steps):
      trainer.step(*batches[i % 4])
    t1.record()
    torch.cuda.synchronize()
    trainer.ctx.check_errors()
    return t0.elapsed_time(t1) / args.steps
  finally:
    del trainer
    gc.collect()
    torch.cuda.empty_cache()


def main():
  ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawTextHelpFormatter)
  ap.add_argument("--steps", type=int, default=30)
  ap.add_argument("--warmup", type=int, default=5)
  ap.add_argument("--repeats", type=int, default=3)
  ap.add_argument("--global-batch", type=int, default=65536)
  ap.add_argument("--max-rows", type=int, default=5_000_000)
  ap.add_argument("--weight-decay", type=float, default=1e-5)
  ap.add_argument("--optimizers", default="adagrad,adam,rowwise_adam",
                  help=f"comma-separated subset of {', '.join(_LR)}")
  args = ap.parse_args()
  kinds = [k for k in args.optimizers.split(",") if k]
  if not kinds or any(k not in _LR for k in kinds):
    ap.error(f"--optimizers: a comma-separated subset of {', '.join(_LR)}")
  if not torch.cuda.is_available():
    raise SystemExit("bench_weight_decay.py needs a CUDA GPU")
  from distributed_embeddings_b200.models.dlrm import DLRM
  torch.cuda.set_device(0)
  dev = torch.device("cuda", 0)
  sizes = mlperf_table_sizes(args.max_rows)
  out = {"gpu": gpu_info(), "max_rows": args.max_rows, "rows": sum(sizes),
         "global_batch": args.global_batch, "steps": args.steps,
         "weight_decay": args.weight_decay}
  pool = make_pool(sizes, args.global_batch)
  batches = [tuple(x.to(dev) for x in p) for p in pool]
  results = []
  for tdt in ("fp32", "bf16"):
    torch.manual_seed(1234)
    model = DLRM(sizes, device=dev, compute_dtype=torch.bfloat16, backend="fused",
                 table_dtype=_DTYPES[tdt])
    runs = {(k, d): [] for k in kinds for d in DECAYS}
    for _ in range(args.repeats):
      for k in kinds:
        for d in DECAYS:
          runs[(k, d)].append(time_step(model, k, d, args, batches))
    for (k, d), ms in runs.items():
      ms = sorted(ms)
      med = ms[len(ms) // 2]
      results.append({"optimizer": k, "table_dtype": tdt, "decay": d, "ms_per_step_median": med,
                      "ms_per_step_min": ms[0], "ms_per_step_max": ms[-1],
                      "samples_per_s": args.global_batch / med * 1e3})
    del model
    gc.collect()
    torch.cuda.empty_cache()
  out["runs"] = results
  print(json.dumps(out))


if __name__ == "__main__":
  main()
