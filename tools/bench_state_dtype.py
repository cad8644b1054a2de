#!/usr/bin/env python
"""fp32 versus bf16 optimizer state (Adagrad accumulator, Adam moments, row-wise Adam's m, FTRL's
n and z, the momentum buffer) in the single-GPU DLRM training step.

  python tools/bench_state_dtype.py [--steps 30] [--warmup 5] [--repeats 3] [--loss-steps 40]
                                    [--profile]
                                    [--optimizers sgd,adagrad,adam,rowwise_adam,ftrl,momentum]

One invocation, one GPU, the MLPerf tables capped at ``--max-rows`` (default 20M:
``dlrm-mlperf-20m`` of ``bench.py``, whose id generator this uses), ``DLRMTrainStep`` (CUDA graph,
bf16 compute) at global batch 65536.  At 20M rows only the bf16-state and the smaller fp32-state
configurations fit one 80 GB card; ``--max-rows 5000000`` fits all of them:

1. ``--optimizers`` (default Adagrad and Adam; ``rowwise_adam`` adds row-wise Adam, whose bf16
   state is its m: v stays one fp32 word per row; ``ftrl`` adds FTRL, two element-wise slots
   like Adam; ``momentum`` adds momentum SGD, one element-wise slot like Adagrad; ``sgd`` adds
   deterministic SGD, the sorted update without state, fp32 state only) x {fp32, bf16} tables x
   {fp32, bf16} state,
   alternating, ``--repeats`` times
   each: device-timed ms per step (CUDA events around ``--steps`` graph replays; median and spread
   over the repeats), samples/s and ``torch.cuda.max_memory_allocated``.  A configuration whose
   tables and state alone exceed the card's memory is reported with its planned GiB and not run;
   one that runs out of memory while building its step is reported as such;
2. for every configuration with both state dtypes, the loss after ``--loss-steps`` seeded steps and
   its difference to the fp32-state run; with Adam and row-wise Adam both run, the loss of each
   after ``--loss-steps`` seeded steps (the two differ by design);
3. with ``--profile``: one extra profiled run per configuration (``torch.profiler``, CUDA
   activities), the update kernels' mean µs per step and the bytes/s they achieve on the bytes the
   update must move (per touched element: weight read + write, state read + write, from the
   unique rows of the batch and the element sizes);
4. the card's name, power limit and max SM clock (``nvidia-smi --query-gpu``, read only).

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
# element-wise state slots
_SLOTS = {"sgd": 0, "adagrad": 1, "adam": 2, "rowwise_adam": 1, "ftrl": 2, "momentum": 1}
# fp32 words per row
_ROW_SLOTS = {"sgd": 0, "adagrad": 0, "adam": 0, "rowwise_adam": 1, "ftrl": 0, "momentum": 0}
_LR = {"sgd": 0.1, "adagrad": 0.01, "adam": 0.0001, "rowwise_adam": 0.0001, "ftrl": 0.01,
       "momentum": 0.01}
_UPDATE_KERNELS = ("segment_update", "balanced_update", "finalize_crossing")
DIM = 128


def gpu_info():
  out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True, check=True)
  name, power, clock = [x.strip() for x in out.stdout.splitlines()[0].split(",")]
  return {"name": name, "power_limit": power, "max_sm_clock": clock}


def planned_gib(sizes, kind, table_dtype, state_dtype):
  elems = sum(sizes) * DIM
  return (elems * (_DTYPES[table_dtype].itemsize + _SLOTS[kind] * _DTYPES[state_dtype].itemsize) +
          sum(sizes) * 4 * _ROW_SLOTS[kind]) / 2**30


def make_pool(sizes, b):
  g = torch.Generator().manual_seed(99)
  pool = []
  for _ in range(4):
    num = torch.rand(b, 13, generator=g)
    cat = torch.stack([gen_ids(s, b, 0.0, g) for s in sizes])
    lab = torch.randint(0, 2, (b,), generator=g).float()
    pool.append((num, cat, lab))
  return pool


def update_bytes(pool, kind, table_dtype, state_dtype):
  """Bytes the fused update moves per step, averaged over the pool: every touched element's
  weight and state are read and written once (row-wise state: one fp32 word per touched row)."""
  per_elem = 2 * (_DTYPES[table_dtype].itemsize + _SLOTS[kind] * _DTYPES[state_dtype].itemsize)
  per_row = DIM * per_elem + 2 * 4 * _ROW_SLOTS[kind]
  rows = [sum(int(torch.unique(c).numel()) for c in cat) for _, cat, _ in pool]
  return sum(rows) / len(rows) * per_row


def run(cfg, args, pool, steps, mode="time"):
  from distributed_embeddings_b200.models.dlrm import DLRM
  from distributed_embeddings_b200.models.dlrm_fast import DLRMTrainStep
  kind, tdt, sdt = cfg
  dev = torch.device("cuda", 0)
  gc.collect()
  torch.cuda.empty_cache()
  torch.cuda.reset_peak_memory_stats(dev)
  res = {"optimizer": kind, "table_dtype": tdt, "state_dtype": sdt}
  model = trainer = None
  try:
    torch.manual_seed(1234)
    model = DLRM(mlperf_table_sizes(args.max_rows), device=dev, compute_dtype=torch.bfloat16,
                 backend="fused", table_dtype=_DTYPES[tdt])
    # SGD keeps no state: the sorted, deterministic update instead of the atomic scatter
    kw = {"state_dtype": _DTYPES[sdt]} if _SLOTS[kind] else {"deterministic": True}
    trainer = DLRMTrainStep(model, lr=_LR[kind], embedding_optimizer=kind, use_cuda_graph=True,
                            embedding_optimizer_kwargs=kw)
    batches = [tuple(x.to(dev) for x in p) for p in pool]
    if mode == "loss":
      loss = None
      for i in range(steps):
        loss = trainer.step(*batches[i % 4])
      torch.cuda.synchronize()
      res["loss"] = float(loss)
      return res
    for i in range(args.warmup):
      trainer.step(*batches[i % 4])
    torch.cuda.synchronize()
    if mode == "profile":
      from torch.profiler import ProfilerActivity, profile
      with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(steps):
          trainer.step(*batches[i % 4])
        torch.cuda.synchronize()
      us = sum(e.device_time_total for e in prof.key_averages()
               if any(k in e.key for k in _UPDATE_KERNELS))
      res["update_us_per_step"] = us / steps
      res["update_bytes_per_step"] = update_bytes(pool, kind, tdt, sdt)
      res["update_achieved_gb_per_s"] = res["update_bytes_per_step"] / (us / steps) / 1e3
      return res
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for i in range(steps):
      trainer.step(*batches[i % 4])
    t1.record()
    torch.cuda.synchronize()
    ms = t0.elapsed_time(t1) / steps
    res.update(ms_per_step=ms, samples_per_s=args.global_batch / ms * 1e3,
               max_memory_allocated_gib=torch.cuda.max_memory_allocated(dev) / 2**30)
    trainer.ctx.check_errors()
    return res
  except torch.OutOfMemoryError:
    res["out_of_memory"] = True
    return res
  finally:
    del trainer, model
    gc.collect()
    torch.cuda.empty_cache()


def main():
  ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawTextHelpFormatter)
  ap.add_argument("--steps", type=int, default=30)
  ap.add_argument("--warmup", type=int, default=5)
  ap.add_argument("--repeats", type=int, default=3)
  ap.add_argument("--loss-steps", type=int, default=40)
  ap.add_argument("--global-batch", type=int, default=65536)
  ap.add_argument("--max-rows", type=int, default=20_000_000)
  ap.add_argument("--profile", action="store_true")
  ap.add_argument("--optimizers", default="adagrad,adam",
                  help="comma-separated subset of " + ", ".join(_SLOTS))
  args = ap.parse_args()
  kinds = [k for k in args.optimizers.split(",") if k]
  if not kinds or any(k not in _SLOTS for k in kinds):
    ap.error(f"--optimizers: a comma-separated subset of {', '.join(_SLOTS)}")
  if not torch.cuda.is_available():
    raise SystemExit("bench_state_dtype.py needs a CUDA GPU")
  torch.cuda.set_device(0)
  card_gib = torch.cuda.get_device_properties(0).total_memory / 2**30
  sizes = mlperf_table_sizes(args.max_rows)
  out = {"gpu": gpu_info(), "max_rows": args.max_rows, "rows": sum(sizes),
         "global_batch": args.global_batch, "steps": args.steps, "card_gib": round(card_gib, 1)}
  pool = make_pool(sizes, args.global_batch)
  cfgs = [(k, t, s) for k in kinds for t in ("fp32", "bf16")
          for s in (("fp32", "bf16") if _SLOTS[k] else ("fp32",))]
  planned = {c: planned_gib(sizes, *c) for c in cfgs}
  # tables and state alone must leave room for the step's buffers (a few GiB at batch 65536)
  runnable = [c for c in cfgs if planned[c] < card_gib - 6.0]
  runs = {c: [] for c in runnable}
  for _ in range(args.repeats):
    for c in runnable:
      if not any(r.get("out_of_memory") for r in runs[c]):
        runs[c].append(run(c, args, pool, args.steps))
  results = []
  for c in cfgs:
    entry = {"optimizer": c[0], "table_dtype": c[1], "state_dtype": c[2],
             "planned_tables_and_state_gib": round(planned[c], 1)}
    rs = runs.get(c)
    if rs is None:
      entry["not_run"] = "tables and state exceed the card"
    elif any(r.get("out_of_memory") for r in rs):
      entry["not_run"] = "out of memory"
    else:
      ms = sorted(r["ms_per_step"] for r in rs)
      med = ms[len(ms) // 2]
      entry.update(ms_per_step_median=med, ms_per_step_min=ms[0], ms_per_step_max=ms[-1],
                   samples_per_s=args.global_batch / med * 1e3,
                   max_memory_allocated_gib=max(r["max_memory_allocated_gib"] for r in rs))
      if args.profile:
        entry["profile"] = run(c, args, pool, 10, mode="profile")
    results.append(entry)
  out["runs"] = results
  ok = {(e["optimizer"], e["table_dtype"], e["state_dtype"]) for e in results if "not_run" not in e}
  losses = []
  for k in kinds:
    for t in ("fp32", "bf16"):
      if (k, t, "fp32") in ok and (k, t, "bf16") in ok:
        l32 = run((k, t, "fp32"), args, pool, args.loss_steps, mode="loss")["loss"]
        l16 = run((k, t, "bf16"), args, pool, args.loss_steps, mode="loss")["loss"]
        losses.append({"optimizer": k, "table_dtype": t, "fp32_state": l32, "bf16_state": l16,
                       "relative_difference": abs(l16 - l32) / abs(l32)})
  out["loss_after_steps"] = {"steps": args.loss_steps, "pairs": losses}
  versus = []
  for t in ("fp32", "bf16"):
    for sd in ("fp32", "bf16"):
      if ("adam", t, sd) in ok and ("rowwise_adam", t, sd) in ok:
        la = run(("adam", t, sd), args, pool, args.loss_steps, mode="loss")["loss"]
        lr_ = run(("rowwise_adam", t, sd), args, pool, args.loss_steps, mode="loss")["loss"]
        versus.append({"table_dtype": t, "state_dtype": sd, "adam": la, "rowwise_adam": lr_,
                       "difference": lr_ - la})
  if versus:
    out["rowwise_adam_vs_adam_loss"] = {"steps": args.loss_steps, "pairs": versus}
  print(json.dumps(out))


if __name__ == "__main__":
  main()
