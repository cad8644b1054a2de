#!/usr/bin/env python
"""Evaluation cost of the single-GPU DLRM step: graph-replayed ``DLRMTrainStep.evaluate`` versus
the autograd module path, next to a training step.

  python tools/bench_eval.py [--batches 4] [--repeats 3] [--train-steps 10] [--warmup 3]
  python tools/bench_eval.py --auc exact [--sizes 1M,16M,89M]

For ``dlrm-mlperf-20m`` (the ``bench.py`` default model) at global batch 65536 with synthetic
uniform ids, once with fp32 and once with bf16 tables, alternating in one process ``--repeats``
times:

(a) ``evaluate`` over ``--batches`` eval batches (one CUDA-graph replay each; binned AUC and log
    loss accumulated on the device), timed with CUDA events;
(b) the path ``examples/dlrm/main.py`` takes without ``--fast``: ``model.eval()``, ``no_grad``,
    ``sigmoid`` of the module's logits, predictions copied to the host and the exact
    ``binary_auc`` over the same batches, timed with a host clock that ends in a synchronise;
(c) ``--train-steps`` training steps (graph replay), timed with CUDA events.

Prints one JSON line per table dtype: ms per batch and samples/s of each (median over the
repeats), the card's name and power limit (read in the same run), and ``|AUC_binned -
AUC_exact|`` of the step's predictions next to ``tie_bound``; asserts the difference is within
the bound.

``--auc exact`` times the exact ROC AUC (``DLRMTrainStep(eval_auc="exact")``) instead, on the same
model with fp32 tables: one JSON line with the per-batch cost of the eval graph with the
``auc_append`` kernel against the binned-only graph (the two graphs alternate ``--repeats`` times,
CUDA events), the exact AUC minus the binned one next to ``tie_bound`` for the step's
predictions, and then for every ``--sizes`` entry the time of ``eval_metrics``' exact part (the
first-party radix sort of the keys and ``auc_count``; CUDA events, median of ``--repeats``, keys
restored before each run) on sigmoid-shaped synthetic probabilities.  Needs a GPU.
"""
import argparse
import gc
import json
import os
import subprocess
import sys
import time

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


def _median(xs):
  xs = sorted(xs)
  return xs[len(xs) // 2]


def run(table_dtype, args, gpu):
  from distributed_embeddings_b200.models.dlrm import DLRM
  from distributed_embeddings_b200.models.dlrm_fast import DLRMTrainStep
  from distributed_embeddings_b200.utils.metrics import binary_auc
  dev = torch.device("cuda", 0)
  torch.manual_seed(1234)
  sizes = table_sizes_for("dlrm-mlperf-20m")
  model = DLRM(sizes, device=dev, compute_dtype=torch.bfloat16, backend="fused",
               table_dtype=_DTYPES[table_dtype])
  step = DLRMTrainStep(model, lr=0.5, embedding_optimizer="sgd", use_cuda_graph=True)
  b = args.global_batch
  g = torch.Generator().manual_seed(99)

  def batch():
    num = torch.rand(b, 13, generator=g)
    cat = torch.stack([gen_ids(s, b, 0.0, g) for s in sizes])
    lab = torch.randint(0, 2, (b,), generator=g).float()
    return num.to(dev), cat.to(dev), lab.to(dev)

  train = [batch() for _ in range(4)]
  evals = [batch() for _ in range(args.batches)]
  ev = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

  def timed_eval():
    ev[0].record()
    for num, cat, lab in evals:
      step.evaluate(num, cat, lab)
    ev[1].record()
    torch.cuda.synchronize()
    step.eval_metrics()
    return ev[0].elapsed_time(ev[1]) / len(evals)

  def timed_module():
    model.eval()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    preds, labels = [], []
    with torch.no_grad():
      for num, cat, lab in evals:
        p = torch.sigmoid(model(num, list(cat)).float())
        preds.append(p.cpu())
        labels.append(lab.cpu())
    binary_auc(torch.cat(labels), torch.cat(preds))
    torch.cuda.synchronize()
    model.train()
    return (time.perf_counter() - t0) * 1e3 / len(evals)

  def timed_train():
    ev[0].record()
    for i in range(args.train_steps):
      step.step(*train[i % 4])
    ev[1].record()
    torch.cuda.synchronize()
    return ev[0].elapsed_time(ev[1]) / args.train_steps

  for i in range(args.warmup):
    step.step(*train[i % 4])
  timed_eval()
  timed_module()
  t_eval, t_mod, t_train = [], [], []
  for _ in range(args.repeats):
    t_eval.append(timed_eval())
    t_mod.append(timed_module())
    t_train.append(timed_train())
  # binned versus exact AUC of the same predictions
  probs, labels = [], []
  for num, cat, lab in evals:
    step.evaluate(num, cat, lab)
    probs.append(step.predict(num, cat).cpu())
    labels.append(lab.cpu())
  met = step.eval_metrics()
  exact = binary_auc(torch.cat(labels), torch.cat(probs))
  diff = abs(met["auc"] - exact)
  assert diff <= met["tie_bound"] + 1e-12, (met, exact)
  step.ctx.check_errors()
  res = {
      "model": "dlrm-mlperf-20m", "table_dtype": table_dtype, "global_batch": b,
      "eval_batches": len(evals), "repeats": args.repeats, "gpu": gpu,
      "eval_graph_ms_per_batch": _median(t_eval),
      "eval_graph_samples_per_s": b / _median(t_eval) * 1e3,
      "module_path_ms_per_batch": _median(t_mod),
      "module_path_samples_per_s": b / _median(t_mod) * 1e3,
      "train_ms_per_step": _median(t_train),
      "module_over_eval": _median(t_mod) / _median(t_eval),
      "auc_binned": met["auc"], "auc_exact": exact, "abs_diff": diff,
      "tie_bound": met["tie_bound"], "log_loss": met["log_loss"], "samples": met["samples"],
      "spread_ms": {"eval": [min(t_eval), max(t_eval)], "module": [min(t_mod), max(t_mod)],
                    "train": [min(t_train), max(t_train)]},
  }
  del step, model, train, evals
  gc.collect()
  torch.cuda.empty_cache()
  return res


def _parse_size(s):
  s = s.strip().upper()
  mult = {"K": 10**3, "M": 10**6}.get(s[-1], 1)
  return int(float(s[:-1] if s[-1] in "KM" else s) * mult)


def run_exact(args, gpu):
  from distributed_embeddings_b200.models.dlrm import DLRM
  from distributed_embeddings_b200.models.dlrm_fast import DLRMTrainStep
  from distributed_embeddings_b200.ops import _native
  from distributed_embeddings_b200.utils.metrics import ExactAUC
  dev = torch.device("cuda", 0)
  torch.manual_seed(1234)
  sizes = table_sizes_for("dlrm-mlperf-20m")
  model = DLRM(sizes, device=dev, compute_dtype=torch.bfloat16, backend="fused",
               table_dtype=torch.float32)
  b = args.global_batch
  step = DLRMTrainStep(model, lr=0.5, embedding_optimizer="sgd", use_cuda_graph=True,
                       eval_auc="exact", eval_capacity=b * args.batches)
  g = torch.Generator().manual_seed(99)

  def batch():
    num = torch.rand(b, 13, generator=g)
    cat = torch.stack([gen_ids(s, b, 0.0, g) for s in sizes])
    lab = torch.randint(0, 2, (b,), generator=g).float()
    return num.to(dev), cat.to(dev), lab.to(dev)

  train = [batch() for _ in range(4)]
  evals = [batch() for _ in range(args.batches)]
  for i in range(args.warmup):
    step.step(*train[i % 4])
  # two captures of the eval schedule: with auc_append (exact) and without (binned only)
  exact_metric = step.exact_auc
  step.exact_auc = None
  step.evaluate(*evals[0])
  graphs = {"binned": (step._eval_graph, None)}
  step._eval_graph, step.exact_auc = None, exact_metric
  step.evaluate(*evals[0])
  graphs["exact"] = (step._eval_graph, exact_metric)
  step.eval_metrics()
  ev = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  times = {"binned": [], "exact": []}
  for _ in range(args.repeats + 1):  # the first round is warm-up
    for mode in ("binned", "exact"):
      step._eval_graph, step.exact_auc = graphs[mode]
      ev[0].record()
      for num, cat, lab in evals:
        step.evaluate(num, cat, lab)
      ev[1].record()
      torch.cuda.synchronize()
      times[mode].append(ev[0].elapsed_time(ev[1]) / len(evals))
      step.eval_metrics()
  step._eval_graph, step.exact_auc = graphs["exact"]
  t_b, t_e = _median(times["binned"][1:]), _median(times["exact"][1:])
  for num, cat, lab in evals:
    step.evaluate(num, cat, lab)
  met = step.eval_metrics()
  assert abs(met["auc"] - met["binned_auc"]) <= met["tie_bound"] + 1e-12, met
  step.ctx.check_errors()
  res = {
      "model": "dlrm-mlperf-20m", "table_dtype": "fp32", "global_batch": b, "auc": "exact",
      "eval_batches": len(evals), "repeats": args.repeats, "gpu": gpu,
      "eval_binned_ms_per_batch": t_b, "eval_exact_ms_per_batch": t_e,
      "append_ms_per_batch": t_e - t_b, "append_share_of_batch": (t_e - t_b) / t_e,
      "spread_ms": {k: [min(v[1:]), max(v[1:])] for k, v in times.items()},
      "auc_exact": met["auc"], "auc_binned": met["binned_auc"],
      "exact_minus_binned": met["auc"] - met["binned_auc"], "tie_bound": met["tie_bound"],
      "samples": met["samples"],
  }
  del step, model, train, evals, graphs, exact_metric
  gc.collect()
  torch.cuda.empty_cache()

  # sort + count at evaluation-set sizes
  ops = _native.require()
  count_ms = {}
  for label in args.sizes.split(","):
    n = _parse_size(label)
    m = ExactAUC(n, device=dev)
    gen = torch.Generator(device=dev).manual_seed(n)
    chunk = 1 << 22
    for s in range(0, n, chunk):
      k = min(chunk, n - s)
      y = (torch.rand(k, generator=gen, device=dev) < 0.25).float()
      p = torch.sigmoid(torch.randn(k, generator=gen, device=dev) * 1.5 - 2.0 + y)
      m.update(p, y)
    want = m.counts()
    saved = m.keys[:n].clone()
    out = torch.zeros(3, dtype=torch.int64, device=dev)
    ts = []
    for _ in range(args.repeats + 1):
      m.keys[:n].copy_(saved)
      torch.cuda.synchronize()
      ev[0].record()
      ops.radix_sort_keys32(m.keys, n, 31)
      ops.auc_count(m.keys, n, out)
      ev[1].record()
      torch.cuda.synchronize()
      ts.append(ev[0].elapsed_time(ev[1]))
    assert tuple(out.tolist()) == want
    count_ms[label] = {"samples": n, "sort_count_ms": _median(ts[1:]),
                       "spread_ms": [min(ts[1:]), max(ts[1:])],
                       "keys_per_s": n / _median(ts[1:]) * 1e3}
    del m, saved, out
    torch.cuda.empty_cache()
  res["eval_metrics_exact"] = count_ms
  return res


def main():
  ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawTextHelpFormatter)
  ap.add_argument("--batches", type=int, default=4, help="eval batches per timing")
  ap.add_argument("--repeats", type=int, default=3)
  ap.add_argument("--train-steps", type=int, default=10)
  ap.add_argument("--warmup", type=int, default=3)
  ap.add_argument("--global-batch", type=int, default=65536)
  ap.add_argument("--table-dtypes", default="fp32,bf16")
  ap.add_argument("--auc", choices=("binned", "exact"), default="binned")
  ap.add_argument("--sizes", default="1M,16M,89M",
                  help="--auc exact: sample counts at which sort + count is timed")
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("bench_eval.py needs a CUDA GPU")
  torch.cuda.set_device(0)
  gpu = gpu_info()
  if args.auc == "exact":
    print(json.dumps(run_exact(args, gpu)), flush=True)
    return
  for dt in args.table_dtypes.split(","):
    print(json.dumps(run(dt, args, gpu)), flush=True)


if __name__ == "__main__":
  main()
