#!/usr/bin/env python
"""Cost of the dense optimizer (``dense_optimizer`` = sgd / adagrad / adam) of the hand-scheduled
steps.

  python tools/bench_dense_optimizer.py [--repeats 3] [--steps 20] [--warmup 3] [--launches 200]

(a) Kernel time: ``dense_sgd`` / ``dense_adagrad`` / ``dense_adam`` on one flat buffer the size
    of the ``DLRMTrainStep`` dense parameters (padded MLPs of the MLPerf DLRM, 2.37 M elements),
    and on one 16 times larger, timed with CUDA events over ``--launches`` launches.  Achieved
    bytes/s from the bytes each kind must move per element (SGD 18: read p32, g32, write p32,
    g32, p16; Adagrad 26: + read / write acc; Adam 34: + read / write m, v) against the H100 SXM
    data-sheet HBM3 bandwidth of 3.35 TB/s.  The DLRM-sized buffers (43-81 MB) largely stay in
    the 50 MB L2 between back-to-back launches, so their rate can exceed HBM bandwidth; the
    larger buffer shows the HBM-bound rate.
(b) Step time: graph-replayed ``DLRMTrainStep`` at global batch 65536 on the ``dlrm-small``
    tables with SGD embeddings, and ``SyntheticTrainStep`` on ``tiny`` with Adagrad embeddings,
    alternating the three dense kinds ``--repeats`` times in one process, timed with CUDA events.

Prints one JSON line per measurement (median over repeats, with the spread) and the card's name
and power limit, read in the same run.  Needs a GPU.
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

KINDS = ("sgd", "adagrad", "adam")
BYTES_PER_ELEM = {"sgd": 18, "adagrad": 26, "adam": 34}
HBM_BYTES_PER_S = 3.35e12


def gpu_info():
  out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True, check=True)
  name, power, clock = [x.strip() for x in out.stdout.splitlines()[0].split(",")]
  return {"name": name, "power_limit": power, "max_sm_clock": clock}


def _median(xs):
  xs = sorted(xs)
  return xs[len(xs) // 2]


def dlrm_dense_numel() -> int:
  """Elements of the DLRMTrainStep flat dense buffers (no replicated tables)."""
  from distributed_embeddings_b200.models.dlrm import DLRM
  from distributed_embeddings_b200.models.dlrm_fast import _pad8
  m = DLRM([4] * 26, device="meta", backend="torch")
  n = 0
  for lin in [x for x in list(m.bottom_mlp.net) + list(m.top_mlp.net)
              if isinstance(x, torch.nn.Linear)]:
    n += lin.out_features * _pad8(lin.in_features) + _pad8(lin.out_features)
  return n


def kernel_times(args, gpu):
  from distributed_embeddings_b200.ops import _native
  ops = _native.require()
  for scale in (1, 16):
    _kernel_times(ops, dlrm_dense_numel() * scale, args, gpu)


def _kernel_times(ops, n, args, gpu):
  dev = torch.device("cuda", 0)
  p32 = torch.randn(n, device=dev)
  p16 = p32.bfloat16()
  g32 = torch.zeros(n, device=dev)
  acc = torch.full((n,), 0.1, device=dev)
  m, v = torch.zeros(n, device=dev), torch.zeros(n, device=dev)
  lr = torch.zeros(1, device=dev)  # the parameters stay put across the launches
  step = torch.ones(1, device=dev)
  launch = {
      "sgd": lambda: ops.dense_sgd(p32, p16, g32, lr, 1.0),
      "adagrad": lambda: ops.dense_adagrad(p32, p16, g32, acc, lr, 1e-7),
      "adam": lambda: ops.dense_adam(p32, p16, g32, m, v, lr, step, 0.9, 0.999, 1e-8),
  }
  ev = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  times = {k: [] for k in KINDS}
  for k in KINDS:
    for _ in range(10):
      launch[k]()
  for _ in range(args.repeats):
    for k in KINDS:
      ev[0].record()
      for _ in range(args.launches):
        launch[k]()
      ev[1].record()
      torch.cuda.synchronize()
      times[k].append(ev[0].elapsed_time(ev[1]) * 1e3 / args.launches)
  for k in KINDS:
    us = _median(times[k])
    bps = n * BYTES_PER_ELEM[k] / (us * 1e-6)
    print(json.dumps({"measure": "kernel", "kind": k, "elements": n,
                      "bytes_per_elem": BYTES_PER_ELEM[k], "us": us,
                      "spread_us": [min(times[k]), max(times[k])], "achieved_TBps": bps / 1e12,
                      "share_of_3.35TBps": bps / HBM_BYTES_PER_S, "gpu": gpu}), flush=True)


def _dlrm_trainer(kind, batch, sizes, dev):
  from distributed_embeddings_b200.models.dlrm import DLRM
  from distributed_embeddings_b200.models.dlrm_fast import DLRMTrainStep
  torch.manual_seed(1234)
  model = DLRM(sizes, device=dev, compute_dtype=torch.bfloat16, backend="fused")
  lr = {"sgd": 0.5, "adagrad": 0.05, "adam": 0.001}[kind]
  step = DLRMTrainStep(model, lr=lr, embedding_optimizer="sgd", dense_optimizer=kind)
  g = torch.Generator().manual_seed(99)
  data = []
  for _ in range(2):
    num = torch.rand(batch, 13, generator=g)
    cat = torch.stack([gen_ids(s, batch, 0.0, g) for s in sizes])
    lab = torch.randint(0, 2, (batch,), generator=g).float()
    data.append((num.to(dev), cat.to(dev), lab.to(dev)))
  return step, model, lambda i: step.step(*data[i % 2])


def _synthetic_trainer(kind, batch, dev):
  from distributed_embeddings_b200.models.configs import synthetic_models_v3
  from distributed_embeddings_b200.models.synthetic import InputGenerator, SyntheticModel
  from distributed_embeddings_b200.models.synthetic_fast import SyntheticTrainStep
  cfg = synthetic_models_v3["tiny"]
  torch.manual_seed(1234)
  model = SyntheticModel(cfg, device=dev, compute_dtype=torch.bfloat16, backend="fused")
  step = SyntheticTrainStep(model, lr=0.001, embedding_optimizer="adagrad", dense_optimizer=kind)
  gen = InputGenerator(cfg, batch, alpha=1.05, device=dev,
                       mp_input_ids=model.embedding.strategy.input_ids_list[0], num_batches=2)
  return step, model, lambda i: step.step(gen[i % 2][0][0], gen[i % 2][0][1], gen[i % 2][1])


def step_times(args, gpu):
  dev = torch.device("cuda", 0)
  sizes = table_sizes_for("dlrm-small")
  ev = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  for name in ("dlrm-small", "synthetic-tiny"):
    times = {k: [] for k in KINDS}
    for _ in range(args.repeats):
      for k in KINDS:
        if name == "dlrm-small":
          step, model, run = _dlrm_trainer(k, args.global_batch, sizes, dev)
        else:
          step, model, run = _synthetic_trainer(k, args.global_batch, dev)
        for i in range(args.warmup):
          run(i)
        torch.cuda.synchronize()
        ev[0].record()
        for i in range(args.steps):
          run(i)
        ev[1].record()
        torch.cuda.synchronize()
        times[k].append(ev[0].elapsed_time(ev[1]) / args.steps)
        step.ctx.check_errors()
        del step, model, run
        gc.collect()
        torch.cuda.empty_cache()
    base = _median(times["sgd"])
    for k in KINDS:
      ms = _median(times[k])
      print(json.dumps({"measure": "step", "model": name, "global_batch": args.global_batch,
                        "dense_optimizer": k, "ms_per_step": ms,
                        "spread_ms": [min(times[k]), max(times[k])],
                        "delta_vs_sgd_us": (ms - base) * 1e3, "repeats": args.repeats,
                        "gpu": gpu}), flush=True)


def main():
  ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawTextHelpFormatter)
  ap.add_argument("--repeats", type=int, default=3)
  ap.add_argument("--steps", type=int, default=20)
  ap.add_argument("--warmup", type=int, default=3)
  ap.add_argument("--launches", type=int, default=200)
  ap.add_argument("--global-batch", type=int, default=65536)
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("bench_dense_optimizer.py needs a CUDA GPU")
  torch.cuda.set_device(0)
  gpu = gpu_info()
  kernel_times(args, gpu)
  step_times(args, gpu)


if __name__ == "__main__":
  main()
