#!/usr/bin/env python
"""DLRM-DCNv2 on the hand-scheduled step: step time, and the cross network's kernels.

  python tools/bench_dcn.py [--batch 65536 8192] [--table-dtype bf16] [--repeats 3]
  python tools/bench_dcn.py --profile [--batch 65536 8192]

Step mode: ``DLRMTrainStep`` on ``DLRM(interaction="dcnv2")`` with the MLPerf layout (bottom MLP
512-256-128, 3 cross layers of rank 512 over D = 3456, top MLP 1024-1024-512-256-1) on the
``mlperf_table_sizes(20M)`` tables, MLPerf DLRM-DCNv2 hotness (214 ids per sample, uniform ids),
SGD.  Graph-replayed steps timed with CUDA events, ``--repeats`` times; prints the median and
min-max step time, samples/s and ``max_memory_allocated`` per batch size.

Profile mode (``--profile``, no tables): ``cross_fwd``, ``cross_bwd`` and ``cross_dx0`` (L = 3) at
``[batch, 3456]``, and the cross layer's six GEMMs, each timed with CUDA events over
``--launches`` launches.  Bytes are computed from the shapes (cross_fwd: 3 reads + 1 write,
cross_bwd: 2 + 1, cross_dx0: 2L + 1 + 1, bf16); achieved bandwidth is given against the H100 SXM
data-sheet HBM3 3.35 TB/s and the GEMMs' TFLOP/s against the 989 TFLOP/s dense bf16 peak.

Every line carries the card's name and power limit, read in the same run.  Needs a GPU.
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

HBM_BYTES_PER_S = 3.35e12
BF16_FLOPS = 989e12
D, RANK, LAYERS = 27 * 128, 512, 3


def gpu_info():
  out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True, check=True)
  name, power, clock = [x.strip() for x in out.stdout.splitlines()[0].split(",")]
  return {"name": name, "power_limit": power, "max_sm_clock": clock}


def _median(xs):
  xs = sorted(xs)
  return xs[len(xs) // 2]


def _time(fn, launches, repeats):
  ev = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  for _ in range(3):
    fn()
  times = []
  for _ in range(repeats):
    ev[0].record()
    for _ in range(launches):
      fn()
    ev[1].record()
    torch.cuda.synchronize()
    times.append(ev[0].elapsed_time(ev[1]) * 1e3 / launches)
  return _median(times), [min(times), max(times)]


def profile(args, gpu):
  from distributed_embeddings_b200.ops import _native
  ops = _native.require()
  dev = torch.device("cuda", 0)
  for b in args.batch:
    mk = lambda *s: torch.randn(*s, device=dev).bfloat16()
    x0, s, xl, out, dy, g = (mk(b, D) for _ in range(6))
    dys, ss = [mk(b, D) for _ in range(LAYERS)], [mk(b, D) for _ in range(LAYERS)]
    d_bottom = mk(b, 128)
    db = torch.zeros(D, device=dev)
    n = b * D
    kernels = {
        "cross_fwd": (lambda: ops.cross_fwd(x0, s, xl, out), 4 * n * 2),
        "cross_bwd": (lambda: ops.cross_bwd(dy, x0, g, db), 3 * n * 2 + D * 4),
        "cross_dx0": (lambda: ops.cross_dx0(dy, dys, ss, out, d_bottom), (2 * LAYERS + 2) * n * 2),
    }
    for name, (fn, nbytes) in kernels.items():
      us, spread = _time(fn, args.launches, args.repeats)
      bps = nbytes / (us * 1e-6)
      print(json.dumps({"measure": "kernel", "kernel": name, "batch": b, "D": D, "bytes": nbytes,
                        "us": us, "spread_us": spread, "achieved_TBps": bps / 1e12,
                        "share_of_3.35TBps": bps / HBM_BYTES_PER_S, "gpu": gpu}), flush=True)
    del dys, ss
    V, W, bW = mk(RANK, D), mk(D, RANK), mk(D)
    u, du = mk(b, RANK), mk(b, RANK)
    gW = torch.empty(D, RANK, device=dev)
    gV = torch.empty(RANK, D, device=dev)
    gemms = {
        "u = x V^T": lambda: torch.mm(xl, V.t(), out=u),
        "s = u W^T + b": lambda: torch.addmm(bW, u, W.t(), out=s),
        "gW = g^T u": lambda: torch.mm(g.t(), u, out_dtype=torch.float32, out=gW),
        "du = g W": lambda: torch.mm(g, W, out=du),
        "gV = du^T x": lambda: torch.mm(du.t(), xl, out_dtype=torch.float32, out=gV),
        "dx = dy + du V": lambda: torch.addmm(dy, du, V, out=out),
    }
    for name, fn in gemms.items():
      us, spread = _time(fn, max(1, args.launches // 4), args.repeats)
      flops = 2.0 * b * D * RANK
      print(json.dumps({"measure": "gemm", "gemm": name, "batch": b, "us": us,
                        "spread_us": spread, "TFLOPs": flops / (us * 1e-6) / 1e12,
                        "share_of_989": flops / (us * 1e-6) / BF16_FLOPS, "gpu": gpu}),
            flush=True)
    del x0, s, xl, out, dy, g, V, W, u, du, gW, gV
    gc.collect()
    torch.cuda.empty_cache()


def steps(args, gpu):
  from distributed_embeddings_b200.models.dlrm import (DLRM, MLPERF_DCNV2_MULTI_HOT_SIZES,
                                                       mlperf_table_sizes)
  from distributed_embeddings_b200.models.dlrm_fast import DLRMTrainStep
  dev = torch.device("cuda", 0)
  sizes = mlperf_table_sizes(20_000_000)
  hots = MLPERF_DCNV2_MULTI_HOT_SIZES
  tdt = {"fp32": torch.float32, "bf16": torch.bfloat16}[args.table_dtype]
  torch.manual_seed(1234)
  model = DLRM(sizes, device=dev, compute_dtype=torch.bfloat16, backend="fused", table_dtype=tdt,
               interaction="dcnv2", multi_hot_sizes=hots)
  step = DLRMTrainStep(model, lr=0.005, embedding_optimizer="sgd")
  ev = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  for b in args.batch:
    g = torch.Generator(device=dev).manual_seed(b)
    data = []
    for _ in range(2):
      num = torch.rand(b, 13, device=dev, generator=g)
      cat = [torch.randint(0, s, (b, h), device=dev, generator=g, dtype=torch.int32)
             for s, h in zip(sizes, hots)]
      lab = torch.randint(0, 2, (b,), device=dev, generator=g).float()
      data.append((num, cat, lab))
    torch.cuda.reset_peak_memory_stats()
    for i in range(args.warmup):
      step.step(*data[i % 2])
    times = []
    for _ in range(args.repeats):
      torch.cuda.synchronize()
      ev[0].record()
      for i in range(args.steps):
        step.step(*data[i % 2])
      ev[1].record()
      torch.cuda.synchronize()
      times.append(ev[0].elapsed_time(ev[1]) / args.steps)
    loss = float(step.loss)
    ms = _median(times)
    print(json.dumps({"measure": "step", "batch": b, "table_dtype": args.table_dtype,
                      "ids_per_sample": sum(hots), "ms_per_step": ms,
                      "spread_ms": [min(times), max(times)], "samples_per_s": b / (ms * 1e-3),
                      "max_memory_allocated_GiB": torch.cuda.max_memory_allocated() / 2**30,
                      "loss": loss, "repeats": args.repeats, "steps": args.steps, "gpu": gpu}),
          flush=True)
    del data
    gc.collect()


def main():
  ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawTextHelpFormatter)
  ap.add_argument("--batch", type=int, nargs="+", default=[65536, 8192])
  ap.add_argument("--table-dtype", default="bf16", choices=["fp32", "bf16"])
  ap.add_argument("--repeats", type=int, default=3)
  ap.add_argument("--steps", type=int, default=20)
  ap.add_argument("--warmup", type=int, default=3)
  ap.add_argument("--launches", type=int, default=100)
  ap.add_argument("--profile", action="store_true", help="time the cross kernels and GEMMs only")
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("bench_dcn.py needs a CUDA GPU")
  torch.cuda.set_device(0)
  gpu = gpu_info()
  if args.profile:
    profile(args, gpu)
  else:
    steps(args, gpu)


if __name__ == "__main__":
  main()
