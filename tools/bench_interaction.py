#!/usr/bin/env python
"""Device time and HBM traffic of the DLRM dot-interaction kernels at the step's shapes.

  python tools/bench_interaction.py [--batch 65536] [--n-emb 26] [--dim 128]
                                    [--applied 0,5,10,15] [--table-rows 20000000]
                                    [--iters 20] [--warmup 5] [--repeats 5]

Times, through the production ops (``interact_fwd`` / ``interact_bwd``):
  * ``fwd``: the forward, z = [tril(F F^T, -1) | bottom | 0 pad];
  * ``bwd``: the backward without the table update (every gradient row stored to a local
    [batch, n_emb * dim] buffer);
  * ``bwd_apply<k>``: the backward with the SGD update of the first k features reduced into fp32
    tables of ``--table-rows`` rows by the kernel (k = 0 is the same launch as ``bwd``).
The applied features read uniform ids over tables of the real row count, so that the reductions
miss L2 as they do in the step.  Five 20M-row fp32 tables (51 GB) are allocated and feature f
updates table f % 5.

Each timing is CUDA events around ``--iters`` back-to-back launches after ``--warmup`` launches;
the configurations alternate within each of ``--repeats`` repeats and the median is reported.
Bytes are the compulsory HBM traffic computed from the shapes (feature rows, dz, dbottom and the
routed gradient rows, ids, and a read and a write of every applied fp32 table row) and the share
is of the 3.35 TB/s data-sheet bandwidth of the H100 SXM.  The card's name, power limit and SM
clocks are read in the same run (``nvidia-smi --query-gpu``, read only).  Prints one JSON line.
Needs a GPU.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
N_TABLES = 5


def gpu_info():
  out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True, check=True)
  name, power, clock, max_clock = [x.strip() for x in out.stdout.splitlines()[0].split(",")]
  return {"name": name, "power_limit": power, "sm_clock": clock, "max_sm_clock": max_clock}


def z_width(n_emb: int, dim: int) -> int:
  return (n_emb * (n_emb + 1) // 2 + dim + 7) // 8 * 8


def traffic_bytes(kind: str, batch: int, n_emb: int, dim: int, applied: int = 0) -> int:
  """Compulsory HBM bytes of one launch."""
  feat = (n_emb + 1) * dim * 2
  dz = z_width(n_emb, dim) * 2
  if kind == "fwd":
    return batch * (feat + dz)
  routed = (n_emb - applied) * dim * 2
  table_rmw = applied * (2 * dim * 4 + 4)  # fp32 row read + write, int32 id
  return batch * (feat + dz + dim * 2 + routed + table_rmw)


def apply_descs(tables, ids, applied: int, n_emb: int) -> torch.Tensor:
  from distributed_embeddings_b200.ops._native import INPUT_DESC
  d = np.zeros(n_emb, dtype=INPUT_DESC)
  for f in range(applied):
    t = tables[f % len(tables)]
    d[f]["table"] = t.data_ptr()
    d[f]["ids"] = ids[f].data_ptr()
    d[f]["sub_rows"] = t.shape[0]
    d[f]["width"] = t.shape[1]
    d[f]["hotness"] = 1
  return torch.from_numpy(d.view(np.uint8).copy())


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--batch", type=int, default=65536)
  ap.add_argument("--n-emb", type=int, default=26)
  ap.add_argument("--dim", type=int, default=128)
  ap.add_argument("--applied", default="0,5,10,15")
  ap.add_argument("--table-rows", type=int, default=20_000_000)
  ap.add_argument("--iters", type=int, default=20)
  ap.add_argument("--warmup", type=int, default=5)
  ap.add_argument("--repeats", type=int, default=5)
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit("bench_interaction.py needs a GPU")
  from distributed_embeddings_b200.ops import _native
  ops = _native.require()
  dev = torch.device("cuda", 0)
  b, n, d = args.batch, args.n_emb, args.dim
  applied = [int(x) for x in args.applied.split(",") if x != ""]
  if any(k > n for k in applied):
    raise SystemExit("--applied cannot exceed --n-emb")
  g = torch.Generator(device=dev).manual_seed(7)
  bf = torch.bfloat16
  bottom = torch.randn(b, d, generator=g, device=dev).to(bf)
  emb = torch.randn(b, n * d, generator=g, device=dev).to(bf)
  zw = z_width(n, d)
  z = torch.zeros(b, zw, dtype=bf, device=dev)
  dz = (torch.randn(b, zw, generator=g, device=dev) * 0.01).to(bf)
  dbottom = torch.empty(b, d, dtype=bf, device=dev)
  demb = torch.empty(b, n * d, dtype=bf, device=dev)
  tables, ids = [], []
  if any(k > 0 for k in applied):
    if d != 128:
      raise SystemExit("the table update needs --dim 128")
    tables = [torch.zeros(args.table_rows, d, dtype=torch.float32, device=dev)
              for _ in range(min(N_TABLES, max(applied)))]
    ids = [torch.randint(0, args.table_rows, (b,), generator=g, device=dev, dtype=torch.int32)
           for _ in range(max(applied))]

  def bwd(descs):
    extra = (descs, -1e-3, 0, False) if descs is not None else ()
    ops.interact_bwd(bottom, emb, n, dz, dbottom, demb.data_ptr(), demb.stride(0), 1.0, None, 0,
                     [], None, 0, *extra)

  configs = {"fwd": (lambda: ops.interact_fwd(bottom, emb, n, z, []),
                     traffic_bytes("fwd", b, n, d))}
  configs["bwd"] = (lambda: bwd(None), traffic_bytes("bwd", b, n, d))
  for k in applied:
    descs = apply_descs(tables, ids, k, n) if k > 0 else None
    configs[f"bwd_apply{k}"] = ((lambda dd=descs: bwd(dd)), traffic_bytes("bwd", b, n, d, k))

  times = {name: [] for name in configs}
  start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  for _ in range(args.repeats):
    for name, (fn, _) in configs.items():
      for _ in range(args.warmup):
        fn()
      torch.cuda.synchronize()
      start.record()
      for _ in range(args.iters):
        fn()
      end.record()
      torch.cuda.synchronize()
      times[name].append(start.elapsed_time(end) * 1e3 / args.iters)
  results = []
  for name, (_, nbytes) in configs.items():
    ts = sorted(times[name])
    med = ts[len(ts) // 2]
    results.append({"kernel": name, "us_median": round(med, 2), "us_min": round(ts[0], 2),
                    "us_max": round(ts[-1], 2), "bytes": nbytes,
                    "tb_per_s": round(nbytes / med * 1e-6, 3),
                    "share_of_3.35TBps": round(nbytes / med * 1e6 / HBM_BYTES_PER_S, 3)})
  print(json.dumps({"gpu": gpu_info(), "batch": b, "n_emb": n, "dim": d,
                    "table_rows": args.table_rows, "iters": args.iters,
                    "repeats": args.repeats, "results": results}))


if __name__ == "__main__":
  main()
