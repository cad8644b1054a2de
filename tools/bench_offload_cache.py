#!/usr/bin/env python
"""Where the HBM row cache of offloaded tables pays off: the DLRM step (``DLRMTrainStep``, CUDA
graph, fp32 tables, one GPU) of ``dlrm-mlperf-20m`` with

  * every table in HBM (no offload),
  * the largest tables in pinned host memory, read and updated zero-copy (offload, no cache),
  * the same offload with caches of ``--cache-fracs`` of the offloaded rows,

each at uniform ids and at the power law of ``--alphas``, repeats alternating over the id
distributions.  Prints one JSON line per (setting, ids) and a table: ms / step, the cache's hit
rate (unique rows, ``offload_cache_stats``) and the PCIe bytes per step (cache: fills, spills and
write-backs x row and state bytes; no cache: every offloaded lookup plus a read and a write of
every unique updated row).  The card's name and power limit are read in the same run.

  python tools/bench_offload_cache.py                       # defaults below
  python tools/bench_offload_cache.py --host-gib 20 --steps 20
"""
import argparse
import gc
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from distributed_embeddings_b200.models.dlrm import DLRM, mlperf_table_sizes  # noqa: E402
from distributed_embeddings_b200.models.dlrm_fast import DLRMTrainStep  # noqa: E402


def gen_ids(rows, n, alpha, gen):
  """Uniform ids, or the reference generator's power law (alpha > 0)."""
  if alpha <= 0:
    return torch.randint(0, rows, (n,), generator=gen, dtype=torch.int32)
  r = torch.rand(n, generator=gen, dtype=torch.float64)
  g = 1.0 - alpha
  y = (r * ((rows + 1.0)**g - 1.0) + 1.0)**(1.0 / g)
  return (y.to(torch.int64) - 1).clamp_(0, rows - 1).to(torch.int32)


def card():
  try:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=30, check=False).stdout
    return out.strip().splitlines()[0]
  except (OSError, IndexError, subprocess.SubprocessError):
    return torch.cuda.get_device_name(0) + ", power limit unknown"


def offload_plan(sizes, dim, host_gib):
  """gpu_embedding_size that sends the largest tables (as many as fit ``host_gib`` of fp32 rows
  and their optimizer state) to the host; returns (budget, offloaded table indices)."""
  order = sorted(range(len(sizes)), key=lambda t: -sizes[t])
  off, gib = [], 0.0
  for t in order:
    g = sizes[t] * dim * 4 / 2**30
    if gib + g > host_gib:
      break
    off.append(t)
    gib += g
  budget = sum(s for t, s in enumerate(sizes) if t not in off) * dim
  return budget, sorted(off)


def main(argv=None):
  ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawTextHelpFormatter)
  ap.add_argument("--max-rows", type=int, default=20_000_000, help="row cap of the MLPerf tables")
  ap.add_argument("--batch", type=int, default=65536)
  ap.add_argument("--steps", type=int, default=20, help="timed steps per repeat")
  ap.add_argument("--warmup", type=int, default=3)
  ap.add_argument("--repeats", type=int, default=2)
  ap.add_argument("--batches", type=int, default=8, help="distinct batches the steps cycle over")
  ap.add_argument("--alphas", default="0,1.05", help="0 = uniform ids")
  ap.add_argument("--cache-fracs", default="0.02,0.1,0.5",
                  help="cache sizes as fractions of the offloaded rows")
  ap.add_argument("--host-gib", type=float, default=None,
                  help="GiB of tables to offload (default: 40 %% of the host's memory, <= 40)")
  ap.add_argument("--lr", type=float, default=0.01)
  args = ap.parse_args(argv)
  if not torch.cuda.is_available():
    raise SystemExit("bench_offload_cache.py measures the GPU step: no CUDA device found")
  dev = torch.device("cuda", 0)
  torch.cuda.set_device(dev)
  host_gib = args.host_gib
  if host_gib is None:
    phys = os.sysconf("SC_PAGE_SIZE") * os.sysconf("SC_PHYS_PAGES") / 2**30
    host_gib = min(0.4 * phys, 40.0)
  sizes = mlperf_table_sizes(args.max_rows)
  dim = 128
  budget, off = offload_plan(sizes, dim, host_gib)
  off_rows = sum(sizes[t] for t in off)
  print(f"card: {card()}")
  print(f"offloaded tables {off}: " +
        ", ".join(f"{sizes[t] * dim * 4 / 2**30:.2f} GiB" for t in off) +
        f" (total {off_rows * dim * 4 / 2**30:.2f} GiB, {off_rows} rows)")
  if not off:
    raise SystemExit("no table fits --host-gib")
  alphas = [float(a) for a in args.alphas.split(",")]
  settings = [("no offload", None, None), ("offload", budget, None)]
  settings += [(f"cache {f:g}", budget, int(f * off_rows) * dim)
               for f in (float(x) for x in args.cache_fracs.split(","))]
  g = torch.Generator().manual_seed(0)
  b = args.batch
  data = {}
  for a in alphas:
    data[a] = [(torch.rand(b, 13, generator=g).to(dev),
                torch.stack([gen_ids(s, b, a, g) for s in sizes]).to(dev),
                torch.randint(0, 2, (b,), generator=g).float().to(dev))
               for _ in range(args.batches)]
  # host-side traffic accounting of the zero-copy path: lookups and unique rows of the
  # offloaded tables per batch
  zc = {a: sum(b * len(off) + sum(int(torch.unique(cat[t]).numel()) for t in off)
               for _, cat, _ in data[a]) / args.batches for a in alphas}
  row_bytes = dim * 4
  results = []
  for name, gpu_size, cache in settings:
    torch.manual_seed(0)
    model = DLRM(sizes, device=dev, compute_dtype=torch.bfloat16, backend="fused",
                 gpu_embedding_size=gpu_size, offload_cache_size=cache)
    t = DLRMTrainStep(model, lr=args.lr, embedding_optimizer="sgd", use_cuda_graph=True)
    times = {a: [] for a in alphas}
    stats = {a: [0, 0, 0, 0] for a in alphas}
    for _ in range(args.repeats):
      for a in alphas:
        bs = data[a]
        for i in range(args.warmup):
          t.step(*bs[i % len(bs)])
        model.embedding.offload_cache_stats(reset=True)
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        for i in range(args.steps):
          t.step(*bs[i % len(bs)])
        end.record()
        torch.cuda.synchronize()
        times[a].append(start.elapsed_time(end) / args.steps)
        for s in model.embedding.offload_cache_stats(reset=True):
          for k, key in enumerate(("hits", "misses", "spills", "writebacks")):
            stats[a][k] += s[key]
    for a in alphas:
      n = args.repeats * args.steps
      hits, misses, spills, wbs = (x / n for x in stats[a])
      if cache is not None:
        pcie = (misses + wbs) * row_bytes
        hit = hits / max(hits + misses, 1)
      elif gpu_size is not None:
        pcie, hit = zc[a] * row_bytes + 0.0, None
        # zc counts one read per lookup and one per unique row; the update also writes it back
        pcie += (zc[a] - b * len(off)) * row_bytes
      else:
        pcie, hit = 0.0, None
      rec = {"setting": name, "ids": "uniform" if a <= 0 else f"alpha {a:g}",
             "ms_per_step": round(min(times[a]), 3), "ms_all": [round(x, 3) for x in times[a]],
             "hit_rate": None if hit is None else round(hit, 4),
             "spills_per_step": round(spills, 1) if cache is not None else None,
             "pcie_mb_per_step": round(pcie / 1e6, 1), "cache_elems": cache,
             "offloaded_tables": off if gpu_size is not None else []}
      results.append(rec)
      print(json.dumps(rec), flush=True)
    del t, model
    gc.collect()
    torch.cuda.empty_cache()
  print(f"\n{'setting':<12} {'ids':<11} {'ms/step':>8} {'hit rate':>9} {'PCIe MB/step':>13}")
  for r in results:
    hr = "-" if r["hit_rate"] is None else f"{r['hit_rate']:.3f}"
    print(f"{r['setting']:<12} {r['ids']:<11} {r['ms_per_step']:>8.3f} {hr:>9} "
          f"{r['pcie_mb_per_step']:>13.1f}")
  print(f"card: {card()}")
  return results


if __name__ == "__main__":
  main()
