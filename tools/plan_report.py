#!/usr/bin/env python
"""Sizing a sharding plan without GPUs: which tables land where, how many bytes each rank holds,
gathers and sends per step, and how unbalanced the plan is.

  python tools/plan_report.py --model dlrm-mlperf --world 8 --data-parallel-threshold 320000
  python tools/plan_report.py --model small --world 8 --strategy traffic_balanced
  python tools/plan_report.py --tables 1000000x128,5000x64,250000000x128 --world 4 \\
      --column-slice-threshold auto --hbm-gib 79

Uses the same planner the run would use (``DistEmbeddingStrategy``, ``traffic_report``,
``memory_report``); nothing is allocated.
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from distributed_embeddings_b200.models.configs import expand, synthetic_models_v3  # noqa: E402
from distributed_embeddings_b200.models.dlrm import mlperf_table_sizes  # noqa: E402
from distributed_embeddings_b200.parallel.offload_cache import cache_bytes, split_budget  # noqa: E402
from distributed_embeddings_b200.parallel.strategy import (DistEmbeddingStrategy,  # noqa: E402
                                                           suggest_column_slice_threshold)


def model_tables(args):
  """-> (configs, input_table_map, hotness)"""
  if args.tables:
    cfgs = []
    for item in args.tables.split(","):
      rows, width = item.lower().split("x")
      cfgs.append({"input_dim": int(rows), "output_dim": int(width), "combiner": "sum"})
    return cfgs, None, None
  if args.model.startswith("dlrm"):
    sizes = {"dlrm-mlperf": mlperf_table_sizes(), "dlrm-small": 26 * [100000],
             "dlrm-tiny": 26 * [1000]}[args.model]
    return [{"input_dim": s, "output_dim": 128, "combiner": None} for s in sizes], None, None
  tables, imap, hots = expand(synthetic_models_v3[args.model])[:3]
  cfgs = [{"input_dim": r, "output_dim": w, "combiner": "sum"} for r, w in tables]
  return cfgs, list(imap), list(hots)


def _thr(v):
  if v is None or str(v).lower() == "none":
    return None
  return v if str(v).lower() == "auto" else int(v)


def main(argv=None):
  ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawTextHelpFormatter)
  ap.add_argument("--model", default="dlrm-mlperf",
                  help="dlrm-mlperf | dlrm-small | dlrm-tiny | " + " | ".join(synthetic_models_v3))
  ap.add_argument("--tables", default=None, help="explicit list ROWSxWIDTH,ROWSxWIDTH,...")
  ap.add_argument("--world", type=int, default=8)
  ap.add_argument("--strategy", default="memory_balanced")
  ap.add_argument("--column-slice-threshold", default=None)
  ap.add_argument("--row-slice-threshold", default=None)
  ap.add_argument("--data-parallel-threshold", default=None)
  ap.add_argument("--global-batch", type=int, default=65536)
  ap.add_argument("--hbm-gib", type=float, default=79.0, help="per-GPU memory to check against")
  ap.add_argument("--optimizer-slots", type=int, default=0,
                  help="state copies per table element (adagrad 1, adam 2)")
  ap.add_argument("--optimizer-row-slots", type=int, default=0,
                  help="fp32 state words per table row of the model-parallel tables (row-wise "
                       "adagrad 1 with --optimizer-slots 0, row-wise adam 1 with --optimizer-slots "
                       "1)")
  ap.add_argument("--state-dtype", default="fp32", choices=["fp32", "bf16"],
                  help="storage of the element-wise Adagrad / Adam / row-wise Adam state of the "
                       "model-parallel tables (set_optimizer(state_dtype=...)); row words and "
                       "replicated tables stay fp32")
  ap.add_argument("--table-dtype", default="fp32", choices=["fp32", "bf16", "fp16"],
                  help="storage of the model-parallel tables (DistributedEmbedding(table_dtype="
                       "...)): their table and gather bytes at its element size; optimizer slots "
                       "and replicated tables stay fp32")
  ap.add_argument("--gpu-embedding-size", type=int, default=None,
                  help="per-rank HBM element budget of the table-parallel tables; the largest "
                       "beyond it go to pinned host memory")
  ap.add_argument("--offload-cache-size", type=int, default=None,
                  help="per-rank HBM element budget of the cache of the offloaded tables' rows "
                       "(fp32 tables): its weight, optimizer-state and spill-region slots are "
                       "reported as cache GiB and counted in HBM GiB")
  ap.add_argument("--json", action="store_true")
  args = ap.parse_args(argv)

  cfgs, imap, hots = model_tables(args)
  if args.offload_cache_size is not None and (args.gpu_embedding_size is None or
                                             args.table_dtype != "fp32"):
    ap.error("--offload-cache-size needs --gpu-embedding-size and fp32 tables")
  if args.offload_cache_size is not None and args.state_dtype != "fp32":
    ap.error("--offload-cache-size needs fp32 optimizer state")
  kw = dict(input_table_map=imap, row_slice_threshold=_thr(args.row_slice_threshold),
            data_parallel_threshold=_thr(args.data_parallel_threshold),
            gpu_embedding_size=args.gpu_embedding_size)
  cst = _thr(args.column_slice_threshold)
  if cst == "auto":
    cst = suggest_column_slice_threshold(cfgs, args.world, args.strategy, hotness=hots,
                                         input_hotness=hots, **kw)
  st = DistEmbeddingStrategy(cfgs, args.world, args.strategy, column_slice_threshold=cst,
                             input_hotness=hots, **kw)
  mem = st.memory_report()
  tr = st.traffic_report(args.global_batch, hots)
  esz = 4 if args.table_dtype == "fp32" else 2
  ssz = 4 if args.state_dtype == "fp32" else 2
  per_elem = esz + ssz * args.optimizer_slots     # model-parallel tables
  per_elem_dp = 4 * (1 + args.optimizer_slots)    # replicated tables are always fp32
  dp_elems = sum(int(c["input_dim"]) * int(c["output_dim"]) for c in st.dp_configs)
  hot = hots or [1] * len(st.input_table_map)
  dp_gather = 0  # bytes gathered from the replicated tables per rank (local batch, fp32 rows)
  for j, gi in enumerate(st.input_groups[0]):
    t = st.table_groups[0][st.map_groups[0][j]]
    dp_gather += args.global_batch // args.world * hot[gi] * int(st.global_configs[t]["output_dim"]) * 4
  ranks = []

  def cache_gib(r):
    """HBM of rank r's offload caches: the budget split like DistributedEmbedding splits it,
    each table's spill region sized to its owner-side batch x hotness."""
    if args.offload_cache_size is None or not st.table_groups[1]:
      return 0.0
    spill = {}
    for li, g in enumerate(st.input_ids_list[r]):
      m = st.local_maps[r][li]
      if st.local_configs[r][m].get("cpu_offload"):
        spill[m] = spill.get(m, 0) + args.global_batch * hot[st.input_groups[1][g]]
    ms = sorted(spill)
    shapes = [(int(st.local_configs[r][m]["input_dim"]), int(st.local_configs[r][m]["output_dim"]))
              for m in ms]
    sets = split_budget(args.offload_cache_size, shapes)
    return sum(cache_bytes(n, spill[m], w, [w] * args.optimizer_slots +
                           [1] * args.optimizer_row_slots)
               for n, m, (_, w) in zip(sets, ms, shapes)) / 2**30

  def row_gib(r):
    """(HBM, host) GiB of rank r's fp32 row words: one per slot and local row of a
    model-parallel table (table-parallel, column slices, row slices)."""
    hbm = host = 0
    if st.table_groups[1]:
      for c in st.local_configs[r]:
        if c.get("cpu_offload"):
          host += int(c["input_dim"])
        else:
          hbm += int(c["input_dim"])
    for gt in range(len(st.table_groups[2])):
      lo, hi = st.row_ranges[gt][r]
      hbm += hi - lo
    words = 4 * args.optimizer_row_slots
    return hbm * words / 2**30, host * words / 2**30

  for r in range(args.world):
    n_tab = len(st.local_configs[r]) if st.table_groups[1] else 0
    cols = sum(int(st.local_configs[r][m]["output_dim"]) for m in st.local_maps[r]) \
        if st.table_groups[1] else 0
    cgib = cache_gib(r)
    rgib, rhost = row_gib(r)
    gib = ((mem[r]["hbm_elements"] - dp_elems) * per_elem + dp_elems * per_elem_dp) / 2**30 + \
        cgib + rgib
    gather = (tr["ranks"][r]["gather_bytes"] - dp_gather) * esz / 4 + dp_gather
    ranks.append({"rank": r, "fused_tables": n_tab, "inputs": len(st.input_ids_list[r]),
                  "exchanged_columns": cols, "hbm_gib": round(gib, 2),
                  "host_gib": round(mem[r]["host_elements"] * per_elem / 2**30 + rhost, 2),
                  "cache_gib": round(cgib, 6),
                  "gather_mb": round(gather / 1e6, 1),
                  "nvlink_out_mb": round(tr["ranks"][r]["nvlink_out_bytes"] / 1e6, 1),
                  "lookups": int(tr["ranks"][r]["lookups"]),
                  "fits": gib <= args.hbm_gib})
  rep = {"world": args.world, "strategy": args.strategy, "column_slice_threshold": cst,
         "table_dtype": args.table_dtype, "state_dtype": args.state_dtype,
         "tables": len(cfgs), "replicated": len(st.table_groups[0]),
         "table_parallel": len(st.table_groups[1]), "row_sliced": len(st.table_groups[2]),
         "gather_imbalance": round(tr["gather_imbalance"], 3),
         "nvlink_imbalance": round(tr["nvlink_imbalance"], 3), "ranks": ranks}
  if args.optimizer_row_slots:
    rep["optimizer_row_slots"] = args.optimizer_row_slots
  if args.json:
    print(json.dumps(rep))
    return rep
  print(f"{len(cfgs)} tables on {args.world} ranks, strategy {args.strategy}, "
        f"column_slice_threshold {cst}, {args.table_dtype} tables, {args.state_dtype} state: "
        f"{rep['replicated']} replicated, "
        f"{rep['table_parallel']} table-parallel, {rep['row_sliced']} row-sliced")
  print(f"{'rank':>4} {'tables':>7} {'inputs':>7} {'columns':>8} {'HBM GiB':>9} {'host GiB':>9} "
        f"{'cache GiB':>10} {'gather MB':>10} {'NVLink out MB':>14} {'lookups':>12}")
  for x in ranks:
    flag = "" if x["fits"] else f"   > {args.hbm_gib:g} GiB!"
    print(f"{x['rank']:>4} {x['fused_tables']:>7} {x['inputs']:>7} {x['exchanged_columns']:>8} "
          f"{x['hbm_gib']:>9.2f} {x['host_gib']:>9.2f} {x['cache_gib']:>10.3f} {x['gather_mb']:>10.1f} "
          f"{x['nvlink_out_mb']:>14.1f} {x['lookups']:>12}{flag}")
  print(f"imbalance (max / mean): gather {rep['gather_imbalance']}, "
        f"NVLink {rep['nvlink_imbalance']}  (per step, global batch {args.global_batch})")
  return rep


if __name__ == "__main__":
  main()
