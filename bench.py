#!/usr/bin/env python
"""Headline benchmark: DLRM (MLPerf Criteo-1TB configuration) training throughput.

``python bench.py --gpus N --steps K --warmup W`` (under torchrun for N > 1) runs K timed hybrid
parallel training steps (forward, loss, backward with the fused embedding update, dense gradient
all-reduce, dense SGD) at global batch 65536 and prints ONE JSON line from rank 0.

* ``value``: global samples/s, device timed (CUDA events), max over ranks.
* ``e2e``: the same metric through the public API with the per-step host->device copy of the
  inputs from pinned memory and the device->host read of the loss inside the timed region.
* ``--impl reference`` reports the unmodified reference (TensorFlow + Horovod) if importable.

Reference counterpart: examples/dlrm/main.py + examples/benchmarks/synthetic_models/main.py
(host wall-clock timing, :132-158); BASELINE.md for the published 8xA100 numbers.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
# more hardware queues than the default 8: the step overlaps kernels of ~6 streams (must be set
# before the CUDA context exists; the package sets the same default on import)
os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")

BASELINE_SAMPLES_PER_SEC = 10416232.0  # 8xA100 AMP, reference examples/dlrm/README.md:8


def parse_args():
  p = argparse.ArgumentParser()
  p.add_argument("--gpus", type=int, default=1)
  p.add_argument("--steps", type=int, default=50)
  p.add_argument("--warmup", type=int, default=10)
  p.add_argument("--impl", default="b200", choices=["b200", "reference"])
  p.add_argument("--global-batch", type=int, default=65536)
  p.add_argument("--model", default="dlrm-mlperf-20m",
                 help="dlrm-mlperf-20m (MLPerf tables capped at 20M rows: 49.6 GiB fp32, fits one "
                 "80 GB H100) | dlrm-mlperf (40M cap: 89.5 GiB, needs 2+ GPUs) | dlrm-small "
                 "(26x100000) | dlrm-tiny (26x1000)")
  p.add_argument("--backend", default="fused", choices=["fused", "torch"])
  p.add_argument("--optimizer", default="sgd")
  p.add_argument("--dtype", default="bf16", choices=["bf16", "fp32"])
  p.add_argument("--lr", type=float, default=24.0)
  p.add_argument("--data-batches", type=int, default=4)
  p.add_argument("--no-e2e", action="store_true")
  p.add_argument("--column-slice-threshold", default="auto",
                 help="elements, 'none', or 'auto' (default) = balance the looked-up columns per "
                 "rank with slices >= 64 wide: 2^32 at 8 GPUs, no slicing at 1-4")
  p.add_argument("--data-parallel-threshold", default="auto",
                 help="replicate tables with at most this many elements (the reference's "
                 "data_parallel_threshold): 'none', a number, or 'auto' (default) = 2500 rows x "
                 "128 at 2+ GPUs: the 11 MLPerf tables with < 2500 rows hold 0.003 %% of the "
                 "parameters but 42 %% of the lookups, replicating them takes 42 %% of the bytes "
                 "off NVLink and their hot rows off a single owner; no effect at 1 GPU")
  p.add_argument("--cuda-graph", type=int, default=1)
  p.add_argument("--gemm", default="cublas", choices=["cublas", "fused_dgrad", "tcgen05", "tcgen05_pair"],
                 help="MLP GEMM path of the fast trainer (see models/dlrm_fast.py)")
  p.add_argument("--profile", default=None, help="write a torch.profiler kernel table (rank 0)")
  p.add_argument("--profile-all-ranks", action="store_true",
                 help="with --profile: every rank writes its kernel table and a chrome trace")
  p.add_argument("--profile-graph", type=int, default=0,
                 help="1 = profile CUDA-graph replays (true device timeline, no launch skew)")
  p.add_argument("--trainer", default="fast", choices=["fast", "autograd"],
                 help="fast = hand-scheduled step + CUDA graph (DLRMTrainStep); autograd = "
                      "nn.Module + HybridTrainer")
  p.add_argument("--alpha", type=float, default=0.0,
                 help="power-law exponent of the synthetic ids (0 = uniform; the reference's "
                      "synthetic benchmark uses 1.05)")
  p.add_argument("--dump-outputs", default=None, metavar="DIR",
                 help="after the timed steps, write what the last timed step computed (rank 0) "
                      "as DIR/<name>.npy: see dump_outputs()")
  p.add_argument("--no-verify", action="store_true",
                 help="skip the pre-flight numerics check (2 steps of a 1/1000-rows plan on all "
                      "ranks vs a single-process fp32 PyTorch oracle on rank 0)")
  return p.parse_args()


def reference_arm(args):
  """Run the unmodified reference through its own API - only possible when TensorFlow and
  Horovod exist; this image has neither (no network), so report unavailability."""
  sys.path.insert(0, os.path.join(ROOT, "baseline", "_ref"))
  why = None
  try:
    import tensorflow  # noqa: F401  pylint: disable=unused-import,import-outside-toplevel
    import horovod.tensorflow  # noqa: F401  pylint: disable=unused-import,import-outside-toplevel
    import distributed_embeddings  # noqa: F401  pylint: disable=unused-import,import-outside-toplevel
  except Exception as e:  # pylint: disable=broad-except
    why = f"{type(e).__name__}: {e}"
  if why is None:
    why = "reference imported but its custom op library (_embedding_lookup_ops.so) is not built"
  rank = int(os.environ.get("RANK", "0"))
  if rank == 0:
    print(json.dumps({"impl": "reference",
                      "unavailable": "reference needs TensorFlow+Horovod (not in image, no "
                                     "network); python package installs to baseline/_ref but "
                                     f"cannot import: {why}"[:300]}))
  return 0


class ClockSampler:
  """Samples SM clocks / throttle reasons with nvidia-smi while the timed region runs."""

  FIELDS = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,"
            "clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
            "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")

  def __init__(self, gpu_index: int):
    self.gpu = gpu_index
    self.path = tempfile.mktemp(suffix=".csv")
    self.proc = None

  def start(self):
    try:
      self.proc = subprocess.Popen(
          ["nvidia-smi", f"--query-gpu={self.FIELDS}", "--format=csv,noheader,nounits", "-lms",
           "100", "-i", str(self.gpu)], stdout=open(self.path, "w"), stderr=subprocess.DEVNULL)
    except Exception:  # pylint: disable=broad-except
      self.proc = None

  def stop(self):
    if self.proc is None:
      return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
    time.sleep(0.15)
    self.proc.terminate()
    try:
      self.proc.wait(timeout=5)
    except Exception:  # pylint: disable=broad-except
      self.proc.kill()
    sm, mx, reasons = [], [], set()
    try:
      for line in open(self.path):
        f = [x.strip() for x in line.split(",")]
        if len(f) < 9:
          continue
        try:
          sm.append(float(f[1]))
          mx.append(float(f[2]))
        except ValueError:
          continue
        for name, val in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown",
                              "sw_power_cap"), f[5:9]):
          if val.lower().startswith("active"):
            reasons.add(name)
    except Exception:  # pylint: disable=broad-except
      pass
    finally:
      try:
        os.remove(self.path)
      except OSError:
        pass
    sm.sort()
    return {"sm_mhz": sm[len(sm) // 2] if sm else None, "sm_max_mhz": max(mx) if mx else None,
            "samples": len(sm), "reasons": sorted(reasons)}


# Criteo Terabyte cardinalities without the MLPerf 40 M cap (882 M rows, 421 GiB at dim 128 fp32:
# only fits sharded over 8 GPUs) - BASELINE.json's "~800M rows total" configuration
CRITEO_1TB_FULL_SIZES = [
    227605432, 39060, 17295, 7424, 20265, 3, 7122, 1543, 63, 130229467, 3067956, 405282, 10, 2209,
    11938, 155, 4, 976, 14, 292775614, 40790948, 187188510, 590152, 12973, 108, 36
]


def table_sizes_for(model: str):
  from distributed_embeddings_b200.models.dlrm import mlperf_table_sizes
  if model == "dlrm-mlperf":
    return mlperf_table_sizes()
  if model == "dlrm-mlperf-20m":
    return mlperf_table_sizes(max_rows=20_000_000)
  if model == "dlrm-full":
    return [s + 1 for s in CRITEO_1TB_FULL_SIZES]
  if model == "dlrm-small":
    return 26 * [100000]
  if model == "dlrm-tiny":
    return 26 * [1000]
  raise ValueError(model)


def auto_column_slice_threshold(sizes, dim, world, data_parallel_threshold=None):
  """Pick the column-slice threshold that minimises the most loaded rank's looked-up columns
  (gather bytes and NVLink bytes per sample are proportional to it); slices stay >= 64 wide.
  Replicated tables (``data_parallel_threshold``) do not take part in the exchange."""
  from distributed_embeddings_b200.parallel.strategy import DistEmbeddingStrategy
  cfgs = [{"input_dim": s, "output_dim": dim, "combiner": None} for s in sizes]
  best, best_cols = None, None
  for thr in [None] + [2**k for k in range(34, 22, -1)]:
    try:
      st = DistEmbeddingStrategy(cfgs, world, "memory_balanced", column_slice_threshold=thr,
                                 data_parallel_threshold=data_parallel_threshold
                                 if world > 1 else None)
    except ValueError:
      continue
    if any(not st.local_configs[r] for r in range(world)):
      continue
    if min(c["output_dim"] for r in range(world) for c in st.local_configs[r]) < 64:
      continue
    cols = max(sum(st.local_configs[r][m]["output_dim"] for m in st.local_maps[r])
               for r in range(world))
    if best_cols is None or cols < best_cols:
      best, best_cols = thr, cols
  return best


def gen_ids(rows: int, n: int, alpha: float, gen):
  """Synthetic categorical ids: uniform, or the reference generator's power law (alpha > 0)."""
  import torch
  if alpha <= 0:
    return torch.randint(0, rows, (n,), generator=gen, dtype=torch.int32)
  r = torch.rand(n, generator=gen, dtype=torch.float64)
  g = 1.0 - alpha
  y = (r * ((rows + 1.0)**g - 1.0) + 1.0)**(1.0 / g)
  return (y.to(torch.int64) - 1).clamp_(0, rows - 1).to(torch.int32)


def dump_outputs(out_dir, model, loss, max_bytes=64 << 20):
  """What a caller of the timed training step receives, as float32 .npy files: the step's loss
  (``loss``), the updated dense parameters (``bottom_mlp_<i>_weight`` / ``_bias``, ``top_mlp_...``)
  and the updated embedding rows of this rank's part of every table ``t`` (``embedding_<t>``, with
  ``_col<c>`` / ``_row<r>`` for column / row slices): all rows of a part with at most 1024 rows,
  else 1024 rows drawn with a generator seeded by ``t``, so the same rows are sampled in every
  run."""
  import numpy as np
  import torch
  os.makedirs(out_dir, exist_ok=True)
  arrays = {"loss": loss.detach().float().reshape(-1)}
  for part in ("bottom_mlp", "top_mlp"):
    lins = [m for m in getattr(model, part).net if isinstance(m, torch.nn.Linear)]
    for i, lin in enumerate(lins):
      arrays[f"{part}_{i}_weight"] = lin.weight.detach().float()
      arrays[f"{part}_{i}_bias"] = lin.bias.detach().float()
  # local tables of the same width are fused into one tensor: cut it back into the plan's tables
  emb, st = model.embedding, model.embedding.strategy
  weights = emb.weights
  n_dp, n_col = len(emb.dp_layers), len(emb.local_embedding_layers)
  parts = [(t, f"embedding_{t}", w) for t, w in zip(st.table_groups[0], weights[:n_dp])]
  for s in st.shards[emb.rank]:
    t = st.table_groups[1][s.table]
    full = s.width == int(st.global_configs[t]["output_dim"])
    name = f"embedding_{t}" if full else f"embedding_{t}_col{s.col_start}"
    parts.append((t, name, weights[n_dp + s.local_table][s.row_offset:s.row_offset + s.rows]))
  for gt, t in enumerate(st.table_groups[2]):
    parts.append((t, f"embedding_{t}_row{emb.rank}", weights[n_dp + n_col + gt]))
  for t, name, w in parts:
    w = w.detach()
    if w.shape[0] > 1024:
      g = torch.Generator().manual_seed(t)
      w = w[torch.randint(0, w.shape[0], (1024,), generator=g).to(w.device)]
    arrays[name] = w.float()
  total = sum(a.numel() * 4 for a in arrays.values())
  if total > max_bytes:
    raise ValueError(f"--dump-outputs: {total} bytes exceed the {max_bytes}-byte budget")
  for name, a in arrays.items():
    np.save(os.path.join(out_dir, name + ".npy"), a.cpu().numpy().astype(np.float32))
  return total


def verify(args, device, world, rank, compute_dtype, cst_for):
  """Pre-flight numerics check that the driver can see at every N: two training steps of a
  scaled-down plan (same 26 tables / MLPs / sharding knobs, 1/1000 of the rows) through the
  benchmarked trainer on all ranks, against a single-process fp32 PyTorch oracle on rank 0 that
  shares nothing with this framework but the initial weights (plain indexing, bmm interaction,
  nn.functional linear layers, autograd, in-place SGD)."""
  import torch
  import torch.distributed as dist
  from distributed_embeddings_b200.models.dlrm import DLRM

  sizes = [max(4, s // 1000) for s in table_sizes_for(args.model)]
  gbv, lr = 256 * world, 0.1
  lbv = gbv // world
  torch.manual_seed(4321)
  cst = cst_for(sizes)
  # same sharding knobs as the timed run, scaled with the rows (replicated tables included)
  dpt = args.data_parallel_threshold
  model = DLRM(sizes, device=device, compute_dtype=compute_dtype, backend=args.backend,
               column_slice_threshold=cst,
               data_parallel_threshold=max(4 * 128, dpt // 1000) if dpt else None)
  from distributed_embeddings_b200 import broadcast_variables
  broadcast_variables(model)
  # oracle copy of the initial state (rank 0 holds the global tables)
  w0 = model.embedding.get_weights()
  dense0 = [(m.weight.detach().float().clone(), m.bias.detach().float().clone())
            for m in list(model.bottom_mlp.net) + list(model.top_mlp.net)
            if isinstance(m, torch.nn.Linear)]
  n_bottom = sum(isinstance(m, torch.nn.Linear) for m in model.bottom_mlp.net)
  if args.trainer == "fast" and args.backend == "fused":
    from distributed_embeddings_b200.models.dlrm_fast import DLRMTrainStep
    trainer = DLRMTrainStep(model, lr=lr, embedding_optimizer="sgd",
                            use_cuda_graph=bool(args.cuda_graph), gemm=args.gemm)
  else:
    from distributed_embeddings_b200.models.trainer import HybridTrainer
    trainer = HybridTrainer(model, lr=lr, embedding_optimizer="sgd")
  g = torch.Generator().manual_seed(7 + rank)
  batches, losses = [], []
  for _ in range(2):
    num = torch.rand(lbv, 13, generator=g)
    cat = torch.stack([gen_ids(s, lbv, args.alpha, g) for s in sizes])
    lab = torch.randint(0, 2, (lbv, 1), generator=g).float()
    batches.append((num.to(device), cat.to(device), lab.to(device)))
  for num, cat, lab in batches:
    if args.trainer == "fast" and args.backend == "fused":
      loss = trainer.step(num, cat, lab)
    else:
      loss = trainer.step(num, list(cat.unbind(0)), lab)
    loss = loss.detach().float().reshape(1).clone()
    if world > 1:
      dist.all_reduce(loss)
      loss /= world
    losses.append(float(loss.item()))
  w1 = model.embedding.get_weights()
  # global batches on rank 0
  glob = []
  for num, cat, lab in batches:
    if world > 1:
      parts = [[torch.empty_like(t) for _ in range(world)] for t in (num, cat, lab)]
      for p, t in zip(parts, (num, cat, lab)):
        dist.all_gather(p, t.contiguous())
      glob.append((torch.cat(parts[0]), torch.cat(parts[1], dim=1), torch.cat(parts[2])))
    else:
      glob.append((num, cat, lab))
  result = None
  if rank == 0:
    n = len(sizes) + 1
    ii, jj = torch.tril_indices(n, n, offset=-1)
    ii, jj = ii.to(device), jj.to(device)

    def oracle(autocast_dtype):
      """Plain PyTorch training of the same model on the global batch: fp32 throughout, or the
      same code under torch.autocast (the precision policy of the benchmarked trainer)."""
      tabs = [torch.from_numpy(w).to(device).requires_grad_(True) for w in w0]
      dense = [(w.clone().requires_grad_(True), b.clone().requires_grad_(True))
               for w, b in dense0]
      params = tabs + [t for wb in dense for t in wb]
      olosses = []
      for num, cat, lab in glob:
        with torch.autocast("cuda", dtype=autocast_dtype or torch.bfloat16,
                            enabled=autocast_dtype is not None):
          x = num
          for w, b in dense[:n_bottom]:
            x = torch.relu(torch.nn.functional.linear(x, w, b))
          embs = [tabs[t][cat[t].long()].to(x.dtype) for t in range(len(sizes))]
          feats = torch.stack([x] + embs, dim=1)
          z = torch.bmm(feats, feats.transpose(1, 2))[:, ii, jj]
          h = torch.cat([z, x], dim=1)
          top = dense[n_bottom:]
          for i, (w, b) in enumerate(top):
            h = torch.nn.functional.linear(h, w, b)
            if i < len(top) - 1:
              h = torch.relu(h)
        loss = torch.nn.functional.binary_cross_entropy_with_logits(h.float(), lab)
        olosses.append(float(loss.item()))
        grads = torch.autograd.grad(loss, params)
        with torch.no_grad():
          for p, gr in zip(params, grads):
            p -= lr * gr
      return [t.detach() for t in tabs], olosses

    def compare(tabs):
      max_err, max_upd, sq_err, sq_upd = 0.0, 0.0, 0.0, 0.0
      for t in range(len(sizes)):
        got = torch.from_numpy(w1[t]).to(device)
        init = torch.from_numpy(w0[t]).to(device)
        err, upd = got - tabs[t], tabs[t] - init
        max_err = max(max_err, float(err.abs().max()))
        max_upd = max(max_upd, float(upd.abs().max()))
        sq_err += float((err.double()**2).sum())
        sq_upd += float((upd.double()**2).sum())
      return max_err, max_upd, (sq_err / max(sq_upd, 1e-30))**0.5

    # The trainer computes the dense side in bf16: against the fp32 oracle the two-step table
    # update agrees to ~10 % (aggregate L2; bf16 has 8 mantissa bits and the error compounds
    # through 9 layers and the second step), against the same plain-PyTorch code under bf16
    # autocast to a few % (the hand-written kernels round at other places than autocast does;
    # the values of a run are in its JSON line's "verify" key).  A wrong routing / missing rank
    # contribution / wrong gradient scale shows up as an error of the order of the update itself
    # (~1.0) against both.
    tabs32, ol32 = oracle(None)
    tabs16, ol16 = oracle(compute_dtype if compute_dtype != torch.float32 else None)
    e32, u32, r32 = compare(tabs32)
    e16, _, r16 = compare(tabs16)
    loss_err = max(abs(a - b) for a, b in zip(losses, ol32))
    tol32, tol16 = 0.30, 0.20
    result = {"max_abs_err": e32, "max_update": u32,
              "rel_l2_err_of_update": r32, "rel_l2_tolerance": tol32,
              "rel_l2_err_vs_autocast_oracle": r16, "rel_l2_tolerance_autocast": tol16,
              "max_abs_err_vs_autocast_oracle": e16,
              "loss": losses, "oracle_loss": ol32, "autocast_oracle_loss": ol16,
              "loss_abs_err": loss_err,
              "tables_rows": int(sum(sizes)), "global_batch": gbv, "steps": 2, "lr": lr,
              "oracle": "single-process plain PyTorch on rank 0: fp32, and the same code under "
                        "autocast(" + str(compute_dtype).replace("torch.", "") + ")",
              "ok": bool(r32 <= tol32 and r16 <= tol16 and loss_err <= 3e-2 and u32 > 0)}
  flag = torch.tensor([1 if (result is None or result["ok"]) else 0], device=device)
  if world > 1:
    dist.broadcast(flag, src=0)
  del trainer, model
  torch.cuda.empty_cache()
  return result, bool(flag.item())


def main():
  args = parse_args()
  if args.impl == "reference":
    return reference_arm(args)

  import torch
  import torch.distributed as dist

  world = int(os.environ.get("WORLD_SIZE", "1"))
  rank = int(os.environ.get("RANK", "0"))
  local_rank = int(os.environ.get("LOCAL_RANK", "0"))
  if world != args.gpus and world > 1:
    args.gpus = world
  torch.cuda.set_device(local_rank)
  device = torch.device("cuda", local_rank)
  if world > 1:
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    dist.init_process_group("nccl", device_id=device)

  from distributed_embeddings_b200.models.dlrm import DLRM
  from distributed_embeddings_b200.models.trainer import HybridTrainer
  from distributed_embeddings_b200.ops import _native

  torch.manual_seed(1234)  # same dense init on every rank (then broadcast anyway)
  sizes = table_sizes_for(args.model)
  compute_dtype = torch.bfloat16 if args.dtype == "bf16" else torch.float32
  gb = args.global_batch
  assert gb % world == 0
  lb = gb // world
  dpt = args.data_parallel_threshold
  if dpt is None or str(dpt).lower() == "none":
    dpt = None
  elif str(dpt).lower() == "auto":
    dpt = 2500 * 128 if (world >= 2 and args.optimizer == "sgd" and
                          args.trainer == "fast" and args.backend == "fused") else None
  else:
    dpt = int(dpt)
  args.data_parallel_threshold = dpt
  cst = args.column_slice_threshold
  if cst == "auto":
    cst = auto_column_slice_threshold(sizes, 128, world, dpt)
  elif cst is None or str(cst).lower() == "none":
    cst = None
  else:
    cst = int(cst)
  verify_result, verify_ok = None, True
  if not args.no_verify:
    raw_cst = args.column_slice_threshold

    def cst_for(vsizes):
      if raw_cst == "auto":
        return auto_column_slice_threshold(vsizes, 128, world,
                                           max(4 * 128, dpt // 1000) if dpt else None)
      if raw_cst is None or str(raw_cst).lower() == "none":
        return None
      return max(1, int(raw_cst) // 1000)
    verify_result, verify_ok = verify(args, device, world, rank, compute_dtype, cst_for)
    if not verify_ok:
      if rank == 0:
        print(json.dumps({"verify": verify_result, "error": "numerics check failed"}))
      if world > 1:
        dist.destroy_process_group()
      return 3
  torch.manual_seed(1234)
  model = DLRM(sizes, device=device, compute_dtype=compute_dtype, backend=args.backend,
               column_slice_threshold=cst, data_parallel_threshold=args.data_parallel_threshold)
  from distributed_embeddings_b200 import broadcast_variables
  broadcast_variables(model)
  use_fast = args.trainer == "fast" and args.backend == "fused"
  # the reference's schedule (examples/dlrm/main.py:192-197): SGD lr 24 reached after 8000
  # warm-up steps, polynomial decay from step 48000; the learning rate lives in device memory so
  # the captured step follows it
  from distributed_embeddings_b200.utils.lr_schedule import LearningRateScheduler
  scheduler = LearningRateScheduler(args.lr, warmup_steps=8000, decay_start_step=48000,
                                    decay_steps=24000)
  if use_fast:
    from distributed_embeddings_b200.models.dlrm_fast import DLRMTrainStep
    trainer = DLRMTrainStep(model, lr=args.lr, embedding_optimizer=args.optimizer,
                            use_cuda_graph=bool(args.cuda_graph), gemm=args.gemm,
                            scheduler=scheduler)
  else:
    trainer = HybridTrainer(model, lr=args.lr, embedding_optimizer=args.optimizer,
                            scheduler=scheduler)

  # ---- synthetic Criteo-shaped data in pinned host memory (uniform ids, random-init tables)
  n_feat = len(sizes)
  g = torch.Generator().manual_seed(99 + rank)
  pool = []
  for _ in range(args.data_batches):
    num = torch.rand(lb, 13, generator=g).pin_memory()
    cat = torch.stack([gen_ids(s, lb, args.alpha, g)
                       for s in sizes]).pin_memory()  # [26, lb] feature major = staging layout
    lab = torch.randint(0, 2, (lb, 1), generator=g).float().pin_memory()
    pool.append((num, cat, lab))
  h2d_bytes = sum(t.numel() * t.element_size() for t in pool[0])

  fused = args.backend == "fused"
  engine = None
  if use_fast:
    engine = trainer.engine
  elif fused:
    from distributed_embeddings_b200.parallel.fused import FusedEngine
    model.embedding._engine = FusedEngine(model.embedding)
    engine = model.embedding._engine
    engine.prepare(lb, [1] * n_feat, ids64=False)
    cat_stage = engine.in_flat[:n_feat * lb].view(n_feat, lb)
  num_d = torch.empty(lb, 13, device=device)
  lab_d = torch.empty(lb, 1, device=device)
  dev_pool = [(n.to(device), c.to(device), l.to(device)) for n, c, l in pool]

  dev_i = [0]

  def step_from_device(i):
    if use_fast:
      # device-resident batches go through the same double-buffered input pipeline as the end
      # to end loop (copies on the copy stream, one select kernel inside the captured step)
      if dev_i[0] == 0:
        trainer.prefetch(*dev_pool[0])
      loss = trainer.run_prefetched()
      dev_i[0] += 1
      trainer.prefetch(*dev_pool[dev_i[0] % len(dev_pool)])
      return loss
    n, c, l = dev_pool[i % len(dev_pool)]
    if fused:
      cat_stage.copy_(c)
      return trainer.step(n, None, l, staged=True)
    return trainer.step(n, list(c.unbind(0)), l)

  # End-to-end loop: every step copies its inputs from pinned host memory and every step's loss
  # is read back to the host.  The read-back is pipelined by one step (async D2H into pinned
  # memory + event), the standard way to log a metric without stalling the launch queue.
  loss_host = torch.zeros(2, 1, dtype=torch.float32).pin_memory()
  loss_events = [torch.cuda.Event(), torch.cuda.Event()]
  e2e_losses = []

  def step_e2e(i):
    n, c, l = pool[i % len(pool)]
    if use_fast:
      # asynchronous input pipeline: batch i was copied (pinned host -> device) on the copy
      # stream while step i-1 ran; batch i+1 is enqueued now and overlaps step i
      if i == 0:
        trainer.prefetch(n, c, l)
      loss = trainer.run_prefetched()
      if i + 1 < args.steps:
        n2, c2, l2 = pool[(i + 1) % len(pool)]
        trainer.prefetch(n2, c2, l2)
      slot = i & 1
      loss_host[slot].copy_(loss.reshape(1), non_blocking=True)
      loss_events[slot].record()
      if i > 0:
        loss_events[slot ^ 1].synchronize()
        e2e_losses.append(float(loss_host[slot ^ 1]))
      if i == args.steps - 1:  # the last step's loss is read inside the timed region as well
        loss_events[slot].synchronize()
        e2e_losses.append(float(loss_host[slot]))
      return None
    num_d.copy_(n, non_blocking=True)
    lab_d.copy_(l, non_blocking=True)
    if fused:
      cat_stage.copy_(c, non_blocking=True)
      loss = trainer.step(num_d, None, lab_d, staged=True)
    else:
      cd = c.to(device, non_blocking=True)
      loss = trainer.step(num_d, list(cd.unbind(0)), lab_d)
    return float(loss.item())  # device -> host read of the step result

  def sync_all():
    torch.cuda.synchronize()
    if world > 1:
      dist.barrier()
      torch.cuda.synchronize()

  last_out = [None]

  def timed(fn, steps):
    sync_all()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for i in range(steps):
      last_out[0] = fn(i)
    end.record()
    sync_all()
    ms = torch.tensor([start.elapsed_time(end)], device=device)
    if world > 1:
      dist.all_reduce(ms, op=dist.ReduceOp.MAX)
    return float(ms.item())

  for i in range(max(3, args.warmup)):
    step_from_device(i)
  sampler = ClockSampler(local_rank)
  if rank == 0:
    sampler.start()
  _native.reset_launch_count()
  total_ms = timed(step_from_device, args.steps)
  if args.dump_outputs and rank == 0:
    dump_outputs(args.dump_outputs, model, last_out[0])
  launches = _native.launch_count()
  if use_fast and args.cuda_graph:
    # kernels replayed from the captured graph are not seen by the python-side counter:
    # count one eager pass of the same schedule
    _native.reset_launch_count()
    trainer._step_impl()
    launches = _native.launch_count() * args.steps
    torch.cuda.synchronize()
  clocks = sampler.stop() if rank == 0 else None
  # the timed steps trained for real: the last loss must be a finite number
  final_loss = step_from_device(0).detach().float().reshape(1).clone()
  if world > 1:
    dist.all_reduce(final_loss)
    final_loss /= world
  final_loss = float(final_loss.item())
  if final_loss != final_loss or abs(final_loss) == float("inf"):
    if rank == 0:
      print(json.dumps({"error": "training diverged: non-finite loss after the timed steps",
                        "final_loss": str(final_loss)}))
    if world > 1:
      dist.destroy_process_group()
    return 4

  if args.profile:
    from torch.profiler import ProfilerActivity, profile
    saved = getattr(trainer, "use_cuda_graph", None)
    if saved is not None and not args.profile_graph:
      trainer.use_cuda_graph = False
    for i in range(3):
      step_from_device(i)
    sync_all()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
      for i in range(5):
        step_from_device(i)
      sync_all()
    if rank == 0 or args.profile_all_ranks:
      # rank 0 -> the given path, other ranks -> path.rankN (the per-rank tables and traces are
      # what shows which rank the barriers / all-reduce are waiting for)
      path = args.profile if rank == 0 else f"{args.profile}.rank{rank}"
      os.makedirs(os.path.dirname(path) or ".", exist_ok=True)
      with open(path, "w") as f:
        f.write(f"# {args.model} world={world} rank={rank} global_batch={gb}, 5 steps, "
                f"{'graph replay' if args.profile_graph else 'eager (no graph)'}\n")
        f.write(prof.key_averages().table(sort_by="cuda_time_total", row_limit=40,
                                          max_name_column_width=70))
      if args.profile_all_ranks:
        prof.export_chrome_trace(f"{path}.trace.json")
    if saved is not None:
      trainer.use_cuda_graph = saved

  e2e = None
  if not args.no_e2e:
    if use_fast:  # build + capture the staged schedule outside the timed region
      for i in range(3):
        trainer.prefetch(*pool[i % len(pool)])
        trainer.run_prefetched()
    else:
      for i in range(3):
        step_e2e(i)
    e2e_ms = timed(step_e2e, args.steps)
    e2e = {"value": gb * args.steps / (e2e_ms / 1e3), "unit": "samples/s",
           "ms_per_step": e2e_ms / args.steps, "h2d_bytes_per_step": h2d_bytes * world,
           "d2h_bytes_per_step": 4 * world}
  if engine is not None:
    engine.ctx.check_errors()

  if rank == 0:
    ms_per_step = total_ms / args.steps
    value = gb / (ms_per_step / 1e3)
    table_gb = sum(sizes) * 128 * 4 / 2**30
    out = {
        "metric": "DLRM global samples/sec (device-timed, max over ranks)",
        "value": value,
        "unit": "samples/s",
        "n_gpus": world,
        "steps": args.steps,
        "warmup": max(3, args.warmup),
        "ms_per_step": ms_per_step,
        "higher_is_better": True,
        "scaling": "strong",
        "vs_baseline": value / BASELINE_SAMPLES_PER_SEC,
        "dtype": args.dtype,
        "data": "synthetic (" + ("uniform" if args.alpha <= 0 else f"power-law alpha={args.alpha}") +
                " Criteo-shaped ids, random-init tables)",
        "impl": "b200",
        "config": {
            "model": f"DLRM {args.model}: 26 tables dim 128 ({sum(sizes)} rows, "
                     f"{table_gb:.1f} GiB fp32), bottom 512-256-128, top 1024-1024-512-256-1",
            "global_batch": gb,
            "seq_len": 1,
            "parallelism": f"hybrid: dp{world} dense + table-parallel embeddings "
                           f"(memory_balanced, column_slice_threshold={cst}, data_parallel_threshold={args.data_parallel_threshold}), backend={args.backend}, trainer={args.trainer}, cuda_graph={int(bool(args.cuda_graph))}, mlp_gemm={args.gemm}, dense_allreduce={getattr(trainer, 'allreduce_kind', 'torch')}",
            "optimizer": f"{args.optimizer} lr={args.lr}, warm-up 8000 / decay from 48000 steps "
                         "like the reference (embedding update fused in backward)",
            "l2_policy": "inputs larger than L2: random rows of "
                         f"{table_gb / world:.1f} GiB tables per GPU vs 50 MB L2",
        },
        "clocks": clocks,
        "e2e": e2e,
        "gpu_launches": launches,
        "final_loss": final_loss,
        "e2e_final_loss": e2e_losses[-1] if e2e_losses else None,
        "verify": verify_result,
    }
    print(json.dumps(out))
  if world > 1:
    dist.destroy_process_group()
  return 0


if __name__ == "__main__":
  sys.exit(main())
