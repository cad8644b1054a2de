#!/usr/bin/env python
"""Benchmark of the synthetic model zoo (reference examples/benchmarks/synthetic_models/main.py).

  torchrun --nproc-per-node 8 --master-addr 127.0.0.1 examples/benchmarks/synthetic_models/main.py \
      --model small --optimizer adagrad --dense_optimizer adagrad --batch_size 65536 --alpha 1.05

The reference applies one optimizer to every variable: its configuration is
``--optimizer adagrad --dense_optimizer adagrad``.  The default ``--dense_optimizer sgd`` updates
the MLP with SGD at the embedding optimizer's learning rate.

Differences from the reference driver: timing is on the device (CUDA events), max over ranks, and
the embedding optimizer runs fused inside the backward kernels.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
sys.path.insert(0, ROOT)

import torch
import torch.distributed as dist

import distributed_embeddings_b200 as de
from distributed_embeddings_b200.models.configs import scaled, summary, synthetic_models_v3
from distributed_embeddings_b200.models.synthetic import (InputGenerator, SyntheticModel,
                                                           SyntheticModelNative)
from distributed_embeddings_b200.models.dense_optimizer import KINDS as DENSE_OPTIMIZERS
from distributed_embeddings_b200.models.trainer import HybridTrainer
from distributed_embeddings_b200.parallel.embedding_optimizers import NAMES as EMBEDDING_OPTIMIZERS


def main():
  p = argparse.ArgumentParser()
  p.add_argument("--batch_size", type=int, default=4, help="Global batch size")
  p.add_argument("--num_data_batches", type=int, default=1)
  p.add_argument("--alpha", type=float, default=1.05, help="power-law exponent, 0 = uniform")
  p.add_argument("--num_steps", type=int, default=100)
  p.add_argument("--dp_input", action="store_true")
  p.add_argument("--model", default="tiny", choices=sorted(synthetic_models_v3))
  p.add_argument("--optimizer", default="sgd", choices=EMBEDDING_OPTIMIZERS)
  p.add_argument("--dense_optimizer", default="sgd", choices=list(DENSE_OPTIMIZERS),
                 help="optimizer of the MLP (--embedding_api de); the reference uses --optimizer's")
  p.add_argument("--momentum", type=float, default=0.9,
                 help="momentum of the 'momentum' optimizers (torch.optim.SGD's, dampening 0)")
  p.add_argument("--nesterov", action="store_true",
                 help="Nesterov momentum for the 'momentum' optimizers")
  p.add_argument("--column_slice_threshold", type=int, default=None)
  p.add_argument("--row_slice_threshold", type=int, default=None)
  p.add_argument("--data_parallel_threshold", type=int, default=None)
  p.add_argument("--embedding_api", default="de", choices=["native", "de"])
  p.add_argument("--dist_strategy", default="memory_balanced",
                 choices=["basic", "memory_balanced", "memory_optimized", "traffic_balanced"],
                 help="placement; traffic_balanced evens out the per-rank lookups of the "
                 "multi-hot features (memory_balanced is what the reference benchmark uses)")
  p.add_argument("--amp", action="store_true", help="bf16 activations / MLP")
  p.add_argument("--table_dtype", default="fp32", choices=["bf16", "fp16", "fp32"],
                 help="storage of the model-parallel embedding tables (--embedding_api de)")
  p.add_argument("--optimizer_state_dtype", default="fp32", choices=["fp32", "bf16"],
                 help="storage of the Adagrad / Adam state of the model-parallel tables "
                      "(--embedding_api de; bf16: half the memory, stochastically rounded)")
  p.add_argument("--backend", default="auto", choices=["auto", "fused", "torch"])
  p.add_argument("--row_scale", type=float, default=1.0, help="shrink tables (smoke runs)")
  p.add_argument("--device", default=None)
  p.add_argument("--cuda_graph", type=int, default=1, help="capture the whole step in a CUDA graph")
  p.add_argument("--trainer", default="auto", choices=["auto", "fast", "autograd"],
                 help="fast = hand-scheduled static step (SyntheticTrainStep); autograd = "
                 "nn.Module + HybridTrainer; auto = fast when the model / back end allow it")
  args = p.parse_args()

  world = int(os.environ.get("WORLD_SIZE", "1"))
  rank = int(os.environ.get("RANK", "0"))
  local_rank = int(os.environ.get("LOCAL_RANK", "0"))
  use_cuda = torch.cuda.is_available() and args.device != "cpu"
  device = torch.device("cuda", local_rank) if use_cuda else torch.device("cpu")
  if use_cuda:
    torch.cuda.set_device(device)
  if world > 1:
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    dist.init_process_group("nccl" if use_cuda else "gloo",
                            device_id=device if use_cuda else None)
  if args.batch_size % world:
    raise ValueError(f"Batch size ({args.batch_size}) is not divisible by world size ({world})")

  cfg = synthetic_models_v3[args.model]
  if args.row_scale != 1.0:
    cfg = scaled(cfg, args.row_scale)
  dtype = torch.bfloat16 if args.amp else torch.float32
  if args.embedding_api == "de":
    model = SyntheticModel(cfg, column_slice_threshold=args.column_slice_threshold,
                           dp_input=args.dp_input, device=device, compute_dtype=dtype,
                           backend=args.backend, row_slice_threshold=args.row_slice_threshold,
                           data_parallel_threshold=args.data_parallel_threshold,
                           strategy=args.dist_strategy,
                           table_dtype={"fp32": torch.float32, "bf16": torch.bfloat16,
                                        "fp16": torch.float16}[args.table_dtype])
    mp_ids = None if args.dp_input else model.embedding.strategy.input_ids_list[rank]
  else:
    if not args.dp_input or args.column_slice_threshold is not None:
      raise ValueError("Model parallel inputs and column slicing need --embedding_api de")
    model = SyntheticModelNative(cfg, device=device, compute_dtype=dtype)
    mp_ids = None
  gen = InputGenerator(cfg, args.batch_size, alpha=args.alpha, mp_input_ids=mp_ids,
                       num_batches=args.num_data_batches, world_size=world, rank=rank,
                       device=device)
  de.broadcast_variables(model)

  if args.embedding_api == "de":
    lr = {"sgd": 0.03, "adagrad": 0.001, "rowwise_adagrad": 0.001, "adam": 0.001,
          "rowwise_adam": 0.001, "ftrl": 0.01, "momentum": 0.01}[args.optimizer]
    opt_kwargs = {"state_dtype": {"fp32": torch.float32,
                                  "bf16": torch.bfloat16}[args.optimizer_state_dtype]}
    momentum = {"momentum": args.momentum, "nesterov": args.nesterov}
    if args.optimizer == "momentum":
      opt_kwargs.update(momentum)
    dense_kwargs = momentum if args.dense_optimizer == "momentum" else None
    from distributed_embeddings_b200.models.synthetic_fast import SyntheticTrainStep
    why = SyntheticTrainStep.unsupported_reason(model) if use_cuda else "needs CUDA"
    if args.trainer == "fast" and why:
      raise ValueError(f"--trainer fast: {why}")
    if args.trainer != "autograd" and not why:
      trainer = SyntheticTrainStep(model, lr=lr, embedding_optimizer=args.optimizer,
                                   use_cuda_graph=bool(args.cuda_graph),
                                   dense_optimizer=args.dense_optimizer,
                                   dense_optimizer_kwargs=dense_kwargs,
                                   embedding_optimizer_kwargs=opt_kwargs)
      trainer_kind = "fast"
    else:
      trainer = HybridTrainer(model, lr=lr, embedding_optimizer=args.optimizer,
                              use_cuda_graph=bool(args.cuda_graph) and use_cuda,
                              dense_optimizer=args.dense_optimizer,
                              dense_optimizer_kwargs=dense_kwargs,
                              embedding_optimizer_kwargs=opt_kwargs)
      trainer_kind = "autograd"
    step = lambda num, cat, lab: trainer.step(num, cat, lab)
  else:
    opt = {"sgd": lambda ps: torch.optim.SGD(ps, lr=0.03),
           "adagrad": lambda ps: torch.optim.Adagrad(ps, lr=0.001),
           "adam": lambda ps: torch.optim.Adam(ps, lr=0.001)}[args.optimizer](model.parameters())
    dopt = de.DistributedOptimizer(opt)
    bce = torch.nn.BCEWithLogitsLoss()

    def step(num, cat, lab):
      dopt.zero_grad()
      loss = bce(model(num, cat).float(), lab)
      loss.backward()
      dopt.step()
      return loss.detach()

  def sync():
    if use_cuda:
      torch.cuda.synchronize()
    if world > 1:
      dist.barrier()

  (num, cat), lab = gen[-1]
  for _ in range(5):
    loss = step(num, cat, lab)
  sync()
  if rank == 0:
    print(f"Initial loss: {float(loss):.3f}")
  if use_cuda:
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
  else:
    import time
    start = time.time()
  for i in range(args.num_steps):
    (num, cat), lab = gen[i % args.num_data_batches]
    loss = step(num, cat, lab)
    if i % 50 == 0 and rank == 0:
      print(f"Benchmark step [{i}/{args.num_steps}]")
  if use_cuda:
    t1.record()
    sync()
    ms = torch.tensor([t0.elapsed_time(t1)], device=device)
    if world > 1:
      dist.all_reduce(ms, op=dist.ReduceOp.MAX)
    ms = float(ms) / args.num_steps
  else:
    sync()
    ms = (time.time() - start) * 1000 / args.num_steps
  if rank == 0:
    print(f"loss: {float(loss):.3f}")
    print(f"Iteration time: {ms:.3f} ms")
    print(json.dumps({"model": args.model, "n_gpus": world, "batch_size": args.batch_size,
                      "ms_per_iter": ms, "samples_per_sec": args.batch_size / ms * 1e3,
                      "optimizer": args.optimizer,
                      "dense_optimizer": args.dense_optimizer if args.embedding_api == "de"
                                         else args.optimizer,
                      "trainer": trainer_kind if args.embedding_api == "de" else "native",
                      **summary(cfg)}))
  if world > 1:
    dist.destroy_process_group()


if __name__ == "__main__":
  main()
