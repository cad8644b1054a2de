#!/usr/bin/env python
"""DLRM training with hybrid-parallel embeddings (reference examples/dlrm/main.py).

  torchrun --nproc-per-node 8 --master-addr 127.0.0.1 examples/dlrm/main.py \
      --dataset_path /data/criteo_split_binary        # real data (split binary Criteo)
  python examples/dlrm/main.py --num_batches 100                       # synthetic data
  python examples/dlrm/main.py --interaction dcnv2 --multi_hot_sizes mlperf   # DLRM-DCNv2

Embeddings are model parallel (memory_balanced placement), MLPs data parallel; SGD lr 24 with
warm-up + polynomial decay; AUC on the eval split; embedding weights saved with np.savez in the
global (sharding independent) layout.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

import numpy as np
import torch
import torch.distributed as dist

import distributed_embeddings_b200 as de
from distributed_embeddings_b200.models.dense_optimizer import KINDS as DENSE_OPTIMIZERS
from distributed_embeddings_b200.models.dlrm import DLRM, MLPERF_DCNV2_MULTI_HOT_SIZES
from distributed_embeddings_b200.models.trainer import HybridTrainer
from distributed_embeddings_b200.parallel.embedding_optimizers import NAMES as EMBEDDING_OPTIMIZERS
from distributed_embeddings_b200.utils.criteo import DummyDataset, RawBinaryDataset
from distributed_embeddings_b200.utils.lr_schedule import LearningRateScheduler
from distributed_embeddings_b200.utils.metrics import binary_auc


TABLE_DTYPES = {"fp32": torch.float32, "bf16": torch.bfloat16, "fp16": torch.float16}
STATE_DTYPES = {"fp32": torch.float32, "bf16": torch.bfloat16}


def parse():
  p = argparse.ArgumentParser()
  p.add_argument("--dataset_path", default=None, help="dir with model_size.json + train/ test/")
  p.add_argument("--learning_rate", type=float, default=24)
  p.add_argument("--batch_size", type=int, default=64 * 1024, help="global batch size")
  p.add_argument("--top_mlp_dims", default="1024,1024,512,256,1")
  p.add_argument("--bottom_mlp_dims", default="512,256,128")
  p.add_argument("--num_numerical_features", type=int, default=13)
  p.add_argument("--num_batches", type=int, default=340, help="synthetic train batches")
  p.add_argument("--table_sizes", default=",".join(["1000"] * 26))
  p.add_argument("--embedding_dim", type=int, default=128)
  p.add_argument("--dp_input", action="store_true")
  p.add_argument("--test_combiner", action="store_true")
  p.add_argument("--dist_strategy", default="memory_balanced")
  p.add_argument("--interaction", default="dot", choices=["dot", "dcnv2"],
                 help="pairwise dot interaction (DLRM) or low-rank cross network (DLRM-DCNv2)")
  p.add_argument("--dcn_num_layers", type=int, default=3)
  p.add_argument("--dcn_low_rank_dim", type=int, default=512)
  p.add_argument("--multi_hot_sizes", default=None,
                 help="ids per sample of every feature (comma-separated, or 'mlperf' for the "
                      "MLPerf DLRM-DCNv2 hotness); synthetic data only, the split-binary reader "
                      "is one-hot")
  p.add_argument("--fast", action="store_true", help="hand-scheduled step + CUDA graph")
  p.add_argument("--eval_interval", type=int, default=0,
                 help="with --fast: every N training steps, evaluate --eval_batches batches of "
                      "the eval split on the GPU (binned AUC, log loss); 0 = off")
  p.add_argument("--eval_batches", type=int, default=8,
                 help="eval batches per periodic evaluation (--eval_interval)")
  p.add_argument("--eval_auc", choices=("binned", "exact"), default="binned",
                 help="with --eval_interval: binned = 8000-threshold ROC AUC (the reference's "
                      "metric); exact = exact ROC AUC from sorted keys on the GPU (4 bytes per "
                      "eval sample), with the binned value beside it")
  p.add_argument("--amp", action="store_true", default=True)
  p.add_argument("--gpu_embedding_size", type=int, default=None,
                 help="per-rank HBM element budget of the tables; the largest beyond it live in "
                      "pinned host memory")
  p.add_argument("--offload_cache_size", type=int, default=None,
                 help="per-rank HBM element budget of the cache of the offloaded tables' rows")
  p.add_argument("--table_dtype", default="fp32", choices=sorted(TABLE_DTYPES),
                 help="storage of the model-parallel embedding tables (bf16 / fp16: half the "
                      "memory, stochastically rounded updates)")
  p.add_argument("--embedding_optimizer", default="sgd",
                 choices=EMBEDDING_OPTIMIZERS,
                 help="fused optimizer of the model-parallel tables")
  p.add_argument("--dense_optimizer", default="sgd", choices=list(DENSE_OPTIMIZERS),
                 help="optimizer of the MLPs (and of replicated tables, which need the embedding "
                      "optimizer's kind)")
  p.add_argument("--momentum", type=float, default=0.9,
                 help="momentum of the 'momentum' optimizers (torch.optim.SGD's, dampening 0)")
  p.add_argument("--nesterov", action="store_true",
                 help="Nesterov momentum for the 'momentum' optimizers")
  p.add_argument("--optimizer_state_dtype", default="fp32", choices=["fp32", "bf16"],
                 help="storage of the Adagrad / Adam / FTRL / momentum state (row-wise Adam: its "
                      "m) of the model-parallel tables (bf16: half the memory, stochastically "
                      "rounded)")
  p.add_argument("--weight_decay", type=float, default=0.0,
                 help="weight decay of the embedding and the dense optimizer (rows a step "
                      "touched / every dense parameter)")
  p.add_argument("--weight_decay_mode", default="l2", choices=["l2", "decoupled"],
                 help="l2: added to the gradient; decoupled: AdamW-style, the weights are scaled "
                      "by 1 - lr * weight_decay before the step (not with ftrl)")
  p.add_argument("--warmup_steps", type=int, default=8000)
  p.add_argument("--decay_start_step", type=int, default=48000)
  p.add_argument("--decay_steps", type=int, default=24000)
  p.add_argument("--epochs", type=int, default=1)
  p.add_argument("--save_path", default="/tmp/embedding_weights")
  p.add_argument("--save_dir", default=None,
                 help="write one global-layout .npy per table into this directory instead; every "
                      "rank writes its own slices in parallel (no gather to rank 0)")
  return p.parse_args()


def main():
  args = parse()
  world = int(os.environ.get("WORLD_SIZE", "1"))
  rank = int(os.environ.get("RANK", "0"))
  local_rank = int(os.environ.get("LOCAL_RANK", "0"))
  cuda = torch.cuda.is_available()
  device = torch.device("cuda", local_rank) if cuda else torch.device("cpu")
  if cuda:
    torch.cuda.set_device(device)
  if world > 1:
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    dist.init_process_group("nccl" if cuda else "gloo", device_id=device if cuda else None)

  if args.dataset_path is not None:
    with open(os.path.join(args.dataset_path, "model_size.json"), encoding="utf-8") as f:
      table_sizes = [s + 1 for s in json.load(f).values()]
  else:
    table_sizes = [int(s) for s in args.table_sizes.split(",")]
  hotness = None
  if args.multi_hot_sizes is not None:
    if args.dataset_path is not None:
      raise SystemExit("--multi_hot_sizes needs synthetic data: the split-binary reader is one-hot")
    hotness = list(MLPERF_DCNV2_MULTI_HOT_SIZES) if args.multi_hot_sizes == "mlperf" else \
        [int(h) for h in args.multi_hot_sizes.split(",")]

  model = DLRM(table_sizes, embedding_dim=args.embedding_dim,
               bottom_mlp_dims=[int(d) for d in args.bottom_mlp_dims.split(",")],
               top_mlp_dims=[int(d) for d in args.top_mlp_dims.split(",")],
               num_numerical_features=args.num_numerical_features, dp_input=args.dp_input,
               dist_strategy=args.dist_strategy, test_combiner=args.test_combiner, device=device,
               compute_dtype=torch.bfloat16 if (args.amp and cuda) else torch.float32,
               table_dtype=TABLE_DTYPES[args.table_dtype], interaction=args.interaction,
               gpu_embedding_size=args.gpu_embedding_size,
               offload_cache_size=args.offload_cache_size,
               dcn_num_layers=args.dcn_num_layers, dcn_low_rank_dim=args.dcn_low_rank_dim,
               multi_hot_sizes=hotness)
  table_ids = list(range(len(table_sizes))) if args.dp_input else \
      model.embedding.strategy.input_ids_list[rank]
  lbs = args.batch_size // world
  if args.dataset_path is not None:
    kw = dict(batch_size=args.batch_size, numerical_features=args.num_numerical_features,
              categorical_features=table_ids, categorical_feature_sizes=table_sizes,
              prefetch_depth=10, drop_last_batch=True, offset=lbs * rank, lbs=lbs,
              dp_input=args.dp_input)
    train = RawBinaryDataset(args.dataset_path, **kw)
    evald = RawBinaryDataset(args.dataset_path, valid=True, **kw)
  else:
    hots = [hotness[t] for t in table_ids] if hotness is not None else None
    train = DummyDataset(args.batch_size, args.num_numerical_features, world, len(table_ids), True,
                         args.dp_input, args.num_batches, hots)
    evald = DummyDataset(args.batch_size, args.num_numerical_features, world, len(table_ids),
                         False, args.dp_input, max(1, args.num_batches // 10), hots)

  sched = LearningRateScheduler(args.learning_rate, warmup_steps=args.warmup_steps,
                                decay_start_step=args.decay_start_step,
                                decay_steps=args.decay_steps)
  de.broadcast_variables(model)
  fast = args.fast and cuda and args.dp_input
  opt_kwargs = {"state_dtype": STATE_DTYPES[args.optimizer_state_dtype]}
  dense_kwargs = {}
  momentum = {"momentum": args.momentum, "nesterov": args.nesterov}
  if args.embedding_optimizer == "momentum":
    opt_kwargs.update(momentum)
  if args.dense_optimizer == "momentum":
    dense_kwargs.update(momentum)
  if args.weight_decay:
    decay = {"weight_decay": args.weight_decay, "weight_decay_mode": args.weight_decay_mode}
    opt_kwargs.update(decay)
    dense_kwargs.update(decay)
  if args.eval_interval > 0 and not fast:
    raise SystemExit("--eval_interval needs the hand-scheduled step: --fast with --dp_input on "
                     "a GPU")
  if fast:
    from distributed_embeddings_b200.models.dlrm_fast import DLRMTrainStep
    trainer = DLRMTrainStep(model, lr=args.learning_rate, scheduler=sched,
                            embedding_optimizer=args.embedding_optimizer,
                            embedding_optimizer_kwargs=opt_kwargs,
                            dense_optimizer=args.dense_optimizer,
                            dense_optimizer_kwargs=dense_kwargs, eval_auc=args.eval_auc,
                            eval_capacity=(args.eval_batches * args.batch_size
                                           if args.eval_auc == "exact" else None))
    if args.interaction == "dcnv2":  # list of [b, h_f] ids
      step = lambda n, c, l: trainer.step(n, [x.to(torch.int32) for x in c], l)
    else:
      step = lambda n, c, l: trainer.step(n, torch.stack([x.to(torch.int32) for x in c]), l)
  else:
    trainer = HybridTrainer(model, lr=args.learning_rate, scheduler=sched,
                            embedding_optimizer=args.embedding_optimizer,
                            embedding_optimizer_kwargs=opt_kwargs,
                            dense_optimizer=args.dense_optimizer,
                            dense_optimizer_kwargs=dense_kwargs)
    step = trainer.step

  def batches():
    for _ in range(args.epochs):
      yield from train

  def periodic_eval(i):
    """Binned AUC (8000 thresholds, as the reference reports; --eval_auc exact: the exact AUC)
    and log loss on the GPU."""
    for k, (num, cat, lab) in enumerate(evald):
      if k >= args.eval_batches:
        break
      num = num.to(device).float()
      lab = lab.reshape(-1)
      if lab.numel() > num.shape[0]:  # global labels: this rank's slice
        lab = lab[rank * num.shape[0]:(rank + 1) * num.shape[0]]
      ids = [c.to(device).to(torch.int32) for c in cat]
      trainer.evaluate(num, ids if args.interaction == "dcnv2" else
                       torch.stack([c.reshape(-1) for c in ids]), lab.to(device).float())
    m = trainer.eval_metrics()  # collective
    if rank == 0:
      binned = f" binned_AUC: {m['binned_auc']:.6f}" if "binned_auc" in m else ""
      print(f"eval step: {i} AUC: {m['auc']:.6f}{binned} tie_bound: {m['tie_bound']:.2e} "
            f"log_loss: {m['log_loss']:.6f}", flush=True)

  for i, (num, cat, lab) in enumerate(batches()):
    num, lab = num.to(device).float(), lab.to(device)
    cat = [c.to(device) for c in cat]
    if args.test_combiner:
      cat = [c.reshape(-1, 1) for c in cat]
    loss = step(num, cat, lab)
    if i % 1000 == 0:
      loss = loss.detach().clone().reshape(())
      if world > 1:
        dist.all_reduce(loss)
        loss /= world
      if rank == 0:
        print("step: ", i, " loss: ", float(loss))
    if args.eval_interval > 0 and (i + 1) % args.eval_interval == 0:
      periodic_eval(i + 1)

  # evaluation: predictions of the local batch gathered on every rank, AUC on rank 0
  preds, labels = [], []
  model.eval()
  with torch.no_grad():
    for num, cat, lab in evald:
      cat = [c.to(device) for c in cat]
      if args.test_combiner:
        cat = [c.reshape(-1, 1) for c in cat]
      p = torch.sigmoid(model(num.to(device).float(), cat).float())
      if world > 1:
        out = [torch.empty_like(p) for _ in range(world)]
        dist.all_gather(out, p)
        p = torch.cat(out)
      preds.append(p.cpu())
      labels.append(lab.reshape(-1, 1).float().cpu())
  if rank == 0 and preds:
    p, y = torch.cat(preds).reshape(-1), torch.cat(labels).reshape(-1)
    n = min(p.numel(), y.numel())
    auc = binary_auc(y[:n], p[:n])
    bce = torch.nn.functional.binary_cross_entropy(p[:n].clamp(1e-7, 1 - 1e-7), y[:n])
    print(f"Evaluation completed, AUC: {auc}, test_loss: {float(bce)}")

  if args.save_dir:
    paths = model.embedding.save_weights(args.save_dir)
    if rank == 0:
      print(f"saved {len(paths)} tables to {args.save_dir}/")
  else:
    weights = model.embedding.get_weights()
    if rank == 0:
      np.savez(args.save_path, *weights)
      print(f"saved {len(weights)} tables to {args.save_path}.npz")
  if world > 1:
    dist.destroy_process_group()


if __name__ == "__main__":
  main()
