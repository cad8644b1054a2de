"""Hybrid-parallel training glue: data-parallel dense parameters are all-reduced (averaged),
model-parallel embedding parameters (tagged ``de_local``) are updated locally.

PyTorch equivalents of the reference's Horovod patches (dist_model_parallel.py:1217-1329):
``DistributedGradientTape`` -> :class:`DistributedGradientTape` / :func:`allreduce_gradients`,
``DistributedOptimizer`` -> :class:`DistributedOptimizer`,
``BroadcastGlobalVariablesCallback`` -> :class:`BroadcastGlobalVariablesCallback`.

On CUDA the dense gradients live in one *symmetric* flat bucket and are reduced by a single
NVLink kernel (reduce-scatter + all-gather over peer memory fused with the 1/world scale, see
``ops/csrc/comm_kernels.cu``); ``torch.distributed.all_reduce`` is the CPU / fallback path.
"""
from __future__ import annotations

from typing import Iterable, List, Optional, Sequence

import numpy as np
import torch
import torch.distributed as dist
from torch import nn

from ..ops.stochastic_rounding import (HALF_DTYPES, STREAM_STATE0, STREAM_STATE1, STREAM_WEIGHT,
                                       stochastic_round)
from .comm import CommContext, dist_ready
from .dist_model_parallel import _is_mp, broadcast_variables
from .embedding_optimizers import (OPTIMIZERS, check_state_dtype, check_weight_decay_mode,
                                   decay_keep, state_slots)


def _world(group=None) -> int:
  return dist.get_world_size(group) if dist_ready() else 1


class GradBucket:
  """Flat gradient bucket for the data-parallel parameters.

  ``param.grad`` of every DP parameter becomes a view into one contiguous buffer (symmetric
  memory on CUDA), so the all-reduce needs no pack / unpack copies.
  """

  def __init__(self, params: Sequence[nn.Parameter], ctx: Optional[CommContext] = None,
               dtype: torch.dtype = torch.float32, group=None):
    self.params = [p for p in params if p.requires_grad]
    self.group = group
    self.dtype = dtype
    self.numel = sum(p.numel() for p in self.params)
    # pad every parameter to 16 bytes so views stay vector aligned
    elem = torch.empty((), dtype=dtype).element_size()
    align = 16 // elem
    self.offsets = []
    pos = 0
    for p in self.params:
      self.offsets.append(pos)
      pos += (p.numel() + align - 1) // align * align
    self.padded = max(pos, align)
    self.ctx = ctx
    self.symm = None
    dev = self.params[0].device if self.params else torch.device("cpu")
    if ctx is not None and ctx.p2p and dev.type == "cuda" and ctx.world_size > 1:
      self.symm = ctx.alloc(self.padded * elem, "dense_grad_bucket")
      self.flat = self.symm.view(dtype, (self.padded,))
    else:
      self.flat = torch.zeros(self.padded, dtype=dtype, device=dev)
    self.views = [self.flat[o:o + p.numel()].view_as(p) for o, p in zip(self.offsets, self.params)]

  def attach(self):
    """Point ``param.grad`` at the bucket views (autograd then accumulates in place)."""
    for p, v in zip(self.params, self.views):
      p.grad = v

  def zero_(self):
    self.flat.zero_()

  def gather_grads_(self):
    """Copy stray ``param.grad`` tensors (not views of the bucket) into the bucket."""
    src, dst = [], []
    for p, v in zip(self.params, self.views):
      g = p.grad
      if g is None:
        v.zero_()
        continue
      if g.data_ptr() == v.data_ptr():
        continue
      if g.is_sparse:
        v.zero_()
        v.add_(g.to_dense().to(v.dtype))
      else:
        src.append(g)
        dst.append(v)
    if src:
      torch._foreach_copy_(dst, src)

  def allreduce_(self, average: bool = True):
    world = _world(self.group)
    if world == 1:
      return
    scale = 1.0 / world if average else 1.0
    if self.symm is not None:
      self.ctx.allreduce_(self.symm, self.padded, self.dtype, scale=scale)
    else:
      dist.all_reduce(self.flat, op=dist.ReduceOp.SUM, group=self.group)
      if average:
        self.flat.mul_(scale)

  def scatter_grads_(self):
    for p, v in zip(self.params, self.views):
      if p.grad is None or p.grad.data_ptr() != v.data_ptr():
        p.grad = v


def allreduce_gradients(params: Iterable[nn.Parameter], group=None, average: bool = True,
                        bucket: Optional[GradBucket] = None):
  """Average the gradients of data-parallel parameters over all ranks (sparse gradients are
  densified, like the reference's ``sparse_as_dense=True``); ``de_local`` parameters are skipped."""
  params = [p for p in params if not _is_mp(p) and p.requires_grad]
  if _world(group) == 1 or not params:
    return
  if bucket is None:
    dense = []
    for p in params:
      if p.grad is None:
        p.grad = torch.zeros_like(p)
      elif p.grad.is_sparse:
        p.grad = p.grad.to_dense()
      dense.append(p.grad)
    flat = torch.cat([g.reshape(-1).float() for g in dense])
    dist.all_reduce(flat, group=group)
    if average:
      flat /= _world(group)
    pos = 0
    for g in dense:
      g.copy_(flat[pos:pos + g.numel()].view_as(g))
      pos += g.numel()
    return
  bucket.gather_grads_()
  bucket.allreduce_(average)
  bucket.scatter_grads_()


class DistributedGradientTape:
  """Functional gradient helper mirroring the reference's tape API.

  >>> tape = DistributedGradientTape()
  >>> grads = tape.gradient(loss, params)   # DP grads averaged over ranks, MP grads local
  """

  def __init__(self, group=None, average: bool = True):
    self.group = group
    self.average = average

  def gradient(self, target: torch.Tensor, sources: Sequence[nn.Parameter]):
    sources = list(sources)
    if target.dim() > 0:
      target = target.sum()
    grads = torch.autograd.grad(target, sources, allow_unused=True)
    out = []
    world = _world(self.group)
    for p, g in zip(sources, grads):
      if g is None:
        out.append(None)
        continue
      if not _is_mp(p) and world > 1:
        if g.is_sparse:
          g = g.to_dense()
        g = g.contiguous()
        dist.all_reduce(g, group=self.group)
        if self.average:
          g = g / world
      out.append(g)
    return out


class DistributedOptimizer:
  """Wrap a ``torch.optim`` optimizer for hybrid parallel training: ``step()`` first averages the
  gradients of data-parallel parameters across ranks, then applies the wrapped optimizer
  (which also owns any model-parallel parameters that are not updated by a fused optimizer)."""

  def __init__(self, optimizer: torch.optim.Optimizer, group=None, average: bool = True,
               use_bucket: bool = True, ctx: Optional[CommContext] = None,
               bucket_dtype: torch.dtype = torch.float32):
    self.optimizer = optimizer
    self.group = group
    self.average = average
    params = [p for g in optimizer.param_groups for p in g["params"]]
    self.dp_params = [p for p in params if not _is_mp(p)]
    self.bucket = None
    if use_bucket and self.dp_params and _world(group) > 1:
      if ctx is None and self.dp_params[0].is_cuda:
        ctx = CommContext.default(self.dp_params[0].device)
      self.bucket = GradBucket(self.dp_params, ctx, bucket_dtype, group)
      self.bucket.attach()

  @property
  def param_groups(self):
    return self.optimizer.param_groups

  def zero_grad(self, set_to_none: bool = False):
    if self.bucket is not None:
      self.bucket.zero_()
      self.bucket.attach()
      for g in self.optimizer.param_groups:
        for p in g["params"]:
          if _is_mp(p):
            p.grad = None
    else:
      self.optimizer.zero_grad(set_to_none=set_to_none)

  def synchronize(self):
    allreduce_gradients(self.dp_params, self.group, self.average, self.bucket)

  def step(self, closure=None):
    self.synchronize()
    return self.optimizer.step(closure)

  def state_dict(self):
    return self.optimizer.state_dict()

  def load_state_dict(self, state):
    self.optimizer.load_state_dict(state)


class BroadcastGlobalVariablesCallback:
  """Broadcast the data-parallel variables of a model from ``root_rank`` (call once after the
  first step / at train begin, reference dist_model_parallel.py:1303-1326)."""

  def __init__(self, root_rank: int = 0, group=None):
    self.root_rank = root_rank
    self.group = group
    self.done = False

  def __call__(self, model: nn.Module):
    if not self.done:
      broadcast_variables(model, self.root_rank, self.group)
      self.done = True

  on_train_begin = __call__
  on_batch_end = __call__


def exclude_model_parallel_from_ddp(module: nn.Module) -> List[str]:
  """Let ``torch.nn.parallel.DistributedDataParallel`` wrap a model that contains a
  :class:`DistributedEmbedding`: the model-parallel tables (``de_local`` parameters, different on
  every rank, updated in place or through row-sparse gradients) are put on DDP's ignore list, so
  DDP neither broadcasts them at construction nor all-reduces their gradients; everything else
  (replicated tables, MLPs) is handled by DDP as usual.  Call it *before* constructing DDP:

      names = exclude_model_parallel_from_ddp(model)
      ddp = torch.nn.parallel.DistributedDataParallel(model)

  The PyTorch counterpart of combining the reference layer with Horovod's
  ``DistributedGradientTape`` (reference dist_model_parallel.py:1241-1290).  Returns the ignored
  parameter names."""
  names = [n for n, p in module.named_parameters() if getattr(p, "de_local", False)]
  from torch.nn.parallel import DistributedDataParallel as DDP  # pylint: disable=import-outside-toplevel
  DDP._set_params_and_buffers_to_ignore_for_model(module, names)  # pylint: disable=protected-access
  return names


class SparseRowOptimizer:
  """Row-sparse optimizer for model-parallel tables whose gradients arrive as (coalesced) sparse
  tensors - the ``torch`` back end of :class:`DistributedEmbedding`, i.e. the NCCL-collectives
  baseline, which has no fused update.  Same math as the fused kernels
  (``ops/csrc/sparse_update_kernels.cu``): ``sgd`` | ``adagrad`` | ``rowwise_adagrad`` | ``adam``
  | ``rowwise_adam`` | ``ftrl`` | ``momentum`` (lazy: only the touched rows advance).  ``ftrl``
  and ``momentum`` take the keyword arguments of their kind in
  ``DistributedEmbedding.set_optimizer`` (``lr_power``, ``l1``, ``l2``, ``l2_shrinkage``,
  ``beta``; ``momentum``, ``nesterov``); the other kinds reject them.  Counterpart of the Keras
  sparse-apply kernels the reference relies on (examples/benchmarks/synthetic_models/main.py:96-101).

  bf16 / fp16 parameters keep fp32 state; their touched rows are updated in fp32 and written
  back with stochastic rounding keyed by (step, row, column), the rule of the fused kernels
  (``ops/stochastic_rounding.py``).

  ``state_dtype=torch.bfloat16`` stores the Adagrad accumulator / Adam moments / row-wise Adam's
  m / FTRL's n and z / the momentum buffer in bf16 like the fused back end: the touched rows'
  state is widened to fp32, the update runs in fp32 with the unrounded new state, and the state
  is stored with stochastic rounding (streams 1 and 2).  Row-wise state (one word per row) stays fp32.

  ``weight_decay_mode``: ``"l2"`` (default) adds ``weight_decay * w`` to the gradient;
  ``"decoupled"`` scales each touched row by the fp32 ``1 - lr * weight_decay`` first and applies
  the step of the undecayed gradient, as :meth:`DistributedEmbedding.set_optimizer` describes."""

  def __init__(self, params: Sequence[nn.Parameter], kind: str = "sgd", lr: float = 0.01,
               eps: Optional[float] = None, beta1: float = 0.9, beta2: float = 0.999,
               initial_accumulator_value: float = 0.1, weight_decay: float = 0.0,
               state_dtype: torch.dtype = torch.float32, weight_decay_mode: str = "l2",
               **hyper):
    kind = kind.lower()
    if kind not in OPTIMIZERS:
      raise ValueError(f"Unsupported optimizer {kind}")
    self.weight_decay_mode = check_weight_decay_mode(kind, weight_decay_mode)
    entry = OPTIMIZERS[kind]
    unknown = sorted(set(hyper) - set(entry.hyper))
    if unknown:
      raise ValueError(f"unknown fused optimizer argument(s) {unknown} for {kind}")
    # the kind's own hyperparameters (FTRL's, momentum's), defaults filled in
    self.hyper = dict(entry.hyper, initial_accumulator_value=initial_accumulator_value, **hyper)
    if entry.check is not None:
      entry.check(self.hyper)
    self.state_dtype = check_state_dtype(kind, state_dtype)
    self.params = [p for p in params if p.requires_grad]
    self.kind, self.lr = kind, float(lr)
    self.eps = entry.eps if eps is None else eps
    self.beta1, self.beta2, self.weight_decay = beta1, beta2, weight_decay
    self.step_count = 0
    self.state = []
    for p in self.params:
      sdt = torch.promote_types(p.dtype, torch.float32)  # half tables: fp32 state
      esdt = torch.bfloat16 if self.state_dtype == torch.bfloat16 else sdt  # element-wise state
      self.state.append(state_slots(kind, p, esdt, sdt, initial_accumulator_value))

  def set_lr(self, lr: float):
    self.lr = float(lr)

  @torch.no_grad()
  def step(self):
    """Update the touched rows of every table in ``promote_types(dtype, float32)``, in the
    kernels' order of operations; store 16-bit weights and bf16 state with stochastic
    rounding."""
    self.step_count += 1
    for p, st in zip(self.params, self.state):
      g = p.grad
      if g is None:
        continue
      p.grad = None
      if g.is_sparse:
        g = g.coalesce()
        idx, val = g.indices()[0], g.values().to(p.dtype)
      else:
        idx = torch.arange(p.shape[0], device=p.device)
        val = g.to(p.dtype)
      if self.kind == "ftrl" and self.lr == 0.0:
        continue  # rows and state keep their bits
      cdt = torch.promote_types(p.dtype, torch.float32)
      w, val = p[idx].to(cdt), val.to(cdt)
      if self.weight_decay and self.weight_decay_mode == "decoupled" and self.kind != "sgd":
        # (1 - lr wd) w in one rounding of the compute dtype, then the undecayed step
        w = w * torch.tensor(decay_keep(self.lr, self.weight_decay), dtype=cdt)
      elif self.weight_decay:
        val = val + self.weight_decay * w
      w, new_state = self._update(w, val, [s[idx].to(cdt) for s in st])
      self._store(p, idx, w, STREAM_WEIGHT)
      for s, x, stream in zip(st, new_state, (STREAM_STATE0, STREAM_STATE1)):
        self._store(s, idx, x, stream)

  def _update(self, w, g, state):
    """One step of the optimizer on rows ``w`` with decayed gradient ``g`` and the rows' state
    slots; returns the new weights and state."""
    b1 = 1 - self.beta1**self.step_count
    b2 = 1 - self.beta2**self.step_count
    if self.kind == "sgd":
      return w - self.lr * g, []
    if self.kind == "adagrad":
      acc = state[0] + g * g
      return w - self.lr * g / (acc.sqrt() + self.eps), [acc]
    if self.kind == "rowwise_adagrad":
      acc = state[0] + (g * g).mean(dim=1)
      return w - self.lr * g / (acc.sqrt().unsqueeze(1) + self.eps), [acc]
    if self.kind == "adam":
      m = self.beta1 * state[0] + (1 - self.beta1) * g
      v = self.beta2 * state[1] + (1 - self.beta2) * g * g
      return w - self.lr * (m / b1) / ((v / b2).sqrt() + self.eps), [m, v]
    if self.kind == "rowwise_adam":
      m = self.beta1 * state[0] + (1 - self.beta1) * g
      v = self.beta2 * state[1] + (1 - self.beta2) * (g * g).mean(dim=1)
      return w - self.lr * (m / b1) / ((v / b2).sqrt().unsqueeze(1) + self.eps), [m, v]
    if self.kind == "momentum":
      return self._momentum(w, g, state[0])
    w, n, z = self._ftrl(w, g, state[0], state[1])
    return w, [n, z]

  def _ftrl(self, w, g, n, z):
    """FTRL-Proximal on rows ``w`` with decayed gradient ``g``, accumulator ``n`` and linear term
    ``z`` (lr != 0); returns the new (w, n, z)."""
    c = self.hyper
    pw = (lambda x: x.sqrt()) if c["lr_power"] == -0.5 else (lambda x: x.pow(-c["lr_power"]))
    n_new = n + g * g
    p_new = pw(n_new)
    z = z + g + 2 * c["l2_shrinkage"] * w - (p_new - pw(n)) / self.lr * w
    q = (c["beta"] + p_new) / self.lr + 2 * c["l2"]
    w = torch.where(z.abs() > c["l1"], (torch.sign(z) * c["l1"] - z) / q, torch.zeros_like(z))
    return w, n_new, z

  def _momentum(self, w, g, b):
    """Momentum SGD on rows ``w`` with decayed gradient ``g`` and buffer ``b``, in the kernels'
    fmaf order (each fma one rounding of its float64 value); returns (w, [b])."""
    cdt = w.dtype
    mu = float(np.float32(self.hyper["momentum"]))
    neg_lr = -float(np.float32(self.lr))
    fma = lambda a, x, y: (a * x.double() + y.double()).to(cdt)
    b = fma(mu, b, g)
    u = fma(mu, b, g) if self.hyper["nesterov"] else b
    return fma(neg_lr, u, w), [b]

  def _store(self, dst, idx, x, stream):
    """Store rows ``x`` at ``idx`` of a table or state slot: as is, or stochastically rounded
    into a 16-bit ``dst``."""
    if dst.dtype in HALF_DTYPES:
      dst[idx] = stochastic_round(x, dst.dtype, self.step_count, idx, stream=stream).to(dst.device)
    else:
      dst[idx] = x
