"""Hybrid-parallel training step: fused model-parallel embedding update + data-parallel dense
update, with an optional whole-step CUDA graph.

One call of :meth:`HybridTrainer.step` does what the reference's ``train_step`` does
(examples/dlrm/main.py:200-209): forward, loss, backward through the embedding exchange, dense
gradient all-reduce, optimizer apply.
"""
from __future__ import annotations

from typing import Callable, List, Optional

import torch
from torch import nn

from ..parallel.comm import CommContext
from ..parallel.hybrid import GradBucket, SparseRowOptimizer
from ..utils.lr_schedule import LearningRateScheduler
from .dense_optimizer import check_state, dense_optimizer_config, slot_init


class HybridTrainer:
  """Owns the dense optimizer state and the gradient bucket of a model whose embeddings are a
  :class:`DistributedEmbedding` with a fused optimizer.

  Args:
    model: module taking ``(numerical, categorical)``; must expose ``embedding``
      (DistributedEmbedding) and ``dense_parameters()``.
    lr: learning rate (dense SGD and fused embedding optimizer share it like the reference).
    embedding_optimizer: ``sgd`` | ``adagrad`` | ``rowwise_adagrad`` | ``adam`` | ``rowwise_adam``
      | ``ftrl`` | ``momentum``; its hyperparameters in ``embedding_optimizer_kwargs`` go to both
      the fused optimizer and the torch back end's :class:`SparseRowOptimizer`.
    scheduler: optional :class:`LearningRateScheduler`.
    dense_optimizer: ``sgd`` | ``adagrad`` | ``adam`` | ``momentum`` for the dense parameters
      (MLPs and replicated tables), hyperparameters in ``dense_optimizer_kwargs`` (see
      ``models/dense_optimizer.py``), ``weight_decay`` / ``weight_decay_mode`` included.
      ``dense_optimizer="momentum"`` (``momentum`` / ``nesterov`` in ``dense_optimizer_kwargs``)
      is the embedding kind's update on device words, so it follows a scheduler inside a
      captured CUDA graph, and takes both decay modes.
    momentum: applies to ``dense_optimizer="sgd"`` only, through ``torch.optim.SGD`` (learning
      rate on the host: no scheduler inside a captured graph).  It takes L2 decay as
      ``torch.optim.SGD(weight_decay=...)`` does (into the gradient, before the momentum
      buffer); ``weight_decay_mode="decoupled"`` with it raises ``ValueError``.
  """

  def __init__(self, model: nn.Module, lr: float = 24.0, embedding_optimizer: str = "sgd",
               scheduler: Optional[LearningRateScheduler] = None, momentum: float = 0.0,
               embedding_optimizer_kwargs: Optional[dict] = None,
               loss_fn: Optional[Callable] = None, use_cuda_graph: bool = False,
               graph_warmup_steps: int = 3, dense_optimizer: str = "sgd",
               dense_optimizer_kwargs: Optional[dict] = None):
    self.dense_cfg = dense_optimizer_config(dense_optimizer, dense_optimizer_kwargs)
    if momentum != 0.0 and self.dense_cfg["kind"] != "sgd":
      raise ValueError("momentum applies to dense_optimizer='sgd' only")
    if momentum != 0.0 and self.dense_cfg["weight_decay"] and \
        self.dense_cfg["weight_decay_mode"] == "decoupled":
      raise ValueError("momentum SGD takes weight_decay_mode='l2' only (torch.optim.SGD's "
                       "weight decay); decoupled decay is for momentum=0")
    self.model = model
    self.emb = model.embedding
    self.emb.set_optimizer(embedding_optimizer, lr=lr, **(embedding_optimizer_kwargs or {}))
    self.dense_params: List[nn.Parameter] = list(model.dense_parameters())
    # Lookups that do not run on the fused engine (torch / NCCL back end, or inputs the engine
    # does not support) hand the model-parallel tables ordinary sparse autograd gradients:
    # a row-sparse optimizer with the same math as the fused kernels applies them.
    self.mp_opt = SparseRowOptimizer(self.emb.mp_parameters(), embedding_optimizer, lr=lr,
                                     **(embedding_optimizer_kwargs or {}))
    self.scheduler = scheduler
    self.lr = lr
    dev = self.dense_params[0].device
    self.ctx = CommContext.default(dev) if dev.type == "cuda" else None
    self.world = self.emb.world_size
    self.bucket = GradBucket(self.dense_params, self.ctx if self.world > 1 else None)
    self.bucket.attach()
    self.opt = torch.optim.SGD(self.dense_params, lr=lr, momentum=momentum,
                               weight_decay=self.dense_cfg["weight_decay"],
                               foreach=dev.type == "cuda")
    # plain SGD keeps its learning rate in device memory: a captured CUDA graph bakes host
    # scalars in, so a scheduler would otherwise leave the dense lr frozen at its capture-time
    # value while the embedding lr (device resident as well) keeps changing
    self.momentum = momentum
    self.lr_t = torch.full((), float(lr), dtype=torch.float32, device=dev)
    # dense Adagrad / Adam: state per bucket parameter, Adam's step count as a device word (both
    # follow a scheduler under graph replay); the gradients are the all-reduced bucket views
    names = {id(p): n for n, p in model.named_parameters()}
    self._dense_names = [names[id(p)] for p in self.bucket.params]
    self.dense_state = [[torch.full_like(p, v, memory_format=torch.contiguous_format)
                         for p in self.bucket.params] for v in slot_init(self.dense_cfg)]
    self.dense_step_t = torch.zeros((), dtype=torch.float32, device=dev)
    self.loss_fn = loss_fn or nn.BCEWithLogitsLoss()
    # whole-step CUDA graph: the first `graph_warmup_steps` calls run eagerly (real steps), the
    # next call captures forward + backward + all-reduce + optimizer and every call replays it
    self.use_cuda_graph = use_cuda_graph and dev.type == "cuda"
    self.graph_warmup_steps = graph_warmup_steps
    self._calls = 0
    self._graph = None
    self._static = None
    # autograd caches each leaf's AccumulateGrad node together with the stream it was first used
    # on; warm-up and capture therefore have to run on the same (non-default) stream
    self._gstream = torch.cuda.Stream(device=dev) if self.use_cuda_graph else None

  def set_lr(self, lr: float):
    self.lr = lr
    for g in self.opt.param_groups:
      g["lr"] = lr
    self.lr_t.fill_(float(lr))
    self.mp_opt.set_lr(lr)
    self.emb.set_learning_rate(lr)

  def _dense_step(self):
    if self.dense_cfg["kind"] != "sgd":
      self._adaptive_dense_step()
      return
    if self.momentum != 0.0:
      if self._graph is not None or (self.use_cuda_graph and self.scheduler is not None):
        raise RuntimeError("momentum SGD keeps its learning rate on the host: it cannot follow a "
                           "scheduler inside a captured CUDA graph (use momentum=0 or "
                           "use_cuda_graph=False)")
      self.opt.step()
      return
    params = [p for p in self.dense_params if p.grad is not None]
    if not params:
      return
    with torch.no_grad():
      grads = [p.grad for p in params]
      wd = self.dense_cfg["weight_decay"]
      if wd:  # p -= lr * (g + wd * p): SGD's update in both decay modes
        grads = torch._foreach_add(grads, params, alpha=wd)
      if params[0].is_cuda:
        upd = torch._foreach_mul(grads, self.lr_t)  # device-resident lr (graph replay safe)
        torch._foreach_sub_(params, upd)
      else:
        for p, g in zip(params, grads):
          p.sub_(g * self.lr_t)

  def _adaptive_dense_step(self):
    """Dense Adagrad / Adam / momentum with the expressions of the fused kernels, on device
    words."""
    c, params, grads = self.dense_cfg, self.bucket.params, self.bucket.views
    if not params:
      return
    with torch.no_grad():
      if c["weight_decay"] and c["weight_decay_mode"] == "decoupled":
        # p = (1 - lr wd) p before the step of the undecayed gradient (device lr: graph safe)
        torch._foreach_mul_(params, 1.0 - self.lr_t * c["weight_decay"])
      elif c["weight_decay"]:
        grads = torch._foreach_add(grads, params, alpha=c["weight_decay"])
      if c["kind"] == "momentum":
        buf = self.dense_state[0]
        torch._foreach_mul_(buf, c["momentum"])
        torch._foreach_add_(buf, grads)
        step = torch._foreach_add(torch._foreach_mul(buf, c["momentum"]), grads) \
            if c["nesterov"] else buf
        torch._foreach_sub_(params, torch._foreach_mul(step, self.lr_t))
        return
      if c["kind"] == "adagrad":
        acc = self.dense_state[0]
        torch._foreach_addcmul_(acc, grads, grads)
        num = grads
        den = torch._foreach_sqrt(acc)
      else:
        m, v = self.dense_state
        self.dense_step_t.add_(1.0)
        torch._foreach_mul_(m, c["beta1"])
        torch._foreach_add_(m, grads, alpha=1.0 - c["beta1"])
        torch._foreach_mul_(v, c["beta2"])
        torch._foreach_addcmul_(v, grads, grads, value=1.0 - c["beta2"])
        bias1 = 1.0 - torch.pow(c["beta1"], self.dense_step_t)
        bias2 = 1.0 - torch.pow(c["beta2"], self.dense_step_t)
        num = torch._foreach_div(m, bias1)
        den = torch._foreach_div(v, bias2)
        torch._foreach_sqrt_(den)
      torch._foreach_add_(den, c["eps"])
      upd = torch._foreach_mul(num, self.lr_t)
      torch._foreach_div_(upd, den)
      torch._foreach_sub_(params, upd)

  def dense_optimizer_state(self) -> dict:
    """``{"kind", "step", "slots": {param_name: [tensor, ...]}}``: the dense optimizer state,
    each slot shaped like its parameter; the format of every trainer."""
    slots = {n: [s[i].detach().clone() for s in self.dense_state]
             for i, n in enumerate(self._dense_names)} if self.dense_state else {}
    step = int(round(float(self.dense_step_t))) if self.dense_cfg["kind"] == "adam" else 0
    return {"kind": self.dense_cfg["kind"], "step": step, "slots": slots}

  def load_dense_optimizer_state(self, state: dict):
    """Restore :meth:`dense_optimizer_state` output (of any trainer); another kind raises."""
    check_state(self.dense_cfg, state, self._dense_names)
    if self.dense_state:
      for i, n in enumerate(self._dense_names):
        for s, src in zip(self.dense_state, state["slots"][n]):
          s[i].copy_(src)
    self.dense_step_t.fill_(float(state.get("step", 0)))

  def step(self, numerical, categorical, labels, staged: bool = False) -> torch.Tensor:
    if self.scheduler is not None:
      self.set_lr(self.scheduler.step())
    self._calls += 1
    if not self.use_cuda_graph or staged:
      return self._step_eager(numerical, categorical, labels, staged)
    if self._calls <= self.graph_warmup_steps:
      self._gstream.wait_stream(torch.cuda.current_stream())
      with torch.cuda.stream(self._gstream):
        loss = self._step_eager(numerical, categorical, labels, staged)
      torch.cuda.current_stream().wait_stream(self._gstream)
      return loss
    if self._static is None:
      self._static = (numerical.clone(), [c.clone() for c in categorical], labels.clone())
    sn, sc, sl = self._static
    sn.copy_(numerical, non_blocking=True)
    sl.copy_(labels, non_blocking=True)
    for d, c in zip(sc, categorical):
      d.copy_(c, non_blocking=True)
    if self._graph is None:
      torch.cuda.synchronize()
      g = torch.cuda.CUDAGraph()
      with torch.cuda.graph(g, stream=self._gstream):
        self._static_loss = self._step_eager(sn, sc, sl, False)
      self._graph = g
    self._graph.replay()
    return self._static_loss

  def _step_eager(self, numerical, categorical, labels, staged: bool = False) -> torch.Tensor:
    self.bucket.zero_()
    logits = self.model(numerical, categorical, staged=staged) if staged else \
        self.model(numerical, categorical)
    loss = self.loss_fn(logits.float(), labels)
    loss.backward()  # embedding tables are updated inside the backward kernels
    self.bucket.gather_grads_()
    self.bucket.allreduce_(average=True)
    self._dense_step()
    self.mp_opt.step()  # no-op when the fused engine already updated the tables in backward
    return loss.detach()
