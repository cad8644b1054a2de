"""Hand-scheduled training step for the synthetic model zoo (no autograd on the hot path) +
whole-step CUDA graph - the counterpart of the reference's single ``tf.function`` + XLA step
(examples/benchmarks/synthetic_models/main.py:122-130).

``SyntheticTrainStep`` runs :class:`SyntheticModel` as one static schedule over preallocated
buffers:

* the embedding lookups write straight into the first-layer input matrix of the MLP
  (``FusedEngine.set_out_row_stride``): the concatenation ``[embeddings | numerical | pad]`` of
  the module costs no kernel, the numerical features are cast into their columns;
* dense parameters live in one flat fp32 master buffer with a bf16 shadow, gradients in one flat
  (symmetric) buffer reduced by the one-kernel NVLink all-reduce, one fused kernel does
  SGD (or Adagrad / Adam, ``dense_optimizer``) + re-cast + gradient zeroing;
* forward layers: bf16 GEMMs with fused bias + ReLU epilogues; backward: weight-gradient and
  data-gradient GEMMs + the fused ReLU-backward / bias-gradient kernel; final layer + BCE loss
  + their backward in one kernel;
* the first layer's data gradient *is* the embedding gradient: ``push_grad`` routes its pieces
  to the table owners over NVLink (gradient all-to-all) and signals them, the fused update
  kernels (atomic SGD or sort / dedup + Adagrad / row-wise Adagrad / Adam) consume it;
* everything is captured in a CUDA graph and replayed.

The pooling interaction of the larger models (``interact_stride``) is a memory-bound kernel pair
between the lookups and the MLP.  Models with replicated tables keep using :class:`HybridTrainer`
(autograd + whole-step graph).
"""
from __future__ import annotations

from typing import List, Optional

import torch
from torch import nn

from ..ops import _native
from ..parallel.comm import CommContext
from ..parallel.fused import FusedEngine
from ..ops.ragged import RaggedIds
from ..utils import nvtx
from .dense_optimizer import FlatDenseOptimizer, dense_optimizer_config
from .dlrm_fast import _Layer, _pad8
from .synthetic import SyntheticModel


class SyntheticTrainStep:
  """Static-schedule training step for :class:`SyntheticModel` on the fused embedding back end.

  ``dense_optimizer`` (``sgd`` | ``adagrad`` | ``adam`` | ``momentum``, hyperparameters in
  ``dense_optimizer_kwargs``) updates the MLP with the shared learning rate; the reference's
  configuration is ``embedding_optimizer="adagrad", dense_optimizer="adagrad"``.
  ``embedding_optimizer`` is any kind of ``DistributedEmbedding.set_optimizer`` (``ftrl`` and
  ``momentum`` included), with its hyperparameters in ``embedding_optimizer_kwargs``."""

  def __init__(self, model: SyntheticModel, lr: float = 0.001, embedding_optimizer: str = "adagrad",
               use_cuda_graph: bool = True, embedding_optimizer_kwargs: Optional[dict] = None,
               dense_optimizer: str = "sgd", dense_optimizer_kwargs: Optional[dict] = None):
    self.dense_cfg = dense_optimizer_config(dense_optimizer, dense_optimizer_kwargs)
    self.model = model
    self.emb = model.embedding
    why = self.unsupported_reason(model)
    if why:
      raise ValueError(f"SyntheticTrainStep: {why}")
    self.dev = self.emb.device
    self.ops = _native.require()
    self.world = self.emb.world_size
    self.ctx = CommContext.for_group(self.emb.group, self.dev)
    self.use_cuda_graph = use_cuda_graph
    self.emb.set_optimizer(embedding_optimizer, lr=lr, **(embedding_optimizer_kwargs or {}))
    if self.emb._engine is None:
      self.emb._engine = FusedEngine(self.emb)
    self.engine: FusedEngine = self.emb._engine
    self.in_pad = model._in_dim + model._in_pad             # first-layer fan-in (multiple of 8)
    tw = self.engine.total_width
    self.pool = model.interact_stride
    if self.pool is None:
      # the lookups write straight into the MLP input matrix
      self.emb_cols = tw
      self.engine.set_out_row_stride(self.in_pad)
    else:
      # pooled interaction: a memory-bound kernel pair sits between the lookups and the MLP
      self.emb_cols = -(-tw // self.pool)
    self.n_num = model._in_dim - self.emb_cols  # numerical features

    lins = [m for m in model.mlp if isinstance(m, nn.Linear)]
    self.hidden = [_Layer(l, True) for l in lins[:-1]]
    self.head = _Layer(lins[-1], False)
    layers = self.hidden + [self.head]
    pos = 0
    for L in layers:
      L.w_off = pos
      pos += L.w_numel
      L.b_off = pos
      pos += L.b_numel
    self.n_flat = pos
    dev = self.dev
    self.p32 = torch.zeros(pos, dtype=torch.float32, device=dev)
    self.p16 = torch.zeros(pos, dtype=torch.bfloat16, device=dev)
    if self.world > 1:
      self.gsym = self.ctx.alloc(pos * 4, "dense_grads")
      self.g32 = self.gsym.view(torch.float32, (pos,))
    else:
      self.gsym = None
      self.g32 = torch.zeros(pos, dtype=torch.float32, device=dev)
    with torch.no_grad():
      for L in layers:
        wv = self.p32[L.w_off:L.w_off + L.w_numel].view(L.out_f, L.in_pad)
        wv[:, :L.in_f].copy_(L.lin.weight)
        L.lin.weight.data = wv[:, :L.in_f]
        bv = self.p32[L.b_off:L.b_off + L.out_f]
        bv.copy_(L.lin.bias)
        L.lin.bias.data = bv
        L.w16 = self.p16[L.w_off:L.w_off + L.w_numel].view(L.out_f, L.in_pad)
        L.b16 = self.p16[L.b_off:L.b_off + L.out_f]
        L.gw = self.g32[L.w_off:L.w_off + L.w_numel].view(L.out_f, L.in_pad)
        L.gb = self.g32[L.b_off:L.b_off + L.b_numel]
      self.p16.copy_(self.p32)
    self.dense_opt = FlatDenseOptimizer(self.dense_cfg, self.p32)
    self.lr = float(lr)
    self.lr_t = torch.full((1,), float(lr), dtype=torch.float32, device=dev)
    self.loss = torch.zeros(1, dtype=torch.float32, device=dev)
    self._batch = None
    self._graph = None
    self._side = torch.cuda.Stream(device=dev)

  @staticmethod
  def unsupported_reason(model) -> Optional[str]:
    """None when the hand-scheduled step can run this model, else why not."""
    if not isinstance(model, SyntheticModel):
      return "needs a SyntheticModel"
    emb = model.embedding
    if emb.backend != "fused":
      return "needs the fused embedding back end"
    if model.compute_dtype != torch.bfloat16:
      return "runs the dense side in bf16 (use --amp / compute_dtype=torch.bfloat16)"
    if len(emb.dp_layers):
      return "replicated tables (data_parallel_threshold) are not part of the static schedule"
    lins = [m for m in model.mlp if isinstance(m, nn.Linear)]
    if len(lins) < 2 or lins[-1].out_features != 1:
      return "the MLP must end in a single logit"
    if lins[-2].out_features not in (64, 128, 256, 512, 1024):
      return "the fused loss kernel needs a last hidden layer of 64..1024 (power of two) units"
    if any(l.out_features % 8 for l in lins[:-1]):
      return "hidden layer widths must be multiples of 8"
    return None

  # ------------------------------------------------------------------ buffers
  def _alloc(self, b: int):
    dev, bf = self.dev, torch.bfloat16
    self.num_in = torch.zeros(b, max(self.n_num, 1), dtype=torch.float32, device=dev)
    self.lab_in = torch.zeros(b, dtype=torch.float32, device=dev)
    for L in self.hidden:
      L.y = torch.empty(b, L.out_f, dtype=bf, device=dev)
      L.dy = torch.empty(b, L.out_f, dtype=bf, device=dev)
    self.dx0 = torch.empty(b, self.in_pad, dtype=bf, device=dev)
    if self.pool is not None:
      self.x0 = torch.zeros(b, self.in_pad, dtype=bf, device=dev)
      self.demb = torch.empty(b, self.engine.total_width, dtype=bf, device=dev)
    self._batch = b
    self._graph = None

  # ------------------------------------------------------------------ the step
  def _forward(self):
    ops, eng = self.ops, self.engine
    tw = eng.total_width
    side = self._side
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
      eng.launch_forward()
    # MLP input [b, in_pad]: embeddings (or their pooled interaction) | numerical | zero pad
    x0 = eng.out_full if self.pool is None else self.x0
    if self.n_num:
      # numerical features into their columns of the MLP input (the pad columns stay zero)
      ops.copy_cast_2d(self.num_in, x0.data_ptr() + self.emb_cols * 2, self.in_pad, 1, 1.0)
    torch.cuda.current_stream().wait_stream(side)
    eng.wait_output()
    if self.pool is not None:
      ops.avgpool_fwd(eng.out, tw, x0, self.pool)
    self._x0 = x0
    x = x0
    for L in self.hidden:
      torch._addmm_activation(L.b16, x, L.w16.t(), out=L.y)
      x = L.y

  def _backward(self):
    ops, eng = self.ops, self.engine
    b = self._batch
    last = self.hidden[-1]
    self.loss.zero_()
    H = self.head
    ops.head_loss(last.y, H.w16.view(-1), H.b16, self.lab_in, 1.0 / b, last.dy,
                  H.gw.view(-1), H.gb, last.gb, self.loss, None)
    for i in range(len(self.hidden) - 1, -1, -1):
      L = self.hidden[i]
      x = self.hidden[i - 1].y if i > 0 else self._x0
      torch.mm(L.dy.t(), x, out_dtype=torch.float32, out=L.gw)
      if i > 0:
        below = self.hidden[i - 1]
        torch.mm(L.dy, L.w16, out=below.dy)
        ops.relu_bwd_bias(below.dy, below.y, below.gb)
      else:
        torch.mm(L.dy, L.w16, out=self.dx0)
    # gradient all-to-all: the embedding columns of the first layer's data gradient go straight
    # to the table owners (NVLink stores + "gradient ready" signal), then the fused update
    tw = eng.total_width
    if self.pool is None:
      demb = self.dx0[:, :tw]
    else:
      ops.avgpool_bwd(self.dx0, self.demb, tw, self.pool)
      demb = self.demb
    if eng.routes_mp is not None:
      ops.push_grad(eng.routes_mp, len(eng.routes_mp_np), demb, eng.act, 1.0,
                    eng.sync_grad_signal())
    side = self._side
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
      eng._backward_mp()
    if self.world > 1:
      self.ctx.allreduce_(self.gsym, self.n_flat, torch.float32, scale=1.0 / self.world)
    self.dense_opt.apply(ops, self.p16, self.g32, self.lr_t)
    torch.cuda.current_stream().wait_stream(side)

  def _step_impl(self):
    with nvtx.range("synthetic_forward"):
      self._forward()
    with nvtx.range("synthetic_backward_update"):
      self._backward()

  def set_lr(self, lr: float):
    self.lr = float(lr)
    self.lr_t.fill_(self.lr)
    self.engine.update_lr(self.lr)

  def load_batch(self, numerical, categorical, labels):
    """Copy one batch into the static buffers.  ``categorical``: the list of id tensors the
    module's ``forward`` takes (data-parallel or model-parallel inputs)."""
    b = int(numerical.shape[0])
    first = self._batch != b
    # staging may (re)build the engine: the captured graph holds the old buffer addresses
    key = self.engine._key
    self.engine.stage(list(categorical))
    if first or key != self.engine._key:
      self._alloc(b)
    self.num_in[:, :self.n_num].copy_(numerical, non_blocking=True)
    self.lab_in.copy_(labels.reshape(-1), non_blocking=True)

  def run(self) -> torch.Tensor:
    """One step on the loaded batch; returns the (device) mean loss of the local batch."""
    eng = self.engine
    if eng.de._fused_optimizer["kind"] != "sgd" and not eng.opt_state:
      eng.reset_optimizer_state()
    if eng._tables_dirty:
      eng._refresh_tables()
    if not self.use_cuda_graph:
      self._step_impl()
      return self.loss
    if self._graph is None:
      # warm up on a side stream with a zero learning rate and dry embedding updates (cuBLAS
      # workspaces, lazy kernel loading; neither weights nor optimizer state move), then capture.
      # A zero rate still moves the dense Adagrad / Adam state and step word: they are put back.
      self.lr_t.zero_()
      eng.update_lr(0.0)
      eng.dry_updates(True)
      dense_snap = self.dense_opt.snapshot()
      s = torch.cuda.Stream(device=self.dev)
      s.wait_stream(torch.cuda.current_stream())
      with torch.cuda.stream(s):
        for _ in range(2):
          self._step_impl()
      torch.cuda.current_stream().wait_stream(s)
      torch.cuda.synchronize()
      eng.dry_updates(False)
      self.dense_opt.restore(dense_snap)
      g = torch.cuda.CUDAGraph()
      with torch.cuda.graph(g):
        self._step_impl()
      self._graph = g
      self.set_lr(self.lr)
    self._graph.replay()
    return self.loss

  def step(self, numerical, categorical, labels) -> torch.Tensor:
    self.load_batch(numerical, categorical, labels)
    return self.run()

  def dense_optimizer_state(self) -> dict:
    """``{"kind", "step", "slots": {param_name: [tensor, ...]}}``: the dense optimizer state,
    each slot shaped like its parameter (no padding); the format of every trainer."""
    return self.dense_opt.state_dict(self.model)

  def load_dense_optimizer_state(self, state: dict):
    """Restore :meth:`dense_optimizer_state` output (of any trainer); another kind raises."""
    self.dense_opt.load_state_dict(self.model, state)
