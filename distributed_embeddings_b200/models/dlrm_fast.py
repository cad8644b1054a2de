"""Hand-scheduled DLRM training step (no autograd on the hot path) + whole-step CUDA graph.

The generic :class:`DLRM` module is convenient but pays for autograd bookkeeping, autocast weight
casts, index-based interaction and ~150 tiny launches per step.  ``DLRMTrainStep`` runs the same
math as one static schedule over preallocated buffers:

* dense parameters live in one flat fp32 master buffer with a bf16 shadow (one fused kernel does
  SGD + re-cast + gradient zeroing); gradients live in one flat buffer (symmetric memory when
  world > 1) that the one-shot NVLink all-reduce kernel reduces in place;
* MLP layers: cuBLASLt bf16 GEMMs forward (fused bias+ReLU epilogues) and for the weight
  gradients (K padded 13->16 and 479->480 so every layer meets the TMA alignment rules of the GEMM
  kernels); the data gradient of a layer above a ReLU is one first-party wgmma GEMM that applies the
  ReLU backward and sums the bias gradient of the layer below in its epilogue;
* dot interaction forward/backward: tensor-core kernels; the forward's head waits for the
  embedding owners' "output ready" signals, the backward pushes every piece of the embedding
  gradient straight into its owner's receive buffer over NVLink and signals "gradient ready";
* final layer + BCE loss + their backward: one kernel;
* embedding forward/backward: the fused P2P engine (``parallel/fused.py``);
* the whole step is captured in a CUDA graph and replayed (launch bound otherwise).

DLRM-DCNv2 (``DLRM(interaction="dcnv2")``) swaps the dot interaction for the low-rank cross
network: the lookups write straight into the columns of ``x0`` (``FusedEngine.set_out_row_stride``),
each cross layer is two cuBLASLt GEMMs and the memory-bound ``cross_fwd`` kernel forward, and
``cross_bwd`` + four GEMMs backward; ``cross_dx0`` gathers the gradient of ``x0``, whose embedding
columns ``push_grad`` routes to the table owners (see :class:`DLRMTrainStep`).

Same model/optimizer as the reference example (examples/dlrm/main.py:76-209): SGD, shared lr.
``dense_optimizer`` swaps the fused dense SGD for fused Adagrad or Adam (see ``dense_optimizer``).
"""
from __future__ import annotations

import copy
import os
from typing import Optional

import torch
from torch import nn

from ..ops import _native
from ..parallel.comm import CommContext
from ..parallel.fused import FusedEngine
from ..utils import nvtx
from ..utils.lr_schedule import LearningRateScheduler
from ..utils.metrics import BinnedAUC, ExactAUC, auc_from_counts, auc_from_histogram
from .dense_optimizer import FlatDenseOptimizer, dense_optimizer_config
from .dlrm import DLRM

# Tables with at least this many rows take their SGD update from the interaction backward
# (fused_table_update).  Chosen by tools/bench_fused_table_update.py (DESIGN §8): the fastest of
# 2500 / 20k / 100k / 1M / 20M rows on uniform and on power-law (alpha 1.05) ids alike.  Smaller
# tables stay in L2 and keep the scatter, which merges repeated ids within a tile.
FUSED_UPDATE_MIN_ROWS = 20000


def _pad8(n: int) -> int:
  return (n + 7) // 8 * 8


def _fused_dgrad(L) -> bool:
  """Whether the data gradient of layer ``L`` (its input a ReLU output) runs as one
  ``gemm_dgrad_relu_bias`` kernel instead of ``torch.mm`` + ``relu_bwd_bias``.  The kernel needs
  N = in_f <= 2048 columns, and 8-element rows (TMA strides of 16 bytes) for dy and W^T.
  tools/bench_dgrad.py times both on the DLRM shapes (DESIGN §8): the fused kernel is faster on
  every one of them."""
  return L.in_f == L.in_pad and L.in_f <= 2048 and L.out_f % 8 == 0


def _dgrad_block_n(L) -> int:
  """Tile width of the fused dgrad GEMM: 128 for K = out_f <= 256, where the shorter main loop
  leaves the epilogue the larger share and the 128-wide tile's deeper pipeline (5 stages instead
  of 3) wins (tools/bench_dgrad.py, DESIGN §8); else the kernel's choice."""
  return 128 if L.out_f <= 256 else 0


class _Layer:
  """One linear layer's slices of the flat buffers."""

  def __init__(self, lin: nn.Linear, relu: bool):
    self.lin = lin
    self.relu = relu
    self.out_f, self.in_f = lin.weight.shape
    self.in_pad = _pad8(self.in_f)
    self.w_off = self.b_off = 0
    self.w_numel = self.out_f * self.in_pad
    self.b_numel = _pad8(self.out_f) if lin.bias is not None else 0  # bias-free: no slot


class DLRMTrainStep:
  """Static-schedule training step for :class:`DLRM` on the fused embedding back end.

  ``dense_optimizer`` (``sgd`` | ``adagrad`` | ``adam`` | ``momentum``, hyperparameters in
  ``dense_optimizer_kwargs``) updates the MLPs and any replicated tables with the shared
  learning rate.  Replicated tables (``data_parallel_threshold``) need
  ``dense_optimizer == embedding_optimizer``, so the row-wise optimizers and ``ftrl`` need a model
  without replicated tables.

  ``fused_table_update``: on one GPU with the atomic SGD embedding update, the interaction
  backward applies the update of the tables with at least ``fused_update_min_rows`` rows
  itself, so their gradient rows skip the receive buffer (:meth:`FusedEngine.producer_update`).
  Other configurations run the same schedule either way; ``False`` keeps every table on the
  staged scatter.

  DLRM-DCNv2 (``model.interaction == "dcnv2"``, cuBLASLt GEMMs only): the engine writes the
  pooled (``sum``, ``model.multi_hot_sizes``) embeddings into the first ``26 * 128`` columns of
  ``x0 = [emb_0 | ... | emb_25 | bottom]`` (``engine.out_full``) and the bottom-MLP output is
  copied into its last 128.  Per cross layer ``l``, forward: ``u = x_l V^T``,
  ``s = u W^T + b`` (cuBLASLt, bias epilogue), ``x_{l+1} = cross_fwd(x0, s, x_l)``; backward,
  in reverse: ``g = cross_bwd(dy, x0)`` (also the bias gradient), ``gW = g^T u``, ``du = g W``,
  ``gV = du^T x_l``, ``dx_l = dy + du V``; then ``cross_dx0`` sums the gradient of ``x0``, its
  embedding columns go to the table owners through ``push_grad`` and its bottom columns into the
  bottom-MLP backward.  The cross parameters live in the flat buffers between the bottom and the
  top MLP.  ``fused_table_update`` does not apply: every table takes the engine's scatter /
  sorted update.  Multi-hot inputs need the ``dcnv2`` model; multi-hot row-sliced tables are
  not supported."""

  def __init__(self, model: DLRM, lr: float = 24.0, embedding_optimizer: str = "sgd",
               scheduler: Optional[LearningRateScheduler] = None, use_cuda_graph: bool = True,
               embedding_optimizer_kwargs: Optional[dict] = None, overlap: bool = True,
               gemm: str = "cublas", eval_thresholds: int = 8000, dense_optimizer: str = "sgd",
               dense_optimizer_kwargs: Optional[dict] = None, fused_table_update: bool = True,
               fused_update_min_rows: int = FUSED_UPDATE_MIN_ROWS, eval_auc: str = "binned",
               eval_capacity: Optional[int] = None):
    if eval_auc not in ("binned", "exact"):
      raise ValueError("eval_auc must be 'binned' or 'exact'")
    if eval_auc == "exact" and (eval_capacity is None or int(eval_capacity) < 1):
      raise ValueError("eval_auc='exact' needs eval_capacity: the number of samples one rank "
                       "evaluates between resets (4 bytes each)")
    if gemm not in ("cublas", "fused_dgrad", "tcgen05", "tcgen05_pair"):
      raise ValueError("gemm must be cublas | fused_dgrad | tcgen05 | tcgen05_pair")
    # Every value runs the data gradients below a ReLU on the first-party wgmma kernel with the
    # ReLU-backward mask + bias gradient fused in its epilogue (see _dgrad_relu).  cublas:
    # cuBLASLt for the forward and weight-gradient GEMMs; fused_dgrad is the same schedule, kept
    # as a name.  tcgen05: forward layers on the first-party kernel as well.  tcgen05_pair: same,
    # with the 2-CTA cluster kernel for layers at least 256 wide.  (The names are historical.)
    self.gemm = gemm
    self.dcn = getattr(model, "interaction", "dot") == "dcnv2"
    hots = getattr(model, "multi_hot_sizes", None)
    if self.dcn and gemm != "cublas":
      raise ValueError("the dcnv2 interaction runs its GEMMs on cuBLASLt: use gemm='cublas'")
    if not self.dcn and hots is not None and any(h != 1 for h in hots):
      raise ValueError("multi-hot features need the dcnv2 interaction in DLRMTrainStep")
    # single GPU with the atomic SGD update: the interaction backward updates the large tables
    # itself (see FusedEngine.producer_update); False keeps every table on the staged scatter
    self.fused_table_update = bool(fused_table_update)
    self.fused_update_min_rows = int(fused_update_min_rows)
    self.dense_cfg = dense_optimizer_config(dense_optimizer, dense_optimizer_kwargs)
    self.model = model
    self.emb = model.embedding
    if self.emb.backend != "fused":
      raise ValueError("DLRMTrainStep needs the fused embedding back end")
    self.dev = self.emb.device
    self.ops = _native.require()
    self.world = self.emb.world_size
    self.ctx = CommContext.for_group(self.emb.group, self.dev)
    self.scheduler = scheduler
    self.use_cuda_graph = use_cuda_graph
    self.overlap = overlap
    self.emb.set_optimizer(embedding_optimizer, lr=lr, **(embedding_optimizer_kwargs or {}))
    if self.emb._engine is None:
      self.emb._engine = FusedEngine(self.emb)
    self.engine: FusedEngine = self.emb._engine
    self.n_emb = len(model.table_sizes)
    self.dim = model.embedding_dim
    self.hots = list(hots) if hots is not None else [1] * self.n_emb
    if self.dcn:
      st = self.emb.strategy
      if self.emb.dp_input and any(self.hots[i] != 1 for i in st.input_groups[2]):
        raise NotImplementedError("the dcnv2 step does not support multi-hot row-sliced inputs")
      if self.dim % 8 or any(l.V.out_features % 8 for l in model.cross_layers):
        raise ValueError("the dcnv2 step needs an embedding width and a cross rank that are "
                         "multiples of 8")
    # gradient all-to-all through local staging + a streaming copy kernel next to the interaction
    # backward (DE_B200_STREAM_PUSH=0: the interaction backward stores into peer memory itself)
    # on from 4 GPUs: at 2 GPUs the copy kernel competes with an interaction backward that keeps
    # every SM busy (not measured on H100); DE_B200_STREAM_PUSH=0/1 overrides
    sp_env = os.environ.get("DE_B200_STREAM_PUSH", "auto")
    self._stream_push = self.world > 1 and (sp_env == "1" or (sp_env == "auto" and self.world >= 4))
    self._push_stream = torch.cuda.Stream(device=self.dev) if self._stream_push else None
    self._push_ready = torch.cuda.Event() if self._stream_push else None

    lins_b = [m for m in model.bottom_mlp.net if isinstance(m, nn.Linear)]
    lins_t = [m for m in model.top_mlp.net if isinstance(m, nn.Linear)]
    self.bottom = [_Layer(l, True) for l in lins_b]
    self.top = [_Layer(l, True) for l in lins_t[:-1]]
    self.head = _Layer(lins_t[-1], False)
    if self.head.out_f != 1:
      raise ValueError("the top MLP must end in a single logit")
    # cross layers (V, W) of the dcnv2 model; after the bottom MLP in the flat buffers, so that
    # they stay out of the top-MLP bucket that is all-reduced early
    self.cross = [(_Layer(c.V, False), _Layer(c.W, False)) for c in model.cross_layers] \
        if self.dcn else []
    layers = self.bottom + [L for pair in self.cross for L in pair] + self.top + [self.head]
    # replicated (data-parallel) embedding tables live in the flat dense buffers too: their
    # local-batch gradient is scattered into the gradient bucket, all-reduced with the MLP
    # gradients and applied densely by the fused dense optimizer kernel (the reference's
    # sparse_as_dense), so the dense and embedding optimizers must agree.  They come first so that
    # they belong to the bucket that is reduced last (DE_B200_AR_OVERLAP).  Covered by the 2- and
    # 8-GPU tests (tests/test_dist_gpu.py: replicated-table cases); bench.py replicates the
    # < 2500-row tables.
    self._dp_slots = []
    pos = 0
    if len(self.emb.dp_layers):
      if embedding_optimizer.lower() != self.dense_cfg["kind"]:
        if embedding_optimizer.lower().startswith("rowwise_"):
          raise ValueError(
              f"replicated tables in the fast step are updated by the dense optimizer kernel, "
              f"which has no row-wise form: embedding_optimizer={embedding_optimizer!r} needs "
              f"data_parallel_threshold=None (no replicated tables)")
        if embedding_optimizer.lower() == "ftrl":
          raise ValueError(
              "replicated tables in the fast step are updated by the dense optimizer kernel, "
              "which has no FTRL: a dense FTRL step would set every row the step does not touch "
              "to the closed form of its z.  embedding_optimizer='ftrl' needs "
              "data_parallel_threshold=None (no replicated tables)")
        raise ValueError("replicated tables in the fast step are updated by the dense optimizer "
                         "kernel: use the same embedding_optimizer and dense_optimizer ('sgd', "
                         "'adagrad', 'adam' or 'momentum') or data_parallel_threshold=None")
      for layer in self.emb.dp_layers:
        w = layer.embeddings
        self._dp_slots.append((pos, tuple(w.shape)))
        pos += _pad8(w.numel())
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
      # prefer an NVSwitch multicast mapping (in-switch reduction), else plain peer mappings
      self.gsym = self.ctx.alloc_multicast(pos * 4, "dense_grads") or \
          self.ctx.alloc(pos * 4, "dense_grads")
      self.allreduce_kind = "nvls_multimem" if getattr(self.gsym, "mc_ptr", 0) else "p2p"
      self.g32 = self.gsym.view(torch.float32, (pos,))
    else:
      self.gsym = None
      self.allreduce_kind = "none"
      self.g32 = torch.zeros(pos, dtype=torch.float32, device=dev)
    # move the module parameters into the flat master buffer (strided views keep the module usable)
    with torch.no_grad():
      dp_targets = []
      for layer, (off, shape) in zip(self.emb.dp_layers, self._dp_slots):
        n = shape[0] * shape[1]
        view = self.p32[off:off + n].view(shape)
        view.copy_(layer.embeddings.data)
        layer.embeddings.data = view
        dp_targets.append(self.g32[off:off + n].view(shape))
      if self._dp_slots:
        self.engine.set_dp_grad_targets(dp_targets)
        self.engine._tables_dirty = True
        self.engine._key = None  # descriptors built earlier point at the old table storage
      for L in layers:
        wv = self.p32[L.w_off:L.w_off + L.w_numel].view(L.out_f, L.in_pad)
        wv[:, :L.in_f].copy_(L.lin.weight)
        L.lin.weight.data = wv[:, :L.in_f]
        if L.lin.bias is not None:
          bv = self.p32[L.b_off:L.b_off + L.out_f]
          bv.copy_(L.lin.bias)
          L.lin.bias.data = bv
        L.w16 = self.p16[L.w_off:L.w_off + L.w_numel].view(L.out_f, L.in_pad)
        L.b16 = self.p16[L.b_off:L.b_off + L.out_f]
        L.gw = self.g32[L.w_off:L.w_off + L.w_numel].view(L.out_f, L.in_pad)
        L.gb = self.g32[L.b_off:L.b_off + L.b_numel]
        L.w16T = torch.empty(L.in_pad, L.out_f, dtype=torch.bfloat16, device=dev)
      self.p16.copy_(self.p32)
      self._refresh_transposes()
    self.dense_opt = FlatDenseOptimizer(self.dense_cfg, self.p32)
    self.lr_t = torch.full((1,), float(lr), dtype=torch.float32, device=dev)
    self.engine.share_lr(self.lr_t)  # dense optimizer and fused embedding update read one word
    self.lr = float(lr)
    self.loss = torch.zeros(1, dtype=torch.float32, device=dev)
    self._batch = None
    self._graph = None
    self._side = torch.cuda.Stream(device=dev) if overlap else None
    # weight-gradient GEMMs are off the critical path (head -> dgrads -> interaction -> embedding
    # backward): they run on a second side stream and join before the all-reduce
    # (at small local batches the full-GPU cuBLAS kernels of the two streams interleave and
    # stretch the critical chain, so it is only enabled for large local batches; not measured on
    # H100; DE_B200_WGRAD_STREAM=0/1 overrides)
    self._wgrad_overlap = os.environ.get("DE_B200_WGRAD_STREAM", "auto")
    self._wstream = torch.cuda.Stream(device=dev) if overlap else None
    # The top-MLP + head gradients (93 % of the dense parameters, complete as soon as the top MLP
    # backward is done) are all-reduced on a third stream while the interaction backward, the
    # embedding exchange and the bottom MLP backward run; only the small bottom-MLP bucket is
    # reduced at the end.  The overlapped kernel is capped at 32 blocks so that its flag spins
    # cannot starve the kernels the peers wait for.  DE_B200_AR_OVERLAP=0/1 overrides the default
    # (on from 4 GPUs).
    ar_env = os.environ.get("DE_B200_AR_OVERLAP", "auto")
    # off at 2 GPUs: the large local batch keeps every SM busy and the overlapped kernel only
    # steals from the interaction backward (not measured on H100)
    ar_on = ar_env == "1" or (ar_env == "auto" and self.world >= 4)
    self._ar_stream = torch.cuda.Stream(device=dev) if (overlap and self.world > 1 and ar_on) \
        else None
    # evaluation metrics, accumulated on the device by the head_eval kernel (see evaluate())
    self.eval_auc = BinnedAUC(eval_thresholds, device=dev)
    self._eval_loss = torch.zeros(1, dtype=torch.float64, device=dev)
    self._eval_count = torch.zeros(1, dtype=torch.int64, device=dev)
    # eval_auc="exact": every evaluated sample's key, appended by auc_append in the eval graph
    self.eval_auc_mode = eval_auc
    self.exact_auc = ExactAUC(eval_capacity, device=dev) if eval_auc == "exact" else None
    self._eval_graph = None

  def _refresh_transposes(self):
    """K-major copies of W^T for the fused dgrad GEMMs (1.9 M elements, a few microseconds)."""
    for L in self.bottom[1:] + self.top[1:]:
      if _fused_dgrad(L):
        L.w16T.copy_(L.w16.t())

  def _linear_fwd(self, L, x):
    if self.gemm in ("tcgen05", "tcgen05_pair"):
      pair = self.gemm == "tcgen05_pair" and L.out_f >= 256
      self.ops.gemm_tn_bias_act(x, L.w16, L.b16, L.y, True, 512 if pair else 0)
    else:
      torch._addmm_activation(L.b16, x, L.w16.t(), out=L.y)
    return L.y

  def _wgrad(self, L, x):
    """gw = dy^T @ x (fp32), on the weight-gradient stream."""
    use = self._wstream is not None and (
        self._wgrad_overlap == "1" or
        (self._wgrad_overlap == "auto" and (self._batch or 0) >= 49152))
    if not use:
      torch.mm(L.dy.t(), x, out_dtype=torch.float32, out=L.gw)
      return
    self._w_used = True
    self._wstream.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(self._wstream):
      torch.mm(L.dy.t(), x, out_dtype=torch.float32, out=L.gw)

  def _dgrad_relu(self, L, x_below, dx, gb_below):
    """dx = (dy @ W) * (x_below > 0); gb_below += colsum(dx)."""
    if _fused_dgrad(L):
      self.ops.gemm_dgrad_relu_bias(L.dy, L.w16T, x_below, dx, gb_below, _dgrad_block_n(L))
    else:
      torch.mm(L.dy, L.w16, out=dx)
      self.ops.relu_bwd_bias(dx, x_below, gb_below)

  # ------------------------------------------------------------------ buffers
  def _alloc(self, b: int):
    dev, bf = self.dev, torch.bfloat16
    if self.dcn:
      self._alloc_dcn(b)
    else:
      if self._stream_push:
        # chunks of >= 1024 samples, at most 16 of them: the last chunk's transfer is the only
        # part of the exchange that does not overlap the interaction backward
        self.engine.enable_streamed_push(max(1024, -(-b // 16)))
      self.engine.prepare(b, [1] * self.n_emb, ids64=False)
      self.cat_stage = self.engine.in_flat[:self.n_emb * b].view(self.n_emb, b)
    self.num_in = torch.zeros(b, self.bottom[0].in_f, dtype=torch.float32, device=dev)
    self.lab_in = torch.zeros(b, dtype=torch.float32, device=dev)
    self.x0 = torch.zeros(b, self.bottom[0].in_pad, dtype=bf, device=dev)
    for L in self.bottom + self.top:
      L.y = torch.empty(b, L.out_f, dtype=bf, device=dev)
      L.dy = torch.empty(b, L.out_f, dtype=bf, device=dev)
    if not self.dcn:
      self.z = torch.zeros(b, self.top[0].in_pad, dtype=bf, device=dev)
      self.dz = torch.empty(b, self.top[0].in_pad, dtype=bf, device=dev)
    self._batch = b
    self._graph = None
    self._eval_graph = None
    self._n_valid = torch.zeros(1, dtype=torch.int64, device=dev)
    self._probs = torch.zeros(b, dtype=torch.float32, device=dev)
    # double-buffered device staging for the asynchronous input pipeline (prefetch())
    self._stage = [(torch.zeros_like(self.cat_stage), torch.zeros_like(self.num_in),
                    torch.zeros_like(self.lab_in)) for _ in range(2)]
    self._slot_dev = torch.zeros(1, dtype=torch.int32, device=dev)
    self._slot_host = torch.tensor([[0], [1]], dtype=torch.int32).pin_memory()
    self._h2d_done = [torch.cuda.Event(), torch.cuda.Event()]
    self._consumed = [torch.cuda.Event(), torch.cuda.Event()]
    self._prefetched = 0   # batches handed to prefetch()
    self._consumed_n = 0   # batches run
    self._use_stage = False

  def _alloc_dcn(self, b: int):
    """Buffers of the cross network: x0 is the engine's output matrix; x_1..x_L, s_l and u_l are
    kept for the backward; dX[l] is the gradient of x_l (dX[0]: the chain part of dx0)."""
    dev, bf = self.dev, torch.bfloat16
    eng = self.engine
    D = self.model.cross_dim
    eng.set_out_row_stride(D)
    eng.prepare(b, self.hots, ids64=False)
    if eng.out_needs_reduce:
      raise NotImplementedError("the dcnv2 step does not support multi-hot row-sliced inputs")
    # ids, feature-major and sample-major within a feature: [sum_f h_f * b] (see prefetch())
    self.cat_stage = eng.in_flat[:sum(self.hots) * b]
    self.emb_cols = eng.total_width
    L = len(self.cross)
    self.xs = [eng.out_full] + [torch.empty(b, D, dtype=bf, device=dev) for _ in range(L)]
    self.ss = [torch.empty(b, D, dtype=bf, device=dev) for _ in range(L)]
    self.us = [torch.empty(b, V.out_f, dtype=bf, device=dev) for V, _ in self.cross]
    self.dX = [torch.empty(b, D, dtype=bf, device=dev) for _ in range(L + 1)]
    self.g = torch.empty(b, D, dtype=bf, device=dev)  # cross_bwd output; dx0 at the end
    self.du = torch.empty(b, max(V.out_f for V, _ in self.cross), dtype=bf, device=dev)

  # ------------------------------------------------------------------ the step
  def _select_stage(self):
    a, b_ = self._stage
    self.ops.select_copy([a[0], a[1], a[2]], [b_[0], b_[1], b_[2]],
                         [self.cat_stage, self.num_in, self.lab_in], self._slot_dev)

  def _forward(self, train: bool = True):
    """Forward up to the top MLP output on the inputs in ``cat_stage`` / ``num_in``; ``train``:
    a training step follows (False: evaluation)."""
    ops = self.ops
    # the embedding exchange (id push, gather + NVLink push of the pooled rows; all signalling
    # folded into those kernels) runs on the side stream while the bottom MLP runs on the main
    # stream; they meet at the interaction, whose head waits for the owners' "output ready"
    eng = self.engine
    if self._side is not None:
      self._side.wait_stream(torch.cuda.current_stream())
      with torch.cuda.stream(self._side):
        eng.launch_forward(train)
    ops.cast_pad(self.num_in, self.x0)
    x = self.x0
    for L in self.bottom:
      x = self._linear_fwd(L, x)
    if self._side is not None:
      torch.cuda.current_stream().wait_stream(self._side)
    else:
      eng.launch_forward(train)
    if eng.out_needs_reduce:  # multi-hot row slices: partial pools are summed first
      eng.wait_output()
      ops.interact_fwd(x, eng.out, self.n_emb, self.z, [])
    else:
      ops.interact_fwd(x, eng.out, self.n_emb, self.z, eng.sync_out_wait())
    x = self.z
    for L in self.top:
      x = self._linear_fwd(L, x)

  def _forward_dcn(self, train: bool = True):
    """Forward of the dcnv2 model up to the top MLP output."""
    ops, eng = self.ops, self.engine
    # lookups (into x0's embedding columns) on the side stream under the bottom MLP
    if self._side is not None:
      self._side.wait_stream(torch.cuda.current_stream())
      with torch.cuda.stream(self._side):
        eng.launch_forward(train)
    ops.cast_pad(self.num_in, self.x0)
    x = self.x0
    for L in self.bottom:
      x = self._linear_fwd(L, x)
    x0 = self.xs[0]
    ops.copy_cast_2d(x, x0.data_ptr() + self.emb_cols * x0.element_size(), x0.stride(0), 1, 1.0)
    if self._side is not None:
      torch.cuda.current_stream().wait_stream(self._side)
    else:
      eng.launch_forward(train)
    eng.wait_output()
    x = x0
    for l, (V, W) in enumerate(self.cross):
      u, s_ = self.us[l], self.ss[l]
      torch.mm(x, V.w16.t(), out=u)
      torch.addmm(W.b16, u, W.w16.t(), out=s_)
      ops.cross_fwd(x0, s_, x, self.xs[l + 1])
      x = self.xs[l + 1]
    for L in self.top:
      x = self._linear_fwd(L, x)

  def _backward_dcn(self):
    ops, eng = self.ops, self.engine
    b = self._batch
    last = self.top[-1]
    self.loss.zero_()
    H = self.head
    ops.head_loss(last.y, H.w16.view(-1), H.b16, self.lab_in, 1.0 / b, last.dy,
                  H.gw.view(-1), H.gb, last.gb, self.loss, None)
    nL = len(self.cross)
    for i in range(len(self.top) - 1, -1, -1):
      L = self.top[i]
      x = self.top[i - 1].y if i > 0 else self.xs[nL]
      self._wgrad(L, x)
      if i > 0:
        self._dgrad_relu(L, x, self.top[i - 1].dy, self.top[i - 1].gb)
      else:  # x_L is no ReLU output: plain dgrad
        torch.mm(L.dy, L.w16, out=self.dX[nL])
    self._allreduce_top_early()
    # cross layers in reverse; their weight gradients stay on this stream (g and du are reused)
    x0 = self.xs[0]
    for l in range(nL - 1, -1, -1):
      V, W = self.cross[l]
      dy = self.dX[l + 1]
      du = self.du[:, :V.out_f]
      ops.cross_bwd(dy, x0, self.g, W.gb)
      torch.mm(self.g.t(), self.us[l], out_dtype=torch.float32, out=W.gw)
      torch.mm(self.g, W.w16, out=du)
      torch.mm(du.t(), self.xs[l], out_dtype=torch.float32, out=V.gw)
      torch.addmm(dy, du, V.w16, out=self.dX[l])
    # dx0 (into g): embedding columns to the table owners, bottom columns to the bottom MLP
    hb = self.bottom[-1]
    ops.cross_dx0(self.dX[0], self.dX[1:], self.ss, self.g, hb.dy)
    if eng.routes_all is not None:
      ops.push_grad(eng.routes_all, len(eng.routes_all_np), self.g[:, :self.emb_cols], eng.act,
                    1.0, eng.sync_grad_signal())
    self._backward_tail(None, False)

  def _allreduce_top_early(self):
    """Top-MLP + head bucket on the all-reduce stream (when enabled), under the rest of the
    backward."""
    if self._ar_stream is not None:
      ar = self._ar_stream
      ar.wait_stream(torch.cuda.current_stream())
      if getattr(self, "_w_used", False):
        ar.wait_stream(self._wstream)
      off = self.top[0].w_off  # flat layout: bottom layers | cross layers | top layers | head
      with torch.cuda.stream(ar):
        self.ctx.allreduce_(self.gsym, self.n_flat - off, torch.float32, scale=1.0 / self.world,
                            byte_offset=off * 4, max_blocks=32)

  def _backward(self):
    ops, eng = self.ops, self.engine
    b = self._batch
    last = self.top[-1]
    self.loss.zero_()
    H = self.head
    # final layer + loss + their backward; also the ReLU mask and bias gradient of the layer below
    ops.head_loss(last.y, H.w16.view(-1), H.b16, self.lab_in, 1.0 / b, last.dy,
                  H.gw.view(-1), H.gb, last.gb, self.loss, None)
    # top MLP backward
    for i in range(len(self.top) - 1, -1, -1):
      L = self.top[i]
      x = self.top[i - 1].y if i > 0 else self.z
      dx = self.top[i - 1].dy if i > 0 else self.dz
      self._wgrad(L, x)
      if i > 0:
        self._dgrad_relu(L, x, dx, self.top[i - 1].gb)
      else:
        torch.mm(L.dy, L.w16, out=dx)
    self._allreduce_top_early()
    # interaction backward: every piece of the embedding gradient is stored straight into the
    # receive buffer of the rank that owns the table (slice) - the gradient all-to-all rides on
    # the kernel's epilogue stores - and its tail signals "gradient ready" to the owners
    hb = self.bottom[-1]
    pushed = eng.streamed_push
    applied = None
    if pushed:
      # pieces of remote owners are staged locally; the copy kernel (own stream, a few blocks)
      # forwards every finished chunk over NVLink while the interaction backward keeps computing.
      # The producer is launched FIRST: the copy kernel spins on the producer's progress, so it
      # must never sit in front of it in a hardware queue the two streams happen to share
      # (streams alias onto CUDA_DEVICE_MAX_CONNECTIONS queues) - launched second it at worst
      # runs after the producer instead of next to it.
      eng.push_counters.zero_()
      self._push_ready.record(torch.cuda.current_stream())
      ops.interact_bwd(hb.y, eng.out, self.n_emb, self.dz, hb.dy, 0, 0, 1.0, eng.routes_stage,
                       len(eng.routes_stage_np), [], eng.push_counters, eng.push_chunk_rows)
      self._push_stream.wait_event(self._push_ready)
      with torch.cuda.stream(self._push_stream):
        eng.launch_streamed_push()
    else:
      # single GPU, SGD: the interaction backward also applies the update of the large tables
      # (FusedEngine.producer_update); their gradient rows never go through the receive buffer
      applied = eng.producer_update(self.dim, self.fused_update_min_rows) \
          if self.fused_table_update else None
      ops.interact_bwd(hb.y, eng.out, self.n_emb, self.dz, hb.dy, 0, 0, 1.0, eng.routes_all,
                       len(eng.routes_all_np), eng.sync_grad_signal(), None, 0,
                       *(applied.interact_args() if applied else ()))
    self._backward_tail(applied, pushed)

  def _backward_tail(self, applied, pushed: bool):
    """Embedding update (side stream) under the bottom-MLP backward, all-reduce, optimizer."""
    ops, eng = self.ops, self.engine
    hb = self.bottom[-1]
    # embedding exchange + fused table update, overlapped with the bottom MLP backward
    if self._side is not None:
      self._side.wait_stream(torch.cuda.current_stream())
      if pushed:  # the update's head waits for every rank's copy kernel: ours must be done first
        self._side.wait_stream(self._push_stream)
      with torch.cuda.stream(self._side):
        eng.backward_inplace(applied)
    else:
      if pushed:
        torch.cuda.current_stream().wait_stream(self._push_stream)
      eng.backward_inplace(applied)
    ops.relu_bwd_bias(hb.dy, hb.y, hb.gb)
    for i in range(len(self.bottom) - 1, -1, -1):
      L = self.bottom[i]
      x = self.bottom[i - 1].y if i > 0 else self.x0
      self._wgrad(L, x)
      if i > 0:
        self._dgrad_relu(L, x, self.bottom[i - 1].dy, self.bottom[i - 1].gb)
    # dense gradient all-reduce (one NVLink kernel, averaged) + fused optimizer / re-cast / zero
    if self._dp_slots and self._side is not None:
      # the replicated tables' gradients are produced by the embedding backward on the side stream
      torch.cuda.current_stream().wait_stream(self._side)
    if getattr(self, "_w_used", False):  # join only a stream that took part in this step
      torch.cuda.current_stream().wait_stream(self._wstream)
      self._w_used = False
    if self.world > 1:
      if self._ar_stream is not None:
        # bottom-MLP bucket, behind the top bucket on the same stream (one flag channel)
        ar = self._ar_stream
        ar.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(ar):
          self.ctx.allreduce_(self.gsym, self.top[0].w_off, torch.float32, scale=1.0 / self.world)
        torch.cuda.current_stream().wait_stream(ar)
      else:
        self.ctx.allreduce_(self.gsym, self.n_flat, torch.float32, scale=1.0 / self.world)
    self.dense_opt.apply(ops, self.p16, self.g32, self.lr_t)
    self._refresh_transposes()
    if self._side is not None:
      torch.cuda.current_stream().wait_stream(self._side)

  def _step_impl(self):
    with nvtx.range("dlrm_forward"):
      if self._use_stage:
        self._select_stage()
      self._forward_dcn() if self.dcn else self._forward()
    with nvtx.range("dlrm_backward_update"):
      self._backward_dcn() if self.dcn else self._backward()

  def set_lr(self, lr: float):
    self.lr = float(lr)
    self.lr_t.fill_(self.lr)  # shared with the embedding engine: one fill per schedule step
    if self.emb._fused_optimizer is not None:
      self.emb._fused_optimizer["lr"] = self.lr

  def load_batch(self, numerical, categorical, labels):
    """Copy one batch into the static input buffers (host pinned or device tensors).
    ``categorical``: ``[n_features, batch]`` tensor (feature major) or list of ``[batch]``; for
    the dcnv2 model a list of ``[batch, h_f]`` (or ``[batch]`` for h_f = 1) tensors, or the flat
    layout of :meth:`prefetch`.
    :meth:`evaluate` / :meth:`predict` overwrite these buffers: do not evaluate between this
    call and the :meth:`run` that consumes the batch."""
    b = int(numerical.shape[0])
    if b != self._batch:
      self._alloc(b)
    self.num_in.copy_(numerical, non_blocking=True)
    self.lab_in.copy_(labels.reshape(-1), non_blocking=True)
    if isinstance(categorical, (list, tuple)):
      for v, c in zip(self.engine.in_views, categorical):
        v.copy_(c.reshape(v.shape), non_blocking=True)
    elif self.dcn:
      self.cat_stage.copy_(categorical.reshape(-1), non_blocking=True)
    else:
      self.cat_stage.copy_(categorical, non_blocking=True)

  def prefetch(self, numerical, categorical, labels):
    """Asynchronous input pipeline: enqueue the H2D copy of the *next* batch (pinned host
    tensors; ``categorical`` as ``[n_features, batch]`` int32) on the copy stream while the
    current step runs.  Consume with :meth:`run_prefetched` in the same order.

    dcnv2 model: ``categorical`` is the engine's packed id layout, one int32 tensor of
    ``sum_f h_f * batch`` ids: feature-major, and within a feature sample-major (the ``h_f`` ids
    of sample 0, then those of sample 1, ...), i.e. ``torch.cat([c.reshape(-1) for c in ids])``
    of the ``[batch, h_f]`` tensors :meth:`step` takes."""
    b = int(numerical.shape[0])
    if b != self._batch:
      self._alloc(b)
    if not self._use_stage:
      self._use_stage = True
      self._graph = None  # the staged schedule starts with select_copy
      self._copy_stream = torch.cuda.Stream(device=self.dev)
    slot = self._prefetched & 1
    cs = self._copy_stream
    if self._prefetched >= 2:
      cs.wait_event(self._consumed[slot])  # the step that used this slot has been enqueued & done
    with torch.cuda.stream(cs):
      st = self._stage[slot]
      st[0].copy_(categorical.reshape(-1) if self.dcn else categorical, non_blocking=True)
      st[1].copy_(numerical, non_blocking=True)
      st[2].copy_(labels.reshape(-1), non_blocking=True)
      self._h2d_done[slot].record(cs)
    self._prefetched += 1

  def run_prefetched(self) -> torch.Tensor:
    """Run one step on the oldest prefetched batch."""
    assert self._consumed_n < self._prefetched, "call prefetch() first"
    slot = self._consumed_n & 1
    main = torch.cuda.current_stream()
    main.wait_event(self._h2d_done[slot])
    self._slot_dev.copy_(self._slot_host[slot], non_blocking=True)
    loss = self.run()
    self._consumed[slot].record(main)
    self._consumed_n += 1
    return loss

  def run(self) -> torch.Tensor:
    """Run one step on the loaded batch; returns the (device) mean loss of the local batch."""
    if self.scheduler is not None:
      self.set_lr(self.scheduler.step())
    if not self.use_cuda_graph:
      self._step_impl()
      return self.loss
    if self._graph is None:
      # warm up on a side stream (cuBLAS handles / workspaces), then capture.  The learning rate
      # is zero while warming up so the extra passes leave the weights untouched.
      self.lr_t.zero_()
      self.engine.dry_updates(True)  # optimizer state (Adagrad / Adam) stays untouched as well
      # a zero rate still moves the dense Adagrad / Adam state and step word: put them back
      dense_snap = self.dense_opt.snapshot()
      s = torch.cuda.Stream(device=self.dev)
      s.wait_stream(torch.cuda.current_stream())
      with torch.cuda.stream(s):
        for _ in range(2):
          self._step_impl()
      torch.cuda.current_stream().wait_stream(s)
      torch.cuda.synchronize()
      self.engine.dry_updates(False)
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

  # ------------------------------------------------------------------ checkpoint
  def dense_optimizer_state(self) -> dict:
    """``{"kind", "step", "slots": {param_name: [tensor, ...]}}``: the dense optimizer state,
    each slot shaped like its parameter (no padding); the format of every trainer."""
    return self.dense_opt.state_dict(self.model)

  def load_dense_optimizer_state(self, state: dict):
    """Restore :meth:`dense_optimizer_state` output (of any trainer); another kind raises."""
    self.dense_opt.load_state_dict(self.model, state)

  # ------------------------------------------------------------------ evaluation
  # The forward-only schedule reuses the step's input and activation buffers and its GEMM back
  # end, and ends in head_eval instead of head_loss + backward.  It changes nothing a training
  # step owns (tables, optimizer state, step_t, p32 / p16 / g32, lr_t, the scheduler, the
  # prefetch slots), so evaluations may sit between run() / run_prefetched() calls and the
  # training graph stays valid.  It does overwrite the static inputs, so an evaluation must not
  # separate load_batch() from the run() that consumes it.
  #
  # At world size > 1 it is collective (every rank runs the same number of chunks) and needs no
  # signal of its own: a requester's next id push is ordered behind its interaction forward,
  # which waited for every owner's "output ready" signal, and each owner sends that from the tail
  # of the lookup that read the ids.  No rank signals "consumed" during an evaluation, so those
  # counts stay equal on all ranks and the next training step's id push waits as before.
  def _eval_impl(self):
    with nvtx.range("dlrm_eval"):
      # a forward-only pass: the offload cache marks no row dirty
      self._forward_dcn(False) if self.dcn else self._forward(False)
      H = self.head
      self.ops.head_eval(self.top[-1].y, H.w16.view(-1), H.b16, self.lab_in, self._n_valid,
                         self._probs, self.eval_auc.hist, self._eval_loss, self._eval_count)
      if self.exact_auc is not None:
        self.ops.auc_append(self._probs, self.lab_in, self._n_valid, self.exact_auc.keys,
                            self.exact_auc.state)

  def _eval_ready(self):
    if self._batch is None:
      raise RuntimeError("evaluation runs in chunks of the training batch: load or run a "
                         "training batch first")
    if self.engine.out_needs_reduce:
      raise NotImplementedError("evaluation does not support multi-hot row-sliced inputs")
    if not self.use_cuda_graph or self._eval_graph is not None:
      return
    # warm up with no valid rows (metrics untouched), then capture the forward-only schedule
    self._n_valid.zero_()
    s = torch.cuda.Stream(device=self.dev)
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
      self._eval_impl()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
      self._eval_impl()
    self._eval_graph = g

  def _eval_chunks(self, numerical, categorical, labels, out=None):
    """Run the forward-only schedule over ``n`` samples in chunks of the training batch; the
    last chunk is padded with id 0 and zero numerical features."""
    n = int(numerical.shape[0])
    if n < 1:
      raise ValueError("evaluation needs at least one sample")
    self._eval_ready()
    b = self._batch
    lab = labels.reshape(-1) if labels is not None else None
    if self.dcn:
      cats = None
    elif isinstance(categorical, (list, tuple)):
      cats = [c.reshape(-1) for c in categorical]
    else:
      cats = None
    for s in range(0, n, b):
      m = min(b, n - s)
      self.num_in[:m].copy_(numerical[s:s + m], non_blocking=True)
      if self.dcn:
        for v, c in zip(self.engine.in_views, categorical):
          v[:m].copy_(c[s:s + m].reshape(m, -1), non_blocking=True)
          if m < b:
            v[m:].zero_()
        if m < b:
          self.num_in[m:].zero_()
      elif cats is None:
        self.cat_stage[:, :m].copy_(categorical[:, s:s + m], non_blocking=True)
      else:
        for f, c in enumerate(cats):
          self.cat_stage[f, :m].copy_(c[s:s + m], non_blocking=True)
      if m < b and not self.dcn:
        self.num_in[m:].zero_()
        self.cat_stage[:, m:].zero_()
      if lab is not None:
        self.lab_in[:m].copy_(lab[s:s + m], non_blocking=True)
      self._n_valid.fill_(m if lab is not None else 0)
      if self.use_cuda_graph:
        self._eval_graph.replay()
      else:
        self._eval_impl()
      if out is not None:
        out[s:s + m].copy_(self._probs[:m])

  def evaluate(self, numerical, categorical, labels):
    """Accumulate the evaluation metrics (binned ROC AUC, log loss; with ``eval_auc="exact"``
    also every sample's exact-AUC key, at most ``eval_capacity`` per rank) over ``n >= 1`` local
    samples: ``numerical [n, 13]``, ``categorical`` ``[n_features, n]`` or a list of ``[n]``
    (dcnv2 model: a list of ``[n, h_f]``), ``labels [n]``.  Nothing is copied to the host; read
    the result with :meth:`eval_metrics`."""
    self._eval_chunks(numerical, categorical, labels)

  def predict(self, numerical, categorical) -> torch.Tensor:
    """fp32 click probabilities ``[n]`` (device) of ``n >= 1`` local samples; the metrics are
    left unchanged."""
    out = torch.empty(int(numerical.shape[0]), dtype=torch.float32, device=self.dev)
    self._eval_chunks(numerical, categorical, None, out)
    return out

  def eval_metrics(self, reset: bool = True) -> dict:
    """``{"auc", "tie_bound", "log_loss", "samples"}`` over everything :meth:`evaluate` saw since
    the last reset, summed over all ranks (collective at world size > 1: one all-reduce).
    ``tie_bound`` bounds ``|auc - exact AUC|`` (see ``utils.metrics.BinnedAUC``).

    ``eval_auc="exact"``: ``{"auc", "binned_auc", "tie_bound", "log_loss", "samples"}`` with the
    exact ROC AUC of every rank's samples (``utils.metrics.ExactAUC``; at world size > 1 the keys
    are all-gathered, so every rank returns the same value) and the binned one beside it.  Raises
    when a rank evaluated more than ``eval_capacity`` samples or saw a NaN probability."""
    hist = self.eval_auc.hist.view(-1)
    packed = torch.cat([hist.double(), self._eval_loss, self._eval_count.double()])
    if self.world > 1:
      import torch.distributed as dist
      dist.all_reduce(packed, group=self.emb.group)
    packed = packed.cpu()  # counts stay exact in float64 below 2^53
    nb = hist.numel()
    res = auc_from_histogram(packed[:nb].round().long().view(2, -1))
    loss, count = float(packed[nb]), int(round(float(packed[nb + 1])))
    exact = None
    if self.exact_auc is not None:
      m = self.exact_auc
      if self.world > 1:
        m = copy.copy(m)  # all_gather replaces the copy's buffers, not the graph's
        m.all_gather(self.emb.group)
      exact = auc_from_counts(*m.counts())
    if reset:
      self.eval_auc.reset()
      self._eval_loss.zero_()
      self._eval_count.zero_()
      if self.exact_auc is not None:
        self.exact_auc.reset()
    log_loss = loss / count if count else float("nan")
    if exact is not None:
      return {"auc": exact, "binned_auc": res.auc, "tie_bound": res.tie_bound,
              "log_loss": log_loss, "samples": count}
    return {"auc": res.auc, "tie_bound": res.tie_bound, "log_loss": log_loss, "samples": count}
