"""Hybrid-parallel embedding wrapper.

``DistributedEmbedding`` distributes a list of embedding tables over the ranks of a process group
(data-parallel small tables, table-parallel + column-sliced tables, row-sliced huge tables) and
runs the index / pooled-vector exchanges.  Two execution back ends share the plan, the weights and
the checkpoint surface:

* ``fused`` (CUDA): descriptor-driven sm_90a kernels that read indices from and write pooled
  vectors / pull gradients to peer HBM over NVLink (see ``fused.py``); no NCCL on the hot path.
* ``torch``: the same data flow expressed with ``torch.distributed`` collectives and autograd
  (works on CPU/gloo and GPU/NCCL, with user-defined embedding layers and host-resident tables).
  This is the measured NCCL baseline and the oracle for the fused path.

Capability parity: ``distributed_embeddings/python/layers/dist_model_parallel.py`` of the
reference (``DistributedEmbedding`` :712-1214, hybrid helpers :1217-1329).
"""
from __future__ import annotations

import os
from typing import Any, Dict, List, Optional, Sequence, Union

import numpy as np
import torch
import torch.distributed as dist
from torch import nn

from ..layers.embedding import Embedding, config_from_layer
from ..ops import embedding_lookup_ops as elo
from ..ops.ragged import RaggedIds, SparseIds
from ..ops.stochastic_rounding import check_state_dtype
from ..utils import initializers
from .comm import dist_ready
from .strategy import DistEmbeddingStrategy, STRATEGIES, suggest_column_slice_threshold


# ------------------------------------------------------------------------- autograd collectives
class _AllToAllSingle(torch.autograd.Function):
  """all_to_all_single whose backward is the reverse exchange scaled by ``grad_scale``."""

  @staticmethod
  def forward(ctx, x, out_splits, in_splits, group, grad_scale):
    ctx.meta = (out_splits, in_splits, group, grad_scale, x.shape)
    out = x.new_empty((sum(out_splits),) + tuple(x.shape[1:]))
    dist.all_to_all_single(out, x.contiguous(), out_splits, in_splits, group=group)
    return out

  @staticmethod
  def backward(ctx, grad):
    out_splits, in_splits, group, grad_scale, shape = ctx.meta
    gin = grad.new_empty(shape)
    dist.all_to_all_single(gin, grad.contiguous(), in_splits, out_splits, group=group)
    if grad_scale != 1.0:
      gin = gin * grad_scale
    return gin, None, None, None, None


class _ReduceScatterSum(torch.autograd.Function):
  """Sum reduce-scatter along dim 0; backward is an all-gather (reference
  ``grouped_reducescatter_unscaled``, dist_model_parallel.py:291-298)."""

  @staticmethod
  def forward(ctx, x, group, grad_scale):
    world = dist.get_world_size(group)
    ctx.meta = (group, grad_scale)
    out = x.new_empty((x.shape[0] // world,) + tuple(x.shape[1:]))
    dist.reduce_scatter_tensor(out, x.contiguous(), op=dist.ReduceOp.SUM, group=group)
    return out

  @staticmethod
  def backward(ctx, grad):
    group, grad_scale = ctx.meta
    world = dist.get_world_size(group)
    gin = grad.new_empty((grad.shape[0] * world,) + tuple(grad.shape[1:]))
    dist.all_gather_into_tensor(gin, grad.contiguous(), group=group)
    if grad_scale != 1.0:
      gin = gin * grad_scale
    return gin, None, None


# ------------------------------------------------------------------------- dp -> mp index exchange
def _batch_of(x) -> int:
  return x.nrows if isinstance(x, RaggedIds) else int(x.shape[0])


def _dp_to_mp_input_dense(dp_inputs: Dict[int, torch.Tensor], rank_to_features: Dict[int, List[int]],
                          rank: int, world: int, group) -> Dict[int, torch.Tensor]:
  """One all-to-all of fixed-hotness ids (reference dist_model_parallel.py:169-221)."""
  if not dp_inputs:
    return {}
  comm_dtype = torch.int32
  for t in dp_inputs.values():
    if t.dtype == torch.int64:
      comm_dtype = torch.int64
  send, send_splits = [], []
  for r in range(world):
    parts = [dp_inputs[k].to(comm_dtype).reshape(-1) for k in rank_to_features[r]]
    send_splits.append(sum(p.numel() for p in parts))
    send += parts
  any_t = next(iter(dp_inputs.values()))
  flat = torch.cat(send) if send else any_t.new_empty(0, dtype=comm_dtype)
  mine = rank_to_features[rank]
  shapes = [tuple(dp_inputs[k].shape) for k in mine]
  per_src = sum(int(np.prod(s)) for s in shapes)
  recv = flat.new_empty(per_src * world)
  dist.all_to_all_single(recv, flat, [per_src] * world, send_splits, group=group)
  recv = recv.reshape(world, per_src)
  out, pos = {}, 0
  for k, shp in zip(mine, shapes):
    n = int(np.prod(shp))
    out[k] = recv[:, pos:pos + n].reshape((world * shp[0],) + tuple(shp[1:]))
    pos += n
  return out


def _dp_to_mp_input_ragged(dp_inputs: Dict[int, RaggedIds], rank_to_features: Dict[int, List[int]],
                           rank: int, world: int, group) -> Dict[int, RaggedIds]:
  """Two all-to-alls (values, row lengths) then worker-major -> feature-major regrouping
  (reference dist_model_parallel.py:90-166)."""
  if not dp_inputs:
    return {}
  any_r = next(iter(dp_inputs.values()))
  dev = any_r.values.device
  val_dtype = torch.int32
  for t in dp_inputs.values():
    if t.values.dtype == torch.int64:
      val_dtype = torch.int64
  local_batch = any_r.nrows
  vals, lens, val_splits, len_splits = [], [], [], []
  for r in range(world):
    n = 0
    for k in rank_to_features[r]:
      vals.append(dp_inputs[k].values.to(val_dtype))
      lens.append(dp_inputs[k].row_lengths().to(torch.int64))
      n += dp_inputs[k].values.numel()
    val_splits.append(n)
    len_splits.append(local_batch * len(rank_to_features[r]))
  mine = rank_to_features[rank]
  flat_lens = torch.cat(lens) if lens else torch.empty(0, dtype=torch.int64, device=dev)
  recv_lens = flat_lens.new_empty(local_batch * len(mine) * world)
  dist.all_to_all_single(recv_lens, flat_lens, [local_batch * len(mine)] * world, len_splits,
                         group=group)
  # how many values every source sends me
  per_src = recv_lens.reshape(world, -1).sum(dim=1)
  recv_val_splits = [int(v) for v in per_src.tolist()]
  flat_vals = torch.cat(vals) if vals else torch.empty(0, dtype=val_dtype, device=dev)
  recv_vals = flat_vals.new_empty(sum(recv_val_splits))
  dist.all_to_all_single(recv_vals, flat_vals, recv_val_splits, val_splits, group=group)
  if not mine:
    return {}
  # recv layout: [source][feature][local sample]; regroup to [feature][source][local sample]
  lens3 = recv_lens.reshape(world, len(mine), local_batch)
  starts = torch.zeros(world * len(mine) + 1, dtype=torch.int64, device=dev)
  torch.cumsum(lens3.sum(dim=2).reshape(-1), 0, out=starts[1:])
  starts = starts.tolist()
  out = {}
  for j, k in enumerate(mine):
    pieces = [recv_vals[starts[s * len(mine) + j]:starts[s * len(mine) + j + 1]]
              for s in range(world)]
    out[k] = RaggedIds.from_row_lengths(torch.cat(pieces), lens3[:, j, :].reshape(-1))
  return out


def dp_to_mp_input(dp_inputs, rank_to_features, rank: int, world: int, group=None):
  """Route data-parallel ids (local batch of every feature) to the ranks owning the features.

  Returns a dict feature -> global-batch ids for the features of this rank (ragged stays ragged).
  """
  if isinstance(dp_inputs, (list, tuple)):
    dp_inputs = dict(enumerate(dp_inputs))
  if world <= 1:
    return {k: dp_inputs[k] for k in rank_to_features[0]}
  ragged, dense = {}, {}
  for k, f in dp_inputs.items():
    if isinstance(f, RaggedIds):
      ragged[k] = f
    elif isinstance(f, SparseIds) or (isinstance(f, torch.Tensor) and f.is_sparse):
      raise ValueError("Sparse tensor data-parallel input is not supported")
    else:
      dense[k] = f
  to_dense = {r: [k for k in rank_to_features[r] if k in dense] for r in range(world)}
  to_ragged = {r: [k for k in rank_to_features[r] if k in ragged] for r in range(world)}
  out = {}
  out.update(_dp_to_mp_input_dense(dense, to_dense, rank, world, group))
  out.update(_dp_to_mp_input_ragged(ragged, to_ragged, rank, world, group))
  return {k: out[k] for k in rank_to_features[rank]}


# ------------------------------------------------------------------------- helpers
def _layer_weight(layer: nn.Module) -> nn.Parameter:
  if hasattr(layer, "embeddings") and isinstance(layer.embeddings, nn.Parameter):
    return layer.embeddings
  for p in layer.parameters():
    if p.dim() == 2:
      return p
  raise ValueError(f"cannot find the embedding matrix of {type(layer)}")


def _shift_ids(ids, offset: int):
  if offset == 0:
    return ids
  if isinstance(ids, RaggedIds):
    return RaggedIds(ids.values.to(torch.int64) + offset, ids.row_splits)
  return ids.to(torch.int64) + offset


class DistributedEmbedding(nn.Module):
  """Hybrid-parallel wrapper around a list of embedding layers.

  Args:
    embeddings: list of (unplaced) embedding layers: ``distributed_embeddings_b200.Embedding``,
      ``torch.nn.Embedding`` / ``EmbeddingBag``, config dicts, or user layers exposing
      ``get_config()`` (with ``input_dim``/``output_dim``) and ``from_config()``.
    strategy: ``basic`` | ``memory_balanced`` | ``memory_optimized`` | ``traffic_balanced``
      (balances the per-step work of the ranks using ``input_hotness``; not in the reference).
    column_slice_threshold: tables with more elements are column sliced (power-of-two count);
      None slices only when there are fewer tables than workers; ``"auto"`` picks the threshold
      that balances the per-rank gather / NVLink bytes (``suggest_column_slice_threshold``).
    row_slice_threshold: tables with at least this many elements are row sliced over all workers.
    dp_input: True -> every rank passes its local batch of *all* features; False -> every rank
      passes the *global* batch of its own features (``strategy.input_ids_list[rank]``).
    input_table_map: ``input[i]`` uses ``table[input_table_map[i]]``.
    data_parallel_threshold: tables with at most this many elements are replicated.
    gpu_embedding_size: per-rank HBM element budget; the largest table-parallel tables beyond it
      live in pinned host memory.
    input_hotness: ids per sample of every input, for ``traffic_balanced`` (keyword only).
    device / process_group / backend / compute_dtype: execution placement (keyword only).
      ``compute_dtype`` is the dtype of the returned activations (bf16 halves the bytes on the
      wire like the reference's mixed precision mode, dist_model_parallel.py:866).
    table_dtype: storage dtype of the model-parallel tables (table-parallel, column slices, row
      slices, CPU-offloaded tables): ``torch.float32`` (default), ``torch.bfloat16`` or
      ``torch.float16`` (keyword only).  Half-precision tables take half the memory; rows are
      pooled in fp32, the optimizer and its state stay fp32 and the new weights are written back
      with stochastic rounding (``ops/stochastic_rounding.py``).  Replicated tables stay fp32.
      The ``dtype`` of a passed ``Embedding`` layer or config is ignored here, as it always was.
      Checkpoints (``get_weights`` / ``save_weights``) are fp32 whatever the table dtype.
    offload_cache_size: per-rank HBM element budget (the unit of ``gpu_embedding_size``) for a
      cache of the rows of this rank's offloaded tables (keyword only; fused back end, fp32
      tables).  None (default) reads and updates offloaded rows zero-copy over PCIe on every
      access.  The budget is split over the offloaded tables in proportion to their rows; each
      also gets optimizer-state rows and a spill region (see ``parallel/offload_cache.py``).
  """

  def __init__(self,
               embeddings: Sequence[Any],
               strategy: str = "basic",
               column_slice_threshold: Optional[int] = None,
               row_slice_threshold: Optional[int] = None,
               dp_input: bool = True,
               input_table_map: Optional[Sequence[int]] = None,
               data_parallel_threshold: Optional[int] = None,
               gpu_embedding_size: Optional[int] = None,
               *,
               device=None,
               process_group=None,
               backend: str = "auto",
               compute_dtype: Optional[torch.dtype] = None,
               rank: Optional[int] = None,
               world_size: Optional[int] = None,
               input_hotness: Optional[Sequence[int]] = None,
               table_dtype: torch.dtype = torch.float32,
               offload_cache_size: Optional[int] = None):
    super().__init__()
    if offload_cache_size is not None:
      if gpu_embedding_size is None:
        raise ValueError("offload_cache_size caches offloaded tables: it needs gpu_embedding_size")
      if table_dtype != torch.float32:
        raise ValueError("offload_cache_size supports fp32 tables only (16-bit tables key their "
                         "stochastic rounding on the row, which a cache slot would change)")
      if int(offload_cache_size) < 0:
        raise ValueError("offload_cache_size must be >= 0")
    self.offload_cache_size = None if offload_cache_size is None else int(offload_cache_size)
    if self.offload_cache_size is not None:
      # module checkpoints (state_dict / load_state_dict) see the host tables: flush the cache
      # before they are read, and drop it before they are overwritten
      self.register_state_dict_pre_hook(_flush_before_state_dict)
      self._register_load_state_dict_pre_hook(_drop_before_load, with_module=True)
    if strategy not in STRATEGIES:
      raise ValueError(f"Unsupported shard strategy {strategy}")
    if table_dtype not in (torch.float32, torch.bfloat16, torch.float16):
      raise ValueError(f"table_dtype must be torch.float32, torch.bfloat16 or torch.float16, "
                       f"got {table_dtype}")
    self.table_dtype = table_dtype
    self.group = process_group
    if world_size is None:
      world_size = dist.get_world_size(process_group) if dist_ready() else 1
      rank = dist.get_rank(process_group) if dist_ready() else 0
    self.world_size, self.rank = int(world_size), int(rank or 0)
    if device is None:
      device = torch.device("cuda", torch.cuda.current_device()) if torch.cuda.is_available() \
          else torch.device("cpu")
    self.device = torch.device(device)
    self.dp_input = dp_input
    self.column_slice_threshold = column_slice_threshold
    self.gpu_embedding_size = gpu_embedding_size
    # a single worker has nothing to replicate or row slice; mp input keeps everything
    # table-parallel for backward compatibility (reference dist_model_parallel.py:764-774)
    if self.offload_cache_size is not None and self.world_size > 1:
      raise ValueError("offload_cache_size is supported on one rank (world size 1) for now")
    if self.world_size > 1:
      self.row_slice_threshold = row_slice_threshold if dp_input else None
      self.data_parallel_threshold = data_parallel_threshold if dp_input else None
    else:
      self.row_slice_threshold = None
      self.data_parallel_threshold = None
    self.compute_dtype = compute_dtype or torch.float32
    # gradients of model-parallel tables follow the global-mean-loss contract: the sum of all
    # ranks' contributions divided by the world size (what Horovod's tape does for local sources)
    self.mp_grad_scale = 1.0 / self.world_size

    configs = [config_from_layer(e) for e in embeddings]
    if column_slice_threshold == "auto":
      # balance the NVLink / gather bytes of the most loaded rank (see traffic_report)
      column_slice_threshold = suggest_column_slice_threshold(
          configs, self.world_size, strategy, input_table_map=input_table_map,
          row_slice_threshold=self.row_slice_threshold,
          data_parallel_threshold=self.data_parallel_threshold,
          gpu_embedding_size=gpu_embedding_size, hotness=input_hotness,
          input_hotness=input_hotness)
      self.column_slice_threshold = column_slice_threshold
    self.strategy = DistEmbeddingStrategy(configs,
                                          self.world_size,
                                          strategy,
                                          input_table_map=input_table_map,
                                          column_slice_threshold=column_slice_threshold,
                                          row_slice_threshold=self.row_slice_threshold,
                                          data_parallel_threshold=self.data_parallel_threshold,
                                          gpu_embedding_size=gpu_embedding_size,
                                          input_hotness=input_hotness)
    st = self.strategy
    self.num_inputs = len(st.input_table_map)

    self.dp_layers = nn.ModuleList()
    for cfg in st.dp_configs:
      self.dp_layers.append(self._create_layer(cfg, local=False))

    self.local_embedding_layers = nn.ModuleList()
    self.col_inputs_offsets: List[int] = []
    if st.table_groups[1]:
      if not all(st.local_configs[r] for r in range(self.world_size)):
        raise ValueError("Not enough table after slicing to run on all worker."
                         "Try decrease column_slice_threshold or decrease worker count")
      for cfg in st.local_configs[self.rank]:
        self.local_embedding_layers.append(self._create_layer(cfg, local=True))
      self.col_inputs_offsets = list(st.local_input_offsets[self.rank])

    self.row_layers = nn.ModuleList()
    self.row_inputs_offsets: List[int] = []
    if st.table_groups[2]:
      for cfg in st.row_sliced_configs[self.rank]:
        self.row_layers.append(self._create_layer(cfg, local=True))
      self.row_inputs_offsets = list(st.row_inputs_offsets[self.rank])

    # native layers (incl. host-resident ones, which the kernels read zero-copy) can run fused
    self._native_layers = all(
        isinstance(l, Embedding) and (l.use_custom_kernel or l.cpu_offloaded)
        for l in list(self.dp_layers) + list(self.local_embedding_layers) + list(self.row_layers))
    if backend == "auto":
      backend = "fused" if (self.device.type == "cuda" and self._native_layers) else "torch"
      if backend == "fused" and self.world_size > 1 and dist_ready():
        # multi-node jobs / GPUs without peer access: same plan, collectives through NCCL
        from .comm import CommContext  # pylint: disable=import-outside-toplevel
        if not CommContext.for_group(process_group, self.device).p2p:
          backend = "torch"
    if backend not in ("fused", "torch"):
      raise ValueError(f"Unsupported backend {backend}")
    if backend == "fused" and not self._native_layers:
      raise ValueError("the fused backend needs native Embedding layers")
    if self.offload_cache_size is not None and backend != "fused":
      raise ValueError("offload_cache_size needs the fused back end (a CUDA device and native "
                       "Embedding layers)")
    self.backend = backend
    self._engine = None
    # ids-per-sample capacity reserved for ragged inputs in the fused back end (None = inferred
    # from the first batch with 2x head room, agreed across ranks)
    self.ragged_capacity: Optional[int] = None
    self._plan_checked = False
    self._fused_optimizer: Optional[Dict[str, Any]] = None

  # ---------------------------------------------------------------------------- construction
  def _create_layer(self, config: Dict[str, Any], local: bool) -> nn.Module:
    config = dict(config)
    layer_type = config.pop("layer_type", None)
    offloaded = bool(config.pop("cpu_offload", False))
    input_dims = config.pop("input_dims", None)
    config.pop("offsets", None)
    if layer_type is None or layer_type in (nn.Embedding, nn.EmbeddingBag) or \
        (isinstance(layer_type, type) and issubclass(layer_type, Embedding)):
      native = True
      layer_type = Embedding if layer_type in (None, nn.Embedding, nn.EmbeddingBag) else layer_type
    else:
      native = False
    dev = torch.device("cpu") if offloaded else self.device
    if native:
      if input_dims is not None and len(input_dims) > 1:
        base = initializers.get(config.get("embeddings_initializer"))
        config["embeddings_initializer"] = initializers.ConcatInitializer(base, input_dims)
      if offloaded:
        config["use_custom_kernel"] = False
      if not local:
        config["sparse_grad"] = False  # replicated tables are all-reduced as dense gradients
      if local and self.table_dtype != torch.float32:
        # created in the table dtype directly: no transient fp32 copy of a large table
        layer = layer_type.from_config(config, device=dev, dtype=self.table_dtype)
      else:
        layer = layer_type.from_config(config, device=dev)
      if offloaded and torch.cuda.is_available():
        layer.embeddings.data = layer.embeddings.data.pin_memory()
    else:
      layer = layer_type.from_config(config)
      layer = layer.to(dev)
    layer.cpu_offloaded = offloaded
    if local:
      for p in layer.parameters():
        p.de_local = True  # model-parallel: never broadcast / all-reduced
    return layer

  # ---------------------------------------------------------------------------- introspection
  @property
  def weights(self) -> List[nn.Parameter]:
    """Local weights in checkpoint order: replicated, table-parallel, row-sliced."""
    return [_layer_weight(l) for l in
            list(self.dp_layers) + list(self.local_embedding_layers) + list(self.row_layers)]

  def mp_parameters(self) -> List[nn.Parameter]:
    return [p for p in self.parameters() if getattr(p, "de_local", False)]

  def dp_parameters(self) -> List[nn.Parameter]:
    return [p for p in self.parameters() if not getattr(p, "de_local", False)]

  def _check_plan_consistency(self, batch_size: Optional[int] = None):
    """Once, at the first forward: all ranks must run the same plan and the same batch size
    (the reference gathers the batch sizes in build(), dist_model_parallel.py:1170-1177)."""
    if self._plan_checked or self.world_size == 1 or not dist_ready():
      self._plan_checked = True
      return
    got: List[Optional[tuple]] = [None] * self.world_size
    dist.all_gather_object(got, (self.strategy.fingerprint(), batch_size), group=self.group)
    if len({g[0] for g in got}) != 1:
      raise RuntimeError(f"sharding plans differ across ranks: {[g[0][:12] for g in got]}")
    sizes = {g[1] for g in got}
    if len(sizes) != 1:
      raise ValueError(f"All input need to have same batchsize. got {sizes}.")
    self._plan_checked = True

  # ---------------------------------------------------------------------------- forward
  def _validate_inputs(self, inputs):
    if not isinstance(inputs, (list, tuple)):
      inputs = [inputs]
    inputs = list(inputs)
    if self.dp_input:
      if len(inputs) != self.num_inputs:
        raise ValueError(f"Expect {self.num_inputs} inputs, got {len(inputs)}.")
    else:
      expect = len(self.strategy.local_maps[self.rank])
      if len(inputs) != expect:
        raise ValueError(f"Expect {expect} inputs, got {len(inputs)}.")
    sizes = {_batch_of(x) for x in inputs}
    if len(sizes) > 1:
      raise ValueError(f"All input need to have same batchsize. got {sizes}.")
    if not self.dp_input and sizes:
      bs = next(iter(sizes))
      if bs % self.world_size > 0:
        raise ValueError(f"Global batchsize {bs} not divisible workers count {self.world_size}.")
    return inputs

  def forward(self, inputs, concat: bool = False):
    """Look up all features.

    Args:
      inputs: list of id tensors (``[batch]``, ``[batch, hotness]``) or :class:`RaggedIds`;
        data-parallel (local batch, all features) when ``dp_input`` else model-parallel (global
        batch, this rank's features in ``strategy.input_ids_list[rank]`` order).
      concat: return a single ``[local_batch, sum(widths)]`` tensor (features concatenated in
        input order) instead of a list - the zero-copy fast path of the fused back end.
    Returns:
      list of ``[local_batch, width]`` tensors in input order (or the concatenation).
    """
    inputs = self._validate_inputs(inputs)
    self._check_plan_consistency(_batch_of(inputs[0]) if inputs else None)
    if self.backend == "fused":
      from .fused import FusedEngine  # pylint: disable=import-outside-toplevel
      if self._engine is None:
        self._engine = FusedEngine(self)
      # a forward whose backward is still outstanding owns the engine's buffers: further calls
      # (two-tower models, gradient accumulation over several forwards) take the torch back end
      if self._engine.supports(inputs) and not self._engine.busy():
        return self._engine.forward(inputs, concat)
    outs = self._forward_torch(inputs)
    return torch.cat(outs, dim=1) if concat else outs

  # -- generic back end -------------------------------------------------------------------
  def _forward_torch(self, inputs):
    st = self.strategy
    dp_in = [inputs[i] for i in st.input_groups[0]] if self.dp_input else []
    dp_out = self._call_data_parallel(dp_in) if dp_in else []
    col_in = [inputs[i] for i in st.input_groups[1]] if self.dp_input else inputs
    col_out = self._call_table_parallel(col_in) if col_in else []
    row_in = [inputs[i] for i in st.input_groups[2]] if self.dp_input else []
    row_out = self._call_row_slice(row_in) if row_in else []
    outs = dp_out + col_out + row_out
    if len(outs) != len(st.rev_group_ids):
      raise RuntimeError(f"internal: {len(dp_out)}+{len(col_out)}+{len(row_out)} outputs for "
                         f"{len(st.rev_group_ids)} inputs")
    return [outs[i] for i in st.rev_group_ids]

  def _call_data_parallel(self, inputs):
    outs = [self.dp_layers[m](inp) for m, inp in zip(self.strategy.map_groups[0], inputs)]
    return [o.to(self.compute_dtype) for o in outs]

  def _lookup_local(self, layer, inp):
    dev = _layer_weight(layer).device
    out = layer(inp.to(dev))  # host-resident (offloaded) tables look up on the host
    return out.to(self.device)

  def _call_table_parallel(self, inputs):
    st = self.strategy
    if self.dp_input:
      mp = dp_to_mp_input(inputs, dict(enumerate(st.input_ids_list)), self.rank, self.world_size,
                          self.group)
      inputs = list(mp.values())
    lmap = st.local_maps[self.rank]
    if len(inputs) != len(lmap):
      raise ValueError(f"Expect {len(lmap)} inputs, got {len(inputs)}.")
    inputs = [_shift_ids(inp, off) for inp, off in zip(inputs, self.col_inputs_offsets)]
    mp_outs = [self._lookup_local(self.local_embedding_layers[m], inp)
               for m, inp in zip(lmap, inputs)]
    mp_outs = [o.to(self.compute_dtype) for o in mp_outs]
    if self.world_size > 1:
      for o in mp_outs:
        if o.dim() != 2:
          raise ValueError("table-parallel outputs must be 2-D [batch, width]; use a combiner or "
                           "1-D inputs")
      global_bs = mp_outs[0].shape[0]
      local_bs = global_bs // self.world_size
      packed = torch.cat([o.reshape(self.world_size, -1) for o in mp_outs], dim=1).reshape(-1)
      n_send = packed.numel() // self.world_size
      recv_splits = [local_bs * sum(int(c[m]["output_dim"]) for m in maps)
                     for c, maps in zip(st.local_configs, st.local_maps)]
      dp_outs = _AllToAllSingle.apply(packed, recv_splits, [n_send] * self.world_size, self.group,
                                      self.mp_grad_scale)
      sizes = [local_bs * w for w in st.widths_list_flat]
      mp_outs = [t.reshape(local_bs, -1) for t in torch.split(dp_outs, sizes)]
    result = [mp_outs[i] for i in st.rev_tp_ids]
    for start, end in st.sliced_out_ranges:
      result[start:end] = [torch.cat(result[start:end], dim=-1)]
    return result

  def _call_row_slice(self, inputs):
    # all-gather ids, shifted local lookup (foreign ids fall outside and add zero), reduce-scatter
    gathered = []
    for inp in inputs:
      if isinstance(inp, RaggedIds):
        raise ValueError("ragged inputs are not supported for row-sliced tables")
      buf = inp.new_empty((inp.shape[0] * self.world_size,) + tuple(inp.shape[1:]))
      dist.all_gather_into_tensor(buf, inp.contiguous(), group=self.group)
      gathered.append(buf)
    # offsets are per row-sliced table; several inputs may share one (input_table_map)
    maps = self.strategy.map_groups[2]
    gathered = [_shift_ids(inp, self.row_inputs_offsets[m]) for m, inp in zip(maps, gathered)]
    outs = [self._lookup_row_shard(self.row_layers[m], inp) for m, inp in zip(maps, gathered)]
    outs = [o.to(self.compute_dtype) for o in outs]
    return [_ReduceScatterSum.apply(o, self.group, self.mp_grad_scale) for o in outs]

  @staticmethod
  def _lookup_row_shard(layer, ids):
    """Look up shifted ids in a row shard: ids of other shards fall outside [0, rows) and must
    contribute zero.  The native layer does that itself; a user layer sees clamped ids and its
    rows are masked afterwards (one id per sample only - pooling inside a user layer cannot be
    masked)."""
    if isinstance(layer, Embedding):
      if layer.use_custom_kernel:
        return layer(ids)
      # library-path layers (F.embedding / embedding_bag) reject the shifted ids that fall
      # outside the shard; the masking lookup (kernel on CUDA, oracle on CPU) zero-fills them
      # like TF's gather does for the reference
      w = layer.embeddings
      ids = ids.to(w.device)
      shape = None
      if ids.dim() == 1:
        shape, ids = (ids.shape[0], w.shape[1]), ids.reshape(-1, 1)
      elif ids.dim() > 2:
        lead = tuple(ids.shape[:-1]) if layer.combiner is not None else tuple(ids.shape)
        shape, ids = lead + (w.shape[1],), ids.reshape(-1, ids.shape[-1])
      elif layer.combiner is None:
        shape = tuple(ids.shape) + (w.shape[1],)
      out = elo.embedding_lookup(w, ids, combiner=layer.combiner, sparse_grad=layer.sparse_grad)
      return out.reshape(shape) if shape is not None else out
    if ids.dim() != 1:
      raise ValueError("row-sliced user-defined layers support one id per sample only")
    rows = _layer_weight(layer).shape[0]
    valid = (ids >= 0) & (ids < rows)
    out = layer(ids.clamp(0, rows - 1))
    return out * valid.unsqueeze(-1).to(out.dtype)

  # ---------------------------------------------------------------------------- fused optimizer
  def set_optimizer(self, kind: str = "sgd", lr: float = 0.01, **kwargs):
    """Attach an optimizer that is applied to the model-parallel tables *inside* the backward
    kernels (no sparse gradient is materialised).  ``kind``: ``sgd`` | ``adagrad`` |
    ``rowwise_adagrad`` | ``adam``.  Only the fused back end consumes it.

    Keyword arguments (any other raises ``ValueError``):

    - ``eps``: added to the square root in the denominator (default 1e-7, Adam 1e-8).
    - ``beta1``, ``beta2``: Adam's moment decay rates (0.9, 0.999).
    - ``initial_accumulator_value``: start value of the Adagrad / row-wise Adagrad accumulator
      (0.1).
    - ``weight_decay``: L2 decay (default 0).  ``weight_decay * w`` is added to the summed,
      scaled gradient of a row before the optimizer sees it, once per step for every row that at
      least one id of the step touched (a row whose ids carry only zero gradients included).  The
      optimizers are lazy: rows no id touched, and their state, do not move.  Row-wise Adagrad
      accumulates the mean square of this decayed gradient.
    - ``deterministic``: SGD only (default False).  False sends SGD without weight decay through
      one atomic scatter of the gradient rows into the tables; True, or any weight decay, takes
      the sorted update, which sums each row's gradient before it applies it.
    - ``step``: Adam's step count to resume from (0).
    - ``state_dtype``: storage of the Adagrad accumulator / Adam moments, ``torch.float32``
      (default) or ``torch.bfloat16`` (half the bytes; the update runs in fp32 and stores the
      state with stochastic rounding, see the user guide, "Half-precision optimizer state")."""
    kind = kind.lower()
    if kind not in ("sgd", "adagrad", "rowwise_adagrad", "adam"):
      raise ValueError(f"Unsupported fused optimizer {kind}")
    state_dtype = check_state_dtype(kind, kwargs.pop("state_dtype", torch.float32))
    if state_dtype != torch.float32 and self.offload_cache_size is not None:
      raise ValueError("state_dtype=torch.bfloat16 is not supported with offload_cache_size: the "
                       "HBM row cache keeps optimizer state rows as fp32 words")
    cfg = {"kind": kind, "lr": float(lr), "eps": 1e-7 if kind != "adam" else 1e-8,
           "beta1": 0.9, "beta2": 0.999, "weight_decay": 0.0, "initial_accumulator_value": 0.1,
           "deterministic": kind != "sgd", "step": 0, "state_dtype": state_dtype}
    unknown = sorted(set(kwargs) - set(cfg))
    if unknown:
      raise ValueError(f"unknown fused optimizer argument(s) {unknown}; the known ones are "
                       f"{sorted(set(cfg) - {'kind', 'lr'})}")
    cfg.update(kwargs)
    self._fused_optimizer = cfg
    if self._engine is not None:
      self._engine.reset_optimizer_state()
    return self

  def set_learning_rate(self, lr: float):
    if self._fused_optimizer is None:
      raise RuntimeError("no fused optimizer attached")
    self._fused_optimizer["lr"] = float(lr)
    if self._engine is not None:
      self._engine.update_lr(float(lr))

  # ---------------------------------------------------------------------------- checkpoint surface
  def _col_table_owner_shards(self):
    """[(group table id, rank, local shard index)] for every placed piece, table order."""
    out = []
    for r, shards in enumerate(self.strategy.shards):
      for j, s in enumerate(shards):
        out.append((s.table, r, j))
    return sorted(out, key=lambda x: (x[0], x[1]))

  def _comm_device(self) -> torch.device:
    if dist_ready() and dist.get_backend(self.group) == "nccl":
      return self.device
    return torch.device("cpu")

  def _bcast_rows(self, src: Optional[torch.Tensor], rows: int, width: int, owner: int,
                  out: Optional[np.ndarray], col_start: int, chunk: int = 1 << 26):
    """Broadcast a [rows, width] shard from ``owner`` in row chunks; collectors copy it into
    ``out[:, col_start:col_start+width]``."""
    dev = self._comm_device() if getattr(self, "_bcast_hook", None) is None else \
        torch.device("cpu")
    step = max(1, chunk // max(1, width))
    for r0 in range(0, rows, step):
      r1 = min(rows, r0 + step)
      if self.rank == owner:
        buf = src[r0:r1].detach().to(dev, torch.float32).contiguous()
      else:
        buf = torch.empty(r1 - r0, width, dtype=torch.float32, device=dev)
      if self.world_size > 1:
        hook = getattr(self, "_bcast_hook", None)  # plan interpreter: ranks are threads
        if hook is not None:
          buf = hook(buf, owner, self.rank)
        else:
          dist.broadcast(buf, src=self._global_rank(owner), group=self.group)
      if out is not None:
        out[r0:r1, col_start:col_start + width] = buf.cpu().numpy()

  def _global_rank(self, group_rank: int) -> int:
    if self.group is None or not dist_ready():
      return group_rank
    return dist.get_global_rank(self.group, group_rank)

  # ---------------------------------------------------------------------------- offload cache
  def flush_offload_cache(self):
    """Write every dirty row of the offload cache, and its optimizer state, back to the host
    tables.  The checkpoint calls do this themselves."""
    if self._engine is not None:
      self._engine.flush_offload_cache()

  def _drop_offload_cache(self):
    """Flush and empty the cache: the host tables are about to be overwritten."""
    if self._engine is not None:
      self._engine.flush_offload_cache(invalidate=True)

  def offload_cache_stats(self, reset: bool = True) -> List[Dict[str, int]]:
    """Per cached table of this rank: ``{"table", "local_table", "hits", "misses", "spills",
    "writebacks"}``, counted on the device in unique rows per step (a row a step looks up many
    times counts once) since the last reset.  ``table`` is the global table index; ``misses``
    include ``spills``.  Reading them synchronises the device."""
    if self._engine is None:
      return []
    st = self.strategy
    out = []
    for m, v in sorted(self._engine.offload_cache_stats(reset).items()):
      shard = next(s for s in st.shards[self.rank] if s.local_table == m)
      out.append({"table": st.table_groups[1][shard.table], "local_table": m, **v})
    return out

  def get_weights(self, all_ranks: bool = False, chunk: int = 1 << 26) -> List[np.ndarray]:
    """Return the *global, unsharded* tables as numpy arrays in original table order.

    The layout is independent of the sharding: a checkpoint written with 8 column-sliced ranks
    loads on one GPU.  Only rank 0 receives the arrays unless ``all_ranks`` (other ranks get an
    empty list for the model-parallel tables they do not own).  Shards are read (and cast to
    fp32) in pieces of at most ``chunk`` elements.
    """
    self.flush_offload_cache()
    weights = self.weights
    n_dp, n_col = len(self.dp_layers), len(self.local_embedding_layers)
    return self._gather_global(weights[:n_dp], weights[n_dp:n_dp + n_col],
                               weights[n_dp + n_col:], all_ranks, chunk=chunk)

  def _gather_global(self, dp_tensors, col_tensors, row_tensors, all_ranks: bool,
                     per_row: bool = False, chunk: int = 1 << 26) -> List[Optional[np.ndarray]]:
    """Assemble global per-table arrays from this rank's local tensors (one per replicated
    layer / fused local table / row shard; ``None`` entries of ``dp_tensors`` are skipped).
    ``per_row``: the local tensors hold one value per row (row-wise optimizer state); the column
    slices of a table then contribute their width-weighted mean."""
    st = self.strategy
    collect = all_ranks or self.rank == 0
    n_tables = len(st.global_configs)
    result: List[Optional[np.ndarray]] = [None] * n_tables
    for t, w in zip(st.table_groups[0], dp_tensors):
      result[t] = None if w is None else w.detach().float().cpu().numpy()
    for gt, t in enumerate(st.table_groups[1]):
      cfg = st.global_configs[t]
      rows, width = int(cfg["input_dim"]), int(cfg["output_dim"])
      if per_row:
        out = np.zeros((rows, 1), dtype=np.float32) if collect else None
      else:
        out = np.empty((rows, width), dtype=np.float32) if collect else None
      for r, shards in enumerate(st.shards):
        for s in shards:
          if s.table != gt:
            continue
          src = None
          if r == self.rank:
            src = col_tensors[s.local_table][s.row_offset:s.row_offset + s.rows]
          if per_row:
            if src is not None:
              src = src.reshape(-1, 1)
            part = np.empty((s.rows, 1), dtype=np.float32) if collect else None
            self._bcast_rows(src, s.rows, 1, r, part, 0, chunk)
            if out is not None:
              out += part * (s.width / width)
          else:
            self._bcast_rows(src, s.rows, s.width, r, out, s.col_start, chunk)
      result[t] = out
    for gt, t in enumerate(st.table_groups[2]):
      cfg = st.global_configs[t]
      rows, width = int(cfg["input_dim"]), int(cfg["output_dim"])
      w_out = 1 if per_row else width
      out = np.empty((rows, w_out), dtype=np.float32) if collect else None
      for r, (lo, hi) in enumerate(st.row_ranges[gt]):
        src = row_tensors[gt] if r == self.rank else None
        if src is not None and per_row:
          src = src.reshape(-1, 1)
        sub = out[lo:hi] if out is not None else None
        self._bcast_rows(src, hi - lo, w_out, r, sub, 0, chunk)
      result[t] = out
    if not collect:
      return []
    return result

  @staticmethod
  def _assign_chunked(param: torch.Tensor, row0: int, arr, chunk: int):
    """Copy ``arr`` ([rows, width], numpy or mmap) into ``param[row0:row0+rows]`` in chunks so a
    device table never needs a second full-size staging copy."""
    rows, width = arr.shape
    step = max(1, chunk // max(1, width))
    with torch.no_grad():
      for r0 in range(0, rows, step):
        r1 = min(rows, r0 + step)
        host = np.ascontiguousarray(arr[r0:r1], dtype=np.float32)
        if not host.flags.writeable:  # read-only memory map: torch wants a writable buffer
          host = host.copy()
        block = torch.from_numpy(host)
        param[row0 + r0:row0 + r1].copy_(block.to(param.device, non_blocking=False))

  def set_weights(self, weights: Sequence[Union[np.ndarray, str, torch.Tensor]],
                  chunk: int = 134217728, use_lock: bool = False):
    """Set all tables from global arrays (or ``.npy`` paths, memory-mapped).

    Args:
      weights: one ``[rows, width]`` array / path per table, original table order.
      chunk: max elements per host->device copy.
      use_lock: load rank by rank in lock step (bounds host memory on shared nodes).
    """
    st = self.strategy
    self._drop_offload_cache()
    if len(weights) != len(st.global_configs):
      raise ValueError(
          f"You called `set_weights(weights)` on layer DistributedEmbedding with a weight list of "
          f"length {len(weights)}, but the layer was expecting {len(st.global_configs)} weights.")
    if use_lock and self.world_size > 1:
      for _ in range(self.rank):
        dist.barrier(group=self.group)

    def load(w):
      if isinstance(w, str):
        return np.load(w, mmap_mode="r")
      if isinstance(w, torch.Tensor):
        return w.detach().cpu().numpy()
      return w

    params = self.weights
    n_dp, n_col = len(self.dp_layers), len(self.local_embedding_layers)
    for t, p in zip(st.table_groups[0], params[:n_dp]):
      arr = load(weights[t])
      self._check_shape(arr, st.global_configs[t], t)
      self._assign_chunked(p.data, 0, arr, chunk)
    col_params = params[n_dp:n_dp + n_col]
    for s in st.shards[self.rank] if st.table_groups[1] else []:
      t = st.table_groups[1][s.table]
      arr = load(weights[t])
      self._check_shape(arr, st.global_configs[t], t)
      self._assign_chunked(col_params[s.local_table].data, s.row_offset,
                           arr[:, s.col_start:s.col_end], chunk)
    row_params = params[n_dp + n_col:]
    for gt, t in enumerate(st.table_groups[2]):
      arr = load(weights[t])
      self._check_shape(arr, st.global_configs[t], t)
      lo, hi = st.row_ranges[gt][self.rank]
      self._assign_chunked(row_params[gt].data, 0, arr[lo:hi], chunk)
    if use_lock and self.world_size > 1:
      for _ in range(self.world_size - self.rank):
        dist.barrier(group=self.group)

  # -- file checkpoints: every rank writes / reads its own slices, no gather -----------------
  def _barrier(self):
    if self.world_size > 1:
      hook = getattr(self, "_barrier_hook", None)  # plan interpreter: ranks are threads
      if hook is not None:
        hook()
      else:
        dist.barrier(group=self.group)

  @staticmethod
  def _write_chunked(mm, row0: int, col0: int, src: torch.Tensor, chunk: int):
    """``mm[row0:row0+rows, col0:col0+width] = src`` in row chunks (one device->host copy of at
    most ``chunk`` elements at a time)."""
    rows, width = int(src.shape[0]), int(src.shape[1])
    step = max(1, chunk // max(1, width))
    for r0 in range(0, rows, step):
      r1 = min(rows, r0 + step)
      mm[row0 + r0:row0 + r1, col0:col0 + width] = \
          src[r0:r1].detach().to(torch.float32).cpu().numpy()

  def save_weights(self, directory: str, chunk: int = 134217728, prefix: str = "table") -> List[str]:
    """Write the tables as ``<directory>/<prefix>_<t>.npy`` in the same *global* layout
    :meth:`get_weights` returns (``[rows, width]`` fp32 per table, original order), without
    gathering them anywhere: rank 0 creates the files, then **every rank writes its own column /
    row slices straight into the memory-mapped files in parallel**.  ``directory`` must be
    visible to all ranks (one host, or a shared file system).  For the 774 GiB synthetic model
    that is 1/W of the bytes per rank and no data collective (two barriers), where :meth:`get_weights`
    funnels every shard through a broadcast.  The files load with :meth:`load_weights` /
    :meth:`set_weights` under any sharding.  Collective: every rank must call it; returns the
    paths."""
    st = self.strategy
    n_tables = len(st.global_configs)
    paths = [os.path.join(directory, f"{prefix}_{t}.npy") for t in range(n_tables)]
    self.flush_offload_cache()
    if self.rank == 0:
      os.makedirs(directory, exist_ok=True)
      for t, path in enumerate(paths):
        cfg = st.global_configs[t]
        mm = np.lib.format.open_memmap(path, mode="w+", dtype=np.float32,
                                       shape=(int(cfg["input_dim"]), int(cfg["output_dim"])))
        del mm
    self._barrier()  # the files exist with their final size
    weights = self.weights
    n_dp, n_col = len(self.dp_layers), len(self.local_embedding_layers)
    if self.rank == 0:  # replicated tables: identical everywhere
      for t, w in zip(st.table_groups[0], weights[:n_dp]):
        mm = np.load(paths[t], mmap_mode="r+")
        self._write_chunked(mm, 0, 0, w, chunk)
        mm.flush()
    col = weights[n_dp:n_dp + n_col]
    for s in st.shards[self.rank] if st.table_groups[1] else []:
      t = st.table_groups[1][s.table]
      mm = np.load(paths[t], mmap_mode="r+")
      self._write_chunked(mm, 0, s.col_start, col[s.local_table][s.row_offset:s.row_offset + s.rows],
                          chunk)
      mm.flush()
    row = weights[n_dp + n_col:]
    for gt, t in enumerate(st.table_groups[2]):
      lo, _ = st.row_ranges[gt][self.rank]
      mm = np.load(paths[t], mmap_mode="r+")
      self._write_chunked(mm, lo, 0, row[gt], chunk)
      mm.flush()
    self._barrier()  # every slice is on disk
    return paths

  def load_weights(self, directory: str, chunk: int = 134217728, use_lock: bool = False,
                   prefix: str = "table"):
    """Load a checkpoint written by :meth:`save_weights` (any world size / sharding): every rank
    memory-maps the files and copies only its own slices."""
    n_tables = len(self.strategy.global_configs)
    paths = [os.path.join(directory, f"{prefix}_{t}.npy") for t in range(n_tables)]
    missing = [p for p in paths if not os.path.exists(p)]
    if missing:
      raise FileNotFoundError(f"checkpoint is incomplete, missing {missing[:3]}")
    self.set_weights(paths, chunk=chunk, use_lock=use_lock)

  @staticmethod
  def _check_shape(arr, cfg, t):
    want = (int(cfg["input_dim"]), int(cfg["output_dim"]))
    if tuple(arr.shape) != want:
      raise ValueError(f"weight {t} has shape {tuple(arr.shape)}, expected {want}")

  # optimizer-state extension of the checkpoint surface (the reference does not cover it)
  def get_optimizer_state(self, all_ranks: bool = False) -> Dict[str, Any]:
    """State of the fused optimizer in the same *global, sharding independent* layout as
    :meth:`get_weights`: ``{"kind", "step", "tables": [per table: None | [slot arrays]]}`` with
    one ``[rows, width]`` array per state slot (Adagrad accumulator; Adam m, v) or ``[rows, 1]``
    for row-wise Adagrad (column slices of a table contribute the width-weighted mean of their
    accumulators).  A state written by 8 column-sliced ranks loads on 4, or on one GPU.
    Replicated tables are trained by the dense optimizer and have no entry (None).  Collective:
    every rank must call it; only rank 0 receives the arrays unless ``all_ranks``."""
    opt = self._fused_optimizer
    eng = self._engine
    self.flush_offload_cache()
    if opt is None or eng is None or not eng.opt_state:
      return {"kind": opt["kind"] if opt else None, "step": eng.step_count() if eng else 0,
              "tables": None}
    kind = opt["kind"]
    n_col = len(self.local_embedding_layers)
    n_slots = len(next(iter(eng.opt_state.values())))
    per_row = kind == "rowwise_adagrad"
    slots = []
    for k in range(n_slots):
      col = [eng.opt_state[m][k] for m in range(n_col)]
      row = [eng.opt_state[n_col + j][k] for j in range(len(self.row_layers))]
      slots.append(self._gather_global([None] * len(self.dp_layers), col, row, all_ranks,
                                       per_row=per_row))
    tables = None
    if slots and slots[0]:
      tables = [None if slots[0][t] is None else [sl[t] for sl in slots]
                for t in range(len(self.strategy.global_configs))]
    return {"kind": kind, "step": eng.step_count(), "tables": tables}

  def set_optimizer_state(self, state: Dict[str, Any], chunk: int = 134217728):
    """Load a state produced by :meth:`get_optimizer_state` (any sharding) - every rank passes
    the same global arrays and keeps its slices, like :meth:`set_weights`.  The older per-rank
    format of ``FusedEngine.optimizer_state_dict`` is still accepted.  Element-wise state is
    copied in pieces of at most ``chunk`` elements and converted to the state's storage dtype
    (bf16 state: round to nearest)."""
    if self._engine is None:
      raise RuntimeError("run a forward pass (or build the engine) before loading optimizer state")
    eng = self._engine
    self._drop_offload_cache()
    if "tables" not in state:
      eng.load_optimizer_state_dict(state)
      return
    if self._fused_optimizer is None or state.get("kind") != self._fused_optimizer["kind"]:
      raise ValueError(f"optimizer state of kind {state.get('kind')} does not match the attached "
                       f"optimizer {self._fused_optimizer and self._fused_optimizer['kind']}")
    if not eng.opt_state:
      eng.reset_optimizer_state()
    tables = state.get("tables")
    if tables is not None:
      st = self.strategy
      per_row = state["kind"] == "rowwise_adagrad"
      n_col = len(self.local_embedding_layers)
      with torch.no_grad():
        for s in st.shards[self.rank] if st.table_groups[1] else []:
          t = st.table_groups[1][s.table]
          for k, arr in enumerate(tables[t]):
            dst = eng.opt_state[s.local_table][k]
            if per_row:
              dst[s.row_offset:s.row_offset + s.rows].copy_(
                  torch.from_numpy(np.array(np.asarray(arr)[:, 0], dtype=np.float32)))
            else:
              self._assign_chunked(dst, s.row_offset, np.asarray(arr)[:, s.col_start:s.col_end],
                                   chunk)
        for gt, t in enumerate(st.table_groups[2]):
          lo, hi = st.row_ranges[gt][self.rank]
          for k, arr in enumerate(tables[t]):
            dst = eng.opt_state[n_col + gt][k]
            if per_row:
              dst.copy_(torch.from_numpy(np.array(np.asarray(arr)[lo:hi, 0], dtype=np.float32)))
            else:
              self._assign_chunked(dst, 0, np.asarray(arr)[lo:hi], chunk)
    step = int(state.get("step", 0))
    eng.step_t.fill_(float(step))
    self._fused_optimizer["step"] = step
    eng._tables_dirty = True

  def save_optimizer_state(self, directory: str, chunk: int = 134217728) -> Optional[str]:
    """File counterpart of :meth:`get_optimizer_state`: ``optimizer.json`` (kind, step, slots)
    plus one ``opt_<t>_slot<k>.npy`` per table and state slot in the global layout.  Adagrad /
    Adam state is element-wise, so every rank writes its own slices in parallel like
    :meth:`save_weights`; row-wise Adagrad needs the width-weighted mean over a table's column
    slices and goes through the gather of :meth:`get_optimizer_state` (rank 0 writes).
    Collective; returns the path of ``optimizer.json`` (None when there is no state)."""
    import json  # pylint: disable=import-outside-toplevel
    opt, eng = self._fused_optimizer, self._engine
    self.flush_offload_cache()
    if opt is None or eng is None or not eng.opt_state:
      return None
    st = self.strategy
    kind = opt["kind"]
    n_slots = len(next(iter(eng.opt_state.values())))
    n_tables = len(st.global_configs)
    meta_path = os.path.join(directory, "optimizer.json")
    has_state = [t not in st.table_groups[0] for t in range(n_tables)]

    def path(t, k):
      return os.path.join(directory, f"opt_{t}_slot{k}.npy")

    if kind == "rowwise_adagrad":
      state = self.get_optimizer_state()
      if self.rank == 0:
        os.makedirs(directory, exist_ok=True)
        for t in range(n_tables):
          if has_state[t]:
            for k, arr in enumerate(state["tables"][t]):
              np.save(path(t, k), arr)
    else:
      if self.rank == 0:
        os.makedirs(directory, exist_ok=True)
        for t in range(n_tables):
          if has_state[t]:
            cfg = st.global_configs[t]
            for k in range(n_slots):
              mm = np.lib.format.open_memmap(
                  path(t, k), mode="w+", dtype=np.float32,
                  shape=(int(cfg["input_dim"]), int(cfg["output_dim"])))
              del mm
      self._barrier()
      n_col = len(self.local_embedding_layers)
      for s in st.shards[self.rank] if st.table_groups[1] else []:
        t = st.table_groups[1][s.table]
        for k in range(n_slots):
          mm = np.load(path(t, k), mmap_mode="r+")
          self._write_chunked(mm, 0, s.col_start,
                              eng.opt_state[s.local_table][k][s.row_offset:s.row_offset + s.rows],
                              chunk)
          mm.flush()
      for gt, t in enumerate(st.table_groups[2]):
        lo, _ = st.row_ranges[gt][self.rank]
        for k in range(n_slots):
          mm = np.load(path(t, k), mmap_mode="r+")
          self._write_chunked(mm, lo, 0, eng.opt_state[n_col + gt][k], chunk)
          mm.flush()
    step = eng.step_count()
    if self.rank == 0:
      with open(meta_path, "w", encoding="utf-8") as f:
        json.dump({"kind": kind, "step": step, "slots": n_slots,
                   "tables": [bool(x) for x in has_state]}, f)
    self._barrier()
    return meta_path

  def load_optimizer_state(self, directory: str, chunk: int = 134217728):
    """Load what :meth:`save_optimizer_state` wrote (any world size / sharding); the arrays stay
    memory mapped, every rank reads only its slices, ``chunk`` elements at a time."""
    import json  # pylint: disable=import-outside-toplevel
    with open(os.path.join(directory, "optimizer.json"), encoding="utf-8") as f:
      meta = json.load(f)
    tables = []
    for t, has in enumerate(meta["tables"]):
      tables.append([np.load(os.path.join(directory, f"opt_{t}_slot{k}.npy"), mmap_mode="r")
                     for k in range(int(meta["slots"]))] if has else None)
    self.set_optimizer_state({"kind": meta["kind"], "step": int(meta["step"]), "tables": tables},
                             chunk=chunk)

  def close(self):
    """Release the fused engine's peer-mapped buffers (collective over the process group).
    Call it before dropping a ``DistributedEmbedding`` in a job that keeps running and builds
    another one; the layer stays usable - buffers are re-created at the next forward."""
    if self._engine is not None:
      self._engine.close()

  def extra_repr(self):
    return (f"world_size={self.world_size}, rank={self.rank}, strategy={self.strategy.strategy}, "
            f"backend={self.backend}, dp_input={self.dp_input}")


def _flush_before_state_dict(module, prefix, keep_vars):  # pylint: disable=unused-argument
  module.flush_offload_cache()


def _drop_before_load(module, *args, **kwargs):  # pylint: disable=unused-argument
  module._drop_offload_cache()  # pylint: disable=protected-access


# ------------------------------------------------------------------------- hybrid-parallel glue
def _is_mp(p) -> bool:
  return bool(getattr(p, "de_local", False))


def broadcast_variables(model_vars, root_rank: int = 0, group=None):
  """Broadcast data-parallel variables from ``root_rank``; model-parallel (``de_local``)
  variables are left alone (reference dist_model_parallel.py:1219-1239)."""
  if isinstance(model_vars, nn.Module):
    model_vars = list(model_vars.parameters()) + list(model_vars.buffers())
  if not dist_ready() or dist.get_world_size(group) == 1:
    return
  src = root_rank if group is None else dist.get_global_rank(group, root_rank)
  for v in model_vars:
    if _is_mp(v):
      continue
    dist.broadcast(v.data if isinstance(v, nn.Parameter) else v, src=src, group=group)
