"""Single-device embedding layers.

Capability parity: ``distributed_embeddings/python/layers/embedding.py`` of the reference
(``Embedding`` :50-170, ``ConcatOneHotEmbedding`` :173-198, ``IntegerLookup`` :202-281).
"""
from __future__ import annotations

from typing import Any, Dict, List, Optional, Sequence

import numpy as np
import torch
from torch import nn

from ..ops import embedding_lookup_ops as elo
from ..ops.ragged import RaggedIds, SparseIds
from ..utils import initializers


def _embedding_lookup_native(param, ids, combiner=None):
  """Library (non-custom-kernel) path, used for host-resident tables.  bf16 / fp16 tables pool
  the gathered rows in fp32 (no fp32 copy of the table) and return the table dtype, like the
  kernels."""
  if param.dtype in (torch.bfloat16, torch.float16) and combiner is not None:
    if isinstance(ids, RaggedIds):
      splits = ids.row_splits.to(torch.int64)
      counts = splits[1:] - splits[:-1]
      values = ids.values.to(torch.int64)
    else:
      values = ids.to(torch.int64).reshape(-1)
      counts = torch.full((ids.shape[0],), ids.shape[1], dtype=torch.int64, device=ids.device)
    rows = nn.functional.embedding(values, param).float()
    sample = torch.repeat_interleave(torch.arange(counts.numel(), device=rows.device),
                                     counts.to(rows.device))
    out = torch.zeros(counts.numel(), param.shape[1], dtype=torch.float32, device=rows.device)
    out = out.index_add(0, sample, rows)
    if combiner == "mean":
      out = out / counts.clamp(min=1).to(out).unsqueeze(1)
    return out.to(param.dtype)
  if isinstance(ids, RaggedIds):
    mode = "sum" if combiner == "sum" else "mean"
    return nn.functional.embedding_bag(ids.values.to(torch.int64),
                                       param,
                                       offsets=ids.row_splits.to(torch.int64),
                                       mode=mode,
                                       include_last_offset=True)
  t = nn.functional.embedding(ids.to(torch.int64), param)
  if combiner == "sum":
    t = t.sum(dim=1)
  elif combiner == "mean":
    t = t.mean(dim=1)
  return t


class Embedding(nn.Module):
  """Turns indices into vectors of fixed size, optionally pooling the last input dimension.

  Args:
    input_dim: size of the vocabulary (max index + 1).
    output_dim: embedding width.
    embeddings_initializer: Keras-style identifier, :class:`Initializer` or callable.
    combiner: ``None`` | ``'sum'`` | ``'mean'``.
    use_custom_kernel: run the sm_90a kernels (True) or the library path (False).
    sparse_grad: parameter gradient as a deduplicated sparse tensor (reference semantics).

  With a combiner the supported inputs / outputs are: N-D tensor ``(d1..dn)`` ->
  ``(d1..dn-1, output_dim)`` (N >= 2); 2-D :class:`RaggedIds` / :class:`SparseIds` ->
  ``(batch, output_dim)``.  Without one the output is ``shape(ids) + (output_dim,)``.
  """

  def __init__(self,
               input_dim: int,
               output_dim: int,
               embeddings_initializer="uniform",
               embeddings_regularizer=None,
               activity_regularizer=None,
               embeddings_constraint=None,
               combiner: Optional[str] = None,
               use_custom_kernel: bool = True,
               sparse_grad: bool = True,
               device=None,
               dtype=torch.float32,
               name: Optional[str] = None,
               **kwargs):
    super().__init__()
    kwargs.pop("input_shape", None)
    kwargs.pop("input_length", None)
    kwargs.pop("mask_zero", None)
    kwargs.pop("trainable", None)
    kwargs.pop("autocast", None)
    if kwargs:
      raise TypeError(f"Unexpected arguments {sorted(kwargs)}")
    if input_dim <= 0 or output_dim <= 0:
      raise ValueError(
          f"Both input_dim and output_dim should be positive, found {input_dim} and {output_dim}")
    if combiner not in (None, "sum", "mean"):
      raise ValueError(f"Unsupported combiner {combiner}")
    self.input_dim = int(input_dim)
    self.output_dim = int(output_dim)
    self.embeddings_initializer = initializers.get(embeddings_initializer)
    self.embeddings_regularizer = embeddings_regularizer
    self.activity_regularizer = activity_regularizer
    self.embeddings_constraint = embeddings_constraint
    self.combiner = combiner
    self.use_custom_kernel = use_custom_kernel
    self.sparse_grad = sparse_grad
    self.layer_name = name
    self.cpu_offloaded = False
    # no autocast: tables stay in their storage dtype, fp32 by default (reference
    # embedding.py:92,111); bf16 / fp16 tables are pooled in fp32
    self.embeddings = nn.Parameter(torch.empty(self.input_dim, self.output_dim, dtype=dtype,
                                               device=device),
                                   requires_grad=True)
    with torch.no_grad():
      self.embeddings_initializer.fill_(self.embeddings.data)

  def compute_output_shape(self, input_shape):
    input_shape = tuple(input_shape)
    if self.combiner is None:
      return input_shape + (self.output_dim,)
    return input_shape[:-1] + (self.output_dim,)

  def forward(self, inputs):
    out_shape = None
    if isinstance(inputs, torch.Tensor) and inputs.is_sparse:
      inputs = SparseIds.from_torch_sparse(inputs)
    if isinstance(inputs, (RaggedIds, SparseIds)):
      if self.combiner is None:
        raise ValueError("ragged / sparse input needs a combiner")
      if inputs.values.dtype not in (torch.int32, torch.int64):
        inputs.values = inputs.values.to(torch.int32)
    else:
      if not isinstance(inputs, torch.Tensor):
        inputs = torch.as_tensor(inputs, device=self.embeddings.device)
      if inputs.dtype not in (torch.int32, torch.int64):
        inputs = inputs.to(torch.int32)
      if inputs.dim() != 2:
        out_shape = self.compute_output_shape(inputs.shape)
      if inputs.dim() == 1:
        if self.combiner is not None:
          raise ValueError("1D input with combiner is ambiguous. Please create batch dimension.")
        inputs = inputs.reshape(-1, 1)
      elif inputs.dim() > 2:
        inputs = inputs.reshape(-1, inputs.shape[-1])
      elif inputs.dim() == 0:
        raise ValueError("scalar input is not supported")

    if self.use_custom_kernel:
      out = elo.embedding_lookup(self.embeddings, inputs, combiner=self.combiner,
                                 sparse_grad=self.sparse_grad)
    else:
      if isinstance(inputs, SparseIds):
        splits = elo.row_to_split(inputs.indices, inputs.dense_shape[0])
        inputs = RaggedIds(inputs.values, splits)
      out = _embedding_lookup_native(self.embeddings, inputs, combiner=self.combiner)
    if out_shape is not None:
      out = out.reshape(out_shape)
    return out

  def regularization_loss(self) -> torch.Tensor:
    """``embeddings_regularizer(embeddings)`` (a callable returning a scalar), 0 if unset.  Keras
    adds this term to the loss automatically; in PyTorch the training loop adds it."""
    if self.embeddings_regularizer is None:
      return self.embeddings.new_zeros(())
    return self.embeddings_regularizer(self.embeddings)

  @torch.no_grad()
  def apply_constraint(self):
    """Project the table with ``embeddings_constraint`` (callable tensor -> tensor) in place; call
    after the optimizer step (Keras applies constraints inside the optimizer)."""
    if self.embeddings_constraint is not None:
      self.embeddings.copy_(self.embeddings_constraint(self.embeddings))

  def get_config(self) -> Dict[str, Any]:
    return {
        "input_dim": self.input_dim,
        "output_dim": self.output_dim,
        "embeddings_initializer": self.embeddings_initializer,
        "embeddings_regularizer": self.embeddings_regularizer,
        "activity_regularizer": self.activity_regularizer,
        "embeddings_constraint": self.embeddings_constraint,
        "combiner": self.combiner,
        "use_custom_kernel": self.use_custom_kernel,
        "sparse_grad": self.sparse_grad,
        "name": self.layer_name,
    }

  @classmethod
  def from_config(cls, config: Dict[str, Any], device=None, dtype=None):
    """Create a layer from a config; stock-embedding configs are accepted
    (``mask_zero`` / ``input_length`` are dropped, reference embedding.py:163-170).  A ``dtype``
    inside the config is dropped as well; the ``dtype`` argument sets the table's storage
    (default fp32)."""
    config = dict(config)
    for k in ("mask_zero", "input_length", "layer_type", "cpu_offload", "input_dims", "offsets",
              "batch_input_shape", "dtype", "trainable", "sparse", "padding_idx", "max_norm",
              "norm_type", "scale_grad_by_freq"):
      config.pop(k, None)
    if dtype is not None:
      config["dtype"] = dtype
    return cls(device=device, **config)

  def extra_repr(self):
    return (f"{self.input_dim}, {self.output_dim}, combiner={self.combiner}, "
            f"custom_kernel={self.use_custom_kernel}")


def config_from_layer(layer) -> Dict[str, Any]:
  """Normalise any supported embedding layer into a planner config dict."""
  if isinstance(layer, dict):
    return dict(layer)
  if hasattr(layer, "get_config"):
    cfg = dict(layer.get_config())
    cfg.setdefault("layer_type", type(layer))
    return cfg
  if isinstance(layer, nn.EmbeddingBag):
    if layer.mode not in ("sum", "mean"):
      raise ValueError(f"EmbeddingBag mode {layer.mode} is not supported")
    return {"input_dim": layer.num_embeddings, "output_dim": layer.embedding_dim,
            "combiner": layer.mode, "layer_type": Embedding,
            "embeddings_initializer": initializers.RandomNormal(0.0, 1.0)}
  if isinstance(layer, nn.Embedding):
    return {"input_dim": layer.num_embeddings, "output_dim": layer.embedding_dim,
            "combiner": None, "layer_type": Embedding,
            "embeddings_initializer": initializers.RandomNormal(0.0, 1.0)}
  raise TypeError(f"Cannot derive an embedding config from {type(layer)}")


class ConcatOneHotEmbedding(nn.Module):
  """One fused table for many one-hot features: ``ids + offsets`` then a single gather.

  Args:
    feature_sizes: vocabulary size of every feature.
    embedding_width: embedding width shared by all features.
  """

  def __init__(self, feature_sizes: Sequence[int], embedding_width: int, device=None,
               embeddings_initializer="uniform"):
    super().__init__()
    self.embedding_width = int(embedding_width)
    offsets = np.concatenate([[0], np.cumsum(np.asarray(feature_sizes, dtype=np.int64))])
    self.register_buffer("offsets", torch.as_tensor(offsets[:-1], dtype=torch.int64, device=device),
                         persistent=False)
    self.num_features = len(feature_sizes)
    self.params = nn.Parameter(torch.empty(int(offsets[-1]), self.embedding_width, device=device))
    with torch.no_grad():
      initializers.get(embeddings_initializer).fill_(self.params.data)

  def forward(self, inputs: torch.Tensor) -> torch.Tensor:
    assert inputs.shape[1] == self.num_features
    ids = inputs.to(torch.int64) + self.offsets
    b, n = ids.shape
    out = elo.embedding_lookup(self.params, ids.reshape(b * n, 1), combiner="sum")
    return out.reshape(b, n, self.embedding_width)


class IntegerLookup(nn.Module):
  """Maps integer features to a contiguous range, building the vocabulary on the fly.

  Keys get indices ``1..max_tokens`` in first-come order; once the vocabulary is full unseen keys
  map to 0 (out of vocabulary).  On the GPU the state is an open-addressed hash table in device
  memory (``table`` with interleaved key/value slots at load factor 2/3, ``count`` with per-index
  frequencies, ``next_index``); all three are buffers and checkpoint with the module.
  The key ``-1`` is the empty-slot marker of the table (as in the reference, whose vocabulary
  starts with ``-1``): it is never inserted and always maps to 0.

  Args:
    max_tokens: vocabulary size (excluding the OOV index 0).
    use_gpu: use the CUDA hash table when the module lives on a GPU; otherwise a host dictionary.
  """

  def __init__(self, max_tokens: int, use_gpu: bool = True, device=None):
    super().__init__()
    max_tokens = int(max_tokens)
    self.max_tokens = max_tokens
    self.capacity = max_tokens + 1
    self.use_gpu = use_gpu
    n_slots = int(1.5 * self.capacity)
    count = torch.zeros(self.capacity, dtype=torch.int32, device=device)
    count[0] = 1  # index 0 is reserved for OOV (reference embedding.py:217-220)
    self.register_buffer("count", count)
    self.register_buffer("table", torch.full((2 * n_slots,), -1, dtype=torch.int64, device=device))
    self.register_buffer("next_index", torch.ones(1, dtype=torch.int64, device=device))
    self._host_vocab: Dict[int, int] = {}

  def _on_gpu(self) -> bool:
    return self.use_gpu and self.table.is_cuda

  def forward(self, inputs: torch.Tensor) -> torch.Tensor:
    if self._on_gpu():
      keys = inputs.to(device=self.table.device, dtype=torch.int64)
      return elo.integer_lookup(self.table, self.count, self.next_index, keys, self.capacity)
    # host path: dictionary with first-occurrence ordering (efficient for power-law data)
    flat = inputs.reshape(-1).to("cpu", torch.int64)
    uniq, inverse = torch.unique(flat, return_inverse=True)
    first = torch.full((uniq.numel(),), flat.numel(), dtype=torch.int64)
    first.scatter_reduce_(0, inverse, torch.arange(flat.numel()), reduce="amin")
    order = torch.argsort(first)
    vals = torch.zeros(uniq.numel(), dtype=torch.int64)
    vocab = self._host_vocab
    for j in order.tolist():
      k = int(uniq[j])
      v = vocab.get(k)
      if v is None and k != -1 and len(vocab) < self.max_tokens:
        v = len(vocab) + 1
        vocab[k] = v
      vals[j] = v or 0
    out = vals[inverse]
    self.count.index_add_(0, out.to(self.count.device),
                          torch.ones_like(out, dtype=torch.int32).to(self.count.device))
    return out.reshape(inputs.shape).to(inputs.device)

  def get_vocabulary(self) -> List[int]:
    """Keys ordered by their assigned index, prefixed with the OOV token -1."""
    if self._on_gpu():
      kv = self.table.view(-1, 2)
      used = kv[(kv[:, 0] != -1) & (kv[:, 1] > 0)]
      order = torch.argsort(used[:, 1])
      return [-1] + used[order, 0].tolist()
    items = sorted(self._host_vocab.items(), key=lambda kv: kv[1])
    return [-1] + [k for k, _ in items]

  def vocabulary_size(self) -> int:
    if self._on_gpu():
      return int(min(int(self.next_index.item()), self.capacity)) - 1
    return len(self._host_vocab)

  def get_extra_state(self):
    return {"host_vocab": dict(self._host_vocab)}

  def set_extra_state(self, state):
    self._host_vocab = dict(state.get("host_vocab", {}))
