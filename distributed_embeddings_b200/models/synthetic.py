"""Synthetic benchmark models and the power-law input generator.

Capability parity: examples/benchmarks/synthetic_models/synthetic_models.py of the reference
(``power_law`` :31-45, ``InputGenerator`` :51-113, ``SyntheticModelTFDE`` :116-176,
``SyntheticModelNative`` :179-234).
"""
from __future__ import annotations

from typing import List, Optional

import numpy as np
import torch
from torch import nn

from ..layers.embedding import Embedding
from ..parallel.dist_model_parallel import DistributedEmbedding
from .configs import ModelConfig, expand


def power_law(k_min, k_max, alpha, r):
  """Map uniform ``r`` in [0,1) to a power-law distributed integer in [k_min, k_max)."""
  gamma = 1.0 - alpha
  y = np.power(r * (np.power(k_max, gamma) - np.power(k_min, gamma)) + np.power(k_min, gamma),
               1.0 / gamma)
  return y.astype(np.int64)


def gen_power_law_data(batch_size, hotness, num_rows, alpha, rng: np.random.Generator):
  """Naive power-law id generator (repetition inside a sample is allowed)."""
  y = power_law(1, num_rows + 1, alpha, rng.random(batch_size * hotness)) - 1
  return torch.from_numpy(y.reshape(batch_size, hotness))


class InputGenerator:
  """Pre-generates ``num_batches`` synthetic batches.

  Args:
    model_config: the synthetic model description.
    global_batch_size: global batch.
    alpha: power-law exponent, 0 = uniform ids.
    mp_input_ids: model-parallel input ids of this rank (global batch of these features), None =
      data-parallel inputs (local batch of all features).
    num_batches: number of distinct batches.
    world_size / rank: data-parallel sharding of the numerical features and labels.
  """

  def __init__(self, model_config: ModelConfig, global_batch_size: int, alpha: float = 0.0,
               mp_input_ids: Optional[List[int]] = None, num_batches: int = 10, world_size: int = 1,
               rank: int = 0, device="cpu", seed: int = 0, id_dtype=torch.int64,
               pin_memory: bool = False):
    tables, imap, hot = expand(model_config)
    self.dp_batch_size = global_batch_size // world_size
    self.cat_batch_size = global_batch_size if mp_input_ids is not None else self.dp_batch_size
    self.num_batches = num_batches
    rng = np.random.default_rng(seed + 1000 * rank)
    ids = mp_input_ids if mp_input_ids is not None else list(range(len(imap)))
    self.input_pool = []
    for _ in range(num_batches):
      cats = []
      for i in ids:
        rows, h = tables[imap[i]][0], hot[i]
        if alpha == 0:
          c = torch.from_numpy(rng.integers(0, rows, size=(self.cat_batch_size, h)))
        else:
          c = gen_power_law_data(self.cat_batch_size, h, rows, alpha, rng)
        c = c.to(id_dtype)
        cats.append(c.pin_memory() if pin_memory else c.to(device))
      num = torch.from_numpy(
          rng.random((self.dp_batch_size, model_config.num_numerical_features), dtype=np.float32) *
          100)
      lab = torch.from_numpy(rng.integers(0, 2, size=(self.dp_batch_size, 1)).astype(np.float32))
      if pin_memory:
        num, lab = num.pin_memory(), lab.pin_memory()
      else:
        num, lab = num.to(device), lab.to(device)
      self.input_pool.append(((num, cats), lab))

  def __len__(self):
    return self.num_batches

  def __getitem__(self, idx):
    return self.input_pool[idx % self.num_batches]


def _interact(x: torch.Tensor, stride: int) -> torch.Tensor:
  """Memory-bound 1-D average pooling over the concatenated embeddings (emulates FM / pooling
  interactions; 'same' padding like Keras AveragePooling1D)."""
  n = x.shape[1]
  out_len = -(-n // stride)
  pad = max(0, (out_len - 1) * stride + stride - n)
  left = pad // 2
  xp = nn.functional.pad(x.unsqueeze(1), (left, pad - left))
  ones = nn.functional.pad(torch.ones(1, 1, n, dtype=x.dtype, device=x.device), (left, pad - left))
  s = nn.functional.avg_pool1d(xp, stride, stride) * stride
  cnt = nn.functional.avg_pool1d(ones, stride, stride) * stride
  return (s / cnt).squeeze(1)


class _SyntheticBase(nn.Module):

  def _build_mlp(self, config: ModelConfig, in_dim: int, device):
    # pad the first layer's fan-in to a multiple of 8 elements (16 bytes of bf16) so the GEMM is
    # eligible for the TMA / tcgen05 library kernels; the pad inputs are zeros
    self._in_dim = in_dim
    self._in_pad = (-in_dim) % 8
    in_dim += self._in_pad
    layers, d = [], in_dim
    for h in config.mlp_sizes:
      layers += [nn.Linear(d, h, device=device), nn.ReLU()]
      d = h
    layers.append(nn.Linear(d, 1, device=device))
    self.mlp = nn.Sequential(*layers)

  def _head(self, outs, numerical):
    amp = self.compute_dtype != torch.float32 and numerical.is_cuda
    x = torch.cat(outs, dim=1) if isinstance(outs, (list, tuple)) else outs
    if self.interact_stride is not None:
      x = _interact(x.float(), self.interact_stride)
    dt = self.compute_dtype if amp else numerical.dtype
    parts = [x.to(dt), numerical.to(dt)]
    if self._in_pad:
      parts.append(torch.zeros(x.shape[0], self._in_pad, dtype=dt, device=x.device))
    with torch.autocast("cuda", dtype=self.compute_dtype, enabled=amp):
      return self.mlp(torch.cat(parts, dim=1))

  def dense_parameters(self):
    return [p for p in self.parameters() if not getattr(p, "de_local", False)]


class SyntheticModel(_SyntheticBase):
  """Synthetic model on :class:`DistributedEmbedding` (``memory_balanced``, sum combiner, shared
  multi-hot inputs through ``input_table_map``).  ``table_dtype``: storage of the model-parallel
  tables (fp32, bf16 or fp16, see :class:`DistributedEmbedding`)."""

  def __init__(self, model_config: ModelConfig, column_slice_threshold=None, dp_input=False,
               device=None, compute_dtype=torch.float32, backend="auto",
               row_slice_threshold=None, data_parallel_threshold=None, strategy="memory_balanced",
               table_dtype=torch.float32):
    super().__init__()
    tables, imap, hots = expand(model_config)[:3]
    self.input_table_map = imap
    self.compute_dtype = compute_dtype
    self.interact_stride = model_config.interact_stride
    embs = [{"input_dim": r, "output_dim": w, "combiner": "sum", "layer_type": Embedding}
            for r, w in tables]
    self.embedding = DistributedEmbedding(embs, strategy=strategy, dp_input=dp_input,
                                          input_table_map=imap,
                                          column_slice_threshold=column_slice_threshold,
                                          row_slice_threshold=row_slice_threshold,
                                          data_parallel_threshold=data_parallel_threshold,
                                          device=device, compute_dtype=compute_dtype,
                                          backend=backend, input_hotness=list(hots),
                                          table_dtype=table_dtype)
    self.embedding.zero_copy_output = True  # consumed inside this module's step
    total = sum(tables[t][1] for t in imap)
    if self.interact_stride is not None:
      total = -(-total // self.interact_stride)
    self._build_mlp(model_config, total + model_config.num_numerical_features, device)

  def forward(self, numerical, categorical, staged: bool = False):
    if staged:
      x = self.embedding._engine.run(concat=True)
    else:
      x = self.embedding(categorical, concat=True)
    return self._head(x, numerical)


class SyntheticModelNative(_SyntheticBase):
  """Undistributed baseline with stock ``torch.nn.EmbeddingBag`` tables (data parallel only)."""

  def __init__(self, model_config: ModelConfig, device=None, compute_dtype=torch.float32):
    super().__init__()
    tables, imap, hots = expand(model_config)[:3]
    self.input_table_map = imap
    self.compute_dtype = compute_dtype
    self.interact_stride = model_config.interact_stride
    self.embeddings = nn.ModuleList(
        [nn.EmbeddingBag(r, w, mode="sum", device=device) for r, w in tables])
    total = sum(tables[t][1] for t in imap)
    if self.interact_stride is not None:
      total = -(-total // self.interact_stride)
    self._build_mlp(model_config, total + model_config.num_numerical_features, device)

  def forward(self, numerical, categorical):
    outs = [self.embeddings[t](c.to(torch.int64)) for t, c in zip(self.input_table_map, categorical)]
    return self._head(outs, numerical)
