"""DLRM (MLPerf configuration) on the hybrid-parallel embedding engine.

Bottom MLP 512-256-128 on 13 numerical features, 26 embedding tables of width 128, pairwise dot
interaction, top MLP 1024-1024-512-256-1 (reference examples/dlrm/main.py:76-145,
examples/dlrm/utils.py:92-113).  Dense layers are data parallel (bf16 compute, fp32 master
weights), embeddings are model parallel through :class:`DistributedEmbedding`.
"""
from __future__ import annotations

import math
from typing import List, Optional, Sequence

import torch
from torch import nn

from ..layers.embedding import Embedding
from ..parallel.dist_model_parallel import DistributedEmbedding
from ..utils.initializers import DLRMInitializer

# Criteo Terabyte table sizes of the MLPerf DLRM benchmark (max_ind_range 40M), before the
# reference's "+1" (examples/dlrm/main.py:68-73 reads them from the dataset's model_size.json).
CRITEO_1TB_MLPERF_SIZES = [
    39884406, 39043, 17289, 7420, 20263, 3, 7120, 1543, 63, 38532951, 2953546, 403346, 10, 2208,
    11938, 155, 4, 976, 14, 39979771, 25641295, 39664984, 585935, 12972, 108, 36
]


def mlperf_table_sizes(max_rows: int = 40_000_000) -> List[int]:
  """Table sizes of the MLPerf configuration; ``max_rows`` below 40M caps the tables further, the
  way a smaller ``max_ind_range`` does (20M: 104 M rows, 49.6 GiB fp32 at dim 128)."""
  return [min(s, max_rows) + 1 for s in CRITEO_1TB_MLPERF_SIZES]


class MLP(nn.Module):
  """Dense stack; Glorot-normal kernels and N(0, sqrt(1/dim)) biases like the reference."""

  def __init__(self, in_dim: int, dims: Sequence[int], final_activation: bool, device=None):
    super().__init__()
    layers = []
    d = in_dim
    for i, h in enumerate(dims):
      lin = nn.Linear(d, h, device=device)
      nn.init.xavier_normal_(lin.weight)
      nn.init.normal_(lin.bias, std=math.sqrt(1.0 / h))
      layers.append(lin)
      if i < len(dims) - 1 or final_activation:
        layers.append(nn.ReLU())
      d = h
    self.net = nn.Sequential(*layers)

  def forward(self, x):
    return self.net(x)


def dot_interact(emb: torch.Tensor, bottom: torch.Tensor, tril: torch.Tensor) -> torch.Tensor:
  """Pairwise dot products of the 26 embeddings + bottom-MLP vector; strict lower triangle,
  concatenated with the bottom-MLP output.  ``emb``: [b, n*d] features concatenated."""
  b, d = bottom.shape
  feats = torch.cat([bottom.unsqueeze(1), emb.view(b, -1, d)], dim=1)  # [b, n+1, d]
  z = torch.bmm(feats, feats.transpose(1, 2))
  flat = z.flatten(1)[:, tril]
  return torch.cat([flat, bottom], dim=1)


class DLRM(nn.Module):

  def __init__(self,
               table_sizes: Sequence[int],
               embedding_dim: int = 128,
               bottom_mlp_dims: Sequence[int] = (512, 256, 128),
               top_mlp_dims: Sequence[int] = (1024, 1024, 512, 256, 1),
               num_numerical_features: int = 13,
               dp_input: bool = True,
               dist_strategy: str = "memory_balanced",
               column_slice_threshold: Optional[int] = None,
               row_slice_threshold: Optional[int] = None,
               data_parallel_threshold: Optional[int] = None,
               test_combiner: bool = False,
               device=None,
               compute_dtype: torch.dtype = torch.bfloat16,
               backend: str = "auto",
               world_size: Optional[int] = None,
               rank: Optional[int] = None,
               table_dtype: torch.dtype = torch.float32):
    """``table_dtype``: storage of the model-parallel embedding tables (fp32, bf16 or fp16, see
    :class:`DistributedEmbedding`); bf16 fits the 40M-row MLPerf tables on one 80 GB GPU."""
    super().__init__()
    if bottom_mlp_dims[-1] != embedding_dim:
      raise ValueError("bottom MLP must end at the embedding width for the dot interaction")
    self.table_sizes = [int(s) for s in table_sizes]
    self.embedding_dim = embedding_dim
    self.compute_dtype = compute_dtype
    self.bottom_mlp = MLP(num_numerical_features, list(bottom_mlp_dims), True, device)
    n = len(self.table_sizes) + 1
    self.num_interactions = n * (n - 1) // 2
    self.top_mlp = MLP(self.num_interactions + embedding_dim, list(top_mlp_dims), False, device)
    embs = [{"input_dim": s, "output_dim": embedding_dim,
             "combiner": "sum" if test_combiner else None,
             "embeddings_initializer": DLRMInitializer(), "layer_type": Embedding}
            for s in self.table_sizes]
    self.embedding = DistributedEmbedding(embs,
                                          strategy=dist_strategy,
                                          dp_input=dp_input,
                                          column_slice_threshold=column_slice_threshold,
                                          row_slice_threshold=row_slice_threshold,
                                          data_parallel_threshold=data_parallel_threshold,
                                          device=device,
                                          compute_dtype=compute_dtype,
                                          backend=backend,
                                          world_size=world_size,
                                          rank=rank,
                                          table_dtype=table_dtype)
    # the activation is consumed inside this module's step: no defensive copy of the engine buffer
    self.embedding.zero_copy_output = True
    ii, jj = torch.tril_indices(n, n, offset=-1)
    self.register_buffer("tril", (ii * n + jj).to(device), persistent=False)

  def dense_parameters(self):
    return [p for p in self.parameters() if not getattr(p, "de_local", False)]

  def forward(self, numerical: torch.Tensor, categorical, staged: bool = False) -> torch.Tensor:
    """``categorical``: list of 26 id tensors (``[b]``), or None with ``staged=True`` when the
    ids were written straight into the engine's staging buffer."""
    amp = self.compute_dtype != torch.float32 and numerical.is_cuda
    with torch.autocast("cuda", dtype=self.compute_dtype, enabled=amp):
      x = self.bottom_mlp(numerical)
    if staged:
      emb = self.embedding._engine.run(concat=True)
    else:
      emb = self.embedding(categorical, concat=True)
    with torch.autocast("cuda", dtype=self.compute_dtype, enabled=amp):
      z = dot_interact(emb.to(x.dtype), x, self.tril)
      return self.top_mlp(z)
