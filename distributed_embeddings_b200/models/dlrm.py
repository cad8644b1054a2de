"""DLRM (MLPerf configuration) on the hybrid-parallel embedding engine.

Bottom MLP 512-256-128 on 13 numerical features, 26 embedding tables of width 128, pairwise dot
interaction, top MLP 1024-1024-512-256-1 (reference examples/dlrm/main.py:76-145,
examples/dlrm/utils.py:92-113).  Dense layers are data parallel (bf16 compute, fp32 master
weights), embeddings are model parallel through :class:`DistributedEmbedding`.

``interaction="dcnv2"`` builds DLRM-DCNv2 instead (the model of the MLPerf Training DLRM benchmark
since v3.0): the dot interaction is replaced by a low-rank cross network over the concatenated
feature vectors, usually with multi-hot, sum-pooled categorical features
(``multi_hot_sizes``, e.g. :data:`MLPERF_DCNV2_MULTI_HOT_SIZES`).
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


# Ids per sample of the 26 categorical features in the MLPerf Training DLRM-DCNv2 reference
# configuration (its multi-hot Criteo 1TB dataset, pooled with "sum"); 214 lookups per sample.
MLPERF_DCNV2_MULTI_HOT_SIZES = [
    3, 2, 1, 2, 6, 1, 1, 1, 1, 7, 3, 8, 1, 6, 9, 5, 1, 1, 1, 12, 100, 27, 10, 3, 1, 1
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


class CrossLayer(nn.Module):
  """One low-rank cross layer: ``x_{l+1} = x0 * (W (V x_l) + b) + x_l``.

  ``V``: ``nn.Linear(D, r, bias=False)``, ``W``: ``nn.Linear(r, D)``.  Both kernels are
  Glorot-normal and the bias is zero (the initialisation of torchrec's ``LowRankCrossNet``): at
  initialisation the layer adds ``x0 * (W V x_l)``, a term of the scale of ``x_l``."""

  def __init__(self, dim: int, rank: int, device=None):
    super().__init__()
    self.V = nn.Linear(dim, rank, bias=False, device=device)
    self.W = nn.Linear(rank, dim, device=device)
    nn.init.xavier_normal_(self.V.weight)
    nn.init.xavier_normal_(self.W.weight)
    nn.init.zeros_(self.W.bias)

  def forward(self, x0, xl):
    return x0 * self.W(self.V(xl)) + xl


class DLRM(nn.Module):
  """``interaction``: ``"dot"`` (pairwise dot products of the 26 embeddings and the bottom-MLP
  vector, the 2019 MLPerf model) or ``"dcnv2"`` (DLRM-DCNv2): a low-rank cross network of
  ``dcn_num_layers`` layers of rank ``dcn_low_rank_dim`` (:class:`CrossLayer`) over

      x0 = [emb_0 | emb_1 | ... | emb_{n-1} | bottom]     (D = (n + 1) * embedding_dim columns)

  with the embeddings first, so that the fused engine's lookups can write straight into ``x0``
  (torchrec puts the dense vector first: a permutation of V's columns and W's rows).  The top MLP
  runs on the last cross layer's output.

  ``multi_hot_sizes``: ids per sample of every feature; each table then pools its ``[b, h_f]``
  ids with ``sum`` (either interaction).  None keeps one-hot ``[b]`` inputs."""

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
               table_dtype: torch.dtype = torch.float32,
               interaction: str = "dot",
               dcn_num_layers: int = 3,
               dcn_low_rank_dim: int = 512,
               multi_hot_sizes: Optional[Sequence[int]] = None,
               gpu_embedding_size: Optional[int] = None,
               offload_cache_size: Optional[int] = None):
    """``table_dtype``: storage of the model-parallel embedding tables (fp32, bf16 or fp16, see
    :class:`DistributedEmbedding`); bf16 fits the 40M-row MLPerf tables on one 80 GB GPU.
    ``gpu_embedding_size`` / ``offload_cache_size``: per-rank HBM element budgets of the tables
    and of the HBM cache of the tables beyond it (pinned host memory), see
    :class:`DistributedEmbedding`."""
    super().__init__()
    if interaction not in ("dot", "dcnv2"):
      raise ValueError("interaction must be 'dot' or 'dcnv2'")
    if bottom_mlp_dims[-1] != embedding_dim:
      raise ValueError("bottom MLP must end at the embedding width for the dot interaction")
    self.table_sizes = [int(s) for s in table_sizes]
    if multi_hot_sizes is not None:
      multi_hot_sizes = [int(h) for h in multi_hot_sizes]
      if len(multi_hot_sizes) != len(self.table_sizes) or min(multi_hot_sizes) < 1:
        raise ValueError("multi_hot_sizes needs one hotness >= 1 per table")
    self.multi_hot_sizes = multi_hot_sizes
    self.interaction = interaction
    self.embedding_dim = embedding_dim
    self.compute_dtype = compute_dtype
    self.bottom_mlp = MLP(num_numerical_features, list(bottom_mlp_dims), True, device)
    n = len(self.table_sizes) + 1
    if interaction == "dot":
      self.num_interactions = n * (n - 1) // 2
      top_in = self.num_interactions + embedding_dim
    else:
      if dcn_num_layers < 1 or dcn_low_rank_dim < 1:
        raise ValueError("the cross network needs at least one layer of rank >= 1")
      self.cross_dim = n * embedding_dim
      self.cross_layers = nn.ModuleList(
          [CrossLayer(self.cross_dim, dcn_low_rank_dim, device) for _ in range(dcn_num_layers)])
      top_in = self.cross_dim
    self.top_mlp = MLP(top_in, list(top_mlp_dims), False, device)
    sum_pool = test_combiner or multi_hot_sizes is not None
    embs = [{"input_dim": s, "output_dim": embedding_dim,
             "combiner": "sum" if sum_pool else None,
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
                                          table_dtype=table_dtype,
                                          gpu_embedding_size=gpu_embedding_size,
                                          offload_cache_size=offload_cache_size)
    # the activation is consumed inside this module's step: no defensive copy of the engine buffer
    self.embedding.zero_copy_output = True
    if interaction == "dot":
      ii, jj = torch.tril_indices(n, n, offset=-1)
      self.register_buffer("tril", (ii * n + jj).to(device), persistent=False)

  def dense_parameters(self):
    return [p for p in self.parameters() if not getattr(p, "de_local", False)]

  def forward(self, numerical: torch.Tensor, categorical, staged: bool = False) -> torch.Tensor:
    """``categorical``: list of 26 id tensors (``[b]``, or ``[b, h_f]`` with ``multi_hot_sizes``),
    or None with ``staged=True`` when the ids were written straight into the engine's staging
    buffer."""
    amp = self.compute_dtype != torch.float32 and numerical.is_cuda
    with torch.autocast("cuda", dtype=self.compute_dtype, enabled=amp):
      x = self.bottom_mlp(numerical)
    if staged:
      emb = self.embedding._engine.run(concat=True)
    else:
      emb = self.embedding(categorical, concat=True)
    with torch.autocast("cuda", dtype=self.compute_dtype, enabled=amp):
      if self.interaction == "dot":
        z = dot_interact(emb.to(x.dtype), x, self.tril)
      else:
        x0 = torch.cat([emb.to(x.dtype), x], dim=1)  # embeddings first, bottom vector last
        z = x0
        for layer in self.cross_layers:
          z = layer(x0, z)
      return self.top_mlp(z)
