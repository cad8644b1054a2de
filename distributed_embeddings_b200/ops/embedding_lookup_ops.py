"""Python op wrappers + autograd glue for the embedding kernels.

CUDA tensors run the hand-written sm_90a kernels (``_C.so``; there is no eager fallback on GPU),
CPU tensors run a plain PyTorch implementation with identical semantics which doubles as the
numerics oracle in the tests.

Capability parity: ``distributed_embeddings/python/ops/embedding_lookup_ops.py`` of the reference
(``embedding_lookup`` :37-102, gradient as deduplicated IndexedSlices :105-122,
``integer_lookup`` :125-128, ``read_var_no_copy`` :26-34).
"""
from __future__ import annotations

from typing import Optional, Tuple, Union

import torch

torch.sparse.check_sparse_tensor_invariants.disable()

from . import _native
from .ragged import RaggedIds, SparseIds

_COMBINERS = {None: -1, "sum": 0, "mean": 1}


def read_var_no_copy(param: torch.Tensor) -> torch.Tensor:
  """Alias of the parameter storage without a copy (PyTorch never copies on read; kept for API
  parity with the reference's ``ReadVariableNoCopy`` op)."""
  return param.detach()


# ----------------------------------------------------------------------------- CPU oracle
def _sample_ids_cpu(values, offsets, hotness, batch):
  """Sample id of every looked-up id and ids per sample."""
  if offsets is None:
    sample = torch.arange(batch, device=values.device).repeat_interleave(hotness)
    counts = torch.full((batch,), hotness, dtype=torch.int64, device=values.device)
  else:
    counts = offsets[1:] - offsets[:-1]
    sample = torch.repeat_interleave(torch.arange(batch, device=values.device), counts)
  return sample, counts


def _lookup_fwd_cpu(param, values, offsets, hotness, batch, combiner):
  """Pooled in fp32 whatever the table dtype; the result has the table's dtype."""
  rows, width = param.shape
  flat = values.reshape(-1).to(torch.int64)
  sample, counts = _sample_ids_cpu(flat, offsets, hotness, batch)
  ok = (flat >= 0) & (flat < rows)
  acc = torch.float32 if param.dtype in (torch.bfloat16, torch.float16) else param.dtype
  gathered = param[flat.clamp(0, rows - 1)].to(acc) * ok.unsqueeze(1).to(acc)
  out = torch.zeros(batch, width, dtype=acc, device=param.device)
  out.index_add_(0, sample, gathered)
  if combiner == 1:
    out = out / counts.clamp(min=1).unsqueeze(1).to(acc)
  return out.to(param.dtype)


def _lookup_grad_cpu(values, offsets, hotness, batch, combiner, grad, num_rows):
  flat = values.reshape(-1).to(torch.int64)
  sample, counts = _sample_ids_cpu(flat, offsets, hotness, batch)
  g = grad.to(torch.float32)[sample]
  if combiner == 1:
    g = g / counts.clamp(min=1)[sample].unsqueeze(1).to(g.dtype)
  ok = (flat >= 0) & (flat < num_rows)
  flat, g = flat[ok], g[ok]
  uniq, inverse = torch.unique(flat, return_inverse=True)
  rows = torch.zeros(uniq.numel(), grad.shape[1], dtype=torch.float32, device=grad.device)
  rows.index_add_(0, inverse, g)
  return uniq, rows


# ----------------------------------------------------------------------------- raw ops
def lookup_forward(param, values, offsets, hotness, batch, combiner, out_bf16=False):
  if param.is_cuda:
    return _native.require().embedding_lookup_fwd(param, values.contiguous(), offsets, hotness,
                                                  batch, combiner, out_bf16)
  out = _lookup_fwd_cpu(param, values, offsets, hotness, batch, combiner)
  return out.to(torch.bfloat16) if out_bf16 else out


def lookup_grad_sparse(values, offsets, hotness, batch, combiner, grad,
                       num_rows) -> Tuple[torch.Tensor, torch.Tensor]:
  """(unique_ids ascending, summed gradient rows) - the IndexedSlices of the reference."""
  if grad.is_cuda:
    if grad.stride(-1) != 1:
      grad = grad.contiguous()
    return _native.require().embedding_lookup_grad(values.contiguous(), offsets, hotness, batch,
                                                   combiner, grad, num_rows)
  return _lookup_grad_cpu(values, offsets, hotness, batch, combiner, grad, num_rows)


def scatter_add_rows(dst, values, offsets, hotness, batch, combiner, grad, scale=1.0):
  """dst[id] += scale * w * grad[sample] for every looked-up id (atomic on GPU)."""
  if dst.is_cuda:
    if grad.stride(-1) != 1:
      grad = grad.contiguous()
    _native.require().embedding_scatter_add(dst, values.contiguous(), offsets, hotness, batch,
                                            combiner, grad, float(scale))
    return dst
  ids, rows = _lookup_grad_cpu(values, offsets, hotness, batch, combiner, grad, dst.shape[0])
  dst.index_add_(0, ids, rows.to(dst.dtype) * scale)
  return dst


class _PooledLookup(torch.autograd.Function):
  """Pooled lookup whose parameter gradient is a deduplicated sparse tensor."""

  @staticmethod
  def forward(ctx, param, values, offsets, hotness, batch, combiner, sparse_grad):
    ctx.save_for_backward(values, offsets)
    ctx.meta = (hotness, batch, combiner, sparse_grad, tuple(param.shape))
    return lookup_forward(param.detach(), values, offsets, hotness, batch, combiner)

  @staticmethod
  def backward(ctx, grad):
    values, offsets = ctx.saved_tensors
    hotness, batch, combiner, sparse_grad, shape = ctx.meta
    if sparse_grad:
      ids, rows = lookup_grad_sparse(values, offsets, hotness, batch, combiner, grad, shape[0])
      g = torch.sparse_coo_tensor(ids.unsqueeze(0), rows, size=shape, is_coalesced=True,
                                  check_invariants=False)
    else:
      g = torch.zeros(shape, dtype=torch.float32, device=grad.device)
      scatter_add_rows(g, values, offsets, hotness, batch, combiner, grad)
    return g, None, None, None, None, None, None


def embedding_lookup_variable_hotness(param: torch.Tensor,
                                      values: torch.Tensor,
                                      row_splits: torch.Tensor,
                                      combiner: str = "sum",
                                      sparse_grad: bool = True) -> torch.Tensor:
  """CSR gather-and-reduce: ``out[i] = combine(param[values[row_splits[i]:row_splits[i+1]]])``."""
  if combiner not in ("sum", "mean"):
    raise ValueError(f"combiner must be 'sum' or 'mean', got {combiner}")
  batch = row_splits.numel() - 1
  return _PooledLookup.apply(param, values, row_splits.to(torch.int64), 0, batch,
                             _COMBINERS[combiner], sparse_grad)


def embedding_lookup_fixed_hotness(param, ids, combiner="sum", sparse_grad=True):
  batch, hot = ids.shape
  return _PooledLookup.apply(param, ids.reshape(-1), None, hot, batch, _COMBINERS[combiner],
                             sparse_grad)


def row_to_split(indices: torch.Tensor, num_rows: int) -> torch.Tensor:
  """COO row indices (sorted by row, shape [nnz, 2]) -> CSR ``row_splits[num_rows + 1]``."""
  indices = indices.to(torch.int64)
  if indices.is_cuda:
    return _native.require().row_to_split(indices.contiguous(), int(num_rows))
  rows = indices[:, 0].contiguous()
  return torch.searchsorted(rows, torch.arange(num_rows + 1, dtype=torch.int64), right=False)


IdsLike = Union[torch.Tensor, RaggedIds, SparseIds]


def embedding_lookup(param: torch.Tensor,
                     ids: IdsLike,
                     combiner: Optional[str] = None,
                     sparse_grad: bool = True) -> torch.Tensor:
  """Look up embeddings for ``ids`` in ``param``.

  Args:
    param: ``[rows, width]`` embedding matrix.
    ids: 2-D int32/int64 tensor, :class:`RaggedIds` (CSR) or :class:`SparseIds` (COO).
    combiner: ``None`` (no reduction, output ``shape(ids) + [width]``), ``'sum'`` or ``'mean'``
      (ids of one row are reduced, output ``[batch, width]``).
    sparse_grad: produce a deduplicated sparse gradient for ``param`` (reference behaviour).
  """
  if not isinstance(param, torch.Tensor):
    raise TypeError("param must be Tensor")
  if combiner not in _COMBINERS:
    raise ValueError(f"Unsupported combiner {combiner}")
  if isinstance(ids, torch.Tensor) and ids.is_sparse:
    ids = SparseIds.from_torch_sparse(ids)
  if isinstance(ids, torch.Tensor):
    if ids.dim() != 2:
      raise ValueError("Only support 2D input")
    if combiner is None:
      b, h = ids.shape
      out = _PooledLookup.apply(param, ids.reshape(-1), None, 1, b * h, 0, sparse_grad)
      return out.reshape(b, h, param.shape[1])
    return embedding_lookup_fixed_hotness(param, ids, combiner, sparse_grad)
  if combiner is None:
    raise ValueError("ragged / sparse ids need a combiner")
  if isinstance(ids, RaggedIds):
    return embedding_lookup_variable_hotness(param, ids.values, ids.row_splits, combiner,
                                             sparse_grad)
  if isinstance(ids, SparseIds):
    splits = row_to_split(ids.indices, ids.dense_shape[0])
    return embedding_lookup_variable_hotness(param, ids.values, splits, combiner, sparse_grad)
  raise TypeError(f"unsupported ids type {type(ids)}")


# ----------------------------------------------------------------------------- IntegerLookup
def integer_lookup_init(table: torch.Tensor):
  """Fill the slot array with the empty sentinel (-1, -1)."""
  if table.is_cuda:
    _native.require().hash_init(table)
  else:
    table.fill_(-1)
  return table


def integer_lookup(table: torch.Tensor, count: torch.Tensor, next_index: torch.Tensor,
                   keys: torch.Tensor, capacity: int) -> torch.Tensor:
  """Map int64 keys to contiguous indices in ``[1, capacity)``, inserting unseen keys while
  indices remain; 0 = out of vocabulary.  ``count[index]`` accumulates key frequencies."""
  if table.is_cuda:
    return _native.require().integer_lookup(table, count, next_index, keys.to(torch.int64),
                                            int(capacity)).reshape(keys.shape)
  return _integer_lookup_cpu(table, count, next_index, keys, capacity)


def _mix64(k: int) -> int:
  m = (1 << 64) - 1
  k &= m
  k ^= k >> 33
  k = (k * 0xff51afd7ed558ccd) & m
  k ^= k >> 33
  k = (k * 0xc4ceb9fe1a85ec53) & m
  k ^= k >> 33
  return k


def _integer_lookup_cpu(table, count, next_index, keys, capacity):
  """Sequential reference with the same slot protocol as the CUDA kernel (first come first served
  in flattened key order)."""
  n_slots = table.numel() // 2
  tab = table.view(-1)
  flat = keys.reshape(-1).to(torch.int64).tolist()
  out = []
  nxt = int(next_index.item())
  for key in flat:
    value = 0
    if key != -1:
      slot = _mix64(key) % n_slots
      for _ in range(n_slots):
        cur = int(tab[2 * slot])
        if cur == -1:
          if nxt >= capacity:
            value = 0
            break
          tab[2 * slot] = key
          value = nxt if nxt < capacity else 0
          nxt += 1
          tab[2 * slot + 1] = value
          break
        if cur == key:
          value = int(tab[2 * slot + 1])
          break
        slot = 0 if slot + 1 == n_slots else slot + 1
    count[value] += 1
    out.append(value)
  next_index.fill_(nxt)
  return torch.tensor(out, dtype=torch.int64).reshape(keys.shape)
