"""Stochastic rounding of fp32 values into bf16 / fp16 tables.

Half-precision embedding tables (``DistributedEmbedding(table_dtype=torch.bfloat16)``) keep their
optimizer math and state in fp32 and write the new weight back with stochastic rounding: an
update smaller than half an ulp (8 significand bits in bf16) would be lost on every step by
round-to-nearest, while stochastic rounding keeps its expected value.

The rule is defined once and implemented twice, here and in ``ops/csrc/common.cuh``
(``round_stochastic``); both agree bit for bit:

* ``lo`` / ``hi`` are the neighbouring representable values of the fp32 ``x`` in the target
  dtype.  If ``lo == hi`` (``x`` is representable) the result is ``x``.
* otherwise ``u = (r >> 8) * 2**-24`` and the result is ``hi`` if ``u * (hi - lo) < x - lo``,
  else ``lo``.  Every fp32 operation of that comparison is exact.
* NaN, +-inf and values beyond the finite range of the target convert as round-to-nearest does.
* ``r`` is a 32-bit hash of (optimizer step, row key, column, stream), see :func:`random_bits`.
  The row key of the fused back end is the row's position in the rank's sorted-update key space
  (the fused local table's ``key_base`` plus the row), of :class:`SparseRowOptimizer` the row
  index.

Half-precision optimizer state (``set_optimizer(..., state_dtype=torch.bfloat16)``) is stored
with the same rule.  Each stored quantity draws from its own stream of the hash, so the rounding
decisions of a weight and of its state are independent:

* stream 0: the weight (the bits of half-precision tables, unchanged by the streams);
* stream 1: ``state0`` (the Adagrad accumulator, Adam's and row-wise Adam's ``m``, FTRL's
  accumulator ``n``);
* stream 2: ``state1`` (Adam's ``v``, FTRL's linear term ``z``; row-wise Adam's ``v`` is one fp32
  word per row and is never rounded).

The stream is folded into the step seed: ``mix((step + 0x9E3779B9 + stream * 0x632BE5AB) mod
2**32)``.  Two streams draw the same bits only at step offsets of about 1.7e9, far beyond the
2**24 steps the fp32 step counter counts exactly.
"""
from __future__ import annotations

from typing import Union

import numpy as np
import torch

HALF_DTYPES = (torch.bfloat16, torch.float16)
_M32 = np.uint64(0xFFFFFFFF)


def _mix(h: np.ndarray) -> np.ndarray:
  """32-bit integer finaliser (values < 2**32 held in uint64)."""
  h = h ^ (h >> np.uint64(16))
  h = (h * np.uint64(0x7FEB352D)) & _M32
  h = h ^ (h >> np.uint64(15))
  h = (h * np.uint64(0x846CA68B)) & _M32
  return h ^ (h >> np.uint64(16))


STREAM_WEIGHT, STREAM_STATE0, STREAM_STATE1 = 0, 1, 2


def random_bits(step: int, keys, cols, stream: int = STREAM_WEIGHT) -> np.ndarray:
  """``r`` of every (row key, column) of ``stream``: ``keys`` and ``cols`` broadcast against each
  other."""
  keys = np.asarray(keys, dtype=np.int64).view(np.uint64)
  cols = np.asarray(cols, dtype=np.int64).astype(np.uint64) & _M32
  seed = (int(step) + 0x9E3779B9 + int(stream) * 0x632BE5AB) & 0xFFFFFFFF
  h = _mix(np.asarray(seed, dtype=np.uint64))
  h = _mix(h ^ (keys & _M32))
  h = _mix(h ^ (keys >> np.uint64(32)))
  return _mix(h ^ cols).astype(np.uint32)


def _ordered(bits: np.ndarray) -> np.ndarray:
  b = bits.astype(np.int32)
  return np.where(b & 0x8000, -(b & 0x7FFF), b)


def _from_ordered(o: np.ndarray) -> np.ndarray:
  return np.where(o >= 0, o, 0x8000 | (-o)).astype(np.uint16)


def _as_float(bits: np.ndarray, dtype: torch.dtype) -> np.ndarray:
  t = torch.from_numpy(np.ascontiguousarray(bits).view(np.int16)).view(dtype)
  return t.float().numpy()


def stochastic_round_bits(x: np.ndarray, dtype: torch.dtype, r: np.ndarray) -> np.ndarray:
  """The rule above on fp32 ``x`` with random words ``r`` (same shape); returns uint16 bits."""
  x = np.ascontiguousarray(x, dtype=np.float32)
  rn = torch.from_numpy(x).to(dtype).view(torch.int16).numpy().view(np.uint16)
  rn_f = _as_float(rn, dtype)
  max_finite = np.float32(torch.finfo(dtype).max)
  with np.errstate(invalid="ignore", over="ignore"):
    keep = (rn_f == x) | ~(np.abs(x) <= max_finite)
    up = rn_f < x
    nb = _from_ordered(_ordered(rn) + np.where(up, 1, -1))
    nb_f = _as_float(nb, dtype)
    lo = np.where(up, rn_f, nb_f).astype(np.float32)
    hi = np.where(up, nb_f, rn_f).astype(np.float32)
    u = (np.asarray(r, dtype=np.uint32) >> np.uint32(8)).astype(np.float32) * np.float32(2.0**-24)
    take_hi = (u * (hi - lo)).astype(np.float32) < (x - lo).astype(np.float32)
  out = np.where(take_hi, np.where(up, nb, rn), np.where(up, rn, nb)).astype(np.uint16)
  return np.where(keep, rn, out).astype(np.uint16)


def stochastic_round(x: torch.Tensor, dtype: torch.dtype, step: int,
                     keys: Union[torch.Tensor, np.ndarray, int], col0: int = 0,
                     stream: int = STREAM_WEIGHT) -> torch.Tensor:
  """Round fp32 rows ``x`` (``[..., width]``) into ``dtype``; ``keys`` (``[...]``) are the row
  keys, columns count from ``col0``, ``stream`` selects the random stream (see the module
  docstring).  Returns a CPU tensor of ``dtype`` and ``x``'s shape."""
  if dtype not in HALF_DTYPES:
    raise ValueError(f"stochastic rounding targets bf16 or fp16, not {dtype}")
  xs = x.detach().to("cpu", torch.float32).contiguous().numpy()
  if isinstance(keys, torch.Tensor):
    keys = keys.detach().cpu().numpy()
  width = xs.shape[-1] if xs.ndim else 1
  cols = np.arange(col0, col0 + width, dtype=np.int64)
  r = random_bits(step, np.asarray(keys, dtype=np.int64)[..., None], cols, stream)
  r = np.broadcast_to(r, xs.shape)
  bits = stochastic_round_bits(xs, dtype, r)
  return torch.from_numpy(bits.view(np.int16).copy()).view(dtype)
