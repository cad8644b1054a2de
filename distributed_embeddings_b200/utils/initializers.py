"""Embedding initializers.

Tables can be hundreds of GB, so initializers fill an already-allocated device tensor in row
chunks instead of materialising a host copy (the reference forces initialisation onto the CPU
to dodge the 2x temporary, embedding.py:28-38; on an 80 GB H100 in-place chunked device init is
both simpler and faster).
"""
from __future__ import annotations

import math
from typing import Any, Callable, Dict, Optional, Sequence, Union

import torch

_CHUNK_ELEMS = 1 << 28  # 256M elements per fill call


class Initializer:
  """Fills ``out`` ([rows, width]) in place; ``logical_rows`` is the table's own row count
  (differs from ``out.shape[0]`` when several tables are fused into one)."""

  def fill_(self, out: torch.Tensor, generator: Optional[torch.Generator] = None):
    raise NotImplementedError

  def get_config(self) -> Dict[str, Any]:
    return {}

  def __call__(self, shape, dtype=torch.float32, device=None, generator=None):
    out = torch.empty(tuple(shape), dtype=dtype, device=device)
    self.fill_(out, generator)
    return out


def _chunked(out: torch.Tensor):
  rows = out.shape[0]
  width = max(1, out[0].numel()) if rows else 1
  step = max(1, _CHUNK_ELEMS // width)
  for start in range(0, rows, step):
    yield out[start:start + step]


class RandomUniform(Initializer):
  """U(minval, maxval); default range is the Keras ``'uniform'`` initializer (+-0.05)."""

  def __init__(self, minval: float = -0.05, maxval: float = 0.05):
    self.minval, self.maxval = float(minval), float(maxval)

  def fill_(self, out, generator=None):
    for chunk in _chunked(out):
      chunk.uniform_(self.minval, self.maxval, generator=generator)
    return out

  def get_config(self):
    return {"minval": self.minval, "maxval": self.maxval}


class RandomNormal(Initializer):

  def __init__(self, mean: float = 0.0, stddev: float = 0.05):
    self.mean, self.stddev = float(mean), float(stddev)

  def fill_(self, out, generator=None):
    for chunk in _chunked(out):
      chunk.normal_(self.mean, self.stddev, generator=generator)
    return out

  def get_config(self):
    return {"mean": self.mean, "stddev": self.stddev}


class Constant(Initializer):

  def __init__(self, value: float = 0.0):
    self.value = float(value)

  def fill_(self, out, generator=None):
    out.fill_(self.value)
    return out

  def get_config(self):
    return {"value": self.value}


class DLRMInitializer(Initializer):
  """U(-1/sqrt(rows), 1/sqrt(rows)) (reference examples/dlrm/utils.py:26-41)."""

  def fill_(self, out, generator=None):
    bound = math.sqrt(1.0 / max(1, out.shape[0]))
    for chunk in _chunked(out):
      chunk.uniform_(-bound, bound, generator=generator)
    return out


class ConcatInitializer(Initializer):
  """Initialise a fused table piecewise so every member sees its own shape
  (reference dist_model_parallel.py:29-40)."""

  def __init__(self, initializer: Initializer, sizes: Sequence[int]):
    self.initializer = initializer
    self.sizes = [int(s) for s in sizes]

  def fill_(self, out, generator=None):
    start = 0
    for n in self.sizes:
      self.initializer.fill_(out[start:start + n], generator)
      start += n
    return out


class FunctionInitializer(Initializer):
  """Wraps a user callable ``fn(shape, dtype=..., device=...) -> Tensor``."""

  def __init__(self, fn: Callable):
    self.fn = fn

  def fill_(self, out, generator=None):
    try:
      val = self.fn(tuple(out.shape), dtype=out.dtype, device=out.device)
    except TypeError:
      val = self.fn(tuple(out.shape))
    out.copy_(torch.as_tensor(val, dtype=out.dtype))
    return out


_REGISTRY = {
    "uniform": RandomUniform,
    "random_uniform": RandomUniform,
    "RandomUniform": RandomUniform,
    "normal": RandomNormal,
    "random_normal": RandomNormal,
    "RandomNormal": RandomNormal,
    "zeros": lambda: Constant(0.0),
    "ones": lambda: Constant(1.0),
    "constant": Constant,
    "Constant": Constant,
    "dlrm": DLRMInitializer,
    "DLRMInitializer": DLRMInitializer,
}


def get(identifier: Union[None, str, dict, Initializer, Callable]) -> Initializer:
  """Resolve a Keras-style initializer identifier."""
  if identifier is None:
    return RandomUniform()
  if isinstance(identifier, Initializer):
    return identifier
  if isinstance(identifier, str):
    if identifier not in _REGISTRY:
      raise ValueError(f"Unknown initializer {identifier}")
    return _REGISTRY[identifier]()
  if isinstance(identifier, dict):
    name = identifier.get("class_name")
    cfg = identifier.get("config", {}) or {}
    if name not in _REGISTRY:
      raise ValueError(f"Unknown initializer {name}")
    cfg = {k: v for k, v in cfg.items() if k in ("minval", "maxval", "mean", "stddev", "value")}
    return _REGISTRY[name](**cfg)
  if callable(identifier):
    return FunctionInitializer(identifier)
  raise ValueError(f"Cannot interpret initializer {identifier!r}")


def serialize(init: Initializer) -> Union[dict, Initializer]:
  for name, cls in _REGISTRY.items():
    if isinstance(cls, type) and type(init) is cls and name[0].isupper():
      return {"class_name": name, "config": init.get_config()}
  return init  # custom objects are carried as-is inside the plan
