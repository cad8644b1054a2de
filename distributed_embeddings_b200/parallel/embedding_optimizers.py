"""The fused optimizers of the model-parallel tables, each described once.

An entry says what every layer needs to know about a kind: its native code (``OPT_*`` of the
update kernels), its state slots, its defaults, and whether a zero gradient still moves it.
:meth:`DistributedEmbedding.set_optimizer`, the fused engine, the plan interpreter,
:class:`SparseRowOptimizer` and the checkpoint code all read it from here.
"""
from __future__ import annotations

import numbers
from typing import Any, Callable, Dict, List, Mapping, NamedTuple, Optional, Tuple

import numpy as np
import torch

from ..ops import _native

# FTRL's hyperparameters and their defaults (Keras ``Ftrl``: learning_rate_power,
# l1_regularization_strength, l2_regularization_strength, l2_shrinkage_regularization_strength,
# beta), in the order they trail the ``segment_update`` op's arguments;
# ``initial_accumulator_value`` is shared with Adagrad
FTRL_DEFAULTS = {"lr_power": -0.5, "l1": 0.0, "l2": 0.0, "l2_shrinkage": 0.0, "beta": 0.0}


def check_ftrl_args(cfg: Mapping[str, Any]):
  """Keras's checks of FTRL's hyperparameters: ``lr_power <= 0``, the others ``>= 0``."""
  if not float(cfg["lr_power"]) <= 0.0:
    raise ValueError(f"ftrl: lr_power must be <= 0, got {cfg['lr_power']}")
  for k in ("initial_accumulator_value", "l1", "l2", "l2_shrinkage", "beta"):
    if not float(cfg[k]) >= 0.0:
      raise ValueError(f"ftrl: {k} must be >= 0, got {cfg[k]}")


# Momentum SGD's hyperparameters and their defaults (torch.optim.SGD's ``momentum`` and
# ``nesterov``, dampening 0), the ``segment_update`` op's arguments of the same names
MOMENTUM_DEFAULTS = {"momentum": 0.9, "nesterov": False}


def check_momentum_args(cfg: Mapping[str, Any]):
  """``momentum`` in [0, 1) and ``nesterov`` a bool."""
  mu = cfg["momentum"]
  if isinstance(mu, bool) or not isinstance(mu, numbers.Real) or not 0.0 <= float(mu) < 1.0:
    raise ValueError(f"momentum: momentum must be a number in [0, 1), got {mu!r}")
  if not isinstance(cfg["nesterov"], bool):
    raise ValueError(f"momentum: nesterov must be a bool, got {cfg['nesterov']!r}")


class Slot(NamedTuple):
  """One state slot: one fp32 word per row (``per_row``), else element-wise ``[rows, width]`` in
  the state dtype; it starts at ``initial_accumulator_value`` (``accumulator``) or at 0."""
  per_row: bool = False
  accumulator: bool = False


class EmbeddingOptimizer(NamedTuple):
  name: str
  code: int                                 # _native.OPT_*
  slots: Tuple[Slot, ...] = ()              # state0, state1 of the kernels' TableDesc
  eps: float = 1e-7
  hyper: Mapping[str, Any] = {}             # keyword arguments of this kind only, with defaults
  check: Optional[Callable[[Mapping[str, Any]], None]] = None  # validates them
  moves_on_zero_grad: bool = False          # a dry (warm-up) update must not run it

  @property
  def elementwise_state(self) -> bool:
    """Whether some slot is element-wise, the state that bf16 can hold."""
    return any(not s.per_row for s in self.slots)


OPTIMIZERS: Dict[str, EmbeddingOptimizer] = {o.name: o for o in (
    EmbeddingOptimizer("sgd", _native.OPT_SGD),
    EmbeddingOptimizer("adagrad", _native.OPT_ADAGRAD, (Slot(accumulator=True),)),
    EmbeddingOptimizer("rowwise_adagrad", _native.OPT_ROWWISE_ADAGRAD,
                       (Slot(per_row=True, accumulator=True),)),
    # m, v
    EmbeddingOptimizer("adam", _native.OPT_ADAM, (Slot(), Slot()), eps=1e-8,
                       moves_on_zero_grad=True),
    # m element-wise, v one word per row
    EmbeddingOptimizer("rowwise_adam", _native.OPT_ROWWISE_ADAM, (Slot(), Slot(per_row=True)),
                       eps=1e-8, moves_on_zero_grad=True),
    # accumulator n, linear term z; on a zero gradient the closed form of z sets the weights
    EmbeddingOptimizer("ftrl", _native.OPT_FTRL, (Slot(accumulator=True), Slot()),
                       hyper=FTRL_DEFAULTS, check=check_ftrl_args, moves_on_zero_grad=True),
    # momentum buffer b; a zero gradient still moves a row by -lr * momentum * b
    EmbeddingOptimizer("momentum", _native.OPT_MOMENTUM, (Slot(),), hyper=MOMENTUM_DEFAULTS,
                       check=check_momentum_args, moves_on_zero_grad=True),
)}
NAMES = tuple(OPTIMIZERS)
BY_CODE = {o.code: o for o in OPTIMIZERS.values()}


# How ``weight_decay`` (lambda) applies, with ``weight_decay_mode``:
# - "l2": lambda * w joins the summed, scaled gradient of a touched row before the optimizer sees
#   it, so Adagrad and Adam divide it by their adaptive denominators;
# - "decoupled" (AdamW-style, FBGEMM's WeightDecayMode.DECOUPLE): the gradient and the state never
#   see it; a touched row is first scaled by 1 - lr * lambda, then the kind's step is applied:
#   w = (1 - lr * lambda) * w - lr * u.  SGD's update is the same in both modes (momentum SGD's is
#   not: its L2 decay passes through the buffer).  FTRL has no decoupled mode: its weight is a
#   closed form of z (use its l2 / l2_shrinkage).
WEIGHT_DECAY_MODES = ("l2", "decoupled")
WEIGHT_DECAY_MODE_CODE = {"l2": 0, "decoupled": 1}  # weight_decay_mode of the native ops


def check_weight_decay_mode(kind: str, mode: Any) -> str:
  """Validate ``weight_decay_mode`` for optimizer ``kind`` ("sgd" ... "momentum"); returns it."""
  if mode not in WEIGHT_DECAY_MODES:
    raise ValueError(f"weight_decay_mode must be one of {', '.join(WEIGHT_DECAY_MODES)}, "
                     f"got {mode!r}")
  if mode == "decoupled" and kind == "ftrl":
    raise ValueError("weight_decay_mode='decoupled' does not apply to ftrl: its weight is a closed "
                     "form of z; use its l2 / l2_shrinkage (or weight_decay_mode='l2')")
  return mode


def decoupled_decay(kind: str, cfg: Mapping[str, Any]) -> bool:
  """Whether an update of ``kind`` with ``cfg`` runs the decoupled kernels: decoupled mode, a
  nonzero decay, and a kind other than SGD (whose decoupled update is its L2 update)."""
  return cfg.get("weight_decay_mode", "l2") == "decoupled" and \
      float(cfg.get("weight_decay", 0.0)) != 0.0 and kind != "sgd"


def decay_keep(lr: float, weight_decay: float) -> float:
  """The factor 1 - lr * weight_decay of a decoupled update as the kernels form it, one fp32 fma
  of the fp32 lr and decay: the product is exact in float64, and the difference is rounded to
  float64 and then to fp32 (the fma's result unless the float64 value is an exact fp32 tie)."""
  lr32, wd32 = np.float32(lr), np.float32(weight_decay)
  return float(np.float32(1.0 - float(lr32) * float(wd32)))


def check_state_dtype(kind: str, state_dtype: torch.dtype) -> torch.dtype:
  """Validate the storage dtype of an optimizer's element-wise state; returns it."""
  if state_dtype not in (torch.float32, torch.bfloat16):
    raise ValueError(
        f"optimizer state_dtype must be torch.float32 or torch.bfloat16, not {state_dtype} "
        "(fp16 cannot hold it: an Adagrad accumulator can pass 65504 and Adam's v underflows)")
  entry = OPTIMIZERS[kind]
  if state_dtype == torch.bfloat16 and not entry.slots:
    raise ValueError(f"state_dtype=torch.bfloat16 needs an optimizer with state: {kind} has none")
  if state_dtype == torch.bfloat16 and not entry.elementwise_state:
    raise ValueError(f"state_dtype=torch.bfloat16 does not apply to {kind}: its one fp32 word "
                     "per row stays fp32")
  return state_dtype


def state_slots(kind: str, weight: torch.Tensor, state_dtype: torch.dtype,
                row_dtype: torch.dtype, initial_accumulator_value: float,
                alloc: Callable[..., torch.Tensor] = torch.full) -> List[torch.Tensor]:
  """The state of one ``[rows, width]`` table, slot by slot: element-wise slots in
  ``state_dtype``, per-row slots in ``row_dtype``.  ``alloc(shape, value, dtype=, device=)``
  makes each one (default ``torch.full``; a bf16 start value is the round-to-nearest of it)."""
  rows, width = weight.shape
  return [alloc((rows,) if s.per_row else (rows, width),
                initial_accumulator_value if s.accumulator else 0.0,
                dtype=row_dtype if s.per_row else state_dtype, device=weight.device)
          for s in OPTIMIZERS[kind].slots]
