"""Dense optimizer of the trainers: SGD, Adagrad, Adam or momentum SGD on the data-parallel
parameters (the MLPs and any replicated embedding tables).

The reference applies one optimizer to every trainable variable; ``dense_optimizer`` lets the
trainers do the same.  The math is that of the fused embedding update (``apply_update`` in
``ops/csrc/sparse_update_kernels.cu``), with the defaults of
:meth:`DistributedEmbedding.set_optimizer`:

* Adagrad: ``acc += g * g; p -= lr * g / (sqrt(acc) + eps)`` (``eps=1e-7``,
  ``initial_accumulator_value=0.1``);
* Adam: ``m = b1 m + (1 - b1) g; v = b2 v + (1 - b2) g^2;
  p -= lr * (m / (1 - b1^t)) / (sqrt(v / (1 - b2^t)) + eps)`` (``beta1=0.9``, ``beta2=0.999``,
  ``eps=1e-8``);
* momentum SGD (``torch.optim.SGD``, dampening 0): ``b = mu b + g; p -= lr * b``, or with
  ``nesterov`` ``p -= lr * (mu b + g)`` (``momentum=0.9``, ``nesterov=False``), each step one
  fp32 fma in this order.

Every kind takes ``weight_decay`` (lambda, default 0) and ``weight_decay_mode``: ``"l2"``
(default) adds ``lambda * p`` to the gradient before the update; ``"decoupled"`` (AdamW-style)
first scales ``p`` by the fp32 ``1 - lr * lambda`` and then applies the step of the undecayed
gradient, ``p = (1 - lr * lambda) * p - lr * u`` (momentum SGD's L2 decay passes through the
buffer, as ``torch.optim.SGD``'s ``weight_decay`` does).  SGD's update is
``p -= lr * (g + lambda * p)`` in both modes.  Unlike the lazy embedding optimizers, the decay
applies to every dense element (MLP weights, biases, replicated tables) on every step; pad elements
of the flat buffers stay 0.

The learning rate is the trainer's device-resident ``lr_t`` word and Adam's step count ``t`` is a
device-resident fp32 word advanced inside the step, so both follow a scheduler under CUDA-graph
replay.

Checkpoints have one format for every trainer: ``{"kind", "step", "slots"}`` where ``slots`` maps
each dense parameter name (``model.named_parameters()``) to its state tensors shaped like the
parameter (Adagrad ``[acc]``, Adam ``[m, v]``, momentum ``[b]``, SGD none) and ``step`` is Adam's
``t`` (0 for the kinds that keep no step count).
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence, Tuple

import torch
from torch import nn

from ..parallel.embedding_optimizers import (MOMENTUM_DEFAULTS, WEIGHT_DECAY_MODE_CODE,
                                              WEIGHT_DECAY_MODES, check_momentum_args)

KINDS = ("sgd", "adagrad", "adam", "momentum")
_DEFAULTS = {
    "sgd": {},
    "adagrad": {"eps": 1e-7, "initial_accumulator_value": 0.1},
    "adam": {"beta1": 0.9, "beta2": 0.999, "eps": 1e-8},
    "momentum": dict(MOMENTUM_DEFAULTS),
}
_DECAY = {"weight_decay": 0.0, "weight_decay_mode": "l2"}  # every kind


def dense_optimizer_config(kind: str, kwargs: Optional[dict] = None) -> dict:
  """``{"kind", **hyperparameters}`` with the defaults of the embedding optimizer filled in."""
  kind = str(kind).lower()
  if kind not in KINDS:
    raise ValueError(f"dense_optimizer must be one of {', '.join(KINDS)}, got {kind!r}")
  cfg = dict(_DEFAULTS[kind], **_DECAY)
  unknown = sorted(set(kwargs or {}) - set(cfg))
  if unknown:
    raise ValueError(f"dense optimizer {kind!r} takes no argument(s) {', '.join(unknown)}")
  kwargs = dict(kwargs or {})
  mode = kwargs.pop("weight_decay_mode", cfg["weight_decay_mode"])
  if mode not in WEIGHT_DECAY_MODES:
    raise ValueError(f"dense optimizer weight_decay_mode must be one of "
                     f"{', '.join(WEIGHT_DECAY_MODES)}, got {mode!r}")
  # nesterov stays a bool; every other hyperparameter is a number
  cfg.update({k: v if k == "nesterov" else float(v) for k, v in kwargs.items()})
  if kind == "momentum":
    check_momentum_args(cfg)
  if not cfg["weight_decay"] >= 0.0:
    raise ValueError(f"dense optimizer weight_decay must be >= 0, got {cfg['weight_decay']}")
  cfg["weight_decay_mode"] = mode
  cfg["kind"] = kind
  return cfg


def decay_args(cfg: dict) -> tuple:
  """The trailing ``(weight_decay, weight_decay_mode)`` of the dense ops, empty without decay
  (the launch then keeps the arguments and kernels of a run without decay)."""
  wd = cfg["weight_decay"]
  return (wd, WEIGHT_DECAY_MODE_CODE[cfg["weight_decay_mode"]]) if wd != 0.0 else ()


def slot_init(cfg: dict) -> List[float]:
  """Initial value of each state slot: Adagrad ``[acc]``, Adam ``[m, v]``, momentum ``[b]``, SGD
  none."""
  return {"sgd": [], "adagrad": [cfg.get("initial_accumulator_value")],
          "adam": [0.0, 0.0], "momentum": [0.0]}[cfg["kind"]]


def dense_named_parameters(model: nn.Module) -> List[Tuple[str, nn.Parameter]]:
  """The data-parallel parameters by name (model-parallel tables are tagged ``de_local``)."""
  return [(n, p) for n, p in model.named_parameters() if not getattr(p, "de_local", False)]


def check_state(cfg: dict, state: dict, names: Sequence[str]):
  if state.get("kind") != cfg["kind"]:
    raise ValueError(f"dense optimizer state of kind {state.get('kind')!r} cannot be loaded into "
                     f"a {cfg['kind']!r} dense optimizer")
  slots = state.get("slots", {})
  missing = sorted(set(names) - set(slots))
  if slot_init(cfg) and missing:
    raise ValueError(f"dense optimizer state misses parameter(s) {', '.join(missing)}")


class FlatDenseOptimizer:
  """Adagrad / Adam / momentum state laid out like a trainer's flat fp32 master buffer ``p32`` and
  the fused update over it (``dense_adagrad`` / ``dense_adam`` / ``dense_momentum``); SGD keeps no
  state and launches ``dense_sgd``.  Pad elements keep ``g = 0``, so they stay at ``p = 0`` and
  their state at its initial value."""

  def __init__(self, cfg: dict, p32: torch.Tensor):
    self.cfg = cfg
    self.kind = cfg["kind"]
    self.p32 = p32
    self.state = [torch.full_like(p32, v) for v in slot_init(cfg)]
    self.step_t = torch.zeros(1, dtype=torch.float32, device=p32.device) \
        if self.kind == "adam" else None

  def apply(self, ops, p16: torch.Tensor, g32: torch.Tensor, lr_t: torch.Tensor):
    """p32 update + ``p16 = bf16(p32)`` + ``g32 = 0``, one launch (Adam: plus the step word)."""
    c = self.cfg
    decay = decay_args(c)
    if self.kind == "sgd":
      ops.dense_sgd(self.p32, p16, g32, lr_t, 1.0, *decay)
    elif self.kind == "adagrad":
      ops.dense_adagrad(self.p32, p16, g32, self.state[0], lr_t, c["eps"], *decay)
    elif self.kind == "momentum":
      ops.dense_momentum(self.p32, p16, g32, self.state[0], lr_t, c["momentum"], c["nesterov"],
                         *decay)
    else:
      self.step_t.add_(1.0)  # device counter: the bias corrections stay right under graph replay
      ops.dense_adam(self.p32, p16, g32, self.state[0], self.state[1], lr_t, self.step_t,
                     c["beta1"], c["beta2"], c["eps"], *decay)

  def snapshot(self) -> List[torch.Tensor]:
    return [s.clone() for s in self.state] + ([self.step_t.clone()] if self.step_t is not None
                                              else [])

  def restore(self, snap: Sequence[torch.Tensor]):
    for dst, src in zip(self.state + ([self.step_t] if self.step_t is not None else []), snap):
      dst.copy_(src)

  def _slot_view(self, s: torch.Tensor, p: torch.Tensor) -> torch.Tensor:
    """The elements of ``s`` that hold the state of parameter ``p`` (a view into ``p32``)."""
    if p.untyped_storage().data_ptr() != self.p32.untyped_storage().data_ptr():
      raise RuntimeError("dense parameter does not live in the flat master buffer")
    return s.as_strided(p.shape, p.stride(), p.storage_offset())

  def state_dict(self, model: nn.Module) -> Dict:
    step = int(round(float(self.step_t.item()))) if self.step_t is not None else 0
    slots = {n: [self._slot_view(s, p).clone() for s in self.state]
             for n, p in dense_named_parameters(model)} if self.state else {}
    return {"kind": self.kind, "step": step, "slots": slots}

  def load_state_dict(self, model: nn.Module, state: Dict):
    named = dense_named_parameters(model)
    check_state(self.cfg, state, [n for n, _ in named])
    if self.state:
      for n, p in named:
        for s, src in zip(self.state, state["slots"][n]):
          self._slot_view(s, p).copy_(src)
    if self.step_t is not None:
      self.step_t.fill_(float(state.get("step", 0)))
