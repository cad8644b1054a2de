"""Decoupled (AdamW-style) weight decay, ``weight_decay_mode="decoupled"``, for the embedding
optimizers and the dense optimizers, against float64.

With lambda = ``weight_decay`` and lr the learning rate, a decoupled update of a touched row is
``w = (1 - lr * lambda) * w - lr * u``: the weight is scaled first (the kernels' fp32
``fmaf(-lr, lambda, 1)``, one rounding of the product), then the kind's step ``u`` from the
undecayed gradient.  The state (Adagrad's accumulator, Adam's moments, the row words of the
row-wise kinds) never sees the decay.  SGD's decoupled update is its L2 update; FTRL has no
decoupled mode.

The float64 model (:func:`decoupled_table_step`) sums each touched row's gradient from its id
occurrences within the bound of ``optim_reference.table_step``, scales the weight by the exact
``1 - lr * lambda`` (bound: two roundings, the factor and the product), and applies the kind's
float64 step with the bounds of ``optim_reference.row_update`` (row-wise Adam:
``test_rowwise_adam.rowwise_adam_update``).  It plugs into the driver of
``test_fused_optimizers.py`` as a ``Spec``, so every step checks every state slot of every shard,
16-bit tables and bf16 state at their rounding keys, and bit-identical untouched rows.

CPU (no GPU):
- argument validation: the mode in ``set_optimizer``, ``SparseRowOptimizer``, the dense
  optimizer config and ``HybridTrainer``; ``ftrl`` with ``"decoupled"`` raises;
- ``SparseRowOptimizer`` on fp32 / bf16 / fp16 tables and bf16 state against the model;
- the plan interpreter at world sizes 1-8 on whole, column-sliced and row-sliced tables;
- SGD: ``"decoupled"`` is bit-identical to ``"l2"`` and launches the same update;
- dry updates leave tables and state bit-identical;
- a modelled defect of the "device" update (the decay added to the gradient, as in L2 mode)
  fails with the table and row named;
- ``HybridTrainer``'s dense AdamW / Adam / Adagrad / SGD with decay against ``torch.optim``.

GPU (one H100):
- every kind on every route (occurrence-balanced, per-row with 4 or 1 columns per lane, row
  slices) at world sizes 2-8 on one GPU through the kernel-authoritative mirror harness of
  ``test_kernel_conformance.py``, on fp32 / bf16 / fp16 tables with fp32 or bf16 state; this
  module's census asserts that each case launched the route, dtypes and decay mode it claims;
- world 1: the same routes on the engine, and offloaded tables through the HBM row cache; the
  cached run equals the uncached one bit for bit;
- SGD's decoupled update bit-identical to L2 on the kernels; dry updates move nothing;
- the dense kernels (``dense_sgd`` / ``dense_adagrad`` / ``dense_adam``) against float64 in both
  modes, and the pad elements of the flat buffers stay zero;
- ``DLRMTrainStep`` against ``HybridTrainer`` with AdamW on the tables and the MLPs over three
  steps.
"""
import collections
import functools
import inspect

import numpy as np
import pytest
import torch

import distributed_embeddings_b200 as de
from distributed_embeddings_b200.ops._native import OPT_EMIT
from distributed_embeddings_b200.parallel import dry_run
from distributed_embeddings_b200.parallel.embedding_optimizers import (BY_CODE, OPTIMIZERS,
                                                                        decay_keep)
from distributed_embeddings_b200.parallel.hybrid import SparseRowOptimizer
from optim_reference import TINY, U, _e_sum, f32, row_update  # pylint: disable=wrong-import-order
import test_fused_optimizers as tfo  # pylint: disable=wrong-import-order
import test_rowwise_adam  # pylint: disable=wrong-import-order
import test_update_conformance as tur  # pylint: disable=wrong-import-order
from test_kernel_conformance import HostDevice  # pylint: disable=wrong-import-order

WD = tfo.WD  # 0.5: a decay applied the wrong way misses the bounds by orders of magnitude
# the kinds whose decoupled update has kernels of its own
KINDS = ("adagrad", "rowwise_adagrad", "adam", "rowwise_adam")
MODE = {"weight_decay_mode": "decoupled"}


# ------------------------------------------------------------------ float64 model
def decoupled_table_step(kind, weights, state, occ_rows, occ_vals, scale, lr, t, cfg):
  """float64 result of one lazy decoupled step of ``kind`` on one table, with bounds: the
  contract of ``optim_reference.table_step`` (state ``[rows, W]``, per-row slots ``[rows]``;
  untouched rows get a bound of zero).  Returns (out, bound, touched)."""
  w = torch.as_tensor(np.asarray(weights, dtype=np.float64))
  rows = w.shape[0]
  occ_rows = np.asarray(occ_rows, dtype=np.int64)
  vals = torch.as_tensor(np.asarray(occ_vals, dtype=np.float64))
  s, wd = f32(scale), f32(cfg["weight_decay"])
  st = [torch.as_tensor(np.asarray(x, dtype=np.float64)) for x in state]
  touched = np.zeros(rows, dtype=bool)
  touched[occ_rows] = True
  idx = torch.as_tensor(np.nonzero(touched)[0])
  occ = torch.as_tensor(occ_rows)
  gsum = torch.zeros_like(w).index_add_(0, occ, vals)
  gabs = torch.zeros_like(w).index_add_(0, occ, vals.abs())
  n_occ = torch.zeros(rows, dtype=torch.float64).index_add_(
      0, occ, torch.ones(len(occ_rows), dtype=torch.float64))
  g = s * gsum[idx]
  e_g = _e_sum(s, n_occ[idx], gabs[idx]) + TINY  # the sum in any order, then the scale
  wk = (1.0 - f32(lr) * wd) * w[idx]  # exact factor; the kernel rounds it and the product
  e_wk = 2.05 * U * wk.abs()
  sel = [x[idx] for x in st]
  if kind == "rowwise_adam":
    o, b = test_rowwise_adam.rowwise_adam_update(wk, g, e_g, sel[0], sel[1], lr, t, cfg)
  else:
    o, b = row_update(kind, wk, g, e_g, sel[0] if sel else None,
                      sel[1] if len(sel) > 1 else None, lr, t, cfg)
  b["p"] = b["p"] + 1.05 * e_wk
  out = {"p": w.clone()}
  bound = {"p": torch.zeros_like(w)}
  for k, x in zip(("s0", "s1"), st):
    out[k], bound[k] = x.clone(), torch.zeros_like(x)
  for k in o:
    out[k][idx] = o[k]
    bound[k][idx] = b[k]
  return out, bound, touched


class DecoupledSpec(tfo.Spec):
  """The driver's ``Spec`` of ``kind`` with ``weight_decay_mode="decoupled"``: the state of the
  kind's own spec, the decoupled float64 model (SGD: the L2 model, the same update)."""

  def __init__(self, kind):
    super().__init__(kind)
    self.base = test_rowwise_adam.SPEC if kind == "rowwise_adam" else tfo.SPECS[kind]

  def opt(self, case):
    return dict(self.base.opt(case), **MODE)

  def initial(self, rows, width, sdt):
    return self.base.initial(rows, width, sdt)

  def model(self, case, before, state, occ, step, scale):
    if self.kind == "sgd":
      return self.base.model(case, before, state, occ, step, scale)
    cfg = {"eps": OPTIMIZERS[self.kind].eps, "beta1": case.get("beta1", 0.9),
           "beta2": case.get("beta2", 0.999), "weight_decay": case.get("wd", 0.0)}
    return decoupled_table_step(self.kind, before, state, occ[0], occ[1], scale,
                                case["lrs"][step], step + 1, cfg)


SPECS = {k: DecoupledSpec(k) for k in ("sgd",) + KINDS}


# ------------------------------------------------------------------ census of update launches
# (route, kind, table dtype, state dtype, decay mode) of every segment_update the interpreter ran
CENSUS = collections.Counter()
_DT = {0: "fp32", 1: "bf16", 2: "fp16"}


@pytest.fixture(autouse=True)
def _count_updates(monkeypatch):
  """Record every ``segment_update`` of the interpreter (which the mirror harness also runs as
  its oracle before each kernel replay, with the same arguments)."""
  orig = dry_run.DryOps.segment_update
  sig = inspect.signature(orig)

  @functools.wraps(orig)
  def counted(self, *args, **kwargs):
    a = sig.bind(self, *args, **kwargs)
    a.apply_defaults()
    a = a.arguments
    if a["kind"] != OPT_EMIT:
      if a["scratch"] is not None and a["vec4"] and a["max_width"] <= 128:
        route = "balanced"
      else:
        route = "per-row " + ("vec4" if a["vec4"] else "vec1")
      kind = BY_CODE[a["kind"]]
      half = bool(a["state_dtype"]) and kind.elementwise_state
      mode = "decoupled" if int(a["weight_decay_mode"]) == 1 and a["weight_decay"] else "l2"
      CENSUS[(route, kind.name, _DT[int(a["table_dtype"])], "bf16" if half else "fp32",
              mode)] += 1
    return orig(self, *args, **kwargs)
  monkeypatch.setattr(dry_run.DryOps, "segment_update", counted)


def _census_delta(before):
  return {k: v - before.get(k, 0) for k, v in CENSUS.items() if v - before.get(k, 0)}


def _state_tag(kind, sdt):
  return "bf16" if sdt == torch.bfloat16 and OPTIMIZERS[kind].elementwise_state else "fp32"


def _expect_census(delta, kind, route, tdt, sdt, mode="decoupled"):
  """``delta`` holds launches of ``kind`` on ``route`` (None: any route) with the given dtypes and
  decay mode, and none in another mode."""
  key = (kind, tur._DT[tdt], _state_tag(kind, sdt), mode)
  assert any(k[1:] == key and route in (None, k[0]) for k in delta), (route, key, delta)
  other = {k for k in delta if k[4] != mode}
  assert not other, f"launches in another decay mode: {sorted(other)}"


# ------------------------------------------------------------------ CPU: arguments
def _layer():
  return de.DistributedEmbedding([{"input_dim": 10, "output_dim": 8, "combiner": "sum"}],
                                 device="cpu", backend="torch", world_size=1, rank=0)


def test_embedding_arguments():
  d = _layer()
  for kind in ("sgd",) + KINDS:
    d.set_optimizer(kind, lr=0.1, weight_decay=0.1, weight_decay_mode="decoupled")
    assert d._fused_optimizer["weight_decay_mode"] == "decoupled"
    d.set_optimizer(kind, lr=0.1)
    assert d._fused_optimizer["weight_decay_mode"] == "l2"
  d.set_optimizer("ftrl", lr=0.1, weight_decay=0.1, weight_decay_mode="l2")
  for bad in ("L2", "adamw", None, 1):
    with pytest.raises(ValueError, match="weight_decay_mode must be one of l2, decoupled"):
      d.set_optimizer("adam", lr=0.1, weight_decay=0.1, weight_decay_mode=bad)
  with pytest.raises(ValueError, match="does not apply to ftrl"):
    d.set_optimizer("ftrl", lr=0.1, weight_decay_mode="decoupled")
  p = torch.nn.Parameter(torch.zeros(10, 8))
  SparseRowOptimizer([p], "adam", weight_decay=0.1, weight_decay_mode="decoupled")
  with pytest.raises(ValueError, match="does not apply to ftrl"):
    SparseRowOptimizer([p], "ftrl", weight_decay_mode="decoupled")
  with pytest.raises(ValueError, match="weight_decay_mode must be one of"):
    SparseRowOptimizer([p], "adagrad", weight_decay_mode="decoupledd")


def test_dense_arguments():
  from distributed_embeddings_b200.models.dense_optimizer import (decay_args,
                                                                  dense_optimizer_config)
  from distributed_embeddings_b200.models.trainer import HybridTrainer
  from test_dense_optimizers import _small_dlrm  # pylint: disable=import-outside-toplevel
  for kind in ("sgd", "adagrad", "adam"):
    cfg = dense_optimizer_config(kind)
    assert cfg["weight_decay"] == 0.0 and cfg["weight_decay_mode"] == "l2"
    assert decay_args(cfg) == ()  # the ops launch with today's arguments
    cfg = dense_optimizer_config(kind, {"weight_decay": 0.25, "weight_decay_mode": "decoupled"})
    assert decay_args(cfg) == (0.25, 1)
    assert decay_args(dense_optimizer_config(kind, {"weight_decay": 0.25})) == (0.25, 0)
    with pytest.raises(ValueError, match="weight_decay_mode must be one of"):
      dense_optimizer_config(kind, {"weight_decay": 0.25, "weight_decay_mode": "adamw"})
    with pytest.raises(ValueError, match="weight_decay must be >= 0"):
      dense_optimizer_config(kind, {"weight_decay": -1.0})
  with pytest.raises(ValueError, match="takes no argument"):
    dense_optimizer_config("sgd", {"weight_decay": 0.1, "beta1": 0.5})
  with pytest.raises(ValueError, match="decoupled decay is for momentum=0"):
    HybridTrainer(_small_dlrm(0), lr=0.1, momentum=0.9,
                  dense_optimizer_kwargs={"weight_decay": 0.1, "weight_decay_mode": "decoupled"})
  HybridTrainer(_small_dlrm(0), lr=0.1, momentum=0.9, dense_optimizer_kwargs={"weight_decay": 0.1})


# ------------------------------------------------------------------ CPU: SparseRowOptimizer
_TABLE_STATE = [(torch.float32, torch.float32), (torch.bfloat16, torch.float32),
                (torch.float16, torch.float32), (torch.float32, torch.bfloat16),
                (torch.bfloat16, torch.bfloat16)]


@pytest.mark.parametrize("tdt,sdt", _TABLE_STATE, ids=lambda x: str(x)[6:])
@pytest.mark.parametrize("kind", KINDS)
def test_sparse_row_optimizer_against_float64(kind, tdt, sdt):
  """Three steps on different touched sets (one at a lower lr): the touched rows and every state
  slot within 3x the model's bounds (torch fp32 ops without fma), 16-bit values at the
  stochastic rounding of a value within them at their (step, row, column) keys, untouched rows
  bit-identical."""
  if sdt == torch.bfloat16 and not OPTIMIZERS[kind].elementwise_state:
    pytest.skip("one fp32 word per row: no bf16 state")
  rows, width = 60, 12
  gen = torch.Generator().manual_seed(50)
  p = torch.nn.Parameter(torch.randn(rows, width, generator=gen).to(tdt))
  # betas exact in fp32, and 1 - beta too: the torch optimizer takes its constants in float64
  case = {"wd": WD, "lrs": [0.05, 0.05, 0.02], "beta1": 0.875, "beta2": 1 - 2.0**-10,
          "table_dtype": tdt, "state_dtype": sdt}
  spec = SPECS[kind]
  opt = SparseRowOptimizer([p], kind, lr=0.05, weight_decay=WD, beta1=case["beta1"],
                           beta2=case["beta2"], state_dtype=sdt, **MODE)
  state = spec.initial(rows, width, sdt)
  for step, lr in enumerate(case["lrs"]):
    opt.set_lr(lr)
    idx = torch.randperm(rows, generator=gen)[:rows // 2 - 7 * step]
    vals = tfo._grad_values(gen, (len(idx), width)).to(tdt)
    before = p.detach().float().numpy().copy()
    p.grad = torch.sparse_coo_tensor(idx[None], vals, (rows, width))
    opt.step()
    out, bound, touched = spec.model(case, before, state, (idx.numpy(), vals.double().numpy()),
                                     step, 1.0)
    slots = [s.float().numpy() for s in opt.state[0]]
    sh = {"rank": 0, "table": 0, "rows": np.arange(rows), "cols": (0, width),
          "keys": np.arange(rows), "slots": slots}
    tfo._check_shard(case, spec, 0, step, sh, out, bound, touched,
                     p.detach().float().numpy(), 3.0)
    state = [s.copy() for s in slots]


def test_model_differs_from_l2():
  """The decoupled model and the L2 model of the same step disagree far outside the bounds (the
  decay divided by the adaptive denominator, or not), so the checks can tell the modes apart."""
  from optim_reference import table_step, worst_table_ratio
  gen = torch.Generator().manual_seed(3)
  w = torch.randn(30, 8, generator=gen).numpy()
  occ_rows = np.arange(0, 30, 2)
  occ_vals = tfo._grad_values(gen, (len(occ_rows), 8)).double().numpy()
  cfg = {"eps": 1e-7, "beta1": 0.9, "beta2": 0.999, "weight_decay": WD}
  for kind in ("adagrad", "rowwise_adagrad", "adam"):
    state = tfo._initial_state(kind, 30, 8)
    out, bound, _ = decoupled_table_step(kind, w, state, occ_rows, occ_vals, 1.0, 0.05, 1, cfg)
    l2, _, _ = table_step(kind, w, state, occ_rows, occ_vals, 1.0, 0.05, 1, cfg)
    assert worst_table_ratio(out, bound, {k: v.numpy() for k, v in out.items()}) == 0.0
    assert worst_table_ratio(out, bound, {k: v.numpy() for k, v in l2.items()}) > 100, kind


# ------------------------------------------------------------------ CPU: plan interpreter
# (world, kind, plan, table dtype, state dtype): whole tables (balanced / per-row vec4), column
# slices off the 4-column grid (per-row vec1), row slices fed ids outside the slice
_INTERP = [
    (1, "adagrad", "balanced", torch.float32, torch.float32),
    (2, "rowwise_adam", "per-row vec1", torch.float32, torch.bfloat16),
    (3, "adam", "rows", torch.bfloat16, torch.float32),
    (4, "rowwise_adagrad", "per-row vec4", torch.float32, torch.float32),
    (5, "adam", "per-row vec1", torch.float16, torch.bfloat16),
    (6, "rowwise_adagrad", "rows", torch.float32, torch.float32),
    (7, "adagrad", "per-row vec1", torch.bfloat16, torch.bfloat16),
    (8, "rowwise_adam", "balanced", torch.float16, torch.float32),
]


def _plan(plan):
  return tur.ROW_SLICES if plan == "rows" else tur.PLANS[plan]


def _route(plan):
  """The route a plan's launches take (row slices: whichever the plan gives the tables)."""
  return None if plan == "rows" else plan


@pytest.mark.parametrize("world,kind,plan,tdt,sdt", _INTERP,
                         ids=[f"w{c[0]}-{c[1]}-{c[2].replace(' ', '_')}" for c in _INTERP])
def test_interpreter_against_float64(world, kind, plan, tdt, sdt):
  """The driver on the plain interpreter: three steps, every state slot of every shard."""
  case, kw = _plan(plan)
  case = dict(case, wd=WD, table_dtype=tdt, state_dtype=sdt, batch=24 * world)
  before = CENSUS.copy()
  tfo._run(case, kind, world, plan=kw, route="any", spec=SPECS[kind])
  _expect_census(_census_delta(before), kind, _route(plan), tdt, sdt)


def test_interpreter_sgd_decoupled_is_l2_bit_for_bit():
  case, kw = tur.PLANS["balanced"]
  case = dict(case, wd=WD, batch=96, lrs=[0.05, 0.02])
  before = CENSUS.copy()
  a = tfo._run(case, "sgd", 3, plan=kw, route="any", spec=SPECS["sgd"])
  assert set(_census_delta(before)) == {("balanced", "sgd", "fp32", "fp32", "l2")}
  b = tfo._run(case, "sgd", 3, plan=kw, route="any")
  for x, y in zip(tfo._weights(a, 3), tfo._weights(b, 3)):
    assert np.array_equal(x.view(np.uint32), y.view(np.uint32))


@pytest.mark.parametrize("kind", KINDS)
def test_interpreter_dry_updates_move_nothing(kind):
  """Dry (warm-up) updates turn the decay off with the rest of the update: tables and every
  state slot keep their bits."""
  case, kw = tur.PLANS["balanced"]
  case = dict(case, wd=WD, batch=48, lrs=[0.05])
  made = []

  def world_cls(n):
    made.append(dry_run.DryWorld(n))
    return made[-1]
  des = tfo._run(case, kind, 2, plan=kw, route="any", world_cls=world_cls, spec=SPECS[kind])
  w0 = tfo._weights(des, 2)
  s0 = [{m: [x.clone() for x in st] for m, st in d._engine.opt_state.items()} for d in des]
  ids, grad = tfo._draw(case, 7)
  for d in des:
    d._engine.dry_updates(True)

  def fn(r):
    out = des[r](tfo._as_inputs(case, ids, des[r].device, r * 24, (r + 1) * 24), concat=True)
    out.backward(grad[r * 24:(r + 1) * 24])
  dry_run.run_ranks(made[0], fn)
  for x, y in zip(w0, tfo._weights(des, 2)):
    assert np.array_equal(x.view(np.uint32), y.view(np.uint32))
  for d, before in zip(des, s0):
    for m, st in d._engine.opt_state.items():
      for x, y in zip(before[m], st):
        assert torch.equal(x, y)


class L2Device(HostDevice):
  """The interpreter as the "kernels", with the decay applied the L2 way (added to the gradient)
  while the engine asked for the decoupled update."""

  def __init__(self):
    super().__init__()
    self.hits = 0

  def op(self, name, rank):
    f = super().op(name, rank)
    if name != "segment_update":
      return f

    def run(*args):
      args = list(args)
      i = tur._ARGS.index("weight_decay_mode")
      if args[i] == 1:
        args[i] = 0
        self.hits += 1
      return f(*args)
    return run


@pytest.mark.parametrize("kind,world", [("adagrad", 2), ("rowwise_adam", 3)])
def test_decay_in_the_gradient_fails(kind, world):
  dev = L2Device()
  case, kw = tur.PLANS["balanced"]
  with pytest.raises(AssertionError, match=r"table \d+ (weight|state slot \d) row \d+"):
    tfo._run(dict(case, wd=WD, lrs=[0.05, 0.02]), kind, world, plan=kw, route="any",
             world_cls=tur._world(dev), slack=3.0, spec=SPECS[kind])
  assert dev.hits > 0


# ------------------------------------------------------------------ CPU: HybridTrainer dense
@pytest.mark.parametrize("kind,mode", [("adam", "decoupled"), ("adam", "l2"),
                                       ("adagrad", "l2"), ("adagrad", "decoupled"),
                                       ("sgd", "l2"), ("sgd", "decoupled")])
def test_hybrid_dense_decay_matches_torch_optim(kind, mode):
  """``HybridTrainer``'s dense step with decay against ``torch.optim``: AdamW for decoupled Adam,
  the optimizers' own ``weight_decay`` (L2) otherwise; decoupled Adagrad against the same
  AdamW-style scaling applied before ``torch.optim.Adagrad``'s step."""
  from distributed_embeddings_b200.models.trainer import HybridTrainer
  from test_dense_optimizers import _batch, _small_dlrm  # pylint: disable=import-outside-toplevel
  model, ref = _small_dlrm(0), _small_dlrm(0)
  lr, wd = 0.01, 0.1
  tr = HybridTrainer(model, lr=lr, embedding_optimizer="sgd", dense_optimizer=kind,
                     dense_optimizer_kwargs={"weight_decay": wd, "weight_decay_mode": mode})
  dense = [p for p in ref.parameters() if not getattr(p, "de_local", False)]
  tables = [p for p in ref.parameters() if getattr(p, "de_local", False)]
  pre = None
  if kind == "adam" and mode == "decoupled":
    opt = torch.optim.AdamW(dense, lr=lr, eps=1e-8, weight_decay=wd)
  elif kind == "adam":
    opt = torch.optim.Adam(dense, lr=lr, eps=1e-8, weight_decay=wd)
  elif kind == "adagrad":
    opt = torch.optim.Adagrad(dense, lr=lr, initial_accumulator_value=0.1, eps=1e-7,
                              weight_decay=0.0 if mode == "decoupled" else wd)
    pre = (1 - lr * wd) if mode == "decoupled" else None
  else:
    opt = torch.optim.SGD(dense, lr=lr, weight_decay=wd)
  topt = torch.optim.SGD(tables, lr=lr)
  for i in range(4):
    num, cat, lab = _batch(model.table_sizes, 32, 100 + i)
    tr.step(num, cat, lab)
    ref.zero_grad()
    torch.nn.functional.binary_cross_entropy_with_logits(ref(num, cat).float(), lab).backward()
    if pre is not None:
      with torch.no_grad():
        for p in dense:
          p.mul_(pre)
    opt.step()
    topt.step()
  for (n, a), b in zip([(n, p) for n, p in model.named_parameters()
                        if not getattr(p, "de_local", False)], dense):
    torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-4 * lr, msg=lambda m, n=n: f"{n}: {m}")


# ------------------------------------------------------------------ GPU
def _cuda():
  return torch.device("cuda", 0)


_WORLDS = (2, 3, 4, 8)
_HALF = [(torch.bfloat16, torch.float32), (torch.float16, torch.float32),
         (torch.float32, torch.bfloat16), (torch.bfloat16, torch.bfloat16),
         (torch.float16, torch.bfloat16)]
GPU_CASES = []
for _i, _k in enumerate(KINDS):
  for _j, _p in enumerate(("balanced", "per-row vec4", "per-row vec1", "rows")):
    GPU_CASES.append((_k, _p, _WORLDS[(_i + _j) % 4], torch.float32, torch.float32))
  for _j, (_t, _s) in enumerate(_HALF):
    if _s == torch.bfloat16 and not OPTIMIZERS[_k].elementwise_state:
      continue
    GPU_CASES.append((_k, ("balanced", "per-row vec4", "per-row vec1", "rows")[(_i + _j) % 4],
                      _WORLDS[(_i + 2 * _j) % 4], _t, _s))


@pytest.mark.gpu
@pytest.mark.parametrize("kind,plan,world,tdt,sdt", GPU_CASES,
                         ids=[f"{c[0]}-{c[1].replace(' ', '_')}-w{c[2]}-{str(c[3])[6:]}_table-"
                              f"{str(c[4])[6:]}_state" for c in GPU_CASES])
def test_gpu_sharded_against_float64(kind, plan, world, tdt, sdt):
  """One case on the kernels through the kernel-authoritative mirror harness, checked at the
  kernels' own bounds; the census must show the route, the dtypes and the decoupled mode."""
  case, kw = _plan(plan)
  case = dict(case, wd=WD, table_dtype=tdt, state_dtype=sdt)
  before = CENSUS.copy()
  tfo._run(case, kind, world, plan=kw, route="any", world_cls=tur._world(tur._gpu()), slack=1.0,
           spec=SPECS[kind])
  _expect_census(_census_delta(before), kind, _route(plan), tdt, sdt)


def test_gpu_cases_cover_every_kind_route_and_dtype():
  got = {(k, _route(p)) for k, p, _, _, _ in GPU_CASES}
  assert got == {(k, r) for k in KINDS for r in tur.ROUTES + (None,)}
  assert {(k, "rows") for k in KINDS} <= {(k, p) for k, p, _, _, _ in GPU_CASES}
  for k in KINDS:
    dts = {(t, _state_tag(k, s)) for kk, _, _, t, s in GPU_CASES if kk == k}
    want = {(t, "fp32") for t in (torch.float32, torch.bfloat16, torch.float16)}
    if OPTIMIZERS[k].elementwise_state:
      want |= {(t, "bf16") for t in (torch.float32, torch.bfloat16, torch.float16)}
    assert want <= dts, (k, want - dts)


_ONE = {"balanced": tfo.MIXED, "per-row vec4": tfo.WIDE, "per-row vec1": tfo.ODD}


@pytest.mark.gpu
@pytest.mark.parametrize("plan", list(_ONE))
@pytest.mark.parametrize("kind", KINDS)
def test_gpu_world1_routes_against_float64(kind, plan):
  """World 1 on the engine: hot rows across many 32-item chunks (``finalize_crossing_kernel``),
  rows touched only by zero gradients, ragged and mean inputs; the route is asserted."""
  tfo._run(dict(_ONE[plan], wd=WD, lrs=[0.05, 0.02]), kind, dev=_cuda(), spec=SPECS[kind],
           route=plan.replace(" ", "_").replace("-", "_"))


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ("sgd",) + KINDS)
def test_gpu_offloaded_against_float64(kind):
  """A host-resident table behind the HBM row cache, against float64 (the case of
  ``test_fused_optimizers.py``'s row-cache cases)."""
  case = tfo._case([(64, 16, "sum"), (6000, 16, "sum")], [0, 1, 1], [1, 2, 1], 512, wd=WD,
                   cache=2000, lrs=[0.05, 0.05], seed=8)
  tfo._run(case, kind, dev=_cuda(), spec=SPECS[kind])


def _pair_ids(step, b, big):
  """Ids of the offloaded table where every row is hit at most twice: each row's gradient is then
  summed exactly the same way on every route and chunking (a + b, in either order)."""
  g = torch.Generator().manual_seed(300 + step)
  rows = torch.randperm(big, generator=g)[:b]
  ids = torch.cat([rows[:b // 2], rows[:b - b // 2]])[torch.randperm(b, generator=g)]
  return ids.view(b, 1).to(torch.int32)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_gpu_cached_equals_uncached_bit_for_bit(kind):
  from test_offload_cache import BIG, SMALL, WAYS, _pair  # pylint: disable=import-outside-toplevel
  cached, plain = _pair(kind, 2 * WAYS * 16, input_table_map=(0, 1), weight_decay=WD, **MODE)
  for step in range(4):
    g = torch.Generator().manual_seed(400 + step)
    ids = [torch.randint(0, SMALL, (128, 1), generator=g, dtype=torch.int32).to(_cuda()),
           _pair_ids(step, 128, BIG).to(_cuda())]
    for d in (cached, plain):
      out = d(ids, concat=True)
      (out * torch.linspace(-1, 1, out.shape[1], device=_cuda())).sum().backward()
  torch.cuda.synchronize()
  for a, b in zip(cached.get_weights(), plain.get_weights()):
    assert np.array_equal(np.asarray(a).view(np.uint32), np.asarray(b).view(np.uint32))
  sc, sp = cached.get_optimizer_state(), plain.get_optimizer_state()
  for ta, tb in zip(sc["tables"], sp["tables"]):
    for a, b in zip(ta or [], tb or []):
      assert np.array_equal(np.asarray(a).view(np.uint32), np.asarray(b).view(np.uint32))


@pytest.mark.gpu
def test_gpu_sgd_decoupled_is_l2_bit_for_bit():
  case = dict(tfo.ODD, wd=WD, lrs=[0.05, 0.02])  # per-row route: a deterministic sum order
  a = tfo._run(case, "sgd", dev=_cuda(), spec=SPECS["sgd"])
  b = tfo._run(case, "sgd", dev=_cuda())
  for x, y in zip(a[0].get_weights(), b[0].get_weights()):
    assert np.array_equal(np.asarray(x).view(np.uint32), np.asarray(y).view(np.uint32))


@pytest.mark.gpu
@pytest.mark.parametrize("kind,tdt", [("adam", torch.bfloat16), ("rowwise_adagrad", torch.float32),
                                      ("rowwise_adam", torch.float16),
                                      ("adagrad", torch.float32)])
def test_gpu_dry_updates_move_nothing(kind, tdt):
  # one table: at world 1 the driver keys 16-bit rounding from the first table's key base
  case = tfo._case([(600, 32, "sum")], [0, 0], [1, 2], 512, edges=True, wd=WD, table_dtype=tdt,
                   seed=5)
  des = tfo._run(case, kind, dev=_cuda(), spec=SPECS[kind])
  d = des[0]
  w0 = [np.asarray(w).copy() for w in d.get_weights()]
  s0 = {m: [x.clone() for x in st] for m, st in d._engine.opt_state.items()}
  ids, grad = tfo._draw(case, 5)
  d._engine.dry_updates(True)
  out = d(tfo._as_inputs(case, ids, _cuda()), concat=True)
  out.backward(grad.to(out.device))
  torch.cuda.synchronize()
  d._engine.dry_updates(False)
  for a, b in zip(w0, d.get_weights()):
    assert np.array_equal(a.view(np.uint32), np.asarray(b).view(np.uint32))
  for m, st in d._engine.opt_state.items():
    for x, y in zip(s0[m], st):
      assert torch.equal(x, y)


# ---- dense kernels
def _dense_model(kind, p, g, s0, s1, lr, t, cfg, mode):
  """float64 result of one dense update with decay, and its bounds."""
  wd = f32(cfg["weight_decay"])
  w = p.double().view(-1, 1)
  gd = g.double().view(-1, 1)
  if kind == "sgd":
    gp = gd + wd * w
    out = w - f32(lr) * gp
    e = 1.05 * (f32(lr) * U * gp.abs() + U * out.abs()) + TINY
    return {"p": out.view(-1)}, {"p": e.view(-1)}
  st0 = s0.double().view(-1, 1)
  st1 = None if s1 is None else s1.double().view(-1, 1)
  if mode == "l2":
    gp = gd + wd * w
    o, b = row_update(kind, w, gp, U * gp.abs() + TINY, st0, st1, lr, t, cfg)
  else:
    wk = (1.0 - f32(lr) * wd) * w
    o, b = row_update(kind, wk, gd, torch.zeros_like(gd), st0, st1, lr, t, cfg)
    b["p"] = b["p"] + 1.05 * 2.05 * U * wk.abs()
  return {k: v.view(-1) for k, v in o.items()}, {k: v.view(-1) for k, v in b.items()}


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["l2", "decoupled"])
@pytest.mark.parametrize("kind", ["sgd", "adagrad", "adam"])
@pytest.mark.parametrize("n", [4, 4 * 1001, 4 * (3 * 2**20 + 1)])
def test_gpu_dense_kernels_against_float64(kind, mode, n):
  from distributed_embeddings_b200.ops import _native
  from test_dense_optimizers import make_inputs  # pylint: disable=import-outside-toplevel
  ops = _native.require()
  dev = _cuda()
  code = {"l2": 0, "decoupled": 1}[mode]
  for t in ((1, 2, 1000) if kind == "adam" else (1,)):
    cfg = {"eps": 1e-8 if kind == "adam" else 1e-7, "beta1": 0.9, "beta2": 0.999,
           "weight_decay": 0.3}
    p, g, s0, s1 = make_inputs("adagrad" if kind == "sgd" else kind, n, 17 + t, dev)
    inp = [x.clone() if x is not None else None for x in (p, g, s0, s1)]
    lr = torch.full((1,), 0.01, dtype=torch.float32, device=dev)
    p16 = torch.empty(n, dtype=torch.bfloat16, device=dev)
    if kind == "sgd":
      ops.dense_sgd(p, p16, g, lr, 1.0, cfg["weight_decay"], code)
    elif kind == "adagrad":
      ops.dense_adagrad(p, p16, g, s0, lr, cfg["eps"], cfg["weight_decay"], code)
    else:
      step = torch.full((1,), float(t), dtype=torch.float32, device=dev)
      ops.dense_adam(p, p16, g, s0, s1, lr, step, cfg["beta1"], cfg["beta2"], cfg["eps"],
                     cfg["weight_decay"], code)
    torch.cuda.synchronize()
    out, bound = _dense_model(kind, *[x.cpu() if x is not None else None for x in inp], 0.01, t,
                              cfg, mode)
    got = {"p": p.cpu(), "s0": s0.cpu(), "s1": None if s1 is None else s1.cpu()}
    for k in out:
      err = (got[k].double() - out[k]).abs()
      assert torch.isfinite(got[k]).all() and bool((err <= bound[k]).all()), \
          (kind, mode, t, k, float((err / bound[k]).max()))
    assert torch.equal(p16.cpu(), p.cpu().bfloat16()) and bool((g == 0).all())


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["sgd", "adagrad", "adam"])
def test_gpu_dense_decay_pad_elements_stay_zero(kind):
  from distributed_embeddings_b200.models.dlrm_fast import DLRMTrainStep
  from test_dense_optimizers import (  # pylint: disable=import-outside-toplevel
      _batch, _dlrm, _pad_mask)
  dev = _cuda()
  sizes = [100 + 7 * i for i in range(26)]
  num, cat, lab = _batch(sizes, 256, 6, dev)
  decay = {"weight_decay": 0.1, "weight_decay_mode": "decoupled"}
  t = DLRMTrainStep(_dlrm(5, dev, sizes=sizes), lr=0.01, embedding_optimizer=kind,
                    dense_optimizer=kind, dense_optimizer_kwargs=decay,
                    embedding_optimizer_kwargs=decay)
  p0 = t.p32.clone()
  for _ in range(3):
    t.step(num, torch.stack([c.int() for c in cat]), lab)
  torch.cuda.synchronize()
  pad = _pad_mask(t)
  assert int(pad.sum()) > 0 and bool((t.p32 != p0)[~pad].any())
  assert bool((t.p32[pad] == 0).all()) and bool((t.p16[pad] == 0).all())
  init = 0.1 if kind == "adagrad" else 0.0
  for s in t.dense_opt.state:
    assert bool((s[pad] == init).all())


@pytest.mark.gpu
def test_gpu_dlrm_step_adamw_matches_hybrid():
  """AdamW on the tables and the MLPs, three steps of ``DLRMTrainStep`` against ``HybridTrainer``:
  the loss of every step; after the first step the moments of every dense parameter and table at
  0.08 relative error (the one-step tolerance of ``test_dense_optimizers.py``; the bf16 paths
  drift apart over later steps); and every step of the fast trainer follows its own moments,
  ``p = (1 - lr wd) p - lr m_hat / (sqrt(v_hat) + eps)``, on the dense parameters and on the
  touched table rows, while untouched rows keep their bits."""
  from distributed_embeddings_b200.models.dlrm_fast import DLRMTrainStep
  from distributed_embeddings_b200.models.trainer import HybridTrainer
  from test_dense_optimizers import (  # pylint: disable=import-outside-toplevel
      _batch, _dense_named, _dlrm, _rel)
  dev = _cuda()
  lr, wd = 0.002, 0.5
  ref, fast = _dlrm(0, dev), _dlrm(0, dev)
  fast.load_state_dict(ref.state_dict())
  fast.embedding.set_weights(ref.embedding.get_weights())
  decay = {"weight_decay": wd, "weight_decay_mode": "decoupled"}
  kw = dict(lr=lr, embedding_optimizer="adam", dense_optimizer="adam",
            embedding_optimizer_kwargs=decay, dense_optimizer_kwargs=decay)
  t_ref = HybridTrainer(ref, **kw)
  t_fast = DLRMTrainStep(fast, use_cuda_graph=False, **kw)
  keep = decay_keep(lr, wd)
  flat = lambda arrays: torch.cat([torch.as_tensor(np.asarray(a)).reshape(-1) for a in arrays])
  for step in range(1, 4):
    num, cat, lab = _batch(ref.table_sizes, 512, step, dev)
    cat = [c.int() for c in cat]
    w0 = [p.detach().clone() for _, p in _dense_named(fast)]
    e0 = fast.embedding.get_weights()
    loss_ref = t_ref.step(num, cat, lab)
    loss_fast = t_fast.step(num, torch.stack(cat), lab).clone()
    torch.cuda.synchronize()
    torch.testing.assert_close(loss_fast[0], loss_ref, rtol=2e-2, atol=2e-3)
    b1, b2 = 1 - 0.9**step, 1 - 0.999**step
    s_ref, s_fast = t_ref.dense_optimizer_state(), t_fast.dense_optimizer_state()
    assert s_ref["step"] == s_fast["step"] == step
    for (name, p), p0 in zip(_dense_named(fast), w0):
      m, v = (x.double() for x in s_fast["slots"][name])
      mr, vr = (x.double() for x in s_ref["slots"][name])
      if step == 1:
        assert _rel(m, mr) < 0.08 and _rel(v.sqrt(), vr.sqrt()) < 0.08, (name, step)
      want = p0.double() * keep - lr * (m / b1) / ((v / b2).sqrt() + 1e-8)
      torch.testing.assert_close(p.detach().double(), want, rtol=1e-5, atol=1e-3 * lr,
                                 msg=lambda msg, n=name: f"{n} step {step}: {msg}")
    e_ref, e_fast = ref.embedding.get_optimizer_state(), fast.embedding.get_optimizer_state()
    for j in range(2):
      a = flat([t[j] for t in e_fast["tables"]]).double()
      r = flat([t[j] for t in e_ref["tables"]]).double()
      if j == 1:
        a, r = a.sqrt(), r.sqrt()
      assert step > 1 or _rel(a, r) < 0.08, ("tables", j, step, _rel(a, r))
    for t, (w_before, w_after) in enumerate(zip(e0, fast.embedding.get_weights())):
      touched = np.zeros(len(w_before), dtype=bool)
      touched[cat[t].cpu().numpy()] = True
      wb, wa = np.asarray(w_before), np.asarray(w_after)
      assert np.array_equal(wb[~touched].view(np.uint32), wa[~touched].view(np.uint32))
      m, v = (torch.as_tensor(np.asarray(x)).double()[touched] for x in e_fast["tables"][t])
      want = torch.as_tensor(wb[touched]).double() * keep - lr * (m / b1) / ((v / b2).sqrt() +
                                                                            1e-8)
      torch.testing.assert_close(torch.as_tensor(wa[touched]).double(), want, rtol=1e-5,
                                 atol=1e-3 * lr, msg=lambda msg, t=t: f"table {t}: {msg}")
