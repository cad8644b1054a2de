"""Every embedding optimizer's fused update at world sizes 2-8 on one GPU, against float64.

SGD with weight decay, Adagrad, row-wise Adagrad, Adam, row-wise Adam and FTRL (Keras defaults,
and every term with ``l1`` large enough to zero weights and ``lr_power = -0.3``) update sharded
tables through the driver of ``test_fused_optimizers.py``: every rank of a plan runs in one
process, and the engines' ops are replayed on the kernels by the mirror harness of
``test_kernel_conformance.py`` in its kernel-authoritative mode.  There the interpreter runs each
``segment_update`` first as the oracle for addressing, the kernel's touched rows become the
tables and state of the run, and rows no key touched must stay bit-identical.  After every step
the float64 models (``optim_reference.py``, ``test_rowwise_adam.py``, ``test_ftrl.py``) check
the kernel's numbers at the kernels' own bounds, shard by shard:

* every state slot, read from each rank's ``opt_state`` at the shard's rows: Adagrad's
  accumulator, row-wise Adagrad's and row-wise Adam's row word of each column slice (the mean
  over that slice's columns), Adam's m and v and its step on every rank, FTRL's n and z;
* 16-bit tables and bf16 state at the kernel's rounding key: ``key_base`` of the rank's local
  table plus the row inside it, and the column inside the slice;
* three steps with different touched sets and a learning-rate change (FTRL: one step at lr = 0,
  which must leave everything bit-identical).

Plans: whole tables (the occurrence-balanced route, width <= 128, or the per-row route with four
columns per lane), column slices whose widths are not multiples of 4 (the per-row route with one
column per lane) and row slices fed ids outside the slice.  Power-law ids give hot rows whose
segments cross many 32-item chunks.  Samples hold at most two ids, so the lookups and gradient
exchanges stay bit-exact on the non-dyadic values the updates produce.  Each case asserts the
routes and dtypes it took from the replay census, and a CPU test checks that the cases together
cover every kind on every route and every 16-bit table / state combination, on row-sliced
tables too.

CPU (no GPU): the kernel-authoritative mode with the interpreter standing in for the kernels
passes at the interpreter's bounds, and four modelled defects of the "device" update fail with
the table and row named: a touched element moved by a few times its bound, a write to a row no
key touched, table descriptors whose ``key_base`` is off by one (wrong 16-bit rounding keys), and
row-wise Adam's v not written back.  A few multi-step cases run the same driver through the plain
interpreter at world 5-8.
"""
import collections
import inspect

import numpy as np
import pytest
import torch

from distributed_embeddings_b200.ops._native import OPT_EMIT, TABLE_DESC
from distributed_embeddings_b200.parallel import dry_run
from distributed_embeddings_b200.parallel.embedding_optimizers import OPTIMIZERS
import test_fused_optimizers as tfo  # pylint: disable=wrong-import-order
import test_ftrl  # pylint: disable=wrong-import-order
import test_rowwise_adam  # pylint: disable=wrong-import-order
from test_kernel_conformance import (  # pylint: disable=wrong-import-order
    REPLAYED, CudaDevice, HostDevice, MirrorWorld)

WD = tfo.WD
# name -> (optimizer kind, driver spec, extra case entries)
KINDS = {
    "sgd": ("sgd", tfo.SPECS["sgd"], {"wd": WD}),
    "adagrad": ("adagrad", tfo.SPECS["adagrad"], {"wd": WD}),
    "rowwise_adagrad": ("rowwise_adagrad", tfo.SPECS["rowwise_adagrad"], {"wd": WD}),
    "adam": ("adam", tfo.SPECS["adam"], {"wd": WD}),
    "rowwise_adam": ("rowwise_adam", test_rowwise_adam.SPEC, {"wd": WD}),
    "ftrl": ("ftrl", test_ftrl.SPEC, {}),
    "ftrl_all_terms": ("ftrl", test_ftrl.SPEC, {"wd": WD, "hp": test_ftrl.ALL_TERMS}),
}
ROUTES = ("balanced", "per-row vec4", "per-row vec1")

# replayed segment_update calls of this module's GPU cases per census tag (kind x route, dtypes)
COVERED = collections.Counter()
_DT = {torch.float32: "fp32", torch.bfloat16: "bf16", torch.float16: "fp16"}


def _world(device):
  return lambda n: MirrorWorld(n, device, inexact=n == 3, authoritative=True)


def _case(tables, imap, hots, **kw):
  kw.setdefault("batch", 192)  # divisible by 2, 3, 4 and 8
  kw.setdefault("lrs", [0.05, 0.05, 0.02])
  return tfo._case(tables, imap, hots, kw.pop("batch"), ragged_max=2, power_law=True, **kw)


# at most two ids per sample; power-law ids: duplicates across the batch make hot rows
PLANS = {
    # whole tables of widths <= 128, multiples of 4: the occurrence-balanced route
    "balanced": (_case([(160, 16, "sum"), (120, 32, "mean"), (96, 8, "sum"), (200, 64, "sum"),
                        (64, 16, "mean"), (128, 32, "sum"), (80, 8, "sum"), (100, 16, "sum")],
                       [0, 1, 2, 3, 4, 5, 6, 7, 0, 3], [1, 2, "ragged", 1, 2, 1, 2, 1, 2, 1]),
                 None),
    # whole tables wider than 128: the per-row route, four columns per lane
    "per-row vec4": (_case([(72, 192, "sum"), (60, 136, "mean"), (48, 132, "sum"),
                            (64, 192, "sum"), (40, 136, "sum"), (56, 144, "mean"),
                            (44, 160, "sum"), (52, 132, "sum")],
                           [0, 1, 2, 3, 4, 5, 6, 7, 0], [2, 1, 2, 1, "ragged", 2, 1, 1, 1]),
                     None),
    # column slices of widths that are not multiples of 4: the per-row route, one column per lane
    "per-row vec1": (_case([(150, 20, "sum"), (120, 36, "mean"), (100, 12, "sum"),
                            (90, 28, "sum")], [0, 1, 2, 3, 1], [2, 1, "ragged", 1, 2]),
                     {"column_slice_threshold": 600}),
}
# a table cut by rows over all ranks (fed the ids of every other rank's rows), beside whole ones
ROW_SLICES = (_case([(900, 16, "sum"), (60, 32, "mean"), (40, 8, "sum")], [0, 1, 2, 0],
                    [1, 2, 1, 2]), {"row_slice_threshold": 8000})


def _run(name, base, world, device, slack, **kw):
  """One case of kind ``name`` on the mirror harness, checked at ``slack`` times the models'
  bounds (1 on the kernels, 3 with the interpreter standing in for them: no fma); returns the
  census tags it added."""
  kind, spec, extra = KINDS[name]
  case, plan = base
  case = dict(case, **extra, **kw)
  if kind == "ftrl":
    case["lrs"] = [0.05, 0.0, 0.02]  # the middle step must move nothing
  before = REPLAYED.copy()
  tfo._run(case, kind, world, plan=plan, route="any", world_cls=_world(device), slack=slack,
           spec=spec)
  return {k: v - before.get(k, 0) for k, v in REPLAYED.items() if v - before.get(k, 0)}


def _expect(delta, *tags):
  for t in tags:
    assert delta.get(t, 0) > 0, (t, delta)


# ---------------------------------------------------------------------------------- CPU self-check
@pytest.mark.parametrize("world,name,plan,dtypes", [
    (2, "rowwise_adam", "per-row vec1", (torch.float32, torch.bfloat16)),
    (3, "ftrl_all_terms", "rows", (torch.bfloat16, torch.float32)),
    (4, "rowwise_adagrad", "per-row vec1", (torch.float16, torch.float32)),
    (4, "adam", "balanced", (torch.bfloat16, torch.bfloat16))])
def test_authoritative_mode_on_the_interpreter(world, name, plan, dtypes):
  """The interpreter as the "kernels": every check of the mode passes at its bounds."""
  base = ROW_SLICES if plan == "rows" else PLANS[plan]
  d = _run(name, base, world, HostDevice(), slack=3.0, table_dtype=dtypes[0], state_dtype=dtypes[1],
           lrs=[0.05, 0.02])
  _expect(d, "segment_update, " + ("balanced" if plan == "rows" else plan) + ", " +
          KINDS[name][0])


_ARGS = list(inspect.signature(dry_run.DryOps.segment_update).parameters)[1:]


class DefectDevice(HostDevice):
  """The interpreter as the "kernels", with one modelled defect in its ``segment_update``."""

  def __init__(self, defect):
    super().__init__()
    self.defect = defect
    self.hits = 0

  def op(self, name, rank):
    f = super().op(name, rank)
    if name != "segment_update":
      return f

    def run(*args):
      a = dict(zip(_ARGS, args))
      if a["kind"] == OPT_EMIT:
        return f(*args)
      T = np.frombuffer(a["tables"].numpy().tobytes(), dtype=TABLE_DESC)[:a["n_tables"]]
      nu = int(a["n_unique"][0])
      keys = a["keys"][a["seg"][:nu].long()].long().numpy()
      live = keys[keys < int(T[-1]["key_base"]) + int(T[-1]["rows"])]
      if self.defect == "key_base":  # every row rounded with the key of the next one
        t2 = T.copy()
        t2["key_base"] += 1
        a["tables"] = torch.from_numpy(np.frombuffer(t2.tobytes(), dtype=np.uint8).copy())
        a["keys"] = a["keys"] + 1
      saved = []
      if self.defect == "v_not_written":
        for t in T:
          v = self.world.tensor(int(t["state1"]), torch.float32, int(t["rows"]))
          saved.append((v, v.clone()))
      out = f(*[a[k] for k in _ARGS])
      for v, old in saved:
        v.copy_(old)
      if live.size and self.defect in ("moved", "stray_row"):
        key = int(live[len(live) // 2])
        m = int(np.searchsorted(T["key_base"], key, side="right")) - 1
        t = T[m]
        width, rows = int(t["width"]), int(t["rows"])
        w = self.world.tensor(int(t["weight"]), torch.float32, rows * width).view(rows, width)
        if self.defect == "moved":  # a touched element, 16 fp32 ulps of its magnitude (or of 1)
          r = key - int(t["key_base"])
          w[r, 0] += 16 * float(np.spacing(np.float32(max(abs(float(w[r, 0])), 1.0))))
        else:  # a row no key of this op touched
          mine = set((live - int(t["key_base"])).tolist())
          r = next(i for i in range(rows) if i not in mine)
          w[r, 0] += 1.0
      self.hits += 1
      return out
    return run


@pytest.mark.parametrize("defect,name,world,dtypes,match", [
    ("moved", "adagrad", 2, (torch.float32, torch.float32),
     r"table \d+ weight row \d+ column \d+"),
    ("stray_row", "sgd", 3, (torch.float32, torch.float32),
     r"row \d+ of table \d+ \(weight, key \d+\) changed, but no key"),
    ("key_base", "adam", 2, (torch.bfloat16, torch.float32), r"table \d+ weight row \d+ column"),
    ("v_not_written", "rowwise_adam", 4, (torch.float32, torch.float32),
     r"table \d+ state slot 1 row \d+ ")])
def test_defects_of_the_device_update_fail(defect, name, world, dtypes, match):
  """Each modelled defect fails with the table and the row named; the 16-bit key and the
  unwritten row word can only be seen by the state and 16-bit checks at world > 1."""
  dev = DefectDevice(defect)
  with pytest.raises(AssertionError, match=match):
    _run(name, PLANS["per-row vec1"] if name == "rowwise_adam" else PLANS["balanced"], world,
         dev, slack=3.0, table_dtype=dtypes[0], state_dtype=dtypes[1], lrs=[0.05, 0.02])
  assert dev.hits > 0


@pytest.mark.parametrize("world,name,plan,dtypes", [
    (5, "rowwise_adagrad", "per-row vec1", (torch.float32, torch.float32)),
    (6, "adam", "rows", (torch.float16, torch.bfloat16)),
    (7, "rowwise_adam", "balanced", (torch.bfloat16, torch.bfloat16)),
    (8, "ftrl_all_terms", "per-row vec1", (torch.float32, torch.bfloat16))])
def test_interpreter_checks_every_slot_over_steps(world, name, plan, dtypes):
  """The driver on the plain interpreter: three steps, every state slot of every shard."""
  kind, spec, extra = KINDS[name]
  case, kw = ROW_SLICES if plan == "rows" else PLANS[plan]
  case = dict(case, **extra, table_dtype=dtypes[0], state_dtype=dtypes[1], batch=24 * world)
  if kind == "ftrl":
    case["lrs"] = [0.05, 0.0, 0.02]
  tfo._run(case, kind, world, plan=kw, route="any", spec=spec)


# ------------------------------------------------------------------------------------------ GPU
_DEVICE = []


def _gpu():
  if not _DEVICE:
    _DEVICE.append(CudaDevice())
  return _DEVICE[0]


_WORLDS = (2, 3, 4, 8)
GPU_CASES = []
for _i, _name in enumerate(KINDS):
  for _j, _route in enumerate(ROUTES):
    GPU_CASES.append((f"{_name}-{_route.replace(' ', '_')}", _name, _route,
                      _WORLDS[(_i + _j) % 4], torch.float32, torch.float32, None))
  GPU_CASES.append((f"{_name}-row_slices", _name, "rows", _WORLDS[(_i + 3) % 4], torch.float32,
                    torch.float32, None))
# 16-bit tables and bf16 state: every combination, every kind that holds element-wise state
_HALF = [(torch.bfloat16, torch.float32), (torch.float16, torch.float32),
         (torch.float32, torch.bfloat16), (torch.bfloat16, torch.bfloat16),
         (torch.float16, torch.bfloat16)]
for _i, _name in enumerate(KINDS):
  for _j, (_tdt, _sdt) in enumerate(_HALF):
    if _sdt == torch.bfloat16 and _name in ("sgd", "rowwise_adagrad"):
      continue
    if (_i + _j) % 2:  # half of the kinds per combination, alternating
      continue
    GPU_CASES.append((f"{_name}-{str(_tdt)[6:]}_table-{str(_sdt)[6:]}_state", _name,
                      ROUTES[(_i + _j) % 3], _WORLDS[(_i + 2 * _j) % 4], _tdt, _sdt, None))
# 16-bit tables and bf16 state on a row-sliced table: the rounding keys of the row-slice local
# table, fed the ids of every other rank's rows
GPU_CASES.append(("adam-bfloat16_table-bfloat16_state-row_slices", "adam", "rows", 4,
                  torch.bfloat16, torch.bfloat16, None))
GPU_CASES.append(("ftrl_all_terms-float16_table-float32_state-row_slices", "ftrl_all_terms",
                  "rows", 8, torch.float16, torch.float32, None))
GPU_CASES.append(("rowwise_adam-bf16_activations", "rowwise_adam", "balanced", 4, torch.float32,
                  torch.float32, torch.bfloat16))


def _route(plan):
  return "balanced" if plan == "rows" else plan


def _state_tag(kind, sdt):
  """The state dtype the update runs with (per-row words and kinds without state stay fp32)."""
  half = sdt == torch.bfloat16 and OPTIMIZERS[kind].elementwise_state
  return "bf16" if half else "fp32"


def _tags(name, plan, tdt, sdt):
  """Census tags a GPU case must add: its kind on its route, its table / state dtypes."""
  kind = KINDS[name][0]
  tags = [f"segment_update, {_route(plan)}, {kind}",
          f"segment_update, {_DT[tdt]} table, {_state_tag(kind, sdt)} state"]
  if tdt != torch.float32:
    tags.append(f"segment_update, {_DT[tdt]} table, {kind}")
  if sdt != torch.float32:
    tags.append(f"segment_update, bf16 state, {kind}")
  return tags


@pytest.fixture(scope="module", autouse=True)
def _census():
  yield
  if COVERED:
    print("\nsegment_update calls replayed at world > 1:")
    for k in sorted(COVERED):
      print(f"  {k}: {COVERED[k]}")


@pytest.mark.gpu
@pytest.mark.parametrize("label,name,plan,world,tdt,sdt,cdt", GPU_CASES,
                         ids=[f"{c[0]}-w{c[3]}" for c in GPU_CASES])
def test_gpu_update_against_float64(label, name, plan, world, tdt, sdt,  # pylint: disable=unused-argument
                                   cdt):
  """One case on the kernels, checked at the kernels' own bounds (slack 1); the census must show
  the route and dtypes the case stands for in the coverage below."""
  kw = {"table_dtype": tdt, "state_dtype": sdt}
  if cdt is not None:
    kw["compute_dtype"] = cdt
  d = _run(name, ROW_SLICES if plan == "rows" else PLANS[plan], world, _gpu(), 1.0, **kw)
  _expect(d, *_tags(name, plan, tdt, sdt))
  for k, v in d.items():
    if k.startswith("segment_update, ") and k.count(",") >= 2:
      COVERED[k] += v


def test_gpu_cases_cover_every_kind_route_and_dtype():
  """The GPU cases cover every optimizer kind on every route and every 16-bit table / state
  combination at world > 1, and every table / state combination of a row-sliced table; each
  case asserts at run time that the census shows its tags, so together they need no run order."""
  got = {t for _, name, plan, world, tdt, sdt, _ in GPU_CASES
         for t in _tags(name, plan, tdt, sdt) if world > 1}
  want = {f"segment_update, {r}, {k}" for k in {v[0] for v in KINDS.values()} for r in ROUTES}
  want |= {f"segment_update, {t} table, {s} state" for t in ("fp32", "bf16", "fp16")
           for s in ("fp32", "bf16")}
  assert not want - got, sorted(want - got)
  rows = {(tdt, _state_tag(KINDS[name][0], sdt)) for _, name, plan, _, tdt, sdt, _ in GPU_CASES
          if plan == "rows"}
  assert {(torch.bfloat16, "bf16"), (torch.float16, "fp32"), (torch.float32, "fp32")} <= rows
