"""The embedding optimizers (SGD, Adagrad, row-wise Adagrad, Adam) on every update route of the
fused engine against the float64 model of ``optim_reference.py``, with and without weight decay.

Every step is checked on the engine's own state: the weights and optimizer state are read with
``get_weights`` / ``get_optimizer_state`` before the step, that one step is computed in float64
from them, and after the step the touched rows and every state slot must lie within bounds
derived from operation counts (no flat tolerance), the untouched rows and their state must be
bit-identical, and Adam's step counter must equal the number of steps.  16-bit tables and state
must equal the stochastic rounding (``ops/stochastic_rounding.py``) of some value within the
bound.  Each case asserts which update op ran, so a route that silently changes fails.

CPU (no GPU): the same cases through the plan interpreter at world 1-4; ``SparseRowOptimizer``
(the torch back end) with weight decay; ``set_optimizer`` rejecting unknown keywords; default
SGD with decay leaving the atomic scatter; and a self-check that the bounds pass the exactly
rounded result and fail each modelled defect.

GPU (one H100, world 1): atomic SGD (staged / unstaged / vec8), the sorted update
(occurrence-balanced, per-row with 4 or 1 columns per lane), the emit route, 16-bit tables, bf16
state, the HBM row cache and bf16 / fp16 activations, on id segments of 1, 31, 32, 33, 65 and 300
occurrences (a segment starting on a 32-item chunk border, a hot row crossing many chunks),
fewer than 32 items, mixed widths in one launch, inputs sharing a table, sum and mean pooling
(fixed and ragged with lengths 0, 1 and many), int32 and int64 ids, gradients from +-1e3 down to
exact zeros and rows touched only by zero gradients, and Adam over 4 steps with different touched
sets and a learning-rate change.
"""
import numpy as np
import pytest
import torch

import distributed_embeddings_b200 as de
from distributed_embeddings_b200.ops.ragged import RaggedIds
from distributed_embeddings_b200.parallel import dry_run
from distributed_embeddings_b200.parallel.embedding_optimizers import OPTIMIZERS
from distributed_embeddings_b200.parallel.hybrid import SparseRowOptimizer
from optim_reference import (TABLE_DEFECTS, f32, half_within,  # pylint: disable=wrong-import-order
                             table_step, worst_table_ratio)

KINDS = ["sgd", "adagrad", "rowwise_adagrad", "adam"]
WD = 0.5  # large enough that a dropped or doubled decay misses the bounds by orders of magnitude
INIT_ACC = 0.1
# occurrence counts of the structured rows 1..6 of the edge table (the table of input 0, first in
# the key space; no other id hits row 0 or rows 1..7): the segments start at sorted positions 0, 1,
# 32 (row 3: a 32-item chunk border), 65, 130 and 162; row 6 crosses nine chunks; row 7 is touched
# by 3 occurrences that all carry zero gradients
EDGE_COUNTS = [1, 31, 33, 65, 32, 300]
ZERO_ROW, ZERO_COUNT = 7, 3


# ------------------------------------------------------------------ inputs
def _grad_values(gen, shape):
  """Gradients from +-1e3 down to 1e-4, 1 in 8 exactly zero."""
  mag = torch.pow(10.0, torch.rand(shape, generator=gen, dtype=torch.float64) * 7 - 4)
  g = (torch.randn(shape, generator=gen, dtype=torch.float64) * mag).clamp(-1e3, 1e3)
  g[torch.rand(shape, generator=gen) < 0.125] = 0.0
  return g.float()


def _draw(case, step):
  """Ids per input (``[B, h]`` int64 arrays or lists of per-sample lists for ragged inputs) and
  the upstream gradient ``[B, sum(widths)]`` in fp32."""
  gen = torch.Generator().manual_seed(1000 * case.get("seed", 0) + step)
  B = case["batch"]
  rows = [t[0] for t in case["tables"]]
  ids = []
  zero_samples = []
  for i, t in enumerate(case["imap"]):
    h = case["hots"][i]
    if h == "ragged":
      most = case.get("ragged_max", 8)
      lens = torch.randint(0, most + 1, (B,), generator=gen).tolist()
      lens[:3] = [0, 1, most]
      lo_id = ZERO_ROW + 1 if case.get("edges") and t == case["imap"][0] else 0
      ids.append([torch.randint(lo_id, rows[t], (n,), generator=gen).tolist() for n in lens])
      continue
    # other inputs of the edge table stay off its structured rows 0..7
    lo_id = ZERO_ROW + 1 if case.get("edges") and t == case["imap"][0] else 0
    if case.get("power_law"):
      x = (torch.rand(B, h, generator=gen).pow(6) * rows[t]).long().clamp(max=rows[t] - 1)
    elif case.get("touch") is not None:  # a step-dependent touched set: fractions of the rows
      lo, hi = case["touch"][step % len(case["touch"])]
      x = torch.randint(int(lo * rows[t]), int(hi * rows[t]), (B, h), generator=gen)
    else:
      x = torch.randint(lo_id, rows[t], (B, h), generator=gen)
    if i == 0 and case.get("edges"):
      col = np.concatenate([np.full(c, r + 1) for r, c in enumerate(EDGE_COUNTS)] +
                           [np.full(ZERO_COUNT, ZERO_ROW)])
      assert h == 1 and len(col) <= B
      x[:len(col), 0] = torch.from_numpy(col)
      x[len(col):, 0] = torch.randint(ZERO_ROW + 1, rows[t], (B - len(col),), generator=gen)
      perm = torch.randperm(B, generator=gen)
      x = x[perm]
      zero_samples = torch.nonzero(x[:, 0] == ZERO_ROW).view(-1).tolist()
    ids.append(x.numpy())
  widths = [case["tables"][t][1] for t in case["imap"]]
  grad = _grad_values(gen, (B, sum(widths)))
  if zero_samples:
    grad[zero_samples, :widths[0]] = 0.0
  return ids, grad


def _occurrences(case, ids, grad, t, lo=0, hi=None):
  """(rows, c_k * g_k) of every id occurrence of table ``t`` from samples [lo, hi), gradients as
  the kernel reads them (already rounded to the compute dtype by the caller)."""
  widths = [case["tables"][j][1] for j in case["imap"]]
  cols = np.cumsum([0] + widths)
  comb = case["tables"][t][2]
  rows_out, vals_out = [], []
  g = grad.double().numpy()
  nrows = case["tables"][t][0]
  for i, tt in enumerate(case["imap"]):
    if tt != t:
      continue
    gi = g[:, cols[i]:cols[i + 1]]
    samples = ids[i] if isinstance(ids[i], list) else [list(r) for r in ids[i]]
    for b in range(lo, len(samples) if hi is None else hi):
      row = [r for r in samples[b] if 0 <= r < nrows]
      n = len(samples[b])
      c = f32(1.0 / n) if (comb == "mean" and n) else 1.0
      for r in row:
        rows_out.append(r)
        vals_out.append(c * gi[b])
  w = case["tables"][t][1]
  return (np.asarray(rows_out, dtype=np.int64),
          np.asarray(vals_out, dtype=np.float64).reshape(-1, w))


def _as_inputs(case, ids, dev, lo=0, hi=None):
  idt = torch.int32 if case.get("ids32") else torch.int64
  out = []
  for x in ids:
    if isinstance(x, list):
      part = x[lo:hi]
      out.append(RaggedIds.from_row_lengths(
          torch.tensor([v for r in part for v in r], dtype=idt, device=dev),
          torch.tensor([len(r) for r in part], dtype=torch.int64, device=dev)))
    else:
      out.append(torch.from_numpy(x[lo:hi]).to(device=dev, dtype=idt))
  return out


def _initial_state(kind, rows, width, sdt=torch.float32):
  if kind == "adagrad":
    return [np.full((rows, width), float(torch.tensor(INIT_ACC).to(sdt).float()), np.float32)]
  if kind == "rowwise_adagrad":
    return [np.full(rows, f32(INIT_ACC), np.float32)]
  if kind == "adam":
    return [np.zeros((rows, width), np.float32)] * 2
  return []


# ------------------------------------------------------------------ per-step check
class Spec:
  """What the driver needs to know about one optimizer kind: its keyword arguments, its state at
  the start, and the float64 model of one step on one column range of a table (a column slice
  keeps its own row words).  The row-wise Adam and FTRL tests pass their own."""

  def __init__(self, kind):
    self.kind = kind
    self.slots = OPTIMIZERS[kind].slots

  def opt(self, case):  # pylint: disable=unused-argument
    return {}

  def initial(self, rows, width, sdt):
    return _initial_state(self.kind, rows, width, sdt)

  def model(self, case, before, state, occ, step, scale):
    cfg = {"eps": OPTIMIZERS[self.kind].eps, "beta1": 0.9, "beta2": 0.999,
           "weight_decay": case.get("wd", 0.0)}
    return table_step(self.kind, before, state, occ[0], occ[1], scale, case["lrs"][step],
                      step + 1, cfg, atomic=_expected_route(case, self.kind) == "atomic")

  def finish(self, case, zeros):
    """Checks over the whole run; ``zeros``: weights that a step with lr > 0 touched and left
    exactly zero."""


SPECS = {k: Spec(k) for k in KINDS}
_SLOT_NAMES = {"p": "weight", "s0": "state slot 0", "s1": "state slot 1"}


def _slices(demb, t, width):
  """Column ranges of table ``t`` that keep their own row words (the whole row unless sliced)."""
  st = demb.strategy
  if t not in st.table_groups[1]:
    return [(0, width)]
  gt = st.table_groups[1].index(t)
  return sorted({(s.col_start, s.col_end) for shards in st.shards for s in shards
                 if s.table == gt})


def _pieces(des, t, width):
  """Where table ``t`` lives: (rank, local table, first local row, first global row, rows, first
  column, end column) of every shard."""
  st = des[0].strategy
  assert t not in st.table_groups[0], "replicated tables are not updated by the engine"
  if t in st.table_groups[1]:
    gt = st.table_groups[1].index(t)
    return [(r, s.local_table, s.row_offset, 0, s.rows, s.col_start, s.col_end)
            for r, shards in enumerate(st.shards) for s in shards if s.table == gt]
  gt = st.table_groups[2].index(t)
  return [(r, len(des[r].local_embedding_layers) + gt, 0, lo, hi - lo, 0, width)
          for r, (lo, hi) in enumerate(st.row_ranges[gt]) if hi > lo]


def _read_shards(des, t, width):
  """Every shard of table ``t`` as the engine of its rank holds it: global rows, columns, the
  16-bit rounding key of each row (``key_base`` of the local table plus the row inside it) and
  the state slots, read from ``opt_state`` at the shard's rows (a per-row slot: the shard's own
  words, not the exported width-weighted mean)."""
  out = []
  for r, m, l0, g0, n, c0, c1 in _pieces(des, t, width):
    eng = des[r]._engine
    st = eng.opt_state.get(m, [])
    slots = [np.asarray(x[l0:l0 + n].float().cpu().numpy(), dtype=np.float32) for x in st]
    out.append({"rank": r, "table": m, "rows": np.arange(g0, g0 + n), "cols": (c0, c1),
                "keys": int(eng.tdesc_np["key_base"][m]) + l0 + np.arange(n), "slots": slots})
  return out


def _read_global(demb, kind, t, rows, width, case):
  """World 1 on the GPU (the table may sit in the HBM row cache): the exported state, rows keyed
  from ``case['key_base']``."""
  st = demb.get_optimizer_state()
  slots = []
  if st["tables"] is not None:
    slots = [np.asarray(a, dtype=np.float32)[:, 0] if s.per_row else np.asarray(a, np.float32)
             for a, s in zip(st["tables"][t], OPTIMIZERS[kind].slots)]
  return [{"rank": 0, "table": t, "rows": np.arange(rows), "cols": (0, width),
           "keys": np.arange(rows) + case.get("key_base", 0), "slots": slots}]


def _check_shard(case, spec, t, step, sh, out, bound, touched, after_t, slack):
  """One shard of table ``t`` after ``step`` against the float64 model of its column range:
  untouched rows bit-identical, touched fp32 values within ``slack`` times the bounds, touched
  16-bit values between the roundings of the bound's ends at the shard's keys.  A failure names
  the table, the slot, the row and the column."""
  rows, (c0, c1) = sh["rows"], sh["cols"]
  tdt = case.get("table_dtype", torch.float32)
  sdt = case.get("state_dtype", torch.float32)
  got = {"p": after_t[rows, c0:c1]}
  dts = {"p": tdt}
  for j, (x, s) in enumerate(zip(sh["slots"], spec.slots)):
    got[f"s{j}"] = x
    dts[f"s{j}"] = torch.float32 if s.per_row else sdt
  hit = touched[rows]
  for k, g in got.items():
    if k not in out:
      continue
    g = torch.as_tensor(np.asarray(g, dtype=np.float64))
    o, b = out[k][rows], slack * bound[k][rows]
    mask = torch.as_tensor(hit).view(-1, *([1] * (g.dim() - 1))).expand_as(g)
    err = (g - o).abs()
    bad = ~torch.isfinite(g) | (~mask & (err != 0))
    if dts[k] == torch.float32:
      bad |= mask & (err > b)
    elif hit.any():
      idx = np.nonzero(hit)[0]
      inside = half_within(g[idx], o[idx], b[idx], dts[k], step + 1, sh["keys"][idx],
                           {"p": 0, "s0": 1, "s1": 2}[k], mask=True)
      bad[torch.as_tensor(idx)] |= torch.as_tensor(~inside)
    if bad.any():
      e = [int(x) for x in torch.nonzero(bad)[0]]
      i = e[0]
      col = f" column {c0 + e[1]}" if len(e) > 1 else ""
      raise AssertionError(
          f"table {t} {_SLOT_NAMES[k]} row {int(rows[i])}{col} after step {step} (rank "
          f"{sh['rank']}, local table {sh['table']}, key {int(sh['keys'][i])}, "
          f"{'touched' if hit[i] else 'untouched'}): got {float(g[tuple(e)])!r}, float64 model "
          f"{float(o[tuple(e)])!r} +- {float(b[tuple(e)])!r} ({dts[k]}); "
          f"{int(bad.sum())} values outside")


class _Counting:
  """Records the update ops the engine launches (name, route)."""

  def __init__(self, ops):
    self._ops, self.routes = ops, []

  def __getattr__(self, name):
    f = getattr(self._ops, name)
    if name not in ("scatter_add_bwd", "segment_update", "interact_bwd"):
      return f

    def call(*a, **k):
      if name == "segment_update":
        from distributed_embeddings_b200.ops import _native
        if a[11] == _native.OPT_EMIT:
          self.routes.append("emit")
        elif a[26] is not None:
          self.routes.append("balanced")
        else:
          self.routes.append("per_row_vec4" if a[25] else "per_row_vec1")
      else:
        self.routes.append(name)
      return f(*a, **k)
    return call


def _expected_route(case, kind):
  if kind == "sgd" and not case.get("wd") and not case.get("deterministic") and \
      case.get("table_dtype", torch.float32) == torch.float32 and not case.get("cache"):
    return "atomic"
  widths = [t[1] for t in case["tables"]]
  if any(w % 4 for w in widths):
    return "per_row_vec1"
  return "balanced" if max(widths) <= 128 else "per_row_vec4"


# ------------------------------------------------------------------ driver (GPU and interpreter)
def _run(case, kind, world=1, dev=None, plan=None, route=None, world_cls=dry_run.DryWorld,
         slack=None, spec=None):
  """Run ``case`` for ``len(case['lrs'])`` steps and check every step: on one GPU rank (``dev``)
  or through the plan interpreter on ``world`` ranks, whose ops ``world_cls`` may replay on the
  kernels.  ``plan``: extra DistributedEmbedding arguments (slicing); ``route``: the update route
  every launch must take ("any": one of the sorted routes); ``slack``: factor on the bounds
  (default 3 for the interpreter, which computes in torch fp32 ops without fma, 1 on the GPU);
  ``spec``: the optimizer's :class:`Spec`.

  The state is read after every step from the engine: on the GPU through
  ``get_optimizer_state``, in the interpreter per shard from ``opt_state`` (the rows of a column
  slice keep their own row words), so every slot is checked at every step and world size, with
  16-bit values rounded at the keys of the rank that owns them."""
  spec = spec or SPECS[kind]
  embs = [{"input_dim": r, "output_dim": w, "combiner": c} for r, w, c in case["tables"]]
  kw = dict(input_table_map=list(case["imap"]), strategy="basic")
  kw.update(plan or {})
  if case.get("table_dtype", torch.float32) != torch.float32:
    kw["table_dtype"] = case["table_dtype"]
  if case.get("compute_dtype"):
    kw["compute_dtype"] = case["compute_dtype"]
  if case.get("cache"):
    small = case["tables"][0]
    kw.update(gpu_embedding_size=small[0] * small[1] + 1, offload_cache_size=case["cache"])
  opt = dict(spec.opt(case), weight_decay=case.get("wd", 0.0))
  if case.get("deterministic"):
    opt["deterministic"] = True
  sdt = case.get("state_dtype", torch.float32)
  if sdt != torch.float32:
    opt["state_dtype"] = sdt
  cdt = case.get("compute_dtype", torch.float32)
  if slack is None:
    slack = 3.0 if dev is None else 1.0
  torch.manual_seed(case.get("seed", 0))
  if dev is None:
    sim, des = dry_run.build_engines(embs, world, world_cls, dp_input=True, **kw)
  else:
    sim, des = None, [de.DistributedEmbedding(embs, device=dev, backend="fused", world_size=1,
                                              rank=0, **kw)]
  gen = np.random.default_rng(case.get("seed", 0))
  tables = [gen.standard_normal((r, w)).astype(np.float32) for r, w, _ in case["tables"]]
  for d in des:
    d.set_weights(tables)
    d.set_optimizer(kind, lr=case["lrs"][0], **opt)
    assert d._fused_optimizer["eps"] == OPTIMIZERS[kind].eps
    if any(h == "ragged" for h in case["hots"]):
      d.ragged_capacity = case.get("ragged_max", 8)
  demb = des[0]
  slices = [_slices(demb, t, w) if dev is None else [(0, w)]
            for t, (_, w, _) in enumerate(case["tables"])]
  states = [{(c0, c1): spec.initial(r, c1 - c0, sdt) for c0, c1 in slices[t]}
            for t, (r, _, _) in enumerate(case["tables"])]
  routes, zeros = set(), 0
  for step, lr in enumerate(case["lrs"]):
    if step and lr != case["lrs"][step - 1]:
      for d in des:
        d.set_learning_rate(lr)
    ids, grad = _draw(case, step)
    grad = grad.to(cdt)  # the values the kernels read
    lb = case["batch"] // world
    before = _weights(des, world)

    def rank_fn(r):
      d = des[r]
      out = d(_as_inputs(case, ids, d.device if dev is None else dev, r * lb, (r + 1) * lb),
              concat=True)
      eng = d._engine
      if not isinstance(eng.ops, _Counting):
        eng.ops = _Counting(eng.ops)
      out.backward(grad[r * lb:(r + 1) * lb].to(out.device))
      return eng.ops.routes
    if dev is None:
      for got in dry_run.run_ranks(sim, rank_fn):
        routes |= set(got)
    else:
      routes |= set(rank_fn(0))
      torch.cuda.synchronize()
    if case.get("edges"):
      _check_edge_layout(case, ids, des[0]._engine)
    after = _weights(des, world)
    if kind in ("adam", "rowwise_adam"):  # the step of the bias corrections, on every rank
      assert [d._engine.step_count() for d in des] == [step + 1] * len(des)
    for t, (r, w, _) in enumerate(case["tables"]):
      rows, vals = _occurrences(case, ids, grad.float(), t)
      shards = _read_shards(des, t, w) if dev is None else _read_global(demb, kind, t, r, w, case)
      touched = None
      for c0, c1 in slices[t]:
        o, b, touched = spec.model(case, before[t][:, c0:c1], states[t][(c0, c1)],
                                   (rows, vals[:, c0:c1]), step, 1.0 / world)
        new = [x.copy() for x in states[t][(c0, c1)]]
        for sh in shards:
          if sh["cols"] != (c0, c1):
            continue
          _check_shard(case, spec, t, step, sh, o, b, touched, after[t], slack)
          for k, x in enumerate(sh["slots"]):
            new[k][sh["rows"]] = x
        states[t][(c0, c1)] = new
      zeros += int((after[t][touched] == 0.0).sum()) if lr > 0 else 0
  spec.finish(case, zeros)
  want = route or _expected_route(case, kind)
  if want == "any":
    assert routes and routes <= {"balanced", "per_row_vec4", "per_row_vec1"}, routes
  else:
    assert routes == {want if want != "atomic" else "scatter_add_bwd"}, (routes, want)
  return des


def _check_edge_layout(case, ids, eng):
  """The edge segments are where the comment at EDGE_COUNTS says: the edge table starts the key
  space and its rows 0..7 are hit exactly EDGE_COUNTS / ZERO_COUNT times."""
  t0 = case["imap"][0]
  occ_rows, _ = _occurrences(case, ids, torch.zeros(case["batch"], sum(
      case["tables"][t][1] for t in case["imap"])), t0)
  counts = np.bincount(occ_rows, minlength=ZERO_ROW + 1)[:ZERO_ROW + 1]
  assert counts.tolist() == [0] + EDGE_COUNTS + [ZERO_COUNT], counts
  widths = {int(d["local_table"]): int(d["width"]) for d in eng.mpdesc_np}
  first = min(range(len(eng.tdesc_np)), key=lambda m: int(eng.tdesc_np[m]["key_base"]))
  edge = [d for d in eng.mpdesc_np if int(d["local_table"]) == first]
  assert int(eng.tdesc_np[first]["key_base"]) == 0 and widths[first] == case["tables"][t0][1]
  assert all(int(d["row_base"]) == 0 for d in edge), "the edge table shares its local table"


def _weights(des, world):
  if world == 1:
    return [np.asarray(w, dtype=np.float32) for w in des[0].get_weights()]
  from test_dry_run import assemble  # pylint: disable=import-outside-toplevel
  return assemble(des)


# ------------------------------------------------------------------ the case matrix
def _case(tables, imap, hots, batch, **kw):
  return dict(tables=tables, imap=imap, hots=hots, batch=batch, lrs=kw.pop("lrs", [0.05]), **kw)


MIXED = _case([(400, 16, "sum"), (300, 32, "mean"), (200, 128, "sum")], [0, 1, 0, 2, 1],
              [1, 3, 2, "ragged", 1], 512, edges=True, seed=1)
WIDE = _case([(400, 16, "sum"), (150, 192, "mean"), (120, 256, "sum")], [0, 1, 2, 0],
             [1, 2, 1, 3], 512, edges=True, seed=2)
ODD = _case([(400, 20, "sum"), (150, 6, "mean"), (90, 12, "sum")], [0, 1, 2, 1],
            [1, 3, "ragged", 1], 512, edges=True, ids32=True, seed=3)
SMALL = _case([(50, 32, "sum"), (40, 16, "mean")], [0, 1], [1, 2], 20, seed=4)


def _with(base, **kw):
  c = dict(base)
  c.update(kw)
  return c


GPU_CASES = []
for _k in KINDS:
  for _wd in (0.0, WD):
    GPU_CASES += [(f"balanced-{_k}-wd{_wd}", _k, _with(MIXED, wd=_wd)),
                  (f"per_row_vec4-{_k}-wd{_wd}", _k, _with(WIDE, wd=_wd)),
                  (f"per_row_vec1-{_k}-wd{_wd}", _k, _with(ODD, wd=_wd)),
                  (f"small-{_k}-wd{_wd}", _k, _with(SMALL, wd=_wd))]
GPU_CASES += [("sgd-deterministic", "sgd", _with(MIXED, deterministic=True))]
for _k in KINDS:
  for _dt in (torch.bfloat16, torch.float16):
    GPU_CASES.append((f"table16-{_k}-{_dt}", _k,
                      _case([(600, 32, "sum")], [0, 0], [1, 2], 512, edges=True, wd=WD,
                            table_dtype=_dt, seed=5)))
for _k in ("adagrad", "adam"):
  GPU_CASES.append((f"bf16state-{_k}", _k,
                    _case([(600, 32, "sum")], [0, 0], [1, 2], 512, edges=True, wd=WD,
                          state_dtype=torch.bfloat16, seed=6)))
  GPU_CASES.append((f"bf16state-bf16table-{_k}", _k,
                    _case([(600, 32, "sum")], [0], [1], 512, edges=True, wd=WD,
                          state_dtype=torch.bfloat16, table_dtype=torch.bfloat16, seed=7)))
for _k in ("sgd", "adagrad", "rowwise_adagrad", "adam"):
  GPU_CASES.append((f"row_cache-{_k}", _k,
                    _case([(64, 16, "sum"), (6000, 16, "sum")], [0, 1, 1], [1, 2, 1], 512,
                          wd=WD, cache=2000, lrs=[0.05, 0.05], seed=8)))
for _cdt in (torch.bfloat16, torch.float16):
  for _k in ("adagrad", "rowwise_adagrad"):
    GPU_CASES.append((f"act-{_cdt}-{_k}", _k, _with(MIXED, wd=WD, compute_dtype=_cdt)))
GPU_CASES.append(("adam-4-steps", "adam",
                  _case([(300, 32, "sum"), (100, 16, "mean")], [0, 1], [2, 3], 256, wd=WD,
                        ids32=True, touch=[(0, 1 / 3), (1 / 6, 2 / 3), (1 / 2, 1), (0, 2 / 15)],
                        lrs=[0.05, 0.05, 0.01, 0.01], seed=9)))


@pytest.mark.gpu
@pytest.mark.parametrize("name,kind,case", GPU_CASES, ids=[c[0] for c in GPU_CASES])
def test_update_routes_against_float64(name, kind, case):  # pylint: disable=unused-argument
  _run(case, kind, dev=torch.device("cuda", 0))


@pytest.mark.gpu
@pytest.mark.parametrize("staged,vec8", [("1", "0"), ("0", "0"), ("1", "1")])
def test_atomic_sgd_scatter_against_float64(monkeypatch, staged, vec8):
  monkeypatch.setenv("DE_B200_SCATTER_STAGED", staged)
  monkeypatch.setenv("DE_B200_VEC8_GRAD", vec8)
  case = _case([(400, 16, "sum"), (300, 32, "mean"), (200, 64, "sum")], [0, 1, 0, 2],
               [1, 3, 2, 1], 512, edges=True, seed=10)
  des = _run(case, "sgd", dev=torch.device("cuda", 0))
  eng = des[0]._engine
  assert eng.staged_update == (staged == "1") and eng.vec8 == (vec8 == "1")


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("width", [16, 32, 128])
@pytest.mark.parametrize("combiner", ["sum", "mean"])
def test_fused_optimizer_on_skewed_ids(kind, width, combiner):
  """Power-law ids (most ids are 0/1/2): segments span many chunks of the balanced update."""
  case = _case([(500, width, combiner)] * 2, [0, 1, 0], [1, 7, 3], 4096, power_law=True,
               deterministic=kind == "sgd", lrs=[0.1], seed=11)
  _run(case, kind, dev=torch.device("cuda", 0))


@pytest.mark.gpu
@pytest.mark.parametrize("ids32", [False, True])
def test_emit_route_against_float64(ids32):
  """Without an optimizer the backward returns deduplicated sparse gradients: each row the sum of
  its occurrences within (n + 1) u sum |c_k g_k|, rows no id touched absent."""
  dev = torch.device("cuda", 0)
  case = _with(MIXED, ids32=ids32)
  embs = [{"input_dim": r, "output_dim": w, "combiner": c} for r, w, c in case["tables"]]
  demb = de.DistributedEmbedding(embs, device=dev, backend="fused", world_size=1, rank=0,
                                 input_table_map=case["imap"], strategy="basic")
  demb.ragged_capacity = 8
  ids, grad = _draw(case, 0)
  out = demb(_as_inputs(case, ids, dev), concat=True)
  eng = demb._engine
  eng.ops = _Counting(eng.ops)
  out.backward(grad.to(dev))
  assert eng.ops.routes == ["emit"]
  for t, layer_w in enumerate(demb.mp_parameters()):
    rows, vals = _occurrences(case, ids, grad, t)
    want = np.zeros((case["tables"][t][0], case["tables"][t][1]))
    np.add.at(want, rows, vals)
    n = np.bincount(rows, minlength=want.shape[0])[:, None]
    ga = np.zeros_like(want)
    np.add.at(ga, rows, np.abs(vals))
    g = layer_w.grad.coalesce()
    dense = np.zeros_like(want)
    dense[g.indices()[0].cpu().numpy()] = g.values().double().cpu().numpy()
    assert set(g.indices()[0].tolist()) == set(rows.tolist())
    assert (np.abs(dense - want) <= (n + 1) * 2.0**-24 * ga + 1e-37).all()


@pytest.mark.gpu
def test_default_sgd_without_decay_keeps_the_atomic_route():
  """Weight decay 0 leaves the default SGD on the atomic scatter; decay moves it to the sorted
  update and a DLRM step's producer update declines."""
  dev = torch.device("cuda", 0)
  demb = de.DistributedEmbedding([{"input_dim": 100, "output_dim": 128, "combiner": None}] * 2,
                                 device=dev, backend="fused", world_size=1, rank=0)
  demb.set_optimizer("sgd", lr=0.1)
  ids = [torch.randint(0, 100, (64,), device=dev) for _ in range(2)]
  demb(ids, concat=True)
  eng = demb._engine
  assert eng._atomic_sgd() and eng.producer_update(128, 10) is not None
  demb.set_optimizer("sgd", lr=0.1, weight_decay=1e-4)
  assert not eng._atomic_sgd() and eng.producer_update(128, 10) is None
  demb(ids, concat=True).sum().backward()


# ------------------------------------------------------------------ CPU: the plan interpreter
CPU_CASES = []
for _k in KINDS:
  for _wd in (0.0, WD):
    CPU_CASES.append((f"{_k}-wd{_wd}", _k,
                      _case([(200, 16, "sum"), (150, 8, "mean"), (90, 12, "sum"),
                             (80, 8, "sum")], [0, 1, 2, 3, 0], [1, 2, 1, 3, 2], 96, edges=False,
                            wd=_wd, seed=20)))


@pytest.mark.parametrize("world", [1, 2, 4])
@pytest.mark.parametrize("name,kind,case", CPU_CASES, ids=[c[0] for c in CPU_CASES])
def test_interpreter_against_float64(world, name, kind, case):  # pylint: disable=unused-argument
  _run(case, kind, world=world)


@pytest.mark.parametrize("kind", KINDS)
def test_interpreter_edges_against_float64(kind):
  """The structured segments (1 ... 300 occurrences, a zero-gradient row) at world 1."""
  case = _case([(400, 8, "sum"), (50, 4, "mean")], [0, 1], [1, "ragged"], 480, edges=True, wd=WD,
               seed=21)
  _run(case, kind, world=1)


def test_default_sgd_applies_weight_decay():
  """Default (non-deterministic) SGD with decay takes the sorted update and decays row 1 once:
  1 - 0.5 * (2 * 0.25 + 0.5 * 1) = 0.5 for a row of ones hit twice."""
  sim, des = dry_run.build_engines([{"input_dim": 10, "output_dim": 8, "combiner": "sum"}], 1,
                                   dp_input=True)
  d = des[0]
  d.set_weights([np.ones((10, 8), np.float32)])
  d.set_optimizer("sgd", lr=0.5, weight_decay=0.5)
  ids = torch.tensor([[1], [2], [1]], dtype=torch.int64)

  def fn(r):  # pylint: disable=unused-argument
    out = d([ids], concat=True)
    out.backward(torch.full_like(out, 0.25))
  dry_run.run_ranks(sim, fn)
  w = d.get_weights()[0]
  assert d._engine.ops.calls.get("scatter_add_bwd", 0) == 0
  assert d._engine.ops.calls.get("segment_update", 0) == 1
  assert (w[1] == 0.5).all() and (w[2] == np.float32(1 - 0.5 * (0.25 + 0.5))).all()
  assert (w[0] == 1).all() and (w[3:] == 1).all()


def test_set_optimizer_rejects_unknown_keywords():
  d = de.DistributedEmbedding([{"input_dim": 10, "output_dim": 8, "combiner": "sum"}],
                              device="cpu", backend="torch", world_size=1, rank=0)
  for bad in ({"weightdecay": 0.1}, {"momentum": 0.9}, {"lr_decay": 1.0}):
    with pytest.raises(ValueError, match="unknown fused optimizer argument"):
      d.set_optimizer("adagrad", lr=0.1, **bad)
  d.set_optimizer("adam", lr=0.1, eps=1e-6, beta1=0.8, beta2=0.99, weight_decay=0.1,
                  initial_accumulator_value=0.0, deterministic=True, step=3,
                  state_dtype=torch.float32)


@pytest.mark.parametrize("kind", KINDS)
def test_sparse_row_optimizer_weight_decay_against_float64(kind):
  """The torch back end's row-sparse optimizer: two steps with decay, duplicate ids and a row
  touched only by zero gradients."""
  torch.manual_seed(30)
  rows, width = 60, 12
  w0 = torch.randn(rows, width)
  p = torch.nn.Parameter(w0.clone())
  # betas exact in fp32: the torch optimizer takes its constants in float64
  b1, b2 = 0.875, 1 - 2.0**-10
  opt = SparseRowOptimizer([p], kind, lr=0.05, weight_decay=WD, beta1=b1, beta2=b2)
  state = _initial_state(kind, rows, width)
  gen = torch.Generator().manual_seed(31)
  for step in range(2):
    idx = torch.randint(0, 30 + 20 * step, (80,), generator=gen)
    idx[:5] = 7
    vals = _grad_values(gen, (80, width))
    vals[:5] = 0.0
    p.grad = torch.sparse_coo_tensor(idx[None], vals, (rows, width))
    before = p.detach().numpy().copy()
    cfg = {"eps": 1e-8 if kind == "adam" else 1e-7, "beta1": b1, "beta2": b2,
           "weight_decay": WD}
    out, bound, touched = table_step(kind, before, state, idx.numpy(), vals.double().numpy(),
                                     1.0, 0.05, step + 1, cfg)
    opt.step()
    got = {"p": p.detach().numpy()}
    for k, s in zip(("s0", "s1"), opt.state[0]):
      got[k] = s.numpy()
    # the torch ops round each product on its own (no fma): allow two more roundings per term
    r = worst_table_ratio(out, {k: 3 * b for k, b in bound.items()}, got)
    assert r <= 1.0 and touched[7], r
    state = [np.asarray(got[k], dtype=np.float32) for k in ("s0", "s1") if k in got]


# ------------------------------------------------------------------ CPU: bound self-check
def _selfcheck_inputs(kind, seed=40):
  gen = torch.Generator().manual_seed(seed)
  rows, width = 64, 16
  w = torch.randn(rows, width, generator=gen).numpy()
  if kind == "adam":  # plausible moments of earlier steps
    m = (torch.randn(rows, width, generator=gen) * 0.1).numpy()
    state = [m, (m * m * 3).astype(np.float32)]
  else:
    state = _initial_state(kind, rows, width)
  occ_rows = np.concatenate([np.full(c, r + 1) for r, c in enumerate([1, 2, 5, 33])] +
                            [np.arange(10, 40)])
  n = np.where(np.arange(len(occ_rows)) % 2 == 0, 1, 3)  # pooling of 1 or 3 ids (mean)
  c = np.asarray([f32(1.0 / k) for k in n])
  g = _grad_values(gen, (len(occ_rows), width)).double().numpy()
  return w, state, occ_rows, c, g


def _rounded_table(out):
  return {k: v.float().numpy() for k, v in out.items()}


def _applies(kind, defect):
  """Whether a modelled defect changes this optimizer's result at all."""
  return not (defect == "bias_t_minus_1" and kind != "adam" or
              defect == "eps_in_sqrt" and kind == "sgd" or
              defect == "rowwise_acc_without_decay" and kind != "rowwise_adagrad" or
              defect == "duplicate_applied_twice" and kind == "sgd")


@pytest.mark.parametrize("kind,defect", [(k, d) for k in KINDS for d in TABLE_DEFECTS
                                         if _applies(k, d)])
def test_bounds_catch_defects(kind, defect):
  """The exactly rounded result passes every bound; each modelled defect fails it."""
  w, state, occ_rows, c, g = _selfcheck_inputs(kind)
  t = 2 if kind == "adam" else 1
  cfg = {"eps": 1e-3 if defect == "eps_in_sqrt" else 1e-7, "beta1": 0.9, "beta2": 0.999,
         "weight_decay": WD}
  vals = c[:, None] * g
  out, bound, _ = table_step(kind, w, state, occ_rows, vals, 1.0, 0.05, t, cfg)
  assert worst_table_ratio(out, bound, _rounded_table(out)) <= 1.0
  if defect == "mean_weight_dropped":
    bad, _, _ = table_step(kind, w, state, occ_rows, g, 1.0, 0.05, t, cfg)
  else:
    bad, _, _ = table_step(kind, w, state, occ_rows, vals, 1.0, 0.05, t, cfg, defect=defect)
  assert worst_table_ratio(out, bound, _rounded_table(bad)) > 1.0, defect
