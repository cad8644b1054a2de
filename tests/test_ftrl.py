"""FTRL-Proximal (``set_optimizer("ftrl")``): accumulator n and linear term z, both element-wise.

Every step is checked against the float64 model below, with bounds from operation counts, on the
engine's own weights and state (the driver of ``test_fused_optimizers.py`` with FTRL's state).

CPU (no GPU): the bound self-check (the exact result passes, one modelled defect per formula term
fails), the plan interpreter at world 1-8 (whole, column- and row-sliced tables, mean pooling,
duplicate, out-of-range and ragged ids, zero-gradient rows, every hyperparameter, 16-bit tables and
bf16 state against the rounding rule), a learning rate of zero, ``SparseRowOptimizer`` against the
model and against the interpreter, optimizer-state round trips, dry updates, argument checks and
the DLRM example's convergence.

GPU (one H100): every kernel route (balanced, crossing segments under skewed ids, per-row with
4 or 1 columns per lane) with fp32, bf16 and fp16 tables and fp32 or bf16 state, a learning rate
of zero, the fused against the torch back end, cached against uncached training and
``DLRMTrainStep`` (CUDA graph, warm-up schedule from lr = 0) against ``HybridTrainer``.
"""
import numpy as np
import pytest
import torch

import distributed_embeddings_b200 as de
from distributed_embeddings_b200.parallel import dry_run
from distributed_embeddings_b200.parallel.hybrid import SparseRowOptimizer
import test_fused_optimizers as tfo  # pylint: disable=wrong-import-order
from optim_reference import (TINY, U, _e_sum, f32,  # pylint: disable=wrong-import-order
                             half_within, worst_table_ratio)
from test_dry_run import assemble  # pylint: disable=wrong-import-order
from test_examples_smoke import run as run_example  # pylint: disable=wrong-import-order

KIND = "ftrl"
WD = tfo.WD
INIT_ACC = 0.1
INIT_ACC_F32 = f32(INIT_ACC)
# every term of the update switched on, and the Keras defaults
ALL_TERMS = {"lr_power": -0.3, "l1": 0.5, "l2": 0.25, "l2_shrinkage": 0.125, "beta": 0.75}
DEFAULTS = {"lr_power": -0.5, "l1": 0.0, "l2": 0.0, "l2_shrinkage": 0.0, "beta": 0.0}


# ------------------------------------------------------------------ float64 model
# One defect per formula term: sigma from P(n') alone, the shrinkage term in the gradient that feeds
# n, l2 without its factor 2, beta not divided by lr, duplicate ids applied one by one.
FTRL_DEFECTS = ("sigma_not_difference", "shrinkage_in_accumulator", "l2_without_2",
                "beta_without_lr", "duplicates_one_by_one")


def _pw(x, lr_power):
  """P(x) = x^(-lr_power) in float64."""
  return x.clamp_min(0).sqrt() if lr_power == -0.5 else x.clamp_min(0).pow(-lr_power)


def _soft(z, q, l1):
  """Step 6: (sign(z) l1 - z) / q where |z| > l1, else 0."""
  return torch.where(z.abs() > l1, (torch.sign(z) * l1 - z) / q, torch.zeros_like(z))


def ftrl_update(w, gp, e_gp, n, z, lr, cfg, defect=None):
  """FTRL on the touched rows from their decayed gradient ``gp`` ([R, W] float64, known to within
  ``e_gp`` of what the kernel computes).  Returns (out, bound) for 'p', 's0' (n) and 's1' (z).

  Bounds, from the kernel's fp32 operations: n' = fma(g, g, n) is exactly rounded; P of n' moves
  with n' (the envelope at n' -/+ e_n) and rounds once (sqrt) or within 4 ulps (powf); sigma
  subtracts and divides (two roundings); z adds four terms (five roundings at most, each within
  u of the sum of the magnitudes); q adds, divides and adds.  Step 6 is continuous and monotone
  in z and, for fixed z, in q, so its input error is the envelope over z -/+ e_z, q -/+ e_q; its
  own subtraction and division add two roundings.  At lr = 0 nothing moves (bound 0)."""
  lr = f32(lr)
  c = {k: f32(cfg[k]) for k in DEFAULTS}
  if lr == 0.0:
    return ({"p": w.clone(), "s0": n.clone(), "s1": z.clone()},
            {"p": torch.zeros_like(w), "s0": torch.zeros_like(n), "s1": torch.zeros_like(z)})
  k_pow = U if c["lr_power"] == -0.5 else 8 * U
  g_n = gp + 2 * c["l2_shrinkage"] * w if defect == "shrinkage_in_accumulator" else gp
  n_new = n + g_n * g_n
  e_n = 2 * gp.abs() * e_gp + e_gp * e_gp + U * n_new.abs() + TINY
  p_new, p_old = _pw(n_new, c["lr_power"]), _pw(n, c["lr_power"])
  env_p = torch.maximum((_pw(n_new + e_n, c["lr_power"]) - p_new).abs(),
                        (_pw((n_new - e_n).clamp_min(0), c["lr_power"]) - p_new).abs())
  e_pn = env_p + k_pow * p_new
  e_po = k_pow * p_old
  sigma = p_new / lr if defect == "sigma_not_difference" else (p_new - p_old) / lr
  e_sigma = (e_pn + e_po + U * (p_new - p_old).abs()) / lr + U * sigma.abs()
  shrink = 2 * c["l2_shrinkage"] * w
  z_new = z + gp + shrink - sigma * w
  e_z = (e_gp + w.abs() * e_sigma +
         5 * U * (z.abs() + gp.abs() + shrink.abs() + (sigma * w).abs()) + TINY)
  two_l2 = c["l2"] if defect == "l2_without_2" else 2 * c["l2"]
  if defect == "beta_without_lr":
    q = c["beta"] + p_new / lr + two_l2
  else:
    q = (c["beta"] + p_new) / lr + two_l2
  e_q = e_pn / lr + 3 * U * q.abs()
  w_new = _soft(z_new, q, c["l1"])
  corners = [_soft(z_new + sz * e_z, q + sq * e_q, c["l1"]) for sz in (-1, 1) for sq in (-1, 1)]
  env_w = torch.stack([(x - w_new).abs() for x in corners]).amax(0)
  e_w = env_w + 3 * U * (z_new.abs() + e_z + c["l1"]) / (q - e_q).clamp_min(TINY)
  out = {"p": w_new, "s0": n_new, "s1": z_new}
  bound = {"p": 1.05 * e_w + TINY, "s0": 1.05 * e_n, "s1": 1.05 * e_z}
  return out, bound


def table_step(weights, state, occ_rows, occ_vals, scale, lr, cfg, defect=None):
  """One lazy FTRL step on a whole table, with bounds: the contract of
  ``optim_reference.table_step`` (the gradient of each touched row summed from its occurrences
  within (n + 2) u |s| sum |c_k g_k|, then one fma of the decay), ``state`` = [n, z], both
  [rows, W].  Untouched rows get a bound of zero.  Returns (out, bound, touched)."""
  w = torch.as_tensor(np.asarray(weights, dtype=np.float64))
  rows = w.shape[0]
  occ_rows = np.asarray(occ_rows, dtype=np.int64)
  vals = torch.as_tensor(np.asarray(occ_vals, dtype=np.float64))
  s = f32(scale)
  wd = f32(cfg.get("weight_decay", 0.0))
  st = [torch.as_tensor(np.asarray(x, dtype=np.float64)) for x in state]
  touched = np.zeros(rows, dtype=bool)
  touched[occ_rows] = True
  idx = torch.as_tensor(np.nonzero(touched)[0])
  occ = torch.as_tensor(occ_rows)
  gsum = torch.zeros_like(w).index_add_(0, occ, vals)
  gabs = torch.zeros_like(w).index_add_(0, occ, vals.abs())
  n_occ = torch.zeros(rows, dtype=torch.float64).index_add_(
      0, occ, torch.ones(len(occ_rows), dtype=torch.float64))
  out = {"p": w.clone(), "s0": st[0].clone(), "s1": st[1].clone()}
  bound = {k: torch.zeros_like(x) for k, x in out.items()}
  if defect == "duplicates_one_by_one":
    for r, v in zip(occ_rows, vals):
      g = s * v[None] + wd * out["p"][r:r + 1]
      o, _ = ftrl_update(out["p"][r:r + 1], g, torch.zeros_like(g), out["s0"][r:r + 1],
                         out["s1"][r:r + 1], lr, cfg)
      for k in out:
        out[k][r] = o[k][0]
    return out, bound, touched
  gp = s * gsum[idx] + wd * w[idx]
  e_gp = _e_sum(s, n_occ[idx], gabs[idx]) + U * gp.abs() + TINY
  o, b = ftrl_update(w[idx], gp, e_gp, st[0][idx], st[1][idx], lr, cfg, defect=defect)
  for k in o:
    out[k][idx] = o[k]
    bound[k][idx] = b[k]
  return out, bound, touched


def _cfg(hp=None, wd=0.0):
  return dict(DEFAULTS, **(hp or {}), weight_decay=wd)


# ------------------------------------------------------------------ driver
def _initial_state(rows, width, sdt=torch.float32):
  n0 = float(torch.tensor(INIT_ACC, dtype=sdt).float())  # bf16 state: 0.1 rounded to nearest
  return [np.full((rows, width), n0, np.float32), np.zeros((rows, width), np.float32)]


def _state_of(demb, t, rows, width, sdt):
  st = demb.get_optimizer_state()
  if st["tables"] is None:
    return _initial_state(rows, width, sdt)
  n, z = st["tables"][t]
  assert n.shape == z.shape == (rows, width)
  return [np.asarray(n, dtype=np.float32), np.asarray(z, dtype=np.float32)]


def _check_step(case, out, bound, touched, after, state_after, slack, weights_only):
  bound = {k: slack * b for k, b in bound.items()}
  got = {"p": after}
  if weights_only:
    out, bound = {"p": out["p"]}, {"p": bound["p"]}
  else:
    got["s0"], got["s1"] = state_after
  tdt = case.get("table_dtype", torch.float32)
  sdt = case.get("state_dtype", torch.float32)
  idx = np.nonzero(touched)[0]
  for k in out:
    g = torch.as_tensor(np.asarray(got[k], dtype=np.float64))
    unt = ~torch.as_tensor(touched)
    assert torch.equal(g[unt], out[k][unt]), f"untouched rows of {k} changed"
    dt = tdt if k == "p" else sdt
    if dt == torch.float32:
      r = worst_table_ratio({k: out[k][idx]}, {k: bound[k][idx]}, {k: g[idx].numpy()})
      assert r <= 1.0, f"{k}: worst error / bound {r}"
    else:
      bad = half_within(g[idx], out[k][idx], bound[k][idx], dt, case["step"] + 1, idx,
                        {"p": 0, "s0": 1, "s1": 2}[k])
      assert bad == 0, f"{k}: {bad} 16-bit values outside the rounding of the bound"


def _run(case, world=1, dev=None, plan=None, route=None):
  """``case`` for ``len(case['lrs'])`` steps, every step checked; ``case['hp']``: FTRL's
  hyperparameters; ``plan``: extra DistributedEmbedding arguments (slicing)."""
  embs = [{"input_dim": r, "output_dim": w, "combiner": c} for r, w, c in case["tables"]]
  kw = dict(input_table_map=list(case["imap"]), strategy="basic")
  kw.update(plan or {})
  if case.get("table_dtype", torch.float32) != torch.float32:
    kw["table_dtype"] = case["table_dtype"]
  if case.get("compute_dtype"):
    kw["compute_dtype"] = case["compute_dtype"]
  hp = case.get("hp", {})
  opt = dict(hp, weight_decay=case.get("wd", 0.0))
  sdt = case.get("state_dtype", torch.float32)
  if sdt != torch.float32:
    opt["state_dtype"] = sdt
  cdt = case.get("compute_dtype", torch.float32)
  torch.manual_seed(case.get("seed", 0))
  if dev is None:
    sim, des = dry_run.build_engines(embs, world, dp_input=True, **kw)
  else:
    sim, des = None, [de.DistributedEmbedding(embs, device=dev, backend="fused", world_size=1,
                                              rank=0, **kw)]
  gen = np.random.default_rng(case.get("seed", 0))
  tables = [gen.standard_normal((r, w)).astype(np.float32) for r, w, _ in case["tables"]]
  for d in des:
    d.set_weights(tables)
    d.set_optimizer(KIND, lr=case["lrs"][0], **opt)
    if any(h == "ragged" for h in case["hots"]):
      d.ragged_capacity = 8
  demb = des[0]
  routes = []
  assert world == 1 or len(case["lrs"]) == 1
  zeros = 0
  for step, lr in enumerate(case["lrs"]):
    if step and lr != case["lrs"][step - 1]:
      for d in des:
        d.set_learning_rate(lr)
    ids, grad = tfo._draw(case, step)
    grad = grad.to(cdt)
    lb = case["batch"] // world
    before = tfo._weights(des, world)
    states = [_state_of(demb, t, r, w, sdt) if world == 1 else _initial_state(r, w, sdt)
              for t, (r, w, _) in enumerate(case["tables"])]

    def rank_fn(r):
      d = des[r]
      out = d(tfo._as_inputs(case, ids, d.device if dev is None else dev, r * lb, (r + 1) * lb),
              concat=True)
      eng = d._engine
      if not isinstance(eng.ops, tfo._Counting):
        eng.ops = tfo._Counting(eng.ops)
      out.backward(grad[r * lb:(r + 1) * lb].to(out.device))
      return eng.ops.routes
    if dev is None:
      routes = list(dry_run.run_ranks(sim, rank_fn)[0])
    else:
      routes = list(rank_fn(0))
      torch.cuda.synchronize()
    if case.get("edges"):
      tfo._check_edge_layout(case, ids, des[0]._engine)
    after = tfo._weights(des, world)
    for t, (r, w, _) in enumerate(case["tables"]):
      occ = tfo._occurrences(case, ids, grad.float(), t)
      out, bound, touched = table_step(before[t], states[t], occ[0], occ[1], 1.0 / world, lr,
                                       _cfg(hp, case.get("wd", 0.0)))
      sa = _state_of(demb, t, r, w, sdt) if world == 1 else None
      # the interpreter computes in torch fp32 ops without fma: three times the kernel's bounds
      _check_step(dict(case, step=step), out, bound, touched, after[t], sa,
                  slack=3.0 if dev is None else 1.0, weights_only=world > 1)
      zeros += int((after[t][touched] == 0.0).sum())
  if hp.get("l1", 0.0) > 0 and all(lr > 0 for lr in case["lrs"]):
    assert zeros > 0, "l1 > 0 left no weight at exactly zero"
  want = route or tfo._expected_route(case, KIND)
  assert routes and set(routes) <= ({want} if want != "any" else
                                    {"balanced", "per_row_vec4", "per_row_vec1"}), (routes, want)
  return des


_case, _with = tfo._case, tfo._with


# ------------------------------------------------------------------ CPU: the float64 model
def _selfcheck_inputs(seed=40):
  gen = torch.Generator().manual_seed(seed)
  rows, width = 64, 16
  w = torch.randn(rows, width, generator=gen).numpy()
  n = (INIT_ACC + torch.rand(rows, width, generator=gen) * 4).numpy()  # after earlier steps
  z = torch.randn(rows, width, generator=gen).numpy()
  occ_rows = np.concatenate([np.full(c, r + 1) for r, c in enumerate([1, 2, 5, 33])] +
                            [np.arange(10, 40)])
  k = np.where(np.arange(len(occ_rows)) % 2 == 0, 1, 3)  # pooling of 1 or 3 ids (mean)
  c = np.asarray([f32(1.0 / x) for x in k])
  g = tfo._grad_values(gen, (len(occ_rows), width)).double().numpy() * 1e-2
  return w, [n, z], occ_rows, c[:, None] * g


@pytest.mark.parametrize("lr_power", [-0.5, -0.3])
@pytest.mark.parametrize("defect", FTRL_DEFECTS)
def test_bounds_catch_defects(defect, lr_power):
  """The exactly rounded result passes every bound; each modelled defect fails it."""
  w, state, occ_rows, vals = _selfcheck_inputs()
  cfg = _cfg(dict(ALL_TERMS, l1=0.05, lr_power=lr_power), WD)
  out, bound, touched = table_step(w, state, occ_rows, vals, 1.0, 0.05, cfg)
  assert touched[1] and not touched[0]
  assert worst_table_ratio(out, bound, tfo._rounded_table(out)) <= 1.0
  assert (out["p"][torch.as_tensor(touched)] == 0).any(), "l1 zeroes some weights"
  bad, _, _ = table_step(w, state, occ_rows, vals, 1.0, 0.05, cfg, defect=defect)
  assert worst_table_ratio(out, bound, tfo._rounded_table(bad)) > 1.0, defect


def test_model_matches_keras_closed_form():
  """With l1 = l2 = beta = shrinkage = 0 and lr_power = -0.5 the weight is -z lr / sqrt(n')."""
  w, state, occ_rows, vals = _selfcheck_inputs()
  out, _, touched = table_step(w, state, occ_rows, vals, 1.0, 0.05, _cfg())
  t = torch.as_tensor(touched)
  torch.testing.assert_close(out["p"][t], -out["s1"][t] * f32(0.05) / out["s0"][t].sqrt(),
                             rtol=1e-12, atol=0)


def test_zero_learning_rate_moves_nothing():
  w, state, occ_rows, vals = _selfcheck_inputs()
  out, bound, _ = table_step(w, state, occ_rows, vals, 1.0, 0.0, _cfg(ALL_TERMS, WD))
  assert all(float(b.abs().max()) == 0 for b in bound.values())
  np.testing.assert_array_equal(out["p"].numpy(), w)


# ------------------------------------------------------------------ CPU: the plan interpreter
TABLES = [(200, 16, "sum"), (150, 8, "mean"), (90, 12, "sum"), (80, 8, "sum")]
PLANS = {"whole": None, "column_slices": {"column_slice_threshold": 1000},
         "row_slices": {"row_slice_threshold": 1500}}
HPS = {"defaults": ({}, 0.0), "all_terms": (ALL_TERMS, WD)}


@pytest.mark.parametrize("world", [1, 2, 3, 4, 5, 6, 7, 8])
@pytest.mark.parametrize("plan", sorted(PLANS))
@pytest.mark.parametrize("hp", sorted(HPS))
def test_interpreter_against_float64(world, plan, hp):
  case = _case(TABLES, [0, 1, 2, 3, 0], [1, 2, 1, 3, 2], 840, hp=HPS[hp][0], wd=HPS[hp][1],
               seed=20 + world)
  des = _run(case, world=world, plan=PLANS[plan], route="any" if PLANS[plan] else None)
  st = des[0].strategy
  if plan == "row_slices" and world > 1:
    assert st.table_groups[2]


@pytest.mark.parametrize("name", ["mixed", "wide", "odd", "skewed", "keras_defaults"])
def test_interpreter_routes_against_float64(name):
  """World 1: the balanced route with crossing segments (1 ... 300 occurrences, a zero-gradient
  row), rows wider than 128, widths that are not a multiple of 4, power-law ids; two steps."""
  case = {"mixed": _with(tfo.MIXED, wd=WD, hp=ALL_TERMS, lrs=[0.05, 0.02]),
          "wide": _with(tfo.WIDE, wd=WD, hp=dict(ALL_TERMS, lr_power=-0.5)),
          "odd": _with(tfo.ODD, wd=0.0, hp=ALL_TERMS),
          "skewed": _case([(500, 32, "mean")] * 2, [0, 1, 0], [1, 7, 3], 512, power_law=True,
                          lrs=[0.1], wd=WD, hp=ALL_TERMS, seed=11),
          "keras_defaults": _with(tfo.MIXED, lrs=[0.05, 0.05])}[name]
  _run(case, world=1)


@pytest.mark.parametrize("table_dtype,state_dtype", [(torch.float32, torch.bfloat16),
                                                     (torch.bfloat16, torch.float32),
                                                     (torch.float16, torch.bfloat16)])
def test_interpreter_16_bit_against_the_rounding_rule(table_dtype, state_dtype):
  case = _case([(600, 32, "sum")], [0, 0], [1, 2], 512, edges=True, wd=WD, hp=ALL_TERMS,
               table_dtype=table_dtype, state_dtype=state_dtype, lrs=[0.05, 0.05], seed=5)
  _run(case, world=1)


def test_interpreter_zero_learning_rate_leaves_everything_bit_identical():
  """The first step of a warm-up schedule (lr = 0): weights, n and z keep their bits, after a
  real step and with 16-bit tables and state."""
  case = _case([(600, 32, "sum")], [0, 0], [1, 2], 512, edges=True, wd=WD, hp=ALL_TERMS,
               table_dtype=torch.bfloat16, state_dtype=torch.bfloat16, lrs=[0.05, 0.0], seed=6)
  _run(case, world=1)
  _run(_with(tfo.MIXED, wd=WD, hp=ALL_TERMS, lrs=[0.0]), world=1)


def _sparse_steps(p, steps=2, seed=31, width=12):
  gen = torch.Generator().manual_seed(seed)
  out = []
  for step in range(steps):
    idx = torch.randint(0, 30 + 10 * step, (80,), generator=gen)
    idx[:5] = 7
    vals = tfo._grad_values(gen, (80, width)).to(p.dtype).float()
    vals[:5] = 0.0
    out.append((idx, vals))
  return out


@pytest.mark.parametrize("hp", sorted(HPS))
def test_sparse_row_optimizer_against_float64(hp):
  """The torch back end's row-sparse optimizer: two steps with duplicate ids and a row touched
  only by zero gradients, then a step at lr = 0."""
  torch.manual_seed(30)
  rows, width = 60, 12
  p = torch.nn.Parameter(torch.randn(rows, width))
  params, wd = HPS[hp]
  opt = SparseRowOptimizer([p], KIND, lr=0.05, weight_decay=wd, **params)
  assert [s.shape for s in opt.state[0]] == [(rows, width)] * 2
  state = _initial_state(rows, width)
  cfg = _cfg(params, wd)
  for step, (idx, vals) in enumerate(_sparse_steps(p, steps=3)):
    lr = 0.0 if step == 2 else 0.05
    opt.set_lr(lr)
    p.grad = torch.sparse_coo_tensor(idx[None], vals, (rows, width))
    before = p.detach().numpy().copy()
    out, bound, touched = table_step(before, state, idx.numpy(), vals.double().numpy(), 1.0, lr,
                                     cfg)
    opt.step()
    got = {"p": p.detach().numpy(), "s0": opt.state[0][0].numpy(), "s1": opt.state[0][1].numpy()}
    r = worst_table_ratio(out, {k: 3 * b for k, b in bound.items()}, got)
    assert r <= 1.0 and touched[7], r
    state = [got["s0"].copy(), got["s1"].copy()]


@pytest.mark.parametrize("table_dtype,state_dtype", [(torch.float32, torch.float32),
                                                     (torch.bfloat16, torch.bfloat16)])
def test_sparse_row_optimizer_matches_the_interpreter(table_dtype, state_dtype):
  """The same steps through SparseRowOptimizer and the plan interpreter (one table, one rank, ids
  as single-id samples): fp32 results agree to rounding, 16-bit ones within one ulp."""
  rows, width = 60, 12
  w0 = np.random.default_rng(3).standard_normal((rows, width)).astype(np.float32)
  p = torch.nn.Parameter(torch.from_numpy(w0.copy()).to(table_dtype))
  opt = SparseRowOptimizer([p], KIND, lr=0.05, weight_decay=WD, state_dtype=state_dtype,
                           **ALL_TERMS)
  steps = _sparse_steps(p)
  for idx, vals in steps:
    p.grad = torch.sparse_coo_tensor(idx[None], vals.to(table_dtype), (rows, width))
    opt.step()
  sim, des = dry_run.build_engines([{"input_dim": rows, "output_dim": width, "combiner": "sum"}],
                                   1, dp_input=True, table_dtype=table_dtype)
  d = des[0]
  d.set_weights([w0])
  kw = {} if state_dtype == torch.float32 else {"state_dtype": state_dtype}
  d.set_optimizer(KIND, lr=0.05, weight_decay=WD, **ALL_TERMS, **kw)
  for idx, vals in steps:
    def fn(r):  # pylint: disable=unused-argument
      out = d([idx[:, None]], concat=True)
      out.backward(vals)
    dry_run.run_ranks(sim, fn)
  got = d.get_weights()[0]
  st = d.get_optimizer_state()["tables"][0]
  want = p.detach().float().numpy()
  if table_dtype == torch.float32:
    np.testing.assert_allclose(got, want, rtol=1e-5, atol=1e-6)
    for k in range(2):
      # z sums terms of up to a few hundred that cancel: compare at the scale of the terms
      ref = opt.state[0][k].float().numpy()
      np.testing.assert_allclose(st[k], ref, rtol=1e-5, atol=1e-6 * np.abs(ref).max())
  else:
    # the same rounding rule and keys; where the fp32 values before a rounding differ in their
    # last bits the decision can flip, and a flipped bf16 z (ulp 2 at |z| ~ 400) moves the next
    # step's weight by ulp(z) / q
    assert (got == want).mean() > 0.9
    assert np.abs(got - want).max() < 1e-2


# ------------------------------------------------------------------ CPU: optimizer state
SIZES = [(30, 8), (12, 16), (50, 8), (21, 16), (64, 8)]


def _plan_engines(world, weights, state_dtype=torch.float32, **kw):
  embs = [{"input_dim": r, "output_dim": w, "combiner": "sum"} for r, w in SIZES]
  sim, des = dry_run.build_engines(embs, world, strategy="memory_balanced", **kw)
  for d in des:
    d.set_weights(weights)
    d.set_optimizer(KIND, lr=0.3, weight_decay=0.1, state_dtype=state_dtype, **ALL_TERMS)
  return sim, des


def _batches(n=2, gb=8, seed=11):
  rng = np.random.default_rng(seed)
  return [([rng.integers(0, r, size=(gb, 2)) for r, _ in SIZES],
           [rng.standard_normal((gb, w)).astype(np.float32) * 0.1 for _, w in SIZES])
          for _ in range(n)]


def _step(sim, des, batch):
  ids, grads = batch
  world = len(des)
  lb = ids[0].shape[0] // world

  def fn(r):
    sl = slice(r * lb, (r + 1) * lb)
    out = des[r]([torch.from_numpy(i[sl]) for i in ids], concat=True)
    out.backward(torch.from_numpy(np.concatenate([g[sl] for g in grads], 1)) * world / 8)
  dry_run.run_ranks(sim, fn)


def _gather(sim, des, fn):
  return dry_run.run_ranks(sim, lambda r: fn(des[r]))[0]


@pytest.mark.parametrize("state_dtype", [torch.float32, torch.bfloat16])
def test_optimizer_state_resharding(state_dtype, tmp_path):
  """Global state layout: n and z ``[rows, width]`` each.  One step on 8 ranks with column-sliced
  tables, state and weights loaded into 4 ranks with a row-sliced table, a second step there ==
  two uninterrupted steps on the 4-rank plan; in memory and through files."""
  rng = np.random.default_rng(11)
  tables = [rng.standard_normal(s).astype(np.float32) for s in SIZES]
  batches = _batches()
  kw4 = {"row_slice_threshold": 500}
  sim_a, des_a = _plan_engines(4, tables, state_dtype, **kw4)
  _step(sim_a, des_a, batches[0])
  _step(sim_a, des_a, batches[1])
  straight = _gather(sim_a, des_a, lambda d: d.get_weights())
  straight_s = _gather(sim_a, des_a, lambda d: d.get_optimizer_state())

  sim_b, des_b = _plan_engines(8, tables, state_dtype, column_slice_threshold=100)
  _step(sim_b, des_b, batches[0])
  saved_w = _gather(sim_b, des_b, lambda d: d.get_weights())
  saved_s = _gather(sim_b, des_b, lambda d: d.get_optimizer_state())
  assert saved_s["step"] == 1 and saved_s["kind"] == KIND
  for t, (rows, w) in enumerate(SIZES):
    n, z = saved_s["tables"][t]
    assert n.shape == z.shape == (rows, w)
    assert (n >= 0.09).all() and (n > 0.1).any() and (z != 0).any()

  sim_c, des_c = _plan_engines(4, saved_w, state_dtype, **kw4)

  def load(r):
    des_c[r]._engine.prepare(8, [2] * len(SIZES))
    des_c[r].set_optimizer_state(saved_s)
  dry_run.run_ranks(sim_c, load)
  _step(sim_c, des_c, batches[1])
  resumed = _gather(sim_c, des_c, lambda d: d.get_weights())
  resumed_s = _gather(sim_c, des_c, lambda d: d.get_optimizer_state())
  # bf16 state: the 8- and 4-rank runs round n and z with different row keys
  tol = dict(rtol=2e-5, atol=2e-6) if state_dtype == torch.float32 else dict(rtol=2e-2, atol=2e-3)
  for a, b in zip(straight, resumed):
    np.testing.assert_allclose(b, a, **tol)
  for ta, tb in zip(straight_s["tables"], resumed_s["tables"]):
    for a, b in zip(ta, tb):
      np.testing.assert_allclose(b, a, **tol)

  ckpt = str(tmp_path / "ckpt")

  def save(r):
    des_b[r].save_weights(ckpt, chunk=64)
    return des_b[r].save_optimizer_state(ckpt, chunk=64)
  metas = dry_run.run_ranks(sim_b, save)
  assert all(m == metas[0] and m.endswith("optimizer.json") for m in metas)
  for t in range(len(SIZES)):
    for k, arr in enumerate(saved_s["tables"][t]):
      np.testing.assert_array_equal(np.load(f"{ckpt}/opt_{t}_slot{k}.npy"), arr)
  sim_d, des_d = _plan_engines(4, tables, state_dtype, **kw4)

  def load_files(r):
    des_d[r]._engine.prepare(8, [2] * len(SIZES))
    des_d[r].load_weights(ckpt)
    des_d[r].load_optimizer_state(ckpt)
  dry_run.run_ranks(sim_d, load_files)
  assert des_d[0]._engine.step_count() == 1
  loaded_s = _gather(sim_d, des_d, lambda d: d.get_optimizer_state())
  for ta, tb in zip(saved_s["tables"], loaded_s["tables"]):
    for a, b in zip(ta, tb):
      np.testing.assert_array_equal(b, a)
  _step(sim_d, des_d, batches[1])
  for a, b in zip(resumed, _gather(sim_d, des_d, lambda d: d.get_weights())):
    np.testing.assert_array_equal(b, a)


def test_state_of_another_kind_is_rejected():
  rng = np.random.default_rng(6)
  tables = [rng.standard_normal(s).astype(np.float32) for s in SIZES]
  sim, des = _plan_engines(1, tables)
  _step(sim, des, _batches(1, gb=4)[0])
  state = des[0].get_optimizer_state()
  des[0].set_optimizer("adam", lr=0.1)
  _step(sim, des, _batches(1, gb=4)[0])
  adam = des[0].get_optimizer_state()
  assert [a.shape for a in adam["tables"][0]] == [a.shape for a in state["tables"][0]]
  with pytest.raises(ValueError, match="does not match"):
    des[0].set_optimizer_state(state)
  des[0].set_optimizer(KIND, lr=0.1)
  with pytest.raises(ValueError, match="does not match"):
    des[0].set_optimizer_state(adam)
  des[0].set_optimizer_state(state)


@pytest.mark.parametrize("weight_decay", [0.0, 0.5])
def test_dry_updates_leave_tables_and_optimizer_state_untouched(weight_decay):
  """Dry passes (graph warm-up, zero gradient) on live state after a real step: tables, n, z and
  the step count come out bit-identical (FTRL's closed form would reset the weights); the next
  real step equals one taken without the dry passes."""
  rng = np.random.default_rng(4)
  tables = [rng.standard_normal(s).astype(np.float32) for s in SIZES]
  batches = _batches(3, seed=12)

  def make():
    sim, des = _plan_engines(2, tables, column_slice_threshold=100)
    for d in des:
      d.set_optimizer(KIND, lr=0.3, weight_decay=weight_decay, **ALL_TERMS)
    return sim, des
  sim_a, des_a = make()
  _step(sim_a, des_a, batches[0])
  w1 = assemble(des_a)
  st1 = [{m: [s.clone() for s in v] for m, v in d._engine.opt_state.items()} for d in des_a]
  for d in des_a:
    d._engine.dry_updates(True)
  _step(sim_a, des_a, batches[1])
  _step(sim_a, des_a, batches[2])
  for got, want in zip(assemble(des_a), w1):
    np.testing.assert_array_equal(got, want)
  for d, before in zip(des_a, st1):
    assert d._engine.step_count() == 1
    for m, slots in before.items():
      for a, b in zip(slots, d._engine.opt_state[m]):
        assert torch.equal(a, b)
    d._engine.dry_updates(False)
  _step(sim_a, des_a, batches[1])
  sim_b, des_b = make()
  _step(sim_b, des_b, batches[0])
  _step(sim_b, des_b, batches[1])
  for a, b in zip(assemble(des_a), assemble(des_b)):
    np.testing.assert_array_equal(a, b)


def test_arguments():
  d = de.DistributedEmbedding([{"input_dim": 10, "output_dim": 8, "combiner": "sum"}],
                              device="cpu", backend="torch", world_size=1, rank=0)
  d.set_optimizer(KIND, lr=0.1)
  cfg = d._fused_optimizer
  assert {k: cfg[k] for k in DEFAULTS} == DEFAULTS
  assert (cfg["initial_accumulator_value"], cfg["weight_decay"]) == (0.1, 0.0)
  d.set_optimizer(KIND, lr=0.1, state_dtype=torch.bfloat16, weight_decay=0.1,
                  initial_accumulator_value=0.0, **ALL_TERMS)
  d.set_optimizer(KIND, lr=0.1, lr_power=0.0)
  for bad in ({"lr_power": 0.5}, {"l1": -1.0}, {"l2": -0.1}, {"l2_shrinkage": -0.1},
              {"beta": -1.0}, {"initial_accumulator_value": -0.1}):
    with pytest.raises(ValueError, match="ftrl"):
      d.set_optimizer(KIND, lr=0.1, **bad)
    with pytest.raises(ValueError, match="ftrl"):
      SparseRowOptimizer([torch.nn.Parameter(torch.zeros(5, 4))], KIND, **bad)
  for other in ("sgd", "adagrad", "rowwise_adagrad", "adam", "rowwise_adam"):
    for key in DEFAULTS:
      with pytest.raises(ValueError, match="unknown fused optimizer argument"):
        d.set_optimizer(other, lr=0.1, **{key: DEFAULTS[key]})
      with pytest.raises(ValueError, match="unknown fused optimizer argument"):
        SparseRowOptimizer([torch.nn.Parameter(torch.zeros(5, 4))], other, **{key: 0.0})
  with pytest.raises(ValueError, match="torch.float32 or torch.bfloat16"):
    d.set_optimizer(KIND, lr=0.1, state_dtype=torch.float16)
  with pytest.raises(ValueError, match="offload_cache_size"):
    de.DistributedEmbedding([{"input_dim": 1000, "output_dim": 8, "combiner": "sum"}],
                            device="cpu", world_size=1, rank=0, offload_cache_size=100,
                            gpu_embedding_size=10).set_optimizer(KIND, lr=0.1,
                                                                  state_dtype=torch.bfloat16)
  p = torch.nn.Parameter(torch.zeros(5, 4, dtype=torch.bfloat16))
  opt = SparseRowOptimizer([p], KIND, state_dtype=torch.bfloat16)
  assert [s.dtype for s in opt.state[0]] == [torch.bfloat16] * 2
  assert float(opt.state[0][0][0, 0]) == float(torch.tensor(0.1, dtype=torch.bfloat16))


def test_dlrm_example_learns_with_ftrl(tmp_path):
  """The DLRM example's convergence run (generated learnable dataset, three epochs) with
  ``--embedding_optimizer ftrl`` and a warm-up that starts at lr = 0: the evaluation AUC climbs
  well above 0.7."""
  data = str(tmp_path / "criteo")
  run_example(["tools/make_synthetic_criteo.py", data, "--train", "16384", "--test", "4096",
               "--table_sizes", "5,300,7000,40,900,60,15,2000"])
  out = run_example(["examples/dlrm/main.py", "--dataset_path", data, "--batch_size", "256",
                     "--embedding_dim", "16", "--bottom_mlp_dims", "32,16", "--top_mlp_dims",
                     "64,32,1", "--learning_rate", "0.05", "--warmup_steps", "20",
                     "--decay_start_step", "100000", "--epochs", "3", "--embedding_optimizer",
                     KIND, "--save_path", str(tmp_path / "w")], timeout=900)
  auc = float(out.split("AUC:")[1].split(",")[0])
  assert auc > 0.7, out[-500:]


# ------------------------------------------------------------------ GPU (one H100)
GPU_CASES = []
for _hp in sorted(HPS):
  _p, _wd = HPS[_hp]
  GPU_CASES += [(f"balanced-{_hp}", _with(tfo.MIXED, wd=_wd, hp=_p, lrs=[0.05, 0.02])),
                (f"per_row_vec4-{_hp}", _with(tfo.WIDE, wd=_wd, hp=_p, lrs=[0.05, 0.02])),
                (f"per_row_vec1-{_hp}", _with(tfo.ODD, wd=_wd, hp=_p, lrs=[0.05, 0.02])),
                (f"small-{_hp}", _with(tfo.SMALL, wd=_wd, hp=_p))]
for _tdt in (torch.float32, torch.bfloat16, torch.float16):
  for _sdt in (torch.float32, torch.bfloat16):
    if _tdt == _sdt == torch.float32:
      continue
    for _w in (32, 192):
      GPU_CASES.append((f"half-{str(_tdt)[6:]}-table-{str(_sdt)[6:]}-state-w{_w}",
                        _case([(600, _w, "sum")], [0, 0], [1, 2], 512, edges=True, wd=WD,
                              hp=ALL_TERMS, table_dtype=_tdt, state_dtype=_sdt,
                              lrs=[0.05, 0.05], seed=5)))
for _cdt in (torch.bfloat16, torch.float16):
  GPU_CASES.append((f"act-{str(_cdt)[6:]}", _with(tfo.MIXED, wd=WD, hp=ALL_TERMS,
                                                  compute_dtype=_cdt)))
GPU_CASES.append(("four-steps-lr-zero-first", _case(
    [(300, 32, "sum"), (100, 16, "mean")], [0, 1], [2, 3], 256, wd=WD, ids32=True, hp=ALL_TERMS,
    touch=[(0, 1 / 3), (1 / 6, 2 / 3), (1 / 2, 1), (0, 2 / 15)], lrs=[0.0, 0.05, 0.01, 0.01],
    seed=9)))
for _name, _base in (("balanced", tfo.MIXED), ("per_row_vec4", tfo.WIDE),
                     ("per_row_vec1", tfo.ODD)):
  GPU_CASES.append((f"lr-zero-{_name}", _with(_base, wd=WD, hp=ALL_TERMS, lrs=[0.05, 0.0])))


@pytest.mark.gpu
@pytest.mark.parametrize("name,case", GPU_CASES, ids=[c[0] for c in GPU_CASES])
def test_gpu_update_routes_against_float64(name, case):  # pylint: disable=unused-argument
  _run(case, dev=torch.device("cuda", 0))


@pytest.mark.gpu
@pytest.mark.parametrize("width", [16, 32, 128])
@pytest.mark.parametrize("combiner", ["sum", "mean"])
def test_gpu_skewed_ids(width, combiner):
  """Power-law ids: segments span many chunks of the balanced update (finalize_crossing)."""
  case = _case([(500, width, combiner)] * 2, [0, 1, 0], [1, 7, 3], 4096, power_law=True,
               lrs=[0.1], wd=WD, hp=ALL_TERMS, seed=11)
  _run(case, dev=torch.device("cuda", 0))


@pytest.mark.gpu
@pytest.mark.parametrize("table_dtype", [torch.float32, torch.bfloat16])
def test_gpu_fused_matches_torch_backend(table_dtype):
  from distributed_embeddings_b200.parallel.dist_model_parallel import DistributedEmbedding
  dev = torch.device("cuda", 0)
  torch.manual_seed(4)
  embs = [{"input_dim": 500, "output_dim": 64, "combiner": "sum"},
          {"input_dim": 300, "output_dim": 16, "combiner": "mean"}]
  w0 = [(np.random.default_rng(i).standard_normal((e["input_dim"], e["output_dim"])) * 0.1)
        .astype(np.float32) for i, e in enumerate(embs)]
  hp = dict(ALL_TERMS, l1=0.01)
  fused = DistributedEmbedding(embs, device=dev, backend="fused", table_dtype=table_dtype,
                               compute_dtype=torch.float32, world_size=1, rank=0)
  fused.set_weights(w0)
  fused.set_optimizer(KIND, lr=0.01, weight_decay=0.01, **hp)
  ref = DistributedEmbedding(embs, device=dev, backend="torch", table_dtype=table_dtype,
                             compute_dtype=torch.float32)
  ref.set_weights(w0)
  opt = SparseRowOptimizer(ref.mp_parameters(), KIND, lr=0.01, weight_decay=0.01, **hp)
  for _ in range(3):
    ids = [torch.randint(0, e["input_dim"], (256, 3), device=dev) for e in embs]
    gout = torch.randn(256, 80, device=dev)
    fused(ids, concat=True).backward(gout)
    ref(ids, concat=True).backward(gout)
    opt.step()
  torch.cuda.synchronize()
  for a, b in zip(fused.get_weights(), ref.get_weights()):
    if table_dtype == torch.float32:
      np.testing.assert_allclose(a, b, rtol=1e-5, atol=1e-6)
    else:
      # the same rounding rule and keys; the fp32 values before the rounding differ in their last
      # bits (gradient summation order), which moves a value by one bf16 ulp where the rounding
      # decision flips
      bad = ~np.isclose(a, b, rtol=2**-6, atol=2e-3)
      assert bad.mean() < 2e-3, bad.mean()
  st = fused.get_optimizer_state()["tables"]
  if table_dtype == torch.float32:
    for t in range(2):
      for k in range(2):
        np.testing.assert_allclose(st[t][k], opt.state[t][k].cpu().numpy(), rtol=1e-5, atol=1e-6)


@pytest.mark.gpu
@pytest.mark.parametrize("skewed", [False, True])
def test_gpu_cached_training_matches_uncached(skewed):
  """fp32 tables and state, a cache far smaller than the working set: tables, n and z equal an
  uncached run to within fp32 rounding (the cached and uncached runs key the sorted update by
  slot id and by row, so the balanced update may sum a row's gradients in another order)."""
  from distributed_embeddings_b200.parallel.dist_model_parallel import DistributedEmbedding
  from distributed_embeddings_b200.parallel.offload_cache import WAYS
  dev = torch.device("cuda", 0)
  small, big, width = 64, 6000, 32
  embs = [{"input_dim": small, "output_dim": width, "combiner": "sum"},
          {"input_dim": big, "output_dim": width, "combiner": "sum"}]
  kw = dict(device=dev, backend="fused", gpu_embedding_size=small * width + 1,
            input_table_map=[0, 1, 1])
  torch.manual_seed(0)
  cached = DistributedEmbedding(embs, offload_cache_size=2 * WAYS * width, **kw)
  plain = DistributedEmbedding(embs, **kw)
  plain.set_weights(cached.get_weights())
  w0 = plain.get_weights()
  for d in (cached, plain):
    d.set_optimizer(KIND, lr=0.05, weight_decay=0.01, **ALL_TERMS)
  for step in range(6):
    g = torch.Generator().manual_seed(100 + step)
    ids = [torch.randint(0, small, (128, 2), generator=g, dtype=torch.int32)]
    for _ in range(2):
      if skewed:
        u = torch.rand(128, 2, generator=g, dtype=torch.float64)
        ids.append((big ** u - 1).floor().clamp(0, big - 1).to(torch.int32))
      else:
        ids.append(torch.randint(0, big, (128, 2), generator=g, dtype=torch.int32))
    ids = [x.to(dev) for x in ids]
    for d in (cached, plain):
      out = d(ids, concat=True)
      (out * torch.linspace(-1, 1, out.shape[1], device=dev)).sum().backward()
  assert cached._engine.caches, "the cache ran"
  for a, b in zip(cached.get_weights(), plain.get_weights()):
    np.testing.assert_allclose(a, b, rtol=1e-5, atol=1e-6)
  assert np.abs(plain.get_weights()[1] - w0[1]).max() > 1e-3, "the offloaded table trained"
  sc, sp = cached.get_optimizer_state(), plain.get_optimizer_state()
  assert sc["step"] == sp["step"] == 6
  for ta, tb in zip(sc["tables"], sp["tables"]):
    for a, b in zip(ta, tb):
      np.testing.assert_allclose(a, b, rtol=1e-5, atol=1e-6)


@pytest.mark.gpu
def test_gpu_dlrm_train_step_matches_hybrid_trainer():
  """DLRMTrainStep (CUDA graph replay) with FTRL and a warm-up schedule whose first step has
  lr = 0 tracks HybridTrainer on the same seeds: the first step moves no table, the second step's
  embedding update and the loss of each of 8 steps agree to bf16-compute accuracy.  The graph
  warm-up passes leave tables, n, z and the step count untouched."""
  from distributed_embeddings_b200.models.dlrm import DLRM
  from distributed_embeddings_b200.models.dlrm_fast import DLRMTrainStep
  from distributed_embeddings_b200.models.trainer import HybridTrainer
  from distributed_embeddings_b200.utils.lr_schedule import LearningRateScheduler
  dev = torch.device("cuda", 0)
  sizes = [300 + 11 * i for i in range(26)]

  def make():
    torch.manual_seed(0)
    return DLRM(sizes, device=dev, compute_dtype=torch.bfloat16, backend="fused")
  ref, fast = make(), make()
  fast.load_state_dict(ref.state_dict())
  fast.embedding.set_weights(ref.embedding.get_weights())
  g = torch.Generator().manual_seed(1)
  batches = [(torch.rand(512, 13, generator=g).to(dev),
              [torch.randint(0, s, (512,), generator=g, dtype=torch.int32).to(dev) for s in sizes],
              torch.randint(0, 2, (512, 1), generator=g).float().to(dev)) for _ in range(8)]
  lr = 0.05
  sched = lambda: LearningRateScheduler(lr, warmup_steps=4, decay_start_step=100, decay_steps=10)
  kw = {"embedding_optimizer_kwargs": dict(ALL_TERMS, l1=1e-4)}
  t_ref = HybridTrainer(ref, lr=lr, embedding_optimizer=KIND, scheduler=sched(), **kw)
  t_fast = DLRMTrainStep(fast, lr=lr, embedding_optimizer=KIND, use_cuda_graph=True,
                         scheduler=sched(), **kw)
  eng = t_fast.engine
  l_ref, l_fast = [], []

  def rel(a, b):
    return float((a - b).norm() / (b.norm() + 1e-12))
  for i, (num, cat, lab) in enumerate(batches):
    e_before = [w.detach().clone() for w in ref.embedding.weights]
    f_before = [w.detach().clone() for w in fast.embedding.weights]
    s_before = {m: [s.clone() for s in v] for m, v in eng.opt_state.items()}
    l_ref.append(float(t_ref.step(num, cat, lab)))
    if i == 2:
      # the dry passes of a graph warm-up on live state (zero lr, dry updates)
      torch.cuda.synchronize()
      step = eng.step_count()
      t_fast.load_batch(num, torch.stack(cat), lab)
      lr_now = float(t_fast.lr_t)
      t_fast.lr_t.zero_()
      eng.dry_updates(True)
      t_fast._step_impl()
      eng.dry_updates(False)
      t_fast.lr_t.fill_(lr_now)
      torch.cuda.synchronize()
      assert eng.step_count() == step == 2
      for m, v in s_before.items():
        for a, b in zip(v, eng.opt_state[m]):
          assert torch.equal(a, b)
      for a, b in zip(f_before, fast.embedding.weights):
        assert torch.equal(a, b.detach())
    l_fast.append(float(t_fast.step(num, torch.stack(cat), lab)))
    torch.cuda.synchronize()
    if i == 0:
      # lr = 0: no table and no state moved, nothing became inf or NaN
      for a, b in zip(f_before, fast.embedding.weights):
        assert torch.equal(a, b.detach())
      for a, b in zip(e_before, ref.embedding.weights):
        assert torch.equal(a, b.detach())
      for n, z in eng.opt_state.values():
        assert bool((n == INIT_ACC_F32).all()) and bool((z == 0).all())
    if i == 1:
      # one step's update (bf16 math on both sides, different summation orders)
      for w_ref, w_fast, r0, f0 in zip(ref.embedding.weights, fast.embedding.weights,
                                       e_before, f_before):
        d_ref, d_fast = w_ref.detach() - r0, w_fast.detach() - f0
        assert d_ref.abs().sum() > 0
        assert rel(d_fast, d_ref) < 0.08, rel(d_fast, d_ref)
  torch.cuda.synchronize()
  assert eng.step_count() == 8
  for v in eng.opt_state.values():
    assert all(torch.isfinite(s).all() for s in v)
  np.testing.assert_allclose(l_fast, l_ref, rtol=2e-2, atol=2e-3)
