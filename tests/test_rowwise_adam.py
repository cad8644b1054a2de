"""Row-wise Adam (``set_optimizer("rowwise_adam")``): m element-wise, v one fp32 word per row.

Every step is checked against the float64 model of ``optim_reference.rowwise_adam_update`` with
bounds from operation counts, on the engine's own weights and state (the driver of
``test_fused_optimizers.py``, with row-wise Adam's state layout).  A column-sliced table keeps one
v word per row in every slice, the mean over that slice's columns: the model is applied per slice.

CPU (no GPU): the bound self-check (the exact result passes, modelled defects fail), the plan
interpreter at world 1-8 (segment / balanced routes, crossing segments, rows wider than 128, mean
pooling, ragged and shared inputs, row and column slices, weight decay, skewed ids),
``SparseRowOptimizer`` against the model and against the interpreter, optimizer-state round trips
in memory, through files and across world sizes, dry updates, argument checks and the DLRM
example's convergence.

GPU (one H100): every kernel route with fp32 tables, 16-bit tables and bf16 m against the
stochastic-rounding rule, the fused against the torch back end, cached against uncached training
(bit for bit) and ``DLRMTrainStep`` (CUDA graph) against ``HybridTrainer``.
"""
import numpy as np
import pytest
import torch

import distributed_embeddings_b200 as de
from distributed_embeddings_b200.parallel import dry_run
from distributed_embeddings_b200.parallel.hybrid import SparseRowOptimizer
import test_fused_optimizers as tfo  # pylint: disable=wrong-import-order
import optim_reference  # pylint: disable=wrong-import-order
from optim_reference import (TINY, U, _e_sum, _ulp32, f32,  # pylint: disable=wrong-import-order
                             worst_table_ratio)
from test_dry_run import assemble  # pylint: disable=wrong-import-order
from test_examples_smoke import run as run_example  # pylint: disable=wrong-import-order

KIND = "rowwise_adam"
WD = tfo.WD


# ------------------------------------------------------------------ float64 model
# Defects the model can add: wrong bias-correction step, eps under the root, decay dropped, and v
# fed the mean square of the undecayed gradient.
ROWWISE_ADAM_DEFECTS = ("bias_t_minus_1", "eps_in_sqrt", "decay_dropped", "v_without_decay")


def rowwise_adam_update(w, gp, e_gp, m, v, lr, t, cfg, defect=None, v_grad=None):
  """Row-wise Adam on the touched rows from their decayed gradient ``gp`` ([R, W] float64, known
  to within ``e_gp`` of what the kernel computes): m ([R, W]) element-wise, v ([R]) one word per
  row, ``v = beta2 v + (1 - beta2) mean_j(gp_j^2)``, ``p -= lr (m / (1 - beta1^t)) /
  (sqrt(v / (1 - beta2^t)) + eps)``.  The mean square is bounded as ``optim_reference`` bounds
  row-wise Adagrad's (a sum of W squares in any order, then / W), the moments and bias
  corrections as it bounds Adam's, then the shared denominator.  ``v_grad``: the gradient v
  averages, if not ``gp`` (a defect).  Returns (out, bound) for 'p', 's0' (m), 's1' (v)."""
  lr, eps = f32(lr), f32(cfg["eps"])
  b1, b2 = f32(cfg["beta1"]), f32(cfg["beta2"])
  c1, c2 = 1.0 - b1, 1.0 - b2  # exact in fp32 (Sterbenz)
  width = gp.shape[1]
  vg = gp if v_grad is None else v_grad
  sq = (vg * vg).sum(1)
  mean = sq / width
  e_mean = ((2 * gp.abs() * e_gp + e_gp * e_gp).sum(1) + (width + 3) * U * sq) / width
  v_new = b2 * v + c2 * mean
  e_v = c2 * e_mean + 3.5 * U * ((b2 * v).abs() + c2 * mean) + TINY
  m_new = b1 * m + c1 * gp
  e_m = c1 * e_gp + 2.5 * U * ((b1 * m).abs() + (c1 * gp).abs()) + TINY
  tt = t - 1 if defect == "bias_t_minus_1" else t
  pw1, pw2 = b1**tt, b2**tt
  bias1, bias2 = 1.0 - pw1, 1.0 - pw2
  rb1 = 4 * float(_ulp32(torch.tensor(pw1))) / bias1 + U
  rb2 = 4 * float(_ulp32(torch.tensor(pw2))) / bias2 + U
  mh = m_new / bias1
  e_mh = e_m / bias1 + mh.abs() * (rb1 + U)
  vh = v_new / bias2
  root = vh.clamp_min(0).sqrt()
  den = (vh + eps).sqrt() if defect == "eps_in_sqrt" else root + eps
  rv = torch.where(v_new > 0, e_v / v_new.clamp_min(1e-300), torch.zeros_like(v_new)) + rb2 + U
  e_den = root * (rv / 2 + U) + U * den
  den, e_den = den.unsqueeze(1), e_den.unsqueeze(1)
  d = lr * mh / den
  e_d = (lr * e_mh + U * lr * mh.abs()) / den + d.abs() * (
      e_den / (den - e_den).clamp_min(TINY) + U)
  out = {"p": w - d, "s0": m_new, "s1": v_new}
  bound = {"p": 1.05 * e_d + U * (w - d).abs() + TINY, "s0": 1.05 * e_m, "s1": 1.05 * e_v}
  return out, bound


def table_step(kind, weights, state, occ_rows, occ_vals, scale, lr, t, cfg, defect=None):
  """One lazy row-wise Adam step on a whole table, with bounds: the contract of
  ``optim_reference.table_step`` (the gradient of each touched row summed from its occurrences
  within (n + 2) u |s| sum |c_k g_k|, then one fma of the decay), with ``state`` = [m [rows, W],
  v [rows]].  Untouched rows get a bound of zero.  Returns (out, bound, touched)."""
  assert kind == KIND
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
  g = s * gsum[idx]
  gp = g if defect == "decay_dropped" else g + wd * w[idx]
  e_gp = _e_sum(s, n_occ[idx], gabs[idx]) + U * gp.abs() + TINY
  o, b = rowwise_adam_update(w[idx], gp, e_gp, st[0][idx], st[1][idx], lr, t, cfg,
                             defect=defect, v_grad=g if defect == "v_without_decay" else None)
  out = {"p": w.clone(), "s0": st[0].clone(), "s1": st[1].clone()}
  bound = {k: torch.zeros_like(x) for k, x in out.items()}
  for k in o:
    out[k][idx] = o[k]
    bound[k][idx] = b[k]
  return out, bound, touched


def _cfg(wd=0.0, eps=1e-8):
  return {"eps": eps, "beta1": 0.9, "beta2": 0.999, "weight_decay": wd}


def _initial_state(rows, width):
  return [np.zeros((rows, width), np.float32), np.zeros(rows, np.float32)]


class _Spec(tfo.Spec):
  """Row-wise Adam for the driver of ``test_fused_optimizers.py``: m element-wise, v per row (per
  column slice: the mean over the slice's columns)."""

  def initial(self, rows, width, sdt):
    return _initial_state(rows, width)

  def model(self, case, before, state, occ, step, scale):
    return table_step(KIND, before, state, occ[0], occ[1], scale, case["lrs"][step], step + 1,
                      _cfg(case.get("wd", 0.0)))


SPEC = _Spec(KIND)
_slices = tfo._slices


def _run(case, world=1, dev=None, plan=None, route=None, **kw):
  """``case`` for ``len(case['lrs'])`` steps through the driver of test_fused_optimizers.py,
  every step and every slot checked; ``plan``: extra DistributedEmbedding arguments (slicing)."""
  return tfo._run(case, KIND, world, dev, plan, route, spec=SPEC, **kw)


_case, _with = tfo._case, tfo._with

# ------------------------------------------------------------------ CPU: the float64 model
def _selfcheck_inputs(seed=40):
  gen = torch.Generator().manual_seed(seed)
  rows, width = 64, 16
  w = torch.randn(rows, width, generator=gen).numpy()
  m = (torch.randn(rows, width, generator=gen) * 0.1).numpy()
  v = (m * m * 3).mean(1).astype(np.float32)  # plausible moments of earlier steps
  occ_rows = np.concatenate([np.full(c, r + 1) for r, c in enumerate([1, 2, 5, 33])] +
                            [np.arange(10, 40)])
  n = np.where(np.arange(len(occ_rows)) % 2 == 0, 1, 3)  # pooling of 1 or 3 ids (mean)
  c = np.asarray([f32(1.0 / k) for k in n])
  g = tfo._grad_values(gen, (len(occ_rows), width)).double().numpy()
  return w, [m, v], occ_rows, c[:, None] * g


@pytest.mark.parametrize("defect", ROWWISE_ADAM_DEFECTS)
def test_bounds_catch_defects(defect):
  """The exactly rounded result passes every bound; each modelled defect fails it."""
  w, state, occ_rows, vals = _selfcheck_inputs()
  cfg = _cfg(WD, eps=1e-3 if defect == "eps_in_sqrt" else 1e-8)
  out, bound, touched = table_step(KIND, w, state, occ_rows, vals, 1.0, 0.05, 2, cfg)
  assert out["s1"].shape == (64,) and touched[1] and not touched[0]
  assert worst_table_ratio(out, bound, tfo._rounded_table(out)) <= 1.0
  bad, _, _ = table_step(KIND, w, state, occ_rows, vals, 1.0, 0.05, 2, cfg, defect=defect)
  assert worst_table_ratio(out, bound, tfo._rounded_table(bad)) > 1.0, defect


def test_model_is_adam_with_a_row_mean_of_v():
  """On a one-column table row-wise Adam is Adam."""
  w, state, occ_rows, vals = _selfcheck_inputs()
  w1, vals1 = w[:, :1], vals[:, :1]
  m1 = state[0][:, :1]
  v1 = (m1 * m1 * 2).astype(np.float32)
  a, _, _ = table_step(KIND, w1, [m1, v1[:, 0]], occ_rows, vals1, 1.0, 0.05, 3, _cfg(WD))
  b, _, _ = optim_reference.table_step("adam", w1, [m1, v1], occ_rows, vals1, 1.0, 0.05, 3,
                                       _cfg(WD))
  torch.testing.assert_close(a["p"], b["p"], rtol=1e-12, atol=0)
  torch.testing.assert_close(a["s1"], b["s1"][:, 0], rtol=1e-12, atol=0)


# ------------------------------------------------------------------ CPU: the plan interpreter
TABLES = [(200, 16, "sum"), (150, 8, "mean"), (90, 12, "sum"), (80, 8, "sum")]
PLANS = {"whole": None, "column_slices": {"column_slice_threshold": 1000},
         "row_slices": {"row_slice_threshold": 1500}}


@pytest.mark.parametrize("world", [1, 2, 3, 4, 5, 6, 7, 8])
@pytest.mark.parametrize("plan", sorted(PLANS))
@pytest.mark.parametrize("wd", [0.0, WD])
def test_interpreter_against_float64(world, plan, wd):
  case = _case(TABLES, [0, 1, 2, 3, 0], [1, 2, 1, 3, 2], 840, wd=wd, seed=20 + world)
  des = _run(case, world=world, plan=PLANS[plan], route="any" if PLANS[plan] else None)
  st = des[0].strategy
  if plan == "column_slices" and world > 1:
    assert any(len(_slices(des[0], t, w)) > 1 for t, (_, w, _) in enumerate(TABLES))
  if plan == "row_slices" and world > 1:
    assert st.table_groups[2]


@pytest.mark.parametrize("name", ["mixed", "wide", "odd", "skewed"])
def test_interpreter_routes_against_float64(name):
  """World 1: the balanced route with crossing segments (1 ... 300 occurrences, a zero-gradient
  row), rows wider than 128, widths that are not a multiple of 4, power-law ids; two steps."""
  case = {"mixed": _with(tfo.MIXED, wd=WD, lrs=[0.05, 0.02]),
          "wide": _with(tfo.WIDE, wd=WD),
          "odd": _with(tfo.ODD, wd=0.0),
          "skewed": _case([(500, 32, "mean")] * 2, [0, 1, 0], [1, 7, 3], 512, power_law=True,
                          lrs=[0.1], wd=WD, seed=11)}[name]
  _run(case, world=1)


@pytest.mark.parametrize("table_dtype,state_dtype", [(torch.float32, torch.bfloat16),
                                                     (torch.bfloat16, torch.float32),
                                                     (torch.float16, torch.bfloat16)])
def test_interpreter_16_bit_against_the_rounding_rule(table_dtype, state_dtype):
  case = _case([(600, 32, "sum")], [0, 0], [1, 2], 512, edges=True, wd=WD,
               table_dtype=table_dtype, state_dtype=state_dtype, lrs=[0.05, 0.05], seed=5)
  _run(case, world=1)


def _sparse_steps(kind_opt, p, steps=2, seed=31, width=12):
  gen = torch.Generator().manual_seed(seed)
  rows = p.shape[0]
  out = []
  for step in range(steps):
    idx = torch.randint(0, 30 + 20 * step, (80,), generator=gen)
    idx[:5] = 7
    vals = tfo._grad_values(gen, (80, width)).to(p.dtype).float()
    vals[:5] = 0.0
    out.append((idx, vals))
    if kind_opt is not None:
      p.grad = torch.sparse_coo_tensor(idx[None], vals.to(p.dtype), (rows, width))
      kind_opt.step()
  return out


def test_sparse_row_optimizer_against_float64():
  """The torch back end's row-sparse optimizer: two steps with decay, duplicate ids and a row
  touched only by zero gradients."""
  torch.manual_seed(30)
  rows, width = 60, 12
  p = torch.nn.Parameter(torch.randn(rows, width))
  b1, b2 = 0.875, 1 - 2.0**-10  # exact in fp32: the torch optimizer takes them in float64
  opt = SparseRowOptimizer([p], KIND, lr=0.05, weight_decay=WD, beta1=b1, beta2=b2)
  assert opt.eps == 1e-8
  assert opt.state[0][0].shape == (rows, width) and opt.state[0][1].shape == (rows,)
  state = _initial_state(rows, width)
  for step, (idx, vals) in enumerate(_sparse_steps(None, p)):
    p.grad = torch.sparse_coo_tensor(idx[None], vals, (rows, width))
    before = p.detach().numpy().copy()
    cfg = {"eps": 1e-8, "beta1": b1, "beta2": b2, "weight_decay": WD}
    out, bound, touched = table_step(KIND, before, state, idx.numpy(), vals.double().numpy(),
                                     1.0, 0.05, step + 1, cfg)
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
  opt = SparseRowOptimizer([p], KIND, lr=0.05, weight_decay=WD, state_dtype=state_dtype)
  steps = _sparse_steps(opt, p)
  sim, des = dry_run.build_engines([{"input_dim": rows, "output_dim": width, "combiner": "sum"}],
                                   1, dp_input=True, table_dtype=table_dtype)
  d = des[0]
  d.set_weights([w0])
  kw = {} if state_dtype == torch.float32 else {"state_dtype": state_dtype}
  d.set_optimizer(KIND, lr=0.05, weight_decay=WD, **kw)
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
    np.testing.assert_allclose(st[0], opt.state[0][0].float().numpy(), rtol=1e-5, atol=1e-7)
    # SparseRowOptimizer takes 1 - beta2 in float64, the kernels and the interpreter in fp32
    np.testing.assert_allclose(st[1][:, 0], opt.state[0][1].numpy(), rtol=3e-5, atol=1e-9)
  else:
    # the same rounding rule and keys: only a last-bit difference of the fp32 value before the
    # rounding can move a result, by one bf16 ulp
    np.testing.assert_allclose(got, want, rtol=2**-7, atol=1e-6)
    assert (got == want).mean() > 0.95


# ------------------------------------------------------------------ CPU: optimizer state
SIZES = [(30, 8), (12, 16), (50, 8), (21, 16), (64, 8)]


def _plan_engines(world, weights, state_dtype=torch.float32, **kw):
  embs = [{"input_dim": r, "output_dim": w, "combiner": "sum"} for r, w in SIZES]
  sim, des = dry_run.build_engines(embs, world, strategy="memory_balanced", **kw)
  for d in des:
    d.set_weights(weights)
    d.set_optimizer(KIND, lr=0.3, weight_decay=0.1, state_dtype=state_dtype)
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
    out.backward(torch.from_numpy(np.concatenate([g[sl] for g in grads], 1)) * world / 2)
  dry_run.run_ranks(sim, fn)


def _gather(sim, des, fn):
  return dry_run.run_ranks(sim, lambda r: fn(des[r]))[0]


@pytest.mark.parametrize("state_dtype", [torch.float32, torch.bfloat16])
def test_optimizer_state_resharding(state_dtype, tmp_path):
  """Global state layout: slot 0 (m) ``[rows, width]``, slot 1 (v) ``[rows, 1]``.  One step on 4
  ranks, state and weights loaded into 2 ranks with a row-sliced table, a second step there ==
  two uninterrupted steps on the 2-rank plan; in memory and through files."""
  rng = np.random.default_rng(11)
  tables = [rng.standard_normal(s).astype(np.float32) for s in SIZES]
  batches = _batches()
  kw2 = {"row_slice_threshold": 500}
  sim_a, des_a = _plan_engines(2, tables, state_dtype, **kw2)
  _step(sim_a, des_a, batches[0])
  _step(sim_a, des_a, batches[1])
  straight = _gather(sim_a, des_a, lambda d: d.get_weights())
  straight_s = _gather(sim_a, des_a, lambda d: d.get_optimizer_state())

  sim_b, des_b = _plan_engines(4, tables, state_dtype)
  _step(sim_b, des_b, batches[0])
  saved_w = _gather(sim_b, des_b, lambda d: d.get_weights())
  saved_s = _gather(sim_b, des_b, lambda d: d.get_optimizer_state())
  assert saved_s["step"] == 1 and saved_s["kind"] == KIND
  for t, (rows, w) in enumerate(SIZES):
    assert [a.shape for a in saved_s["tables"][t]] == [(rows, w), (rows, 1)]
    assert (saved_s["tables"][t][1] >= 0).all() and (saved_s["tables"][t][1] > 0).any()

  sim_c, des_c = _plan_engines(2, saved_w, state_dtype, **kw2)

  def load(r):
    des_c[r]._engine.prepare(4, [2] * len(SIZES))
    des_c[r].set_optimizer_state(saved_s)
  dry_run.run_ranks(sim_c, load)
  _step(sim_c, des_c, batches[1])
  resumed = _gather(sim_c, des_c, lambda d: d.get_weights())
  resumed_s = _gather(sim_c, des_c, lambda d: d.get_optimizer_state())
  # bf16 m: the 4- and 2-rank runs round m with different row keys (stochastic rounding)
  tol = dict(rtol=2e-5, atol=2e-6) if state_dtype == torch.float32 else dict(rtol=2e-2, atol=2e-3)
  for a, b in zip(straight, resumed):
    np.testing.assert_allclose(b, a, **tol)
  for ta, tb in zip(straight_s["tables"], resumed_s["tables"]):
    np.testing.assert_allclose(tb[1], ta[1], rtol=1e-5, atol=1e-12)  # v: fp32 everywhere

  ckpt = str(tmp_path / "ckpt")

  def save(r):
    des_b[r].save_weights(ckpt, chunk=64)
    return des_b[r].save_optimizer_state(ckpt, chunk=64)
  metas = dry_run.run_ranks(sim_b, save)
  assert all(m == metas[0] and m.endswith("optimizer.json") for m in metas)
  for t in range(len(SIZES)):
    for k, arr in enumerate(saved_s["tables"][t]):
      np.testing.assert_array_equal(np.load(f"{ckpt}/opt_{t}_slot{k}.npy"), arr)
  sim_d, des_d = _plan_engines(2, tables, state_dtype, **kw2)

  def load_files(r):
    des_d[r]._engine.prepare(4, [2] * len(SIZES))
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


def test_column_slices_keep_their_own_row_word_and_export_the_weighted_mean():
  """A table cut into column slices: each slice's v word is the mean over its own columns; the
  exported word is the width-weighted mean of the slices' words (exact for the linear EMA), and
  an import gives every slice that global word."""
  rng = np.random.default_rng(5)
  tables = [rng.standard_normal(s).astype(np.float32) for s in SIZES]
  sim, des = _plan_engines(4, tables, column_slice_threshold=100)
  _step(sim, des, _batches(1)[0])
  st = des[0].strategy
  sliced = [(gt, t) for gt, t in enumerate(st.table_groups[1])
            if len({(s.col_start, s.col_end) for sh in st.shards for s in sh if s.table == gt}) > 1]
  assert sliced
  saved = _gather(sim, des, lambda d: d.get_optimizer_state())
  for gt, t in sliced:
    width = SIZES[t][1]
    mean = np.zeros(SIZES[t][0])
    for r, shards in enumerate(st.shards):
      for s in shards:
        if s.table == gt:
          local = des[r]._engine.opt_state[s.local_table][1][s.row_offset:s.row_offset + s.rows]
          mean += local.numpy() * (s.width / width)
    np.testing.assert_allclose(saved["tables"][t][1][:, 0], mean, rtol=1e-6, atol=1e-12)
  dry_run.run_ranks(sim, lambda r: des[r].set_optimizer_state(saved))
  for gt, t in sliced:
    for r, shards in enumerate(st.shards):
      for s in shards:
        if s.table == gt:
          local = des[r]._engine.opt_state[s.local_table][1][s.row_offset:s.row_offset + s.rows]
          np.testing.assert_array_equal(local.numpy(), saved["tables"][t][1][:, 0])


def test_state_of_another_kind_is_rejected():
  rng = np.random.default_rng(6)
  tables = [rng.standard_normal(s).astype(np.float32) for s in SIZES]
  sim, des = _plan_engines(1, tables)
  _step(sim, des, _batches(1, gb=4)[0])
  state = des[0].get_optimizer_state()
  des[0].set_optimizer("adam", lr=0.1)
  with pytest.raises(ValueError, match="does not match"):
    des[0].set_optimizer_state(state)
  des[0].set_optimizer(KIND, lr=0.1)
  des[0].set_optimizer_state(state)
  adam = dict(state, kind="rowwise_adagrad")
  with pytest.raises(ValueError, match="does not match"):
    des[0].set_optimizer_state(adam)


@pytest.mark.parametrize("weight_decay", [0.0, 0.5])
def test_dry_updates_leave_tables_and_optimizer_state_untouched(weight_decay):
  """Dry passes (graph warm-up) on live state after a real step: tables, m, v and the step count
  come out bit-identical; the next real step equals one taken without the dry passes."""
  rng = np.random.default_rng(4)
  tables = [rng.standard_normal(s).astype(np.float32) for s in SIZES]
  batches = _batches(3, seed=12)

  def make():
    sim, des = _plan_engines(2, tables, column_slice_threshold=100)
    for d in des:
      d.set_optimizer(KIND, lr=0.3, weight_decay=weight_decay)
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
  assert des_a[0]._engine.step_count() == des_b[0]._engine.step_count() == 2


def test_arguments():
  d = de.DistributedEmbedding([{"input_dim": 10, "output_dim": 8, "combiner": "sum"}],
                              device="cpu", backend="torch", world_size=1, rank=0)
  d.set_optimizer(KIND, lr=0.1)
  cfg = d._fused_optimizer
  assert (cfg["eps"], cfg["beta1"], cfg["beta2"], cfg["weight_decay"]) == (1e-8, 0.9, 0.999, 0.0)
  assert cfg["state_dtype"] == torch.float32
  d.set_optimizer(KIND, lr=0.1, state_dtype=torch.bfloat16, eps=1e-6, beta1=0.8, beta2=0.99,
                  weight_decay=0.1, step=3)
  with pytest.raises(ValueError, match="torch.float32 or torch.bfloat16"):
    d.set_optimizer(KIND, lr=0.1, state_dtype=torch.float16)
  with pytest.raises(ValueError, match="unknown fused optimizer argument"):
    d.set_optimizer(KIND, lr=0.1, momentum=0.9)
  with pytest.raises(ValueError, match="offload_cache_size"):
    de.DistributedEmbedding([{"input_dim": 1000, "output_dim": 8, "combiner": "sum"}],
                            device="cpu", world_size=1, rank=0, offload_cache_size=100,
                            gpu_embedding_size=10).set_optimizer(KIND, lr=0.1,
                                                                  state_dtype=torch.bfloat16)
  p = torch.nn.Parameter(torch.zeros(5, 4, dtype=torch.bfloat16))
  opt = SparseRowOptimizer([p], KIND, state_dtype=torch.bfloat16)
  assert opt.state[0][0].dtype == torch.bfloat16 and opt.state[0][1].dtype == torch.float32


def test_plan_report_counts_row_words():
  """tools/plan_report.py: row-wise Adam = one element slot (state dtype) + one fp32 row word."""
  import json  # pylint: disable=import-outside-toplevel
  rows, width = 100_000_000, 128
  base = ["tools/plan_report.py", "--tables", f"{rows}x{width}", "--world", "1", "--json",
          "--table-dtype", "bf16", "--hbm-gib", "1000"]

  def gib(*extra):
    rep = json.loads(run_example(base + list(extra)).strip().splitlines()[-1])
    return rep["ranks"][0]["hbm_gib"], rep
  plain, rep = gib()
  assert "optimizer_row_slots" not in rep
  assert gib("--optimizer-row-slots", "0")[0] == plain
  fp32_m, rep = gib("--optimizer-slots", "1", "--optimizer-row-slots", "1")
  assert rep["optimizer_row_slots"] == 1
  assert abs(fp32_m - plain - (rows * width * 4 + rows * 4) / 2**30) <= 0.01
  bf16_m, _ = gib("--optimizer-slots", "1", "--state-dtype", "bf16", "--optimizer-row-slots", "1")
  assert abs(bf16_m - plain - (rows * width * 2 + rows * 4) / 2**30) <= 0.01


def test_dlrm_example_learns_with_rowwise_adam(tmp_path):
  """The DLRM example's convergence run (generated learnable dataset, three epochs) with
  ``--embedding_optimizer rowwise_adam``: the evaluation AUC climbs well above 0.7."""
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
for _wd in (0.0, WD):
  GPU_CASES += [(f"balanced-wd{_wd}", _with(tfo.MIXED, wd=_wd, lrs=[0.05, 0.02])),
                (f"per_row_vec4-wd{_wd}", _with(tfo.WIDE, wd=_wd, lrs=[0.05, 0.02])),
                (f"per_row_vec1-wd{_wd}", _with(tfo.ODD, wd=_wd, lrs=[0.05, 0.02])),
                (f"small-wd{_wd}", _with(tfo.SMALL, wd=_wd))]
for _tdt in (torch.float32, torch.bfloat16, torch.float16):
  for _sdt in (torch.float32, torch.bfloat16):
    if _tdt == _sdt == torch.float32:
      continue
    GPU_CASES.append((f"half-{str(_tdt)[6:]}-table-{str(_sdt)[6:]}-m",
                      _case([(600, 32, "sum")], [0, 0], [1, 2], 512, edges=True, wd=WD,
                            table_dtype=_tdt, state_dtype=_sdt, lrs=[0.05, 0.05], seed=5)))
for _cdt in (torch.bfloat16, torch.float16):
  GPU_CASES.append((f"act-{str(_cdt)[6:]}", _with(tfo.MIXED, wd=WD, compute_dtype=_cdt)))
GPU_CASES.append(("four-steps", _case([(300, 32, "sum"), (100, 16, "mean")], [0, 1], [2, 3], 256,
                                      wd=WD, ids32=True,
                                      touch=[(0, 1 / 3), (1 / 6, 2 / 3), (1 / 2, 1), (0, 2 / 15)],
                                      lrs=[0.05, 0.05, 0.01, 0.01], seed=9)))


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
               lrs=[0.1], wd=WD, seed=11)
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
  fused = DistributedEmbedding(embs, device=dev, backend="fused", table_dtype=table_dtype,
                               compute_dtype=torch.float32, world_size=1, rank=0)
  fused.set_weights(w0)
  fused.set_optimizer(KIND, lr=0.01, weight_decay=0.01)
  ref = DistributedEmbedding(embs, device=dev, backend="torch", table_dtype=table_dtype,
                             compute_dtype=torch.float32)
  ref.set_weights(w0)
  opt = SparseRowOptimizer(ref.mp_parameters(), KIND, lr=0.01, weight_decay=0.01)
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
      # the same rounding rule and keys, but the fp32 values before the rounding differ in their
      # last bits (gradient summation order; 1 - beta2 in float64 in SparseRowOptimizer), which
      # moves a value by one bf16 ulp where the rounding decision flips
      bad = ~np.isclose(a, b, rtol=2**-6, atol=2e-3)
      assert bad.mean() < 2e-3, bad.mean()
  st = fused.get_optimizer_state()["tables"]
  for t in range(2):
    # SparseRowOptimizer takes 1 - beta2 in float64, the kernels in fp32; with bf16 tables v also
    # sees the weight-decay term of weights that differ by an ulp here and there
    np.testing.assert_allclose(st[t][1][:, 0], opt.state[t][1].cpu().numpy(),
                               rtol=3e-5 if table_dtype == torch.float32 else 1e-2, atol=1e-12)


@pytest.mark.gpu
@pytest.mark.parametrize("skewed", [False, True])
def test_gpu_cached_training_matches_uncached_bit_for_bit(skewed):
  """fp32 tables, fp32 m, a cache far smaller than the working set.  Width 132 takes the per-row
  update, which sums a row's gradient rows in input order whatever the keys are (the balanced
  update of narrower tables splits runs at borders that depend on the keys, which are slot ids
  with the cache): tables, m and v equal an uncached run bit for bit."""
  from distributed_embeddings_b200.parallel.dist_model_parallel import DistributedEmbedding
  from distributed_embeddings_b200.parallel.offload_cache import WAYS
  dev = torch.device("cuda", 0)
  small, big, width = 64, 6000, 132
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
    d.set_optimizer(KIND, lr=0.01, weight_decay=0.01)
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
    np.testing.assert_array_equal(a, b)
  assert np.abs(plain.get_weights()[1] - w0[1]).max() > 1e-3, "the offloaded table trained"
  sc, sp = cached.get_optimizer_state(), plain.get_optimizer_state()
  assert sc["step"] == sp["step"] == 6
  for ta, tb in zip(sc["tables"], sp["tables"]):
    for a, b in zip(ta, tb):
      np.testing.assert_array_equal(a, b)


@pytest.mark.gpu
def test_gpu_dlrm_train_step_matches_hybrid_trainer():
  """DLRMTrainStep (CUDA graph replay) with row-wise Adam tracks HybridTrainer on the same seeds:
  the first step's embedding update and the loss of each of 8 steps agree to bf16-compute
  accuracy.  The graph warm-up passes leave tables, m, v and the step count untouched."""
  from distributed_embeddings_b200.models.dlrm import DLRM
  from distributed_embeddings_b200.models.dlrm_fast import DLRMTrainStep
  from distributed_embeddings_b200.models.trainer import HybridTrainer
  dev = torch.device("cuda", 0)
  sizes = [300 + 11 * i for i in range(26)]

  def make():
    torch.manual_seed(0)
    return DLRM(sizes, device=dev, compute_dtype=torch.bfloat16, backend="fused")
  ref, fast = make(), make()
  fast.load_state_dict(ref.state_dict())
  fast.embedding.set_weights(ref.embedding.get_weights())
  e0 = [w.detach().clone() for w in ref.embedding.weights]
  g = torch.Generator().manual_seed(1)
  batches = [(torch.rand(512, 13, generator=g).to(dev),
              [torch.randint(0, s, (512,), generator=g, dtype=torch.int32).to(dev) for s in sizes],
              torch.randint(0, 2, (512, 1), generator=g).float().to(dev)) for _ in range(8)]
  lr = 0.01
  t_ref = HybridTrainer(ref, lr=lr, embedding_optimizer=KIND)
  t_fast = DLRMTrainStep(fast, lr=lr, embedding_optimizer=KIND, use_cuda_graph=True)
  eng = t_fast.engine
  l_ref, l_fast = [], []

  def rel(a, b):
    return float((a - b).norm() / (b.norm() + 1e-12))
  for i, (num, cat, lab) in enumerate(batches):
    l_ref.append(float(t_ref.step(num, cat, lab)))
    if i == 1:
      # the dry passes of a graph warm-up on live state (zero lr, dry updates)
      torch.cuda.synchronize()
      before = {m: [s.clone() for s in v] for m, v in eng.opt_state.items()}
      w_before = [w.detach().clone() for w in fast.embedding.weights]
      step = eng.step_count()
      t_fast.load_batch(num, torch.stack(cat), lab)
      t_fast.lr_t.zero_()
      eng.dry_updates(True)
      t_fast._step_impl()
      eng.dry_updates(False)
      t_fast.lr_t.fill_(lr)
      torch.cuda.synchronize()
      assert eng.step_count() == step == 1
      for m, v in before.items():
        for a, b in zip(v, eng.opt_state[m]):
          assert torch.equal(a, b)
      for a, b in zip(w_before, fast.embedding.weights):
        assert torch.equal(a, b.detach())
    l_fast.append(float(t_fast.step(num, torch.stack(cat), lab)))
    if i == 0:
      # one step's update (bf16 math on both sides, different summation orders)
      for w_ref, w_fast, w0_ in zip(ref.embedding.weights, fast.embedding.weights, e0):
        d_ref, d_fast = w_ref.detach() - w0_, w_fast.detach() - w0_
        assert d_ref.abs().sum() > 0
        assert rel(d_fast, d_ref) < 0.08, rel(d_fast, d_ref)
  torch.cuda.synchronize()
  assert eng.step_count() == 8
  np.testing.assert_allclose(l_fast, l_ref, rtol=2e-2, atol=2e-3)


@pytest.mark.gpu
@pytest.mark.parametrize("state_dtype", [torch.float32, torch.bfloat16])
def test_gpu_synthetic_train_step(state_dtype):
  """SyntheticTrainStep (CUDA graph) trains with row-wise Adam: m in the state dtype, v fp32."""
  from distributed_embeddings_b200.models.configs import expand, scaled, synthetic_models_v3
  from distributed_embeddings_b200.models.synthetic import SyntheticModel
  from distributed_embeddings_b200.models.synthetic_fast import SyntheticTrainStep
  dev = torch.device("cuda", 0)
  cfg = scaled(synthetic_models_v3["tiny"], 2e-4)
  tables, imap, hots = expand(cfg)[:3]
  torch.manual_seed(5)
  m = SyntheticModel(cfg, dp_input=True, device=dev, compute_dtype=torch.bfloat16,
                     backend="fused")
  t = SyntheticTrainStep(m, lr=0.01, embedding_optimizer=KIND, use_cuda_graph=True,
                         embedding_optimizer_kwargs={"state_dtype": state_dtype})
  g = torch.Generator().manual_seed(4)
  num = (torch.rand(128, cfg.num_numerical_features, generator=g) * 2).to(dev)
  cat = [torch.randint(0, tables[imap[i]][0], (128, h), generator=g).to(dev)
         for i, h in enumerate(hots)]
  lab = torch.randint(0, 2, (128, 1), generator=g).float().to(dev)
  losses = [float(t.step(num, cat, lab)) for _ in range(6)]
  torch.cuda.synchronize()
  assert all(np.isfinite(losses)) and losses[-1] < losses[0], losses
  assert t.engine.step_count() == 6
  for st in t.engine.opt_state.values():
    assert st[0].dtype == state_dtype and st[1].dtype == torch.float32 and st[1].dim() == 1
