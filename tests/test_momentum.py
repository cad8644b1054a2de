"""Momentum SGD (``set_optimizer("momentum")``, ``dense_optimizer="momentum"``) for the embedding
tables and the dense parameters, against float64.

The update follows ``torch.optim.SGD(momentum=mu, nesterov=..., dampening=0)`` with an
element-wise buffer b that starts at 0, in the kernels' fmaf order.  For a touched row with the
summed, scaled gradient g:

    l2 decay:         g = fmaf(wd, w, g)                   (before the buffer)
    decoupled decay:  w = w * fmaf(-lr, wd, 1)             (first)
    b = fmaf(mu, b, g)
    plain:     w = fmaf(-lr, b, w)
    nesterov:  w = fmaf(-lr, fmaf(mu, b, g), w)

The float64 model (:func:`momentum_table_step`) sums each touched row's gradient from its id
occurrences within the bound of ``optim_reference.table_step`` and follows each fma with one
rounding.  It plugs into the driver of ``test_fused_optimizers.py`` as a ``Spec``, so every step
checks the buffer of every shard, 16-bit tables and bf16 buffers at their rounding keys, and
bit-identical untouched rows.

CPU (no GPU):
- argument checks; other kinds still reject ``momentum=``;
- the plan interpreter at world 1-8 on whole, column-sliced and row-sliced tables, ragged inputs,
  16-bit tables, bf16 buffers, both decay modes and nesterov, three steps with an lr change;
- momentum 0 equals deterministic SGD bit for bit; dry updates move nothing;
- ``SparseRowOptimizer`` against float64, and against ``torch.optim.SGD`` when every row is
  touched in every step;
- ``HybridTrainer``'s dense kind against ``torch.optim.SGD`` (L2 decay) and float64 (decoupled);
- the buffer through checkpoints saved at world 2 and loaded at world 3;
- the GPU cases cover every route x table dtype x state dtype.

GPU (one H100):
- world 1 on every route, 16-bit tables and bf16 buffers; world 2-8 on one GPU through the
  kernel-authoritative mirror harness of ``test_kernel_conformance.py``, state read per shard;
- momentum 0 against deterministic SGD bit for bit (fp32, bf16 and fp16 tables);
- offloaded tables against float64, and cached training equal to uncached bit for bit;
- ``dense_momentum`` against float64;
- ``DLRMTrainStep`` (CUDA graph, scheduler) against ``HybridTrainer``, and ``SyntheticTrainStep``
  against ``HybridTrainer``'s plain-PyTorch dense step.
"""
import numpy as np
import pytest
import torch

import distributed_embeddings_b200 as de
from distributed_embeddings_b200.parallel import dry_run
from distributed_embeddings_b200.parallel.hybrid import SparseRowOptimizer
from optim_reference import TINY, U, _e_sum, f32  # pylint: disable=wrong-import-order
import test_fused_optimizers as tfo  # pylint: disable=wrong-import-order
import test_update_conformance as tur  # pylint: disable=wrong-import-order

KIND = "momentum"
WD = tfo.WD
MU = 0.9


# ------------------------------------------------------------------ float64 model
def momentum_table_step(weights, state, occ_rows, occ_vals, scale, lr, cfg):
  """float64 result of one lazy momentum step on one table with bounds, the contract of
  ``optim_reference.table_step``: returns (out, bound, touched) with 'p' and 's0' (the buffer)."""
  w = torch.as_tensor(np.asarray(weights, dtype=np.float64))
  rows = w.shape[0]
  occ = torch.as_tensor(np.asarray(occ_rows, dtype=np.int64))
  vals = torch.as_tensor(np.asarray(occ_vals, dtype=np.float64))
  s, wd, mu, lr = f32(scale), f32(cfg["weight_decay"]), f32(cfg["momentum"]), f32(lr)
  b0 = torch.as_tensor(np.asarray(state[0], dtype=np.float64))
  touched = np.zeros(rows, dtype=bool)
  touched[occ.numpy()] = True
  idx = torch.as_tensor(np.nonzero(touched)[0])
  gsum = torch.zeros_like(w).index_add_(0, occ, vals)
  gabs = torch.zeros_like(w).index_add_(0, occ, vals.abs())
  n_occ = torch.zeros(rows, dtype=torch.float64).index_add_(
      0, occ, torch.ones(len(occ), dtype=torch.float64))
  g = s * gsum[idx]
  e_g = _e_sum(s, n_occ[idx], gabs[idx]) + TINY
  wi, e_w = w[idx], 0.0
  if wd and cfg.get("weight_decay_mode", "l2") == "decoupled":
    wi = (1.0 - lr * wd) * wi  # the kernel rounds the factor and the product
    e_w = 2.05 * U * wi.abs()
  elif wd:
    g = g + wd * wi  # one fma
    e_g = e_g + U * g.abs() + TINY
  b = mu * b0[idx] + g
  e_b = e_g + U * b.abs() + TINY
  u, e_u = b, e_b
  if cfg["nesterov"]:
    u = mu * b + g
    e_u = mu * e_b + e_g + U * u.abs() + TINY
  p = wi - lr * u
  e_p = lr * e_u + e_w + U * p.abs() + TINY
  out, bound = {"p": w.clone(), "s0": b0.clone()}, {"p": torch.zeros_like(w),
                                                   "s0": torch.zeros_like(b0)}
  out["p"][idx], bound["p"][idx] = p, 1.05 * e_p
  out["s0"][idx], bound["s0"][idx] = b, 1.05 * e_b
  return out, bound, touched


class MomentumSpec(tfo.Spec):
  """The driver's ``Spec`` of momentum SGD: hyperparameters from the case's ``hp`` and ``mode``."""

  def __init__(self):
    super().__init__(KIND)

  def opt(self, case):
    return dict(case.get("hp", {}), weight_decay_mode=case.get("mode", "l2"))

  def initial(self, rows, width, sdt):  # pylint: disable=unused-argument
    return [np.zeros((rows, width), np.float32)]

  def model(self, case, before, state, occ, step, scale):
    hp = dict({"momentum": MU, "nesterov": False}, **case.get("hp", {}))
    cfg = dict(hp, weight_decay=case.get("wd", 0.0), weight_decay_mode=case.get("mode", "l2"))
    return momentum_table_step(before, state, occ[0], occ[1], scale, case["lrs"][step], cfg)


SPEC = MomentumSpec()
NESTEROV = {"momentum": 0.75, "nesterov": True}


# ------------------------------------------------------------------ CPU: arguments
def _layer():
  return de.DistributedEmbedding([{"input_dim": 10, "output_dim": 8, "combiner": "sum"}],
                                 device="cpu", backend="torch", world_size=1, rank=0)


def test_arguments():
  d = _layer()
  d.set_optimizer(KIND, lr=0.1)
  assert d._fused_optimizer["momentum"] == 0.9 and d._fused_optimizer["nesterov"] is False
  assert d._fused_optimizer["deterministic"]
  d.set_optimizer(KIND, lr=0.1, momentum=0.0, nesterov=True, weight_decay=0.1,
                  weight_decay_mode="decoupled", state_dtype=torch.bfloat16)
  for bad in (1.0, -0.1, 1.5, float("nan"), True, "0.9"):
    with pytest.raises(ValueError, match="momentum must be a number in"):
      d.set_optimizer(KIND, lr=0.1, momentum=bad)
  for bad in (1, 0, "yes", None):
    with pytest.raises(ValueError, match="nesterov must be a bool"):
      d.set_optimizer(KIND, lr=0.1, nesterov=bad)
  for kind in ("sgd", "adagrad", "adam", "rowwise_adam", "ftrl"):
    with pytest.raises(ValueError, match="unknown fused optimizer argument"):
      d.set_optimizer(kind, lr=0.1, momentum=0.9)
  p = torch.nn.Parameter(torch.zeros(10, 8))
  opt = SparseRowOptimizer([p], KIND, momentum=0.5, nesterov=True, state_dtype=torch.bfloat16,
                           weight_decay=0.1, weight_decay_mode="decoupled")
  assert opt.hyper["momentum"] == 0.5 and opt.hyper["nesterov"] is True
  with pytest.raises(ValueError, match="momentum must be a number in"):
    SparseRowOptimizer([p], KIND, momentum=1.0)
  with pytest.raises(ValueError, match="unknown fused optimizer argument"):
    SparseRowOptimizer([p], "adagrad", momentum=0.9)


def test_dense_arguments():
  from distributed_embeddings_b200.models.dense_optimizer import (dense_optimizer_config,
                                                                  slot_init)
  cfg = dense_optimizer_config(KIND)
  assert cfg["momentum"] == 0.9 and cfg["nesterov"] is False and slot_init(cfg) == [0.0]
  cfg = dense_optimizer_config(KIND, {"momentum": 0, "nesterov": True, "weight_decay": 0.1,
                                      "weight_decay_mode": "decoupled"})
  assert cfg["momentum"] == 0.0 and cfg["nesterov"] is True
  with pytest.raises(ValueError, match="momentum must be a number in"):
    dense_optimizer_config(KIND, {"momentum": 1.0})
  with pytest.raises(ValueError, match="nesterov must be a bool"):
    dense_optimizer_config(KIND, {"nesterov": 1})
  with pytest.raises(ValueError, match="takes no argument"):
    dense_optimizer_config("adagrad", {"momentum": 0.9})


# ------------------------------------------------------------------ CPU: plan interpreter
# (world, plan, table dtype, state dtype, decay mode or None, hyperparameters)
_INTERP = [
    (1, "balanced", torch.float32, torch.float32, None, {}),
    (2, "per-row vec1", torch.float32, torch.bfloat16, "decoupled", NESTEROV),
    (3, "rows", torch.bfloat16, torch.float32, "l2", NESTEROV),
    (4, "per-row vec4", torch.float32, torch.float32, "decoupled", {}),
    (5, "per-row vec1", torch.float16, torch.bfloat16, "l2", {}),
    (6, "rows", torch.float32, torch.float32, "decoupled", NESTEROV),
    (7, "balanced", torch.bfloat16, torch.bfloat16, "decoupled", {}),
    (8, "balanced", torch.float16, torch.float32, "l2", NESTEROV),
]


def _plan(plan):
  return tur.ROW_SLICES if plan == "rows" else tur.PLANS[plan]


def _with_decay(case, mode):
  return dict(case, wd=WD, mode=mode) if mode else dict(case, wd=0.0)


@pytest.mark.parametrize("world,plan,tdt,sdt,mode,hp", _INTERP,
                         ids=[f"w{c[0]}-{c[1].replace(' ', '_')}" for c in _INTERP])
def test_interpreter_against_float64(world, plan, tdt, sdt, mode, hp):
  """Three steps (the last at a lower lr), every buffer of every shard at the model's bounds."""
  case, kw = _plan(plan)
  case = dict(_with_decay(case, mode), hp=hp, table_dtype=tdt, state_dtype=sdt,
              batch=24 * world)
  tfo._run(case, KIND, world, plan=kw, route="any", spec=SPEC)


def _dyadic_run(kind, tdt, **opt):
  """Two steps at world 2 on a dyadic grid (power-of-two lr, weights, gradients and decay), where
  every fp32 operation of SGD and momentum 0 is exact; returns (weights, buffers)."""
  embs = [{"input_dim": 40, "output_dim": 8, "combiner": "sum"},
          {"input_dim": 30, "output_dim": 12, "combiner": "mean"}]
  sim, des = dry_run.build_engines(embs, 2, dp_input=True, column_slice_threshold=200,
                                   table_dtype=tdt)
  rng = np.random.default_rng(5)
  tables = [rng.integers(-32, 32, (r, w)).astype(np.float32) / 16 for r, w in ((40, 8), (30, 12))]
  for d in des:
    d.set_weights(tables)
    d.set_optimizer(kind, lr=0.25, weight_decay=0.5, **opt)
  for step in range(2):
    ids = [torch.from_numpy(rng.integers(0, r, (16, 2))) for r in (40, 30)]
    grad = torch.from_numpy(rng.integers(-8, 8, (16, 20)).astype(np.float32) / 8)

    def fn(r, ids=ids, grad=grad):
      out = des[r]([i[r * 8:(r + 1) * 8] for i in ids], concat=True)
      out.backward(grad[r * 8:(r + 1) * 8])
    dry_run.run_ranks(sim, fn)
  bufs = dry_run.run_ranks(sim, lambda r: des[r].get_optimizer_state())[0]
  return tfo._weights(des, 2), bufs


@pytest.mark.parametrize("tdt", [torch.float32, torch.bfloat16, torch.float16],
                         ids=lambda x: str(x)[6:])
def test_interpreter_momentum_zero_is_sgd_bit_for_bit(tdt):
  a, state = _dyadic_run(KIND, tdt, momentum=0.0, nesterov=True)
  b, _ = _dyadic_run("sgd", tdt, deterministic=True)
  for x, y in zip(a, b):
    assert np.array_equal(np.asarray(x, np.float32).view(np.uint32),
                          np.asarray(y, np.float32).view(np.uint32))
  assert any((np.asarray(t[0]) != 0).any() for t in state["tables"])


def test_interpreter_dry_updates_move_nothing():
  """A zero gradient still moves a row by -lr mu b: dry (warm-up) updates must not run momentum."""
  case, kw = tur.PLANS["balanced"]
  case = dict(case, wd=WD, batch=48, lrs=[0.05])
  made = []

  def world_cls(n):
    made.append(dry_run.DryWorld(n))
    return made[-1]
  des = tfo._run(case, KIND, 2, plan=kw, route="any", world_cls=world_cls, spec=SPEC)
  w0 = tfo._weights(des, 2)
  s0 = [{m: [x.clone() for x in st] for m, st in d._engine.opt_state.items()} for d in des]
  assert any((x != 0).any() for s in s0 for st in s.values() for x in st)
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


# ------------------------------------------------------------------ CPU: SparseRowOptimizer
_TABLE_STATE = [(torch.float32, torch.float32), (torch.bfloat16, torch.float32),
                (torch.float16, torch.float32), (torch.float32, torch.bfloat16),
                (torch.bfloat16, torch.bfloat16)]


@pytest.mark.parametrize("mode,hp", [("l2", {}), ("decoupled", NESTEROV)], ids=["l2", "nesterov"])
@pytest.mark.parametrize("tdt,sdt", _TABLE_STATE, ids=lambda x: str(x)[6:])
def test_sparse_row_optimizer_against_float64(tdt, sdt, mode, hp):
  """Three steps on different touched sets (one at a lower lr): touched rows and the buffer within
  3x the model's bounds, 16-bit values at their rounding keys, untouched rows bit-identical."""
  rows, width = 60, 12
  gen = torch.Generator().manual_seed(50)
  p = torch.nn.Parameter(torch.randn(rows, width, generator=gen).to(tdt))
  case = {"wd": WD, "mode": mode, "hp": hp, "lrs": [0.05, 0.05, 0.02], "table_dtype": tdt,
          "state_dtype": sdt}
  opt = SparseRowOptimizer([p], KIND, lr=0.05, weight_decay=WD, weight_decay_mode=mode,
                           state_dtype=sdt, **hp)
  state = SPEC.initial(rows, width, sdt)
  for step, lr in enumerate(case["lrs"]):
    opt.set_lr(lr)
    idx = torch.randperm(rows, generator=gen)[:rows // 2 - 7 * step]
    if tdt == torch.float32:  # duplicate ids (a 16-bit sparse gradient coalesces in 16 bits)
      idx = torch.cat([idx, idx[:5]])
    vals = tfo._grad_values(gen, (len(idx), width)).to(tdt)
    before = p.detach().float().numpy().copy()
    p.grad = torch.sparse_coo_tensor(idx[None], vals, (rows, width))
    opt.step()
    out, bound, touched = SPEC.model(case, before, state, (idx.numpy(), vals.double().numpy()),
                                     step, 1.0)
    slots = [s.float().numpy() for s in opt.state[0]]
    sh = {"rank": 0, "table": 0, "rows": np.arange(rows), "cols": (0, width),
          "keys": np.arange(rows), "slots": slots}
    tfo._check_shard(case, SPEC, 0, step, sh, out, bound, touched, p.detach().float().numpy(),
                     3.0)
    state = [s.copy() for s in slots]


@pytest.mark.parametrize("nesterov", [False, True])
def test_sparse_row_optimizer_matches_torch_sgd_when_every_row_is_touched(nesterov):
  """Every row touched in every step: the lazy update is the dense ``torch.optim.SGD``."""
  gen = torch.Generator().manual_seed(7)
  w0 = torch.randn(40, 16, generator=gen)
  p, q = torch.nn.Parameter(w0.clone()), torch.nn.Parameter(w0.clone())
  opt = SparseRowOptimizer([p], KIND, lr=0.05, momentum=MU, nesterov=nesterov, weight_decay=0.1)
  ref = torch.optim.SGD([q], lr=0.05, momentum=MU, nesterov=nesterov, weight_decay=0.1)
  for step, lr in enumerate([0.05, 0.05, 0.01, 0.01]):
    opt.set_lr(lr)
    for group in ref.param_groups:
      group["lr"] = lr
    g = torch.randn(40, 16, generator=gen)
    idx = torch.cat([torch.arange(40), torch.arange(0, 40, 3)])
    vals = torch.cat([g, torch.zeros(len(idx) - 40, 16)])
    p.grad = torch.sparse_coo_tensor(idx[None], vals, (40, 16))
    q.grad = g.clone()
    opt.step()
    ref.step()
    torch.testing.assert_close(p.detach(), q.detach(), rtol=1e-6, atol=1e-6,
                               msg=lambda m, s=step: f"step {s}: {m}")
    torch.testing.assert_close(opt.state[0][0], ref.state[q]["momentum_buffer"], rtol=1e-6,
                               atol=1e-6)


# ------------------------------------------------------------------ CPU: HybridTrainer dense
@pytest.mark.parametrize("mode", ["l2", "decoupled"])
@pytest.mark.parametrize("nesterov", [False, True])
def test_hybrid_dense_momentum(mode, nesterov):
  """``HybridTrainer(dense_optimizer="momentum")`` against ``torch.optim.SGD(momentum, nesterov,
  weight_decay)`` with L2 decay, and against a float64 model of the decoupled step (the weights
  scaled by 1 - lr wd first) otherwise; under a scheduler that changes the lr every step."""
  from distributed_embeddings_b200.models.trainer import HybridTrainer
  from distributed_embeddings_b200.utils.lr_schedule import LearningRateScheduler
  from test_dense_optimizers import _batch, _small_dlrm  # pylint: disable=import-outside-toplevel
  model, ref = _small_dlrm(0), _small_dlrm(0)
  lr, wd = 0.05, 0.1
  tr = HybridTrainer(model, lr=lr, embedding_optimizer="sgd", dense_optimizer=KIND,
                     scheduler=LearningRateScheduler(lr, 2, 3, 4),
                     dense_optimizer_kwargs={"momentum": MU, "nesterov": nesterov,
                                             "weight_decay": wd, "weight_decay_mode": mode})
  sched = LearningRateScheduler(lr, 2, 3, 4)
  dense = [p for p in ref.parameters() if not getattr(p, "de_local", False)]
  tables = [p for p in ref.parameters() if getattr(p, "de_local", False)]
  opt = torch.optim.SGD(dense, lr=lr, momentum=MU, nesterov=nesterov, weight_decay=wd)
  p64 = [p.detach().double() for p in dense]
  b64 = [torch.zeros_like(p) for p in p64]
  topt = torch.optim.SGD(tables, lr=lr)
  for i in range(5):
    step_lr = sched.step()
    for group in opt.param_groups + topt.param_groups:
      group["lr"] = step_lr
    num, cat, lab = _batch(model.table_sizes, 32, 100 + i)
    tr.step(num, cat, lab)
    ref.zero_grad()
    torch.nn.functional.binary_cross_entropy_with_logits(ref(num, cat).float(), lab).backward()
    if mode == "l2":
      opt.step()
    else:
      with torch.no_grad():
        for p, x, b in zip(dense, p64, b64):
          g = p.grad.double()
          x.mul_(1 - f32(step_lr) * f32(wd))
          b.mul_(f32(MU)).add_(g)
          x.sub_(f32(step_lr) * (f32(MU) * b + g if nesterov else b))
          p.copy_(x.float())
    topt.step()
  named = [(n, p) for n, p in model.named_parameters() if not getattr(p, "de_local", False)]
  for (n, a), b in zip(named, dense):
    torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-4 * lr, msg=lambda m, n=n: f"{n}: {m}")
  state = tr.dense_optimizer_state()
  assert state["kind"] == KIND and state["step"] == 0
  assert all(len(s) == 1 and s[0].shape == p.shape for (_, p), s in
             zip(named, [state["slots"][n] for n, _ in named]))


# ------------------------------------------------------------------ CPU: checkpoints
SIZES = [(30, 8), (12, 16), (50, 8), (21, 16), (64, 8)]


def _plan_engines(world, weights, state_dtype=torch.float32, **kw):
  embs = [{"input_dim": r, "output_dim": w, "combiner": "sum"} for r, w in SIZES]
  sim, des = dry_run.build_engines(embs, world, strategy="memory_balanced", **kw)
  for d in des:
    d.set_weights(weights)
    d.set_optimizer(KIND, lr=0.3, weight_decay=0.1, state_dtype=state_dtype, **NESTEROV)
  return sim, des


def _step(sim, des, batch):
  ids, grads = batch
  world = len(des)
  lb = ids[0].shape[0] // world

  def fn(r):
    sl = slice(r * lb, (r + 1) * lb)
    out = des[r]([torch.from_numpy(i[sl]) for i in ids], concat=True)
    out.backward(torch.from_numpy(np.concatenate([g[sl] for g in grads], 1)) * world / 6)
  dry_run.run_ranks(sim, fn)


def _gather(sim, des, fn):
  return dry_run.run_ranks(sim, lambda r: fn(des[r]))[0]


@pytest.mark.parametrize("state_dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
def test_buffer_survives_checkpoints_from_world_2_to_3(state_dtype, tmp_path):
  """The buffer is one element-wise slot ``[rows, width]`` per table in the global layout: saved
  at world 2 (column-sliced tables), loaded at world 3 (a row-sliced table) in memory and through
  files, it comes back bit for bit, and the next step there matches an uninterrupted 3-rank run."""
  rng = np.random.default_rng(11)
  tables = [rng.standard_normal(s).astype(np.float32) for s in SIZES]
  batches = [([rng.integers(0, r, size=(6, 2)) for r, _ in SIZES],
              [rng.standard_normal((6, w)).astype(np.float32) * 0.1 for _, w in SIZES])
             for _ in range(2)]
  kw3 = {"row_slice_threshold": 500}
  sim_a, des_a = _plan_engines(3, tables, state_dtype, **kw3)
  for b in batches:
    _step(sim_a, des_a, b)
  straight = _gather(sim_a, des_a, lambda d: d.get_weights())

  sim_b, des_b = _plan_engines(2, tables, state_dtype, column_slice_threshold=100)
  _step(sim_b, des_b, batches[0])
  saved_w = _gather(sim_b, des_b, lambda d: d.get_weights())
  saved_s = _gather(sim_b, des_b, lambda d: d.get_optimizer_state())
  assert saved_s["kind"] == KIND
  for t, (rows, w) in enumerate(SIZES):
    (b,) = saved_s["tables"][t]
    assert b.shape == (rows, w) and (b != 0).any()
  ckpt = str(tmp_path / "ckpt")

  def save(r):
    des_b[r].save_weights(ckpt, chunk=64)
    return des_b[r].save_optimizer_state(ckpt, chunk=64)
  dry_run.run_ranks(sim_b, save)

  for from_files in (False, True):
    sim_c, des_c = _plan_engines(3, saved_w, state_dtype, **kw3)

    def load(r, des_c=des_c, from_files=from_files):
      des_c[r]._engine.prepare(6, [2] * len(SIZES))
      if from_files:
        des_c[r].load_weights(ckpt)
        des_c[r].load_optimizer_state(ckpt)
      else:
        des_c[r].set_optimizer_state(saved_s)
    dry_run.run_ranks(sim_c, load)
    loaded = _gather(sim_c, des_c, lambda d: d.get_optimizer_state())
    for ta, tb in zip(saved_s["tables"], loaded["tables"]):
      for a, b in zip(ta, tb):
        np.testing.assert_array_equal(b, a)
    _step(sim_c, des_c, batches[1])
    # bf16 buffers: the 2- and 3-rank runs round b with different row keys
    tol = dict(rtol=2e-5, atol=2e-6) if state_dtype == torch.float32 else \
        dict(rtol=2e-2, atol=2e-3)
    for a, b in zip(straight, _gather(sim_c, des_c, lambda d: d.get_weights())):
      np.testing.assert_allclose(b, a, **tol)


# ------------------------------------------------------------------ GPU cases
def _cuda():
  return torch.device("cuda", 0)


ROUTE_TABLES = {"balanced": (600, 32), "per-row vec4": (300, 192), "per-row vec1": (400, 22)}
_DTS = [(t, s) for t in (torch.float32, torch.bfloat16, torch.float16)
        for s in (torch.float32, torch.bfloat16)]
# world 1 on the engine: one table (the driver keys 16-bit rounding from its key base 0), every
# route x table dtype x state dtype, decay mode and nesterov alternating
WORLD1 = []
for _i, _route in enumerate(ROUTE_TABLES):
  for _j, (_t, _s) in enumerate(_DTS):
    WORLD1.append((_route, _t, _s, ("l2", "decoupled")[(_i + _j) % 2],
                   NESTEROV if (_i + _j) % 3 == 0 else {}))
# world 2-8 on one GPU through the mirror harness: every route and row slices
SHARDED = [
    ("balanced", 2, torch.float32, torch.float32, "l2", {}),
    ("per-row vec4", 3, torch.float32, torch.float32, "decoupled", NESTEROV),
    ("per-row vec1", 4, torch.float16, torch.float32, "l2", NESTEROV),
    ("rows", 8, torch.float32, torch.float32, "decoupled", {}),
    ("rows", 4, torch.bfloat16, torch.bfloat16, "l2", {}),
    ("balanced", 8, torch.float32, torch.bfloat16, "decoupled", NESTEROV),
    ("per-row vec1", 2, torch.bfloat16, torch.bfloat16, "decoupled", {}),
]


def test_gpu_cases_cover_every_route_and_dtype():
  """World 1 covers every route x table dtype x state dtype; the sharded cases every route at
  world > 1 and row-sliced tables with 16-bit tables and bf16 buffers."""
  want = {(r, t, s) for r in ROUTE_TABLES for t, s in _DTS}
  assert {(r, t, s) for r, t, s, _, _ in WORLD1} == want
  assert {r for r, *_ in SHARDED} == set(ROUTE_TABLES) | {"rows"}
  assert {(t, s) for r, _, t, s, _, _ in SHARDED if r == "rows"} >= {
      (torch.float32, torch.float32), (torch.bfloat16, torch.bfloat16)}
  for cases in (WORLD1, SHARDED):
    assert {c[-2] for c in cases} == {"l2", "decoupled"}
    assert {bool(c[-1]) for c in cases} == {False, True}


def _world1_case(route, tdt, sdt, mode, hp, seed=5):
  rows, width = ROUTE_TABLES[route]
  return tfo._case([(rows, width, "sum")], [0, 0], [1, 2], 512, edges=True, wd=WD, mode=mode,
                   hp=hp, table_dtype=tdt, state_dtype=sdt, lrs=[0.05, 0.05, 0.02], seed=seed)


@pytest.mark.gpu
@pytest.mark.parametrize("route,tdt,sdt,mode,hp", WORLD1,
                         ids=[f"{c[0].replace(' ', '_')}-{str(c[1])[6:]}_table-"
                              f"{str(c[2])[6:]}_state" for c in WORLD1])
def test_gpu_world1_against_float64(route, tdt, sdt, mode, hp):
  """Hot rows across many 32-item chunks (``finalize_crossing_kernel``), a row touched only by
  zero gradients, three steps with an lr change; the route is asserted."""
  tfo._run(_world1_case(route, tdt, sdt, mode, hp), KIND, dev=_cuda(), spec=SPEC,
           route=route.replace(" ", "_").replace("-", "_"))


@pytest.mark.gpu
@pytest.mark.parametrize("plan,world,tdt,sdt,mode,hp", SHARDED,
                         ids=[f"{c[0].replace(' ', '_')}-w{c[1]}-{str(c[2])[6:]}_table-"
                              f"{str(c[3])[6:]}_state" for c in SHARDED])
def test_gpu_sharded_against_float64(plan, world, tdt, sdt, mode, hp):
  """The kernels through the kernel-authoritative mirror harness, the buffer read per shard."""
  case, kw = _plan(plan)
  case = dict(case, wd=WD, mode=mode, hp=hp, table_dtype=tdt, state_dtype=sdt)
  before = tur.REPLAYED.copy()
  tfo._run(case, KIND, world, plan=kw, route="any", world_cls=tur._world(tur._gpu()), slack=1.0,
           spec=SPEC)
  got = {k for k, v in tur.REPLAYED.items() if v > before.get(k, 0)}
  state = "bf16" if sdt == torch.bfloat16 else "fp32"
  want = {f"segment_update, {tur._DT[tdt]} table, {state} state"}
  if plan != "rows":
    want.add(f"segment_update, {plan}, {KIND}")
  assert want <= got, (want, got)


@pytest.mark.gpu
@pytest.mark.parametrize("tdt", [torch.float32, torch.bfloat16, torch.float16],
                         ids=lambda x: str(x)[6:])
def test_gpu_momentum_zero_is_sgd_bit_for_bit(tdt):
  """At momentum 0, plain and nesterov, the kernels give deterministic SGD's weights exactly (the
  per-row route: a fixed sum order), with the same 16-bit rounding keys."""
  case = _world1_case("per-row vec1", tdt, torch.float32, "l2", {})
  sgd = tfo._run(dict(case, deterministic=True), "sgd", dev=_cuda())
  for nesterov in (False, True):
    mom = tfo._run(dict(case, hp={"momentum": 0.0, "nesterov": nesterov}), KIND, dev=_cuda(),
                   spec=SPEC)
    for x, y in zip(mom[0].get_weights(), sgd[0].get_weights()):
      x, y = np.asarray(x, np.float32), np.asarray(y, np.float32)
      assert np.array_equal(x.view(np.uint32), y.view(np.uint32))


@pytest.mark.gpu
@pytest.mark.parametrize("mode,hp", [("l2", {}), ("decoupled", NESTEROV)], ids=["l2", "nesterov"])
def test_gpu_offloaded_against_float64(mode, hp):
  """A host-resident table behind the HBM row cache (fp32 buffer rows in the cache)."""
  case = tfo._case([(64, 16, "sum"), (6000, 16, "sum")], [0, 1, 1], [1, 2, 1], 512, wd=WD,
                   mode=mode, hp=hp, cache=2000, lrs=[0.05, 0.05], seed=8)
  tfo._run(case, KIND, dev=_cuda(), spec=SPEC)


@pytest.mark.gpu
def test_gpu_cached_equals_uncached_bit_for_bit():
  from test_decoupled_weight_decay import _pair_ids  # pylint: disable=import-outside-toplevel
  from test_offload_cache import BIG, SMALL, WAYS, _pair  # pylint: disable=import-outside-toplevel
  cached, plain = _pair(KIND, 2 * WAYS * 16, input_table_map=(0, 1), weight_decay=WD,
                        weight_decay_mode="decoupled", **NESTEROV)
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
  assert any((np.asarray(t[0]) != 0).any() for t in sp["tables"])
  for ta, tb in zip(sc["tables"], sp["tables"]):
    for a, b in zip(ta, tb):
      assert np.array_equal(np.asarray(a).view(np.uint32), np.asarray(b).view(np.uint32))


def _dense_model(p, g, b, lr, mu, nesterov, wd, mode):
  """float64 result of one ``dense_momentum`` update with its bounds (the fma order)."""
  lr, mu, wd = f32(lr), f32(mu), f32(wd)
  p, g, b = p.double(), g.double(), b.double()
  e_w = torch.zeros_like(p)
  e_g = torch.zeros_like(p)
  if wd and mode == "decoupled":
    p = (1 - lr * wd) * p
    e_w = 2.05 * U * p.abs()
  elif wd:
    g = g + wd * p
    e_g = U * g.abs()
  b = mu * b + g
  e_b = e_g + U * b.abs()
  u, e_u = b, e_b
  if nesterov:
    u = mu * b + g
    e_u = mu * e_b + e_g + U * u.abs()
  p = p - lr * u
  return {"p": p, "b": b}, {"p": 1.05 * (lr * e_u + e_w + U * p.abs()) + TINY,
                             "b": 1.05 * e_b + TINY}


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["none", "l2", "decoupled"])
@pytest.mark.parametrize("nesterov", [False, True])
@pytest.mark.parametrize("n", [4, 4 * 1001, 4 * (3 * 2**20 + 1)])
def test_gpu_dense_momentum_against_float64(n, nesterov, mode):
  from distributed_embeddings_b200.ops import _native
  from test_dense_optimizers import make_inputs  # pylint: disable=import-outside-toplevel
  ops = _native.require()
  dev = _cuda()
  wd = 0.0 if mode == "none" else 0.3
  p, g, b, _ = make_inputs("adam", n, 23, dev)  # s0: a plausible buffer of earlier steps
  inp = [x.cpu() for x in (p, g, b)]
  lr = torch.full((1,), 0.01, dtype=torch.float32, device=dev)
  p16 = torch.empty(n, dtype=torch.bfloat16, device=dev)
  decay = () if mode == "none" else (wd, {"l2": 0, "decoupled": 1}[mode])
  ops.dense_momentum(p, p16, g, b, lr, MU, nesterov, *decay)
  torch.cuda.synchronize()
  out, bound = _dense_model(*inp, 0.01, MU, nesterov, wd, mode)
  for k, got in (("p", p.cpu()), ("b", b.cpu())):
    err = (got.double() - out[k]).abs()
    assert torch.isfinite(got).all() and bool((err <= bound[k]).all()), \
        (k, float((err / bound[k]).max()))
  assert torch.equal(p16.cpu(), p.cpu().bfloat16()) and bool((g == 0).all())


@pytest.mark.gpu
def test_gpu_dlrm_step_matches_hybrid():
  """Momentum on the tables and the MLPs, ``DLRMTrainStep`` with a CUDA graph and a scheduler that
  changes the lr on every step, against ``HybridTrainer`` with the same kinds: the loss of every
  step, the buffers after the first step at 0.08 relative error (the one-step tolerance of
  ``test_dense_optimizers.py``; the bf16 paths drift apart later), and every step of the fast
  trainer follows its own buffer, ``p = p0 - lr_t * b``, on the dense parameters and the touched
  table rows, while untouched rows keep their bits."""
  from distributed_embeddings_b200.models.dlrm_fast import DLRMTrainStep
  from distributed_embeddings_b200.models.trainer import HybridTrainer
  from distributed_embeddings_b200.utils.lr_schedule import LearningRateScheduler
  from test_dense_optimizers import (  # pylint: disable=import-outside-toplevel
      _batch, _dense_named, _dlrm, _rel)
  dev = _cuda()
  lr = 0.05
  ref, fast = _dlrm(0, dev), _dlrm(0, dev)
  fast.load_state_dict(ref.state_dict())
  fast.embedding.set_weights(ref.embedding.get_weights())
  mk = lambda: LearningRateScheduler(lr, 2, 2, 4)
  hp = {"momentum": MU}
  kw = dict(lr=lr, embedding_optimizer=KIND, dense_optimizer=KIND,
            embedding_optimizer_kwargs=hp, dense_optimizer_kwargs=hp)
  t_ref = HybridTrainer(ref, scheduler=mk(), **kw)
  t_fast = DLRMTrainStep(fast, use_cuda_graph=True, scheduler=mk(), **kw)
  sched = mk()
  for step in range(1, 6):
    step_lr = f32(sched.step())
    num, cat, lab = _batch(ref.table_sizes, 512, step, dev)
    cat = [c.int() for c in cat]
    w0 = [p.detach().clone() for _, p in _dense_named(fast)]
    e0 = fast.embedding.get_weights()
    loss_ref = t_ref.step(num, cat, lab)
    loss_fast = t_fast.step(num, torch.stack(cat), lab).clone()
    torch.cuda.synchronize()
    torch.testing.assert_close(loss_fast[0], loss_ref, rtol=2e-2, atol=2e-3)
    s_ref, s_fast = t_ref.dense_optimizer_state(), t_fast.dense_optimizer_state()
    assert s_ref["kind"] == s_fast["kind"] == KIND
    for (name, p), p0 in zip(_dense_named(fast), w0):
      (b,) = (x.double() for x in s_fast["slots"][name])
      if step == 1:
        assert _rel(b, s_ref["slots"][name][0].double()) < 0.08, name
      torch.testing.assert_close(p.detach().double(), p0.double() - step_lr * b, rtol=1e-5,
                                 atol=1e-7, msg=lambda m, n=name, s=step: f"{n} step {s}: {m}")
    e_ref, e_fast = ref.embedding.get_optimizer_state(), fast.embedding.get_optimizer_state()
    if step == 1:
      flat = lambda ts: torch.cat([torch.as_tensor(np.asarray(t[0])).reshape(-1) for t in ts])
      assert _rel(flat(e_fast["tables"]).double(), flat(e_ref["tables"]).double()) < 0.08
    for t, (w_before, w_after) in enumerate(zip(e0, fast.embedding.get_weights())):
      touched = np.zeros(len(w_before), dtype=bool)
      touched[cat[t].cpu().numpy()] = True
      wb, wa = np.asarray(w_before), np.asarray(w_after)
      assert np.array_equal(wb[~touched].view(np.uint32), wa[~touched].view(np.uint32))
      b = torch.as_tensor(np.asarray(e_fast["tables"][t][0])).double()[touched]
      torch.testing.assert_close(torch.as_tensor(wa[touched]).double(),
                                 torch.as_tensor(wb[touched]).double() - step_lr * b, rtol=1e-5,
                                 atol=1e-7, msg=lambda m, t=t: f"table {t}: {m}")


@pytest.mark.gpu
def test_gpu_synthetic_step_matches_hybrid():
  """``SyntheticTrainStep`` with momentum on both halves against ``HybridTrainer``, whose dense
  step is plain PyTorch ``_foreach`` ops: the buffers of every dense parameter after one step at
  0.08 relative error, and the fast step's update follows its own buffer."""
  from distributed_embeddings_b200.models.configs import scaled, synthetic_models_v3
  from distributed_embeddings_b200.models.synthetic import InputGenerator, SyntheticModel
  from distributed_embeddings_b200.models.synthetic_fast import SyntheticTrainStep
  from distributed_embeddings_b200.models.trainer import HybridTrainer
  from test_dense_optimizers import _dense_named, _rel  # pylint: disable=import-outside-toplevel
  dev = _cuda()
  cfg = scaled(synthetic_models_v3["tiny"], 2e-4)
  mk = lambda: SyntheticModel(cfg, device=dev, compute_dtype=torch.bfloat16, backend="fused")
  torch.manual_seed(21)
  ref = mk()
  torch.manual_seed(21)
  fast = mk()
  fast.load_state_dict(ref.state_dict())
  fast.embedding.set_weights(ref.embedding.get_weights())
  (num, cat), lab = InputGenerator(cfg, 256, alpha=1.05, device=dev,
                                   mp_input_ids=ref.embedding.strategy.input_ids_list[0])[0]
  w0 = [p.detach().clone() for p in ref.dense_parameters()]
  lr = 0.05
  kw = dict(lr=lr, embedding_optimizer=KIND, dense_optimizer=KIND,
            dense_optimizer_kwargs=NESTEROV, embedding_optimizer_kwargs=NESTEROV)
  t_ref = HybridTrainer(ref, **kw)
  t_ref.step(num, cat, lab)
  t_fast = SyntheticTrainStep(fast, use_cuda_graph=True, **kw)
  t_fast.step(num, cat, lab)
  torch.cuda.synchronize()
  s_ref, s_fast = t_ref.dense_optimizer_state(), t_fast.dense_optimizer_state()
  mu = f32(NESTEROV["momentum"])
  for (name, p_ref), (_, p_fast), p0 in zip(_dense_named(ref), _dense_named(fast), w0):
    b, br = s_fast["slots"][name][0].double(), s_ref["slots"][name][0].double()
    assert (p_ref.detach() - p0).abs().sum() > 0
    assert _rel(b, br) < 0.08, name
    # first step from b = 0: b = g, and nesterov's step is lr * (mu * g + g)
    torch.testing.assert_close(p_fast.detach().double(), p0.double() - f32(lr) * (mu * b + b),
                               rtol=1e-5, atol=1e-7, msg=lambda m, n=name: f"{n}: {m}")
