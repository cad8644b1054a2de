"""Evaluation of the DLRM step: the binned ROC AUC (``utils.metrics.BinnedAUC``), the forward-only
``head_eval`` kernel and ``DLRMTrainStep.evaluate`` / ``predict`` / ``eval_metrics``.

CPU: the metric against an independent float64 port of the Keras AUC formula and against the
exact AUC within ``tie_bound``; its all-reduce at gloo world 2; the plan interpreter running a
forward-only step between two training steps at world 1-8.
GPU: ``head_eval`` against float64 with the bounds of ``test_dense_conformance.py`` (its
histogram bit for bit against the binning of its own output, its logits bit for bit against
``head_loss``), and the step's evaluation: no side effects on anything training owns, forward
equality with the training step, chunking and padding, graph versus eager, interleaving with
training steps and with the input pipeline.  The world-2 / world-8 cases skip on smaller boxes.
"""
import math
import os
import random
import socket
import sys
import traceback

import numpy as np
import pytest
import torch

from distributed_embeddings_b200.parallel import dry_run
from distributed_embeddings_b200.utils.metrics import BinnedAUC, auc_from_histogram, binary_auc
from test_dry_run import SMALL_PROFILE, _draw_grads, _draw_tables, assemble  # pylint: disable=wrong-import-order


# ------------------------------------------------------------------ metric (CPU)
def keras_auc(probs, labels, T):
  """float64 port of tf.keras.metrics.AUC(num_thresholds=T, curve='ROC',
  summation_method='interpolation'): a prediction counts above threshold t when p > t."""
  p = np.asarray(probs, dtype=np.float64)
  y = np.asarray(labels) > 0.5
  thr = np.concatenate([[-1e-7], np.arange(1, T - 1, dtype=np.float64) / (T - 1), [1 + 1e-7]])
  pos, neg = np.sort(p[y]), np.sort(p[~y])
  tp = len(pos) - np.searchsorted(pos, thr, side="right")
  fp = len(neg) - np.searchsorted(neg, thr, side="right")
  tpr, fpr = tp / len(pos), fp / len(neg)
  return float(np.sum((fpr[:-1] - fpr[1:]) * (tpr[:-1] + tpr[1:]) / 2))


def _exact_product(p32, T):
  """Predictions whose fp32 product with T - 1 is exact (no threshold within one rounding)."""
  prod = (p32 * np.float32(T - 1)).astype(np.float64)
  return p32[prod == p32.astype(np.float64) * (T - 1)]


def _grid_probs(rng, n, T):
  parts = [
      rng.integers(0, 1025, n).astype(np.float32) / np.float32(1024),  # dyadic: many ties
      _exact_product(rng.random(4 * n).astype(np.float32), T),
      np.array([0.0, 1.0, 0.0, 1.0], dtype=np.float32),
  ]
  thr = np.arange(T, dtype=np.float64) / (T - 1)
  exact = thr[thr.astype(np.float32).astype(np.float64) == thr].astype(np.float32)
  parts.append(np.repeat(exact, 3))
  p = np.concatenate(parts)
  return p[rng.permutation(len(p))]


@pytest.mark.parametrize("T", [2, 3, 200, 8000])
def test_binned_auc_matches_keras_formula(T):
  rng = np.random.default_rng(T)
  for _ in range(3):
    p = _grid_probs(rng, 3000, T)
    y = (rng.random(len(p)) < 0.3 + 0.4 * p).astype(np.float32)
    m = BinnedAUC(T)
    m.update(torch.from_numpy(p), torch.from_numpy(y))
    assert m.hist.shape == (2, T - 1) and m.hist.dtype == torch.int64
    assert int(m.hist.sum()) == len(p)
    got = m.result().auc
    assert abs(got - keras_auc(p, y, T)) <= 1e-12, (got, keras_auc(p, y, T))
  if T == 3:  # exact thresholds lie in the lower bucket (Keras: p > t)
    m = BinnedAUC(3)
    m.update(torch.tensor([0.0, 0.5, 0.50000006, 1.0]), torch.tensor([0.0, 1.0, 0.0, 1.0]))
    assert m.hist.tolist() == [[1, 1], [1, 1]]


@pytest.mark.parametrize("T", [200, 8000])
@pytest.mark.parametrize("kind", ["random", "tied", "separable"])
def test_binned_auc_within_tie_bound_of_exact(T, kind):
  g = torch.Generator().manual_seed(T)
  n = 20000
  y = (torch.rand(n, generator=g) < 0.25).float()
  if kind == "random":
    p = torch.sigmoid(torch.randn(n, generator=g) + 1.5 * y)
  elif kind == "tied":
    p = torch.tensor([0.01, 0.2, 0.2001, 0.5, 0.97])[torch.randint(0, 5, (n,), generator=g)]
    p = torch.where((y > 0) & (torch.rand(n, generator=g) < 0.5), p.roll(1), p)
  else:
    p = torch.where(y > 0, 0.7 + 0.3 * torch.rand(n, generator=g), 0.3 * torch.rand(n, generator=g))
  m = BinnedAUC(T)
  m.update(p, y)
  res = m.result()
  exact = binary_auc(y, p)
  assert abs(res.auc - exact) <= res.tie_bound + 1e-12, (res, exact)
  if kind == "separable":
    assert res.auc == 1.0 and res.tie_bound == 0.0
  if kind == "tied":
    assert res.tie_bound > 0.01  # the bound is not vacuous here


def test_binned_auc_single_class_chunks_and_reset():
  g = torch.Generator().manual_seed(5)
  p = torch.rand(1001, generator=g)
  m = BinnedAUC(50)
  m.update(p, torch.ones(1001))
  assert math.isnan(m.result().auc) and math.isnan(m.result().tie_bound)
  m.reset()
  assert int(m.hist.abs().sum()) == 0
  y = (torch.rand(1001, generator=g) < 0.5).float()
  whole, parts = BinnedAUC(50), BinnedAUC(50)
  whole.update(p, y)
  for s in range(0, 1001, 97):
    parts.update(p[s:s + 97].reshape(-1, 1), y[s:s + 97].reshape(-1, 1))
  assert torch.equal(whole.hist, parts.hist)
  assert auc_from_histogram(whole.hist) == whole.result()
  with pytest.raises(ValueError):
    BinnedAUC(1)


# ------------------------------------------------------------------ multi-process helper
def _free_port():
  with socket.socket() as s:
    s.bind(("127.0.0.1", 0))
    return s.getsockname()[1]


def _worker(rank, world, port, case, device_type, errq):
  try:
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank),
                      WORLD_SIZE=str(world))
    torch.set_num_threads(1)
    if device_type == "cuda":
      torch.cuda.set_device(rank)
      dist.init_process_group("nccl", rank=rank, world_size=world,
                              device_id=torch.device("cuda", rank))
    else:
      dist.init_process_group("gloo", rank=rank, world_size=world)
    globals()[case](rank, world)
    if device_type == "cuda":
      torch.cuda.synchronize()
    dist.barrier()
    dist.destroy_process_group()
  except Exception:  # pylint: disable=broad-except
    errq.put((rank, traceback.format_exc()))
    raise


def _launch(case, world, device_type="cpu", timeout=600):
  """One process per rank running ``case(rank, world)`` of this module (as tests/dist_utils.py
  does for the cases of dist_cases.py)."""
  import torch.multiprocessing as mp
  ctx = mp.get_context("spawn")
  errq = ctx.SimpleQueue()
  port = _free_port()
  procs = [ctx.Process(target=_worker, args=(r, world, port, case, device_type, errq))
           for r in range(world)]
  for p in procs:
    p.start()
  failed = False
  for p in procs:
    p.join(timeout)
    if p.is_alive():
      p.terminate()
      p.join()
      failed = True
    elif p.exitcode != 0:
      failed = True
  msgs = []
  while not errq.empty():
    msgs.append(errq.get())
  if failed or msgs:
    detail = "\n".join(f"--- rank {r} ---\n{tb}" for r, tb in msgs) or "timeout / crash"
    raise AssertionError(f"case {case} failed (world={world}):\n{detail}")


def _case_all_reduce(rank, world):
  g = torch.Generator().manual_seed(17)
  p = torch.rand(world * 500, generator=g)
  y = (torch.rand(world * 500, generator=g) < 0.4).float()
  m = BinnedAUC(300)
  m.update(p[rank * 500:(rank + 1) * 500], y[rank * 500:(rank + 1) * 500])
  m.all_reduce()
  one = BinnedAUC(300)
  one.update(p, y)
  assert torch.equal(m.hist, one.hist)
  assert m.result() == one.result()


def test_binned_auc_all_reduce_gloo_world2():
  _launch("_case_all_reduce", 2)


# ------------------------------------------------------------------ plan interpreter (CPU)
def _eval_plan(seed, world, kind, with_eval):
  """A one-hot plan like the DLRM step's: training steps (lookup, gradient push through
  ``routes_all``, ``backward_inplace``) and, if ``with_eval``, a forward-only step between them.
  Returns (tables after the last step, the forward-only outputs or None, the tables before it)."""
  prof = {**SMALL_PROFILE, "rows": (3, 60), "local_batch": (3, 5, 8)}
  rng = random.Random(seed)
  nrng = np.random.default_rng(seed)
  n_tables = rng.randint(max(2, world // 2), 2 * world + 2)
  sizes = [(rng.randint(*prof["rows"]), rng.choice(prof["widths"])) for _ in range(n_tables)]
  imap = list(range(n_tables)) + [rng.randint(0, n_tables - 1) for _ in range(rng.randint(0, 2))]
  kw = {"strategy": rng.choice(["basic", "memory_balanced", "memory_optimized"]),
        "input_table_map": imap}
  if rng.random() < 0.5:
    kw["column_slice_threshold"] = rng.choice([60, 150, 300])
  if world > 1 and rng.random() < 0.6:
    kw["data_parallel_threshold"] = rng.choice([40, 100])
  embs = [{"input_dim": r, "output_dim": w, "combiner": None} for r, w in sizes]
  try:
    sim, des = dry_run.build_engines(embs, world, **kw)
  except ValueError as e:
    if "Not enough table" in str(e):
      return None
    raise
  tables = _draw_tables(nrng, sizes, True)
  lb = rng.choice(prof["local_batch"])
  B = lb * world
  dp_tables = list(des[0].strategy.table_groups[0])
  for de in des:
    de.set_weights(tables)
    de.set_optimizer(kind, lr=0.5)
    de._engine.set_dp_grad_targets([torch.zeros(sizes[t]) for t in dp_tables])
    de._engine.prepare(lb, [1] * len(imap), ids64=False)
  batches = [[nrng.integers(0, sizes[t][0], B).astype(np.int32) for t in imap] for _ in range(3)]
  grads = [_draw_grads(nrng, [(B, sizes[t][1]) for t in imap], True) for _ in range(2)]

  def forward(eng, r, ids):
    sl = slice(r * lb, (r + 1) * lb)
    for v, i in zip(eng.input_views, ids):
      v.copy_(torch.from_numpy(i[sl]).reshape(v.shape))
    eng.launch_forward()
    eng.wait_output()  # the consumer's "output ready" wait (folded into interact_fwd on the GPU)

  def train(ids, g):
    def fn(r):
      eng = des[r]._engine
      with torch.no_grad():
        forward(eng, r, ids)
        gr = torch.from_numpy(np.concatenate([x[r * lb:(r + 1) * lb] for x in g], 1))
        eng.ops.push_grad(eng.routes_all, len(eng.routes_all_np), gr, eng.act, 1.0,
                          eng.sync_grad_signal())
        eng.backward_inplace()
    dry_run.run_ranks(sim, fn)

  def evaluate(ids):
    def fn(r):
      eng = des[r]._engine
      with torch.no_grad():
        forward(eng, r, ids)
        return eng.out.float().numpy().copy()
    return dry_run.run_ranks(sim, fn)

  train(batches[0], grads[0])
  outs, mid = None, None
  if with_eval:
    mid = assemble(des)
    outs = evaluate(batches[2])
  train(batches[1], grads[1])
  return assemble(des), outs, mid, (imap, batches[2], lb)


@pytest.mark.parametrize("world", [1, 2, 3, 4, 8])
@pytest.mark.parametrize("kind", ["sgd", "adagrad"])
def test_forward_only_step_between_training_steps(world, kind):
  """[train, forward-only, train] leaves every table bit for bit where [train, train] does, and
  the forward-only step reads the tables of the first training step."""
  ok = 0
  for s in range(4 if world < 8 else 2):
    seed = 7100 * world + 31 * s + (kind == "adagrad")
    a = _eval_plan(seed, world, kind, True)
    if a is None:
      continue
    b = _eval_plan(seed, world, kind, False)
    for t, (x, y) in enumerate(zip(a[0], b[0])):
      assert np.array_equal(x.view(np.int32), y.view(np.int32)), f"table {t}"
    imap, ids, lb = a[3]
    exp = np.concatenate([a[2][t][i] for t, i in zip(imap, ids)], 1)
    for r, o in enumerate(a[1]):
      np.testing.assert_array_equal(o, exp[r * lb:(r + 1) * lb], err_msg=f"rank {r}")
    ok += 1
  assert ok >= 1


# ------------------------------------------------------------------ GPU: head_eval kernel
def _ops():
  from distributed_embeddings_b200.ops import _native
  return _native.require()


def _sms():
  return torch.cuda.get_device_properties(0).multi_processor_count


def _np_bins(probs, labels, T):
  """NumPy binning of fp32 predictions (the BinnedAUC rule, computed independently)."""
  p = probs.cpu().numpy().astype(np.float32)
  k = np.ceil(p * np.float32(T - 1)).astype(np.int64) - 1
  k = np.clip(k, 0, T - 2)
  h = np.zeros((2, T - 1), dtype=np.int64)
  np.add.at(h, ((labels.cpu().numpy() > 0.5).astype(np.int64), k), 1)
  return h


def _eval_accumulators(T, seed):
  g = torch.Generator().manual_seed(seed)
  hist = torch.randint(0, 1000, (2, T - 1), generator=g).cuda()
  loss = torch.tensor([123.25], dtype=torch.float64, device="cuda")
  count = torch.tensor([77], dtype=torch.int64, device="cuda")
  return hist, loss, count


@pytest.mark.gpu
@pytest.mark.parametrize("k", [64, 128, 256, 512, 1024])
def test_head_eval(k):
  from test_dense_conformance import TINY, U32, _head_inputs, acc_bound, check_close, head_ref
  ops = _ops()
  big = 4 * _sms() * 256 + 45  # more rows than one wave of the grid: warps loop
  T = 8000
  for b in (1, 7, 1000, big):
    x, w, bias, labels = _head_inputs(b, k, seed=k + b, frac_labels=False)
    for nv in sorted({0, b // 2, b}):
      hist, loss, count = _eval_accumulators(T, k + b + nv)
      hist0, loss0, count0 = hist.clone(), loss.clone(), count.clone()
      probs = torch.full((b,), 9.0, device="cuda")
      n_valid = torch.tensor([nv], dtype=torch.int64, device="cuda")
      ops.head_eval(x, w, bias, labels, n_valid, probs, hist, loss, count)
      torch.cuda.synchronize()
      where = f"K={k} batch={b} n_valid={nv}"
      zeros = torch.zeros_like(labels)
      h0 = head_ref(x, w, bias, zeros, 1.0)  # label 0, 1 / batch = 1: dl = sigmoid(logit)
      check_close(f"head_eval/probs {where}", probs, h0["dl"], h0["e_dl"] + TINY)
      # the histogram is the binning of the kernel's own predictions, bit for bit
      exp_hist = hist0.cpu().numpy() + _np_bins(probs[:nv], labels[:nv], T)
      assert np.array_equal(hist.cpu().numpy(), exp_hist), where
      assert int(count) == int(count0) + nv, where
      h = head_ref(x[:nv], w, bias, labels[:nv], 1.0)
      lt = h["loss_terms"]
      check_close(f"head_eval/loss {where}", loss, loss0.double() + lt.sum(),
                  h["e_loss_terms"].sum() + acc_bound(nv + 2, lt.abs().sum()) +
                  U32 * float(loss0.abs()))
      if nv == 0:
        assert torch.equal(loss, loss0) and torch.equal(hist, hist0), where


@pytest.mark.gpu
@pytest.mark.parametrize("k", [64, 256, 1024])
def test_head_eval_logits_equal_head_loss(k):
  """head_eval's sigmoid input is head_loss's logit bit for bit: with label 0 and 1 / batch = 1,
  head_loss's bias gradient of a one-row batch is exactly its sigmoid(logit), the value
  head_eval writes; the one-row logits equal the full-batch logits of head_loss."""
  from test_dense_conformance import _head_inputs, check_bits
  ops = _ops()
  b = 300
  x, w, bias, labels = _head_inputs(b, k, seed=5 + k, frac_labels=False)
  probs = torch.empty(b, device="cuda")
  hist = torch.zeros(2, 99, dtype=torch.int64, device="cuda")
  f = lambda n: torch.zeros(n, device="cuda")  # noqa: E731
  ops.head_eval(x, w, bias, labels, torch.zeros(1, dtype=torch.int64, device="cuda"), probs, hist,
                torch.zeros(1, dtype=torch.float64, device="cuda"),
                torch.zeros(1, dtype=torch.int64, device="cuda"))
  full = f(b)
  ops.head_loss(x, w, bias, labels, 1.0 / b, torch.empty_like(x), f(k), f(1), f(k), f(1), full)
  rows = list(range(0, b, 7)) + [b - 1]
  sig, logit = f(len(rows)), f(len(rows))
  for j, s in enumerate(rows):
    db = f(1)
    lg = f(1)
    ops.head_loss(x[s:s + 1], w, bias, torch.zeros(1, device="cuda"), 1.0, torch.empty_like(x[:1]),
                  f(k), db, f(k), f(1), lg)
    sig[j], logit[j] = db[0], lg[0]
  check_bits("head_eval/logit one row vs batch", logit, full[rows])
  check_bits("head_eval/probs vs head_loss sigmoid", probs[rows], sig)


@pytest.mark.gpu
def test_head_eval_rejects_bad_arguments():
  ops = _ops()
  b, k = 16, 256
  from test_dense_conformance import _head_inputs
  x, w, bias, labels = _head_inputs(b, k, seed=1, frac_labels=False)
  i64 = lambda *s: torch.zeros(*s, dtype=torch.int64, device="cuda")  # noqa: E731

  def call(**kw):
    a = dict(x=x, w=w, bias=bias, labels=labels, n_valid=i64(1),
             probs=torch.zeros(b, device="cuda"), hist=i64(2, 99),
             loss=torch.zeros(1, dtype=torch.float64, device="cuda"), count=i64(1))
    a.update(kw)
    ops.head_eval(a["x"], a["w"], a["bias"], a["labels"], a["n_valid"], a["probs"], a["hist"],
                  a["loss"], a["count"])

  bad = [
      ("K in", dict(x=torch.zeros(b, 96, dtype=torch.bfloat16, device="cuda"))),
      ("x must", dict(x=x.float())),
      ("x must be contiguous",
       dict(x=torch.zeros(b, 2 * k, dtype=torch.bfloat16, device="cuda")[:, :k])),
      ("w must hold K", dict(w=w[:k // 2])),
      ("w must be", dict(w=w.float())),
      ("bias must", dict(bias=bias.float())),
      ("labels must hold", dict(labels=labels[:b - 1])),
      ("labels must be", dict(labels=labels.double())),
      ("n_valid must be one", dict(n_valid=i64(2))),
      ("n_valid must be an int64", dict(n_valid=torch.zeros(1, dtype=torch.int32, device="cuda"))),
      ("n_valid must be an int64", dict(n_valid=torch.zeros(1, dtype=torch.int64))),
      ("probs must hold", dict(probs=torch.zeros(b + 1, device="cuda"))),
      ("probs must be", dict(probs=torch.zeros(b, dtype=torch.float64, device="cuda"))),
      ("hist must be \\[2", dict(hist=i64(3, 99))),
      ("hist must be \\[2", dict(hist=i64(2, 0))),
      ("hist must be \\[2", dict(hist=i64(198))),
      ("hist must be a", dict(hist=torch.zeros(2, 99, dtype=torch.int32, device="cuda"))),
      ("loss_sum must be", dict(loss=torch.zeros(1, device="cuda"))),
      ("loss_sum must hold", dict(loss=torch.zeros(2, dtype=torch.float64, device="cuda"))),
      ("count must be", dict(count=torch.zeros(1, device="cuda"))),
      ("count must hold", dict(count=i64(2))),
  ]
  for msg, kw in bad:
    with pytest.raises(RuntimeError, match=msg):
      call(**kw)
  torch.cuda.synchronize()


# ------------------------------------------------------------------ GPU: the DLRM step
SIZES = [300 + 11 * i for i in range(26)]
LR = 0.5


def _make_step(gemm, use_graph, table_dtype, opt, seed=0):
  from distributed_embeddings_b200.models.dlrm import DLRM
  from distributed_embeddings_b200.models.dlrm_fast import DLRMTrainStep
  torch.manual_seed(seed)
  model = DLRM(SIZES, device=torch.device("cuda", 0), compute_dtype=torch.bfloat16,
               backend="fused", table_dtype=table_dtype)
  step = DLRMTrainStep(model, lr=LR if opt == "sgd" else 0.05, embedding_optimizer=opt,
                       use_cuda_graph=use_graph, gemm=gemm)
  return model, step


def _batch(b, seed, device="cuda"):
  g = torch.Generator().manual_seed(seed)
  num = torch.rand(b, 13, generator=g)
  cat = torch.stack([torch.randint(0, s, (b,), generator=g, dtype=torch.int32) for s in SIZES])
  lab = torch.randint(0, 2, (b,), generator=g).float()
  return num.to(device), cat.to(device), lab.to(device)


def _tensors(obj):
  if isinstance(obj, torch.Tensor):
    yield obj
  elif isinstance(obj, dict):
    for v in obj.values():
      yield from _tensors(v)
  elif isinstance(obj, (list, tuple)):
    for v in obj:
      yield from _tensors(v)


def _snapshot(model, step):
  """Bytes of everything a training step owns."""
  eng = step.engine
  parts = [p.detach() for p in model.embedding.parameters()]
  parts += list(_tensors(eng.opt_state)) + [eng.step_t, step.p32, step.p16, step.g32, step.lr_t]
  parts += list(_tensors(step._stage))
  return [t.contiguous().reshape(-1).view(torch.uint8).clone() for t in parts]


def _check_snapshot(before, after, what):
  assert len(before) == len(after)
  for i, (a, b) in enumerate(zip(before, after)):
    assert torch.equal(a, b), f"{what}: tensor {i} of the training state changed"


STEP_CASES = [(g, graph, dt, opt) for g in ("cublas", "tcgen05") for graph in (False, True)
              for dt in ("fp32", "bf16") for opt in ("sgd", "adagrad")]
_DT = {"fp32": torch.float32, "bf16": torch.bfloat16}


@pytest.mark.gpu
@pytest.mark.parametrize("gemm,use_graph,table_dtype,opt", STEP_CASES)
def test_step_evaluation(gemm, use_graph, table_dtype, opt):
  from test_dense_conformance import TINY, U32, acc_bound, check_bits, check_close, head_ref
  model, step = _make_step(gemm, use_graph, _DT[table_dtype], opt)
  b = 512
  for s in range(2):
    step.step(*_batch(b, s))
  torch.cuda.synchronize()
  before = _snapshot(model, step)

  # chunking and padding: 2.5 batches, last chunk padded
  n = b * 5 // 2
  num, cat, lab = _batch(n, 11)
  step.evaluate(num, cat, lab)
  probs = step.predict(num, cat)
  torch.cuda.synchronize()
  _check_snapshot(before, _snapshot(model, step), "evaluate / predict")
  ref = BinnedAUC(step.eval_auc.num_thresholds, device="cuda")
  ref.update(probs, lab)
  assert torch.equal(step.eval_auc.hist, ref.hist)
  # per-chunk predictions (a chunk of its own, padded differently) equal the long run's
  H = step.head
  w, bias = H.w16.view(-1), H.b16
  loss_ref, loss_bound = 0.0, 0.0
  for s0 in range(0, n, b):
    m = min(b, n - s0)
    p = step.predict(num[s0:s0 + m], cat[:, s0:s0 + m])
    check_bits("predict chunk vs long run", p, probs[s0:s0 + m])
    x = step.top[-1].y[:m]
    h = head_ref(x, w, bias, lab[s0:s0 + m], 1.0)
    loss_ref += float(h["loss_terms"].sum())
    loss_bound += float(h["e_loss_terms"].sum())
    h0 = head_ref(x, w, bias, torch.zeros_like(lab[s0:s0 + m]), 1.0)
    check_close("step predict vs float64 sigmoid", p, h0["dl"], h0["e_dl"] + TINY)
  met = step.eval_metrics(reset=False)
  assert met["samples"] == n
  loss_bound += acc_bound(n + 2, abs(loss_ref))
  assert abs(met["log_loss"] * n - loss_ref) <= loss_bound + n * U32 * abs(loss_ref), met
  res = ref.result()
  assert met["auc"] == res.auc and met["tie_bound"] == res.tie_bound
  assert abs(met["auc"] - binary_auc(lab, probs)) <= met["tie_bound"] + 1e-12
  met2 = step.eval_metrics()  # reset=True
  assert met2 == met
  assert step.eval_metrics()["samples"] == 0
  _check_snapshot(before, _snapshot(model, step), "eval_metrics")

  # graph and eager predict agree bit for bit
  saved = step.use_cuda_graph
  step.use_cuda_graph = not saved
  try:
    other = step.predict(num, cat)
  finally:
    step.use_cuda_graph = saved
  check_bits("predict graph vs eager", other, probs)

  # forward equality with the training step: run a step with learning rate 0 (weights and
  # tables unchanged), keep its top-MLP output, evaluate the same batch
  tb = _batch(b, 21)
  step.set_lr(0.0)
  step.step(*tb)
  torch.cuda.synchronize()
  y_train = step.top[-1].y.clone()
  step.set_lr(step.lr if step.lr else LR)
  p_step = step.predict(tb[0], tb[1])
  check_bits("eval top-MLP output vs training forward", step.top[-1].y, y_train)
  h0 = head_ref(y_train, w, bias, torch.zeros_like(tb[2]), 1.0)
  check_close("step predict vs sigmoid of the training forward", p_step, h0["dl"],
              h0["e_dl"] + TINY)
  # ... and the autograd module
  model.eval()
  with torch.no_grad():
    p_mod = torch.sigmoid(model(tb[0], list(tb[1])).float()).reshape(-1)
  model.train()
  torch.testing.assert_close(p_step, p_mod, rtol=2e-2, atol=2e-3)


@pytest.mark.gpu
def test_evaluate_before_a_training_batch_raises():
  _, step = _make_step("cublas", True, torch.float32, "sgd")
  num, cat, lab = _batch(8, 0)
  with pytest.raises(RuntimeError, match="training batch first"):
    step.evaluate(num, cat, lab)


INTERLEAVE_CASES = [("cublas", True, "fp32", "sgd"), ("tcgen05", True, "bf16", "adagrad"),
                    ("cublas", False, "bf16", "sgd"), ("tcgen05", False, "fp32", "adagrad")]


@pytest.mark.gpu
@pytest.mark.parametrize("gemm,use_graph,table_dtype,opt", INTERLEAVE_CASES)
def test_evaluation_between_training_steps(gemm, use_graph, table_dtype, opt):
  """[3 steps, evaluate, 3 steps] trains like [6 steps]; with the input pipeline, an evaluation
  between prefetch() and run_prefetched() as well.  Not bitwise: the ReLU-bias and head kernels
  use float atomics."""
  b = 256
  batches = [_batch(b, 40 + i) for i in range(6)]
  ev = _batch(b * 3 // 2, 99)
  losses = []
  models = []
  for with_eval in (True, False):
    model, step = _make_step(gemm, use_graph, _DT[table_dtype], opt, seed=3)
    ls = []
    for i in range(3):
      ls.append(float(step.step(*batches[i])))
    if with_eval:
      step.evaluate(*ev)
      step.predict(ev[0], ev[1])
    for i in range(3, 6):
      ls.append(float(step.step(*batches[i])))
    losses.append(ls)
    models.append(model)
  torch.cuda.synchronize()
  assert losses[0] == pytest.approx(losses[1], rel=1e-5)
  for p, q in zip(models[0].dense_parameters(), models[1].dense_parameters()):
    torch.testing.assert_close(p, q, rtol=1e-4, atol=1e-5)

  # prefetch -> evaluate -> run_prefetched
  pinned = [tuple(t.cpu().pin_memory() for t in bt) for bt in batches]
  losses, models = [], []
  for with_eval in (True, False):
    model, step = _make_step(gemm, use_graph, _DT[table_dtype], opt, seed=4)
    ls = []
    step.prefetch(*pinned[0])
    for i in range(len(pinned)):
      if with_eval and i == 2:
        step.evaluate(*ev)
      loss = step.run_prefetched()
      if i + 1 < len(pinned):
        step.prefetch(*pinned[i + 1])
      if with_eval and i == 3:
        step.evaluate(*ev)  # between prefetch() and the run_prefetched() that consumes it
      ls.append(float(loss))
    losses.append(ls)
    models.append(model)
  torch.cuda.synchronize()
  assert losses[0] == pytest.approx(losses[1], rel=1e-5)
  for p, q in zip(models[0].dense_parameters(), models[1].dense_parameters()):
    torch.testing.assert_close(p, q, rtol=1e-4, atol=1e-5)


# ------------------------------------------------------------------ GPU: world 2 and 8
def _case_dist_eval(rank, world):
  """Every rank trains on its slice of the global batch with an evaluation in between; the
  result must match the single-process step on the global batch (built on every rank, seeded
  alike), and eval_metrics() must equal one process's metrics over the global eval batch."""
  import torch.distributed as dist
  from distributed_embeddings_b200.models.dlrm import DLRM
  from distributed_embeddings_b200.models.dlrm_fast import DLRMTrainStep
  dev = torch.device("cuda", rank)
  torch.manual_seed(7)
  ref_model = DLRM(SIZES, device=dev, compute_dtype=torch.bfloat16, backend="fused",
                   world_size=1, rank=0)
  torch.manual_seed(7)
  model = DLRM(SIZES, device=dev, compute_dtype=torch.bfloat16, backend="fused")
  model.load_state_dict({k: v for k, v in ref_model.state_dict().items() if "embedding" not in k},
                        strict=False)
  model.embedding.set_weights(ref_model.embedding.get_weights(all_ranks=True))
  ref = DLRMTrainStep(ref_model, lr=LR, embedding_optimizer="sgd", use_cuda_graph=False)
  step = DLRMTrainStep(model, lr=LR, embedding_optimizer="sgd", use_cuda_graph=True)
  lb = 128
  B = lb * world
  sl = slice(rank * lb, (rank + 1) * lb)
  batches = [_batch(B, 70 + i, dev) for i in range(4)]
  ev = _batch(B * 3 // 2, 98, dev)
  evl = B * 3 // 2 // world
  esl = slice(rank * evl, (rank + 1) * evl)
  for i, (num, cat, lab) in enumerate(batches):
    l_ref = ref.step(num, cat, lab).clone()
    loss = step.step(num[sl], cat[:, sl].contiguous(), lab[sl]).clone()
    dist.all_reduce(loss)
    torch.testing.assert_close(loss / world, l_ref, rtol=1e-2, atol=1e-3)
    if i == 1:
      step.evaluate(ev[0][esl], ev[1][:, esl].contiguous(), ev[2][esl])
      met = step.eval_metrics()
      probs = step.predict(ev[0][esl], ev[1][:, esl].contiguous())
      gathered = [torch.empty_like(probs) for _ in range(world)]
      dist.all_gather(gathered, probs)
      one = BinnedAUC(step.eval_auc.num_thresholds, device=dev)
      one.update(torch.cat(gathered), ev[2][:evl * world])
      res = one.result()
      assert met["samples"] == evl * world
      assert met["auc"] == res.auc and met["tie_bound"] == res.tie_bound, (met, res)
      # the single-process step's predictions on the global eval batch
      p_ref = ref.predict(ev[0][:evl * world], ev[1][:, :evl * world])
      torch.testing.assert_close(torch.cat(gathered), p_ref, rtol=2e-2, atol=2e-3)
  step.ctx.check_errors()
  for (n1, p1), (_, p2) in zip(ref_model.named_parameters(), model.named_parameters()):
    if "embedding" not in n1:
      torch.testing.assert_close(p2, p1, rtol=3e-2, atol=3e-3)


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 8])
def test_distributed_evaluation(world):
  if torch.cuda.device_count() < world:
    pytest.skip(f"needs {world} GPUs")
  _launch("_case_dist_eval", world, "cuda")
