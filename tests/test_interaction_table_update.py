"""The single-GPU DLRM step with the SGD update of the large tables applied by the interaction
backward (``DLRMTrainStep(fused_table_update=True)``, ``FusedEngine.producer_update``).

GPU:
  * one eager step and three graph replays against ``fused_table_update=False`` on identical
    weights and batches, at batch 777 and 8192, uniform and power-law (alpha 1.05) ids, with 4-row,
    medium and 1M-row tables: the forward and the interaction backward are bit identical, every
    table row is within the fp32 accumulation bound of the float64 update, untouched rows are bit
    identical;
  * the zero-rate warm-up passes leave every table bit identical;
  * ineligible configurations (Adagrad, bf16 tables) run the schedule of ``fused_table_update=False``;
  * ``interact_bwd`` rejects malformed apply records before any launch.
CPU (plan interpreter): the descriptor split at world 1, the configurations that get none, and a
step whose producer applies the large tables against the unsharded SGD reference.
"""
import numpy as np
import pytest
import torch

from distributed_embeddings_b200.parallel import dry_run

SIZES = [4, 4, 97, 2499, 2500, 3001, 40_000, 1_000_000]
LR = 0.5
U32 = 2.0 ** -24


def _ids(rows, b, alpha, g):
  if alpha <= 0:
    return torch.randint(0, rows, (b,), generator=g, dtype=torch.int32)
  # power law over a random permutation of the rows: a few hot rows take most of the samples
  k = min(rows, 100_000)
  p = torch.arange(1, k + 1, dtype=torch.float64) ** -alpha
  hot = torch.multinomial(p / p.sum(), b, replacement=True, generator=g)
  perm = torch.randperm(rows, generator=g)[:k]
  return perm[hot].to(torch.int32)


def _batch(b, alpha, seed):
  g = torch.Generator().manual_seed(seed)
  num = torch.rand(b, 13, generator=g).cuda()
  cat = torch.stack([_ids(s, b, alpha, g) for s in SIZES]).cuda()
  lab = torch.randint(0, 2, (b,), generator=g).float().cuda()
  return num, cat, lab


def _pair(use_graph, seed=0, **kw):
  """Two steps on identical weights: the producer update on (a) and off (b)."""
  from distributed_embeddings_b200.models.dlrm import DLRM
  from distributed_embeddings_b200.models.dlrm_fast import DLRMTrainStep
  dev = torch.device("cuda", 0)
  torch.manual_seed(seed)
  ma = DLRM(SIZES, device=dev, compute_dtype=torch.bfloat16, backend="fused")
  mb = DLRM(SIZES, device=dev, compute_dtype=torch.bfloat16, backend="fused")
  mb.load_state_dict(ma.state_dict())
  mb.embedding.set_weights(ma.embedding.get_weights())
  sa = DLRMTrainStep(ma, lr=LR, use_cuda_graph=use_graph, fused_table_update=True,
                     fused_update_min_rows=2500, **kw)
  sb = DLRMTrainStep(mb, lr=LR, use_cuda_graph=use_graph, fused_table_update=False, **kw)
  return ma, mb, sa, sb


def _tables(model):
  return [torch.from_numpy(w).cuda() for w in model.embedding.get_weights()]


def _watch(step):
  """Record the ops the step and its engine launch."""
  proxy = _Calls(step.ops)
  step.ops = step.engine.ops = proxy
  return proxy


class _Calls:
  """Forwards every op; records how interact_bwd and scatter_add_bwd were called."""

  def __init__(self, ops):
    self._ops = ops
    self.calls = []

  def __getattr__(self, name):
    fn = getattr(self._ops, name)

    def call(*args, **kwargs):
      if name == "interact_bwd":
        self.calls.append((name, len(args) > 13))
      elif name == "scatter_add_bwd":
        self.calls.append((name, int(args[1])))
      else:
        self.calls.append((name, None))
      return fn(*args, **kwargs)

    return call


def _grad_rows(step):
  """[batch, n_emb, dim] bf16 embedding gradient of a step without the producer update (its
  receive buffer holds every feature's gradient row)."""
  eng, dim = step.engine, step.dim
  g = torch.empty(step._batch, step.n_emb, dim, dtype=torch.float64, device="cuda")
  for i, d in enumerate(eng.cdesc_np):
    f = int(d["dst_col"]) // dim
    rc = int(eng.mpdesc_np[i]["dst_col"])
    g[:, f] = eng.recv[:step._batch, rc:rc + dim].double()
  return g


def _check_tables(name, old, new, cats, grads):
  """new = old - LR * sum of the gradient rows of the samples that hit a row, within the fp32
  accumulation bound (any order of the fp32 additions); untouched rows bit identical."""
  for t in range(len(SIZES)):
    rows = old[t].shape[0]
    o = old[t].double()
    gsum = torch.zeros(rows, o.shape[1], dtype=torch.float64, device="cuda")
    gabs = torch.zeros_like(gsum)
    occ = torch.zeros(rows, dtype=torch.float64, device="cuda")
    for cat, g in zip(cats, grads):
      ids = cat[t].long()
      gsum.index_add_(0, ids, g[:, t])
      gabs.index_add_(0, ids, g[:, t].abs())
      occ.index_add_(0, ids, torch.ones_like(ids, dtype=torch.float64))
    touched = occ > 0
    ref = o - LR * gsum
    bound = 2 * (occ[:, None] + 1) * U32 * (o.abs() + LR * gabs) + 1e-30
    err = (new[t].double() - ref).abs()
    bad = (err > bound) & touched[:, None]
    assert not bool(bad.any()), \
        f"{name}: table {t} ({rows} rows): {int(bad.sum())} elements beyond the bound, max " \
        f"excess {float((err - bound)[bad].max()):.3e}"
    assert torch.equal(new[t][~touched], old[t][~touched]), f"{name}: table {t} untouched rows"


@pytest.mark.gpu
@pytest.mark.parametrize("b", [777, 8192])
@pytest.mark.parametrize("alpha", [0.0, 1.05])
def test_one_step_matches_scatter(b, alpha):
  ma, mb, sa, sb = _pair(use_graph=False)
  proxy = _watch(sa)
  num, cat, lab = _batch(b, alpha, seed=b)
  old = _tables(mb)
  p0 = sb.p32.clone()
  sa.step(num, cat, lab)
  sb.step(num, cat, lab)
  torch.cuda.synchronize()
  small = sum(1 for s in SIZES if s < sa.fused_update_min_rows)
  assert ("interact_bwd", True) in proxy.calls
  assert ("scatter_add_bwd", small) in proxy.calls
  ea, eb = sa.engine, sb.engine
  for what, x, y in (("eng.out", ea.out, eb.out), ("z", sa.z, sb.z), ("dz", sa.dz, sb.dz),
                     ("hb.dy", sa.bottom[-1].dy, sb.bottom[-1].dy),
                     ("hb.y", sa.bottom[-1].y, sb.bottom[-1].y)):
    assert torch.equal(x, y), what
  # dense parameters: not bit for bit.  The bias gradients are fp32 atomics whose order depends
  # on how the streams overlap, and the overlap changes with the update's split (the scatter
  # left on the side stream is shorter).  1e-3 of the update covers that reordering (about
  # 1e-6 of it in practice) and still fails on any missing or doubled term.
  upd = (sb.p32 - p0).abs()
  assert bool(((sa.p32 - sb.p32).abs() <= 1e-3 * upd + 2 * U32 * sb.p32.abs()).all())
  grads = [_grad_rows(sb)]
  _check_tables("fused", old, _tables(ma), [cat], grads)
  _check_tables("scatter", old, _tables(mb), [cat], grads)


@pytest.mark.gpu
@pytest.mark.parametrize("alpha", [0.0, 1.05])
def test_graph_replays_match_scatter(alpha):
  ma, mb, sa, sb = _pair(use_graph=True, seed=3)
  old = _tables(mb)
  batches = [_batch(777, alpha, seed=70 + i) for i in range(3)]
  la, lb = [], []
  for num, cat, lab in batches:
    la.append(float(sa.step(num, cat, lab)))
    lb.append(float(sb.step(num, cat, lab)))
  torch.cuda.synchronize()
  assert la == pytest.approx(lb, rel=1e-3)
  ta, tb = _tables(ma), _tables(mb)
  hit = [torch.zeros(s, dtype=torch.bool, device="cuda") for s in SIZES]
  for _, cat, _ in batches:
    for t in range(len(SIZES)):
      hit[t][cat[t].long()] = True
  for t in range(len(SIZES)):
    moved = (tb[t] - old[t]).abs().max()
    assert float(moved) > 0, t
    assert float((ta[t] - tb[t]).abs().max()) <= 1e-2 * float(moved) + 1e-7, t
    assert torch.equal(ta[t][~hit[t]], old[t][~hit[t]]), t


@pytest.mark.gpu
def test_zero_rate_warmup_leaves_tables():
  ma, _, sa, _ = _pair(use_graph=True, seed=5)
  proxy = _watch(sa)
  num, cat, lab = _batch(777, 0.0, seed=1)
  old = _tables(ma)
  sa.load_batch(num, cat, lab)
  # the warm-up of run(): zero learning rate, dry updates, eager passes of the captured schedule
  sa.lr_t.zero_()
  sa.engine.dry_updates(True)
  for _ in range(2):
    sa._step_impl()
  sa.engine.dry_updates(False)
  torch.cuda.synchronize()
  assert ("interact_bwd", True) in proxy.calls
  for t, (a, b) in enumerate(zip(old, _tables(ma))):
    assert torch.equal(a, b), t


@pytest.mark.gpu
@pytest.mark.parametrize("kw", [{"embedding_optimizer": "adagrad"}, {"table_dtype": "bf16"}])
def test_ineligible_steps_run_todays_schedule(kw):
  from distributed_embeddings_b200.models.dlrm import DLRM
  from distributed_embeddings_b200.models.dlrm_fast import DLRMTrainStep
  dev = torch.device("cuda", 0)
  sizes = [3000, 5000, 4]
  runs = []
  for fused in (True, False):
    torch.manual_seed(0)
    mkw = {"table_dtype": torch.bfloat16} if "table_dtype" in kw else {}
    model = DLRM(sizes, device=dev, compute_dtype=torch.bfloat16, backend="fused", **mkw)
    step = DLRMTrainStep(model, lr=0.1, use_cuda_graph=False, fused_table_update=fused,
                         embedding_optimizer=kw.get("embedding_optimizer", "sgd"))
    proxy = _watch(step)
    g = torch.Generator().manual_seed(2)
    cat = torch.stack([torch.randint(0, s, (256,), generator=g, dtype=torch.int32)
                       for s in sizes]).to(dev)
    step.step(torch.rand(256, 13, generator=g).to(dev), cat,
              torch.randint(0, 2, (256,), generator=g).float().to(dev))
    torch.cuda.synchronize()
    assert step.engine.producer_update(step.dim, 1) is None
    runs.append(proxy.calls)
  assert runs[0] == runs[1]
  assert ("interact_bwd", False) in runs[0]


@pytest.mark.gpu
def test_interact_bwd_rejects_bad_apply_records():
  from distributed_embeddings_b200.ops import _native
  ops = _native.require()
  b, n_emb, dim = 64, 2, 128
  bf = dict(dtype=torch.bfloat16, device="cuda")
  bottom, emb = torch.randn(b, dim, **bf), torch.randn(b, n_emb * dim, **bf)
  dz = torch.randn(b, 512, **bf)
  dbottom = torch.empty(b, dim, **bf)
  demb = torch.zeros(b, n_emb * dim, **bf)
  table = torch.zeros(1000, dim, device="cuda")
  ids = torch.zeros(b, dtype=torch.int32, device="cuda")

  def rec(**over):
    a = np.zeros(n_emb, dtype=_native.INPUT_DESC)
    a[1]["table"], a[1]["ids"], a[1]["sub_rows"] = table.data_ptr(), ids.data_ptr(), 1000
    a[1]["width"], a[1]["hotness"] = dim, 1
    for k, v in over.items():
      a[1][k] = v
    return torch.from_numpy(a.view(np.uint8).copy())

  def call(apply, d=dim, e=emb, bt=bottom, db=dbottom):
    ops.interact_bwd(bt, e, n_emb, dz, db, demb.data_ptr(), demb.stride(0), 1.0, None, 0, [],
                     None, 0, apply, -0.5, 0, False)

  before = table.clone()
  cases = [
      (rec().cuda(), "CPU tensor"),
      (rec().view(torch.int8), "uint8"),
      (rec()[:-8], "one InputDesc per embedding row"),
      (rec(width=64), "128 wide"),
      (rec(hotness=2), "one-hot"),
      (rec(offsets=16), "one-hot"),
      (rec(ids=0), "one-hot"),
      (rec(table=table.data_ptr() + 4), "16-byte aligned"),
      (rec(ids=ids.data_ptr() + 2), "aligned to their element size"),
      (rec(row_base=-1), "negative"),
  ]
  for apply, msg in cases:
    with pytest.raises(RuntimeError, match=msg):
      call(apply)
  # a 64-wide interaction cannot take applied rows
  with pytest.raises(RuntimeError, match="128 wide"):
    call(rec(), bt=bottom[:, :64].contiguous(), e=emb[:, :2 * 64].contiguous(),
         db=dbottom[:, :64].contiguous())
  torch.cuda.synchronize()
  assert torch.equal(table, before)
  # a well-formed record updates the table: every sample hits row 0 with -0.5 x its gradient
  call(rec())
  ref = torch.zeros(b, n_emb * dim, **bf)
  ops.interact_bwd(bottom, emb, n_emb, dz, dbottom, ref.data_ptr(), ref.stride(0), 1.0, None, 0,
                   [], None, 0)
  torch.cuda.synchronize()
  want = -0.5 * ref[:, dim:].double().sum(0)
  bound = 2 * (b + 1) * U32 * 0.5 * ref[:, dim:].double().abs().sum(0) + 1e-30
  assert bool(((table[0].double() - want).abs() <= bound).all())
  assert torch.equal(table[1:], before[1:])
  assert torch.equal(demb[:, :dim], ref[:, :dim])  # the routed feature is stored as before


# ------------------------------------------------------------------ CPU: the plan interpreter
def _dry_engine(world, sizes, hot=1, kind="sgd", width=128):
  embs = [{"input_dim": r, "output_dim": width, "combiner": "sum" if hot > 1 else None}
          for r in sizes]
  sim, des = dry_run.build_engines(embs, world, dry_run.DryWorld, strategy="memory_balanced")
  rng = np.random.default_rng(0)
  tables = [rng.standard_normal((r, width)).astype(np.float32) for r in sizes]
  for de in des:
    de.set_weights(tables)
    de.set_optimizer(kind, lr=0.5)
  return sim, des, tables


def test_split_at_world_one():
  sizes = [3, 40, 9, 70]
  sim, des, _ = _dry_engine(1, sizes)
  de, eng = des[0], des[0]._engine
  lb = 6
  ids = [torch.zeros(lb, dtype=torch.int64) for _ in sizes]
  dry_run.run_ranks(sim, lambda r: de(ids, concat=True))
  split = eng.producer_update(128, min_rows=10)
  assert split is not None
  recs = np.frombuffer(split.apply_descs.numpy().tobytes(), dtype=dry_run.INPUT_DESC)
  assert len(recs) == len(sizes)
  applied = [f for f in range(len(sizes)) if int(recs[f]["table"])]
  assert applied == [f for f, s in enumerate(sizes) if s >= 10]
  assert split.scale == -1.0 and split.scale_ptr == eng.lr_t.data_ptr()
  assert split.n_rest == sum(1 for s in sizes if s < 10)
  # applied and scattered descriptors cover the model-parallel inputs once each
  kept = dry_run.DryOps._descs(split.rest_descs, split.n_rest)
  key = lambda d: (int(d["table"]), int(d["row_base"]), int(d["ids"]))  # noqa: E731
  got = sorted([key(d) for d in kept] + [key(recs[f]) for f in applied])
  assert got == sorted(key(d) for d in eng.mpdesc_np)
  eng.dry_updates(True)
  assert eng.producer_update(128, min_rows=10).scale == 0.0
  eng.dry_updates(False)
  assert eng.producer_update(128, min_rows=1000) is None  # nothing large enough


def test_stale_producer_update_is_rejected():
  """A split built for another plan (here: another batch size) must not pick the scattered
  tables of the current one."""
  sizes = [3, 40]
  sim, des, _ = _dry_engine(1, sizes)
  de, eng = des[0], des[0]._engine

  def fwd(lb):
    dry_run.run_ranks(sim, lambda r: de([torch.zeros(lb, dtype=torch.int64) for _ in sizes],
                                        concat=True))

  fwd(4)
  stale = eng.producer_update(128, min_rows=10)
  fwd(6)
  with pytest.raises(ValueError, match="another plan"):
    dry_run.run_ranks(sim, lambda r: eng.backward_inplace(stale))


def _engine_step(world, sizes, fused, hot=1, kind="sgd", width=128, min_rows=1):
  """One forward + gradient push + backward of the hand-scheduled steps' engine calls on the
  plan interpreter, with (``fused``) or without the producer's table update.  Returns every
  rank's op calls and the updated tables."""
  sim, des, _ = _dry_engine(world, sizes, hot=hot, kind=kind, width=width)
  lb = 4
  rng = np.random.default_rng(3)
  shape = (lb * world, hot) if hot > 1 else (lb * world,)
  ids = [torch.from_numpy(rng.integers(0, s, shape)) for s in sizes]
  g = torch.from_numpy(rng.standard_normal((lb * world, len(sizes) * width))
                       .astype(np.float32)).bfloat16()

  def rank_fn(r):
    de, eng = des[r], des[r]._engine
    sl = slice(r * lb, (r + 1) * lb)
    with torch.no_grad():
      de([x[sl] for x in ids], concat=True)
      split = eng.producer_update(width, min_rows) if fused else None
      eng.ops.push_grad(eng.routes_all, len(eng.routes_all_np), g[sl], eng.act, 1.0,
                        eng.sync_grad_signal())
      if split is not None:
        eng.ops.interact_bwd_apply(g[sl], *split.interact_args())
      eng.backward_inplace(split)
    return dict(eng.ops.calls), de.get_weights()  # get_weights is collective: every rank calls

  outs = dry_run.run_ranks(sim, rank_fn)
  return [c for c, _ in outs], outs[0][1]


@pytest.mark.parametrize("case", ["world2", "adagrad", "multi_hot", "width64"])
def test_ineligible_engine_steps_run_todays_ops(case):
  kw = {"world": 2 if case == "world2" else 1, "sizes": [40, 50, 60],
        "hot": 2 if case == "multi_hot" else 1, "kind": "adagrad" if case == "adagrad" else "sgd",
        "width": 64 if case == "width64" else 128}
  calls_on, w_on = _engine_step(fused=True, **kw)
  calls_off, w_off = _engine_step(fused=False, **kw)
  assert calls_on == calls_off
  assert "interact_bwd_apply" not in calls_on[0]
  for a, b in zip(w_on, w_off):
    np.testing.assert_array_equal(a, b)


def test_eligible_engine_step_moves_the_large_tables_to_the_producer():
  calls_on, w_on = _engine_step(1, [3, 40, 9, 70], fused=True, min_rows=10)
  calls_off, w_off = _engine_step(1, [3, 40, 9, 70], fused=False, min_rows=10)
  assert calls_on[0].pop("interact_bwd_apply") == 1
  assert calls_on == calls_off  # the scatter still runs for the two small tables
  for a, b in zip(w_on, w_off):
    np.testing.assert_allclose(a, b, rtol=1e-6, atol=1e-6)


def test_producer_applied_step_matches_reference():
  """World 1: the producer applies tables >= min_rows (DryOps.interact_bwd_apply), the scatter
  the rest; the result is the unsharded SGD step."""
  sizes = [3, 40, 9, 70]
  sim, des, tables = _dry_engine(1, sizes)
  de, eng = des[0], des[0]._engine
  lb = 8
  rng = np.random.default_rng(1)
  ids = [rng.integers(0, s, lb) for s in sizes]
  grads = rng.standard_normal((lb, len(sizes) * 128)).astype(np.float32)
  gb = torch.from_numpy(grads).bfloat16()

  def rank_fn(_):
    with torch.no_grad():
      de([torch.from_numpy(x) for x in ids], concat=True)
      split = eng.producer_update(128, min_rows=10)
      eng.ops.push_grad(eng.routes_all, len(eng.routes_all_np), gb, eng.act, 1.0, [])
      eng.ops.interact_bwd_apply(gb, *split.interact_args())
      eng.backward_inplace(split)

  dry_run.run_ranks(sim, rank_fn)
  assert eng.ops.calls["scatter_add_bwd"] == 1
  got = de.get_weights()
  g32 = gb.float().numpy()
  for t, s in enumerate(sizes):
    want = tables[t].copy()
    np.add.at(want, ids[t], -0.5 * g32[:, t * 128:(t + 1) * 128])
    np.testing.assert_allclose(got[t], want, rtol=1e-6, atol=1e-6, err_msg=f"table {t}")
