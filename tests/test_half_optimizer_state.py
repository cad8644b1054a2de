"""bf16 optimizer state (``set_optimizer(..., state_dtype=torch.bfloat16)``): the random streams
of the rounding hash, argument checks, the plan interpreter at world sizes 1-8 against an
unsharded model of the documented rule, checkpoints across state dtypes and world sizes, the plan
report and - on an H100 - the fused kernels bit for bit against an fp32-state run, the torch back
end, the trainers and offloaded tables."""
import os
import random
import subprocess
import sys

import numpy as np
import pytest
import torch

from distributed_embeddings_b200.ops import stochastic_rounding as sr
from distributed_embeddings_b200.parallel import dry_run

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BF16_ULP = 2.0**-7  # relative spacing of bf16 values (8 significand bits)


@pytest.fixture(autouse=True)
def _tests_on_path():
  sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
  yield
  sys.path.remove(os.path.dirname(os.path.abspath(__file__)))


def _bits(t):
  return t.detach().cpu().contiguous().view(torch.int16).numpy().view(np.uint16)


def _rn(x):
  """fp32 -> bf16 (round to nearest) -> fp32."""
  return torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).to(torch.bfloat16).float() \
      .numpy()


# ----------------------------------------------------------------------------- random streams
def test_stream_zero_is_the_weight_hash():
  def mix(h):
    h ^= h >> 16
    h = (h * 0x7FEB352D) & 0xFFFFFFFF
    h ^= h >> 15
    h = (h * 0x846CA68B) & 0xFFFFFFFF
    return h ^ (h >> 16)

  def documented(step, key, col, stream):
    h = mix((step + 0x9E3779B9 + stream * 0x632BE5AB) & 0xFFFFFFFF)
    h = mix(h ^ (key & 0xFFFFFFFF))
    h = mix(h ^ (key >> 32))
    return mix(h ^ col)

  rng = np.random.default_rng(0)
  keys = rng.integers(0, 1 << 40, 64)
  cols = rng.integers(0, 512, 64)
  for step in (0, 1, 12, 1 << 23):
    base = sr.random_bits(step, keys, cols)
    assert np.array_equal(base, sr.random_bits(step, keys, cols, sr.STREAM_WEIGHT))
    for stream in (0, 1, 2):
      got = sr.random_bits(step, keys, cols, stream)
      assert [int(x) for x in got] == [documented(step, int(k), int(c), stream)
                                       for k, c in zip(keys, cols)]


def test_streams_draw_uncorrelated_rounding_decisions():
  keys = np.arange(1000, dtype=np.int64)[:, None]
  cols = np.arange(1000, dtype=np.int64)[None, :]
  draws = [sr.random_bits(7, keys, cols, s).reshape(-1) for s in (0, 1, 2)]
  n = draws[0].size
  assert n == 10**6
  # a rounding decision compares u = (r >> 8) * 2^-24 with the position of x between its
  # neighbours; the midpoint decision (u < 1/2) of two streams must be independent
  dec = [(d >> np.uint32(31)).astype(np.float64) for d in draws]
  for i in range(3):
    assert abs(dec[i].mean() - 0.5) < 5 * 0.5 / np.sqrt(n)
    for j in range(i + 1, 3):
      assert not np.array_equal(draws[i], draws[j])
      corr = np.corrcoef(dec[i], dec[j])[0, 1]
      assert abs(corr) < 5 / np.sqrt(n), (i, j, corr)
      u_i = (draws[i] >> np.uint32(8)).astype(np.float64) * 2.0**-24
      u_j = (draws[j] >> np.uint32(8)).astype(np.float64) * 2.0**-24
      assert abs(np.corrcoef(u_i, u_j)[0, 1]) < 5 / np.sqrt(n)


# ----------------------------------------------------------------------------- argument checks
def _cpu_de(**kw):
  from distributed_embeddings_b200.parallel.dist_model_parallel import DistributedEmbedding
  return DistributedEmbedding([{"input_dim": 8, "output_dim": 4}], device="cpu", **kw)


@pytest.mark.parametrize("target", ["set_optimizer", "SparseRowOptimizer"])
def test_invalid_state_dtype_is_rejected(target):
  from distributed_embeddings_b200.parallel.hybrid import SparseRowOptimizer

  def attach(kind, dtype):
    if target == "set_optimizer":
      _cpu_de().set_optimizer(kind, lr=0.1, state_dtype=dtype)
    else:
      SparseRowOptimizer([torch.nn.Parameter(torch.zeros(8, 4))], kind, lr=0.1, state_dtype=dtype)

  with pytest.raises(ValueError, match="65504"):
    attach("adagrad", torch.float16)
  with pytest.raises(ValueError, match="float32 or torch.bfloat16"):
    attach("adam", torch.float64)
  with pytest.raises(ValueError, match="sgd has none"):
    attach("sgd", torch.bfloat16)
  with pytest.raises(ValueError, match="rowwise_adagrad"):
    attach("rowwise_adagrad", torch.bfloat16)
  attach("adagrad", torch.bfloat16)
  attach("adam", torch.bfloat16)
  attach("sgd", torch.float32)


# ----------------------------------------------------------------------------- plan interpreter
def _reference_update(tables, dense, kind, lr):
  """Unsharded model of one step of the documented rule from fresh state: fp32 math, the weight
  update from the unrounded fp32 state.  Returns the fp32 state of every table (slots)."""
  states = []
  for t, g in enumerate(dense):
    touched = np.abs(g).sum(1) != 0
    gt = g[touched]
    if kind == "adagrad":
      acc = np.full_like(tables[t], _rn(np.float32(0.1))[()])  # initial value: round to nearest
      acc[touched] = acc[touched] + gt * gt
      tables[t][touched] -= lr * gt / (np.sqrt(acc[touched]) + np.float32(1e-7))
      states.append([acc])
    else:  # lazy Adam, step 1
      b1, b2 = np.float32(0.9), np.float32(0.999)
      m = np.zeros_like(tables[t])
      v = np.zeros_like(tables[t])
      m[touched] = (np.float32(1) - b1) * gt
      v[touched] = (np.float32(1) - b2) * gt * gt
      mh = m[touched] / (np.float32(1) - b1)
      vh = v[touched] / (np.float32(1) - b2)
      tables[t][touched] -= lr * mh / (np.sqrt(vh) + np.float32(1e-8))
      states.append([m, v])
  return states


def run_state_plan(seed, world, kind, table_dtype, ragged=False):
  """One step of a random plan with bf16 optimizer state against the unsharded model."""
  rng = random.Random(seed)
  nrng = np.random.default_rng(seed)
  n_tables = rng.randint(max(1, world // 2), 2 * world + 2)
  sizes = [(rng.randint(3, 50), rng.choice([4, 8, 12, 16])) for _ in range(n_tables)]
  combiners = [rng.choice(["sum", "mean"]) for _ in sizes]
  imap = list(range(n_tables))
  hots = {t: rng.choice([1, 1, 2, 3]) for t in range(n_tables)}
  kw = {"strategy": rng.choice(["basic", "memory_balanced", "memory_optimized"]),
        "input_table_map": imap, "dp_input": True, "table_dtype": table_dtype}
  if rng.random() < 0.5:
    kw["column_slice_threshold"] = rng.choice([40, 100, 250])
  if world > 1 and rng.random() < 0.5 and not ragged:
    kw["data_parallel_threshold"] = rng.choice([30, 80])
  if world > 1 and rng.random() < 0.5 and not ragged:
    kw["row_slice_threshold"] = rng.choice([300, 500])
  embs = [{"input_dim": r, "output_dim": w, "combiner": c} for (r, w), c in zip(sizes, combiners)]
  try:
    sim, des = dry_run.build_engines(embs, world, **kw)
  except ValueError as e:
    if "Not enough table" in str(e):
      return "infeasible"
    raise
  tables = [torch.from_numpy(nrng.standard_normal(s).astype(np.float32)).to(table_dtype).float()
            .numpy() for s in sizes]
  lr = 0.5
  for de in des:
    de.set_weights(tables)
    de.set_optimizer(kind, lr=lr, state_dtype=torch.bfloat16)
  lb = rng.choice([2, 3, 5])
  B = lb * world
  glob = [nrng.integers(0, sizes[t][0], size=(B, hots[t])) for t in imap]
  rag = [ragged and rng.random() < 0.6 for _ in imap]
  for i, t in enumerate(imap):
    if rag[i]:
      glob[i] = [list(nrng.integers(0, sizes[t][0], size=rng.randint(0, 4))) for _ in range(B)]
  if ragged:
    for de in des:
      de.ragged_capacity = 4

  def as_input(i, lo, hi):
    from distributed_embeddings_b200.ops.ragged import RaggedIds
    if rag[i]:
      rows = glob[i][lo:hi]
      return RaggedIds.from_row_lengths(
          torch.tensor([v for row in rows for v in row], dtype=torch.int64),
          torch.tensor([len(row) for row in rows], dtype=torch.int64))
    return torch.from_numpy(glob[i][lo:hi])

  widths = [sizes[t][1] for t in imap]
  grads = [nrng.standard_normal((B, w)).astype(np.float32) * 0.1 for w in widths]
  dp_tables = set(des[0].strategy.table_groups[0])

  def rank_fn(r):
    de = des[r]
    out = de([as_input(i, r * lb, (r + 1) * lb) for i in range(len(imap))], concat=True)
    gout = torch.from_numpy(np.concatenate([g[r * lb:(r + 1) * lb] for g in grads], 1))
    out.backward(gout)
    for st in de._engine.opt_state.values():
      assert all(s.dtype == torch.bfloat16 for s in st)
    return de._engine.ops.calls.get("segment_update", 0)

  calls = dry_run.run_ranks(sim, rank_fn)
  assert sum(calls) > 0
  from test_dry_run import reference_step  # noqa: E402  pylint: disable=import-outside-toplevel
  _, dense = reference_step([t.copy() for t in tables], imap, glob, combiners, grads, lr, world,
                            "none", {})
  ref = [t.copy() for t in tables]
  ref_state = _reference_update(ref, dense, kind, lr)
  got = des[0].get_weights() if world == 1 else dry_run.run_ranks(
      sim, lambda r: des[r].get_weights(all_ranks=True))[0]
  state = des[0].get_optimizer_state() if world == 1 else dry_run.run_ranks(
      sim, lambda r: des[r].get_optimizer_state(all_ranks=True))[0]
  tol = 2 * BF16_ULP if table_dtype == torch.bfloat16 else 1e-5
  for t in range(n_tables):
    if t in dp_tables:
      np.testing.assert_array_equal(got[t], tables[t])
      assert state["tables"][t] is None
      continue
    np.testing.assert_allclose(got[t], ref[t], rtol=tol, atol=1e-3 if tol > 1e-5 else 1e-5,
                               err_msg=f"table {t} after the {kind} step")
    for k, (s_got, s_ref) in enumerate(zip(state["tables"][t], ref_state[t])):
      assert s_got.dtype == np.float32
      assert np.array_equal(s_got, _rn(s_got)), "state values are bf16 values, upcast exactly"
      # one stochastic rounding of the fp32 state: one of its two bf16 neighbours
      np.testing.assert_allclose(s_got, s_ref, rtol=1.01 * BF16_ULP, atol=1e-30,
                                 err_msg=f"table {t} slot {k}")
  return "ok"


@pytest.mark.parametrize("table_dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("world", [1, 2, 4, 8])
@pytest.mark.parametrize("kind", ["adagrad", "adam"])
def test_random_plans_bf16_state(world, kind, table_dtype):
  n = 3 if world < 8 else 2
  outcomes = [run_state_plan(17000 * world + 31 * s + len(kind), world, kind, table_dtype)
              for s in range(n)]
  assert outcomes.count("ok") >= 1, outcomes


@pytest.mark.parametrize("world", [1, 2, 4])
@pytest.mark.parametrize("kind", ["adagrad", "adam"])
def test_random_plans_bf16_state_ragged(world, kind):
  outcomes = [run_state_plan(19000 * world + s, world, kind, torch.bfloat16, ragged=True)
              for s in range(3)]
  assert outcomes.count("ok") >= 1, outcomes


def test_interpreter_catches_out_of_bounds_at_the_bf16_state_element_size():
  from distributed_embeddings_b200.ops._native import TABLE_DESC
  sim, des = dry_run.build_engines([{"input_dim": 10, "output_dim": 8, "combiner": "sum"}], 1)
  de = des[0]
  de.set_optimizer("adagrad", lr=0.1, state_dtype=torch.bfloat16)
  eng = de._engine
  calls = []
  real = eng.ops.segment_update

  def spy(*args):
    calls.append(args)
    return real(*args)

  eng.ops.segment_update = spy
  de([torch.tensor([[9]])], concat=True).sum().backward()  # the last row: the state's last bytes
  args = list(calls[0])
  assert args[-1] == 1, "the launch carries the bf16 state code"
  # the same launch again: in bounds at 2 bytes per element (4 would end 160 bytes past the
  # buffer); with state0 moved by one bf16 element the last row ends 2 bytes past it
  real(*args)
  t = np.frombuffer(args[1].numpy().tobytes(), dtype=TABLE_DESC).copy()
  t[0]["state0"] += 2
  args[1] = torch.from_numpy(np.frombuffer(t.tobytes(), dtype=np.uint8).copy())
  with pytest.raises(RuntimeError, match="outside any buffer"):
    real(*args)


@pytest.mark.parametrize("table_dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("kind", ["adagrad", "adam"])
def test_dry_updates_leave_bf16_state_bit_identical(kind, table_dtype):
  sim, des = dry_run.build_engines([{"input_dim": 30, "output_dim": 8, "combiner": "sum"},
                                    {"input_dim": 20, "output_dim": 16, "combiner": "mean"}], 1,
                                   table_dtype=table_dtype)
  de = des[0]
  de.set_optimizer(kind, lr=0.5, state_dtype=torch.bfloat16)
  ids = [torch.randint(0, 30, (6, 2)), torch.randint(0, 20, (6, 3))]
  de(ids, concat=True).sum().backward()  # one real step: the state is non-trivial
  before = [w.detach().clone() for w in de.weights]
  state = {m: [s.clone() for s in v] for m, v in de._engine.opt_state.items()}
  step = de._engine.step_count()
  de._engine.dry_updates(True)
  for _ in range(2):
    de(ids, concat=True).sum().backward()
  de._engine.dry_updates(False)
  for a, b in zip(before, de.weights):
    assert torch.equal(a.view(-1).view(torch.int16) if a.dtype != torch.float32 else a,
                       b.detach().view(-1).view(torch.int16) if b.dtype != torch.float32 else b)
  for m, v in state.items():
    for a, b in zip(v, de._engine.opt_state[m]):
      assert b.dtype == torch.bfloat16
      assert torch.equal(a.view(torch.int16), b.view(torch.int16))
  assert de._engine.step_count() == step


# ----------------------------------------------------------------------------- checkpoints
_EMBS = [{"input_dim": 40, "output_dim": 8, "combiner": "sum"},
         {"input_dim": 25, "output_dim": 16, "combiner": "sum"},
         {"input_dim": 33, "output_dim": 4, "combiner": "sum"}]


def _stepped(world, state_dtype, kind="adam", **kw):
  """Engines at ``world`` after one step, so that every slot holds values of its own."""
  sim, des = dry_run.build_engines(_EMBS, world, **kw)
  ids = [torch.randint(0, e["input_dim"], (2 * world, 2), generator=torch.Generator()
                       .manual_seed(i)) for i, e in enumerate(_EMBS)]

  def fn(r):
    des[r].set_optimizer(kind, lr=0.1, state_dtype=state_dtype)
    out = des[r]([x[2 * r:2 * r + 2] for x in ids], concat=True)
    out.backward(torch.ones_like(out) * 0.37)

  dry_run.run_ranks(sim, fn)
  return sim, des


def test_checkpoint_crosses_state_dtype_and_world_size(tmp_path):
  # fp32 state at W=1
  _, des1 = _stepped(1, torch.float32)
  st32 = des1[0].get_optimizer_state()
  assert st32["step"] == 1
  # into a bf16-state run at W=2 (column slices): round to nearest
  sim2, des2 = _stepped(2, torch.bfloat16, column_slice_threshold=200)
  dry_run.run_ranks(sim2, lambda r: des2[r].set_optimizer_state(st32, chunk=24))
  for de in des2:
    for st in de._engine.opt_state.values():
      assert all(s.dtype == torch.bfloat16 for s in st)
  got2 = dry_run.run_ranks(sim2, lambda r: des2[r].get_optimizer_state(all_ranks=True))[0]
  assert got2["step"] == 1
  for a, b in zip(got2["tables"], st32["tables"]):
    for x, y in zip(a, b):
      assert x.dtype == np.float32
      np.testing.assert_array_equal(x, _rn(y))
  # file at W=2, into an fp32-state run at W=3: exact upcast
  dry_run.run_ranks(sim2, lambda r: des2[r].save_optimizer_state(str(tmp_path), chunk=24))
  sim3, des3 = _stepped(3, torch.float32)
  dry_run.run_ranks(sim3, lambda r: des3[r].load_optimizer_state(str(tmp_path), chunk=24))
  got3 = dry_run.run_ranks(sim3, lambda r: des3[r].get_optimizer_state(all_ranks=True))[0]
  for a, b in zip(got3["tables"], got2["tables"]):
    for x, y in zip(a, b):
      np.testing.assert_array_equal(x, y)
  # and back from the fp32 file into bf16 at W=1: nothing changes (the values are bf16 values)
  _, des1b = _stepped(1, torch.bfloat16)
  des1b[0].load_optimizer_state(str(tmp_path))
  for a, b in zip(des1b[0].get_optimizer_state()["tables"], got2["tables"]):
    for x, y in zip(a, b):
      np.testing.assert_array_equal(x, y)


def test_checkpoint_chunks_bound_every_fp32_staging_buffer_of_bf16_state(tmp_path):
  from test_half_tables import _Fp32Sizes  # noqa: E402  pylint: disable=import-outside-toplevel
  _, des = _stepped(1, torch.bfloat16, kind="adagrad")
  de = des[0]
  chunk = 64  # 8 rows of the first table, 1/5 of it
  st = de.get_optimizer_state(all_ranks=True)  # the global fp32 arrays are its result
  with _Fp32Sizes() as mode:
    de.set_optimizer_state(st, chunk=chunk)
    de.save_optimizer_state(str(tmp_path), chunk=chunk)
    de.load_optimizer_state(str(tmp_path), chunk=chunk)
  assert mode.sizes, "no fp32 staging observed"
  assert max(mode.sizes) <= chunk, max(mode.sizes)
  after = de.get_optimizer_state()
  for a, b in zip(after["tables"], st["tables"]):
    np.testing.assert_array_equal(a[0], b[0])


# ----------------------------------------------------------------------------- torch back end
@pytest.mark.parametrize("kind", ["adagrad", "adam"])
def test_sparse_row_optimizer_applies_the_rule(kind):
  from distributed_embeddings_b200.parallel.hybrid import SparseRowOptimizer
  torch.manual_seed(0)
  w0 = torch.randn(50, 12)
  ids = torch.tensor([3, 7, 7, 49, 0])
  vals = torch.randn(5, 12)
  grad = torch.sparse_coo_tensor(ids[None], vals, (50, 12)).coalesce()
  runs = {}
  for sdt in (torch.float32, torch.bfloat16):
    p = torch.nn.Parameter(w0.clone())
    opt = SparseRowOptimizer([p], kind, lr=0.1, state_dtype=sdt)
    if kind == "adagrad":  # a start every dtype stores exactly
      opt.state[0][0].fill_(0.125)
    p.grad = grad.clone()
    opt.step()
    runs[sdt] = (p.detach(), opt.state[0])
  (w32, s32), (w16, s16) = runs[torch.float32], runs[torch.bfloat16]
  torch.testing.assert_close(w16, w32, rtol=1e-6, atol=1e-7)
  rows = torch.unique(ids)
  for k, (a, b) in enumerate(zip(s16, s32)):
    assert a.dtype == torch.bfloat16
    stream = sr.STREAM_STATE0 if k == 0 else sr.STREAM_STATE1
    expect = sr.stochastic_round(b[rows], torch.bfloat16, 1, rows, stream=stream)
    assert np.array_equal(_bits(a[rows]), _bits(expect))
    untouched = torch.ones(50, dtype=torch.bool)
    untouched[rows] = False
    assert torch.equal(a[untouched].float(), b[untouched])


# ----------------------------------------------------------------------------- plan report
def test_plan_report_state_dtype_sizes_the_slots():
  from distributed_embeddings_b200.models.dlrm import mlperf_table_sizes
  tables = ",".join(f"{s}x128" for s in mlperf_table_sizes(20_000_000))

  def gib(*extra):
    out = subprocess.run([sys.executable, "tools/plan_report.py", "--tables", tables, "--world",
                          "1", "--table-dtype", "bf16", "--json"] + list(extra), cwd=ROOT,
                         capture_output=True, text=True, check=True).stdout
    return float(__import__("json").loads(out)["ranks"][0]["hbm_gib"])

  assert gib() == pytest.approx(24.8, abs=0.05)
  assert gib("--optimizer-slots", "1") == pytest.approx(74.4, abs=0.05)
  assert gib("--optimizer-slots", "1", "--state-dtype", "bf16") == pytest.approx(49.6, abs=0.05)
  assert gib("--optimizer-slots", "2") == pytest.approx(124.0, abs=0.05)
  assert gib("--optimizer-slots", "2", "--state-dtype", "bf16") == pytest.approx(74.4, abs=0.05)


# ----------------------------------------------------------------------------- GPU (one H100)
def _cuda():
  return torch.device("cuda", 0)


def _de(embs, table_dtype=torch.float32, **kw):
  from distributed_embeddings_b200.parallel.dist_model_parallel import DistributedEmbedding
  return DistributedEmbedding(embs, device=_cuda(), backend="fused", table_dtype=table_dtype,
                              compute_dtype=torch.float32, **kw)


def _start_state(kind, rows, width, seed):
  """Global optimizer state of one table that bf16 stores exactly (Adam at step 5)."""
  g = np.random.default_rng(seed)
  if kind == "adagrad":
    return {"kind": kind, "step": 0, "tables": [[_rn(g.uniform(0.01, 2.0, (rows, width)))]]}
  m = _rn(g.standard_normal((rows, width)) * 0.01)
  v = _rn(g.uniform(1e-6, 1e-3, (rows, width)))
  return {"kind": kind, "step": 5, "tables": [[m, v]]}


@pytest.mark.gpu
@pytest.mark.parametrize("skewed", [False, True])
@pytest.mark.parametrize("width", [6, 64, 192])  # 1-column kernel, balanced 4-column, per-row 4
@pytest.mark.parametrize("table_dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("kind", ["adagrad", "adam"])
def test_gpu_one_step_is_bit_exact(kind, table_dtype, width, skewed):
  rows, n = 3000, 4096
  g = torch.Generator().manual_seed(width + 7 * skewed)
  w0 = torch.randn(rows, width, generator=g).to(table_dtype).float().numpy()
  if skewed:  # a third of all ids on one row: its segment crosses many chunks of the balanced
    ids = torch.randint(0, rows, (n,), generator=g)
    ids[torch.rand(n, generator=g) < 0.35] = 17
  else:  # duplicates of a uniform draw
    ids = torch.randint(0, rows, (n,), generator=g)
  # gradients on a 2^-12 grid: every fp32 sum of them is exact, so the order in which the
  # balanced kernel's vector reductions add up the segments that cross chunk borders does not
  # change the result, and two runs see the same summed gradient bit for bit
  grad = torch.randint(-200, 200, (n, width), generator=g).float() * 2.0**-12
  start = _start_state(kind, rows, width, width)
  runs = {}
  for sdt in (torch.float32, torch.bfloat16):
    de = _de([{"input_dim": rows, "output_dim": width, "combiner": None}], table_dtype)
    de.set_weights([w0])
    de.set_optimizer(kind, lr=0.05, state_dtype=sdt)
    de([ids.to(_cuda())], concat=True)  # builds the engine
    de.set_optimizer_state(start)
    de([ids.to(_cuda())], concat=True).backward(grad.to(_cuda()))
    torch.cuda.synchronize()
    runs[sdt] = (de.weights[0].detach().cpu(), [s.cpu() for s in de._engine.opt_state[0]],
                 de._engine.step_count())
  (w32, s32, step), (w16, s16, step16) = runs[torch.float32], runs[torch.bfloat16]
  assert step == step16 == start["step"] + 1
  assert np.array_equal(_bits(w16) if table_dtype != torch.float32 else w16.numpy().view(np.uint32),
                        _bits(w32) if table_dtype != torch.float32 else w32.numpy().view(np.uint32))
  keys = np.arange(rows, dtype=np.int64)[:, None]
  cols = np.arange(width, dtype=np.int64)[None, :]
  for k, (a, b) in enumerate(zip(s16, s32)):
    assert a.dtype == torch.bfloat16 and b.dtype == torch.float32
    r = sr.random_bits(step, keys, cols, sr.STREAM_STATE0 if k == 0 else sr.STREAM_STATE1)
    assert np.array_equal(_bits(a), sr.stochastic_round_bits(b.numpy(), torch.bfloat16, r)), k
  touched = torch.unique(ids)
  assert not np.array_equal(_bits(s16[0][touched]), _bits(torch.from_numpy(
      start["tables"][0][0][touched.numpy()]).to(torch.bfloat16)))


@pytest.mark.gpu
def test_gpu_sub_ulp_accumulator_increments_are_unbiased():
  rows, width, steps = 64, 128, 200
  de = _de([{"input_dim": rows, "output_dim": width, "combiner": None}])
  de.set_optimizer("adagrad", lr=0.0, initial_accumulator_value=1.0, state_dtype=torch.bfloat16)
  ids = torch.arange(rows, device=_cuda())
  g = np.float32(np.sqrt(0.1 * BF16_ULP))  # g^2: 0.1 ulp of the accumulator at 1.0
  inc = float(np.float32(g) * np.float32(g))
  for _ in range(steps):
    de([ids], concat=True).backward(torch.full((rows, width), float(g), device=_cuda()))
  torch.cuda.synchronize()
  acc = de._engine.opt_state[0][0].float()
  expect = 1.0 + steps * inc
  se = BF16_ULP * np.sqrt(steps * 0.25) / np.sqrt(rows * width)
  assert abs(float(acc.mean()) - expect) < 5 * se + 1e-6, (float(acc.mean()), expect, se)
  assert float(acc.mean()) > 1.0 + 0.5 * steps * inc, "round to nearest would not move it"


@pytest.mark.gpu
@pytest.mark.parametrize("table_dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("kind", ["adagrad", "adam"])
def test_gpu_fused_matches_torch_backend(kind, table_dtype):
  from distributed_embeddings_b200.parallel.dist_model_parallel import DistributedEmbedding
  from distributed_embeddings_b200.parallel.hybrid import SparseRowOptimizer
  torch.manual_seed(4)
  embs = [{"input_dim": 500, "output_dim": 64, "combiner": "sum"},
          {"input_dim": 300, "output_dim": 16, "combiner": "mean"}]
  w0 = [(np.random.default_rng(i).standard_normal((e["input_dim"], e["output_dim"])) * 0.1)
        .astype(np.float32) for i, e in enumerate(embs)]
  fused = _de(embs, table_dtype)
  fused.set_weights(w0)
  fused.set_optimizer(kind, lr=0.05, state_dtype=torch.bfloat16)
  ref = DistributedEmbedding(embs, device=_cuda(), backend="torch", table_dtype=table_dtype,
                             compute_dtype=torch.float32)
  ref.set_weights(w0)
  opt = SparseRowOptimizer(ref.mp_parameters(), kind, lr=0.05, state_dtype=torch.bfloat16)
  for _ in range(3):
    ids = [torch.randint(0, e["input_dim"], (256, 3), device=_cuda()) for e in embs]
    gout = torch.randn(256, 80, device=_cuda())
    fused(ids, concat=True).backward(gout)
    ref(ids, concat=True).backward(gout)
    opt.step()
  torch.cuda.synchronize()
  for a, b in zip(fused.get_weights(), ref.get_weights()):
    if kind != "adam":
      np.testing.assert_allclose(a, b, rtol=2 * BF16_ULP, atol=2e-3)
      continue
    # as in the fp32-state comparison: near-zero gradient elements may differ in sign between
    # the two back ends' gradient sums; those are rare, all others agree
    bad = ~np.isclose(a, b, rtol=2 * BF16_ULP, atol=2e-3)
    assert bad.mean() < 2e-3, bad.mean()
    assert np.abs(a - b).max() <= 3 * 3 * 0.05


def _dot_batches(sizes, n, b=512, seed=3):
  g = torch.Generator().manual_seed(seed)
  return [(torch.rand(b, 13, generator=g).to(_cuda()),
           torch.stack([torch.randint(0, s, (b,), generator=g, dtype=torch.int32)
                        for s in sizes]).to(_cuda()),
           torch.randint(0, 2, (b,), generator=g).float().to(_cuda())) for _ in range(n)]


def _trainer_pair(interaction):
  """(model, batches) twice: identical models and data, one per state dtype."""
  from distributed_embeddings_b200.models.dlrm import DLRM
  out = []
  for _ in range(2):
    if interaction == "dot":
      sizes = [200 + 13 * i for i in range(26)]
      torch.manual_seed(7)
      model = DLRM(sizes, device=_cuda(), compute_dtype=torch.bfloat16, backend="fused")
      batches = _dot_batches(sizes, 20)
    else:
      from test_dcn import _gpu_batch, _gpu_model  # noqa: E402  pylint: disable=import-outside-toplevel
      hots = [1, 3, 2, 1, 5, 1, 2, 1]
      model = _gpu_model(11, hots)
      sizes = [300 + 11 * i for i in range(8)]
      batches = [_gpu_batch(sizes, hots, 512, 100 + s) for s in range(20)]
    out.append((model, batches))
  return out


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["adagrad", "adam"])
@pytest.mark.parametrize("interaction", ["dot", "dcnv2"])
def test_gpu_dlrm_train_step_with_bf16_state(interaction, kind):
  """DLRMTrainStep (CUDA graph) with bf16 state tracks the fp32-state run: the loss after each of
  20 steps within 2e-2 (the state's stochastic rounding perturbs the embedding update by up to
  one bf16 ulp of the state, a relative 2^-8 of the step size).  The graph warm-up leaves the
  state bit-identical, and evaluation runs."""
  from distributed_embeddings_b200.models.dlrm_fast import DLRMTrainStep
  (m32, batches), (m16, _) = _trainer_pair(interaction)
  lr = 0.05 if kind == "adagrad" else 0.001
  losses = {}
  for sdt, model in ((torch.float32, m32), (torch.bfloat16, m16)):
    t = DLRMTrainStep(model, lr=lr, embedding_optimizer=kind, use_cuda_graph=True,
                      embedding_optimizer_kwargs={"state_dtype": sdt})
    eng = t.engine
    if sdt == torch.bfloat16:
      # the passes before the capture (zero lr, dry updates) on live, non-trivial state
      t.step(*batches[0])
      torch.cuda.synchronize()
      before = {m: [s.clone() for s in v] for m, v in eng.opt_state.items()}
      step = eng.step_count()
      t.load_batch(*batches[1])
      t.lr_t.zero_()
      eng.dry_updates(True)
      for _ in range(2):
        t._step_impl()
      eng.dry_updates(False)
      t.lr_t.fill_(lr)
      torch.cuda.synchronize()
      assert eng.step_count() == step
      for m, v in before.items():
        for a, b in zip(v, eng.opt_state[m]):
          assert b.dtype == torch.bfloat16
          assert torch.equal(a.view(torch.int16), b.view(torch.int16))
      losses[sdt] = [float(t.step(*b)) for b in batches[1:]]
    else:
      losses[sdt] = [float(t.step(*b)) for b in batches]
      losses[sdt] = losses[sdt][1:]
    torch.cuda.synchronize()
    t.evaluate(*batches[0])
    met = t.eval_metrics()
    assert met["samples"] == batches[0][0].shape[0] and 0.0 <= met["auc"] <= 1.0, met
  diff = max(abs(a - b) for a, b in zip(losses[torch.float32], losses[torch.bfloat16]))
  assert diff <= 2e-2, (losses[torch.float32], losses[torch.bfloat16])


@pytest.mark.gpu
def test_gpu_synthetic_train_step_bf16_state_adagrad():
  from distributed_embeddings_b200.models.configs import expand, scaled, synthetic_models_v3
  from distributed_embeddings_b200.models.synthetic import SyntheticModel
  from distributed_embeddings_b200.models.synthetic_fast import SyntheticTrainStep
  cfg = scaled(synthetic_models_v3["tiny"], 2e-4)
  tables, imap, hots = expand(cfg)[:3]
  losses = {}
  for sdt in (torch.float32, torch.bfloat16):
    torch.manual_seed(5)
    m = SyntheticModel(cfg, dp_input=True, device=_cuda(), compute_dtype=torch.bfloat16,
                       backend="fused")
    t = SyntheticTrainStep(m, lr=0.01, embedding_optimizer="adagrad", use_cuda_graph=True,
                           embedding_optimizer_kwargs={"state_dtype": sdt})
    g = torch.Generator().manual_seed(4)
    out = []
    for _ in range(10):
      num = (torch.rand(128, cfg.num_numerical_features, generator=g) * 2).to(_cuda())
      cat = [torch.randint(0, tables[imap[i]][0], (128, h), generator=g).to(_cuda())
             for i, h in enumerate(hots)]
      lab = torch.randint(0, 2, (128, 1), generator=g).float().to(_cuda())
      out.append(float(t.step(num, cat, lab)))
    torch.cuda.synchronize()
    for st in t.engine.opt_state.values():
      assert all(s.dtype == sdt for s in st)
    losses[sdt] = out
  diff = max(abs(a - b) for a, b in zip(losses[torch.float32], losses[torch.bfloat16]))
  assert diff <= 2e-2, losses


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["adagrad", "adam"])
def test_gpu_bf16_state_halves_the_state_bytes(kind):
  embs = [{"input_dim": 100000, "output_dim": 128, "combiner": None},
          {"input_dim": 30000, "output_dim": 64, "combiner": None}]
  ids = [torch.randint(0, e["input_dim"], (256,), device=_cuda()) for e in embs]
  nbytes = {}
  for sdt in (torch.float32, torch.bfloat16):
    de = _de(embs)
    de(ids, concat=True)  # builds the engine
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    de.set_optimizer(kind, lr=0.1, state_dtype=sdt)
    torch.cuda.synchronize()
    alloc = torch.cuda.memory_allocated() - base
    st = [s for v in de._engine.opt_state.values() for s in v]
    assert all(s.dtype == sdt and s.is_cuda for s in st)
    nbytes[sdt] = (sum(s.numel() * s.element_size() for s in st), alloc)
    del de, st
    torch.cuda.empty_cache()
  elems = sum(e["input_dim"] * e["output_dim"] for e in embs) * (2 if kind == "adam" else 1)
  assert nbytes[torch.float32][0] == 4 * elems and nbytes[torch.bfloat16][0] == 2 * elems
  assert nbytes[torch.bfloat16][1] <= nbytes[torch.float32][1] // 2 + (1 << 21)
  assert nbytes[torch.bfloat16][1] >= 2 * elems


@pytest.mark.gpu
def test_gpu_offloaded_table_keeps_pinned_bf16_state():
  embs = [{"input_dim": 700, "output_dim": 32, "combiner": "sum"},
          {"input_dim": 5000, "output_dim": 32, "combiner": "mean"}]
  w0 = [(np.random.default_rng(i).standard_normal((e["input_dim"], e["output_dim"])) * 0.1)
        .astype(np.float32) for i, e in enumerate(embs)]
  runs = []
  for offload in (True, False):
    kw = {"gpu_embedding_size": 700 * 32 + 1} if offload else {}
    de = _de(embs, **kw)
    assert any(getattr(l, "cpu_offloaded", False) for l in de.local_embedding_layers) == offload
    de.set_weights(w0)
    de.set_optimizer("adagrad", lr=0.05, state_dtype=torch.bfloat16)
    g = torch.Generator().manual_seed(1)
    for _ in range(3):
      ids = [torch.randint(0, e["input_dim"], (256, 4), generator=g).to(_cuda()) for e in embs]
      de(ids, concat=True).backward(torch.randn(256, 64, generator=g).to(_cuda()))
    torch.cuda.synchronize()
    eng = de._engine
    for m, layer in enumerate(eng.mp_layers):
      for s in eng.opt_state[m]:
        assert s.dtype == torch.bfloat16
        if getattr(layer, "cpu_offloaded", False):
          assert not s.is_cuda and s.is_pinned()
    runs.append((de.get_weights(), de.get_optimizer_state()))
  (w_off, s_off), (w_hbm, s_hbm) = runs
  for a, b in zip(w_off, w_hbm):
    np.testing.assert_allclose(a, b, rtol=1e-5, atol=1e-6)
  for a, b in zip(s_off["tables"], s_hbm["tables"]):
    np.testing.assert_allclose(a[0], b[0], rtol=1.01 * BF16_ULP, atol=1e-30)


@pytest.mark.gpu
def test_gpu_bf16_state_is_rejected_with_the_offload_cache():
  de = _de([{"input_dim": 700, "output_dim": 32, "combiner": "sum"},
            {"input_dim": 5000, "output_dim": 32, "combiner": "sum"}],
           gpu_embedding_size=700 * 32 + 1, offload_cache_size=4096)
  with pytest.raises(ValueError, match="offload_cache_size"):
    de.set_optimizer("adagrad", lr=0.1, state_dtype=torch.bfloat16)
  de.set_optimizer("adagrad", lr=0.1)
