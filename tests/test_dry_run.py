"""The fused engine's plan -> descriptor logic, exercised for every rank of a plan in one process
on the CPU (parallel/dry_run.py): forward outputs and in-kernel optimizer updates of all ranks
must equal an unsharded numpy model, for random plans at world sizes 1-8."""
import random

import numpy as np
import pytest
import torch

from distributed_embeddings_b200.parallel import dry_run


def _dense_grad(p):
  g = p.grad
  if g is None:
    return torch.zeros_like(p, dtype=torch.float32)
  return (g.to_dense() if g.is_sparse else g).float()


def assemble(des, get=lambda p: p.detach().float()):
  """Global tables from the local shards of all ranks (what get_weights does with collectives);
  ``get`` picks what to read from every local parameter (the weights, or their gradients)."""
  st = des[0].strategy
  n_tables = len(st.global_configs)
  out = [None] * n_tables
  n_dp = len(des[0].dp_layers)
  for j, t in enumerate(st.table_groups[0]):
    out[t] = get(des[0].weights[j]).numpy().copy()
  for gt, t in enumerate(st.table_groups[1]):
    cfg = st.global_configs[t]
    full = np.full((cfg["input_dim"], cfg["output_dim"]), np.nan, dtype=np.float32)
    for r, shards in enumerate(st.shards):
      n_col = len(des[r].local_embedding_layers)
      col_w = des[r].weights[n_dp:n_dp + n_col]
      for s in shards:
        if s.table == gt:
          full[:, s.col_start:s.col_end] = \
              get(col_w[s.local_table])[s.row_offset:s.row_offset + s.rows].numpy()
    assert not np.isnan(full).any()
    out[t] = full
  for gt, t in enumerate(st.table_groups[2]):
    parts = []
    for r in range(len(des)):
      n_col = len(des[r].local_embedding_layers)
      parts.append(get(des[r].weights[n_dp + n_col + gt]).numpy())
    out[t] = np.concatenate(parts, 0)
  return out


def reference_step(tables, imap, glob_ids, combiners, grads, lr, world, kind, state,
                   weight_decay=0.0):
  """Unsharded model: returns outputs [global batch, width] per input and updates ``tables``
  in place with the mean-of-ranks gradient contract (sum over the global batch / world).  The
  optimizers are lazy: a row is touched when at least one id hits it (zero gradients included),
  and only touched rows get the decay and advance their state."""
  outs = []
  dense = [np.zeros_like(t) for t in tables]
  touched_rows = [np.zeros(t.shape[0], dtype=bool) for t in tables]
  for i, t in enumerate(imap):
    ids = glob_ids[i]
    if isinstance(ids, list):  # ragged: one id list per sample
      out = np.zeros((len(ids), tables[t].shape[1]), dtype=np.float32)
      for b, row in enumerate(ids):
        n = len(row)
        if n == 0:
          continue
        scale = 1.0 / n if combiners[t] == "mean" else 1.0
        out[b] = tables[t][row].sum(0) * scale
        np.add.at(dense[t], np.asarray(row, dtype=np.int64), grads[i][b] * scale)
        touched_rows[t][np.asarray(row, dtype=np.int64)] = True
      outs.append(out)
      continue
    # ids outside the table (fed to row-sliced tables) pool to zero and get no gradient
    ok = (ids >= 0) & (ids < tables[t].shape[0])
    rows = tables[t][np.where(ok, ids, 0)] * ok[..., None]  # [B, h, w]
    n = ids.shape[1]
    outs.append(rows.sum(1) / (n if combiners[t] == "mean" else 1))
    g = grads[i] / (n if combiners[t] == "mean" else 1)
    per_id = np.repeat(g, n, axis=0)
    flat_ok = ok.reshape(-1)
    np.add.at(dense[t], ids.reshape(-1)[flat_ok], per_id[flat_ok])
    touched_rows[t][ids.reshape(-1)[flat_ok]] = True
  if kind == "none":
    return outs, [g / world for g in dense]
  for t, g in enumerate(dense):
    touched = touched_rows[t]
    g = g / world
    g[touched] += weight_decay * tables[t][touched]
    if kind == "sgd":
      tables[t][touched] -= lr * g[touched]
    elif kind == "adagrad":
      acc = state.setdefault(t, np.full_like(tables[t], 0.1))
      acc[touched] += g[touched]**2
      tables[t][touched] -= lr * g[touched] / (np.sqrt(acc[touched]) + 1e-7)
    elif kind == "rowwise_adagrad":
      acc = state.setdefault(t, np.full(tables[t].shape[0], 0.1, dtype=np.float32))
      acc[touched] += (g[touched]**2).mean(1)
      tables[t][touched] -= lr * g[touched] / (np.sqrt(acc[touched])[:, None] + 1e-7)
    elif kind == "adam":  # first step of lazy Adam: m/bias1 = g, v/bias2 = g^2 (0/eps = 0)
      tables[t][touched] -= lr * g[touched] / (np.abs(g[touched]) + 1e-8)
  return outs


# Size profile of the random plans.  The default keeps the interpreter fast; other profiles (the
# GPU kernel conformance tests) draw larger shapes from the same generator.
#   rows / widths / hotness / local_batch: (lo, hi) range of table rows, choices for the others;
#   ragged_len: most ids of a ragged sample; power_law: skewed ids (hot rows) instead of uniform;
#   dyadic: tables, gradients and mean weights on a coarse power-of-two grid, so that every fp32
#     sum is exact in any order; out_of_table: one-hot inputs of row-sliced tables also get ids
#     below / above the table (they pool to zero); table_dtype: storage of model-parallel tables.
SMALL_PROFILE = {"rows": (3, 50), "widths": (4, 8, 12, 16), "hotness": (1, 1, 2, 3),
                 "local_batch": (2, 3, 5), "ragged_len": 4, "power_law": False, "dyadic": False,
                 "out_of_table": False, "table_dtype": torch.float32}


def _pow2_floor(n):
  return 1 << (int(n).bit_length() - 1) if n > 0 else 0


def _draw_ids(nrng, rows, size, power_law):
  if power_law:  # P(id < k) = (k / rows)^(1/4): a few very hot rows, a long tail
    return np.minimum((rows * nrng.random(size)**4).astype(np.int64), rows - 1)
  return nrng.integers(0, rows, size=size)


def _draw_tables(nrng, sizes, dyadic):
  tables = [nrng.standard_normal(s).astype(np.float32) for s in sizes]
  if dyadic:  # multiples of 1/16 in [-4, 4]: exact in bf16 / fp16 as well; "+ 0" drops the
    # sign of -0.0 (the kernels keep it through a one-id pool, the interpreter's sum does not)
    tables = [np.clip(np.round(t * 16) / 16, -4, 4).astype(np.float32) + 0 for t in tables]
  return tables


def _draw_grads(nrng, shapes, dyadic):
  if dyadic:  # multiples of 1/64
    return [(np.round(nrng.standard_normal(s) * 8) / 64).astype(np.float32) + 0 for s in shapes]
  return [nrng.standard_normal(s).astype(np.float32) * 0.1 for s in shapes]


def run_plan(seed, world, kind="sgd", dtype=torch.float32, ragged=False, profile=None,
             world_cls=dry_run.DryWorld, weight_decay=0.0):
  prof = dict(SMALL_PROFILE, **(profile or {}))
  rng = random.Random(seed)
  nrng = np.random.default_rng(seed)
  n_tables = rng.randint(max(1, world // 2), 2 * world + 2)
  if kind == "rowwise_adagrad":
    n_tables = max(n_tables, world)  # no automatic column slicing (see below)
  sizes = [(rng.randint(*prof["rows"]), rng.choice(prof["widths"])) for _ in range(n_tables)]
  combiners = [rng.choice(["sum", "mean"]) for _ in sizes]
  imap = list(range(n_tables)) + [rng.randint(0, n_tables - 1) for _ in range(rng.randint(0, 3))]
  rng.shuffle(imap)
  if sorted(set(imap)) != list(range(n_tables)):
    imap = list(range(n_tables))
  hots = {t: rng.choice(prof["hotness"]) for t in range(n_tables)}
  if prof["dyadic"]:  # mean pooling by a power of two
    hots = {t: _pow2_floor(h) if combiners[t] == "mean" else h for t, h in hots.items()}
  kw = {"strategy": rng.choice(["basic", "memory_balanced", "memory_optimized",
                                 "traffic_balanced"]),
        "input_table_map": imap}
  if kw["strategy"] == "traffic_balanced" and not ragged and kind != "rowwise_adagrad":
    kw["input_hotness"] = [hots[t] for t in imap]
  # a column slice keeps its own per-row accumulator (mean of g^2 over *its* columns), so the
  # unsharded reference only applies to row-wise Adagrad when tables are not column sliced
  if rng.random() < 0.5 and kind != "rowwise_adagrad":
    kw["column_slice_threshold"] = rng.choice([40, 100, 250])
  if rng.random() < 0.2:
    kw["gpu_embedding_size"] = rng.choice([150, 400])  # some tables become "host resident"
  dp_input = rng.random() < 0.75
  kw["dp_input"] = dp_input
  plain = ragged or kind == "rowwise_adagrad"  # keep every table in the table-parallel group
  if dp_input and world > 1 and rng.random() < 0.4 and not plain:
    kw["data_parallel_threshold"] = rng.choice([30, 80])
  if dp_input and world > 1 and rng.random() < 0.4 and not plain:
    kw["row_slice_threshold"] = rng.choice([300, 500])
  if prof["table_dtype"] != torch.float32:
    kw["table_dtype"] = prof["table_dtype"]
  embs = [{"input_dim": r, "output_dim": w, "combiner": c} for (r, w), c in zip(sizes, combiners)]
  try:
    sim, des = dry_run.build_engines(embs, world, world_cls, compute_dtype=dtype, **kw)
  except ValueError as e:
    if "Not enough table" in str(e):
      return "infeasible"
    raise
  tables = _draw_tables(nrng, sizes, prof["dyadic"])
  for de in des:
    de.set_weights(tables)
    if kind != "none":
      de.set_optimizer(kind, lr=0.5, weight_decay=weight_decay)
  lb = rng.choice(prof["local_batch"])
  B = lb * world
  glob = [_draw_ids(nrng, sizes[t][0], (B, hots[t]), prof["power_law"]) for t in imap]
  id_dtype = rng.choice([np.int64, np.int32])
  rag = [ragged and rng.random() < 0.6 for _ in imap]
  for i, t in enumerate(imap):
    if rag[i]:
      # 0 ids is legal: the sample pools to zero and contributes no gradient
      lens = [rng.randint(0, prof["ragged_len"]) for _ in range(B)]
      if prof["dyadic"] and combiners[t] == "mean":
        lens = [_pow2_floor(n) for n in lens]
      glob[i] = [list(_draw_ids(nrng, sizes[t][0], n, prof["power_law"])) for n in lens]
  if ragged:
    for de in des:
      de.ragged_capacity = prof["ragged_len"]
  if prof["out_of_table"]:
    row_sliced = set(des[0].strategy.table_groups[2])
    for i, t in enumerate(imap):
      if t in row_sliced and not rag[i] and hots[t] == 1:
        bad = nrng.random(B) < 0.15
        glob[i][bad, 0] = nrng.choice([-7, -1, sizes[t][0], sizes[t][0] + 3], size=int(bad.sum()))

  def as_input(i, lo, hi):
    from distributed_embeddings_b200.ops.ragged import RaggedIds
    if rag[i]:
      rows = glob[i][lo:hi]
      return RaggedIds.from_row_lengths(
          torch.tensor([v for row in rows for v in row], dtype=torch.int64),
          torch.tensor([len(row) for row in rows], dtype=torch.int64))
    return torch.from_numpy(glob[i][lo:hi].astype(id_dtype))

  widths = [sizes[t][1] for t in imap]
  grads = _draw_grads(nrng, [(B, w) for w in widths], prof["dyadic"])
  st = des[0].strategy
  dp_tables = set(st.table_groups[0])

  def rank_fn(r):
    de = des[r]
    sl = slice(r * lb, (r + 1) * lb)
    if dp_input:
      inputs = [as_input(i, r * lb, (r + 1) * lb) for i in range(len(imap))]
    else:
      inputs = [as_input(i, 0, B) for i in st.input_ids_list[r]]
    out = de(inputs, concat=True)
    assert de._engine.ops.calls.get("lookup_fwd", 0) > 0, "the interpreter did not run"
    gout = torch.from_numpy(np.concatenate([g[sl] for g in grads], 1)).to(out.dtype)
    out.backward(gout)
    dp_grads = [p.grad for layer in de.dp_layers for p in layer.parameters()]
    return out.detach().float().numpy(), dp_grads

  results = dry_run.run_ranks(sim, rank_fn)
  ref_tables = [t.copy() for t in tables]
  # replicated tables are not updated by the engine (their dense gradient goes to the all-reduce)
  ref_outs = reference_step(ref_tables, imap, glob, combiners, grads, 0.5, world, kind, {},
                            weight_decay)
  ref_grads = None
  if kind == "none":
    ref_outs, ref_grads = ref_outs
  tol = 1e-4 if dtype == torch.float32 else 3e-2
  # 16-bit tables: one stochastic rounding per element, within one ulp of the fp32 result
  half = {torch.bfloat16: 2.0**-7, torch.float16: 2.0**-10}.get(prof["table_dtype"])
  tab_rtol, tab_atol = (2 * half, 1e-3) if half else (10 * tol, 10 * tol)
  for r, (out, dp_grads) in enumerate(results):
    exp = np.concatenate([o[r * lb:(r + 1) * lb] for o in ref_outs], 1)
    np.testing.assert_allclose(out, exp, rtol=tol, atol=tol, err_msg=f"forward, rank {r}")
  if ref_grads is not None:
    # no fused optimizer: the engine returns deduplicated sparse gradients (reference semantics)
    got_g = assemble(des, _dense_grad)
    for t in range(n_tables):
      if t not in dp_tables:
        np.testing.assert_allclose(got_g[t], ref_grads[t], rtol=tab_rtol, atol=tab_atol,
                                   err_msg=f"sparse gradient of table {t}")
  got = assemble(des)
  for t in range(n_tables):
    if t in dp_tables:
      np.testing.assert_allclose(got[t], tables[t], rtol=0, atol=0)  # untouched by the engine
      continue
    np.testing.assert_allclose(got[t], ref_tables[t], rtol=tab_rtol, atol=tab_atol,
                               err_msg=f"table {t} after the {kind} step")
  # dense gradients of replicated tables: local-batch contribution of each rank
  for j, t in enumerate(st.table_groups[0]):
    for r, (_, dp_grads) in enumerate(results):
      exp = np.zeros_like(tables[t])
      for i, ti in enumerate(imap):
        if ti == t:
          assert not rag[i]
          ids = glob[i][r * lb:(r + 1) * lb]
          n = ids.shape[1]
          g = grads[i][r * lb:(r + 1) * lb] / (n if combiners[t] == "mean" else 1)
          np.add.at(exp, ids.reshape(-1), np.repeat(g, n, axis=0))
      np.testing.assert_allclose(dp_grads[j].numpy(), exp, rtol=10 * tol, atol=10 * tol)
  return "ok"


@pytest.mark.parametrize("world", [1, 2, 3, 4, 8])
def test_random_plans_sgd(world):
  n = 8 if world < 8 else 4
  outcomes = [run_plan(1000 * world + s, world, "sgd") for s in range(n)]
  assert outcomes.count("ok") >= n // 2 + 1, outcomes
  # SGD with weight decay leaves the atomic scatter for the sorted update
  outcomes = [run_plan(1000 * world + s, world, "sgd", weight_decay=0.25) for s in range(2)]
  assert outcomes.count("ok") >= 1, outcomes


@pytest.mark.parametrize("world", [1, 2, 4])
@pytest.mark.parametrize("kind", ["adagrad", "rowwise_adagrad", "adam"])
def test_random_plans_stateful_optimizers(world, kind):
  outcomes = [run_plan(5000 * world + s, world, kind) for s in range(5)]
  assert outcomes.count("ok") >= 3, outcomes
  # weight decay (dyadic, so exact on the dyadic grid of the GPU conformance profile as well)
  outcomes = [run_plan(5000 * world + s, world, kind, weight_decay=0.25) for s in range(5)]
  assert outcomes.count("ok") >= 3, outcomes


@pytest.mark.parametrize("world", [1, 2, 4, 8])
def test_random_plans_sparse_gradients(world):
  n = 8 if world < 8 else 3
  outcomes = [run_plan(3000 * world + s, world, "none") for s in range(n)]
  assert outcomes.count("ok") >= n // 2 + 1, outcomes


@pytest.mark.parametrize("world", [1, 2, 4])
@pytest.mark.parametrize("kind", ["sgd", "adagrad"])
def test_random_plans_ragged(world, kind):
  outcomes = [run_plan(7000 * world + s, world, kind, ragged=True) for s in range(5)]
  assert outcomes.count("ok") >= 3, outcomes


def test_bf16_activations_world4():
  outcomes = [run_plan(9000 + s, 4, "sgd", torch.bfloat16) for s in range(6)]
  assert outcomes.count("ok") >= 4, outcomes


def test_out_of_bounds_descriptor_is_caught():
  """A corrupted descriptor must trip the interpreter's address check, not pass silently."""
  embs = [{"input_dim": 10, "output_dim": 8, "combiner": "sum"} for _ in range(2)]
  sim, des = dry_run.build_engines(embs, 1)
  de = des[0]
  de.set_optimizer("sgd", lr=0.1)
  ids = [torch.randint(0, 10, (4, 2)) for _ in range(2)]
  de(ids, concat=True)
  eng = de._engine
  eng.cdesc_np[0]["row_base"] = 1000  # beyond the fused table
  eng._upload()
  with pytest.raises((RuntimeError, IndexError)):
    eng._run_forward()


def test_sparse_gradient_values_have_canonical_strides():
  """One unique row of a table narrower than the widest one: the emitted values must not be a
  padded view (PyTorch's sparse -> dense kernels address the destination with the values' row
  stride; found by the fuzzer as an intermittent heap corruption at world size 8)."""
  embs = [{"input_dim": 6, "output_dim": 4, "combiner": "sum"},
          {"input_dim": 9, "output_dim": 8, "combiner": "sum"}]
  _, des = dry_run.build_engines(embs, 1)
  de = des[0]
  ids = [torch.full((5, 2), 3, dtype=torch.int64), torch.randint(0, 9, (5, 2))]
  out = de(ids, concat=True)
  out.backward(torch.ones_like(out))
  for p in de.parameters():
    g = p.grad
    assert g.is_sparse
    v = g._values()
    assert v.stride() == (v.shape[1], 1), (tuple(v.shape), v.stride())
    dense = g.to_dense()
    assert torch.isfinite(dense).all()
  narrow = [p for p in de.parameters() if p.shape[1] == 4][0].grad.to_dense()
  assert narrow[3].tolist() == [10.0] * 4 and float(narrow.abs().sum()) == 40.0


def _run_steps(seed, world, kind, n_steps=3):
  """Several steps on one plan, with a different local batch size on the second step (the
  engines rebuild their buffers): optimizer state, row-slice partial buffers and id staging must
  carry over / be reset correctly from step to step."""
  rng = random.Random(seed)
  nrng = np.random.default_rng(seed)
  n_tables = rng.randint(world, 2 * world + 1)
  sizes = [(rng.randint(5, 40), rng.choice([4, 8, 16])) for _ in range(n_tables)]
  combiners = [rng.choice(["sum", "mean"]) for _ in sizes]
  imap = list(range(n_tables)) + [rng.randint(0, n_tables - 1) for _ in range(2)]
  hots = [rng.choice([1, 2, 3]) for _ in imap]
  kw = {"strategy": rng.choice(["basic", "memory_balanced", "memory_optimized",
                                 "traffic_balanced"]),
        "input_table_map": imap, "input_hotness": hots}
  if rng.random() < 0.5:
    kw["column_slice_threshold"] = rng.choice([60, 150])
  if world > 1 and rng.random() < 0.5:
    kw["row_slice_threshold"] = 400
  embs = [{"input_dim": r, "output_dim": w, "combiner": c} for (r, w), c in zip(sizes, combiners)]
  try:
    sim, des = dry_run.build_engines(embs, world, **kw)
  except ValueError as e:
    if "Not enough table" in str(e):
      return "infeasible"
    raise
  tables = [nrng.standard_normal(s).astype(np.float32) for s in sizes]
  lr = 0.3
  for de in des:
    de.set_weights(tables)
    de.set_optimizer(kind, lr=lr)
  ref = [t.copy() for t in tables]
  state = {}
  for step in range(n_steps):
    lb = [3, 5, 3, 2][step % 4]
    B = lb * world
    glob = [nrng.integers(0, sizes[t][0], size=(B, h)) for t, h in zip(imap, hots)]
    grads = [nrng.standard_normal((B, sizes[t][1])).astype(np.float32) * 0.1 for t in imap]

    def rank_fn(r, lb=lb, glob=glob, grads=grads):
      inputs = [torch.from_numpy(g[r * lb:(r + 1) * lb]) for g in glob]
      out = des[r](inputs, concat=True)
      out.backward(torch.from_numpy(np.concatenate([g[r * lb:(r + 1) * lb] for g in grads], 1)))
      return out.detach().numpy()

    outs = dry_run.run_ranks(sim, rank_fn)
    # reference: forward on the current tables, then the update
    dense = [np.zeros_like(t) for t in ref]
    exp_cols = []
    for i, t in enumerate(imap):
      n = glob[i].shape[1]
      scale = 1.0 / n if combiners[t] == "mean" else 1.0
      exp_cols.append(ref[t][glob[i]].sum(1) * scale)
      np.add.at(dense[t], glob[i].reshape(-1), np.repeat(grads[i] * scale, n, axis=0))
    exp = np.concatenate(exp_cols, 1)
    for r in range(world):
      np.testing.assert_allclose(outs[r], exp[r * lb:(r + 1) * lb], rtol=2e-4, atol=2e-4,
                                 err_msg=f"step {step} forward rank {r}")
    t_step = step + 1
    for t, g in enumerate(dense):
      g = g / world
      # lazy: the rows an id hit, whatever their gradient (Adam decays the moments of a row hit
      # by zero gradients)
      touched = np.zeros(ref[t].shape[0], dtype=bool)
      for i, ti in enumerate(imap):
        if ti == t:
          touched[glob[i].reshape(-1)] = True
      if kind == "sgd":
        ref[t] -= lr * g
      elif kind == "adagrad":
        acc = state.setdefault(t, np.full_like(ref[t], 0.1))
        acc[touched] += g[touched]**2
        ref[t][touched] -= lr * g[touched] / (np.sqrt(acc[touched]) + 1e-7)
      elif kind == "adam":
        m, v = state.setdefault(t, (np.zeros_like(ref[t]), np.zeros_like(ref[t])))
        m[touched] = 0.9 * m[touched] + 0.1 * g[touched]
        v[touched] = 0.999 * v[touched] + 0.001 * g[touched]**2
        mh = m[touched] / (1 - 0.9**t_step)
        vh = v[touched] / (1 - 0.999**t_step)
        ref[t][touched] -= lr * mh / (np.sqrt(vh) + 1e-8)
  got = assemble(des)
  for t in range(n_tables):
    np.testing.assert_allclose(got[t], ref[t], rtol=2e-3, atol=2e-3,
                               err_msg=f"table {t} after {n_steps} {kind} steps")
  return "ok"


@pytest.mark.parametrize("world", [2, 8])
@pytest.mark.parametrize("kind", ["sgd", "adagrad", "adam"])
def test_multi_step_with_batch_size_change(world, kind):
  n = 3 if world < 8 else 1
  outcomes = [_run_steps(400 * world + s, world, kind, n_steps=3 if world < 8 else 2)
              for s in range(n)]
  assert outcomes.count("ok") >= max(1, n - 1), outcomes


@pytest.mark.parametrize("world,streamed", [(1, False), (2, False), (4, False), (2, True),
                                            (3, True), (4, True), (5, True), (8, True)])
def test_backward_inplace_with_replicated_tables(world, streamed):
  """The hand-scheduled step's path: gradient pushed by a fused producer, replicated tables
  accumulate their local-batch dense gradient into persistent targets (later all-reduced with
  the dense parameters), model-parallel tables are updated in place.  ``streamed``: the
  producer stages the pieces of remote owners locally (``routes_stage``) and the copy kernel of
  the streamed push forwards them (the default of the DLRM step from 4 GPUs)."""
  rng = np.random.default_rng(77 + world)
  sizes = [(6, 8), (40, 8), (9, 16), (300, 16), (25, 8), (500, 8)]
  embs = [{"input_dim": r, "output_dim": w, "combiner": None} for r, w in sizes]
  kw = {"strategy": "memory_balanced", "data_parallel_threshold": 150} if world > 1 else {}
  sim, des = dry_run.build_engines(embs, world, **kw)
  tables = [rng.standard_normal(s).astype(np.float32) for s in sizes]
  lr, lb = 0.25, 6
  B = lb * world
  for de in des:
    de.set_weights(tables)
    de.set_optimizer("sgd", lr=lr)
  dp_tables = des[0].strategy.table_groups[0]
  assert (len(dp_tables) > 0) == (world > 1)
  targets = [[torch.zeros(sizes[t]) for t in dp_tables] for _ in range(world)]
  chunk = 4  # two chunks per local batch, the second one partial
  for r, de in enumerate(des):
    de._engine.set_dp_grad_targets(targets[r])
    if streamed:
      de._engine.enable_streamed_push(chunk)
  ids = [rng.integers(0, r_, size=B) for r_, _ in sizes]
  grads = [rng.standard_normal((B, w)).astype(np.float32) * 0.1 for _, w in sizes]

  def rank_fn(r):
    de, eng = des[r], des[r]._engine
    sl = slice(r * lb, (r + 1) * lb)
    with torch.no_grad():
      out = de([torch.from_numpy(i[sl]) for i in ids], concat=True)
      exp = np.concatenate([tables[t][ids[t][sl]] for t in range(len(sizes))], 1)
      np.testing.assert_allclose(out.numpy(), exp, rtol=1e-5, atol=1e-5)
      # what the fused producer (the DLRM interaction backward) does: every piece of the local
      # gradient rows goes through `routes_all` to its owner (replicated inputs: to the local
      # requester-layout buffer), "gradient ready" is signalled from the same launch
      g = torch.from_numpy(np.concatenate([g[sl] for g in grads], 1))
      if streamed:
        assert eng.streamed_push and len(eng.push_plan[0]) == world - 1
        eng.push_counters.zero_()
        eng.ops.push_grad(eng.routes_stage, len(eng.routes_stage_np), g, eng.act, 1.0, [])
        for c in range(eng.push_counters.numel()):  # the producer's per-chunk progress
          eng.push_counters[c] = min(chunk, lb - c * chunk)
        eng.launch_streamed_push()
      else:
        eng.ops.push_grad(eng.routes_all, len(eng.routes_all_np), g, eng.act, 1.0,
                          eng.sync_grad_signal())
      eng.backward_inplace()

  dry_run.run_ranks(sim, rank_fn)
  got = assemble(des)
  for t, (rows, _) in enumerate(sizes):
    dense = np.zeros_like(tables[t])
    np.add.at(dense, ids[t], grads[t])
    if t in dp_tables:
      np.testing.assert_array_equal(got[t], tables[t])  # applied later, with the dense params
      j = dp_tables.index(t)
      for r in range(world):
        loc = np.zeros_like(tables[t])
        np.add.at(loc, ids[t][r * lb:(r + 1) * lb], grads[t][r * lb:(r + 1) * lb])
        np.testing.assert_allclose(targets[r][j].numpy(), loc, rtol=1e-5, atol=1e-6)
    else:
      np.testing.assert_allclose(got[t], tables[t] - lr * dense / world, rtol=1e-5, atol=1e-5)
  with pytest.raises(ValueError):
    des[0]._engine.set_dp_grad_targets([torch.zeros(1)] * (len(dp_tables) + 1))


@pytest.mark.parametrize("kind", ["adagrad", "adam"])
def test_optimizer_state_checkpoint_resume(kind):
  """get_weights + get_optimizer_state after step 1, loaded into freshly built engines, then
  step 2 == two uninterrupted steps (same plan on both sides; world size 2)."""
  rng = np.random.default_rng(5)
  sizes = [(30, 8), (12, 16), (50, 8), (21, 16)]
  embs = [{"input_dim": r, "output_dim": w, "combiner": "sum"} for r, w in sizes]
  world, lb = 2, 4
  tables = [rng.standard_normal(s).astype(np.float32) for s in sizes]
  batches = [([rng.integers(0, r, size=(lb * world, 2)) for r, _ in sizes],
              [rng.standard_normal((lb * world, w)).astype(np.float32) * 0.1 for _, w in sizes])
             for _ in range(2)]

  def make(weights):
    sim, des = dry_run.build_engines(embs, world, strategy="memory_balanced",
                                     column_slice_threshold=200)
    for de in des:
      de.set_weights(weights)
      de.set_optimizer(kind, lr=0.3)
    return sim, des

  def step(sim, des, batch):
    ids, grads = batch

    def fn(r):
      sl = slice(r * lb, (r + 1) * lb)
      out = des[r]([torch.from_numpy(i[sl]) for i in ids], concat=True)
      out.backward(torch.from_numpy(np.concatenate([g[sl] for g in grads], 1)))

    dry_run.run_ranks(sim, fn)

  sim_a, des_a = make(tables)
  step(sim_a, des_a, batches[0])
  step(sim_a, des_a, batches[1])
  straight = assemble(des_a)

  sim_b, des_b = make(tables)
  step(sim_b, des_b, batches[0])
  saved_w = assemble(des_b)
  saved_s = [de._engine.optimizer_state_dict() for de in des_b]
  assert all(s["state"] for s in saved_s) and saved_s[0]["step"] == 1
  sim_c, des_c = make(saved_w)
  for de, st in zip(des_c, saved_s):
    de.set_optimizer_state(st)  # per-rank (sharding dependent) format
  step(sim_c, des_c, batches[1])
  resumed = assemble(des_c)
  for a, b in zip(straight, resumed):
    np.testing.assert_allclose(b, a, rtol=1e-5, atol=1e-6)
  # and without the optimizer state the result differs (the test is sensitive to it)
  sim_d, des_d = make(saved_w)
  step(sim_d, des_d, batches[1])
  assert any(not np.allclose(a, b, rtol=1e-5, atol=1e-6) for a, b in zip(straight, assemble(des_d)))


@pytest.mark.parametrize("kind", ["adagrad", "adam", "rowwise_adagrad"])
def test_optimizer_state_resharding(kind, tmp_path):
  """The global optimizer-state layout is sharding independent: one step on 4 column-sliced
  ranks, state + weights loaded into a 2-rank plan (different slicing, a row-sliced table), a
  second step there == two uninterrupted steps on the 2-rank plan."""
  rng = np.random.default_rng(11)
  sizes = [(30, 8), (12, 16), (50, 8), (21, 16), (64, 8)]
  embs = [{"input_dim": r, "output_dim": w, "combiner": "sum"} for r, w in sizes]
  gb = 8
  tables = [rng.standard_normal(s).astype(np.float32) for s in sizes]
  batches = [([rng.integers(0, r, size=(gb, 2)) for r, _ in sizes],
              [rng.standard_normal((gb, w)).astype(np.float32) * 0.1 for _, w in sizes])
             for _ in range(2)]

  def make(world, weights, **kw):
    sim, des = dry_run.build_engines(embs, world, strategy="memory_balanced", **kw)
    for de in des:
      de.set_weights(weights)
      de.set_optimizer(kind, lr=0.3)
    return sim, des

  def step(sim, des, batch):
    ids, grads = batch
    world = len(des)
    lb = gb // world

    def fn(r):
      sl = slice(r * lb, (r + 1) * lb)
      out = des[r]([torch.from_numpy(i[sl]) for i in ids], concat=True)
      out.backward(torch.from_numpy(np.concatenate([g[sl] for g in grads], 1)) * world / 2)

    dry_run.run_ranks(sim, fn)

  def gather(sim, des, fn):
    return dry_run.run_ranks(sim, lambda r: fn(des[r]))[0]

  kw2 = {"column_slice_threshold": 300, "row_slice_threshold": 500}
  # row-wise state of a column-sliced table is per slice: keep tables whole in that case
  kw4 = {"column_slice_threshold": 100 if kind != "rowwise_adagrad" else None}
  if kind == "rowwise_adagrad":
    kw2 = {"row_slice_threshold": 500}
  sim_a, des_a = make(2, tables, **kw2)
  step(sim_a, des_a, batches[0])
  step(sim_a, des_a, batches[1])
  straight = gather(sim_a, des_a, lambda de: de.get_weights())

  sim_b, des_b = make(4, tables, **kw4)
  step(sim_b, des_b, batches[0])
  saved_w = gather(sim_b, des_b, lambda de: de.get_weights())
  saved_s = gather(sim_b, des_b, lambda de: de.get_optimizer_state())
  assert saved_s["step"] == 1 and saved_s["kind"] == kind
  for t, (rows, w) in enumerate(sizes):
    want = (rows, 1) if kind == "rowwise_adagrad" else (rows, w)
    assert all(a.shape == want for a in saved_s["tables"][t])
  sim_c, des_c = make(2, saved_w, **kw2)

  def load(r):
    des_c[r]._engine.prepare(gb // 2, [2] * len(sizes))
    des_c[r].set_optimizer_state(saved_s)
  dry_run.run_ranks(sim_c, load)
  step(sim_c, des_c, batches[1])
  resumed = gather(sim_c, des_c, lambda de: de.get_weights())
  for a, b in zip(straight, resumed):
    np.testing.assert_allclose(b, a, rtol=2e-5, atol=2e-6)

  # the same through files: every rank of the 4-rank job writes its slices (weights and state),
  # the 2-rank job maps the files and reads its own
  ckpt = str(tmp_path / "ckpt")

  def save(r):
    des_b[r].save_weights(ckpt, chunk=64)
    return des_b[r].save_optimizer_state(ckpt, chunk=64)
  metas = dry_run.run_ranks(sim_b, save)
  assert all(m == metas[0] and m.endswith("optimizer.json") for m in metas)
  for t in range(len(sizes)):
    for k, arr in enumerate(saved_s["tables"][t]):
      np.testing.assert_allclose(np.load(f"{ckpt}/opt_{t}_slot{k}.npy"), arr, rtol=1e-6, atol=0)
  sim_d, des_d = make(2, tables, **kw2)

  def load_files(r):
    des_d[r]._engine.prepare(gb // 2, [2] * len(sizes))
    des_d[r].load_weights(ckpt)
    des_d[r].load_optimizer_state(ckpt)
  dry_run.run_ranks(sim_d, load_files)
  assert des_d[0]._engine.step_count() == 1
  step(sim_d, des_d, batches[1])
  resumed_files = gather(sim_d, des_d, lambda de: de.get_weights())
  for a, b in zip(straight, resumed_files):
    np.testing.assert_allclose(b, a, rtol=2e-5, atol=2e-6)


def test_second_forward_before_backward_takes_the_torch_path():
  """Two forwards of one layer before any backward (two-tower models, gradient accumulation):
  the first owns the engine's buffers, the second runs on the torch back end; neither output nor
  gradient of the first call is disturbed (the reference layer can be called any number of
  times)."""
  rng = np.random.default_rng(11)
  sizes = [(30, 8), (12, 16), (50, 8)]
  embs = [{"input_dim": r, "output_dim": w, "combiner": None} for r, w in sizes]
  sim, des = dry_run.build_engines(embs, 1)
  de = des[0]
  tables = [rng.standard_normal(s).astype(np.float32) for s in sizes]
  de.set_weights(tables)
  b = 5
  ids1 = [rng.integers(0, r, size=b) for r, _ in sizes]
  ids2 = [rng.integers(0, r, size=b) for r, _ in sizes]
  g1 = rng.standard_normal((b, sum(w for _, w in sizes))).astype(np.float32)
  g2 = rng.standard_normal((b, sum(w for _, w in sizes))).astype(np.float32)
  seen = {}

  def rank_fn(r):
    out1 = de([torch.from_numpy(i) for i in ids1], concat=True)
    assert de._engine.busy()
    calls = dict(de._engine.ops.calls)
    out2 = de([torch.from_numpy(i) for i in ids2], concat=True)
    assert dict(de._engine.ops.calls) == calls, "the second forward must not touch the engine"
    exp1 = np.concatenate([tables[t][ids1[t]] for t in range(len(sizes))], 1)
    exp2 = np.concatenate([tables[t][ids2[t]] for t in range(len(sizes))], 1)
    np.testing.assert_allclose(out1.detach().numpy(), exp1, rtol=1e-6, atol=1e-6)
    np.testing.assert_allclose(out2.detach().numpy(), exp2, rtol=1e-6, atol=1e-6)
    (out1 * torch.from_numpy(g1)).sum().backward()
    assert not de._engine.busy()
    seen["first"] = assemble(des, _dense_grad)
    for p in de.parameters():
      p.grad = None
    (out2 * torch.from_numpy(g2)).sum().backward()
    seen["second"] = assemble(des, _dense_grad)
    out3 = de([torch.from_numpy(i) for i in ids2], concat=True)  # the engine is free again
    assert dict(de._engine.ops.calls) != calls
    np.testing.assert_allclose(out3.detach().numpy(), exp2, rtol=1e-6, atol=1e-6)

  dry_run.run_ranks(sim, rank_fn)
  col = 0
  for t, (rows, w) in enumerate(sizes):
    for ids, g, key in ((ids1, g1, "first"), (ids2, g2, "second")):
      dense = np.zeros((rows, w), dtype=np.float32)
      np.add.at(dense, ids[t], g[:, col:col + w])
      np.testing.assert_allclose(seen[key][t], dense, rtol=1e-5, atol=1e-6,
                                 err_msg=f"{key} backward, table {t}")
    col += w


@pytest.mark.parametrize("world", [1, 2, 3])
def test_output_row_stride(world):
  """``set_out_row_stride``: the lookups of every owner write into a wider requester matrix (the
  synthetic step's MLP input: embeddings first, other features behind them); the columns behind
  the embeddings are never touched and the gradient push reads the same strided layout."""
  rng = np.random.default_rng(21 + world)
  sizes = [(30, 8), (12, 16), (50, 8), (9, 8)]
  embs = [{"input_dim": r, "output_dim": w, "combiner": "sum"} for r, w in sizes]
  sim, des = dry_run.build_engines(embs, world, strategy="memory_balanced")
  tables = [rng.standard_normal(s).astype(np.float32) for s in sizes]
  lr, lb, hot = 0.5, 4, 2
  B = lb * world
  tw = sum(w for _, w in sizes)
  stride = tw + 24
  for de in des:
    de.set_weights(tables)
    de.set_optimizer("sgd", lr=lr)
    de._engine.set_out_row_stride(stride)
  with pytest.raises(ValueError):
    des[0]._engine.set_out_row_stride(tw + 4)  # not a multiple of 8
  with pytest.raises(ValueError):
    des[0]._engine.set_out_row_stride(tw - 8)  # narrower than the embeddings
  ids = [rng.integers(0, r, size=(B, hot)) for r, _ in sizes]
  grads = rng.standard_normal((B, stride)).astype(np.float32) * 0.1

  def rank_fn(r):
    de, eng = des[r], des[r]._engine
    sl = slice(r * lb, (r + 1) * lb)
    with torch.no_grad():
      eng.stage([torch.from_numpy(i[sl]) for i in ids])
      eng.out_full[:, tw:] = 7.0  # the consumer's other features
      eng.launch_forward()
      eng.wait_output()
      assert eng.out_full.shape == (lb, stride) and eng.out.shape == (lb, tw)
      exp = np.concatenate([tables[t][ids[t][sl]].sum(1) for t in range(len(sizes))], 1)
      np.testing.assert_allclose(eng.out.float().numpy(), exp, rtol=1e-5, atol=1e-5)
      assert bool((eng.out_full[:, tw:] == 7.0).all())
      # gradient of the whole strided matrix (a first-layer dgrad): only the embedding columns
      # are routed to the owners
      g = torch.from_numpy(grads[sl])
      eng.ops.push_grad(eng.routes_all, len(eng.routes_all_np), g, eng.act, 1.0,
                        eng.sync_grad_signal())
      eng.backward_inplace()

  dry_run.run_ranks(sim, rank_fn)
  got = assemble(des)
  col = 0
  for t, (rows, w) in enumerate(sizes):
    dense = np.zeros((rows, w), dtype=np.float32)
    np.add.at(dense, ids[t].reshape(-1), np.repeat(grads[:, col:col + w], hot, axis=0))
    np.testing.assert_allclose(got[t], tables[t] - lr * dense / world, rtol=1e-5, atol=1e-5,
                               err_msg=f"table {t}")
    col += w


def run_inplace_plan(seed, world, streamed, profile=None, world_cls=dry_run.DryWorld):
  """Random plan for the hand-scheduled steps' backward (``routes_all`` / ``routes_stage`` +
  ``backward_inplace``): column slices, shared tables, multi-hot sum / mean pooling, replicated
  tables, one SGD step against the unsharded model.  ``profile``: see ``SMALL_PROFILE`` (rows,
  widths, hotness, dyadic)."""
  prof = {**SMALL_PROFILE, "rows": (3, 60), "local_batch": (3, 5, 8), **(profile or {})}
  rng = random.Random(seed)
  nrng = np.random.default_rng(seed)
  n_tables = rng.randint(max(2, world // 2), 2 * world + 2)
  sizes = [(rng.randint(*prof["rows"]), rng.choice(prof["widths"])) for _ in range(n_tables)]
  hot = rng.choice(prof["hotness"])
  if prof["dyadic"]:
    hot = _pow2_floor(hot)
  combiners = [rng.choice(["sum", "mean"]) if hot > 1 else None for _ in sizes]
  imap = list(range(n_tables)) + [rng.randint(0, n_tables - 1) for _ in range(rng.randint(0, 2))]
  kw = {"strategy": rng.choice(["basic", "memory_balanced", "memory_optimized"]),
        "input_table_map": imap}
  if rng.random() < 0.5:
    kw["column_slice_threshold"] = rng.choice([60, 150, 300])
  if world > 1 and rng.random() < 0.6:
    kw["data_parallel_threshold"] = rng.choice([40, 100])
  embs = [{"input_dim": r, "output_dim": w, "combiner": c} for (r, w), c in zip(sizes, combiners)]
  try:
    sim, des = dry_run.build_engines(embs, world, world_cls, **kw)
  except ValueError as e:
    if "Not enough table" in str(e):
      return "infeasible"
    raise
  tables = _draw_tables(nrng, sizes, prof["dyadic"])
  lr = 0.5
  lb = rng.choice(prof["local_batch"])
  chunk = rng.choice([2, 3, 8])
  B = lb * world
  st = des[0].strategy
  dp_tables = list(st.table_groups[0])
  targets = [[torch.zeros(sizes[t]) for t in dp_tables] for _ in range(world)]
  for r, de in enumerate(des):
    de.set_weights(tables)
    de.set_optimizer("sgd", lr=lr)
    de._engine.set_dp_grad_targets(targets[r])
    if streamed:
      de._engine.enable_streamed_push(chunk)
  shape = (B,) if hot == 1 and rng.random() < 0.5 else (B, hot)
  glob = [_draw_ids(nrng, sizes[t][0], shape, prof["power_law"]) for t in imap]
  widths = [sizes[t][1] for t in imap]
  grads = _draw_grads(nrng, [(B, w) for w in widths], prof["dyadic"])

  def rank_fn(r):
    de, eng = des[r], des[r]._engine
    sl = slice(r * lb, (r + 1) * lb)
    with torch.no_grad():
      out = de([torch.from_numpy(g[sl]) for g in glob], concat=True)
      g = torch.from_numpy(np.concatenate([x[sl] for x in grads], 1))
      if streamed and eng.streamed_push:
        eng.push_counters.zero_()
        eng.ops.push_grad(eng.routes_stage, len(eng.routes_stage_np), g, eng.act, 1.0, [])
        for c in range(eng.push_counters.numel()):
          eng.push_counters[c] = min(chunk, lb - c * chunk)
        eng.launch_streamed_push()
      else:
        eng.ops.push_grad(eng.routes_all, len(eng.routes_all_np), g, eng.act, 1.0,
                          eng.sync_grad_signal())
      eng.backward_inplace()
      return out.numpy().copy()

  outs = dry_run.run_ranks(sim, rank_fn)
  ref = [t.copy() for t in tables]
  ids2d = [g.reshape(B, -1) for g in glob]
  comb = [c or "sum" for c in combiners]
  ref_outs = reference_step(ref, imap, ids2d, comb, grads, lr, world, "sgd", {})
  for r in range(world):
    exp = np.concatenate([o[r * lb:(r + 1) * lb] for o in ref_outs], 1)
    np.testing.assert_allclose(outs[r], exp, rtol=1e-4, atol=1e-4, err_msg=f"forward, rank {r}")
  got = assemble(des)
  for t in range(n_tables):
    if t in dp_tables:
      np.testing.assert_array_equal(got[t], tables[t])
      j = dp_tables.index(t)
      for r in range(world):
        loc = np.zeros_like(tables[t])
        for i, ti in enumerate(imap):
          if ti == t:
            ids = ids2d[i][r * lb:(r + 1) * lb]
            n = ids.shape[1]
            g = grads[i][r * lb:(r + 1) * lb] / (n if comb[t] == "mean" else 1)
            np.add.at(loc, ids.reshape(-1), np.repeat(g, n, axis=0))
        np.testing.assert_allclose(targets[r][j].numpy(), loc, rtol=1e-4, atol=1e-5,
                                   err_msg=f"replicated table {t}, rank {r}")
    else:
      np.testing.assert_allclose(got[t], ref[t], rtol=1e-3, atol=1e-3, err_msg=f"table {t}")
  return "ok"


@pytest.mark.parametrize("world", [1, 2, 3, 4, 8])
@pytest.mark.parametrize("streamed", [False, True])
def test_random_plans_backward_inplace(world, streamed):
  n = 6 if world < 8 else 3
  outcomes = [run_inplace_plan(11000 * world + 17 * s + int(streamed), world, streamed)
              for s in range(n)]
  assert outcomes.count("ok") >= n // 2 + 1, outcomes


@pytest.mark.parametrize("world_save,world_load", [(1, 3), (4, 2), (8, 1), (3, 5)])
def test_file_checkpoint_is_sharding_independent(world_save, world_load, tmp_path):
  """save_weights: every rank writes its own column / row slices into global-layout .npy files
  (no gather); load_weights under a different world size and plan restores the same tables."""
  rng = np.random.default_rng(3)
  sizes = [(6, 8), (40, 8), (9, 16), (300, 16), (25, 8), (500, 8), (64, 12)]
  embs = [{"input_dim": r, "output_dim": w, "combiner": "sum"} for r, w in sizes]
  tables = [rng.standard_normal(s).astype(np.float32) for s in sizes]

  def plan(world, i):
    kw = {"strategy": ["memory_balanced", "memory_optimized"][i % 2]}
    if world > 1:
      kw.update(data_parallel_threshold=100, row_slice_threshold=3500,
                column_slice_threshold=[1200, 960][i % 2] // world)
    return dry_run.build_engines(embs, world, **kw)

  sim, des = plan(world_save, 0)
  for de in des:
    de.set_weights(tables)
  ckpt = str(tmp_path / "ckpt")
  paths = dry_run.run_ranks(sim, lambda r: des[r].save_weights(ckpt, chunk=256))
  assert all(p == paths[0] for p in paths) and len(paths[0]) == len(sizes)
  for t, path in enumerate(paths[0]):
    np.testing.assert_array_equal(np.load(path), tables[t])
  sim2, des2 = plan(world_load, 1)
  dry_run.run_ranks(sim2, lambda r: des2[r].load_weights(ckpt, chunk=128))
  for got, want in zip(assemble(des2), tables):
    np.testing.assert_array_equal(got, want)
  os_missing = str(tmp_path / "nothing")
  with pytest.raises(FileNotFoundError):
    des2[0].load_weights(os_missing)


@pytest.mark.parametrize("kind", ["sgd", "adagrad", "adam"])
def test_shared_learning_rate_word_is_owned_by_the_trainer(kind):
  """A hand-scheduled trainer shares one device-resident learning-rate word with the engine
  (``share_lr``) and zeroes it while it warms up before graph capture.  The engine's table
  refresh - triggered in the middle of that warm-up when lazily created optimizer state appears -
  must not re-arm the rate (regression: dense weights drifted during the warm-up of the Adagrad
  DLRM step)."""
  rng = np.random.default_rng(2)
  sizes = [(30, 8), (12, 16), (50, 8)]
  embs = [{"input_dim": r, "output_dim": w, "combiner": "sum"} for r, w in sizes]
  world, lb = 2, 4
  sim, des = dry_run.build_engines(embs, world, strategy="memory_balanced")
  tables = [rng.standard_normal(s).astype(np.float32) for s in sizes]
  lrs = [torch.zeros(1) for _ in range(world)]
  for r, de in enumerate(des):
    de.set_weights(tables)
    de.set_optimizer(kind, lr=0.5)
    de._engine.share_lr(lrs[r])
  ids = [rng.integers(0, r_, size=(lb * world, 2)) for r_, _ in sizes]
  grads = [rng.standard_normal((lb * world, w)).astype(np.float32) for _, w in sizes]

  def step(r):
    sl = slice(r * lb, (r + 1) * lb)
    out = des[r]([torch.from_numpy(i[sl]) for i in ids], concat=True)
    out.backward(torch.from_numpy(np.concatenate([g[sl] for g in grads], 1)))

  dry_run.run_ranks(sim, step)  # warm-up pass: the shared word is zero
  assert all(float(t) == 0.0 for t in lrs), "the engine wrote a trainer-owned learning rate"
  for got, want in zip(assemble(des), tables):
    np.testing.assert_array_equal(got, want)
  for t in lrs:  # the trainer arms the rate: now the tables move
    t.fill_(0.5)
  dry_run.run_ranks(sim, step)
  moved = [np.abs(g - w).max() for g, w in zip(assemble(des), tables)]
  assert min(moved) > 1e-3, moved
  # an engine that owns its rate keeps following set_optimizer / set_learning_rate
  sim2, des2 = dry_run.build_engines(embs, 1)
  des2[0].set_weights(tables)
  des2[0].set_optimizer(kind, lr=0.25)
  dry_run.run_ranks(sim2, lambda r: des2[0]([torch.from_numpy(i[:lb]) for i in ids],
                                            concat=True).sum().backward())
  assert abs(float(des2[0]._engine.lr_t) - 0.25) < 1e-7


@pytest.mark.parametrize("kind", ["sgd", "adagrad", "rowwise_adagrad", "adam"])
def test_dry_updates_leave_tables_and_optimizer_state_untouched(kind):
  """Graph warm-up passes of the hand-scheduled trainers run with ``dry_updates(True)``: every
  kernel is launched, but tables, optimizer state and the step counter must come out exactly as
  they went in - then a real step must equal a step taken without any warm-up.  With weight decay
  as well: a dry pass applies none."""
  for weight_decay in (0.0, 0.5):
    _dry_updates_case(kind, weight_decay)


def _dry_updates_case(kind, weight_decay):
  rng = np.random.default_rng(4)
  sizes = [(30, 8), (12, 16), (50, 8), (21, 16)]
  embs = [{"input_dim": r, "output_dim": w, "combiner": "sum"} for r, w in sizes]
  world, lb = 2, 4
  tables = [rng.standard_normal(s).astype(np.float32) for s in sizes]
  ids = [rng.integers(0, r_, size=(lb * world, 2)) for r_, _ in sizes]
  grads = [rng.standard_normal((lb * world, w)).astype(np.float32) * 0.1 for _, w in sizes]

  def make():
    sim, des = dry_run.build_engines(embs, world, strategy="memory_balanced")
    for de in des:
      de.set_weights(tables)
      de.set_optimizer(kind, lr=0.3, weight_decay=weight_decay)
    return sim, des

  def step(sim, des):
    def fn(r):
      sl = slice(r * lb, (r + 1) * lb)
      out = des[r]([torch.from_numpy(i[sl]) for i in ids], concat=True)
      out.backward(torch.from_numpy(np.concatenate([g[sl] for g in grads], 1)))
    dry_run.run_ranks(sim, fn)

  sim_a, des_a = make()
  for de in des_a:
    de._engine.dry_updates(True)
  step(sim_a, des_a)
  step(sim_a, des_a)
  for got, want in zip(assemble(des_a), tables):
    np.testing.assert_array_equal(got, want)
  for de in des_a:
    assert de._engine.step_count() == 0
    for slots in de._engine.opt_state.values():
      for k, s in enumerate(slots):
        init = 0.1 if kind in ("adagrad", "rowwise_adagrad") else 0.0
        assert float((s - init).abs().max()) == 0.0, (kind, k)
    de._engine.dry_updates(False)
  step(sim_a, des_a)
  sim_b, des_b = make()
  step(sim_b, des_b)
  for a, b in zip(assemble(des_a), assemble(des_b)):
    np.testing.assert_array_equal(a, b)
  # SGD counts steps on the sorted update only, which it takes with weight decay
  assert des_a[0]._engine.step_count() == des_b[0]._engine.step_count() == \
      (0 if kind == "sgd" and not weight_decay else 1)


@pytest.mark.parametrize("world", [1, 3])
def test_prepared_engine_with_direct_input_views(world):
  """The data-loader fast path: ``prepare()`` allocates the staging buffers, the loader writes
  the ids straight into ``input_views`` (int32 here), ``run()`` does the forward without any
  staging copy, and a second batch reuses the same buffers."""
  rng = np.random.default_rng(8)
  sizes = [(30, 8), (12, 16), (50, 8), (21, 4)]
  hots = [1, 3, 2, 1]
  embs = [{"input_dim": r, "output_dim": w, "combiner": "sum"} for r, w in sizes]
  sim, des = dry_run.build_engines(embs, world, strategy="memory_balanced")
  tables = [rng.standard_normal(s).astype(np.float32) for s in sizes]
  lb = 5
  for de in des:
    de.set_weights(tables)
    de._engine.prepare(lb, hots, ids64=False)
  ptrs = [[v.data_ptr() for v in de._engine.input_views] for de in des]
  for batch in range(2):
    ids = [rng.integers(0, r_, size=(lb * world, h)).astype(np.int32)
           for (r_, _), h in zip(sizes, hots)]

    def fn(r):
      eng = des[r]._engine
      sl = slice(r * lb, (r + 1) * lb)
      for v, i in zip(eng.input_views, ids):
        assert v.dtype == torch.int32 and tuple(v.shape) == i[sl].shape
        v.copy_(torch.from_numpy(i[sl]))
      with torch.no_grad():
        return eng.run(concat=True).numpy().copy()

    outs = dry_run.run_ranks(sim, fn)
    exp = np.concatenate([tables[t][ids[t]].sum(1) for t in range(len(sizes))], 1)
    for r in range(world):
      np.testing.assert_allclose(outs[r], exp[r * lb:(r + 1) * lb], rtol=1e-5, atol=1e-5)
    assert ptrs == [[v.data_ptr() for v in de._engine.input_views] for de in des]
