"""HBM row cache of host-offloaded tables (``DistributedEmbedding(offload_cache_size=)``): the
Python policy, argument validation and - on an H100 - the cache pass against the policy, and
cached training against the same training without a cache."""
import numpy as np
import pytest
import torch

from distributed_embeddings_b200.parallel.offload_cache import (WAYS, CachePolicy, cache_bytes,
                                                                cache_set, split_budget)


# ----------------------------------------------------------------------------- policy (CPU)
def _rows_of_set(st, n_sets, count, start=0):
  """The first ``count`` rows >= start that hash to set ``st``."""
  out, r = [], start
  while len(out) < count:
    if cache_set(r, n_sets) == st:
      out.append(r)
    r += 1
  return out


def test_hash_is_fixed():
  # pins the mixing function shared with offload_cache.cu
  assert [cache_set(r, 1000) for r in (0, 1, 2, 12345, 2**40 + 3)] == [0, 734, 501, 596, 912]
  assert cache_set(0, 7) == 0
  assert len({cache_set(r, 64) for r in range(4096)}) == 64


def test_hits_refresh_and_misses_fill_in_row_order():
  p = CachePolicy(n_sets=2, n_spill=64)
  rows = _rows_of_set(0, 2, 3)
  slot_of, wb, fills = p.step(list(reversed(rows)) + rows, train=False)
  # ascending rows take ways 0, 1, 2 of set 0
  assert [slot_of[r] for r in rows] == [0, 1, 2]
  assert fills == [(0, rows[0]), (1, rows[1]), (2, rows[2])] and wb == []
  assert p.stats == {"hits": 0, "misses": 3, "spills": 0, "writebacks": 0}
  assert not p.dirty.any(), "a forward-only pass marks nothing dirty"
  slot_of, _, fills = p.step([rows[1]], train=True)
  assert fills == [] and slot_of[rows[1]] == 1 and p.ticks[1] == 2 and p.ticks[0] == 1
  assert p.dirty[1] == 1 and p.dirty[0] == 0
  assert p.stats["hits"] == 1


def test_lru_victims_and_dirty_write_back():
  p = CachePolicy(n_sets=1, n_spill=64)
  first = list(range(32))
  p.step(first, train=True)            # tick 1: every way, dirty
  p.step(first[16:], train=False)      # tick 2: ways 16..31 refreshed
  new = list(range(100, 104))
  slot_of, wb, fills = p.step(new, train=False)  # tick 3: LRU = ways 0..3 (tick 1, by way)
  assert [slot_of[r] for r in new] == [0, 1, 2, 3]
  assert wb == [(0, 0), (1, 1), (2, 2), (3, 3)], "dirty victims go back to the host first"
  assert fills == [(w, r) for w, r in zip(range(4), new)]
  # clean victims are not written back
  p2 = CachePolicy(n_sets=1, n_spill=64)
  p2.step(first, train=False)
  _, wb2, _ = p2.step([200], train=True)
  assert wb2 == []


def test_way_used_this_tick_is_never_evicted_and_overflow_spills():
  p = CachePolicy(n_sets=1, n_spill=64)
  p.step(list(range(32)), train=True)
  # 30 hits + 5 misses: only the two ways not used in this tick are free
  rows = list(range(2, 32)) + [40, 41, 42, 43, 44]
  slot_of, wb, fills = p.step(rows, train=True)
  assert slot_of[40] == 0 and slot_of[41] == 1
  uniq = sorted(rows)
  for r in (42, 43, 44):
    assert slot_of[r] == 32 + uniq.index(r), "spill slot = base + unique index"
  assert p.stats["spills"] == 3 and wb == [(0, 0), (1, 1)]
  assert sorted(s for s, _ in fills) == [0, 1, 32 + uniq.index(42), 32 + uniq.index(43),
                                         32 + uniq.index(44)]
  # the next pass writes the (dirty) spilled rows back and empties the spill region
  slot_of, wb, _ = p.step([42], train=False)
  assert wb[:3] == [(32 + uniq.index(r), r) for r in (42, 43, 44)]
  # every way was used in the last tick: 42 takes the least recently used one, way 0
  assert slot_of[42] == 0 and (p.tags[32:] == -1).all()


def test_flush_writes_dirty_rows_once():
  p = CachePolicy(n_sets=4, n_spill=16)
  p.step([1, 2, 3, -1], train=True)
  out = p.flush()
  assert sorted(r for _, r in out) == [1, 2, 3]
  assert p.flush() == []


def test_budget_split_and_bytes():
  sets = split_budget(64 * 100 * 32, [(1000, 64), (3000, 64)])
  assert sets == [25, 75]
  assert split_budget(0, [(1000, 16)]) == [1], "at least one set"
  assert cache_bytes(2, 10, 16, [16]) == (64 + 10) * 4 * 32 + (64 + 10) * 12 + 64 * 4 + 36


def test_cache_without_offload_is_rejected():
  from distributed_embeddings_b200.parallel.dist_model_parallel import DistributedEmbedding
  embs = [{"input_dim": 100, "output_dim": 8}]
  with pytest.raises(ValueError, match="gpu_embedding_size"):
    DistributedEmbedding(embs, offload_cache_size=1000, device="cpu", world_size=1, rank=0)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_cache_with_16_bit_tables_is_rejected(dtype):
  from distributed_embeddings_b200.parallel.dist_model_parallel import DistributedEmbedding
  embs = [{"input_dim": 100, "output_dim": 8}]
  with pytest.raises(ValueError, match="fp32 tables only"):
    DistributedEmbedding(embs, offload_cache_size=1000, gpu_embedding_size=10, device="cpu",
                         world_size=1, rank=0, table_dtype=dtype)


def test_cache_needs_the_fused_back_end():
  from distributed_embeddings_b200.parallel.dist_model_parallel import DistributedEmbedding
  embs = [{"input_dim": 100, "output_dim": 8}]
  with pytest.raises(ValueError, match="fused back end"):
    DistributedEmbedding(embs, offload_cache_size=1000, gpu_embedding_size=10, device="cpu",
                         world_size=1, rank=0, backend="torch")


def test_cache_is_rejected_on_more_than_one_rank():
  from distributed_embeddings_b200.parallel.dist_model_parallel import DistributedEmbedding
  embs = [{"input_dim": 100, "output_dim": 8}, {"input_dim": 200, "output_dim": 8}]
  with pytest.raises(ValueError, match="world size 1"):
    DistributedEmbedding(embs, offload_cache_size=1000, gpu_embedding_size=10, device="cpu",
                         world_size=2, rank=0)


def test_plan_report_counts_the_cache_bytes():
  import json
  import os
  import subprocess
  import sys
  root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
  base = [sys.executable, "tools/plan_report.py", "--tables", "1000x64,200000x64,300000x32",
          "--world", "1", "--gpu-embedding-size", str(1000 * 64 + 1), "--global-batch", "512",
          "--optimizer-slots", "1", "--json"]

  def run(*extra):
    out = subprocess.run(base + list(extra), cwd=root, capture_output=True, text=True,
                         check=False)
    assert out.returncode == 0, out.stderr[-1000:]
    return json.loads(out.stdout.strip().splitlines()[-1])["ranks"][0]
  plain, cached = run(), run("--offload-cache-size", "204800")
  assert plain["cache_gib"] == 0 and plain["host_gib"] > 0
  # 204800 elements split by rows: 81920 -> 1280 rows of width 64 -> 40 sets;
  # 122880 -> 3840 rows of width 32 -> 120 sets; spill regions of 512 ids each
  exp = cache_bytes(40, 512, 64, [64]) + cache_bytes(120, 512, 32, [32])
  assert abs(cached["cache_gib"] - exp / 2**30) < 1e-6
  assert cached["hbm_gib"] == pytest.approx(plain["hbm_gib"] + cached["cache_gib"], abs=0.02)


def test_default_dlrm_is_unchanged():
  from distributed_embeddings_b200.models.dlrm import DLRM
  a = DLRM([50, 60], device="cpu", backend="torch", compute_dtype=torch.float32)
  b = DLRM([50, 60], device="cpu", backend="torch", compute_dtype=torch.float32,
           gpu_embedding_size=None, offload_cache_size=None)
  assert list(a.state_dict()) == list(b.state_dict())
  assert a.embedding.offload_cache_size is None


# ----------------------------------------------------------------------------- GPU (one H100)
def _cuda():
  return torch.device("cuda", 0)


SMALL, BIG, WIDTH = 64, 6000, 16


def _pair(kind, cache_elems, input_table_map=(0, 1, 1), **opt):
  """A cached and an uncached layer with the same tables: table 1 (BIG rows) is offloaded."""
  from distributed_embeddings_b200.parallel.dist_model_parallel import DistributedEmbedding
  embs = [{"input_dim": SMALL, "output_dim": WIDTH, "combiner": "sum"},
          {"input_dim": BIG, "output_dim": WIDTH, "combiner": "sum"}]
  kw = dict(device=_cuda(), backend="fused", gpu_embedding_size=SMALL * WIDTH + 1,
            input_table_map=list(input_table_map))
  torch.manual_seed(0)
  cached = DistributedEmbedding(embs, offload_cache_size=cache_elems, **kw)
  plain = DistributedEmbedding(embs, **kw)
  plain.set_weights(cached.get_weights())
  assert any(l.cpu_offloaded for l in cached.local_embedding_layers)
  if kind is not None:
    cached.set_optimizer(kind, lr=0.05, **opt)
    plain.set_optimizer(kind, lr=0.05, **opt)
  return cached, plain


def _ids(step, b, hot, skewed, n_inputs=3):
  g = torch.Generator().manual_seed(100 + step)
  out = [torch.randint(0, SMALL, (b, hot), generator=g, dtype=torch.int32)]
  for _ in range(n_inputs - 1):
    if skewed:  # power law over the rows (density ~ 1 / row): log-uniform
      u = torch.rand(b, hot, generator=g, dtype=torch.float64)
      r = (BIG ** u - 1).floor().clamp(0, BIG - 1).long()
      out.append(r.to(torch.int32))
    else:
      out.append(torch.randint(0, BIG, (b, hot), generator=g, dtype=torch.int32))
  # out-of-range ids contribute zero and must not take a slot
  out[1][0, 0] = BIG + 5
  out[2][1, 0] = -3
  return [x.to(_cuda()) for x in out]


def _cache_of(de):
  (m, c), = de._engine.caches.items()
  return c


@pytest.mark.gpu
@pytest.mark.parametrize("skewed", [False, True])
def test_gpu_cache_pass_matches_the_python_policy(skewed):
  """Tags, ticks and dirty bits after every pass equal the Python policy exactly; every spilled
  row appears exactly once; the lookups through the cache equal the zero-copy lookups."""
  cached, plain = _pair("adagrad", 2 * WAYS * WIDTH)  # 2 sets: every step evicts and spills
  pol = None
  for step in range(5):
    ids = _ids(step, 64, 3, skewed)
    train = step != 2  # one forward-only pass (no grad): marks nothing dirty
    with torch.set_grad_enabled(train):
      out_c, out_p = cached(ids, concat=True), plain(ids, concat=True)
    assert torch.equal(out_c, out_p), "lookups through the cache differ from zero-copy ones"
    if train:
      (out_c * 1.0).sum().backward()
      (out_p * 1.0).sum().backward()
    c = _cache_of(cached)
    if pol is None:
      pol = CachePolicy(c.n_sets, c.n_spill)
    rows = [int(r) for x in ids[1:] for r in x.view(-1).tolist() if 0 <= r < BIG]
    pol.step(rows, train)
    torch.cuda.synchronize()
    assert np.array_equal(c.tags.cpu().numpy(), pol.tags), step
    assert np.array_equal(c.ticks.cpu().numpy(), pol.ticks), step
    assert np.array_equal(c.dirty.cpu().numpy(), pol.dirty), step
    spill = c.tags[c.n_sets * WAYS:].cpu().numpy()
    held = np.concatenate([c.tags[:c.n_sets * WAYS].cpu().numpy(), spill])
    held = held[held >= 0]
    assert len(held) == len(set(held.tolist())), "a row holds two slots"
  stats = cached.offload_cache_stats()
  assert stats[0]["table"] == 1
  assert {k: stats[0][k] for k in pol.stats} == pol.stats
  assert cached.offload_cache_stats()[0]["hits"] == 0, "reset"


def _train(de, steps, b, hot, skewed, scale=1.0):
  outs = []
  for s in range(steps):
    ids = _ids(s, b, hot, skewed)
    out = de(ids, concat=True)
    w = torch.linspace(-1, 1, out.shape[1], device=_cuda()) * scale
    (out * w).sum().backward()
    outs.append(out.detach())
  return outs


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["adagrad", "rowwise_adagrad", "adam", "sgd"])
@pytest.mark.parametrize("skewed", [False, True])
def test_gpu_cached_training_matches_uncached(kind, skewed):
  """Several steps through a cache far smaller than the working set.  The sorted update sums a
  row's gradient rows in the same (input) order with and without the cache, but the
  occurrence-balanced kernel splits long runs at tile borders that depend on the keys, and the
  keys are slot ids here: a row's partial sums may be associated differently.  Tables and state
  therefore agree to fp32 rounding: at most a few ulps of the per-step update, far below it."""
  opt = {"deterministic": True} if kind == "sgd" else {}
  cached, plain = _pair(kind, 2 * WAYS * WIDTH, **opt)
  w0 = plain.get_weights()
  outs_c = _train(cached, 6, 128, 2, skewed)
  outs_p = _train(plain, 6, 128, 2, skewed)
  assert torch.equal(outs_c[0], outs_p[0])
  for a, b in zip(outs_c, outs_p):
    torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-6)
  wc, wp = cached.get_weights(), plain.get_weights()
  for a, b in zip(wc, wp):
    np.testing.assert_allclose(a, b, rtol=1e-5, atol=1e-6)
  # the offloaded table moved by far more than the tolerance above
  assert np.abs(wp[1] - w0[1]).max() > 1e-3, "the offloaded table trained"
  sc, sp = cached.get_optimizer_state(), plain.get_optimizer_state()
  assert sc["step"] == sp["step"]
  if sp["tables"] is not None:
    for ta, tb in zip(sc["tables"], sp["tables"]):
      for a, b in zip(ta or [], tb or []):
        np.testing.assert_allclose(a, b, rtol=1e-5, atol=1e-6)


@pytest.mark.gpu
def test_gpu_flush_round_trips_rows_and_state_bit_for_bit():
  """Fill + flush without an update moves rows and state unchanged: after dry updates (zero
  gradient) the host tables and Adam state are bit-identical."""
  cached, _ = _pair("adam", 2 * WAYS * WIDTH)
  _train(cached, 1, 64, 2, False)
  before_w = [w.copy() for w in cached.get_weights()]
  before_s = cached.get_optimizer_state()
  cached._engine.dry_updates(True)
  _train(cached, 4, 64, 2, True)
  cached._engine.dry_updates(False)
  for a, b in zip(before_w, cached.get_weights()):
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
  after_s = cached.get_optimizer_state()
  for ta, tb in zip(before_s["tables"], after_s["tables"]):
    for a, b in zip(ta or [], tb or []):
      assert np.array_equal(a.view(np.uint32), b.view(np.uint32))


@pytest.mark.gpu
def test_gpu_checkpoint_round_trip_with_a_dirty_cache(tmp_path):
  cached, plain = _pair("adagrad", 4 * WAYS * WIDTH)
  _train(cached, 3, 64, 2, True)
  _train(plain, 3, 64, 2, True)
  c = _cache_of(cached)
  assert int(c.dirty.sum()) > 0
  cached.save_weights(str(tmp_path / "w"))
  saved = [np.load(str(tmp_path / "w" / f"table_{t}.npy")) for t in range(2)]
  for a, b in zip(saved, plain.get_weights()):
    np.testing.assert_allclose(a, b, rtol=1e-5, atol=1e-6)
  cached.load_weights(str(tmp_path / "w"))
  assert int((c.tags >= 0).sum()) == 0, "loading invalidates the cache"
  ids = _ids(9, 64, 2, True)
  with torch.no_grad():
    out = cached(ids, concat=True)
  ref = [torch.from_numpy(w).to(_cuda()) for w in saved]
  exp = []
  for t, x in zip([0, 1, 1], ids):
    xl = x.long()
    ok = (xl >= 0) & (xl < ref[t].shape[0])
    exp.append((ref[t][xl.clamp(0, ref[t].shape[0] - 1)] * ok.unsqueeze(-1)).sum(1))
  torch.testing.assert_close(out, torch.cat(exp, 1), rtol=1e-6, atol=1e-6)


def _dlrm(cache, sizes, **kw):
  from distributed_embeddings_b200.models.dlrm import DLRM
  torch.manual_seed(7)
  big = sum(sizes) - max(sizes) - sorted(sizes)[-2]
  return DLRM(sizes, device=_cuda(), compute_dtype=torch.bfloat16, backend="fused",
              gpu_embedding_size=big * 128 + 1, offload_cache_size=cache, **kw)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["adagrad", "rowwise_adagrad", "adam", "sgd"])
@pytest.mark.parametrize("interaction", ["dot", "dcnv2"])
def test_gpu_dlrm_train_step_with_a_cache(kind, interaction):
  """DLRMTrainStep (CUDA graph, several replays) on a model whose two largest tables are
  offloaded with a tiny cache, against the same step without a cache, with an evaluate between
  training steps.  Losses and tables agree to fp32 rounding (see above)."""
  from distributed_embeddings_b200.models.dlrm_fast import DLRMTrainStep
  sizes = [200 + 13 * i for i in range(24)] + [5000, 7000]
  kw = {}
  if interaction == "dcnv2":
    kw = dict(interaction="dcnv2", dcn_num_layers=1, dcn_low_rank_dim=64,
              multi_hot_sizes=[1] * 24 + [3, 2])
  cached = _dlrm(2 * WAYS * 128, sizes, **kw)
  plain = _dlrm(None, sizes, **kw)
  plain.load_state_dict(cached.state_dict())
  assert sum(l.cpu_offloaded for l in cached.embedding.local_embedding_layers) == 2
  opt = {"embedding_optimizer_kwargs": {"deterministic": True}} if kind == "sgd" else {}
  b = 256
  g = torch.Generator().manual_seed(3)
  hots = kw.get("multi_hot_sizes", [1] * 26)
  batches = []
  for _ in range(4):
    u = torch.rand(26, b * max(hots), generator=g, dtype=torch.float64)
    cat = [(torch.tensor(s, dtype=torch.float64) ** u[f, :b * h] - 1).floor()
           .clamp(0, s - 1).to(torch.int32) for f, (s, h) in enumerate(zip(sizes, hots))]
    cat = torch.cat(cat) if interaction == "dcnv2" else torch.stack(cat)
    batches.append((torch.rand(b, 13, generator=g).to(_cuda()), cat.to(_cuda()),
                    torch.randint(0, 2, (b,), generator=g).float().to(_cuda())))
  res = []
  for model in (cached, plain):
    t = DLRMTrainStep(model, lr=0.05, embedding_optimizer=kind, use_cuda_graph=True, **opt)
    losses = [float(t.step(*batches[0])), float(t.step(*batches[1]))]
    # a forward-only pass between training steps (marks nothing dirty, updates nothing)
    ev = t.predict(batches[2][0], batches[2][1]).cpu() if interaction == "dot" else None
    losses += [float(t.step(*batches[2])), float(t.step(*batches[3]))]
    torch.cuda.synchronize()
    res.append((losses, ev, model.embedding.get_weights()))
  (lc, evc, wc), (lp, evp, wp) = res
  np.testing.assert_allclose(lc, lp, rtol=1e-5, atol=1e-6)
  if evc is not None:
    torch.testing.assert_close(evc, evp, rtol=1e-5, atol=1e-6)
  for a, bb in zip(wc, wp):
    np.testing.assert_allclose(a, bb, rtol=1e-4, atol=1e-6)
  st = cached.embedding.offload_cache_stats()
  assert len(st) == 2 and all(s["spills"] > 0 and s["writebacks"] > 0 for s in st)


def _batches(sizes, b, n, seed=3):
  g = torch.Generator().manual_seed(seed)
  out = []
  for _ in range(n):
    u = torch.rand(len(sizes), b, generator=g, dtype=torch.float64)
    cat = torch.stack([(torch.tensor(float(s), dtype=torch.float64) ** u[f] - 1).floor()
                       .clamp(0, s - 1).to(torch.int32) for f, s in enumerate(sizes)])
    out.append((torch.rand(b, 13, generator=g).to(_cuda()), cat.to(_cuda()),
                torch.randint(0, 2, (b,), generator=g).float().to(_cuda())))
  return out


@pytest.mark.gpu
def test_gpu_no_grad_forward_before_the_train_step_keeps_updates():
  """A forward-only module call (no grad) before DLRMTrainStep must not turn the step's cache
  passes into forward-only ones: every update reaches the host tables after a flush."""
  from distributed_embeddings_b200.models.dlrm_fast import DLRMTrainStep
  sizes = [200 + 13 * i for i in range(24)] + [5000, 7000]
  cached, plain = _dlrm(2 * WAYS * 128, sizes), _dlrm(None, sizes)
  plain.load_state_dict(cached.state_dict())
  w0 = plain.embedding.get_weights()
  batches = _batches(sizes, 256, 4)
  res = []
  for model in (cached, plain):
    with torch.no_grad():
      model.embedding([c for c in batches[0][1]])
    t = DLRMTrainStep(model, lr=0.05, embedding_optimizer="adagrad", use_cuda_graph=True)
    res.append([float(t.step(*bt)) for bt in batches])
    t2 = DLRMTrainStep(model, lr=0.05, embedding_optimizer="adagrad", use_cuda_graph=False)
    res[-1] += [float(t2.step(*bt)) for bt in batches[:2]]
  np.testing.assert_allclose(res[0], res[1], rtol=1e-5, atol=1e-6)
  # Six steps of a bf16 dense side: an fp32-rounding difference of a table value can flip the
  # bf16 rounding of an activation and so change the gradients by bf16 ulps, which Adagrad's
  # normalisation turns into relative changes of the small updates (about 0.1 measured on an
  # H100).  Compare the updates, not the values, with the bound bench.py's verify uses (0.3): with
  # a cache of one set per table nearly every row is evicted each step, so updates dropped on
  # eviction would make this error about 1.
  wc, wp = cached.embedding.get_weights(), plain.embedding.get_weights()
  err = sum(float(((a.astype(np.float64) - b)**2).sum()) for a, b in zip(wc, wp))
  upd = sum(float(((b.astype(np.float64) - c)**2).sum()) for b, c in zip(wp, w0))
  assert upd > 0 and (err / upd)**0.5 <= 0.3, (err, upd)


@pytest.mark.gpu
def test_gpu_train_predict_train_equals_train_train():
  """After a flush, [train, predict, train] leaves the cached tables where [train, train] does
  (the predict only changes which rows the cache holds; fp32-rounding bound as above)."""
  from distributed_embeddings_b200.models.dlrm_fast import DLRMTrainStep
  sizes = [200 + 13 * i for i in range(24)] + [5000, 7000]
  a, b = _dlrm(2 * WAYS * 128, sizes), _dlrm(2 * WAYS * 128, sizes)
  b.load_state_dict(a.state_dict())
  batches = _batches(sizes, 256, 3)
  ta = DLRMTrainStep(a, lr=0.05, embedding_optimizer="adam", use_cuda_graph=True)
  tb = DLRMTrainStep(b, lr=0.05, embedding_optimizer="adam", use_cuda_graph=True)
  ta.step(*batches[0])
  ta.predict(batches[2][0], batches[2][1])
  ta.step(*batches[1])
  tb.step(*batches[0])
  tb.step(*batches[1])
  torch.cuda.synchronize()
  for x, y in zip(a.embedding.get_weights(), b.embedding.get_weights()):
    np.testing.assert_allclose(x, y, rtol=1e-5, atol=1e-6)
  sa, sb = a.embedding.get_optimizer_state(), b.embedding.get_optimizer_state()
  for ta_, tb_ in zip(sa["tables"], sb["tables"]):
    for x, y in zip(ta_ or [], tb_ or []):
      np.testing.assert_allclose(x, y, rtol=1e-5, atol=1e-6)


@pytest.mark.gpu
def test_gpu_hybrid_trainer_and_module_checkpoint_on_a_cached_model():
  """HybridTrainer (autograd path) on a cached DLRM against the uncached one; the module's
  state_dict flushes the cache first and load_state_dict drops it."""
  from distributed_embeddings_b200.models.trainer import HybridTrainer
  sizes = [200 + 13 * i for i in range(24)] + [5000, 7000]
  cached, plain = _dlrm(2 * WAYS * 128, sizes), _dlrm(None, sizes)
  plain.load_state_dict(cached.state_dict())
  batches = _batches(sizes, 256, 3)
  losses = []
  for model in (cached, plain):
    tr = HybridTrainer(model, lr=0.05, embedding_optimizer="rowwise_adagrad")
    losses.append([float(tr.step(n, list(c), l.view(-1, 1))) for n, c, l in batches])
  np.testing.assert_allclose(losses[0], losses[1], rtol=1e-5, atol=1e-6)
  sd_c = {k: v.detach().cpu().clone() for k, v in cached.state_dict().items()}
  sd_p = plain.state_dict()
  for k, v in sd_p.items():
    torch.testing.assert_close(sd_c[k], v.detach().cpu(), rtol=1e-4, atol=1e-6)
  # load the uncached model's tables into the cached one: the cache must not serve old rows
  cached.load_state_dict(plain.state_dict())
  c = next(iter(cached.embedding._engine.caches.values()))
  assert int((c.tags >= 0).sum()) == 0
  for x, y in zip(cached.embedding.get_weights(), plain.embedding.get_weights()):
    assert np.array_equal(x, y)
