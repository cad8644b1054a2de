"""Exact ROC AUC for the DLRM evaluation: ``utils.metrics.ExactAUC``, the ``auc_append`` /
``radix_sort_keys32`` / ``auc_count`` kernels and ``DLRMTrainStep(eval_auc="exact")``.

CPU: the key encoding (order of scores and labels, -0.0, rejection of NaN and out-of-range
values); the numpy ``(P, N, U2)`` against scipy's Mann-Whitney U and ``binary_auc`` on random,
heavily tied, all-equal and one-class data; the CPU metric's chunking, overflow and reset; its
``all_gather`` at gloo world 2 and 3 with a different sample count on each rank.
GPU: the kernels equal the CPU integers exactly (n = 1 .. millions, appends with ``n_valid <
batch``, ties, scores of exactly 0 and 1), a NaN probability and an overflow raise and nothing is
written past the buffer, a CUDA-graph replay equals eager launches; the DLRM step in exact mode on
the dot and dcnv2 models.
"""
import copy
import math
import os
import traceback

import numpy as np
import pytest
import torch
from scipy import stats

from distributed_embeddings_b200.utils.metrics import (ExactAUC, auc_counts_from_keys,
                                                       auc_from_counts, auc_keys, binary_auc)


def _draw(kind, n, seed):
  rng = np.random.default_rng(seed)
  y = (rng.random(n) < 0.3).astype(np.float32)
  if kind == "random":
    p = rng.random(n).astype(np.float32)
  elif kind == "tied":  # a few distinct scores, positives shifted up a little
    p = rng.integers(0, 5, n).astype(np.float32) / np.float32(4)
    p = np.where((y > 0) & (rng.random(n) < 0.5), np.minimum(p + np.float32(0.25), 1), p)
  elif kind == "equal":
    p = np.full(n, 0.375, dtype=np.float32)
  elif kind == "ends":  # exactly 0 and 1 and their neighbours
    vals = np.array([0.0, 1.0, np.nextafter(np.float32(0), np.float32(1)),
                     np.nextafter(np.float32(1), np.float32(0)), 0.5], dtype=np.float32)
    p = vals[rng.integers(0, len(vals), n)]
  elif kind == "one_class":
    p = rng.random(n).astype(np.float32)
    y = np.ones(n, dtype=np.float32)
  else:
    raise ValueError(kind)
  return p.astype(np.float32), y


# ------------------------------------------------------------------ CPU: encoding and counts
def test_keys_order_scores_then_labels():
  rng = np.random.default_rng(0)
  base = np.concatenate([rng.random(5000).astype(np.float32),
                         np.array([0.0, 1.0, 0.5, 1e-30, 1e-45], dtype=np.float32)])
  nb = np.concatenate([np.nextafter(base, np.float32(0)), np.nextafter(base, np.float32(1))])
  p = np.concatenate([base, nb]).astype(np.float32)
  p = p[(p >= 0) & (p <= 1)]
  y = (rng.random(p.size) < 0.5).astype(np.float32)
  k = auc_keys(p, y)
  assert k.dtype == np.uint32 and int(k.max()) < 2**31
  assert int(auc_keys(np.float32([1.0]), np.float32([1]))[0]) == (0x3F800000 << 1) | 1
  order = np.argsort(k, kind="stable")
  ps, ys = p[order].astype(np.float64), y[order]
  assert np.all(np.diff(ps) >= 0)  # monotone in the score
  same = np.diff(ps) == 0
  assert np.all(ys[1:][same] >= ys[:-1][same])  # negatives first within one score
  # distinct fp32 values get distinct keys, equal ones equal keys (-0.0 == 0.0)
  assert auc_keys(np.float32([-0.0]), np.float32([0]))[0] == auc_keys(np.float32([0.0]),
                                                                       np.float32([0]))[0]
  assert len(np.unique(k >> 1)) == len(np.unique(p))
  for bad in (np.nan, -1e-8, 1.0000001, np.inf):
    with pytest.raises(ValueError, match="NaN or outside"):
      auc_keys(np.float32([0.5, bad]), np.float32([0, 1]))


@pytest.mark.parametrize("kind", ["random", "tied", "equal", "ends", "one_class"])
@pytest.mark.parametrize("n", [1, 2, 37, 20000])
def test_counts_match_mann_whitney_and_binary_auc(kind, n):
  p, y = _draw(kind, n, seed=n)
  P, N, U2 = auc_counts_from_keys(auc_keys(p, y))
  assert (P, N) == (int((y > 0.5).sum()), int((y <= 0.5).sum()))
  auc = auc_from_counts(P, N, U2)
  if P == 0 or N == 0:
    assert U2 == 0 and math.isnan(auc)
    assert math.isnan(binary_auc(torch.from_numpy(y), torch.from_numpy(p)))
    return
  pos, neg = p[y > 0.5].astype(np.float64), p[y <= 0.5].astype(np.float64)
  assert U2 == round(2 * stats.mannwhitneyu(pos, neg).statistic)
  assert abs(auc - binary_auc(torch.from_numpy(y), torch.from_numpy(p))) <= 1e-12
  if kind == "equal":
    assert auc == 0.5


def test_cpu_metric_chunks_overflow_and_reset():
  p, y = _draw("tied", 1000, seed=3)
  whole = auc_counts_from_keys(auc_keys(p, y))
  m = ExactAUC(1000)
  for s in range(0, 1000, 96):
    m.update(torch.from_numpy(p[s:s + 128]), torch.from_numpy(y[s:s + 128]),
             n_valid=min(96, 1000 - s))
  assert m.counts() == whole and m.result() == auc_from_counts(*whole)
  m.update(torch.tensor([0.5]), torch.tensor([1.0]))  # one past the capacity
  with pytest.raises(RuntimeError, match="1001 samples .* holds 1000"):
    m.counts()
  m.reset()
  assert m.counts() == (0, 0, 0) and math.isnan(m.result())
  m.update(torch.tensor([0.5, float("nan")]), torch.tensor([1.0, 0.0]))
  with pytest.raises(RuntimeError, match="1 of 2 probabilities were NaN"):
    m.result()
  with pytest.raises(ValueError):
    ExactAUC(0)


def _case_all_gather(rank, world):
  p, y = _draw("tied", 3000, seed=11)
  bounds = [0, 700, 1900, 3000] if world == 3 else [0, 1234, 3000]
  lo, hi = bounds[rank], bounds[rank + 1]
  m = ExactAUC(hi - lo + 5)
  m.update(torch.from_numpy(p[lo:hi]), torch.from_numpy(y[lo:hi]))
  local = copy.copy(m)
  m.all_gather()
  assert int(m.state[0]) == 3000
  assert m.counts() == auc_counts_from_keys(auc_keys(p, y))
  assert local.counts() == auc_counts_from_keys(auc_keys(p[lo:hi], y[lo:hi]))


def _gloo_worker(rank, world, port, errq):
  try:
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.set_num_threads(1)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    _case_all_gather(rank, world)
    dist.barrier()
    dist.destroy_process_group()
  except Exception:  # pylint: disable=broad-except
    errq.put((rank, traceback.format_exc()))
    raise


@pytest.mark.parametrize("world", [2, 3])
def test_all_gather_gloo(world):
  import torch.multiprocessing as mp
  from dist_utils import _free_port
  ctx = mp.get_context("spawn")
  errq = ctx.SimpleQueue()
  port = _free_port()
  procs = [ctx.Process(target=_gloo_worker, args=(r, world, port, errq)) for r in range(world)]
  for pr in procs:
    pr.start()
  for pr in procs:
    pr.join(240)
    if pr.is_alive():
      pr.terminate()
      pr.join()
  msgs = []
  while not errq.empty():
    msgs.append(errq.get())
  assert not msgs and all(pr.exitcode == 0 for pr in procs), msgs


# ------------------------------------------------------------------ GPU: kernels
def _ops():
  from distributed_embeddings_b200.ops import _native
  return _native.require()


def _device_metric(p, y, capacity, batch, n_valid_step):
  """Append (p, y) through auc_append in chunks of `batch` rows, n_valid_step of them valid."""
  m = ExactAUC(capacity, device="cuda")
  pd, yd = torch.from_numpy(p).cuda(), torch.from_numpy(y).cuda()
  for s in range(0, p.size, n_valid_step):
    m_ = min(n_valid_step, p.size - s)
    chunk_p = torch.rand(batch, device="cuda")  # rows past n_valid must be ignored
    chunk_y = torch.ones(batch, device="cuda")
    chunk_p[:m_] = pd[s:s + m_]
    chunk_y[:m_] = yd[s:s + m_]
    m.update(chunk_p, chunk_y, n_valid=torch.full((1,), m_, dtype=torch.int64, device="cuda"))
  return m


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 31, 65536 + 17, 3_000_017])
@pytest.mark.parametrize("kind", ["random", "tied", "ends"])
def test_kernels_equal_cpu_integers(n, kind):
  p, y = _draw(kind, n, seed=n + 1)
  batch = 65536
  step = min(batch - 5, max(1, n // 3 + 1))
  m = _device_metric(p, y, n + 3, batch, step)
  assert int(m.state[0]) == n and int(m.state[1]) == 0 and int(m.state[2]) == 0
  want_keys = auc_keys(p, y)
  assert np.array_equal(m.keys[:n].cpu().numpy().view(np.uint32), want_keys)
  want = auc_counts_from_keys(want_keys)
  assert m.counts() == want
  assert np.array_equal(m.keys[:n].cpu().numpy().view(np.uint32), np.sort(want_keys))
  assert m.counts() == want  # sorting sorted keys again changes nothing
  auc = m.result()
  assert auc == auc_from_counts(*want) or (math.isnan(auc) and (want[0] == 0 or want[1] == 0))


@pytest.mark.gpu
def test_keys_only_sort_and_empty_count():
  ops = _ops()
  g = torch.Generator().manual_seed(1)
  for n, bits in [(1, 31), (4097, 31), (100_000, 31), (70_000, 12), (50_000, 9)]:
    k = torch.randint(0, 2**bits, (n + 7,), generator=g, dtype=torch.int64).to(torch.int32)
    d = k.cuda()
    ops.radix_sort_keys32(d, n, bits)
    got = d.cpu()
    assert torch.equal(got[:n], torch.sort(k[:n]).values), (n, bits)
    assert torch.equal(got[n:], k[n:])  # keys past n untouched
  out = torch.full((3,), 7, dtype=torch.int64, device="cuda")
  ops.auc_count(torch.zeros(4, dtype=torch.int32, device="cuda"), 0, out)
  assert out.tolist() == [0, 0, 0]


@pytest.mark.gpu
def test_nan_and_overflow_raise_and_stay_in_bounds():
  cap = 1000
  guard = torch.full((cap + 256,), 0x5A5A5A5A, dtype=torch.int32, device="cuda")
  m = ExactAUC(cap, device="cuda")
  m.keys = guard[:cap]
  p = torch.rand(600, device="cuda")
  y = (torch.rand(600, device="cuda") < 0.5).float()
  m.update(p, y)
  m.update(p, y)  # 1200 > 1000: dropped whole
  torch.cuda.synchronize()
  assert m.state[:3].tolist() == [600, 600, 0]
  assert torch.all(guard[600:] == 0x5A5A5A5A)
  with pytest.raises(RuntimeError, match="1200 samples .* holds 1000"):
    m.counts()
  m.reset()
  p[17] = float("nan")
  p[18] = 1.5
  m.update(p, y)
  with pytest.raises(RuntimeError, match="2 of 600 probabilities were NaN or outside"):
    m.result()
  assert torch.all(guard[cap:] == 0x5A5A5A5A)
  m.reset()
  q = torch.tensor([0.0, 1.0, -0.0, 0.0, 1.0, 0.0], device="cuda")
  m.update(q, torch.tensor([1.0, 0.0, 0.0, 1.0, 1.0, 0.0], device="cuda"))
  assert m.counts() == auc_counts_from_keys(auc_keys(q.cpu(), [1, 0, 0, 1, 1, 0]))


@pytest.mark.gpu
def test_graph_replay_equals_eager():
  ops = _ops()
  batch, cap = 4096, 40000
  p, y = _draw("tied", 9 * batch, seed=5)
  pd, yd = torch.from_numpy(p).cuda(), torch.from_numpy(y).cuda()
  sp = torch.zeros(batch, device="cuda")
  sy = torch.zeros(batch, device="cuda")
  nv = torch.zeros(1, dtype=torch.int64, device="cuda")
  g_m, e_m = ExactAUC(cap, device="cuda"), ExactAUC(cap, device="cuda")
  s = torch.cuda.Stream()
  s.wait_stream(torch.cuda.current_stream())
  with torch.cuda.stream(s):
    ops.auc_append(sp, sy, nv, g_m.keys, g_m.state)  # warm-up with no valid rows
  torch.cuda.current_stream().wait_stream(s)
  graph = torch.cuda.CUDAGraph()
  with torch.cuda.graph(graph):
    ops.auc_append(sp, sy, nv, g_m.keys, g_m.state)
  valid = [batch, 17, batch - 1, 0, 1000, batch, 3, batch, 2222]
  for i, v in enumerate(valid):
    sp.copy_(pd[i * batch:(i + 1) * batch])
    sy.copy_(yd[i * batch:(i + 1) * batch])
    nv.fill_(v)
    graph.replay()
    e_m.update(sp, sy, n_valid=v)
  torch.cuda.synchronize()
  n = sum(valid)
  assert g_m.state.tolist() == e_m.state.tolist() == [n, 0, 0, 0]
  assert torch.equal(g_m.keys[:n], e_m.keys[:n])
  sel = np.concatenate([np.arange(i * batch, i * batch + v) for i, v in enumerate(valid)])
  assert g_m.counts() == e_m.counts() == auc_counts_from_keys(auc_keys(p[sel], y[sel]))


# ------------------------------------------------------------------ GPU: the DLRM step
def _dot_setup(mode, capacity, seed=0):
  from distributed_embeddings_b200.models.dlrm import DLRM
  from distributed_embeddings_b200.models.dlrm_fast import DLRMTrainStep
  from test_dlrm_eval import SIZES, _batch
  torch.manual_seed(seed)
  model = DLRM(SIZES, device=torch.device("cuda", 0), compute_dtype=torch.bfloat16,
               backend="fused")
  kw = dict(eval_auc="exact", eval_capacity=capacity) if mode == "exact" else {}
  step = DLRMTrainStep(model, lr=0.5, use_cuda_graph=True, **kw)

  def batch(b, s):
    num, cat, lab = _batch(b, s)
    return num, cat, lab, (num, cat)
  return model, step, batch


def _dcn_setup(mode, capacity, seed=0):
  from distributed_embeddings_b200.models.dlrm_fast import DLRMTrainStep
  from test_dcn import MLPERF_LIKE, _gpu_batch, _gpu_model
  model = _gpu_model(seed, MLPERF_LIKE)
  kw = dict(eval_auc="exact", eval_capacity=capacity) if mode == "exact" else {}
  step = DLRMTrainStep(model, lr=0.3, use_cuda_graph=True, **kw)

  def batch(b, s):
    num, cat, lab = _gpu_batch(model.table_sizes, MLPERF_LIKE, b, s)
    return num, cat, lab, (num, cat)
  return model, step, batch


@pytest.mark.gpu
@pytest.mark.parametrize("arch", ["dot", "dcnv2"])
def test_step_exact_auc(arch):
  from test_dlrm_eval import _check_snapshot, _snapshot
  setup = _dot_setup if arch == "dot" else _dcn_setup
  b = 256
  n = 3 * b + 77  # four chunks, the last one short
  model, step, batch = setup("exact", capacity=n)
  for s in range(3):
    num, cat, lab, _ = batch(b, s)
    step.step(num, cat, lab)
  torch.cuda.synchronize()
  before = _snapshot(model, step)
  num, cat, lab, inp = batch(n, 50)
  step.evaluate(num, cat, lab)
  probs = step.predict(*inp)  # leaves the keys untouched
  met = step.eval_metrics(reset=False)
  torch.cuda.synchronize()
  _check_snapshot(before, _snapshot(model, step), "exact evaluate / predict / eval_metrics")
  assert set(met) == {"auc", "binned_auc", "tie_bound", "log_loss", "samples"}
  assert met["samples"] == n and int(step.exact_auc.state[0]) == n
  want = auc_counts_from_keys(auc_keys(probs, lab))
  assert step.exact_auc.counts() == want
  assert met["auc"] == auc_from_counts(*want)
  assert abs(met["auc"] - binary_auc(lab, probs)) <= 1e-12
  assert abs(met["binned_auc"] - met["auc"]) <= met["tie_bound"] + 1e-12
  assert step.eval_metrics() == met  # reset=True clears the keys with the other metrics
  assert int(step.exact_auc.state[0]) == 0
  after = step.eval_metrics()
  assert after["samples"] == 0 and math.isnan(after["auc"])
  # the binned-mode step reports the same binned value and no exact one
  _, ref, _ = setup("binned", capacity=None)
  for s in range(3):
    ref.step(*batch(b, s)[:3])
  ref.evaluate(num, cat, lab)
  rmet = ref.eval_metrics()
  assert set(rmet) == {"auc", "tie_bound", "log_loss", "samples"}
  assert rmet["samples"] == n
  # more samples than eval_capacity: raises with the counts
  step.evaluate(num, cat, lab)
  small = batch(10, 51)
  step.evaluate(*small[:3])
  with pytest.raises(RuntimeError, match=f"{n + 10} samples .* holds {n}"):
    step.eval_metrics()


@pytest.mark.gpu
def test_step_exact_eval_between_training_steps():
  """An exact-mode evaluation between training steps leaves everything a training step owns
  bit for bit as it was, so the following steps see the state a run without it would see; the
  following losses match such a run (to the float-atomic tolerance of test_dlrm_eval)."""
  from test_dlrm_eval import _check_snapshot, _snapshot
  losses = []
  for with_eval in (True, False):
    model, step, batch = _dot_setup("exact" if with_eval else "binned", capacity=2000, seed=3)
    ls = [float(step.step(*batch(256, 40 + i)[:3])) for i in range(3)]
    if with_eval:
      torch.cuda.synchronize()
      before = _snapshot(model, step)
      num, cat, lab, _ = batch(384, 99)
      step.evaluate(num, cat, lab)
      step.eval_metrics()
      torch.cuda.synchronize()
      _check_snapshot(before, _snapshot(model, step), "exact evaluation")
    ls += [float(step.step(*batch(256, 40 + i)[:3])) for i in range(3, 6)]
    losses.append(ls)
  assert losses[0] == pytest.approx(losses[1], rel=1e-5)


@pytest.mark.gpu
def test_step_rejects_bad_eval_auc_arguments():
  from distributed_embeddings_b200.models.dlrm import DLRM
  from distributed_embeddings_b200.models.dlrm_fast import DLRMTrainStep
  model = DLRM([300] * 4, embedding_dim=32, bottom_mlp_dims=(64, 32), top_mlp_dims=(128, 64, 1),
               device=torch.device("cuda", 0), backend="fused")
  with pytest.raises(ValueError, match="eval_auc must be"):
    DLRMTrainStep(model, eval_auc="roc")
  with pytest.raises(ValueError, match="needs eval_capacity"):
    DLRMTrainStep(model, eval_auc="exact")
