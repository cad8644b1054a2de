"""Evaluation metrics and structured logging helpers."""
from __future__ import annotations

import json
import time
from typing import Any, Dict, NamedTuple

import numpy as np
import torch


def binary_auc(labels: torch.Tensor, scores: torch.Tensor) -> float:
  """Exact ROC AUC by rank statistics (ties get the average rank).

  The reference example uses a Keras AUC metric with 8000 thresholds (examples/dlrm/main.py:
  223-243); the exact value is cheaper and deterministic."""
  labels = labels.reshape(-1).double()
  scores = scores.reshape(-1).double()
  n_pos = float(labels.sum())
  n_neg = float(labels.numel() - n_pos)
  if n_pos == 0 or n_neg == 0:
    return float("nan")
  order = torch.argsort(scores)
  s = scores[order]
  ranks = torch.arange(1, s.numel() + 1, dtype=torch.float64)
  # average ranks over ties
  uniq, inv, counts = torch.unique_consecutive(s, return_inverse=True, return_counts=True)
  ends = torch.cumsum(counts, 0).double()
  starts = ends - counts.double() + 1
  avg = ((starts + ends) / 2)[inv]
  pos_rank_sum = float(avg[labels[order] > 0.5].sum())
  return (pos_rank_sum - n_pos * (n_pos + 1) / 2) / (n_pos * n_neg)


class AUCResult(NamedTuple):
  auc: float        # trapezoidal ROC AUC over the threshold grid (NaN when a class is empty)
  tie_bound: float  # |auc - exact AUC| <= tie_bound: half the share of pairs that share a bucket


def auc_from_histogram(hist) -> AUCResult:
  """ROC AUC of a ``[2, T - 1]`` histogram (row 0 negatives, row 1 positives), in float64.

  Equals the trapezoid over the ``T`` threshold points, i.e. Mann-Whitney over bucket indices
  with ties counted as one half: ``(sum_k pos_k neg_<k + 1/2 sum_k pos_k neg_k) / (P N)``."""
  h = np.asarray(torch.as_tensor(hist).detach().cpu().to(torch.float64))
  neg, pos = h[0], h[1]
  n_neg, n_pos = float(neg.sum()), float(pos.sum())
  if n_neg == 0 or n_pos == 0:
    return AUCResult(float("nan"), float("nan"))
  neg_below = np.cumsum(neg) - neg
  tied = float(np.dot(pos, neg))
  auc = (float(np.dot(pos, neg_below)) + 0.5 * tied) / (n_pos * n_neg)
  return AUCResult(auc, 0.5 * tied / (n_pos * n_neg))


class BinnedAUC:
  """Streaming ROC AUC over ``num_thresholds`` evenly spaced thresholds, the metric the reference
  example reports (``tf.keras.metrics.AUC(num_thresholds=8000, curve='ROC',
  summation_method='interpolation')``), kept as a histogram so it accumulates on the device.

  ``hist`` (int64 ``[2, T - 1]``): row 0 counts negatives, row 1 positives (label > 0.5), one
  column per bucket between neighbouring thresholds.  A prediction ``p`` in [0, 1] falls into
  bucket ``k(p) = clamp(ceil(fp32(p * (T - 1))) - 1, 0, T - 2)``: the number of interior
  thresholds ``i / (T - 1)`` (``i = 1 .. T - 2``) strictly below ``p``.  That is Keras's ``p > t``
  rule with outer thresholds ``-1e-7`` and ``1 + 1e-7``, except for a ``p`` within one fp32
  rounding of a threshold.  The DLRM evaluation kernel (``head_eval``) adds into the same tensor
  with the same rule."""

  def __init__(self, num_thresholds: int = 8000, device=None):
    if int(num_thresholds) < 2:
      raise ValueError("num_thresholds must be >= 2")
    self.num_thresholds = int(num_thresholds)
    self.hist = torch.zeros(2, self.num_thresholds - 1, dtype=torch.int64, device=device)

  def bucket(self, probs: torch.Tensor) -> torch.Tensor:
    """Bucket index of every prediction (int64, same shape)."""
    nb = self.num_thresholds - 1
    k = torch.ceil(probs.float() * float(nb)) - 1
    return k.clamp_(0, nb - 1).long()

  def update(self, probs: torch.Tensor, labels: torch.Tensor):
    """Add a batch of predictions in [0, 1] and their labels (any device)."""
    nb = self.num_thresholds - 1
    p = probs.reshape(-1).to(self.hist.device)
    y = labels.reshape(-1).to(self.hist.device)
    if p.numel() != y.numel():
      raise ValueError("probs and labels must have the same number of elements")
    key = self.bucket(p) + (y > 0.5).long() * nb
    self.hist.view(-1).add_(torch.bincount(key, minlength=2 * nb))

  def reset(self):
    self.hist.zero_()

  def all_reduce(self, group=None):
    """Sum ``hist`` over the ranks of ``group`` (collective)."""
    import torch.distributed as dist
    dist.all_reduce(self.hist, group=group)

  def result(self) -> AUCResult:
    """``(auc, tie_bound)`` of the accumulated histogram (host float64)."""
    return auc_from_histogram(self.hist)


def auc_keys(probs, labels) -> np.ndarray:
  """Exact-AUC keys ``(bits(p) << 1) | (y > 0.5)`` (uint32, below 2^31) of fp32 probabilities in
  [0, 1]; -0.0 is keyed as 0.0.  Raises on a probability that is NaN or outside [0, 1]."""
  p = np.ascontiguousarray(np.asarray(torch.as_tensor(probs).detach().cpu().float()).reshape(-1))
  y = np.asarray(torch.as_tensor(labels).detach().cpu().float()).reshape(-1)
  if p.size != y.size:
    raise ValueError("probs and labels must have the same number of elements")
  bad = int(np.count_nonzero(~((p >= 0) & (p <= 1))))
  if bad:
    raise ValueError(f"{bad} probabilities are NaN or outside [0, 1]")
  bits = p.view(np.uint32) & np.uint32(0x7FFFFFFF)
  return (bits << np.uint32(1)) | (y > 0.5).astype(np.uint32)


def auc_counts_from_keys(keys) -> tuple:
  """``(P, N, U2)`` of exact-AUC keys (any order), with numpy integers: ``U2`` is twice the
  Mann-Whitney U of the positives' scores over the negatives' (ties count one half),
  ``sum over positives j of 2 #{neg: p < p_j} + #{neg: p == p_j}``."""
  k = np.sort(np.asarray(keys).astype(np.uint32).reshape(-1))
  n = k.size
  if n == 0:
    return 0, 0, 0
  neg = (1 - (k & 1)).astype(np.int64)
  np_before = np.cumsum(neg) - neg  # negatives before each position: score <= its own
  score = k >> 1
  head = np.ones(n, dtype=bool)
  head[1:] = score[1:] != score[:-1]
  run_start = np.maximum.accumulate(np.where(head, np.arange(n), 0))
  pos = neg == 0
  # negatives before the score run: score strictly below
  u2 = int(np_before[pos].sum()) + int(np_before[run_start[pos]].sum())
  n_neg = int(neg.sum())
  return n - n_neg, n_neg, u2


def auc_from_counts(n_pos: int, n_neg: int, u2: int) -> float:
  """``U2 / (2 P N)`` in float64; NaN when a class is empty."""
  if n_pos == 0 or n_neg == 0:
    return float("nan")
  return u2 / (2 * n_pos * n_neg)


class ExactAUC:
  """Exact ROC AUC (Mann-Whitney, ties count one half) over every sample since the last reset,
  accumulated without floating-point sums: each sample is kept as one 31-bit key (4 bytes, see
  :func:`auc_keys`) in a ``capacity``-key buffer, and :meth:`counts` sorts the keys and counts
  ``(P, N, U2)`` in 64-bit integers.  The value equals :func:`binary_auc`.

  On CUDA, :meth:`update` is one ``auc_append`` kernel with the sample count and every offset on
  the device (it replays inside a CUDA graph), and :meth:`counts` runs the first-party radix sort
  and ``auc_count``; they need ``4 * n`` bytes of temporary space for ``n`` keys.  On CPU the same
  integers come from a numpy sort (the reference the kernels are tested against).

  ``state`` (int64): ``[keys stored, samples dropped because they would pass capacity, samples
  whose probability is NaN or outside [0, 1], kernel ticket]``.  Overflow drops the whole update
  (nothing is written past the buffer) and a bad probability is not stored; either makes
  :meth:`counts` and :meth:`result` raise until :meth:`reset`."""

  def __init__(self, capacity: int, device=None):
    if int(capacity) < 1:
      raise ValueError("capacity must be >= 1")
    self.capacity = int(capacity)
    self.keys = torch.zeros(self.capacity, dtype=torch.int32, device=device)
    self.state = torch.zeros(4, dtype=torch.int64, device=device)

  def update(self, probs: torch.Tensor, labels: torch.Tensor, n_valid=None):
    """Append the first ``n_valid`` (default all) predictions in [0, 1] and their labels.  On
    CUDA ``n_valid`` may be an int64 device word, read by the kernel."""
    p = probs.reshape(-1)
    y = labels.reshape(-1)
    if p.numel() != y.numel():
      raise ValueError("probs and labels must have the same number of elements")
    if self.keys.is_cuda:
      from ..ops import _native
      if not isinstance(n_valid, torch.Tensor):
        n = p.numel() if n_valid is None else int(n_valid)
        n_valid = torch.full((1,), n, dtype=torch.int64, device=self.keys.device)
      _native.require().auc_append(p.float().contiguous(), y.float().contiguous(), n_valid,
                                   self.keys, self.state)
      return
    n = p.numel() if n_valid is None else int(n_valid)
    n = max(0, min(n, p.numel()))
    p, y = p[:n].float().numpy(), y[:n].float().numpy()
    ok = (p >= 0) & (p <= 1)
    self.state[2] += int(np.count_nonzero(~ok))
    count = int(self.state[0])
    if count + n > self.capacity:
      self.state[1] += n
      return
    keys = auc_keys(np.where(ok, p, 0).astype(np.float32), y)
    self.keys[count:count + n] = torch.from_numpy(keys.view(np.int32))
    self.state[0] = count + n

  def reset(self):
    self.state.zero_()

  def all_gather(self, group=None):
    """Collective: afterwards every rank of ``group`` holds every rank's keys (counts may differ
    between ranks) and the summed dropped / bad counts.  The buffers are replaced by new ones of
    ``max(capacity, total keys)`` keys, so a CUDA graph that appends to the old ones no longer
    reaches this object."""
    import torch.distributed as dist
    world = dist.get_world_size(group)
    st = self.state[:3].clone()
    states = [torch.empty_like(st) for _ in range(world)]
    dist.all_gather(states, st, group=group)
    states = torch.stack(states).cpu()
    counts = [int(c) for c in states[:, 0]]
    width = max(max(counts), 1)
    send = torch.zeros(width, dtype=torch.int32, device=self.keys.device)
    send[:counts[dist.get_rank(group)]] = self.keys[:counts[dist.get_rank(group)]]
    recv = [torch.empty_like(send) for _ in range(world)]
    dist.all_gather(recv, send, group=group)
    total = sum(counts)
    self.capacity = max(self.capacity, total)
    keys = torch.zeros(self.capacity, dtype=torch.int32, device=self.keys.device)
    keys[:total] = torch.cat([r[:c] for r, c in zip(recv, counts)])
    state = torch.zeros(4, dtype=torch.int64, device=self.state.device)
    state[:3] = states.sum(0).to(state.device)
    self.keys, self.state = keys, state

  def counts(self) -> tuple:
    """``(P, N, U2)`` over the stored keys (host ints).  Raises when samples were dropped for
    lack of capacity or a probability was NaN or outside [0, 1]."""
    stored, dropped, bad = (int(v) for v in self.state[:3].tolist())
    if dropped:
      raise RuntimeError(
          f"ExactAUC overflow: {stored + dropped} samples were evaluated but the key buffer holds "
          f"{self.capacity}; {dropped} were not stored (raise the capacity)")
    if bad:
      raise RuntimeError(
          f"ExactAUC: {bad} of {stored + dropped} probabilities were NaN or outside [0, 1] "
          f"(capacity {self.capacity})")
    if not self.keys.is_cuda:
      return auc_counts_from_keys(self.keys[:stored].numpy())
    from ..ops import _native
    ops = _native.require()
    out = torch.zeros(3, dtype=torch.int64, device=self.keys.device)
    ops.radix_sort_keys32(self.keys, stored, 31)  # in place: the order of the keys is free
    ops.auc_count(self.keys, stored, out)
    return tuple(int(v) for v in out.tolist())

  def result(self) -> float:
    """Exact ROC AUC in float64 (NaN when a class is empty)."""
    return auc_from_counts(*self.counts())


class MetricsLogger:
  """Structured (JSON lines) metrics: one record per call, rank-0 only by default."""

  def __init__(self, path=None, rank: int = 0, enabled_ranks=(0,)):
    self.path, self.rank, self.enabled = path, rank, rank in enabled_ranks
    self.t0 = time.time()

  def log(self, **record: Any) -> Dict[str, Any]:
    record = {"t": round(time.time() - self.t0, 3), "rank": self.rank, **record}
    if self.enabled:
      line = json.dumps(record)
      if self.path:
        with open(self.path, "a", encoding="utf-8") as f:
          f.write(line + "\n")
      else:
        print(line, flush=True)
    return record


def bus_bandwidth_gbs(bytes_per_rank_out: float, seconds: float) -> float:
  """All-to-all bus bandwidth per GPU (bytes leaving one GPU / time)."""
  return bytes_per_rank_out / max(seconds, 1e-12) / 1e9
