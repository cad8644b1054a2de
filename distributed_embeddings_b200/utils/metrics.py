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
