"""HBM row cache of host-offloaded embedding tables (``DistributedEmbedding(offload_cache_size=)``).

Tables that ``gpu_embedding_size`` puts in pinned host memory are read and updated by the fused
kernels zero-copy over PCIe.  With a cache, each step first moves the rows it touches into HBM
(``ops/csrc/offload_cache.cu``); the lookup and the sorted update then run on the cache arrays.

Policy (:class:`CachePolicy` is the reference the kernels are tested against, bit for bit):

* ``n_sets`` sets of 32 ways; the set of a row is :func:`cache_set`, a fixed integer hash of the
  row mod ``n_sets``.  Every way has a tag (row or -1), a last-use tick and a dirty bit.
* A pass advances the tick by one.  It first writes the dirty rows of the previous pass's spill
  region back to the host and empties it.  Then, over the unique rows of the step:
  a hit refreshes its way's tick; a set's misses, in ascending row order, take its least recently
  used ways (ties by way index), never a way used in this tick.  A dirty victim is written back
  before its way is refilled.  Misses a set cannot take go to spill slot ``n_sets * 32 + u``
  (``u``: the row's index among the step's unique rows, ascending), so every id has an HBM slot.
* A training pass marks every slot it touches dirty; a forward-only pass marks nothing (a filled
  slot starts clean).

Memory per cached table: ``(n_sets * 32 + n_spill)`` rows of weight and optimizer state, plus 12
bytes of tag / dirty per slot and 4 bytes of tick per way.  ``n_spill`` is the static bound on
unique rows per step: the sum of owner-side batch x hotness over the table's cached inputs.
"""
from __future__ import annotations

from typing import Dict, List, Sequence, Tuple

import numpy as np
import torch

WAYS = 32
_M64 = (1 << 64) - 1


def cache_set(row: int, n_sets: int) -> int:
  """Set of a host row (the same mixing as ``cache_set`` in ``offload_cache.cu``)."""
  x = int(row) & _M64
  x ^= x >> 33
  x = (x * 0xff51afd7ed558ccd) & _M64
  x ^= x >> 33
  return x % int(n_sets)


def cache_geometry(budget_rows: int) -> int:
  """Number of sets for a budget of ``budget_rows`` cached rows (at least one set)."""
  return max(1, int(budget_rows) // WAYS)


def split_budget(budget_elems: int, tables: Sequence[Tuple[int, int]]) -> List[int]:
  """Sets per table for an element budget split over ``tables`` = [(rows, width)] in
  proportion to their rows."""
  total = sum(r for r, _ in tables)
  out = []
  for rows, width in tables:
    share = budget_elems * rows // max(total, 1)
    out.append(cache_geometry(min(share // max(width, 1), rows)))
  return out


def cache_bytes(n_sets: int, n_spill: int, width: int, state_widths: Sequence[int]) -> int:
  """HBM bytes of one table's cache: weight and state rows of every slot, tags, dirty, ticks."""
  slots = n_sets * WAYS + n_spill
  return slots * 4 * (width + sum(state_widths)) + slots * (8 + 4) + n_sets * WAYS * 4 + 4 + 32


class CachePolicy:
  """Python reference of one table's cache state and pass (tags, ticks, dirty bits)."""

  def __init__(self, n_sets: int, n_spill: int):
    self.n_sets, self.n_spill = int(n_sets), int(n_spill)
    slots = self.n_sets * WAYS + self.n_spill
    self.tags = np.full(slots, -1, dtype=np.int64)
    self.ticks = np.zeros(self.n_sets * WAYS, dtype=np.int32)
    self.dirty = np.zeros(slots, dtype=np.int32)
    self.tick = 0
    self.stats = {"hits": 0, "misses": 0, "spills": 0, "writebacks": 0}

  def step(self, rows, train: bool):
    """One pass over the rows a step touches (any order, duplicates allowed; rows < 0 are
    out-of-shard ids).  Returns ``(slot_of, writebacks, fills)``: the slot of every unique row,
    ``[(slot, row)]`` written back to the host (spill region first, then victims) and
    ``[(slot, row)]`` filled from it."""
    now = self.tick + 1
    base = self.n_sets * WAYS
    writebacks, fills = [], []
    for s in range(base, base + self.n_spill):
      if self.tags[s] >= 0:
        if self.dirty[s]:
          writebacks.append((s, int(self.tags[s])))
          self.stats["writebacks"] += 1
        self.tags[s], self.dirty[s] = -1, 0
    uniq = sorted({int(r) for r in rows if int(r) >= 0})
    if len(uniq) > self.n_spill:
      raise ValueError("more unique rows than spill slots")
    slot_of: Dict[int, int] = {}
    misses: Dict[int, List[Tuple[int, int]]] = {}
    for u, row in enumerate(uniq):
      st = cache_set(row, self.n_sets)
      ways = np.nonzero(self.tags[st * WAYS:(st + 1) * WAYS] == row)[0]
      if len(ways):
        slot = st * WAYS + int(ways[0])
        self.ticks[slot] = now
        if train:
          self.dirty[slot] = 1
        slot_of[row] = slot
        self.stats["hits"] += 1
      else:
        misses.setdefault(st, []).append((u, row))
    for st in sorted(misses):
      lst = misses[st]
      ways = [w for w in range(WAYS) if self.ticks[st * WAYS + w] != now]
      ways.sort(key=lambda w: (int(self.ticks[st * WAYS + w]), w))
      self.stats["misses"] += len(lst)
      for i, (u, row) in enumerate(lst):
        if i < len(ways):
          slot = st * WAYS + ways[i]
          old = int(self.tags[slot])
          if old >= 0 and self.dirty[slot]:
            writebacks.append((slot, old))
            self.stats["writebacks"] += 1
          self.ticks[slot] = now
        else:
          slot = base + u
          self.stats["spills"] += 1
        self.tags[slot] = row
        self.dirty[slot] = 1 if train else 0
        slot_of[row] = slot
        fills.append((slot, row))
    self.tick = now
    return slot_of, writebacks, fills

  def flush(self) -> List[Tuple[int, int]]:
    out = [(int(s), int(self.tags[s])) for s in np.nonzero((self.tags >= 0) & (self.dirty != 0))[0]]
    self.dirty[:] = 0
    self.stats["writebacks"] += len(out)
    return out


class OffloadCache:
  """Device state of one cached table: HBM weight / optimizer-state rows of every slot, the
  policy words, and the host table it caches (pinned, addressed through its UVA mapping)."""

  def __init__(self, host_weight: torch.Tensor, n_sets: int, n_spill: int, device, ptr):
    self.host_weight = host_weight
    self.rows, self.width = int(host_weight.shape[0]), int(host_weight.shape[1])
    self.n_sets, self.n_spill = int(n_sets), int(n_spill)
    self.slots = self.n_sets * WAYS + self.n_spill
    self.device = device
    self._ptr = ptr
    self.weight = torch.zeros(self.slots, self.width, dtype=torch.float32, device=device)
    self.tags = torch.full((self.slots,), -1, dtype=torch.int64, device=device)
    self.ticks = torch.zeros(self.n_sets * WAYS, dtype=torch.int32, device=device)
    self.dirty = torch.zeros(self.slots, dtype=torch.int32, device=device)
    self.tick_word = torch.zeros(1, dtype=torch.int32, device=device)
    self.stats = torch.zeros(4, dtype=torch.int64, device=device)
    self.host_state: List[torch.Tensor] = []
    self.state: List[torch.Tensor] = []

  def set_state(self, host_state: Sequence[torch.Tensor]):
    """Optimizer-state tensors of the host table (cached alongside its rows).  Call only on an
    empty cache (after :meth:`invalidate`)."""
    self.host_state = list(host_state)
    self.state = [torch.zeros((self.slots,) + tuple(s.shape[1:]), dtype=torch.float32,
                              device=self.device) for s in self.host_state]

  def tensors(self) -> List[torch.Tensor]:
    empty = torch.empty(0, dtype=torch.float32, device=self.device)
    st = self.state + [empty] * (2 - len(self.state))
    return [self.weight, st[0], st[1], self.tags, self.ticks, self.dirty, self.tick_word,
            self.stats]

  def host_ptrs(self) -> List[int]:
    hs = [self._ptr(s) for s in self.host_state]
    return [self._ptr(self.host_weight)] + hs + [0] * (2 - len(hs))

  def flush(self, ops):
    ops.offload_cache_flush(self.tensors(), self.host_ptrs(), self.n_sets, self.n_spill,
                            self.rows)

  def invalidate(self):
    self.tags.fill_(-1)
    self.ticks.zero_()
    self.dirty.zero_()
    self.tick_word.zero_()

  def hbm_bytes(self) -> int:
    return cache_bytes(self.n_sets, self.n_spill, self.width,
                       [int(np.prod(s.shape[1:])) for s in self.state])

  def read_stats(self, reset: bool) -> Dict[str, int]:
    v = self.stats.tolist()
    if reset:
      self.stats.zero_()
    return dict(zip(("hits", "misses", "spills", "writebacks"), (int(x) for x in v)))
