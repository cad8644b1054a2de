"""Sharding planner for hybrid-parallel embeddings.

The planner is pure Python and deterministic: every rank computes the *global* plan, so no
communication is needed to agree on where a table (or a column / row slice of it) lives.

Behavioural parity target: ``DistEmbeddingStrategy`` of the reference
(``distributed_embeddings/python/layers/dist_model_parallel.py:301-709``).  The observable
outputs (``table_ids``, ``input_ids_list``, ``local_maps``, ``local_configs``, ``rev_tp_ids``,
``sliced_out_ranges`` ...) match the golden vectors in SURVEY.md Appendix A.  The implementation
is organised differently: every placed piece of a table is an explicit :class:`Shard` that
carries its own column range, so weight slicing (set/get_weights) and the device-side routing
descriptors are derived from the shards instead of being re-derived from slice counts.
"""
from __future__ import annotations

import copy
import hashlib
import json
from dataclasses import dataclass
from typing import Any, Dict, List, Optional, Sequence

STRATEGIES = ("basic", "memory_balanced", "memory_optimized", "traffic_balanced")


def _numel(cfg: Dict[str, Any]) -> int:
  return int(cfg["input_dim"]) * int(cfg["output_dim"])


@dataclass
class Shard:
  """One placed piece of a table-parallel (column group) table on one rank."""
  table: int  # id inside the column group
  rank: int
  rows: int
  col_start: int
  col_end: int
  local_table: int = -1  # index of the (fused) local table on the owning rank
  row_offset: int = 0  # first row of this shard inside the fused local table
  cpu_offload: bool = False

  @property
  def width(self) -> int:
    return self.col_end - self.col_start


@dataclass
class OutputPiece:
  """Where one (owner rank, local input) result lands in the requester's output.

  ``group_input`` is the position of the input inside the column group; ``col_offset`` is the
  first output column this piece fills inside that input's (concatenated) output.
  """
  rank: int
  local_input: int
  group_input: int
  col_offset: int
  width: int


class DistEmbeddingStrategy:
  """Compute the global distribution of embedding tables over ``world_size`` ranks.

  Args:
    embeddings: list of embedding layer objects exposing ``get_config()`` (with at least
      ``input_dim`` and ``output_dim``), or plain config dicts.
    world_size: number of model-parallel workers.
    strategy: ``basic`` (round robin) | ``memory_balanced`` (size-sorted snake, even table
      count) | ``memory_optimized`` (greedy least-loaded memory) | ``traffic_balanced`` (greedy
      least-loaded *work*: ids looked up x slice width, i.e. the bytes a rank gathers and sends
      per step; not in the reference - with multi-hot features the size-based placements leave
      the busiest rank of the synthetic models with 2-2.5x the mean work).
    input_table_map: ``input[i]`` reads ``table[input_table_map[i]]``; None = identity.
    column_slice_threshold: tables with more elements are split along width into the smallest
      power-of-two number of slices that brings each slice under the threshold.
    row_slice_threshold: tables with at least this many elements are split by rows onto all
      ranks.
    data_parallel_threshold: tables with at most this many elements are replicated.
    gpu_embedding_size: per-rank element budget for table-parallel tables kept in HBM; the
      largest tables beyond it are placed in host memory.
    input_hotness: ids per sample of every input (default 1); only ``traffic_balanced`` uses it.

  Attributes mirror the reference (DMP:319-345) so that user code such as
  ``strategy.input_ids_list[rank]`` keeps working.
  """

  def __init__(self,
               embeddings: Sequence[Any],
               world_size: int,
               strategy: str = "basic",
               input_table_map: Optional[Sequence[int]] = None,
               column_slice_threshold: Optional[int] = None,
               row_slice_threshold: Optional[int] = None,
               data_parallel_threshold: Optional[int] = None,
               gpu_embedding_size: Optional[int] = None,
               input_hotness: Optional[Sequence[int]] = None):
    if strategy not in STRATEGIES:
      raise ValueError(f"Unsupported shard strategy {strategy}")
    self.world_size = int(world_size)
    # a single worker always round-robins (i.e. keeps table order), reference DMP:357
    self.strategy = "basic" if self.world_size == 1 else strategy
    self.column_slice_threshold = column_slice_threshold
    self.row_slice_threshold = row_slice_threshold
    self.data_parallel_threshold = data_parallel_threshold
    self.gpu_embedding_size = gpu_embedding_size

    self.global_configs: List[Dict[str, Any]] = []
    for emb in embeddings:
      cfg = dict(emb) if isinstance(emb, dict) else dict(emb.get_config())
      cfg.setdefault("layer_type", None if isinstance(emb, dict) else type(emb))
      self.global_configs.append(cfg)
    if input_table_map is None:
      input_table_map = list(range(len(self.global_configs)))
    self.input_table_map = [int(t) for t in input_table_map]
    if input_hotness is None:
      input_hotness = [1] * len(self.input_table_map)
    if len(input_hotness) != len(self.input_table_map):
      raise ValueError("input_hotness needs one entry per input")
    self.input_hotness = [max(1, int(h)) for h in input_hotness]

    self.table_groups = self._group_tables()
    self.input_groups, self.map_groups, self.rev_group_ids = self._group_inputs()

    # group 0: replicated tables
    self.dp_configs = [copy.copy(self.global_configs[t]) for t in self.table_groups[0]]

    # group 2: row slices on every rank
    self.row_sliced_configs: List[List[Dict[str, Any]]] = [[] for _ in range(self.world_size)]
    self.row_inputs_offsets: List[List[int]] = [[] for _ in range(self.world_size)]
    self.row_ranges: List[List[List[int]]] = []  # [table][rank] -> [start, end)
    if self.table_groups[2]:
      self._plan_row_slices()

    # group 1: table parallel with optional column slicing
    self.sliced_out_ranges: List[List[int]] = []
    self.input_ids_list: List[List[int]] = [[] for _ in range(self.world_size)]
    self.local_maps: List[List[int]] = [[] for _ in range(self.world_size)]
    self.local_configs: List[List[Dict[str, Any]]] = [[] for _ in range(self.world_size)]
    self.local_input_offsets: List[List[int]] = [[] for _ in range(self.world_size)]
    self.local_weight_offsets: List[List[List[int]]] = [[] for _ in range(self.world_size)]
    self.local_group_list: List[List[List[int]]] = [[] for _ in range(self.world_size)]
    self.table_ids: List[List[int]] = [[] for _ in range(self.world_size)]
    self.widths_list_flat: List[int] = []
    self.rev_tp_ids: List[int] = []
    self.shards: List[List[Shard]] = [[] for _ in range(self.world_size)]
    self.output_pieces: List[OutputPiece] = []
    if self.table_groups[1]:
      self._plan_table_parallel()

  # ------------------------------------------------------------------ grouping
  def _group_tables(self) -> List[List[int]]:
    """Split table ids into [data-parallel, table/column-parallel, row-sliced] by size."""
    dp, col, row = [], [], []
    for i, cfg in enumerate(self.global_configs):
      n = _numel(cfg)
      if self.data_parallel_threshold and n <= self.data_parallel_threshold:
        dp.append(i)
      elif self.row_slice_threshold and n >= self.row_slice_threshold:
        row.append(i)
      else:
        col.append(i)
    return [dp, col, row]

  def _group_inputs(self):
    where = {}
    for g, tables in enumerate(self.table_groups):
      for pos, t in enumerate(tables):
        where[t] = (g, pos)
    inputs = [[], [], []]
    maps = [[], [], []]
    for i, t in enumerate(self.input_table_map):
      if t not in where:
        raise ValueError("Wrong input initializing input/map groups.")
      g, pos = where[t]
      inputs[g].append(i)
      maps[g].append(pos)
    flat = inputs[0] + inputs[1] + inputs[2]
    rev = sorted(range(len(flat)), key=lambda j: flat[j])
    return inputs, maps, rev

  # ------------------------------------------------------------------ row slicing
  def _plan_row_slices(self):
    per_table_cfgs, per_table_offs = [], []
    for t in self.table_groups[2]:
      cfg = self.global_configs[t]
      rows = int(cfg["input_dim"])
      base, rem = divmod(rows, self.world_size)
      start = 0
      cfgs, offs, ranges = [], [], []
      for r in range(self.world_size):
        n = base + (1 if r < rem else 0)
        c = copy.copy(cfg)
        c["input_dim"] = n
        cfgs.append(c)
        offs.append(-start)  # shifting ids makes foreign ids fall out of [0, n)
        ranges.append([start, start + n])
        start += n
      per_table_cfgs.append(cfgs)
      per_table_offs.append(offs)
      self.row_ranges.append(ranges)
    self.row_sliced_configs = [list(x) for x in zip(*per_table_cfgs)]
    self.row_inputs_offsets = [list(x) for x in zip(*per_table_offs)]

  # ------------------------------------------------------------------ column slicing
  @staticmethod
  def slice_widths(cfg: Dict[str, Any], threshold: Optional[float], world_size: int) -> List[int]:
    """Widths of the column slices of one table (a single entry = not sliced)."""
    if threshold is None:
      threshold = float("inf")
    size = float(_numel(cfg))
    n = 1
    while size > threshold:
      n *= 2
      size /= 2
    if n == 1:
      return [int(cfg["output_dim"])]
    n = min(n, world_size, int(cfg["output_dim"]))
    base, rem = divmod(int(cfg["output_dim"]), n)
    return [base + (1 if i < rem else 0) for i in range(n)]

  def _auto_threshold(self, configs) -> Optional[int]:
    """With fewer tables than workers, pick a threshold that yields >= world_size slices."""
    sizes = [_numel(c) for c in configs]
    threshold = None
    while self.world_size > len(sizes):
      sizes.sort()
      largest = sizes.pop()
      threshold = largest - 1
      sizes += [largest // 2, largest // 2]
    return threshold

  def _place(self, slice_table_ids: List[int], slice_sizes: List[int],
             slice_costs: Optional[List[int]] = None) -> List[List[int]]:
    """Distribute slices (identified by their table id) to ranks."""
    w = self.world_size
    if self.strategy == "traffic_balanced":
      # longest-processing-time greedy on the per-step work, memory as the tie breaker
      todo = sorted(zip(slice_costs, slice_sizes, slice_table_ids), reverse=True)
      bins = [[0, 0, r, []] for r in range(w)]  # work, memory, rank, tables
      for cost, size, t in todo:
        b = min(bins, key=lambda x: (x[0], x[1], x[2]))
        b[0] += cost
        b[1] += size
        b[3].append(t)
      return [b[3] for b in bins]
    if self.strategy == "basic":
      return [slice_table_ids[r::w] for r in range(w)]
    if self.strategy == "memory_balanced":
      order = [t for _, t in sorted(zip(slice_sizes, slice_table_ids), reverse=True)]
      return [order[r::2 * w] + order[2 * w - 1 - r::2 * w] for r in range(w)]
    if self.strategy == "memory_optimized":
      todo = sorted(zip(slice_sizes, slice_table_ids))
      bins = [[0, []] for _ in range(w)]
      while todo:
        size, t = todo.pop()
        bins[0][0] += size
        bins[0][1].append(t)
        bins.sort()
      return [b[1] for b in bins]
    raise ValueError(f"Unsupported strategy {self.strategy}")

  def _plan_table_parallel(self):
    col_tables = self.table_groups[1]
    col_map = self.map_groups[1]
    configs = [self.global_configs[t] for t in col_tables]
    threshold = self.column_slice_threshold
    if threshold is None:
      threshold = self._auto_threshold(configs)

    widths = [self.slice_widths(c, threshold, self.world_size) for c in configs]
    # per-sample work of every table of the group, in "rows of one column": every id is a row
    # gathered (and read-modify-written in the backward), every input one pooled vector out and
    # one gradient vector in over NVLink, worth about two row accesses each at HBM / NVLink rates
    lookups = [0] * len(configs)
    for k, t in enumerate(col_map):
      lookups[t] += self.input_hotness[self.input_groups[1][k]] + 2
    if self.strategy == "traffic_balanced" and self.world_size > 1:
      # a table whose work alone exceeds a rank's fair share is column sliced further (power of
      # two, slices stay >= 32 columns = one 128-byte row segment)
      fair = sum(lookups[t] * int(c["output_dim"]) for t, c in enumerate(configs)) / self.world_size
      for t, c in enumerate(configs):
        width, n = int(c["output_dim"]), len(widths[t])
        while lookups[t] * width / n > fair and 2 * n <= self.world_size and width // (2 * n) >= 32:
          n *= 2
        if n != len(widths[t]):
          base, rem = divmod(width, n)
          widths[t] = [base + (1 if i < rem else 0) for i in range(n)]
    flat_ids, flat_sizes, flat_costs = [], [], []
    for t, ws in enumerate(widths):
      for w_ in ws:
        flat_ids.append(t)
        flat_sizes.append(int(configs[t]["input_dim"]) * w_)
        flat_costs.append(lookups[t] * w_)
    placement = self._place(flat_ids, flat_sizes, flat_costs)

    # Hand out slices in rank order; slices of one table meeting on a rank are merged into one
    # wider shard.  Column ranges therefore grow with the rank, which is also the order in
    # which the pieces of an output are concatenated.
    remaining = [list(ws) for ws in widths]
    next_col = [0] * len(configs)
    for rank, ids in enumerate(placement):
      shards: List[Shard] = []
      for t in ids:
        w_ = remaining[t].pop(0)
        mine = next((s for s in shards if s.table == t), None)
        if mine is None:
          shards.append(
              Shard(table=t,
                    rank=rank,
                    rows=int(configs[t]["input_dim"]),
                    col_start=next_col[t],
                    col_end=next_col[t] + w_))
        else:
          mine.col_end += w_
        next_col[t] += w_
      self.shards[rank] = shards
      self.table_ids[rank] = [s.table for s in shards]

    # number of output pieces per table after merging
    pieces_per_table = [0] * len(configs)
    for shards in self.shards:
      for s in shards:
        pieces_per_table[s.table] += 1
    # ranges of consecutive outputs (progressively merged list) to concatenate, input order
    for k, t in enumerate(col_map):
      if len(widths[t]) > 1:
        self.sliced_out_ranges.append([k, k + pieces_per_table[t]])

    for rank, shards in enumerate(self.shards):
      rank_configs = []
      for s in shards:
        c = copy.copy(configs[s.table])
        c["output_dim"] = s.width
        rank_configs.append(c)
      # inputs served by this rank, grouped by local table order
      in_ids, in_map = [], []
      for m, s in enumerate(shards):
        for k, t in enumerate(col_map):
          if t == s.table:
            in_ids.append(k)
            in_map.append(m)
      self._mark_offload(rank_configs)
      for s, c in zip(shards, rank_configs):
        s.cpu_offload = c["cpu_offload"]
      fused, new_map, in_offsets, groups, w_offsets = self._fuse_tables(rank_configs, in_map)
      for gid, (group, offs) in enumerate(zip(groups, w_offsets)):
        for j, m in enumerate(group):
          shards[m].local_table = gid
          shards[m].row_offset = offs[j]
      self.input_ids_list[rank] = in_ids
      self.local_configs[rank] = fused
      self.local_maps[rank] = new_map
      self.local_input_offsets[rank] = in_offsets
      self.local_group_list[rank] = groups
      self.local_weight_offsets[rank] = w_offsets

    for cfgs, lmap in zip(self.local_configs, self.local_maps):
      self.widths_list_flat += [int(cfgs[m]["output_dim"]) for m in lmap]
    worker_order = [k for ids in self.input_ids_list for k in ids]
    self.rev_tp_ids = sorted(range(len(worker_order)), key=lambda j: (worker_order[j], j))

    # Explicit routing of every (rank, local input) result into the requester's output
    col_fill = [0] * len(col_map)
    by_input: Dict[int, List[OutputPiece]] = {}
    for rank, ids in enumerate(self.input_ids_list):
      for li, k in enumerate(ids):
        w_ = int(self.local_configs[rank][self.local_maps[rank][li]]["output_dim"])
        by_input.setdefault(k, []).append(
            OutputPiece(rank=rank, local_input=li, group_input=k, col_offset=0, width=w_))
    for k in range(len(col_map)):
      for p in by_input.get(k, []):  # already in rank order
        p.col_offset = col_fill[k]
        col_fill[k] += p.width
        self.output_pieces.append(p)
    self.col_output_widths = col_fill

  def _mark_offload(self, configs: List[Dict[str, Any]]):
    """Flag the largest tables for host placement once the HBM element budget is exceeded."""
    if self.gpu_embedding_size is None:
      for c in configs:
        c["cpu_offload"] = False
      return
    total = 0
    for i in sorted(range(len(configs)), key=lambda j: _numel(configs[j])):
      total += _numel(configs[i])
      configs[i]["cpu_offload"] = total > self.gpu_embedding_size

  @staticmethod
  def _fuse_tables(configs: List[Dict[str, Any]], input_map: List[int]):
    """Fuse local tables with equal width and combiner (and not offloaded) into one table.

    Returns (fused_configs, new_input_map, input_row_offsets, groups, weight_offsets).
    """
    groups: List[List[int]] = []
    fused: List[Dict[str, Any]] = []
    offsets: List[List[int]] = []
    for tid, cfg in enumerate(configs):
      for g, fc, offs in zip(groups, fused, offsets):
        if (cfg["output_dim"] == fc["output_dim"] and cfg.get("combiner") == fc.get("combiner") and
            not cfg["cpu_offload"] and not fc["cpu_offload"]):
          g.append(tid)
          fc["input_dim"] += cfg["input_dim"]
          fc["input_dims"].append(cfg["input_dim"])
          offs.append(offs[-1] + cfg["input_dim"])
          break
      else:
        groups.append([tid])
        fc = copy.copy(cfg)
        fc["input_dims"] = [cfg["input_dim"]]
        fused.append(fc)
        offsets.append([0, cfg["input_dim"]])
    new_map, in_offsets = [], []
    for m in input_map:
      for gid, g in enumerate(groups):
        if m in g:
          new_map.append(gid)
          in_offsets.append(offsets[gid][g.index(m)])
          break
    return fused, new_map, in_offsets, groups, offsets

  # ------------------------------------------------------------------ helpers
  def column_range(self, rank: int, local_shard: int) -> List[int]:
    s = self.shards[rank][local_shard]
    return [s.col_start, s.col_end]

  def fingerprint(self) -> str:
    """Stable hash of the plan; ranks compare it at init to detect mismatched plans."""
    desc = {
        "world": self.world_size,
        "groups": self.table_groups,
        "table_ids": self.table_ids,
        "inputs": self.input_ids_list,
        "maps": self.local_maps,
        "cfg": [[[c["input_dim"], c["output_dim"], bool(c.get("cpu_offload"))] for c in r]
                for r in self.local_configs],
        "row": [[[c["input_dim"], c["output_dim"]] for c in r] for r in self.row_sliced_configs],
        "ranges": self.sliced_out_ranges,
    }
    return hashlib.sha256(json.dumps(desc, sort_keys=True).encode()).hexdigest()

  def memory_report(self) -> List[Dict[str, int]]:
    """Per-rank element counts (HBM / host) of the model-parallel tables."""
    rep = []
    for r in range(self.world_size):
      hbm = sum(_numel(c) for c in self.local_configs[r] if not c.get("cpu_offload"))
      host = sum(_numel(c) for c in self.local_configs[r] if c.get("cpu_offload"))
      row = sum(_numel(c) for c in self.row_sliced_configs[r])
      dp = sum(_numel(c) for c in self.dp_configs)
      rep.append({"rank": r, "hbm_elements": hbm + row + dp, "host_elements": host})
    return rep

  def traffic_report(self, global_batch: int, hotness: Optional[Sequence[int]] = None,
                     activation_bytes: int = 2, id_bytes: int = 4) -> Dict[str, Any]:
    """Per-rank bytes per step implied by the plan (forward; the backward moves the same
    activation bytes in the other direction): rows gathered from the tables, pooled vectors
    leaving the rank over NVLink, ids pulled from the other ranks.  ``hotness[i]`` is the number
    of ids per sample of input ``i`` (default 1).  The step time of the embedding exchange is set
    by the most loaded rank, so ``imbalance`` (max / mean) is what a threshold search minimises.
    """
    w_ = self.world_size
    n_inputs = len(self.input_table_map)
    hot = [1] * n_inputs if hotness is None else [int(h) for h in hotness]
    if len(hot) != n_inputs:
      raise ValueError(f"expected {n_inputs} hotness values, got {len(hot)}")
    away = (w_ - 1) / w_ if w_ > 1 else 0.0
    local_batch = global_batch // w_
    ranks = [{"rank": r, "gather_bytes": 0.0, "nvlink_out_bytes": 0.0, "id_pull_bytes": 0.0,
              "lookups": 0.0} for r in range(w_)]
    # table-parallel / column-sliced: the owner looks up the global batch of its inputs
    for r in range(w_):
      for li, gi_group in enumerate(self.input_ids_list[r] if self.table_groups[1] else []):
        gi = self.input_groups[1][gi_group]
        width = int(self.local_configs[r][self.local_maps[r][li]]["output_dim"])
        n_ids = global_batch * hot[gi]
        ranks[r]["lookups"] += n_ids
        ranks[r]["gather_bytes"] += n_ids * width * 4
        ranks[r]["nvlink_out_bytes"] += global_batch * width * activation_bytes * away
        ranks[r]["id_pull_bytes"] += n_ids * id_bytes * away
    # row-sliced: every rank sees all ids, gathers its share, sends fp32 partial pools
    for j, gi in enumerate(self.input_groups[2]):
      t = self.table_groups[2][self.map_groups[2][j]]
      width = int(self.global_configs[t]["output_dim"])
      n_ids = global_batch * hot[gi]
      for r in range(w_):
        ranks[r]["lookups"] += n_ids / w_
        ranks[r]["gather_bytes"] += n_ids / w_ * width * 4
        ranks[r]["nvlink_out_bytes"] += global_batch * width * 4 * away
        ranks[r]["id_pull_bytes"] += n_ids * id_bytes * away
    # replicated: local batch only, nothing on the wire
    for j, gi in enumerate(self.input_groups[0]):
      t = self.table_groups[0][self.map_groups[0][j]]
      width = int(self.global_configs[t]["output_dim"])
      for r in range(w_):
        ranks[r]["lookups"] += local_batch * hot[gi]
        ranks[r]["gather_bytes"] += local_batch * hot[gi] * width * 4

    def imbalance(key):
      vals = [x[key] for x in ranks]
      mean = sum(vals) / len(vals)
      return max(vals) / mean if mean > 0 else 1.0

    return {"ranks": ranks,
            "max_gather_bytes": max(x["gather_bytes"] for x in ranks),
            "max_nvlink_out_bytes": max(x["nvlink_out_bytes"] for x in ranks),
            "gather_imbalance": imbalance("gather_bytes"),
            "nvlink_imbalance": imbalance("nvlink_out_bytes")}


def suggest_column_slice_threshold(embeddings: Sequence[Any], world_size: int,
                                   strategy: str = "memory_balanced",
                                   input_table_map: Optional[Sequence[int]] = None,
                                   hotness: Optional[Sequence[int]] = None,
                                   min_slice_width: int = 64, **plan_kwargs) -> Optional[int]:
  """Column-slice threshold (``None`` or a power of two) that minimises the bytes the most
  loaded rank gathers and sends per step (``traffic_report``), keeping every slice at least
  ``min_slice_width`` columns wide (narrow slices waste the 128-byte vector accesses of the
  lookup kernels).  What ``column_slice_threshold="auto"`` of ``DistributedEmbedding`` uses."""
  best, best_cost = None, None
  for thr in [None] + [2**k for k in range(34, 22, -1)]:
    try:
      st = DistEmbeddingStrategy(embeddings, world_size, strategy, input_table_map=input_table_map,
                                 column_slice_threshold=thr, **plan_kwargs)
    except ValueError:
      continue
    if st.table_groups[1] and any(not st.local_configs[r] for r in range(world_size)):
      continue
    widths = [int(c["output_dim"]) for r in range(world_size) for c in st.local_configs[r]]
    full = [int(c["output_dim"]) for c in st.global_configs]
    if widths and min(widths) < min(min_slice_width, min(full)):
      continue
    rep = st.traffic_report(world_size * 1024, hotness)
    cost = (rep["max_nvlink_out_bytes"], rep["max_gather_bytes"])
    if best_cost is None or cost < best_cost:
      best, best_cost = thr, cost
  return best

