"""Planner tests against golden vectors (SURVEY.md Appendix A: produced by running the
reference's own DistEmbeddingStrategy, dist_model_parallel.py:301-709)."""
import pytest

from distributed_embeddings_b200.parallel.strategy import DistEmbeddingStrategy


def cfgs(sizes, combiner=None):
  return [{"input_dim": r, "output_dim": w, "combiner": combiner} for r, w in sizes]


def lc(strategy):
  return [[[c["input_dim"], c["output_dim"]] for c in rank] for rank in strategy.local_configs]


def test_column_slice_merge():
  s = DistEmbeddingStrategy(cfgs([[100, 8], [5, 8], [10, 8], [25, 4]]),
                            4,
                            "memory_balanced",
                            column_slice_threshold=45)
  assert s.table_ids == [[0, 3], [0, 3, 1], [0, 3, 2], [0, 2]]
  assert s.input_ids_list == s.table_ids
  assert s.local_maps == [[0, 0], [0, 1, 2], [0, 1, 2], [0, 1]]
  assert s.local_input_offsets == [[0, 100], [0, 0, 0], [0, 0, 0], [0, 0]]
  assert lc(s) == [[[125, 2]], [[100, 2], [25, 1], [5, 8]], [[100, 2], [25, 1], [10, 4]],
                   [[100, 2], [10, 4]]]
  assert s.local_group_list == [[[0, 1]], [[0], [1], [2]], [[0], [1], [2]], [[0], [1]]]
  assert s.local_weight_offsets == [[[0, 100, 125]], [[0, 100], [0, 25], [0, 5]],
                                    [[0, 100], [0, 25], [0, 10]], [[0, 100], [0, 10]]]
  assert s.widths_list_flat == [2, 2, 2, 1, 8, 2, 1, 4, 2, 4]
  assert s.rev_tp_ids == [0, 2, 5, 8, 4, 7, 9, 1, 3, 6]
  assert s.sliced_out_ranges == [[0, 4], [2, 4], [3, 6]]
  # explicit column ranges: rank 0 holds columns [0,2) of table 3 (two merged width-1 slices)
  assert [s.column_range(0, 1), s.column_range(1, 1), s.column_range(2, 1)] == [[0, 2], [2, 3],
                                                                              [3, 4]]


def test_column_slice_dup_worker():
  s = DistEmbeddingStrategy(cfgs([[10, 4], [11, 2], [4, 2], [4, 2]]),
                            4,
                            "memory_balanced",
                            column_slice_threshold=10)
  assert s.table_ids == [[1, 2], [1, 3], [0], [0]]
  assert lc(s) == [[[11, 1], [4, 2]], [[11, 1], [4, 2]], [[10, 2]], [[10, 2]]]
  assert s.widths_list_flat == [1, 2, 1, 2, 2, 2]
  assert s.rev_tp_ids == [4, 5, 0, 2, 1, 3]
  assert s.sliced_out_ranges == [[0, 2], [1, 3]]


def test_auto_concat():
  s = DistEmbeddingStrategy(
      cfgs([[10, 2], [11, 2], [4, 2], [4, 2], [10, 2], [11, 2], [4, 2], [4, 2]]), 2,
      "memory_balanced")
  assert s.table_ids == [[5, 7, 0, 2], [1, 6, 4, 3]]
  assert lc(s) == [[[29, 2]], [[29, 2]]]
  assert s.local_maps == [[0, 0, 0, 0], [0, 0, 0, 0]]
  assert s.local_input_offsets == [[0, 11, 15, 25], [0, 11, 15, 25]]
  assert s.local_weight_offsets == [[[0, 11, 15, 25, 29]], [[0, 11, 15, 25, 29]]]
  assert s.rev_tp_ids == [2, 4, 3, 7, 6, 0, 5, 1]


def test_fewer_tables_than_workers():
  s = DistEmbeddingStrategy(cfgs([[16, 12]]), 4, "basic")
  assert s.table_ids == [[0], [0], [0], [0]]
  assert lc(s) == 4 * [[[16, 3]]]
  assert s.widths_list_flat == [3, 3, 3, 3]
  assert s.sliced_out_ranges == [[0, 4]]


def test_shared_inputs():
  s = DistEmbeddingStrategy(cfgs([[10, 4], [20, 4], [30, 8]]),
                            2,
                            "basic",
                            input_table_map=[0, 1, 2, 0, 2])
  assert s.table_ids == [[0, 2], [1]]
  assert s.input_ids_list == [[0, 3, 2, 4], [1]]
  assert s.local_maps == [[0, 0, 1, 1], [0]]
  assert s.widths_list_flat == [4, 4, 8, 8, 4]
  assert s.rev_tp_ids == [0, 4, 2, 1, 3]


def test_all_modes():
  s = DistEmbeddingStrategy(cfgs([[5, 8], [10, 8], [50, 8], [100, 8], [200, 8], [7, 4]]),
                            4,
                            "memory_balanced",
                            data_parallel_threshold=100,
                            column_slice_threshold=200,
                            row_slice_threshold=1000)
  assert s.table_groups == [[0, 1, 5], [2, 3], [4]]
  assert s.rev_group_ids == [0, 1, 3, 4, 5, 2]
  assert s.table_ids == [[1], [1], [1, 0], [1, 0]]
  assert lc(s) == [[[100, 2]], [[100, 2]], [[100, 2], [50, 4]], [[100, 2], [50, 4]]]
  assert s.widths_list_flat == [2, 2, 2, 4, 2, 4]
  assert s.rev_tp_ids == [3, 5, 0, 1, 2, 4]
  assert s.sliced_out_ranges == [[0, 2], [1, 5]]
  assert [[[c["input_dim"], c["output_dim"]] for c in r] for r in s.row_sliced_configs
         ] == 4 * [[[50, 8]]]
  assert s.row_inputs_offsets == [[0], [-50], [-100], [-150]]


def test_memory_optimized():
  s = DistEmbeddingStrategy(
      cfgs([[100, 8], [50, 8], [40, 8], [30, 8], [20, 8], [10, 8], [5, 8]]), 3, "memory_optimized")
  assert s.table_ids == [[2, 3, 6], [1, 4, 5], [0]]
  assert lc(s) == [[[75, 8]], [[80, 8]], [[100, 8]]]
  assert s.rev_tp_ids == [6, 3, 0, 1, 4, 5, 2]


def test_cpu_offload():
  s = DistEmbeddingStrategy(cfgs(4 * [[100, 32]] + 4 * [[1000, 64]]),
                            2,
                            "basic",
                            gpu_embedding_size=32000)
  assert s.table_ids == [[0, 2, 4, 6], [1, 3, 5, 7]]
  got = [[[c["input_dim"], c["output_dim"], c["cpu_offload"]] for c in r] for r in s.local_configs]
  assert got == 2 * [[[200, 32, False], [1000, 64, True], [1000, 64, True]]]


def test_dlrm_like():
  s = DistEmbeddingStrategy(cfgs(26 * [[1000, 128]]), 8, "memory_balanced")
  assert s.table_ids == [[25, 9, 10], [24, 8, 11], [23, 7, 12], [22, 6, 13], [21, 5, 14],
                         [20, 4, 15], [19, 3, 16, 0], [18, 2, 17, 1]]
  assert lc(s) == 6 * [[[3000, 128]]] + 2 * [[[4000, 128]]]


def test_single_worker_forces_basic():
  s = DistEmbeddingStrategy(cfgs([[10, 4], [30, 4], [20, 8]]), 1, "memory_balanced")
  assert s.strategy == "basic"
  assert s.table_ids == [[0, 1, 2]]
  assert lc(s) == [[[40, 4], [20, 8]]]
  assert s.local_maps == [[0, 0, 1]]
  assert s.local_input_offsets == [[0, 10, 0]]


def test_output_pieces_cover_outputs():
  s = DistEmbeddingStrategy(cfgs([[100, 8], [5, 8], [10, 8], [25, 4]]),
                            4,
                            "memory_balanced",
                            column_slice_threshold=45)
  assert s.col_output_widths == [8, 8, 8, 4]
  seen = {}
  for p in s.output_pieces:
    seen.setdefault(p.group_input, []).append((p.col_offset, p.width))
  for k, pieces in seen.items():
    pos = 0
    for off, w in pieces:
      assert off == pos
      pos += w
    assert pos == s.col_output_widths[k]


def test_shared_input_with_slices_ranges():
  # two inputs share a sliced table: every input of that table needs a concat range
  s = DistEmbeddingStrategy(cfgs([[100, 8], [4, 4]]),
                            2,
                            "basic",
                            input_table_map=[0, 1, 0],
                            column_slice_threshold=500)
  assert s.sliced_out_ranges == [[0, 2], [2, 4]]


def test_bad_strategy():
  with pytest.raises(ValueError):
    DistEmbeddingStrategy(cfgs([[4, 4]]), 1, "nope")


def test_fingerprint_is_stable():
  a = DistEmbeddingStrategy(cfgs(26 * [[1000, 128]]), 8, "memory_balanced").fingerprint()
  b = DistEmbeddingStrategy(cfgs(26 * [[1000, 128]]), 8, "memory_balanced").fingerprint()
  c = DistEmbeddingStrategy(cfgs(26 * [[1000, 128]]), 8, "basic").fingerprint()
  assert a == b and a != c


def test_traffic_report_dlrm_mlperf():
  """Bytes per step implied by a plan: the 1-GPU gather volume of the MLPerf DLRM is one fp32
  row of every table per sample (65536 x 26 x 128 x 4 B = 872 MB), and column slicing the six
  big tables evens out the 8-GPU load."""
  from distributed_embeddings_b200.models.dlrm import mlperf_table_sizes
  cfgs = [{"input_dim": s, "output_dim": 128, "combiner": None} for s in mlperf_table_sizes()]
  one = DistEmbeddingStrategy(cfgs, 1, "memory_balanced").traffic_report(65536)
  assert one["max_gather_bytes"] == 65536 * 26 * 128 * 4 and one["max_nvlink_out_bytes"] == 0
  plain = DistEmbeddingStrategy(cfgs, 8, "memory_balanced").traffic_report(65536)
  sliced = DistEmbeddingStrategy(cfgs, 8, "memory_balanced",
                                 column_slice_threshold=2**32).traffic_report(65536)
  assert sliced["nvlink_imbalance"] < plain["nvlink_imbalance"] <= 1.3
  total_out = sum(r["nvlink_out_bytes"] for r in sliced["ranks"])
  assert total_out == pytest.approx(65536 * 26 * 128 * 2 * 7 / 8)
  # multi-hot, row slices and replicated tables are accounted separately
  cfgs = [{"input_dim": 1000, "output_dim": 16, "combiner": "sum"},
          {"input_dim": 10, "output_dim": 8, "combiner": "sum"},
          {"input_dim": 100000, "output_dim": 32, "combiner": "sum"}]
  st = DistEmbeddingStrategy(cfgs, 4, "basic", data_parallel_threshold=100,
                             row_slice_threshold=1000000)
  rep = st.traffic_report(4096, hotness=[3, 1, 5])
  assert st.table_groups == [[1], [0], [2]]
  r0 = rep["ranks"][0]
  # the single table-parallel table is column sliced onto all 4 ranks (fewer tables than
  # workers): each looks up the whole batch; replicated: 1024 local lookups per rank; row slice:
  # a quarter of the 4096 x 5 ids on every rank
  assert sum(r["lookups"] for r in rep["ranks"]) == 4 * 4096 * 3 + 4 * 1024 + 4096 * 5
  assert r0["nvlink_out_bytes"] >= 4096 * 32 * 4 * 3 / 4


def test_auto_column_slice_threshold():
  from distributed_embeddings_b200 import DistributedEmbedding
  from distributed_embeddings_b200.models.dlrm import mlperf_table_sizes
  from distributed_embeddings_b200.parallel.strategy import suggest_column_slice_threshold
  cfgs = [{"input_dim": s, "output_dim": 128, "combiner": None} for s in mlperf_table_sizes()]
  assert [suggest_column_slice_threshold(cfgs, w) for w in (1, 2, 4, 8)] == \
      [None, None, None, 2**32]
  # the wrapper accepts "auto" (planning only: no process group needed with explicit rank/world)
  small = [{"input_dim": 5000, "output_dim": 128, "combiner": "sum"}] + \
      [{"input_dim": 50, "output_dim": 128, "combiner": "sum"} for _ in range(3)]
  de = DistributedEmbedding(small, strategy="memory_balanced", column_slice_threshold="auto",
                            device="cpu", backend="torch", world_size=4, rank=0)
  rep = de.strategy.traffic_report(4096)
  base = DistributedEmbedding(small, strategy="memory_balanced", device="cpu", backend="torch",
                              world_size=4, rank=0).strategy.traffic_report(4096)
  assert rep["max_nvlink_out_bytes"] <= base["max_nvlink_out_bytes"]
  assert min(c["output_dim"] for r in range(4) for c in de.strategy.local_configs[r]) >= 64


def test_traffic_balanced_placement():
  """The work-balancing placement (not in the reference): on the synthetic "small" model at 8
  ranks the size-based snake leaves one rank with 2.5x the mean gather bytes."""
  from distributed_embeddings_b200.models.configs import expand, synthetic_models_v3
  tables, imap, hots = expand(synthetic_models_v3["small"])[:3]
  cfgs = [{"input_dim": int(r), "output_dim": int(w), "combiner": "sum"} for r, w in tables]
  mem = DistEmbeddingStrategy(cfgs, 8, "memory_balanced", input_table_map=imap)
  tra = DistEmbeddingStrategy(cfgs, 8, "traffic_balanced", input_table_map=imap,
                              input_hotness=hots)
  a, b = mem.traffic_report(65536, hots), tra.traffic_report(65536, hots)
  assert a["gather_imbalance"] > 2.0 and b["gather_imbalance"] < 1.25
  assert b["max_gather_bytes"] < 0.6 * a["max_gather_bytes"]
  assert b["nvlink_imbalance"] < 1.5
  # every table is still placed exactly once per column and the plan is deterministic
  cover = {}
  for r, shards in enumerate(tra.shards):
    for s in shards:
      cover.setdefault(s.table, []).append((s.col_start, s.col_end))
  for t, pieces in cover.items():
    pieces.sort()
    assert pieces[0][0] == 0 and all(x[1] == y[0] for x, y in zip(pieces, pieces[1:]))
  again = DistEmbeddingStrategy(cfgs, 8, "traffic_balanced", input_table_map=imap,
                                input_hotness=hots)
  assert again.fingerprint() == tra.fingerprint()
  # a single dominant multi-hot table gets column sliced beyond what its size asks for
  hot = [{"input_dim": 1000, "output_dim": 128, "combiner": "sum"}] + \
      [{"input_dim": 1000, "output_dim": 128, "combiner": "sum"} for _ in range(7)]
  st = DistEmbeddingStrategy(hot, 4, "traffic_balanced", input_hotness=[50] + [1] * 7)
  assert len([s for sh in st.shards for s in sh if s.table == 0]) == 4
  with pytest.raises(ValueError):
    DistEmbeddingStrategy(hot, 4, "traffic_balanced", input_hotness=[1, 2])
