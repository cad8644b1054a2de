"""bench.py driver contract, the parts that can be checked without a GPU: the reference arm always
prints one JSON line and exits 0, the default flags are the BASELINE configuration, and the
automatic column-slice threshold yields a plan every rank participates in."""
import importlib.util
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _load_bench():
  spec = importlib.util.spec_from_file_location("de_bench", os.path.join(ROOT, "bench.py"))
  mod = importlib.util.module_from_spec(spec)
  spec.loader.exec_module(mod)
  return mod


def test_reference_arm_prints_one_json_line():
  out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference",
                        "--gpus", "1", "--steps", "2", "--warmup", "1"],
                       capture_output=True, text=True, timeout=600, cwd=ROOT, check=False)
  assert out.returncode == 0, out.stderr[-2000:]
  lines = [l for l in out.stdout.splitlines() if l.startswith("{")]
  assert len(lines) == 1
  rec = json.loads(lines[0])
  assert rec["impl"] == "reference"
  # either the reference ran (metric/value present) or it says why it could not
  assert "unavailable" in rec or ("metric" in rec and "value" in rec)


def test_defaults_are_the_baseline_config(monkeypatch):
  bench = _load_bench()
  monkeypatch.setattr(sys, "argv", ["bench.py"])
  args = bench.parse_args()
  assert args.gpus == 1 and args.warmup >= 3
  assert args.global_batch == 65536 and args.model == "dlrm-mlperf-20m" and args.dtype == "bf16"
  with open(os.path.join(ROOT, "BASELINE.json"), encoding="utf-8") as f:
    base = json.load(f)
  assert "samples" in json.dumps(base).lower()
  sizes = bench.table_sizes_for("dlrm-mlperf")
  assert len(sizes) == 26 and sum(sizes) == 187767425
  # the default model: the same tables capped at 20M rows, 49.6 GiB fp32 on one 80 GB GPU
  sizes = bench.table_sizes_for(args.model)
  assert len(sizes) == 26 and sum(sizes) == 104064018 and max(sizes) == 20000001


@pytest.mark.parametrize("world", [1, 2, 4, 8])
def test_auto_column_slice_threshold(world):
  from distributed_embeddings_b200.parallel.strategy import DistEmbeddingStrategy
  bench = _load_bench()
  sizes = bench.table_sizes_for("dlrm-mlperf")
  thr = bench.auto_column_slice_threshold(sizes, 128, world)
  cfgs = [{"input_dim": s, "output_dim": 128, "combiner": None} for s in sizes]
  st = DistEmbeddingStrategy(cfgs, world, "memory_balanced", column_slice_threshold=thr)
  cols = [sum(st.local_configs[r][m]["output_dim"] for m in st.local_maps[r]) for r in range(world)]
  assert all(c > 0 for c in cols)
  # looked-up columns per rank (what sets gather and NVLink bytes) within 35% of perfect balance
  assert max(cols) <= 1.35 * (26 * 128 / world) + 64
  assert min(c["output_dim"] for r in range(world) for c in st.local_configs[r]) >= 64


@pytest.mark.parametrize("world", [2, 4, 8])
def test_default_plan_with_replicated_tables(world):
  """The plan bench.py times by default at N > 1: tables of at most 2500 rows are replicated, the
  column-slice rule only looks at the tables that are still exchanged."""
  from distributed_embeddings_b200.parallel.strategy import DistEmbeddingStrategy
  bench = _load_bench()
  sizes = bench.table_sizes_for("dlrm-mlperf")
  dpt = 2500 * 128
  thr = bench.auto_column_slice_threshold(sizes, 128, world, dpt)
  cfgs = [{"input_dim": s, "output_dim": 128, "combiner": None} for s in sizes]
  st = DistEmbeddingStrategy(cfgs, world, "memory_balanced", column_slice_threshold=thr,
                             data_parallel_threshold=dpt)
  n_dp = len(st.table_groups[0])
  assert n_dp == sum(1 for s in sizes if s * 128 <= dpt) == 11
  assert len(st.table_groups[1]) == 26 - n_dp and not st.table_groups[2]
  cols = [sum(st.local_configs[r][m]["output_dim"] for m in st.local_maps[r]) for r in range(world)]
  assert all(c > 0 for c in cols), "every rank owns part of the exchange"
  mean = (26 - n_dp) * 128 / world
  assert max(cols) <= max(1.25 * mean, mean + 128), (cols, thr)


def _bench_dump(out_dir, steps):
  out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--steps",
                        str(steps), "--warmup", "1", "--model", "dlrm-tiny", "--global-batch",
                        "4096", "--no-e2e", "--dump-outputs", str(out_dir)],
                       capture_output=True, text=True, timeout=900, cwd=ROOT, check=False)
  assert out.returncode == 0, out.stderr[-2000:]
  lines = [l for l in out.stdout.splitlines() if l.startswith("{")]
  assert len(lines) == 1
  return json.loads(lines[0])


@pytest.mark.gpu
def test_dump_outputs_of_the_timed_step(tmp_path):
  """--steps sets the timed steps; --dump-outputs writes the last timed step's loss, dense
  parameters and sampled embedding rows as float .npy files within 64 MB.  Two runs with the same
  arguments agree; a run with one timed step fewer differs by far more than that, so the dump
  reflects the last timed step and not a stale or earlier state."""
  import numpy as np
  rec = _bench_dump(tmp_path / "a", 3)
  assert rec["steps"] == 3
  names = sorted(os.listdir(tmp_path / "a"))
  for want in ("loss.npy", "bottom_mlp_0_weight.npy", "top_mlp_4_bias.npy", "embedding_0.npy",
               "embedding_25.npy"):
    assert want in names, names
  total = 0
  for name in names:
    a = np.load(tmp_path / "a" / name)
    assert a.dtype in (np.float32, np.float64) and np.isfinite(a).all(), name
    total += a.nbytes
  assert total <= 64 << 20
  assert np.load(tmp_path / "a" / "embedding_0.npy").shape == (1000, 128)
  assert _bench_dump(tmp_path / "b", 3)["steps"] == 3
  assert _bench_dump(tmp_path / "c", 2)["steps"] == 2

  def l1_diff(x, y, name):
    return float(np.abs(np.load(tmp_path / x / name).astype(np.float64) -
                        np.load(tmp_path / y / name).astype(np.float64)).sum())

  for name in names:
    # identical seeded inputs; only the order of atomic float additions may differ
    np.testing.assert_allclose(np.load(tmp_path / "b" / name), np.load(tmp_path / "a" / name),
                               rtol=1e-3, atol=1e-5, err_msg=name)
  # early in the learning-rate warm-up a step moves every touched element by little, but all of
  # them, while reordered atomics move a few elements by an ulp or two: compare summed differences
  for name in ("loss.npy", "top_mlp_0_weight.npy", "bottom_mlp_0_weight.npy", "embedding_0.npy"):
    noise, step = l1_diff("a", "b", name), l1_diff("a", "c", name)
    assert step > 0 and step > 10 * noise, (name, noise, step)
