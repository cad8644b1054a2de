"""The offline analysis tools: timelines, step budgets, SASS and plan reports (no GPU)."""
import os
import shutil
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run(*args):
  return subprocess.run([sys.executable] + list(args), capture_output=True, text=True, cwd=ROOT,
                        timeout=300, check=False)


def _trace(rank_delay, steps=3):
  """A chrome trace of ``bench.py --profile-all-ranks`` shape: ``steps`` steps of six kernels (id
  push, lookup, dense GEMM, interaction, all-reduce, embedding update), 400 us apart."""
  ev, t = [], 1000.0
  for _ in range(steps):
    t0 = t + rank_delay
    for name, dur in (("void de::(anonymous namespace)::push_segments_kernel<int>(...)", 10),
                      ("void de::(anonymous namespace)::lookup_fwd_kernel<int, bf16, 4>(...)", 40),
                      ("nvjet_tst_128x256_64x6_2x2_2cta_v_bz_relubias", 30),
                      ("void de::(anonymous namespace)::interact_fwd_kernel<128>(...)", 25),
                      ("void de::(anonymous namespace)::allreduce_p2p_kernel<false>(...)", 20),
                      ("void de::(anonymous namespace)::scatter_add_staged_kernel<int, bf16>(...)",
                       35)):
      ev.append({"ph": "X", "cat": "kernel", "name": name, "ts": t0, "dur": dur})
      t0 += dur + 1
    t += 400
  return {"traceEvents": ev}


def _write_traces(prof, delays):
  import json
  for rank, delay in enumerate(delays):
    suffix = ".trace.json" if rank == 0 else f".rank{rank}.trace.json"
    with open(prof + suffix, "w", encoding="utf-8") as f:
      json.dump(_trace(delay), f)


def test_step_budget_on_an_eight_rank_timeline(tmp_path):
  prof = str(tmp_path / "prof.txt")
  _write_traces(prof, [1.5 * r for r in range(8)])
  timeline = _run("tools/critical_path.py", prof, "--step", "1")
  assert timeline.returncode == 0, timeline.stderr[-1000:]
  path = tmp_path / "timeline.txt"
  path.write_text(timeline.stdout, encoding="utf-8")
  out = _run("tools/step_budget.py", str(path))
  assert out.returncode == 0, out.stderr[-1000:]
  text = out.stdout
  assert text.count("== rank ") == 8
  assert "mean / max over 8 ranks" in text
  for cat in ("dense GEMM", "embedding lookup", "embedding update", "interaction", "exchange"):
    assert cat in text
  # per-rank rows ("   <category>  busy  exposed"): exposed time never exceeds busy time
  per_rank = text.split("== mean / max")[0]
  checked = 0
  for line in per_rank.splitlines():
    parts = line.split()
    if line.startswith("   ") and len(parts) >= 3 and not line.strip().startswith("category"):
      try:
        busy, exposed = float(parts[-2]), float(parts[-1])
      except ValueError:
        continue
      assert exposed <= busy + 1e-6, line
      checked += 1
  assert checked >= 8 * 5


@pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="CUDA toolkit not on PATH")
def test_resource_usage_lists_the_hot_kernels():
  so = os.path.join(ROOT, "distributed_embeddings_b200", "_C.so")
  if not os.path.exists(so):
    pytest.skip("extension not built")
  out = _run("tools/resource_usage.py")
  assert out.returncode == 0, out.stderr[-1000:]
  for k in ("lookup_fwd_kernel<int, __nv_bfloat16, 4, float>", "scatter_add_staged_kernel",
            "interact_bwd_v2_kernel<128>", "stream_push_kernel", "gemm_tn_pair_kernel",
            "digit_scatter_kernel", "integer_lookup_kernel"):
    assert k in out.stdout, k


@pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="CUDA toolkit not on PATH")
def test_sass_census_shows_the_hopper_opcodes():
  so = os.path.join(ROOT, "distributed_embeddings_b200", "_C.so")
  if not os.path.exists(so):
    pytest.skip("extension not built")
  out = _run("tools/sass_census.py")
  assert out.returncode == 0, out.stderr[-1000:]
  text = out.stdout
  for op in ("HGMMA", "UTMALDG", "REDG", "LDGSTS", "HMMA", "STRONG.SYS", "MATCH.ANY"):
    assert op in text, op


def test_plan_report_cli():
  import json
  out = _run("tools/plan_report.py", "--model", "dlrm-mlperf", "--world", "8",
             "--data-parallel-threshold", "320000", "--json")
  assert out.returncode == 0, out.stderr[-1000:]
  rep = json.loads(out.stdout.strip().splitlines()[-1])
  assert rep["replicated"] == 11 and rep["table_parallel"] == 15 and rep["row_sliced"] == 0
  assert len(rep["ranks"]) == 8 and all(x["fits"] for x in rep["ranks"])
  assert max(x["exchanged_columns"] for x in rep["ranks"]) == 256
  assert 1.0 <= rep["nvlink_imbalance"] < 1.1
  # human-readable form, a synthetic model with shared multi-hot inputs, explicit tables
  out = _run("tools/plan_report.py", "--model", "tiny", "--world", "4", "--strategy",
             "traffic_balanced")
  assert out.returncode == 0 and "imbalance (max / mean)" in out.stdout, out.stderr[-1000:]
  out = _run("tools/plan_report.py", "--tables", "1000000x128,5000x64,3000000x32", "--world", "2",
             "--column-slice-threshold", "auto", "--hbm-gib", "0.1")
  assert out.returncode == 0 and "GiB!" in out.stdout, out.stdout[-500:] + out.stderr[-500:]


def test_critical_path_and_step_budget_on_a_synthetic_trace(tmp_path):
  """tools/critical_path.py merges the per-rank chrome traces of `bench.py --profile-all-ranks`
  into one timeline; tools/step_budget.py reads that text.  Two ranks, three steps each."""
  prof = str(tmp_path / "prof.txt")
  _write_traces(prof, [0.0, 7.0])
  out = _run("tools/critical_path.py", prof, "--step", "1")
  assert out.returncode == 0, out.stderr[-1000:]
  text = out.stdout
  assert "== rank 0: 6 kernels" in text and "== rank 1: 6 kernels" in text
  assert "cross-GPU waits" in text and "skew 7.0 us" in text
  assert "last in rank 1" in text
  timeline = tmp_path / "timeline.txt"
  timeline.write_text(text, encoding="utf-8")
  bud = _run("tools/step_budget.py", str(timeline))
  assert bud.returncode == 0, bud.stderr[-1000:]
  assert bud.stdout.count("== rank ") == 2 and "embedding lookup" in bud.stdout
  assert "embedding update" in bud.stdout and "dense GEMM" in bud.stdout
