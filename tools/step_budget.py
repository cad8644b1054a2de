#!/usr/bin/env python
"""Where the time of one training step goes, from a `tools/critical_path.py` timeline (text).

For every rank: kernel time per category (dense GEMMs, dense element-wise, embedding lookups,
embedding updates, interaction, collectives / pushes, copies), the part of the step span during
which exactly one / several / no kernels were running, and the *exposed* time of every category:
the wall-clock during which only kernels of that category were running (what would have to shrink
for the step to get shorter).  No GPU needed.

  python tools/step_budget.py critical_path_n8.txt > step_budget_n8.txt
"""
import re
import sys
from collections import defaultdict

CATS = [
    ("dense GEMM (cuBLASLt nvjet / splitK)", ("nvjet", "splitKreduce", "gemm_tn_")),
    ("dense element-wise (relu-bwd+bias, loss, cast, SGD)",
     ("relu_bwd_bias", "head_loss", "cast_pad", "sgd_update", "vectorized_elementwise",
      "select_copy")),
    ("embedding lookup (+ pooled-row push)", ("lookup_fwd",)),
    ("embedding update (scatter / sort / segment)",
     ("scatter_add", "segment_update", "balanced_update", "build_keys", "digit_", "head_c",
      "head_s", "finalize_crossing", "finish_segments")),
    ("interaction fwd / bwd (+ gradient routing)", ("interact_",)),
    ("exchange / collectives (id push, grad push, all-reduce, waits)",
     ("push_segments", "push_grad", "stream_push", "allreduce_", "sync_only", "barrier_kernel",
      "rowslice_reduce")),
    ("copies (Memcpy / Memset)", ("Memcpy", "Memset")),
]
LINE = re.compile(r"^\s+([0-9.]+) \+\s+([0-9.]+)\s+(.*)$")


def category(name):
  for i, (_, keys) in enumerate(CATS):
    if any(k in name for k in keys):
      return i
  return len(CATS)


def parse(path):
  ranks, cur = {}, None
  with open(path, encoding="utf-8") as f:
    for line in f:
      m = re.match(r"^== rank (\d+): (\d+) kernels, step span ([0-9.]+) us", line)
      if m:
        cur = int(m.group(1))
        ranks[cur] = {"span": float(m.group(3)), "k": []}
        continue
      if line.startswith("== cross-GPU"):
        cur = None
      m = LINE.match(line)
      if m and cur is not None and "idle" not in line:
        ranks[cur]["k"].append((float(m.group(1)), float(m.group(2)), m.group(3).strip()))
  return ranks


def budget(kernels):
  """Sweep over kernel start / end events: time with 0, 1, >1 kernels active, per-category busy
  time and per-category exposed time (only that category active)."""
  ev = []
  for s, d, name in kernels:
    c = category(name)
    ev.append((s, 1, c))
    ev.append((s + d, -1, c))
  ev.sort(key=lambda e: (e[0], e[1]))
  active = defaultdict(int)
  t_prev = ev[0][0]
  t_first, t_last = ev[0][0], max(e[0] for e in ev)
  conc = defaultdict(float)
  exposed = defaultdict(float)
  for t, delta, c in ev:
    dt = t - t_prev
    if dt > 0:
      n = sum(active.values())
      conc[min(n, 2)] += dt
      cats = [k for k, v in active.items() if v > 0]
      if len(cats) == 1:
        exposed[cats[0]] += dt
    active[c] += delta
    t_prev = t
  busy = defaultdict(float)
  for _, d, name in kernels:
    busy[category(name)] += d
  return t_last - t_first, conc, busy, exposed


def main():
  path = sys.argv[1]
  ranks = parse(path)
  names = [c[0] for c in CATS] + ["other"]
  print(f"# step budget from {path} (one graph replay; times in us)")
  agg_busy, agg_exp = defaultdict(list), defaultdict(list)
  for r in sorted(ranks):
    span, conc, busy, exposed = budget(ranks[r]["k"])
    print(f"\n== rank {r}: span {span:.1f}, no kernel {conc[0]:.1f}, one kernel {conc[1]:.1f}, "
          f"two or more {conc[2]:.1f}")
    print(f"   {'category':<62} {'busy':>8} {'exposed':>8}")
    for i, n in enumerate(names):
      if busy[i] == 0:
        continue
      print(f"   {n:<62} {busy[i]:8.1f} {exposed[i]:8.1f}")
      agg_busy[i].append(busy[i])
      agg_exp[i].append(exposed[i])
  n = len(ranks)
  if n > 1:
    print(f"\n== mean / max over {n} ranks")
    print(f"   {'category':<62} {'busy mean':>10} {'busy max':>9} {'exposed mean':>13} "
          f"{'exposed max':>12}")
    for i, nm in enumerate(names):
      if not agg_busy[i]:
        continue
      b, e = agg_busy[i], agg_exp[i]
      print(f"   {nm:<62} {sum(b) / len(b):10.1f} {max(b):9.1f} {sum(e) / len(e):13.1f} "
            f"{max(e):12.1f}")
    spans = [budget(ranks[r]["k"])[0] for r in ranks]
    print(f"   step span mean {sum(spans) / n:.1f}, max {max(spans):.1f}")


if __name__ == "__main__":
  main()
