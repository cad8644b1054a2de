#!/usr/bin/env python
"""Per-kernel SASS mnemonic census of the built extension (cuobjdump runs without a GPU):
   python tools/sass_census.py"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SO = os.path.join(ROOT, "distributed_embeddings_b200", "_C.so")
NOTABLE = re.compile(r"^(HGMMA|WARPGROUP|UTMALDG|UTMASTG|UTCBAR|UTCATOMSWS|UBLKCP|SYNCS|HMMA|LDGSTS|LDSM|REDG|"
                     r"ATOMG|ATOMS|MATCH|LDGMC|STGMC|REDGMC|LDG\.E\.128|STG\.E\.128|LDTM|STTM|MULTIMEM|MEMBAR|"
                     r"LDG\.E\.STRONG\.SYS|STG\.E\.STRONG\.SYS|LD\.E\.STRONG\.SYS|ST\.E\.STRONG\.SYS|"
                     r"CCTL|UCGABAR|ELECT|REDUX|SHFL)")


def main():
  sass = subprocess.run(["cuobjdump", "-sass", SO], capture_output=True, text=True, check=True).stdout
  demangle = {}
  names = re.findall(r"Function : (\S+)", sass)
  if names:
    out = subprocess.run(["cu++filt"] + names, capture_output=True, text=True, check=False).stdout
    for n, d in zip(names, out.splitlines()):
      demangle[n] = d
  print(f"# SASS mnemonic census of distributed_embeddings_b200/_C.so (sm_90a), per kernel")
  print("# columns: kernel | instructions | notable opcodes (count)\n")
  cur, counts, total = None, None, 0
  rows = []

  def flush():
    if cur is not None:
      name = demangle.get(cur, cur)
      name = re.sub(r"\(anonymous namespace\)::", "", name)
      rows.append((name, total, dict(counts)))

  for line in sass.splitlines():
    m = re.search(r"Function : (\S+)", line)
    if m:
      flush()
      cur, counts, total = m.group(1), collections.Counter(), 0
      continue
    m = re.match(r"\s+/\*[0-9a-f]{4}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)", line)
    if m and cur is not None:
      op = m.group(1)
      total += 1
      k = NOTABLE.match(op)
      if k:
        # keep the qualifiers that carry meaning (2CTA, MULTICAST, F32x4, sizes)
        key = op if op.startswith(("HGMMA", "UTMA", "REDG", "HMMA", "MATCH", "MULTIMEM", "LDTM", "LDGMC", "STGMC", "REDGMC",
                                   "UBLKCP")) else k.group(1)
        counts[key] += 1
  flush()
  for name, tot, c in rows:
    ops = ", ".join(f"{k}:{v}" for k, v in sorted(c.items(), key=lambda kv: -kv[1]))
    print(f"{name[:150]} | {tot} | {ops}")


if __name__ == "__main__":
  sys.exit(main())
