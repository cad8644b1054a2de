#!/usr/bin/env python
"""Per-kernel resource usage of ``_C.so`` (registers, shared memory, stack / spills, constant
bank) from ``cuobjdump -res-usage`` - the ``-Xptxas -v`` numbers of the binary that actually ships,
no GPU needed:

    python tools/resource_usage.py > resource_usage.txt
"""
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SO = os.path.join(ROOT, "distributed_embeddings_b200", "_C.so")


def main():
  out = subprocess.run(["cuobjdump", "-res-usage", SO], capture_output=True, text=True,
                       check=True).stdout
  rows, src = [], ""
  lines = out.splitlines()
  for i, line in enumerate(lines):
    m = re.match(r"identifier = (.*)", line)
    if m:
      src = os.path.basename(m.group(1))
    m = re.match(r"\s*Function (\S+):", line)
    if m and i + 1 < len(lines):
      res = dict(re.findall(r"(REG|STACK|SHARED|LOCAL|CONSTANT\[0\]):(\d+)", lines[i + 1]))
      rows.append((src, m.group(1), res))
  names = subprocess.run(["cu++filt"] + [r[1] for r in rows], capture_output=True, text=True,
                         check=False).stdout.splitlines()
  print("# cuobjdump -res-usage of distributed_embeddings_b200/_C.so (sm_90a); static shared "
        "memory only - dynamic shared memory is set at launch")
  print(f"{'source':<26} {'regs':>5} {'stack':>6} {'local':>6} {'smem':>7} {'const0':>7}  kernel")
  for (src, _, res), name in sorted(zip(rows, names), key=lambda x: (x[0][0], x[1])):
    name = re.sub(r"\(anonymous namespace\)::|<unnamed>::", "", name)
    name = re.sub(r"\((int|bool|unsigned int)\)", "", name)
    name = re.sub(r"^void ", "", name).split("(")[0]
    print(f"{src:<26} {res.get('REG', '?'):>5} {res.get('STACK', '0'):>6} "
          f"{res.get('LOCAL', '0'):>6} {res.get('SHARED', '0'):>7} "
          f"{res.get('CONSTANT[0]', '0'):>7}  {name}")


if __name__ == "__main__":
  main()
