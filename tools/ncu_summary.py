#!/usr/bin/env python
"""Compact per-kernel summary of an ncu report (runs without a GPU):
   python tools/ncu_summary.py x.ncu-rep > x_summary.txt"""
import csv
import io
import subprocess
import sys

WANT = [
    ("gpu__time_duration.sum", "time"),
    ("dram__bytes_read.sum", "dram read"),
    ("dram__bytes_write.sum", "dram write"),
    ("gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "dram % of peak"),
    ("lts__t_sector_hit_rate.pct", "L2 hit %"),
    ("sm__throughput.avg.pct_of_peak_sustained_elapsed", "SM % of peak"),
    ("sm__warps_active.avg.pct_of_peak_sustained_active", "warps active %"),
    ("sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active", "tensor pipe %"),
    ("launch__registers_per_thread", "regs/thread"),
    ("launch__shared_mem_per_block_dynamic", "dyn smem/block"),
    ("launch__occupancy_limit_registers", "occ limit regs (blocks)"),
    ("launch__occupancy_limit_shared_mem", "occ limit smem (blocks)"),
    ("smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio", "stall long_scoreboard"),
    ("smsp__average_warps_issue_stalled_lg_throttle_per_issue_active.ratio", "stall lg_throttle"),
    ("smsp__average_warps_issue_stalled_short_scoreboard_per_issue_active.ratio", "stall short_scoreboard"),
    ("smsp__average_warps_issue_stalled_barrier_per_issue_active.ratio", "stall barrier"),
    ("smsp__average_warps_issue_stalled_mio_throttle_per_issue_active.ratio", "stall mio_throttle"),
    ("smsp__average_warps_issue_stalled_drain_per_issue_active.ratio", "stall drain"),
    ("smsp__average_warps_issue_stalled_wait_per_issue_active.ratio", "stall wait"),
    ("lts__t_sectors_op_red.sum", "L2 RED sectors"),
    ("lts__t_sectors_op_atom.sum", "L2 ATOM sectors"),
    ("l1tex__t_sectors_pipe_lsu_mem_global_op_ld.sum", "L1 global load sectors"),
    ("l1tex__t_sectors_pipe_lsu_mem_global_op_st.sum", "L1 global store sectors"),
    ("smsp__inst_executed.sum", "warp instructions"),
]


def main():
  rep = sys.argv[1]
  out = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True,
                       text=True, check=True).stdout
  rows = list(csv.reader(io.StringIO(out)))
  hdr, units = rows[0], rows[1]
  col = {}
  for i, h in enumerate(hdr):
    col.setdefault(h.split(".", 2)[-1] if h.count(".") > 2 and h.split(".")[1] in
                   ("TriageCompute",) else h, i)
    col.setdefault(h, i)
  print(f"# {rep}: ncu --set full --clock-control none (one launch per row, cold L2 per replay)")
  for r in rows[2:]:
    name = r[hdr.index("Kernel Name")]
    print(f"\n== {name}  grid {r[hdr.index('Grid Size')]} block {r[hdr.index('Block Size')]}")
    for key, label in WANT:
      i = col.get(key)
      if i is None or r[i] == "":
        continue
      print(f"   {label:28s} {r[i]:>18s} {units[i]}")


if __name__ == "__main__":
  main()
