#!/usr/bin/env python
"""Summarise an ncu report (--set full) into a small JSON:  python tools/ncu_summary.py <report.ncu-rep> <out.json> [note]"""
import csv
import io
import json
import subprocess
import sys

rep, out = sys.argv[1], sys.argv[2]
note = sys.argv[3] if len(sys.argv) > 3 else ""
raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
rows = list(csv.reader(io.StringIO(raw)))
h = rows[0]
KEYS = {
    "gpu__time_duration.sum": "duration_us", "smsp__inst_executed.sum": "warp_instructions", "launch__registers_per_thread": "registers",
    "launch__grid_size": "grid", "launch__block_size": "block", "sm__warps_active.avg.pct_of_peak_sustained_active": "warps_active_pct",
    "smsp__issue_active.avg.pct_of_peak_sustained_active": "issue_active_pct", "sm__cycles_active.avg": "sm_cycles_active", "sm__cycles_elapsed.avg": "sm_cycles_elapsed",
    "dram__bytes_read.sum": "dram_read", "dram__bytes_write.sum": "dram_write", "dram__throughput.avg.pct_of_peak_sustained_elapsed": "dram_throughput_pct",
    "lts__t_bytes.sum": "l2_bytes", "l1tex__t_bytes.sum": "l1_bytes", "launch__occupancy_limit_registers": "occ_limit_regs", "launch__occupancy_limit_shared_mem": "occ_limit_smem",
    "smsp__average_warp_latency_per_inst_issued.ratio": "warp_latency_per_inst",
    "smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio": "stall_long_scoreboard",
    "smsp__average_warps_issue_stalled_short_scoreboard_per_issue_active.ratio": "stall_short_scoreboard",
    "smsp__average_warps_issue_stalled_wait_per_issue_active.ratio": "stall_wait",
    "smsp__average_warps_issue_stalled_not_selected_per_issue_active.ratio": "stall_not_selected",
    "smsp__average_warps_issue_stalled_math_pipe_throttle_per_issue_active.ratio": "stall_math_pipe",
    "smsp__average_warps_issue_stalled_lg_throttle_per_issue_active.ratio": "stall_lg_throttle",
    "smsp__average_warps_issue_stalled_barrier_per_issue_active.ratio": "stall_barrier",
}
units = rows[1]
res = []
for row in rows[2:]:
    d = dict(zip(h, row))
    u = dict(zip(h, units))
    k = {"kernel": d.get("Kernel Name"), "id": d.get("ID")}
    for src, dst in KEYS.items():
        if src in d and d[src] != "":
            try:
                v = float(d[src].replace(",", ""))
            except ValueError:
                continue
            unit = u.get(src, "")
            if dst in ("dram_read", "dram_write", "l2_bytes", "l1_bytes"):
                mult = {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}.get(unit, 1)
                v *= mult
            if dst == "duration_us":
                v *= {"ns": 1e-3, "us": 1, "ms": 1e3, "s": 1e6}.get(unit, 1)
            k[dst] = v
    if "dram_read" in k:
        k["dram_bytes"] = k.get("dram_read", 0) + k.get("dram_write", 0)
    res.append(k)
json.dump({"report": rep, "note": note, "kernels": res}, open(out, "w"), indent=1)
for k in res:
    print(f"{k['kernel'][:60]:60s} {k.get('duration_us', 0):8.1f} us  inst {k.get('warp_instructions', 0) / 1e6:7.2f} M  regs {k.get('registers', 0):3.0f}  "
          f"issue {k.get('issue_active_pct', 0):5.1f}%  warps {k.get('warps_active_pct', 0):5.1f}%  dram {k.get('dram_bytes', 0) / 1e6:7.2f} MB  L2 {k.get('l2_bytes', 0) / 1e6:8.2f} MB")
