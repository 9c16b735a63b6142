"""Summarise an `ncu --page raw --csv` export: one JSON object per captured launch with the headline numbers
(duration, DRAM bytes read / written, executed warp instructions, registers, occupancy, SM-active cycles).
Usage: python scripts/ncu_summary.py <raw.csv> [<raw.csv> ...]"""
import csv
import json
import sys

csv.field_size_limit(10 ** 9)
WANT = {"Kernel Name": "kernel", "gpu__time_duration.sum": "duration", "dram__bytes_read.sum": "dram_bytes_read",
        "dram__bytes_write.sum": "dram_bytes_write", "smsp__inst_executed.sum": "warp_instructions", "launch__registers_per_thread": "registers",
        "launch__grid_size": "grid", "launch__block_size": "block", "sm__warps_active.avg.pct_of_peak_sustained_active": "achieved_occupancy_pct",
        "sm__cycles_active.avg": "sm_active_cycles", "gpc__cycles_elapsed.max": "elapsed_cycles",
        "dram__throughput.avg.pct_of_peak_sustained_elapsed": "dram_pct_of_peak", "sm__inst_executed_pipe_fp64.sum": "fp64_pipe_instructions",
        "smsp__inst_executed.avg.per_cycle_active": "ipc_per_smsp"}
UNIT = {"Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9, "byte": 1.0, "us": 1e-6, "ms": 1e-3, "ns": 1e-9, "s": 1.0, "usecond": 1e-6, "msecond": 1e-3, "nsecond": 1e-9}
for path in sys.argv[1:]:
    rows = list(csv.reader(open(path)))
    hdr, units = rows[0], rows[1]
    for r in rows[2:]:
        out = {"file": path.split("/")[-1]}
        for i, h in enumerate(hdr):
            if h in WANT and i < len(r):
                v = r[i]
                try:
                    v = float(v.replace(",", ""))
                    if units[i] in UNIT and WANT[h] in ("duration", "dram_bytes_read", "dram_bytes_write"):
                        v *= UNIT[units[i]]
                except ValueError:
                    pass
                out[WANT[h]] = v
        if "duration" in out:
            out["duration_us"] = out.pop("duration") * 1e6
        print(json.dumps(out))
