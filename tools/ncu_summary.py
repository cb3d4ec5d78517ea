#!/usr/bin/env python3
"""Turn an .ncu-rep (read here, without a GPU) into the files kept under profiles/: the raw metric page as CSV, and - for the scan kernel - the
record of profiles/ncu_traffic_r02.json that bench.py reads for `roofline.traffic`.

    python tools/ncu_summary.py prof_scan_C3.ncu-rep profiles/ncu_k_substr_scan_r02.csv --traffic C3 400000000 "<command>"
    python tools/ncu_summary.py prof_zstd.ncu-rep profiles/ncu_zstd_r02.csv
"""
import csv
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KEY = ["gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum", "dram__throughput.avg.pct_of_peak_sustained_elapsed", "launch__registers_per_thread", "launch__grid_size",
       "launch__block_size", "launch__occupancy_limit_registers", "launch__occupancy_limit_shared_mem", "sm__warps_active.avg.pct_of_peak_sustained_active",
       "smsp__issue_active.avg.pct_of_peak_sustained_active", "smsp__inst_executed.sum", "sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active",
       "smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio", "smsp__average_warps_issue_stalled_short_scoreboard_per_issue_active.ratio",
       "smsp__average_warps_issue_stalled_barrier_per_issue_active.ratio", "smsp__average_warps_issue_stalled_wait_per_issue_active.ratio",
       "smsp__average_warps_issue_stalled_mio_throttle_per_issue_active.ratio", "smsp__average_warps_issue_stalled_lg_throttle_per_issue_active.ratio",
       "smsp__average_warps_issue_stalled_branch_resolving_per_issue_active.ratio", "smsp__average_warps_issue_stalled_not_selected_per_issue_active.ratio",
       "lts__t_sector_hit_rate.pct", "l1tex__t_sector_hit_rate.pct", "smsp__thread_inst_executed_per_inst_executed.ratio"]


def to_bytes(v, unit):
    return float(v) * {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9, "Tbyte": 1e12}[unit]


def main():
    rep, out = sys.argv[1], sys.argv[2]
    raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True, check=True).stdout
    open(out, "w").write(raw)
    rows = list(csv.reader(raw.splitlines()))
    hdr, units, launches = rows[0], rows[1], rows[2:]
    col = {h: i for i, h in enumerate(hdr)}
    for r in launches:
        print(r[col["Kernel Name"]][:60])
        for k in KEY:
            if k in col:
                print("   %-84s %s %s" % (k, r[col[k]], units[col[k]]))
    if "--traffic" in sys.argv:
        i = sys.argv.index("--traffic")
        workload, nrows, cmd = sys.argv[i + 1], int(sys.argv[i + 2]), sys.argv[i + 3]
        r = launches[0]
        rd = to_bytes(r[col["dram__bytes_read.sum"]], units[col["dram__bytes_read.sum"]])
        wr = to_bytes(r[col["dram__bytes_write.sum"]], units[col["dram__bytes_write.sum"]])
        path = os.path.join(ROOT, "profiles", "ncu_traffic_r02.json")
        recs = [x for x in json.load(open(path)) if not (x["workload"] == workload and int(x["rows"]) == nrows)] if os.path.exists(path) else []
        alg = int(sys.argv[i + 4]) if len(sys.argv) > i + 4 else None
        recs.append({"workload": workload, "rows": nrows, "kernel": r[col["Kernel Name"]].split("(")[0], "dram_bytes_read": int(rd), "dram_bytes_write": int(wr),
                     "dram_bytes_per_launch": int(rd + wr), "algorithmic_bytes_per_launch": alg, "ratio": round((rd + wr) / alg, 4) if alg else None,
                     "gpu_time_ms_under_ncu": float(r[col["gpu__time_duration.sum"]]),
                     "source": "%s (%s; dram__bytes_read.sum + dram__bytes_write.sum)" % (os.path.relpath(out, ROOT), cmd)})
        json.dump(recs, open(path, "w"), indent=1)


if __name__ == "__main__":
    main()
