"""Summarise an .ncu-rep (read here, no GPU needed) into profiles/<name>.summary.txt and,
with --traffic, profiles/roofline_traffic.json (DRAM bytes per launch of the dominant kernel).

    python tools/ncu_summary.py profiles/tiled_step.ncu-rep [--traffic]
"""
import csv
import io
import json
import os
import subprocess
import sys

KEYS = [
    "gpu__time_duration.sum", "dram__bytes_read.sum", "dram__bytes_write.sum",
    "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "lts__t_sector_hit_rate.pct",
    "l1tex__t_sector_hit_rate.pct", "lts__throughput.avg.pct_of_peak_sustained_elapsed",
    "l1tex__throughput.avg.pct_of_peak_sustained_elapsed",
    "l1tex__data_pipe_lsu_wavefronts.avg.pct_of_peak_sustained_elapsed",
    "sm__warps_active.avg.pct_of_peak_sustained_active", "launch__registers_per_thread",
    "launch__grid_size", "launch__block_size", "launch__shared_mem_per_block_dynamic",
    "launch__occupancy_limit_shared_mem", "launch__occupancy_limit_registers",
    "smsp__issue_active.avg.pct_of_peak_sustained_active", "smsp__inst_executed.sum",
    "sm__inst_executed_pipe_lsu.avg.pct_of_peak_sustained_active",
    "l1tex__t_sectors_pipe_lsu_mem_global_op_ld.sum", "lts__t_sectors_srcunit_tex_op_read.sum",
    "smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_short_scoreboard_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_wait_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_not_selected_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_math_pipe_throttle_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_barrier_per_issue_active.ratio",
]


def main():
    rep = sys.argv[1]
    raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True,
                         text=True).stdout
    rows = list(csv.reader(io.StringIO(raw)))
    head, units = rows[0], rows[1]
    out = ["# %s" % os.path.basename(rep)]
    launches = []
    for r in rows[2:]:
        name = r[head.index("Kernel Name")]
        out.append("\n## %s" % name[:150])
        rec = {}
        for k in KEYS:
            if k in head:
                i = head.index(k)
                out.append("%-85s %18s %s" % (k, r[i], units[i]))
                rec[k] = r[i]
        launches.append((name, rec))
    dst = rep.replace(".ncu-rep", ".summary.txt")
    open(dst, "w").write("\n".join(out) + "\n")
    print(dst)
    if "--traffic" in sys.argv:
        def to_bytes(v, key):
            u = units[head.index(key)].lower()
            scale = {"byte": 1, "kbyte": 1e3, "mbyte": 1e6, "gbyte": 1e9}[u]
            return float(v.replace(",", "")) * scale
        vals = [to_bytes(rec["dram__bytes_read.sum"], "dram__bytes_read.sum") +
                to_bytes(rec["dram__bytes_write.sum"], "dram__bytes_write.sum")
                for _, rec in launches]
        path = os.path.join(os.path.dirname(rep), "roofline_traffic.json")
        json.dump({"kernel": launches[0][0][:120], "source": os.path.basename(rep),
                   "dram_bytes_per_launch": sum(vals) / len(vals), "launches_captured": len(vals)},
                  open(path, "w"), indent=1)
        print(path)


if __name__ == "__main__":
    main()
