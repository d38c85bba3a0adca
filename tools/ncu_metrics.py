#!/usr/bin/env python
"""Extract the per-launch metrics the rooflines cite from an .ncu-rep capture (ncu --set full) into a small CSV:
duration, grid/block, registers, DRAM bytes read / written, L2 hit rate, tensor-pipe activity, issue activity.
    python tools/ncu_metrics.py x.ncu-rep > x_metrics.csv      (no GPU needed: ncu -i ... --page raw)
The first two rows are header and units (ncu's raw page)."""
import csv
import io
import subprocess
import sys

WANT = ["gpu__time_duration.sum", "launch__grid_size", "launch__block_size", "launch__registers_per_thread",
        "dram__bytes_read.sum", "dram__bytes_write.sum", "lts__t_sector_hit_rate.pct",
        "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active",
        "sm__inst_executed_pipe_tensor.sum", "smsp__issue_active.avg.pct_of_peak_sustained_active",
        "sm__warps_active.avg.pct_of_peak_sustained_active", "l1tex__throughput.avg.pct_of_peak_sustained_elapsed",
        "lts__throughput.avg.pct_of_peak_sustained_elapsed", "dram__throughput.avg.pct_of_peak_sustained_elapsed",
        "sm__throughput.avg.pct_of_peak_sustained_elapsed"]


def main(path):
    raw = subprocess.run(["ncu", "-i", path, "--page", "raw", "--csv"], capture_output=True, text=True, check=True).stdout
    rows = list(csv.reader(io.StringIO(raw)))
    hdr, units = rows[0], rows[1]
    ix = {h: i for i, h in enumerate(hdr)}
    cols = [c for c in WANT if c in ix]
    w = csv.writer(sys.stdout)
    w.writerow(["kernel"] + cols)
    w.writerow([""] + [units[ix[c]] for c in cols])
    for r in rows[2:]:
        name = r[ix["Kernel Name"]].replace("p3d::", "").replace("(anonymous namespace)::", "").replace("<unnamed>::", "")
        name = name[:name.find("(")] if "(" in name and not name.startswith("void") else name.replace("void ", "")
        w.writerow([name[:90]] + [r[ix[c]] for c in cols])


if __name__ == "__main__":
    main(sys.argv[1])
