#!/usr/bin/env python
"""Per-kernel share of ONE frame from an `ncu --metrics gpu__time_duration.sum --csv` launch list of bench.py
(cold-cache, serialised launch times: compare SHARES, not absolutes).  The frame = the launches between the last two
`vox_init` kernels.    python tools/launch_shares.py launches.csv [> shares.txt]"""
import collections
import csv
import re
import sys


def main(path):
    rows = list(csv.reader(open(path, newline="")))
    hi = [i for i, r in enumerate(rows) if "Kernel Name" in r][0]
    ix = {h: i for i, h in enumerate(rows[hi])}
    launches = []
    for r in rows[hi + 1:]:
        if len(r) <= ix["Metric Value"] or r[ix["Metric Name"]] != "gpu__time_duration.sum":
            continue
        v = float(r[ix["Metric Value"]].replace(",", ""))
        unit = r[ix["Metric Unit"]]
        us = v / 1e3 if unit in ("ns", "nsecond") else v * 1e3 if unit in ("ms", "msecond") else v
        launches.append((r[ix["Kernel Name"]], us))
    idx = [i for i, (n, _) in enumerate(launches) if "vox_init" in n]
    if len(idx) < 2:
        raise SystemExit("need at least two frames in the capture")
    frame = launches[idx[-2]:idx[-1]]
    agg = collections.OrderedDict()
    for n, t in frame:
        k = re.sub(r"<.*", "", n.replace("(anonymous namespace)::", "").replace("<unnamed>::", "").split("(")[0]).replace("void ", "").replace("p3d::", "")
        m = re.search(r"<\(int\)(\d+), \(int\)(\d+)", n)
        if m and ("conv_f16" in n):
            k += "<%s,%s..>" % (m.group(1), m.group(2))
        agg.setdefault(k, [0, 0.0])
        agg[k][0] += 1
        agg[k][1] += t
    tot = sum(v[1] for v in agg.values())
    print("# one frame = %d launches, %.1f us of serialised cold-cache kernel time (%s)" % (len(frame), tot, path))
    for k, v in sorted(agg.items(), key=lambda kv: -kv[1][1]):
        print("%-64s n %3d  %9.1f us  %5.1f%%" % (k[:64], v[0], v[1], 100 * v[1] / tot))


if __name__ == "__main__":
    main(sys.argv[1])
