"""Per-kernel totals of an ncu launch list (`--metrics gpu__time_duration.sum --csv`).

    python tools/launch_summary.py launches.csv "command that was profiled" > profiles/launches.summary.txt
"""
import collections
import csv
import os
import sys


def main():
    path = sys.argv[1]
    what = sys.argv[2] if len(sys.argv) > 2 else "?"
    rows = [r for r in csv.reader(open(path)) if len(r) > 10]
    hdr = rows[0]
    ki, vi = hdr.index("Kernel Name"), hdr.index("Metric Value")
    agg = collections.OrderedDict()
    for r in rows[1:]:
        try:
            v = float(r[vi].replace(",", ""))
        except ValueError:
            continue
        a = agg.setdefault(r[ki], [0, 0.0])
        a[0] += 1
        a[1] += v
    total = sum(t for _, t in agg.values())
    print("# ncu launch list of `%s` (%s)" % (what, os.path.basename(path)))
    print("# per-kernel totals: device time, launches, average, share of all GPU time in the run\n")
    for k, (c, t) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
        print("%9.3f ms %5d launches avg %9.1f us %5.1f%%  %s" % (t / 1e6, c, t / c / 1e3, 100 * t / total, k[:100]))


if __name__ == "__main__":
    main()
