#!/usr/bin/env python3
"""Summarise an `ncu --csv` launch list (one row per launch and metric) into a markdown table.

    python tools/launch_summary.py launches_c3.csv > launches_c3.md
"""
import collections
import csv
import sys


def summarise(path):
    rows = [r for r in csv.reader(l for l in open(path) if l.startswith('"'))]
    ix = {h: i for i, h in enumerate(rows[0])}
    per = collections.OrderedDict()
    for r in rows[1:]:
        key = (r[ix["ID"]], r[ix["Kernel Name"]])
        per.setdefault(key, {})[r[ix["Metric Name"]]] = float(r[ix["Metric Value"]].replace(",", ""))
    agg = collections.OrderedDict()
    for (_, k), m in per.items():
        a = agg.setdefault(k, [0, 0.0, 0.0, 0.0])
        a[0] += 1
        a[1] += m.get("gpu__time_duration.sum", 0.0)
        a[2] += m.get("dram__bytes_read.sum", 0.0) + m.get("dram__bytes_write.sum", 0.0)
        a[3] += m.get("smsp__inst_executed.sum", 0.0)
    return agg


def main():
    for path in sys.argv[1:]:
        agg = summarise(path)
        print(f"### {path}\n")
        print("| kernel | launches | avg µs | DRAM MB / launch | warp-instr (M) / launch |")
        print("|---|---|---|---|---|")
        for k, a in agg.items():
            name = k.replace("<unnamed>::", "").replace("void ", "")
            name = name.split("(")[0]
            print(f"| `{name}` | {a[0]} | {a[1] / a[0] / 1000:.1f} | {a[2] / a[0] / 1e6:.2f} | {a[3] / a[0] / 1e6:.2f} |")
        print()


if __name__ == "__main__":
    main()
