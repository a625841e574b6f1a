#!/usr/bin/env python
"""Turns the CSV of `ncu --metrics gpu__time_duration.sum --clock-control none --csv --log-file X ...` into the
per-kernel table (shares of the step; absolute times under ncu are cold-cache and serialised)."""
import csv
import sys
from collections import defaultdict


def main(path, title):
    rows = []
    with open(path, newline="") as f:
        lines = [l for l in f if not l.startswith("==")]
    rd = csv.DictReader(lines)
    for r in rd:
        if r.get("Metric Name") != "gpu__time_duration.sum":
            continue
        val = float(r["Metric Value"].replace(",", ""))
        unit = r.get("Metric Unit", "ns")
        scale = {"ns": 1e-6, "us": 1e-3, "usecond": 1e-3, "nsecond": 1e-6, "ms": 1.0, "msecond": 1.0, "s": 1e3, "second": 1e3}.get(unit, 1e-6)
        rows.append((r["Kernel Name"], val * scale))
    tot = defaultdict(float)
    cnt = defaultdict(int)
    for k, ms in rows:
        name = k.split("(")[0]
        tot[name] += ms
        cnt[name] += 1
    total = sum(tot.values())
    print("# %s\n" % title)
    print("| kernel | launches | total ms | share |\n|---|---|---|---|")
    for k in sorted(tot, key=lambda k: -tot[k]):
        print("| %s | %d | %.2f | %.1f%% |" % (k, cnt[k], tot[k], 100 * tot[k] / total))


if __name__ == "__main__":
    main(sys.argv[1], sys.argv[2] if len(sys.argv) > 2 else "ncu launch list")
