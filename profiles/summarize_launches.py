"""Summarise an `ncu --metrics gpu__time_duration.sum --csv` launch list into per-kernel totals and shares.

    python profiles/summarize_launches.py step0_launches.csv > launches_summary.md
"""
import csv
import re
import sys
from collections import defaultdict


def main(path):
    rows = []
    with open(path, newline="") as f:
        lines = [l for l in f if not l.startswith("==")]
    rd = csv.DictReader(lines)
    for r in rd:
        if r.get("Metric Name") != "gpu__time_duration.sum":
            continue
        try:
            v = float(r["Metric Value"].replace(",", ""))
        except ValueError:
            continue
        unit = r.get("Metric Unit", "ns")
        scale = {"ns": 1e-6, "us": 1e-3, "ms": 1.0, "s": 1e3, "nsecond": 1e-6, "usecond": 1e-3, "msecond": 1.0, "second": 1e3}.get(unit, 1e-6)
        name = re.sub(r"\(.*", "", r["Kernel Name"]).strip()
        name = re.sub(r"^void\s+", "", name)
        rows.append((name, v * scale))
    tot = defaultdict(float)
    cnt = defaultdict(int)
    for n, ms in rows:
        tot[n] += ms
        cnt[n] += 1
    total = sum(tot.values())
    print(f"# ncu launch list summary: {path}\n")
    print(f"{len(rows)} launches, {total:.1f} ms of kernel time (cold-cache, serialised: compare SHARES, not absolutes)\n")
    print("| kernel | launches | total ms | share | avg us |")
    print("|---|---:|---:|---:|---:|")
    for n in sorted(tot, key=tot.get, reverse=True)[:25]:
        print(f"| `{n[:90]}` | {cnt[n]} | {tot[n]:.2f} | {100 * tot[n] / total:.1f}% | {1000 * tot[n] / cnt[n]:.1f} |")


if __name__ == "__main__":
    main(sys.argv[1])
