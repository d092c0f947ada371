#!/usr/bin/env python
"""Summarises an `ncu --csv` launch list (metrics gpu__time_duration.sum and, when captured, dram__bytes_read.sum /
dram__bytes_write.sum): per kernel count, mean / min / max duration and DRAM bytes per launch, plus the totals of ONE
build (centre_bounds_kernel .. the last build kernel before the next build or the first traversal).

    python scripts/summarize_launches.py launches.csv [--traffic traffic.json --key build_soup_1000000]
"""
import argparse
import collections
import csv
import json
import re

UNIT = {"ns": 1e-3, "us": 1.0, "usecond": 1.0, "ms": 1e3, "msecond": 1e3, "s": 1e6, "nsecond": 1e-3, "second": 1e6,
        "byte": 1.0, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}
BUILD = ("centre_bounds_kernel", "morton_kernel", "rs_", "hierarchy_", "treelet_kernel", "compact_", "wide_collapse", "wide_init")


def short(name):
    name = re.sub(r"\(.*", "", name)
    name = re.sub(r"^void ", "", name)
    name = name.replace("bvhb200::<unnamed>::", "").replace("bvhb200::", "")
    return name[:90]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("csv")
    ap.add_argument("--traffic")
    ap.add_argument("--key")
    a = ap.parse_args()
    lines = [l for l in open(a.csv) if not l.startswith("==")]
    launches = collections.OrderedDict()               # id -> {name, metrics}
    for row in csv.DictReader(lines):
        lid = row["ID"]
        rec = launches.setdefault(lid, {"name": short(row["Kernel Name"]), "m": {}})
        try:
            rec["m"][row["Metric Name"]] = float(row["Metric Value"].replace(",", "")) * UNIT.get(row["Metric Unit"], 1.0)
        except ValueError:
            pass
    agg = collections.OrderedDict()
    for rec in launches.values():
        agg.setdefault(rec["name"], []).append(rec["m"])
    print(f"{'kernel':92s} {'n':>4s} {'mean us':>9s} {'min':>8s} {'max':>8s} {'dram rd MB':>10s} {'dram wr MB':>10s}")
    for name, ms in agg.items():
        t = [m.get("gpu__time_duration.sum", 0.0) for m in ms]
        rd = [m.get("dram__bytes_read.sum", 0.0) / 1e6 for m in ms]
        wr = [m.get("dram__bytes_write.sum", 0.0) / 1e6 for m in ms]
        print(f"{name:92s} {len(ms):4d} {sum(t) / len(t):9.1f} {min(t):8.1f} {max(t):8.1f} {sum(rd) / len(rd):10.2f} {sum(wr) / len(wr):10.2f}")
    # one build = from the LAST centre_bounds_kernel launch to the last consecutive build kernel after it
    recs = list(launches.values())
    starts = [i for i, r in enumerate(recs) if r["name"].startswith("centre_bounds_kernel")]
    if starts:
        i = starts[-1]
        t = rd = wr = 0.0
        names = []
        while i < len(recs) and any(recs[i]["name"].startswith(b) for b in BUILD):
            m = recs[i]["m"]
            t += m.get("gpu__time_duration.sum", 0.0); rd += m.get("dram__bytes_read.sum", 0.0); wr += m.get("dram__bytes_write.sum", 0.0)
            names.append(recs[i]["name"].split("<")[0])
            i += 1
        print(f"\none build: {len(names)} launches, {t:.1f} us of kernel time (serialised, cold caches), DRAM {rd / 1e6:.1f} MB read + {wr / 1e6:.1f} MB written")
        if a.traffic and a.key and (rd + wr) > 0:
            try:
                db = json.load(open(a.traffic))
            except Exception:
                db = {}
            db[a.key] = rd + wr
            json.dump(db, open(a.traffic, "w"), indent=1, sort_keys=True)
            print(f"{a.traffic}: {a.key} = {rd + wr:.0f}")


if __name__ == "__main__":
    main()
