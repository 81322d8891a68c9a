#!/usr/bin/env python
"""DRAM traffic of the conv launches of one step from an `ncu --set full` raw CSV export (ncu -i x.ncu-rep --page raw --csv),
written as the JSON bench.py reads for roofline.traffic.  The file is stamped with the SHA-256 of the kernel sources it was
captured from (bench.py refuses it when the sources have changed since).

    python tools/ncu_traffic.py ncu_raw_f16f8.csv --config 2 --mode f16f8 --batch 32 > profiles/conv_traffic_cfg2_f16f8.json
"""
import argparse
import csv
import json
import os
import re
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import sources_sha256  # noqa: E402


def to_bytes(v, unit):
    f = float(v.replace(",", ""))
    return f * {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}[unit]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("csv")
    ap.add_argument("--config", type=int, default=2)
    ap.add_argument("--mode", default="f16f8")
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--sha-file", default="", help="sources_sha256.txt written on the box by tools/capture_profiles.sh (default: hash the local tree)")
    a = ap.parse_args()
    rows = list(csv.reader(open(a.csv)))
    i0 = next(i for i, r in enumerate(rows) if "Kernel Name" in r)
    hdr, units, data = rows[i0], rows[i0 + 1], [r for r in rows[i0 + 2:] if len(r) >= len(rows[i0])]
    kn, rd, wr, tm = (hdr.index(k) for k in ("Kernel Name", "dram__bytes_read.sum", "dram__bytes_write.sum", "gpu__time_duration.sum"))
    launches = []
    for r in data:
        m = re.search(r"conv_tc_kernel<([^>]*)>", r[kn])
        if not m:
            continue
        tpl = [int(x) for x in re.findall(r"\)(\d+)", m.group(1))] or [int(x) for x in re.findall(r"\d+", m.group(1))]
        if len(tpl) >= 3 and tpl[2] != 9:
            continue                                   # the 1x1 GEMMs are not part of the conv roofline
        launches.append({"template": m.group(1).replace("(int)", ""), "dram_read": to_bytes(r[rd], units[rd]),
                         "dram_write": to_bytes(r[wr], units[wr]), "time": r[tm] + " " + units[tm]})
    out = {"config": a.config, "mode": a.mode, "batch": a.batch, "launches": len(launches),
           "dram_bytes_per_step": sum(l["dram_read"] + l["dram_write"] for l in launches),
           "per_launch": launches, "sources_sha256": open(a.sha_file).read().strip() if a.sha_file else sources_sha256(),
           "how": "ncu --set full --clock-control none -k regex:conv_tc, one step of tools/ncu_step.py; dram__bytes_read.sum + dram__bytes_write.sum"}
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
