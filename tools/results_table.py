#!/usr/bin/env python
"""Markdown table of bench JSON lines (files holding bench.py output).

    python tools/results_table.py bench_cfg2.json bench_cfg3.json ...
"""
import json
import sys

print("| file | config / mode | GPUs | images/s (device-resident) | e2e images/s (host in, host out) | + text lines | ms/step | conv roofline frac (TFLOP/s) | SM MHz (median) | CPU oracle images/s |")
print("|---|---|---|---|---|---|---|---|---|---|")
for f in sys.argv[1:]:
    for line in open(f):
        if not line.startswith("{"):
            continue
        d = json.loads(line)
        if d.get("impl") == "reference":
            print("| `%s` | reference arm (CPU oracle port, %d threads) | - | %.2f | - | - | %.0f | - | - | %.2f |" % (
                f.split("/")[-1], d["cpu_baseline"]["cores"], d["value"], d["ms_per_step"], d["value"]))
            continue
        r = d["roofline"]
        cfg = d["config"]
        print("| `%s` | %s, `%s` | %d | **%.0f** | %.0f | %s | %.2f | %.3f (%.0f) | %s | %s |" % (
            f.split("/")[-1], cfg.get("baseline_config", "").replace("BASELINE.json ", ""), cfg.get("mode"), d["n_gpus"], d["value"], d["e2e"]["value"],
            "%.0f" % d["e2e_text_lines"]["value"] if "e2e_text_lines" in d else ("(e2e is lines)" if "lines" in d["e2e"].get("api", "") else "-"),
            d["ms_per_step"], r["frac"], r["achieved"], (d.get("clocks") or {}).get("sm_mhz"),
            "%.2f" % d["cpu_baseline"]["value"] if "cpu_baseline" in d else "-"))
        for k, v in (d.get("alt_modes") or {}).items():
            print("| ↳ same process | `%s` | %d | %.0f | - | - | %.2f | %.3f (%.0f) | - | - |" % (
                k, d["n_gpus"], v["value"], v["ms_per_step"], v["conv_tflops"] / r["peak"], v["conv_tflops"]))
